"""GPU: the RRDBNet upscalers (RealESRGAN_x4plus, BSRGAN x4 / x2) on the wgmma convolutions.  The forward against the
f16 restatement (tests/rrdb_oracle.py; the margins are recorded by tests/test_rrdb_cpu.py::test_f16_budget), one
dense block and one RRDB against float64 on the engine's own stored inputs, run_esrgan's chain for both network scales
and both model-name quirks, the tiled host path, the merged_pipeline driver, and one 3840x1080 x4 forward."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle.sr import preprocess_esr
from tests import rrdb_oracle as RO
from visiondepth3d_b200 import _lib
from visiondepth3d_b200 import merged_pipeline as MP
from visiondepth3d_b200 import render_3d as R
from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu

_ENGINES = {}


def _engine(nb, scale):
    if (nb, scale) not in _ENGINES:
        e = MP.SrEngine(MP.random_rrdb_state_dict(nb, scale, seed=0))
        e.lib.vd3d_depth_get_buffer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
        e.lib.vd3d_depth_get_buffer.restype = C.c_int
        _ENGINES[(nb, scale)] = e
    return _ENGINES[(nb, scale)]


def _buf(e, name, shape, dtype):
    out = np.empty(shape, dtype)
    e.check(e.lib.vd3d_depth_get_buffer(e.h, name.encode(), out.ctypes.data, out.nbytes))
    return out


@pytest.mark.parametrize("scale,nb,w,h", [(4, 23, 64, 48), (4, 23, 67, 45), (2, 23, 64, 48), (2, 23, 67, 45),
                                          (4, 1, 64, 48), (2, 1, 67, 45), (4, 2, 160, 90), (2, 2, 160, 90)])
def test_forward_matches_f16_oracle(scale, nb, w, h):
    """u8 output: at most 1 LSB off rrdb_forward_f16 on at most 5 % of the bytes; float output of conv_last within
    2e-3 (the CPU test measures up to 2.5 % and 1e-3 between two accumulation orders of the same f16 graph; an H100
    gave 2.8-3.8 % and 1.1e-3 at nb = 23, 0.4-0.6 % and 1.4e-4 at nb <= 2).  Against
    fp32 rrdb_forward only loosely (<= 6 LSB, mean <= 0.5): f16 storage through ~350 convs, the cost the CPU test
    records for the restatement itself."""
    e = _engine(nb, scale)
    sd = MP.random_rrdb_state_dict(nb, scale, seed=0)
    fr = synth_frame(3, w, h, "natural")[0]
    got = e.upscale(fr)
    assert got.shape == (scale * h, scale * w, 3)
    x = torch.from_numpy(preprocess_esr(fr))
    ref = RO.rrdb_forward_f16(sd, x)
    d = np.abs(got.astype(int) - RO.postprocess_esr(ref.numpy()))
    print(f"x{scale} nb={nb} {w}x{h}: vs f16 oracle max {d.max()} differing {(d > 0).mean():.4f}", end="; ")
    assert d.max() <= 1 and (d > 0).mean() <= 0.05, (d.max(), (d > 0).mean())
    raw = _buf(e, "rr.u0" if scale == 4 else "rr.u1", (scale * h, scale * w, 32), np.float32)[..., :3]
    fd = np.abs(raw - ref[0].permute(1, 2, 0).numpy()).max()
    d32 = np.abs(got.astype(int) - RO.postprocess_esr(RO.rrdb_forward(sd, x).numpy()))
    print(f"float max {fd:.2e}; vs fp32 oracle max {d32.max()} mean {d32.mean():.3f}")
    assert fd <= 2e-3
    assert d32.max() <= 6 and d32.mean() <= 0.5


def _conv64(x, w, b):
    """float64 3x3 conv (pad 1) of NHWC x with torch weights [Cout, Cin, 3, 3] (f16-rounded as the engine stores
    them); also the conv of |x| with |w| plus |b| (the scale of the fp32 accumulation error)."""
    import torch.nn.functional as F
    xt = torch.from_numpy(x.astype(np.float64)).permute(2, 0, 1)[None]
    wt = torch.from_numpy(w.astype(np.float16).astype(np.float64))
    bt = torch.from_numpy(b.astype(np.float64))
    y = F.conv2d(xt, wt, bt, padding=1)[0].permute(1, 2, 0).numpy()
    s = F.conv2d(xt.abs(), wt.abs(), bt.abs(), padding=1)[0].permute(1, 2, 0).numpy()
    return y, s


def _check(got, exp, s, what):
    """One f16 store (half an ulp, 2^-11 relative, 2^-25 absolute below the normal range) after fp32 accumulation
    (4e-5 of the sum of |terms|: K up to 2880 in groups of 256)."""
    err = np.abs(got.astype(np.float64) - exp)
    bound = np.abs(exp) * 2.0 ** -11 + 2.0 ** -25 + 4e-5 * s
    print(f"{what}: max err/bound {(err / bound).max():.3f}", end="; ")
    assert (err <= bound).all(), (what, float((err / bound).max()))


def test_dense_block_and_rrdb_on_the_engine_buffers():
    """nb = 1, x4, 64x48.  After the forward: rr.feat holds the RRDB input, rr.d1 the second dense block (its input in
    channels 0..63 and x1..x4 in the growth slices), rr.d2 the third, and rr.d0's channels 0..63 the RRDB output.  Each
    conv of the second dense block, its output (x + 0.2 x5 in rr.d2) and the RRDB output (x + 0.2 (y + 0.2 x5)) are
    checked against float64 on the engine's own f16 inputs; the padding channels stay zero."""
    e = _engine(1, 4)
    sd = RO._t(MP.random_rrdb_state_dict(1, 4, seed=0))
    w, h = 64, 48
    e.upscale(synth_frame(5, w, h, "natural")[0])
    feat = _buf(e, "rr.feat", (h, w, 64), np.float16)
    d = [_buf(e, f"rr.d{i}", (h, w, 320), np.float16) for i in range(3)]
    cols = lambda k: list(range(64)) + [64 * (s + 1) + c for s in range(k - 1) for c in range(32)]
    for i in range(3):
        for k in range(1, 5):
            assert not d[i][..., 64 * k + 32:64 * (k + 1)].any(), (i, k)
    X = d[1]
    for k in range(1, 6):
        wk, bk = sd[f"body.0.rdb2.conv{k}.weight"].numpy(), sd[f"body.0.rdb2.conv{k}.bias"].numpy()
        y, s = _conv64(X[..., cols(k)], wk, bk)
        if k < 5:
            exp = np.where(y > 0, y, 0.2 * y)
            _check(X[..., 64 * k:64 * k + 32], exp, s, f"rdb2.conv{k}")
        else:
            _check(d[2][..., :64], X[..., :64].astype(np.float64) + 0.2 * y, 0.2 * s, "rdb2 output")
    w5, b5 = sd["body.0.rdb3.conv5.weight"].numpy(), sd["body.0.rdb3.conv5.bias"].numpy()
    y, s = _conv64(d[2][..., cols(5)], w5, b5)
    exp = feat.astype(np.float64) + 0.2 * (d[2][..., :64].astype(np.float64) + 0.2 * y)
    _check(d[0][..., :64], exp, 0.04 * s, "RRDB output")
    print()


_CASES = [dict(), dict(input_res_pct=50), dict(input_res_pct=75), dict(input_res_pct=150),
          dict(target_size=(200, 120)), dict(input_res_pct=50, target_size=(97, 61)), dict(blend_mode="LOW"),
          dict(blend_mode="MEDIUM", input_res_pct=75), dict(blend_mode="HIGH", input_res_pct=50)]


@pytest.mark.parametrize("scale", [4, 2])
@pytest.mark.parametrize("model_name", ["RealESRGAN_x4_fp16", "BSRGANx2_fp16"])
def test_run_esrgan_chain(scale, model_name):
    """vd3d_sr_upscale with an RRDBNet engine against (a) the per-stage composition on the device (SrEngine.upscale,
    then the INTER_CUBIC resizes one by one: bit-identical) and (b) the oracle chain (cv2 restatements of the resizes
    and addWeighted) fed with the engine's network output: within 2 LSB, at most 1e-3 of the bytes beyond 1 LSB, like
    the SRVGGNetCompact chain tests."""
    e = _engine(2, scale)
    MP.esrgan_session = e
    try:
        for i, (w, h) in enumerate(((96, 64), (91, 57))):
            fr = synth_frame(7 + i, w, h, "natural")[0]
            for kw in _CASES:
                got = MP.run_esrgan(fr, model_name=model_name, **kw)
                pct, tgt = kw.get("input_res_pct", 100), kw.get("target_size")
                small = fr
                if pct != 100:
                    nw, nh = int(w * pct / 100), int(h * pct / 100)
                    small = R.resize_area(fr, nw, nh) if pct < 100 else MP._resize_cubic(fr, nw, nh)
                up = e.upscale(small)
                q = 2 if "x2" in model_name.lower() else 4
                if up.shape[:2] != (q * small.shape[0], q * small.shape[1]):
                    up = MP._resize_cubic(up, q * small.shape[1], q * small.shape[0])
                up = MP._resize_cubic(up, w, h)
                if tgt:
                    up = MP._resize_cubic(up, *tgt)
                ref_dev = MP.blend_images(fr, up, kw.get("blend_mode", "OFF"))
                assert got.shape == ref_dev.shape and np.array_equal(got, ref_dev), (scale, model_name, kw)
                ref = RO.run_esrgan(None, fr, kw.get("blend_mode", "OFF"), pct, model_name, tgt, network=e.upscale)
                dd = np.abs(got.astype(int) - ref)
                assert dd.max() <= 2 and (dd > 1).mean() <= 1e-3, (scale, model_name, kw, dd.max(), (dd > 1).mean())
    finally:
        MP.esrgan_session = None


@pytest.mark.parametrize("scale", [4, 2])
def test_run_esrgan_tiled_host_path(scale):
    """run_esrgan(tile=...) keeps its host path on an RRDBNet engine: tiles through SrEngine.upscale (net_scale x the
    tile), cropped into an input-size canvas as the reference does, then the INTER_CUBIC chain."""
    e = _engine(2, scale)
    MP.esrgan_session = e
    try:
        fr = synth_frame(9, 80, 56, "natural")[0]
        got = MP.run_esrgan(fr, "OFF", 100, "BSRGANx2_fp16", tile=32, tile_pad=8)
        canvas = MP._esrgan_tiled(fr, 32, 8)
        ref = RO.run_esrgan(None, fr, "OFF", 100, "BSRGANx2_fp16", network=lambda f: canvas)
        assert got.shape == fr.shape
        dd = np.abs(got.astype(int) - ref)
        assert dd.max() <= 2 and (dd > 1).mean() <= 1e-3
        # the canvas holds the network output: its first tile is the top-left of the first padded crop's upscale
        assert np.array_equal(canvas[:32, :32], e.upscale(fr[:40, :40])[:32, :32]) and canvas.std() > 1
    finally:
        MP.esrgan_session = None


def _write_folder(tmp_path, w, h, n):
    import cv2
    d = tmp_path / "frames"
    d.mkdir()
    for i in range(n):
        cv2.imwrite(str(d / f"frame_{i + 1:04d}.png"), synth_frame(20 + i, w, h, "natural")[0])
    return d


@pytest.mark.parametrize("fname,scale", [("BSRGANx2_fp16", 2), ("RealESRGANx4_fp16", 4), ("BSRGANx4_fp16", 4)])
def test_driver_serves_rrdb_weights(tmp_path, fname, scale):
    """iter_merged_frames with <stem>.pth next to the GUI's ONNX path (old-ESRGAN naming for BSRGAN, basicsr with
    params_ema for Real-ESRGAN) yields what per-frame run_esrgan (default model name: quirk scale 4) gives."""
    import cv2
    d = _write_folder(tmp_path, 64, 48, 5)
    naming = "esrgan" if fname.startswith("BSRGAN") else "basicsr"
    sd = MP.random_rrdb_state_dict(1, scale, seed=0, naming=naming)
    t = {k: torch.from_numpy(v) for k, v in sd.items()}
    torch.save({"params_ema": t} if naming == "basicsr" else t, str(tmp_path / f"{fname}.pth"))
    srcs = [cv2.imread(str(d / f)) for f in sorted(os.listdir(d))]
    try:
        for kw in (dict(width=128, height=96), dict(width=64, height=48, blend_mode="MEDIUM", input_res_pct=75)):
            s = dict(frames_folder=str(d), output_file=str(tmp_path / "o.mp4"), codec="libx264", fps=24,
                     fps_multiplier=2, enable_rife=False, enable_upscale=True, blend_mode="OFF", input_res_pct=100,
                     model_path=str(tmp_path / f"{fname}.onnx"))
            s.update(kw)
            got = list(MP.iter_merged_frames(s))
            assert MP.esrgan_session.net_scale == scale
            ref = [MP.run_esrgan(f, s["blend_mode"], s["input_res_pct"], target_size=(s["width"], s["height"]))
                   for f in srcs]
            assert len(got) == len(ref) == 5
            assert all(np.array_equal(a, b) for a, b in zip(got, ref)), kw
    finally:
        MP.esrgan_session = None


def test_forward_3840x1080_x4_memory():
    """One nb = 23 x4 forward of a Full-SBS-shaped 3840x1080 frame (config 4's SR input) completes; the device memory
    the engine took is printed."""
    free0 = torch.cuda.mem_get_info()[0]
    e = MP.SrEngine(MP.random_rrdb_state_dict(23, 4, seed=0))
    fr = np.concatenate([synth_frame(21 + i, 1920, 1080, "natural")[0] for i in range(2)], axis=1)
    try:
        out = e.upscale(fr)
        free1 = torch.cuda.mem_get_info()[0]
        print(f"3840x1080 x4 RRDBNet forward: device memory taken {(free0 - free1) / 2 ** 30:.2f} GiB")
        assert out.shape == (4320, 15360, 3)
        assert out[::97, ::89].std() > 10
    finally:
        e.close()
