"""GPU: run_esrgan's untiled chain as one device call (vd3d_sr_upscale, with k_sr_tail_cubic resampling the x4 output
straight from the last conv) against the explicit per-stage composition it replaces, and the merged_pipeline driver
(iter_merged_frames / start_merged_pipeline) against per-frame run_esrgan."""
import ctypes as C
import os

import numpy as np
import pytest

from visiondepth3d_b200 import _lib
from visiondepth3d_b200 import merged_pipeline as MP
from visiondepth3d_b200 import render_3d as R
from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = MP.SrEngine(MP.random_srvgg_state_dict(4, seed=1))
    e.lib.vd3d_depth_launch_count.argtypes = [C.c_void_p]
    e.lib.vd3d_depth_launch_count.restype = C.c_uint64
    e.lib.vd3d_depth_get_buffer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
    e.lib.vd3d_depth_get_buffer.restype = C.c_int
    yield e
    e.close()


def old_chain(eng, frame, blend_mode="OFF", pct=100, scale=4, target=None):
    """The untiled run_esrgan as it was composed before vd3d_sr_upscale: SrEngine.upscale -> _resize_cubic(x scale) ->
    _resize_cubic(original) -> [_resize_cubic(target)] -> blend_images, one host round trip per stage."""
    original = frame
    if pct != 100:
        h, w = frame.shape[:2]
        nw, nh = int(w * pct / 100), int(h * pct / 100)
        frame = R.resize_area(frame, nw, nh) if pct < 100 else MP._resize_cubic(frame, nw, nh)
    up = eng.upscale(frame)
    up = MP._resize_cubic(up, frame.shape[1] * scale, frame.shape[0] * scale)
    up = MP._resize_cubic(up, original.shape[1], original.shape[0])
    if target:
        up = MP._resize_cubic(up, target[0], target[1])
    return MP.blend_images(original, up, mode=blend_mode)


def new_chain(eng, frames, blend_mode="OFF", pct=100, scale=4, target=None, mem=_lib.MEM_HOST):
    p = MP.upscale_params(blend_mode, pct, "RealESR_x2" if scale == 2 else "RealESR_Gx4_fp16", target)
    h, w = frames[0].shape[:2]
    size = tuple(target) if target else (w, h)
    if mem == _lib.MEM_HOST:
        return eng.upscale_chain(frames, p, size)
    import torch
    fd = [torch.from_numpy(f).cuda() for f in frames]
    od = [torch.empty((size[1], size[0], 3), dtype=torch.uint8, device="cuda") for _ in frames]
    torch.cuda.synchronize()
    eng.upscale_ptrs([t.data_ptr() for t in fd], h, w, p, [t.data_ptr() for t in od], _lib.MEM_DEVICE)
    return [t.cpu().numpy() for t in od]


def _frames(w, h, n=1, seed=3):
    return [synth_frame(seed + i, w, h, "natural")[0] for i in range(n)]


@pytest.mark.parametrize("w,h", [(160, 90), (157, 93)])
@pytest.mark.parametrize("pct", [25, 50, 75, 100, 150])
@pytest.mark.parametrize("scale", [4, 2])
@pytest.mark.parametrize("tgt", [None, "larger", "smaller"])
def test_sr_upscale_bit_identical_to_old_chain(eng, w, h, pct, scale, tgt):
    target = {None: None, "larger": (2 * w + 3, 2 * h + 1), "smaller": (w // 2 + 1, h // 2 + 3)}[tgt]
    fr = _frames(w, h)[0]
    ref = old_chain(eng, fr, "OFF", pct, scale, target)
    got = new_chain(eng, [fr], "OFF", pct, scale, target)[0]
    assert got.shape == ref.shape and np.array_equal(got, ref), (w, h, pct, scale, target)


@pytest.mark.parametrize("mode", ["LOW", "MEDIUM", "HIGH", "low", "Sharp"])
@pytest.mark.parametrize("pct,scale", [(100, 4), (50, 4), (75, 2)])
def test_sr_upscale_blend_modes(eng, mode, pct, scale):
    fr = _frames(157, 93)[0]
    for target in (None, (157, 93)):  # a target of the frame's own size is the identity resize
        ref = old_chain(eng, fr, mode, pct, scale, target)
        got = new_chain(eng, [fr], mode, pct, scale, target)[0]
        assert np.array_equal(got, ref), (mode, pct, scale, target)


@pytest.mark.parametrize("mem", [_lib.MEM_HOST, _lib.MEM_DEVICE])
def test_sr_upscale_batches_and_memory_kinds(eng, mem):
    frs = _frames(160, 90, n=5, seed=11)
    for kw in (dict(), dict(pct=50, target=(320, 180)), dict(blend_mode="MEDIUM", pct=75), dict(scale=2, pct=100)):
        ref = [old_chain(eng, f, kw.get("blend_mode", "OFF"), kw.get("pct", 100), kw.get("scale", 4), kw.get("target"))
               for f in frs]
        got = new_chain(eng, frs, mem=mem, **kw)
        one = [new_chain(eng, [f], mem=mem, **kw)[0] for f in frs]
        for a, b, c in zip(ref, got, one):
            assert np.array_equal(a, b) and np.array_equal(a, c), kw


def test_sr_upscale_sbs_frame_shape(eng):
    """A 3840x1080 Full-SBS-shaped frame (config 4's SR input), to a 7680x2160 target and to its own size."""
    fr = np.concatenate(_frames(1920, 1080, n=2, seed=21), axis=1)
    for target in ((7680, 2160), None):
        assert np.array_equal(new_chain(eng, [fr], target=target)[0], old_chain(eng, fr, target=target)), target


def test_sr_upscale_refuses_blend_of_two_sizes(eng):
    fr = _frames(160, 90)[0]
    out = np.empty((180, 320, 3), np.uint8)
    p = MP.upscale_params("MEDIUM", 100, target_size=(320, 180))
    fp = (C.c_void_p * 1)(fr.ctypes.data)
    op = (C.c_void_p * 1)(out.ctypes.data)
    rc = eng.lib.vd3d_sr_upscale(eng.ctx.h, eng.h, 1, fp, 90, 160, eng.num_conv, C.byref(p), op, _lib.MEM_HOST)
    assert rc == -2  # VD3D_ERR_ARG
    with pytest.raises(AssertionError):
        MP.esrgan_session, saved = eng, MP.esrgan_session
        try:
            MP.run_esrgan(fr, "MEDIUM", target_size=(320, 180))
        finally:
            MP.esrgan_session = saved


def test_no_x4_buffer_at_pct_100():
    e = MP.SrEngine(MP.random_srvgg_state_dict(2, seed=4))
    w, h = 160, 90
    fr = _frames(w, h)[0]
    for target, mode in (((320, 180), "OFF"), (None, "HIGH")):
        e.upscale_chain([fr], MP.upscale_params(mode, 100, target_size=target), target or (w, h))
    buf = np.empty(16 * w * h * 3, np.uint8)
    get = e.lib.vd3d_depth_get_buffer
    get.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
    assert get(e.h, b"sr.outu8", buf.ctypes.data, 1) != 0          # the x4 image of vd3d_sr_forward never existed
    assert get(e.h, b"up.0", buf.ctypes.data, w * h * 3) == 0        # the only intermediate: one frame-size image
    assert get(e.h, b"up.0", buf.ctypes.data, 16 * w * h * 3) != 0
    assert get(e.h, b"up.in", buf.ctypes.data, 1) != 0
    e.close()


def test_launch_count_per_frame_is_fixed(eng):
    lc = lambda: eng.ctx.launches + int(eng.lib.vd3d_depth_launch_count(eng.h))  # noqa: E731
    fr = _frames(160, 90)[0]
    l0 = lc()
    eng.upscale(fr)
    net = lc() - l0 - 1  # vd3d_sr_forward = k_sr_in + the convs + k_sr_out
    # pct 50 / scale 2 on 160x90: the tail lands on 160x90 itself, so the second cubic resize is skipped
    cases = [(dict(), 1), (dict(pct=50), 2), (dict(pct=50, scale=2), 2), (dict(pct=75, scale=2), 3),
             (dict(target=(320, 180)), 2),
             (dict(blend_mode="LOW"), 2), (dict(pct=150, scale=2, target=(80, 45)), 4)]
    for kw, extra in cases:
        frs = _frames(160, 90, n=3)
        l0 = lc()
        new_chain(eng, frs, **kw)
        assert lc() - l0 == 3 * (net + extra), kw


def _write_folder(tmp_path, w, h, n):
    import cv2
    d = tmp_path / "frames"
    d.mkdir()
    for i in range(n):
        cv2.imwrite(str(d / f"frame_{i + 8}.png"), synth_frame(i, w, h, "natural")[0])
    (d / "notes.txt").write_text("not a frame")
    (d / "broken_3.png").write_bytes(b"\x89PNG not really")
    return d


def _settings(d, tmp_path, **kw):
    s = dict(frames_folder=str(d), output_file=str(tmp_path / "out.mp4"), codec="libx264", width=160, height=90,
             fps=24, fps_multiplier=2, enable_rife=True, enable_upscale=True, blend_mode="OFF", input_res_pct=100,
             model_path=str(tmp_path / "RealESR_Gx4_fp16.onnx"))
    s.update(kw)
    return s


def test_driver_equals_per_frame_run_esrgan(tmp_path, monkeypatch):
    import cv2
    import shutil
    import torch
    d = _write_folder(tmp_path, 160, 90, 6)
    sd = MP.random_srvgg_state_dict(4, seed=9)
    torch.save({"params_ema": {k: torch.from_numpy(v) for k, v in sd.items()}}, str(tmp_path / "RealESR_Gx4_fp16.pth"))
    files = MP.natural_sort([str(d / f) for f in os.listdir(d) if f.lower().endswith((".jpg", ".jpeg", ".png"))])
    srcs = [cv2.imread(f) for f in files]
    srcs = [s for s in srcs if s is not None]
    for kw in (dict(), dict(input_res_pct=50, width=320, height=180), dict(blend_mode="MEDIUM"),
               dict(enable_upscale=False, width=96, height=54), dict(enable_upscale=False, width=200, height=120)):
        s = _settings(d, tmp_path, **kw)
        got = list(MP.iter_merged_frames(s))
        if s["enable_upscale"]:
            ref = [MP.run_esrgan(f, s["blend_mode"], s["input_res_pct"], target_size=(s["width"], s["height"]))
                   for f in srcs]
        else:
            ref = [R.resize_area(f, s["width"], s["height"]) if f.shape[1] > s["width"]
                   else MP._resize_cubic(f, s["width"], s["height"]) for f in srcs]
        assert len(got) == len(ref) == 6, kw
        assert all(np.array_equal(a, b) for a, b in zip(got, ref)), kw
    # the whole driver with its writer thread: the recorded writer gets the same frames, fps x multiplier (RIFE on)
    rec = {}

    class FakeProc:
        def __init__(self):
            self.frames = []

            class In:
                def write(_s, b):
                    self.frames.append(bytes(b))

                def close(_s):
                    pass
            self.stdin = In()

        def wait(self):
            return 0

    def fake_writer(path, w, h, fps, codec):
        rec.update(args=(path, w, h, fps, codec), proc=FakeProc())
        return rec["proc"]

    monkeypatch.setattr(MP, "start_ffmpeg_writer", fake_writer)
    monkeypatch.setattr(shutil, "which", lambda name: "/usr/bin/ffmpeg")
    s = _settings(d, tmp_path)
    MP.start_merged_pipeline(s, None, None)
    assert rec["args"] == (s["output_file"], 160, 90, 48, "libx264")
    ref = [MP.run_esrgan(f, target_size=(160, 90)).tobytes() for f in srcs]
    assert rec["proc"].frames == ref
    MP.cancel_flag.set()
    try:
        assert len(list(MP.iter_merged_frames(s))) == 1  # the first frame is written before the loop checks the flag
    finally:
        MP.cancel_flag.clear()
    MP.esrgan_session = None


def test_config4_composition_matches_host_path():
    """Depth + Full-SBS (preserve_original_aspect) on the device, then vd3d_sr_upscale on the device frames, equals the
    host-buffer vd3d_render_clip_depth followed by run_esrgan per frame."""
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200.depth_engine import DepthEngine, processed_size
    from visiondepth3d_b200.depth_weights import hf_config
    w, h, n = 320, 180, 3
    ctx = _lib.default_context(0)
    torch.manual_seed(0)
    sd = DepthAnythingForDepthEstimation(hf_config("vits")).eval().state_dict()
    ih, iw = processed_size(w, h)
    deng = DepthEngine("vits", ih, iw, ctx=ctx)
    deng.load_state_dict(sd)
    rp = R.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, "Full-SBS", 16 / 9, 0.0, preserve_original_aspect=True)
    oshape = R.output_shape(rp, R.plan_sizes(w, h, rp))
    frames = [synth_frame(i, w, h, "natural")[0] for i in range(n)]
    sr = MP.load_esrgan(MP.random_srvgg_state_dict(4, seed=2))
    target = (2 * oshape[1], 2 * oshape[0])
    # host path
    ctx.reset()
    outs = [np.empty(oshape, np.uint8) for _ in range(n)]
    ctx.check(ctx.lib.vd3d_render_clip_depth(ctx.h, deng.h, n, (C.c_void_p * n)(*[f.ctypes.data for f in frames]), h, w,
                                             C.byref(rp), (C.c_void_p * n)(*[o.ctypes.data for o in outs]),
                                             _lib.MEM_HOST))
    ref = [MP.run_esrgan(o, target_size=target) for o in outs]
    # device path
    ctx.reset()
    fd = [torch.from_numpy(f).cuda() for f in frames]
    od = [torch.empty(oshape, dtype=torch.uint8, device="cuda") for _ in range(n)]
    ud = [torch.empty((target[1], target[0], 3), dtype=torch.uint8, device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    ctx.check(ctx.lib.vd3d_render_clip_depth(ctx.h, deng.h, n, (C.c_void_p * n)(*[t.data_ptr() for t in fd]), h, w,
                                             C.byref(rp), (C.c_void_p * n)(*[t.data_ptr() for t in od]),
                                             _lib.MEM_DEVICE))
    sr.upscale_ptrs([t.data_ptr() for t in od], oshape[0], oshape[1], MP.upscale_params(target_size=target),
                    [t.data_ptr() for t in ud], _lib.MEM_DEVICE)
    for a, b in zip(ud, ref):
        assert np.array_equal(a.cpu().numpy(), b)
    ctx.check(ctx.lib.vd3d_release_depth(ctx.h, deng.h))
    MP.esrgan_session = None


def test_driver_against_merged_oracle(tmp_path):
    """The drop-in driver against the numpy / cv2 restatement (tests/merged_oracle.py on oracle/sr.py): the loader's
    INTER_AREA exact, its INTER_CUBIC <= 1 LSB, the upscaled frames within the network tolerance of
    test_run_esrgan_chain_matches_oracle."""
    import torch
    from oracle import sr as S
    from tests import merged_oracle as MO
    from tests.util import u8_diff
    d = _write_folder(tmp_path, 128, 72, 4)
    sd = S.srvgg_state_dict(num_conv=4, seed=6)
    torch.save({"params_ema": sd}, str(tmp_path / "RealESR_Gx4_fp16.pth"))
    cases = [(dict(enable_upscale=False, width=96, height=54), 0), (dict(enable_upscale=False, width=200, height=120), 1),
             (dict(input_res_pct=50, width=256, height=144), 2), (dict(blend_mode="MEDIUM", width=128, height=72), 2)]
    for kw, tol in cases:
        s = _settings(d, tmp_path, **kw)
        got = list(MP.iter_merged_frames(s))
        ref = MO.merged_frames(s, sd if s["enable_upscale"] else None)
        assert len(got) == len(ref) == 4, kw
        for a, b in zip(got, ref):
            mx, f0, f1 = u8_diff(a, b)
            assert a.shape == b.shape and mx <= tol, (kw, mx)
            if tol == 1:
                assert f0 < 0.002, (kw, f0)
            if tol == 2:
                assert f1 <= 1e-3 and f0 <= 0.06, (kw, f0, f1)
    s = _settings(d, tmp_path, model_path=str(tmp_path / "missing" / "x.onnx"))  # no model: source frames
    assert all(np.array_equal(a, b) for a, b in zip(MP.iter_merged_frames(s), MO.merged_frames(s, None)))
    MP.esrgan_session = None


@pytest.mark.parametrize("name", ["merged_area_rife.npz", "merged_cubic_rife.npz", "merged_sr_pct50_x2target.npz",
                                  "merged_sr_medium.npz", "merged_sr_nomodel.npz"])
def test_driver_against_reference_fixtures(name, tmp_path, golden_dir, monkeypatch):
    """The drop-in driver against the frames and writer arguments the unmodified reference driver recorded: the
    loader's INTER_AREA and the no-model source frames exact, its INTER_CUBIC <= 1 LSB / < 0.2 %, the upscaled frames
    within the network tolerance of test_run_esrgan_chain_matches_oracle."""
    import shutil
    import torch
    from oracle import sr as S
    from tests.test_merged_pipeline_cpu import fixture_settings
    from tests.merged_oracle import MERGED_SR
    from tests.util import u8_diff
    g = np.load(os.path.join(golden_dir, name))
    s, has_model = fixture_settings(name, tmp_path)
    if has_model:
        os.makedirs(os.path.dirname(s["model_path"]), exist_ok=True)
        torch.save({"params_ema": S.srvgg_state_dict(**MERGED_SR)}, s["model_path"][:-len(".onnx")] + ".pth")
    rec = {"frames": []}

    class Proc:
        class stdin:  # noqa: N801
            write = staticmethod(lambda b: rec["frames"].append(bytes(b)))
            close = staticmethod(lambda: None)

        def wait(self):
            return 0

    def writer(path, w, h, fps, codec):
        rec["args"] = (w, h, fps, codec)
        return Proc()

    monkeypatch.setattr(MP, "start_ffmpeg_writer", writer)
    monkeypatch.setattr(shutil, "which", lambda n: "/usr/bin/ffmpeg")
    try:
        got = list(MP.iter_merged_frames(s))
        MP.start_merged_pipeline(s, None, None)
    finally:
        MP.esrgan_session = None
    assert rec["args"] == (*[int(v) for v in g["writer_size"]], float(g["writer_fps"]), str(g["codec"]))
    ref = g["frames"]
    assert len(got) == len(rec["frames"]) == len(ref)
    for a, raw, b in zip(got, rec["frames"], ref):
        assert a.shape == b.shape and raw == a.tobytes(), name
        mx, f0, f1 = u8_diff(a, b)
        if not s["enable_upscale"] and s["width"] < 128 or not has_model:
            assert mx == 0, (name, mx)
        elif not s["enable_upscale"]:
            assert mx <= 1 and f0 < 0.002, (name, mx, f0)
        else:
            assert mx <= 2 and f1 <= 1e-3 and f0 <= 0.06, (name, mx, f0, f1)


def test_run_esrgan_raises_on_caller_sizes_and_falls_back_on_engine_refusal(eng):
    """Empty sizes raise like the reference's cv2.resize calls; only what the engine refuses (a network input below
    8 x 8) returns the source frame, as a failed network run does in the reference."""
    fr = _frames(160, 90)[0]
    saved, MP.esrgan_session = MP.esrgan_session, eng
    try:
        for kw in (dict(target_size=(0, 0)), dict(target_size=(-4, 90)), dict(input_res_pct=0)):
            with pytest.raises(ValueError):
                MP.run_esrgan(fr, **kw)
        assert MP.run_esrgan(fr, input_res_pct=3) is fr   # 4 x 2 network input
    finally:
        MP.esrgan_session = saved
