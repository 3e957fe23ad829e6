"""GPU: MiDaS 3.0 (DPT-Hybrid) on the depth engine -- the forward against tests/dpt_hybrid_oracle.py (fp32), a batch
against single forwards, each BiT kernel (stem conv, GroupNorm statistics and apply, max-pool, SAME im2col) against
float64 through vd3d_bit_kernel, the family's argument checks, and the image / video drivers of render_depth with a
hybrid model written by save_pretrained."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import dpt_hybrid_oracle as OH

pytestmark = pytest.mark.gpu

PROC128 = dict(size=(128, 128), resample=3, mean=(0.5,) * 3, std=(0.5,) * 3)


def _depth_u8(d):
    d = d.astype(np.float32)
    return ((d - d.min()) / (d.max() - d.min() + np.float32(1e-6)) * 255).astype(np.uint8)


def _engine(sd, cfg, processor=None):
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine(cfg, family="dpt-hybrid", processor=processor)
    e.load_state_dict(sd)
    return e


@pytest.fixture(scope="module")
def default_model():
    return OH.random_model()


def _forward_err(sd, cfg, seed, processor=None):
    import torch
    e = _engine(sd, cfg, processor)
    S = cfg["image_size"]
    assert (e.image_h, e.image_w) == (S, S)
    px = torch.randn(3, S, S, generator=torch.Generator().manual_seed(seed))
    with torch.no_grad():
        ref = OH.forward(sd, cfg, px).numpy()
    out = e.forward(px.numpy())
    e.close()
    assert np.isfinite(out).all()
    err = float(np.abs(out - ref).max() / (ref.max() - ref.min()))
    lsb = int(np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int)).max())
    return err, lsb


def test_forward_matches_oracle_default(default_model):
    sd, cfg = default_model
    err, lsb = _forward_err(sd, cfg, 3)
    print("MiDaS 3.0 (norm3 gamma x 0.25) B=1 max-abs error / range", err, "u8 LSB", lsb)
    # the f16 emulation of the engine's storage (tests/test_oracle_dpt_hybrid.py) alone gives 1.03e-3
    assert err <= 1.5e-3 and lsb <= 1, (err, lsb)


def test_forward_matches_oracle_stress():
    sd, cfg = OH.random_model(gamma3=1.0)
    err, lsb = _forward_err(sd, cfg, 3)
    print("MiDaS 3.0 stress (HF init, gamma 1) B=1 max-abs error / range", err, "u8 LSB", lsb)
    assert err <= 5e-3 and lsb <= 2, (err, lsb)


def test_forward_matches_oracle_small():
    sd, cfg = OH.random_model(small=True)
    err, lsb = _forward_err(sd, cfg, 4, PROC128)
    print("DPT-Hybrid small ViT at 128 max-abs error / range", err, "u8 LSB", lsb)
    assert err <= 1.5e-3 and lsb <= 1, (err, lsb)


def test_batch_of_four_equals_single_forwards(default_model):
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = default_model
    e = _engine(sd, cfg)
    frames = [synth_frame(i, 640, 360, k)[0] for i, k in ((1, "natural"), (2, "noise"), (3, "smooth"), (4, "natural"))]
    batch = e.infer_batch(frames)
    for f, (d32, d8) in zip(frames, batch):
        s32, s8 = e.infer(f)
        assert np.array_equal(d32, s32) and np.array_equal(d8, s8)
    e.close()


# ---- each BiT kernel against float64, through vd3d_bit_kernel ----
EPS32 = 2.0 ** -24


@pytest.fixture(scope="module")
def keng():
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine(OH.SMALL | dict(patch=16, ln_eps=1e-12), family="dpt-hybrid", processor=PROC128)
    yield e
    e.close()


def test_stem_conv_against_float64(keng):
    import torch
    from visiondepth3d_b200.depth_weights import standardize_weight
    rng = np.random.default_rng(0)
    H, W = 70, 46  # edge columns and rows on both sides of the 2 / 3 padding
    px = rng.standard_normal((3, H, W)).astype(np.float32)
    w = np.asarray(standardize_weight(torch.from_numpy(rng.standard_normal((64, 3, 7, 7)))), np.float32)
    out = keng.bit_kernel(0, (H, W), {"t.in": px, "t.w": w.reshape(64, 147)}, (H // 2 * (W // 2), 64), np.float32)
    xp = torch.from_numpy(px.astype(np.float64))[None]
    ref = OH.conv_same(xp, torch.from_numpy(w.astype(np.float64)), 2, ws=False)[0].permute(1, 2, 0).reshape(-1, 64)
    absum = OH.conv_same(xp.abs(), torch.from_numpy(np.abs(w).astype(np.float64)), 2, ws=False)[0]
    absum = absum.permute(1, 2, 0).reshape(-1, 64).numpy()
    tol = 147 * EPS32 * absum + 1e-30  # fp32 fmaf chain of at most 147 terms
    d = np.abs(out - ref.numpy())
    print("stem conv max error / bound", float((d / tol).max()))
    assert (d <= tol).all()


def _gn64(y, g, b):
    """GroupNorm(32) in float64 on [rows, C]: (normalised, mean, var) per group."""
    rows, C = y.shape
    yg = y.reshape(rows, 32, C // 32)
    m = yg.mean(axis=(0, 2))
    v = ((yg - m[None, :, None]) ** 2).mean(axis=(0, 2))
    return ((yg - m[None, :, None]) / np.sqrt(v[None, :, None] + 1e-5)).reshape(rows, C) * g + b, m, v


@pytest.mark.parametrize("rows,C,flags", [(96 * 96, 64, 1), (48 * 48, 256, 1), (24 * 24, 1024, 4 | 1),
                                          (48 * 48, 512, 2 | 1), (1000, 128, 0), (37, 1024, 2 | 4 | 1)])
def test_groupnorm_against_float64(keng, rows, C, flags):
    """Statistics and apply, every variant; group 5 has a mean of ~100 x its standard deviation, so that a
    sum-of-squares variance would cancel."""
    rng = np.random.default_rng(rows + C + flags)
    cpg = C // 32

    def src():
        y = (rng.standard_normal((rows, C)) * rng.uniform(0.2, 3.0, C)).astype(np.float32)
        y[:, 5 * cpg:6 * cpg] = (300.0 + 3.0 * rng.standard_normal((rows, cpg))).astype(np.float32)
        return y
    y, g, b = src(), rng.uniform(0.5, 1.5, C).astype(np.float32), rng.standard_normal(C).astype(np.float32)
    t = {"t.in": y, "t.g": g, "t.b": b}
    want, m, v = _gn64(y.astype(np.float64), g, b)
    if flags & 2:
        y2, g2, b2 = src(), rng.uniform(0.5, 1.5, C).astype(np.float32), rng.standard_normal(C).astype(np.float32)
        t.update({"t.in2": y2, "t.g2": g2, "t.b2": b2})
        want = want + _gn64(y2.astype(np.float64), g2, b2)[0]
    if flags & 4:
        res = rng.standard_normal((rows, C)).astype(np.float16)
        t["t.res"] = res
        want = want + res.astype(np.float64)
    if flags & 1:
        want = np.maximum(want, 0)
    out = keng.bit_kernel(1, (rows, C, flags), t, (rows, C), np.float16).astype(np.float64)
    # partials: the chunks' (mean, M2), merged in float64, give the float64 statistics to fp32 accuracy
    chunk = -(-rows // 128)
    nch = -(-rows // chunk)
    part = keng.get_buffer("t.part", (nch, 32, 2), np.float32).astype(np.float64)
    n = np.array([(min(rows, (k + 1) * chunk) - k * chunk) * cpg for k in range(nch)], np.float64)[:, None]
    N = rows * cpg
    pm = (part[..., 0] * n).sum(0) / N
    pM2 = (part[..., 1] + n * (part[..., 0] - pm[None]) ** 2).sum(0)
    sd = np.sqrt(v)
    assert (np.abs(pm - m) <= 64 * EPS32 * (np.abs(m) + sd)).all()
    assert (np.abs(pM2 / N - v) <= 64 * EPS32 * v + 1e-30).all()
    # apply: fp32 statistics (mean off by a few ulp of |mean| + sd) carried through the affine, then f16 rounding
    grp = np.arange(C) // cpg
    tol = 2.0 ** -11 * np.abs(want) + 2.0 ** -24
    for gam, mm, vv, yy in ((g, m, v, y),) + (((t["t.g2"],) + _gn64(t["t.in2"].astype(np.float64), g, b)[1:]
                                                + (t["t.in2"],),) if flags & 2 else ()):
        z = (yy.astype(np.float64) - mm[grp]) / np.sqrt(vv[grp] + 1e-5)
        rel = 64 * EPS32 * (np.abs(mm[grp]) + np.sqrt(vv[grp])) / np.sqrt(vv[grp] + 1e-5)
        tol = tol + np.abs(gam) * (rel * (1 + np.abs(z)) + 8 * EPS32 * np.abs(z)) + 8 * EPS32 * np.abs(want)
    d = np.abs(out - want)
    print("GroupNorm", rows, C, flags, "max error / bound", float((d / tol).max()))
    assert (d <= tol).all()


@pytest.mark.parametrize("H,W", [(192, 192), (34, 50)])
def test_maxpool_edges_equal_float64(keng, H, W):
    """The last output row and column take the 0 before / 1 after padding with pad value 0: on negative inputs the
    edge outputs are 0, inside they are the window maximum."""
    import torch
    import torch.nn.functional as F
    rng = np.random.default_rng(H)
    x = rng.standard_normal((H, W, 64)).astype(np.float16)
    x[-1] = -np.abs(x[-1])
    x[:, -1] = -np.abs(x[:, -1])
    out = keng.bit_kernel(2, (H, W, 64), {"t.in": x}, (H // 2, W // 2, 64), np.float16)
    t = torch.from_numpy(x.astype(np.float64)).permute(2, 0, 1)[None]
    ref = F.max_pool2d(F.pad(t, (0, 1, 0, 1), value=0.0), 3, 2)[0].permute(1, 2, 0).numpy()
    assert np.array_equal(out.astype(np.float64), ref)
    assert (out[-1] >= 0).all() and (out[:, -1] >= 0).all()


@pytest.mark.parametrize("k,pb", [(3, 0), (1, 0)])
def test_same_im2col_equals_float64(keng, k, pb):
    """The stride-2 3x3 SAME rows (0 before, 1 after) and the stride-2 1x1 subsample, as a conv on them equals
    torch's SAME conv of the map: checked bit for bit against the unfolded float64 map."""
    import torch
    import torch.nn.functional as F
    H, W, Cc = 24, 18, 128
    x = np.random.default_rng(k).standard_normal((H, W, Cc)).astype(np.float16)
    out = keng.bit_kernel(3, (H, W, Cc, k, pb), {"t.in": x}, (H // 2 * (W // 2), k * k * Cc), np.float16)
    t = torch.from_numpy(x.astype(np.float64)).permute(2, 0, 1)[None]
    if k == 3:
        t = F.pad(t, (0, 1, 0, 1))
    cols = F.unfold(t, k, stride=2)[0]  # [C * k * k, L], rows c-major
    ref = cols.reshape(Cc, k * k, -1).permute(2, 1, 0).reshape(-1, k * k * Cc).numpy()
    assert np.array_equal(out.astype(np.float64), ref)


def test_create_ex_arguments():
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200.depth_engine import DepthConfig, DepthConfigEx, _bind
    lib = _lib.load()
    _bind(lib)
    ctx = _lib.default_context(0)

    def make(size=(384, 384), patch=16, neck=(256, 512, 768, 768), head=0):
        dc = DepthConfig(768, 12, 12, (C.c_int32 * 4)(3, 6, 9, 12), (C.c_int32 * 4)(*neck), 256, *size)
        dx = DepthConfigEx(dc, 2, patch, 1e-12, 3, (C.c_float * 3)(0.5, 0.5, 0.5), (C.c_float * 3)(0.5, 0.5, 0.5),
                           head, 1.0 if head == 0 else 10.0)
        h = C.c_void_p()
        rc = lib.vd3d_depth_create_ex(C.byref(dx), lib.vd3d_stream(ctx.h), C.byref(h))
        if rc == 0:
            lib.vd3d_depth_destroy(h)
        return rc
    assert make() == 0 and make((128, 128)) == 0
    assert make(head=1) == -2
    assert make(patch=14, size=(392, 392)) == -2
    assert make(size=(384, 512)) == -2
    assert make(size=(400, 400)) == -2
    assert make(neck=(128, 512, 768, 768)) == -2


# ---- the drivers with a random-init hybrid written by save_pretrained ----
@pytest.fixture(scope="module")
def midas(default_model, tmp_path_factory):
    from visiondepth3d_b200 import render_depth as RD
    sd, _ = default_model
    root = tmp_path_factory.mktemp("w")
    model = OH.hf_model(sd)
    folder = root / "weights" / "Intel_dpt-hybrid-midas"
    model.save_pretrained(str(folder))
    old = RD.local_model_dir
    RD.local_model_dir = str(root / "weights")
    RD.update_pipeline("MiDaS 3.0", None, None, None).join()
    yield RD, model, folder
    RD.local_model_dir = old
    RD.USE_TILED_DEPTH = False


class Var:
    def __init__(self, v):
        self.v = v

    def get(self):
        return self.v


def test_update_pipeline_publishes_pipe(midas):
    RD, _, folder = midas
    assert {"model.safetensors", "config.json"} <= set(os.listdir(folder))
    assert RD._arch == "dpt-hybrid-midas" and RD.pipe is not None and RD.pipe_type == "hf"


def test_process_image_matches_transformers_pipeline(midas, tmp_path):
    """A 1920x1080 image through process_image against transformers' pipeline("depth-estimation") on the same weights
    on the CPU, then the min-max u8 of convert_depth_to_grayscale: the path the reference runs."""
    import torch
    from PIL import Image
    from transformers import pipeline
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    RD, model, _ = midas
    from visiondepth3d_b200.synth import synth_frame
    fr, _ = synth_frame(5, 1920, 1080, "natural")
    img = Image.fromarray(fr[..., ::-1].copy())
    src = tmp_path / "in.png"
    img.save(src)
    RD.process_image(str(src), Var("default"), Var(False), Var(str(tmp_path / "o")), Var("Original"), None, None, None,
                     None)
    got = np.array(Image.open(tmp_path / "o" / "in_depth.png"))
    assert got.shape == (1080, 1920)
    pipe = pipeline("depth-estimation", model=model, image_processor=DPTImageProcessor(), device="cpu")
    with torch.no_grad():
        d = pipe(img)["predicted_depth"]
    want = RD.convert_depth_to_grayscale(d)
    if want.shape != got.shape:
        want = RD.resize_cubic_u8(want, 1920, 1080)
    diff = np.abs(got.astype(int) - want.astype(int))
    print("process_image vs transformers pipeline: max LSB", int(diff.max()), "share > 0", float((diff > 0).mean()))
    assert diff.max() <= 1


def test_folder_driver_writes_source_sizes(midas, tmp_path):
    import torch
    from PIL import Image
    RD, model, _ = midas
    src = tmp_path / "in"
    src.mkdir()
    rng = np.random.default_rng(2)
    sizes = [(640, 360), (333, 500), (384, 384)]
    for k, (w, h) in enumerate(sizes):
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(src / f"im{k}.png")
    RD.process_images_in_folder(str(src), Var("8"), Var(str(tmp_path / "o")), Var("Original"), None, None, None,
                                Var(False))
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    proc = DPTImageProcessor()
    for k, (w, h) in enumerate(sizes):
        got = np.array(Image.open(tmp_path / "o" / f"im{k}_depth.png"))
        assert got.shape == (h, w)
        img = Image.open(src / f"im{k}.png").convert("RGB")
        pv = proc(images=img, return_tensors="pt")["pixel_values"]
        with torch.no_grad():
            d = model(pixel_values=pv).predicted_depth
            d = torch.nn.functional.interpolate(d[None], size=(h, w), mode="bicubic", align_corners=False)[0, 0]
        want = RD.convert_depth_to_grayscale(d)
        assert np.abs(got.astype(int) - want.astype(int)).max() <= 1, k


def test_depth_frames_equal_per_frame_inference(midas):
    from tests import letterbox_oracle as L
    from tests.test_letterbox_cpu import _Cap
    RD, _, _ = midas
    frames = L.track_frames()[:6]
    got = list(RD.iter_depth_frames(_Cap(frames, 2), 320, 180, False, None, batch_size=4))
    assert len(got) == len(frames)
    for f, g in zip(frames, got):
        want = RD.resize_cubic_u8(RD.depth_u8_from_frame(f), 320, 180)
        assert np.abs(g.astype(int) - want.astype(int)).max() <= 1


def test_tiled_depth_is_refused_before_files_exist(midas, tmp_path):
    RD, _, _ = midas
    RD.USE_TILED_DEPTH = True
    try:
        with pytest.raises(ValueError, match="USE_TILED_DEPTH"):
            RD.depth_video_from_video(str(tmp_path / "missing.mp4"), str(tmp_path / "o.mkv"))
        with pytest.raises(ValueError, match="USE_TILED_DEPTH"):
            RD.process_images_in_folder(str(tmp_path), 2, str(tmp_path / "out"), "Original", None, None, None, False)
        assert os.listdir(tmp_path) == []
    finally:
        RD.USE_TILED_DEPTH = False


def test_clip_depth_refuses_hybrid(default_model):
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R3
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = default_model
    e = _engine(sd, cfg)
    w, h = 320, 180
    rp = R3.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, "Half-SBS", 16 / 9, 0.0, 10.0, 9, True, True)
    frames = [synth_frame(i, w, h, "smooth")[0] for i in range(2)]
    outs = [np.empty((h, w, 3), np.uint8) for _ in frames]
    fp = (C.c_void_p * 2)(*[f.ctypes.data for f in frames])
    op = (C.c_void_p * 2)(*[o.ctypes.data for o in outs])
    ctx = e.ctx
    assert ctx.lib.vd3d_render_clip_depth(ctx.h, e.h, 2, fp, h, w, C.byref(rp), op, _lib.MEM_HOST) == -3  # UNSUPPORTED
    e.close()
