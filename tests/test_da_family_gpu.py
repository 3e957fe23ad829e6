"""GPU: the Depth-Anything family beyond V2 on the depth engine -- Depth Anything V1 (the last four layers as taps),
Distill-Any-Depth and the V2 metric models (max_depth * sigmoid head): the forward against the fp32 oracle, the
metric EPI_HEAD against float64 on the engine's own head input, and every driver (batches, still images, the video
pass, tiled depth, the joined render with its engine clone and graphs) carrying the model's spec."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

from tests import da_family_oracle as DO
from tests import depth_kernel_refs as R
from visiondepth3d_b200 import depth_weights as DW

pytestmark = pytest.mark.gpu

V1 = {k: DW.da_spec(k, taps=DW.V1_TAPS[k]) for k in ("vits", "vitb", "vitl")}
METRIC_S = DW.da_spec("vits", head="metric", max_depth=20.0)


def _depth_u8(d):
    d = d.astype(np.float32)
    return ((d - d.min()) / (d.max() - d.min() + np.float32(1e-6)) * 255).astype(np.uint8)


def _engine(sd, spec, h=518, w=924):
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine(spec, h, w)
    e.load_state_dict(sd)
    return e


# max-abs error / depth range of the forward: test_depth_gpu.test_forward_matches_oracle's 1e-3 for S and B.  ViT-L
# gets DPT-Large's 1.5e-3 (test_dpt_gpu): V1-Large, which taps the last four of its 24 layers, measured 1.08e-3 on an
# H100, the f16 rounding of every layer's operands reaching all four taps
GATE = {"vits": 1e-3, "vitb": 1e-3, "vitl": 1.5e-3}


def _gate(out, ref, what, gate):
    """<= gate of the range, <= 1 LSB after min-max u8"""
    scale = float(ref.max() - ref.min())
    assert scale > 1e-2 * float(np.abs(ref).max()), "degenerate test model: output range cancels"
    err = np.abs(out - ref).max() / scale
    print(f"[da-family] {what}: max-abs error / range {err:.2e}")
    assert err <= gate, (what, err)
    assert np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int)).max() <= 1, what


@pytest.mark.parametrize("name", ["vits", "vitb", "vitl"])
def test_v1_forward_matches_oracle(name):
    sd, spec = DO.random_model(V1[name])
    e = _engine(sd, spec)
    px = torch.randn(3, 518, 924, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        ref = DO.forward(sd, spec, px).numpy()
    _gate(e.forward(px.numpy()), ref, f"V1 {name}", GATE[name])
    e.close()


@pytest.fixture(scope="module")
def metric_large():
    """V2-Metric-Large at 518 x 924: the scaled head (calibrated on the test input) and the oracle's pre-sigmoid
    value, which does not depend on max_depth."""
    px = torch.randn(3, 518, 924, generator=torch.Generator().manual_seed(4))
    sd, _ = DO.random_model("vitl")  # non-negative conv3 weights, zero bias
    with torch.no_grad():
        s = DO.pre_activation(sd, DO.head_input(sd, DW.da_spec("vitl"), px))
    # the scale and bias random_model gives a metric head calibrated on this input, applied to the oracle's value
    a = 8.0 / float(s.max() - s.min())
    b = -4.0 - a * float(s.min())
    sd["head.conv3.weight"] = sd["head.conv3.weight"] * a
    sd["head.conv3.bias"] = torch.tensor([b])
    return sd, px, s * a + b


@pytest.mark.parametrize("max_depth", [20.0, 80.0])
def test_metric_forward_matches_oracle(metric_large, max_depth):
    sd, px, pre = metric_large
    assert float(pre.min()) < -3.5 and float(pre.max()) > 3.5  # both tails and the middle of the sigmoid
    spec = DW.da_spec("vitl", head="metric", max_depth=max_depth)
    ref = (torch.sigmoid(pre) * max_depth).numpy()
    e = _engine(sd, spec)
    out = e.forward(px.numpy())
    assert 0.0 <= out.min() and out.max() <= max_depth
    # The gate applies to the pre-sigmoid value, whose error the sigmoid passes on scaled by its slope there.  In
    # the middle (slope 1/4) that is twice the error relative to the depth range of a linear head: the output range
    # over a [-4, 4] span is 0.96 max_depth, but max_depth / 4 * 8 of pre-activation range maps onto it.
    pre64 = pre.double().numpy()
    slope = 1.0 / (2.0 + np.exp(pre64) + np.exp(-pre64))
    delta = GATE["vitl"] * float(pre64.max() - pre64.min())
    tol = 1.02 * max_depth * slope * delta + 8 * R.F32_EPS * max_depth
    ratio = float((np.abs(out - ref) / tol).max())
    print(f"[da-family] V2-Metric-Large max_depth {max_depth}: error / range {np.abs(out - ref).max() / np.ptp(ref):.2e}, "
          f"observed / bound {ratio:.3f}")
    assert ratio <= 1.0
    assert np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int)).max() <= 1
    e.close()


def test_metric_head_epilogue_against_float64():
    """max_depth * sigmoid(sum_c relu(conv3x3(h1u) + b2)[c] * w3[c] + b3) in float64 from the f16 head input the
    engine stored: the pre-activation bound of test_depth_kernels_gpu.test_neck_and_head, propagated through the
    sigmoid's slope <= 1/4, plus the fp32 expf / division / scale."""
    h, w = 140, 252
    px = torch.randn(3, h, w, generator=torch.Generator().manual_seed(9))
    sd, spec = DO.random_model(METRIC_S, calib=px)
    e = _engine(sd, spec, h, w)
    e.forward(px.numpy())
    P = DW.prepare(sd, spec, h, w)
    F2 = (spec["fusion"] // 2 + 63) // 64 * 64
    h1u = e.get_buffer("h1u", (h, w, F2), np.float16)
    depth = e.get_buffer("depth", (h, w), np.float32)
    t = np.maximum(R.conv3x3(h1u, P["h.c2.w"], P["h.c2.b"]), 0)
    w3, b3 = R.f64(P["h.c3.w"]), float(P["h.c3.b"][0])
    s = t @ w3 + b3
    md = spec["max_depth"]
    ref = md / (1.0 + np.exp(-s))
    acc = 2 * min(9 * F2, 256) / 16 + math.ceil(9 * F2 / 256) + 4  # ACC of test_depth_kernels_gpu, in units of 2^-24
    tol_s = (acc * R.F32_EPS * R.conv3x3_abs(h1u, P["h.c2.w"], P["h.c2.b"])) @ np.abs(w3) \
        + 40 * R.F32_EPS * (t @ np.abs(w3) + abs(b3))
    tol = 0.25 * md * tol_s + 8 * R.F32_EPS * np.abs(ref) + 1e-30
    ratio = float((np.abs(R.f64(depth) - ref) / tol).max())
    print(f"[da-family] metric EPI_HEAD: observed / bound = {ratio:.3f}")
    assert ratio <= 1.0
    assert s.min() < -3.0 and s.max() > 3.0, "the fixture no longer exercises both tails of the sigmoid"
    e.close()


def test_create_ex_arguments():
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200.depth_engine import DepthConfig, DepthConfigEx, _bind
    lib = _lib.load()
    _bind(lib)
    ctx = _lib.default_context(0)
    c = DW.CONFIGS["vits"]

    def create(family=0, head=0, max_depth=1.0, patch=14, h=70, w=98):
        dc = DepthConfig(c["hidden"], c["layers"], c["heads"], (C.c_int32 * 4)(*c["taps"]), (C.c_int32 * 4)(*c["neck"]),
                         c["fusion"], h, w)
        dx = DepthConfigEx(dc, family, patch, 1e-6, 3, (C.c_float * 3)(0.5, 0.5, 0.5), (C.c_float * 3)(0.5, 0.5, 0.5),
                           head, max_depth)
        p = C.c_void_p()
        rc = lib.vd3d_depth_create_ex(C.byref(dx), lib.vd3d_stream(ctx.h), C.byref(p))
        if rc == 0:
            lib.vd3d_depth_destroy(p)
        return rc
    assert create() == 0 and create(head=1, max_depth=20.0) == 0
    for bad in (dict(head=2), dict(head=-1), dict(head=1, max_depth=0.0), dict(head=1, max_depth=-20.0),
                dict(head=1, max_depth=float("nan")), dict(head=1, max_depth=float("inf")), dict(max_depth=0.0),
                dict(family=1, patch=16, h=384, w=384, head=1, max_depth=20.0)):
        assert create(**bad) == -2, bad  # VD3D_ERR_ARG


# ---------------------------------------------------------------------------------------------------------------------
# drivers, for a V1 model and a metric model: every engine built from the loaded weights carries the spec
# ---------------------------------------------------------------------------------------------------------------------
SPECS = {"v1": V1["vits"], "metric": METRIC_S}


@pytest.fixture(scope="module", params=list(SPECS))
def model(request):
    return DO.random_model(SPECS[request.param], seed=5)


@pytest.fixture
def loaded(model):
    from visiondepth3d_b200 import render_depth as RD
    sd, spec = model
    if RD._state_dict is not sd:
        _, meta = RD.load_depth_model(spec, sd, 320, 180)
        assert meta["config"] == spec and RD._spec == spec
    yield RD, sd, spec
    RD.USE_TILED_DEPTH, RD.TILE_SIZE, RD.TILE_PAD = False, 512, 32


def test_engines_carry_the_spec(loaded):
    """Engines for every processed size differ from the V2-tapped / ReLU-headed model on the same weights."""
    from visiondepth3d_b200.synth import synth_frame
    RD, sd, spec = loaded
    for (w, h) in ((320, 180), (400, 400), (200, 120)):
        fr = synth_frame(1, w, h, "natural")[0]
        got = RD._engine_for(w, h).infer(fr)[0]
        assert RD._engine_for(w, h).cfg == spec
        v2 = _engine(sd, DW.da_spec("vits"), *RD.model_processed_size(w, h))
        other = v2.infer(fr)[0]
        v2.close()
        assert np.abs(got - other).max() > 1e-3 * np.abs(got).max()
        if spec["head"] == "metric":
            assert 0 <= got.min() and got.max() <= spec["max_depth"]


def test_batch_of_four_equals_single_forwards(loaded):
    from visiondepth3d_b200.synth import synth_frame
    RD, _, _ = loaded
    frames = [synth_frame(i, 640, 360, k)[0] for i, k in ((1, "natural"), (2, "noise"), (3, "smooth"), (4, "natural"))]
    e = RD._engine_for(640, 360)
    batch = e.infer_batch(frames)
    for f, (d32, d8) in zip(frames, batch):
        s32, s8 = e.infer(f)
        assert np.array_equal(d32, s32) and np.array_equal(d8, s8)


def test_infer_images_mixed_sizes_equal_single_images(loaded):
    from visiondepth3d_b200.depth_engine import processed_size
    from visiondepth3d_b200.synth import synth_frame
    RD, _, _ = loaded
    sizes = [(640, 480), (1024, 768), (800, 600)]
    e = RD._engine_for(*sizes[0])
    assert all(processed_size(*s) == (e.image_h, e.image_w) for s in sizes)
    rgbs = [synth_frame(20 + k, w, h, "natural")[0][..., ::-1].copy() for k, (w, h) in enumerate(sizes)]
    for invert in (False, True):
        got = e.infer_images(rgbs, invert=invert, want_f32=True)
        for a, (u8, f32) in zip(rgbs, got):
            d32, d8 = e.infer(np.ascontiguousarray(a[..., ::-1]), invert=invert)
            assert np.array_equal(u8, d8)
            assert np.abs(f32 - d32).max() <= 1e-6 * np.abs(d32).max()


class _Bars:
    def __init__(self, bars):
        self.bars = bars

    def update_batch(self, frames, first_idx=0):
        return [self.bars] * len(frames)


@pytest.mark.parametrize("inf,bars,invert", [(None, None, False), (None, (12, 10), True), ((224, 126), None, True)])
def test_depth_frames_equal_host_composition(loaded, inf, bars, invert):
    from PIL import Image
    from tests import letterbox_oracle as L
    from tests.test_letterbox_cpu import _Cap
    RD, _, _ = loaded
    frames = L.track_frames()[:10]
    got = list(RD.iter_depth_frames(_Cap(frames, 2), 320, 180, invert, inf, batch_size=4,
                                    tracker=_Bars(bars) if bars else None))
    assert len(got) == len(frames)
    for f, g in zip(frames, got):
        d = RD.hf_batch_safe_pipe([Image.fromarray(f[..., ::-1].copy())], inf)[0]["predicted_depth"]
        want = RD.convert_depth_to_grayscale(d)
        if invert:
            want = 255 - want
        want = RD.resize_cubic_u8(want, 320, 180)
        if bars:
            want = RD.letterbox_repad(want, *bars)
        assert np.abs(g.astype(int) - want.astype(int)).max() <= 1


def test_tiled_depth_equals_tile_composition(loaded):
    """USE_TILED_DEPTH: the tiled video pass equals infer_depth_tile through the pipe frame by frame, and
    infer_depth_tile equals the blend of the pipe's own tile predictions (tile-size engines carry the spec)."""
    from tests import tiled_oracle as T
    from tests.test_letterbox_cpu import _Cap
    from tests.test_tiled_depth_gpu import _engine_preds, _oracle_crops, _oracle_outer
    RD, _, _ = loaded
    rng = np.random.default_rng(11)
    rgb = np.clip(rng.normal(128, 50, (120, 200, 3)), 0, 255).astype(np.uint8)
    got = RD.infer_depth_tile(RD.pipe, rgb, None, tile=96, pad=16)
    img = _oracle_outer(rgb, None)
    plan = T.plan(img.shape[1], img.shape[0], 96, 16)
    want = T.blend(_engine_preds(RD, _oracle_crops(img, plan)), plan, img.shape[1], img.shape[0], 96, 16)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    W, H = 176, 100
    frames = [np.clip(rng.normal(120, 50, (H, W, 3)), 0, 255).astype(np.uint8) for _ in range(6)]
    RD.USE_TILED_DEPTH, RD.TILE_SIZE, RD.TILE_PAD = True, 96, 16
    try:
        out = list(RD.iter_depth_frames(_Cap(frames, 2), W, H, True, None, 4))
        ref = [RD._normalize_to_u8(RD.infer_depth_tile(RD.pipe, f[..., ::-1].copy(), None, 96, 16), (W, H), True)
               for f in frames]
    finally:
        RD.USE_TILED_DEPTH, RD.TILE_SIZE, RD.TILE_PAD = False, 512, 32
    for a, b in zip(out, ref):
        assert np.array_equal(a, b)


def test_clip_depth_pipeline_equals_stagewise(loaded):
    """vd3d_render_clip_depth (a clone of the engine on a second stream, CUDA graphs) against depth inference then
    vd3d_render_frame: the clone and the graphs run the model's taps and head."""
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R3
    from visiondepth3d_b200.synth import synth_frame
    _, sd, spec = loaded
    w, h = 640, 360
    e = _engine(sd, spec, 364, 644)
    rp = R3.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, "Half-SBS", 16 / 9, 0.0, 10.0, 9, True, True,
                               zero_parallax_strength=0.01)
    frames = [synth_frame(i, w, h, "smooth")[0] for i in range(11)]
    ctx = e.ctx
    ctx.reset()
    ref = [R3.render_frame(f, e.infer(f, check_size=False)[1], rp, ctx=ctx) for f in frames]
    ctx.reset()
    n = len(frames)
    outs = [np.empty_like(ref[0]) for _ in range(n)]
    fp = (C.c_void_p * n)(*[f.ctypes.data for f in frames])
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    for _ in range(2):  # the second clip replays the captured graphs
        ctx.reset()
        ctx.check(ctx.lib.vd3d_render_clip_depth(ctx.h, e.h, n, fp, h, w, C.byref(rp), op, _lib.MEM_HOST))
        for i, (a, b) in enumerate(zip(ref, outs)):
            assert np.array_equal(a, b), i
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
# the menu: update_pipeline on folders written by save_pretrained, in the reference's cache layout
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("label,spec", [("Depth Anything V1 Small", V1["vits"]),
                                        ("Distil-Any-Depth-Small", DW.da_spec("vits")),
                                        ("V2-Metric-Indoor-Large", DW.da_spec("vitl", head="metric", max_depth=20.0))])
def test_update_pipeline_from_saved_folder(tmp_path, monkeypatch, label, spec):
    from PIL import Image
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200 import render_depth as RD
    from tests.test_da_family_cpu import _processor
    sd, spec = DO.random_model(spec, seed=2)
    model = DepthAnythingForDepthEstimation(DW.hf_config(spec)).eval()
    model.load_state_dict(sd)
    ck = RD.supported_models[label][0]
    folder = tmp_path / "weights" / ck.replace("/", "_")
    model.save_pretrained(str(folder))
    _processor().save_pretrained(str(folder))
    monkeypatch.setattr(RD, "local_model_dir", str(tmp_path / "weights"))
    RD.update_pipeline(label, None, None, None).join()
    assert RD._spec == DW.da_config_from_json(json.load(open(folder / "config.json"))) == spec
    img = Image.fromarray(np.random.default_rng(1).integers(0, 256, (300, 500, 3), dtype=np.uint8))
    got = RD.pipe([img])[0]["predicted_depth"].numpy()
    RD.load_depth_model(spec, sd, 384, 384)
    assert np.array_equal(got, RD.pipe([img])[0]["predicted_depth"].numpy())
    if spec["taps"] != DW.CONFIGS[DW.da_arch(spec)]["taps"]:  # V1: the same weights loaded as V2 give other depth
        RD.load_depth_model(DW.da_arch(spec), sd, 384, 384)
        other = RD.pipe([img])[0]["predicted_depth"].numpy()
        assert np.abs(got - other).max() > 1e-3 * np.abs(got).max()
    # tampered files are refused before anything loads
    cfg = json.load(open(folder / "config.json"))
    json.dump(dict(cfg, head_hidden_size=64), open(folder / "config.json", "w"))
    assert RD.ensure_model_downloaded(ck) == (None, None)
    json.dump(cfg, open(folder / "config.json", "w"))
    pj = json.load(open(folder / "preprocessor_config.json"))
    json.dump(dict(pj, keep_aspect_ratio=False), open(folder / "preprocessor_config.json", "w"))
    assert RD.ensure_model_downloaded(ck) == (None, None)
    before = RD._state_dict
    RD.update_pipeline(label, None, None, None).join()
    assert RD._state_dict is before
