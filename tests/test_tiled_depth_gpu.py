"""GPU: the tiled depth path (tiled_depth.cu, vd3d_tile_* / vd3d_normalize_u8 / vd3d_depth_tiled) against the
restatement in tests/tiled_oracle.py and the tiled_* fixtures recorded from the reference."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from oracle import dibr as O
from tests import tiled_oracle as T

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = sorted(p for p in glob.glob(os.path.join(GOLDEN, "tiled_*.npz")) if "tiled_video_" not in p)
IDS = [os.path.basename(p)[6:-4] for p in FIXTURES]


def _ctx():
    from visiondepth3d_b200 import _lib
    return _lib, _lib.default_context(0)


def _tiles(plan):
    _lib, _ = _ctx()
    arr = (_lib.Tile * len(plan))()
    for k, r in enumerate(plan):
        arr[k] = _lib.Tile(*r, 0)
    return arr


def _fixture(path):
    g = np.load(path)
    w, h = (int(v) for v in g["size"])
    inf = tuple(int(v) for v in g["inference_size"])
    inf = None if inf == (0, 0) else inf
    return g, w, h, inf, int(g["tile"]), int(g["pad"])


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_crops(path):
    _lib, ctx = _ctx()
    g, w, h, inf, tile, pad = _fixture(path)
    img = np.ascontiguousarray(T.outer_resize(g["rgb"], inf)[:, :, ::-1])  # BGR, as the engine sees frames
    ih, iw = img.shape[:2]
    plan = T.plan(iw, ih, tile, pad)
    total = sum(r[8] * r[9] * 3 for r in plan)
    out = np.empty(total, np.uint8)
    ctx.check(ctx.lib.vd3d_tile_crops(ctx.h, img.ctypes.data, ih, iw, tile, pad, _tiles(plan), len(plan),
                                      out.ctypes.data, _lib.MEM_HOST))
    o = 0
    ref_crops = T.crops(img[:, :, ::-1], plan)  # RGB, recorded order
    for r, rc in zip(plan, ref_crops):
        y0, y1, x0, x1, yp0, yp1, xp0, xp1, rh, rw = r
        got = out[o:o + rh * rw * 3].reshape(rh, rw, 3)
        o += rh * rw * 3
        src = img[yp0:yp1, xp0:xp1]
        if src.shape[:2] == (rh, rw):
            want = src
        else:  # the oracle's cv2 arithmetic per channel: exact
            want = np.stack([O.resize_cubic_u8(np.ascontiguousarray(src[..., c]), rw, rh) for c in range(3)], -1)
        assert np.array_equal(got, want), r
        assert np.abs(got[:, :, ::-1].astype(int) - rc.astype(int)).max() <= 1  # cv2 itself: within 1 LSB
    assert np.abs(np.concatenate([c.ravel() for c in ref_crops]).astype(int) - g["crops"].astype(int)).max() <= 1


def _blend(plan, preds, wts, ih, iw, tile, pad, mem):
    _lib, ctx = _ctx()
    n = len(plan)
    out = np.empty((ih, iw), np.float32)
    mm = np.empty(2, np.float32)
    if mem == _lib.MEM_HOST:
        pp = (C.c_void_p * n)(*[p.ctypes.data for p in preds])
        wp = (C.c_void_p * n)(*[x.ctypes.data for x in wts])
        ctx.check(ctx.lib.vd3d_tile_blend(ctx.h, ih, iw, tile, pad, _tiles(plan), n, pp, wp, out.ctypes.data,
                                          mm.ctypes.data, mem))
        return out, mm
    import torch
    pd = [torch.from_numpy(p).cuda() for p in preds]
    wd = [torch.from_numpy(x).cuda() for x in wts]
    od = torch.empty((ih, iw), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.check(ctx.lib.vd3d_tile_blend(ctx.h, ih, iw, tile, pad, _tiles(plan), n,
                                      (C.c_void_p * n)(*[p.data_ptr() for p in pd]),
                                      (C.c_void_p * n)(*[x.data_ptr() for x in wd]), od.data_ptr(), mm.ctypes.data,
                                      mem))
    return od.cpu().numpy(), mm


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_blend_bit_exact(path):
    _lib, _ = _ctx()
    g, w, h, inf, tile, pad = _fixture(path)
    img = T.outer_resize(g["rgb"], inf)
    ih, iw = img.shape[:2]
    plan = T.plan(iw, ih, tile, pad)
    preds = [T.prediction(c, str(g["kind"])) for c in T.crops(img, plan)]
    wts = [np.ascontiguousarray(T.weights(r[1] - r[0], r[3] - r[2], tile, pad)) for r in plan]
    for mem in (_lib.MEM_HOST, _lib.MEM_DEVICE):
        out, mm = _blend(plan, preds, wts, ih, iw, tile, pad, mem)
        assert np.array_equal(out.view(np.uint32), g["depth"].view(np.uint32)), mem
        assert mm[0] == np.nanmin(g["depth"]) and mm[1] == np.nanmax(g["depth"])


def _normalize(d, out_size, invert=False, pclip=(1.0, 99.0)):
    _lib, ctx = _ctx()
    d = np.ascontiguousarray(d, np.float32)
    ow, oh = out_size
    out = np.empty((oh, ow), np.uint8)
    st = np.empty(4, np.float32)
    ctx.check(ctx.lib.vd3d_normalize_u8(ctx.h, d.ctypes.data, d.shape[0], d.shape[1], pclip[0], pclip[1], int(invert),
                                        out.ctypes.data, oh, ow, st.ctypes.data, _lib.MEM_HOST))
    return out, st


@pytest.mark.parametrize("path", FIXTURES, ids=IDS)
def test_normalize_fixture(path):
    from visiondepth3d_b200 import render_depth as R
    g, w, h, *_ = _fixture(path)
    u8, st = _normalize(g["depth"], (w, h), bool(g["invert"]))
    # exact against the restatement with the cv2-pinned resize oracle; the recorded cv2 frame within its 1 LSB
    assert np.array_equal(u8, T.normalize_u8(g["depth"], (w, h), bool(g["invert"]), resize=O.resize_cubic_u8))
    assert np.abs(u8.astype(int) - g["u8"].astype(int)).max() <= 1
    if g["depth"].shape == (h, w):
        assert np.array_equal(u8, g["u8"])
    assert np.array_equal(st[:2], g["pct"])
    assert np.array_equal(R._normalize_to_u8(g["depth"], (w, h), bool(g["invert"])), u8)


def _planes():
    rng = np.random.default_rng(11)
    out = [rng.standard_normal((90, 160)).astype(np.float32),
           (rng.standard_normal((37, 53)) * 1e30).astype(np.float32),
           np.full((20, 30), 2.5, np.float32),                       # flat: both fallbacks -> 128
           np.full((1, 1), -4.0, np.float32),                        # n = 1
           np.array([[1.0, -2.0]], np.float32),                      # n = 2
           rng.integers(-2, 3, (64, 64)).astype(np.float32),         # duplicates
           rng.standard_normal((1080, 1920)).astype(np.float32) * 3 - 7]
    lohi = np.full((50, 60), 5.0, np.float32)
    lohi[0, :4] = -1.0                                                # p1 == p99, range -> min-max
    out.append(lohi)
    bad = rng.standard_normal((70, 70)).astype(np.float32)
    bad[::5, ::3], bad[1::7, ::2], bad[2::9] = np.nan, np.inf, -np.inf
    out.append(bad)
    neg0 = np.zeros((16, 16), np.float32)
    neg0[::2] = -0.0
    neg0[3, 3] = 1e-3
    out.append(neg0)
    return out


@pytest.mark.parametrize("k", range(10))
def test_normalize_planes(k):
    d = _planes()[k]
    h, w = d.shape
    for invert in (False, True):
        for size in ((w, h), (max(1, w * 3 // 2), max(1, h // 2 + 1))):
            got, _ = _normalize(d, size, invert)
            assert np.array_equal(got, T.normalize_u8(d, size, invert, resize=O.resize_cubic_u8)), (k, invert, size)
    got, _ = _normalize(d, (w, h), False, (5.0, 95.0))
    assert np.array_equal(got, T.normalize_u8(d, (w, h), False, (5.0, 95.0)))


@pytest.fixture(scope="module")
def model():
    from visiondepth3d_b200 import render_depth as R
    R.load_depth_model("vits", None, 128, 128, seed=3)
    yield R


def _oracle_crops(img, plan):
    """T.crops with the cv2-pinned cubic oracle (the device's arithmetic) in place of cv2."""
    out = []
    for y0, y1, x0, x1, yp0, yp1, xp0, xp1, rh, rw in plan:
        c = img[yp0:yp1, xp0:xp1]
        if c.shape[:2] != (rh, rw):
            c = np.stack([O.resize_cubic_u8(np.ascontiguousarray(c[..., k]), rw, rh) for k in range(3)], -1)
        out.append(np.ascontiguousarray(c))
    return out


def _engine_preds(R, crops):
    """The pipe's own predictions of the crops (RGB), batched by size in plan order as vd3d_depth_tiled batches them."""
    from PIL import Image
    preds = [None] * len(crops)
    by = {}
    for k, c in enumerate(crops):
        by.setdefault(c.shape[:2], []).append(k)
    for (rh, rw), idx in by.items():
        res = R.pipe([Image.fromarray(crops[k]) for k in idx], inference_size=(rw, rh))
        for k, r in zip(idx, res):
            preds[k] = r["predicted_depth"].numpy()
    return preds


def _oracle_outer(rgb, inf):
    """infer_depth_tile's first resize with the device's arithmetic: cv2 INTER_AREA when shrinking (vd3d_fit_eye
    reproduces it exactly), the cv2-pinned cubic oracle per channel when enlarging."""
    h, w = rgb.shape[:2]
    tw, th = inf or (w, h)
    if (tw, th) == (w, h) or (tw <= w and th <= h):
        return T.outer_resize(rgb, inf)
    return np.stack([O.resize_cubic_u8(np.ascontiguousarray(rgb[..., k]), tw, th) for k in range(3)], -1)


@pytest.mark.parametrize("case", [((200, 120), None, 96, 16), ((256, 144), (200, 112), 96, 16),
                                  ((160, 90), (208, 117), 96, 16), ((100, 64), None, 64, 24)])
def test_infer_depth_tile_composition(model, case):
    R = model
    (w, h), inf, tile, pad = case
    rng = np.random.default_rng(w + h)
    rgb = np.clip(rng.normal(128, 50, (h, w, 3)), 0, 255).astype(np.uint8)
    got = R.infer_depth_tile(R.pipe, rgb, inf, tile=tile, pad=pad)
    img = _oracle_outer(rgb, inf)
    plan = T.plan(img.shape[1], img.shape[0], tile, pad)
    crops = _oracle_crops(img, plan)
    want = T.blend(_engine_preds(R, crops), plan, img.shape[1], img.shape[0], tile, pad)
    assert got.dtype == np.float32
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_infer_depth_tile_matches_fp32_oracle():
    """infer_depth_tile(pipe, ...) at the default tile 512 / pad 32 against oracle/depth.py on the CPU, per tile and
    blended.  A 1000x600 frame gives 6 tiles: 546x546 crops (processed at 518x518, the native position-embedding grid)
    and narrow edge crops (140 wide).  The model is the random-init vits of test_depth_gpu.py with its non-negative
    last conv.

    Error model.  Per tile, the engine's prediction p_i differs from the oracle's by e_i with |e_i| <= 1e-3 * S_i (S_i
    the tile's range; the north-star gate, asserted here per tile).  The blend is out = sum(w_i p_i) / max(sum(w_i),
    1e-8) with the same float32 operations on both sides, so at a pixel
        |out - out_ref| <= A * (E + 3e-7 * C),   A = sum(|w_i|) / max(sum(w_i), 1e-8),
    E = max_i 1e-3 * S_i, C = max_i |p_i| (the 3e-7 * C term covers the float32 roundings of the two sums).  A = 1
    where every weight is positive (most of the frame); it grows at border pixels covered only by Hann tails.
    For the u8 frame: every pixel stays within [ref - b_p, ref + b_p] (b_p the bound above), and a percentile is
    monotone in the data, so lo lies between the percentiles of ref - b and ref + b: |lo - lo_ref| <= dlo, likewise
    dhi.  With t = (d - lo) / (hi - lo) in [0, 1], |t - t_ref| <= (b_p + dlo + (dlo + dhi)) / (hi - lo - dlo - dhi),
    and after x255 and truncation |u8 - u8_ref| <= ceil(255 * that) + 1 at each pixel (the output is written at the
    depth's own size, so the final resize is a copy).  Border pixels with a large A get a loose bound; the percentiles,
    and so every other pixel, do not."""
    import torch
    import torch.nn.functional as F
    from oracle import depth as OD
    from tests.test_depth_gpu import _model
    from visiondepth3d_b200 import render_depth as R
    from visiondepth3d_b200.depth_weights import CONFIGS
    sd = _model("vits")
    R.load_depth_model("vits", sd, 518, 518)
    W, H = 1000, 600
    rng = np.random.default_rng(4)
    base = np.clip(rng.normal(128, 40, (H // 8, W // 8, 3)), 0, 255).astype(np.uint8)
    import cv2
    rgb = cv2.resize(base, (W, H), interpolation=cv2.INTER_LINEAR)  # smooth content, like a picture
    plan = T.plan(W, H, 512, 32)
    assert len(plan) == 6 and {(r[8], r[9]) for r in plan} >= {(546, 546)}
    assert any(r[9] < 200 for r in plan)
    got = R.infer_depth_tile(R.pipe, rgb, None)
    crops = _oracle_crops(rgb, plan)
    ref_preds, S, C = [], [], 0.0
    for crop, r in zip(crops, plan):
        rh, rw = r[8], r[9]
        eng = R._engine_for(rw, rh)
        d32, _ = eng.infer(np.ascontiguousarray(crop[..., ::-1]))  # the engine alone on this crop
        px = eng.get_buffer("px", (3, eng.image_h, eng.image_w), np.float32)
        with torch.no_grad():
            ref = OD.forward(sd, CONFIGS["vits"], torch.from_numpy(px.copy()))
            ref = F.interpolate(ref[None, None], size=(rh, rw), mode="bicubic", align_corners=False)[0, 0].numpy()
        s = float(ref.max() - ref.min())
        assert s > 0 and np.abs(d32 - ref).max() / s <= 1e-3, (r, np.abs(d32 - ref).max() / s)
        ref_preds.append(ref.astype(np.float32))
        S.append(s)
        C = max(C, float(np.abs(ref).max()))
    want = T.blend(ref_preds, plan, W, H, 512, 32)
    wsum = np.zeros((H, W), np.float32)
    wabs = np.zeros((H, W), np.float32)
    for r in plan:
        wm = T.weights(r[1] - r[0], r[3] - r[2], 512, 32)
        wsum[r[0]:r[1], r[2]:r[3]] += wm
        wabs[r[0]:r[1], r[2]:r[3]] += np.abs(wm)
    A = wabs.astype(np.float64) / np.maximum(wsum, 1e-8)
    bound = A * (1e-3 * max(S) + 3e-7 * C)
    err = np.abs(got.astype(np.float64) - want)
    assert (err <= bound).all(), (err.max(), float(bound[err.argmax() // W, err.argmax() % W]))
    # the bulk of the frame (all weights positive): the plain 1e-3-of-range gate
    inner = A <= 1.0 + 1e-6
    assert inner.mean() > 0.9 and err[inner].max() <= 1e-3 * max(S) + 3e-7 * C
    w64 = want.astype(np.float64)
    lo, hi = float(T.percentile(want, 1.0)), float(T.percentile(want, 99.0))
    slack = 1e-6 * max(abs(lo), abs(hi))  # float32 vs float64 evaluation of the same interpolation
    dlo = max(abs(np.percentile(w64 + s_ * bound, 1.0) - lo) for s_ in (-1, 1)) + slack
    dhi = max(abs(np.percentile(w64 + s_ * bound, 99.0) - hi) for s_ in (-1, 1)) + slack
    assert hi - lo > dlo + dhi
    u8_bound = np.ceil(255 * (bound + 2 * dlo + dhi) / (hi - lo - dlo - dhi)) + 1
    du = np.abs(R._normalize_to_u8(got, (W, H)).astype(int) - T.normalize_u8(want, (W, H)).astype(int))
    assert (du <= u8_bound).all(), (du.max(), float(u8_bound[inner].max()))
    print(f"tiled vs fp32 oracle: err/range {err[inner].max() / max(S):.2e} (interior), u8 max diff {du.max()}, "
          f"bound {int(u8_bound[inner].max())} where all weights are positive")


def test_infer_depth_tile_refuses_mixed_resize(model):
    R = model
    with pytest.raises(ValueError):
        R.infer_depth_tile(R.pipe, np.zeros((60, 80, 3), np.uint8), (60, 70))


def test_run_pipe_or_tile_prints_range(model, capsys):
    from PIL import Image
    R = model
    rgb = np.random.default_rng(1).integers(0, 256, (90, 130, 3), dtype=np.uint8)
    R.USE_TILED_DEPTH, R.TILE_SIZE, R.TILE_PAD, R.TILE_DEBUG = True, 64, 16, True
    try:
        out = R._run_pipe_or_tile([Image.fromarray(rgb)], None)
    finally:
        R.USE_TILED_DEPTH, R.TILE_SIZE, R.TILE_PAD, R.TILE_DEBUG = False, 512, 32, False
    dep = out[0]["predicted_depth"]
    lines = capsys.readouterr().out.splitlines()
    assert lines[:-1] == T.debug_lines(T.plan(130, 90, 64, 16))
    assert lines[-1] == f"[tile] range min={float(np.nanmin(dep)):.6f} max={float(np.nanmax(dep)):.6f}"


class _Cap:
    def __init__(self, frames):
        self.frames = list(frames)

    def read(self):
        return (True, self.frames.pop(0)) if self.frames else (False, None)


class _Bars:
    """Stand-in tracker: fixed bars after every batch."""

    def __init__(self, bars):
        self.bars = bars

    def update_batch(self, frames, first_idx=0):
        return [self.bars] * len(frames)


@pytest.mark.parametrize("inf,tracker,invert", [(None, None, False), ((160, 96), None, True), (None, (8, 6), False)])
def test_video_pass_tiled(model, inf, tracker, invert):
    from PIL import Image
    R = model
    W, H = 176, 100
    rng = np.random.default_rng(5)
    frames = [np.clip(rng.normal(120, 50, (H, W, 3)), 0, 255).astype(np.uint8) for _ in range(11)]
    R.USE_TILED_DEPTH, R.TILE_SIZE, R.TILE_PAD = True, 96, 16
    try:
        got = list(R.iter_depth_frames(_Cap(frames), W, H, invert, inf, 4,
                                       tracker=_Bars(tracker) if tracker else None))
        want = []
        for f in frames:
            rgb = f[..., ::-1].copy()
            if inf is not None:
                rgb = np.asarray(Image.fromarray(rgb).resize(inf, Image.BICUBIC))
            d8 = R._normalize_to_u8(R.infer_depth_tile(R.pipe, rgb, None, 96, 16), (W, H), invert)
            if tracker:
                d8 = R.letterbox_repad(d8, *tracker)
            want.append(d8)
    finally:
        R.USE_TILED_DEPTH, R.TILE_SIZE, R.TILE_PAD = False, 512, 32
    assert len(got) == len(want) == 11
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def test_video_pass_debug_log_per_image(model, capsys):
    """TILE_DEBUG in the video pass: each image's tile lines, then its range line, image after image."""
    R = model
    frames = [np.random.default_rng(k).integers(0, 256, (100, 150, 3), dtype=np.uint8) for k in range(3)]
    R.USE_TILED_DEPTH, R.TILE_SIZE, R.TILE_PAD, R.TILE_DEBUG = True, 96, 16, True
    try:
        list(R.iter_depth_frames(_Cap(frames), 150, 100, False, None, 3))
    finally:
        R.USE_TILED_DEPTH, R.TILE_SIZE, R.TILE_PAD, R.TILE_DEBUG = False, 512, 32, False
    lines = capsys.readouterr().out.splitlines()
    per = T.debug_lines(T.plan(150, 100, 96, 16))
    assert len(lines) == 3 * (len(per) + 1)
    for k in range(3):
        chunk = lines[k * (len(per) + 1):(k + 1) * (len(per) + 1)]
        assert chunk[:-1] == per and chunk[-1].startswith("[tile] range min=")


def test_tile_crops_beyond_grid_z_limit():
    """More tile jobs than gridDim.z allows (65535) in one gather: 4112 x 4096 with tile 16 / pad 0 is 65792 tiles."""
    _lib, ctx = _ctx()
    h, w = 4096, 4112
    img = np.random.default_rng(2).integers(0, 256, (h, w, 3), dtype=np.uint8)
    plan = T.plan(w, h, 16, 0)
    assert len(plan) > 65535
    out = np.empty(sum(r[8] * r[9] * 3 for r in plan), np.uint8)
    ctx.check(ctx.lib.vd3d_tile_crops(ctx.h, img.ctypes.data, h, w, 16, 0, _tiles(plan), len(plan), out.ctypes.data,
                                      _lib.MEM_HOST))
    per = 28 * 28 * 3
    for k in (0, 65534, 65535, len(plan) - 1):
        y0, y1, x0, x1, yp0, yp1, xp0, xp1, rh, rw = plan[k]
        src = img[yp0:yp1, xp0:xp1]
        want = np.stack([O.resize_cubic_u8(np.ascontiguousarray(src[..., c]), rw, rh) for c in range(3)], -1)
        assert np.array_equal(out[k * per:(k + 1) * per].reshape(rh, rw, 3), want), k


def test_depth_tiled_refuses_engine_on_other_stream(model):
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200.depth_engine import DepthEngine
    R = model
    ctx = _lib.default_context(0)
    other = _lib.Context(0)
    eng = DepthEngine("vits", 70, 84, ctx=other)
    plan = R._plan_for(60, 50, 96, 16)
    frame = np.zeros((50, 60, 3), np.uint8)
    u8 = np.empty((50, 60), np.uint8)
    vp = C.c_void_p
    rc = ctx.lib.vd3d_depth_tiled(ctx.h, (vp * 1)(eng.h), 1, 1, (vp * 1)(frame.ctypes.data), 50, 60, 96, 16, plan.tiles,
                                  len(plan.rects), plan.weight_ptrs, 0, 50, 60, (vp * 1)(u8.ctypes.data), None, None,
                                  _lib.MEM_HOST)
    assert rc != 0 and b"vd3d_stream" in ctx.lib.vd3d_last_error(ctx.h)
    eng.close()
    other.close()


def test_depth_tiled_device_frames(model):
    import torch
    R = model
    rng = np.random.default_rng(8)
    frames = [rng.integers(0, 256, (120, 200, 3), dtype=np.uint8) for _ in range(3)]
    u_h, f_h, mm_h = R.depth_tiled(frames, 200, 120, (240, 150), True, 96, 16, want_f32=True)
    dev = torch.from_numpy(np.stack(frames)).cuda()
    u_d, f_d, mm_d = R.depth_tiled(dev, 200, 120, (240, 150), True, 96, 16, want_f32=True)
    for k in range(3):
        assert np.array_equal(u_h[k], u_d[k].cpu().numpy())
        assert np.array_equal(f_h[k], f_d[k].cpu().numpy())
    assert mm_h == mm_d


def test_untiled_pass_issues_no_tiled_call(model, monkeypatch):
    R = model

    def boom(*a, **k):
        raise AssertionError("tiled call with USE_TILED_DEPTH False")

    monkeypatch.setattr(R, "depth_tiled", boom)
    frames = [np.full((64, 96, 3), 90, np.uint8)] * 3
    assert len(list(R.iter_depth_frames(_Cap(frames), 96, 64, False, None, 2))) == 3
