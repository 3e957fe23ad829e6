"""GPU: auto_crop_black_bars on the device (k_black_bars -> ingest rectangle from two device words).

k_black_bars against the oracle's detect_black_bars; the loop fixtures of the unmodified reference in both arithmetic
modes (exact: bit for bit with the oracle); frames without bars unchanged by the option; graphs, pipelining, the
depth + stereo clip and the sharded state chain unchanged by it; the per-frame (top, bottom) reports; launch counts;
render_sbs_3d end to end."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from oracle import dibr as O
from tests import autocrop_oracle as A
from tests.test_autocrop_cpu import AUTOCROP_CASES, oracle_params
from tests.util import u8_diff
from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu

MODES = ["fast", "exact"]
W, H = 320, 180


@pytest.fixture
def ctx():
    from visiondepth3d_b200 import _lib
    c = _lib.Context()
    yield c
    c.close()


def _rp(o):
    """vd3d_render_params of an oracle RenderParams."""
    from visiondepth3d_b200 import render_3d as R
    return R.make_render_params(
        o.output_width, o.output_height, o.fg_shift, o.mg_shift, o.bg_shift, o.sharpness_factor, o.output_format,
        o.aspect_ratio, o.dof_strength, o.feather_strength, o.blur_ksize, o.use_subject_tracking, o.use_floating_window,
        o.max_pixel_shift_percent, o.preserve_original_aspect, o.zero_parallax_strength, o.enable_edge_masking,
        o.enable_feathering, o.original_video_width, o.original_video_height, o.convergence_strength,
        o.enable_dynamic_convergence, o.ipd_factor, o.color_saturation, o.color_contrast, o.color_brightness,
        o.auto_crop_black_bars)


def _params(**kw):
    a = dict(output_width=W, output_height=H, sharpness_factor=0.2, output_format="Half-SBS", feather_strength=10.0,
             blur_ksize=9, use_subject_tracking=True, use_floating_window=True, zero_parallax_strength=0.01,
             auto_crop_black_bars=True)
    a.update(kw)
    o = A.RenderParams(**a)
    return _rp(o), o


def detect(ctx, frame, mem="host"):
    from visiondepth3d_b200 import _lib
    t, b = C.c_int(), C.c_int()
    h, w = frame.shape[:2]
    if mem == "host":
        ctx.check(ctx.lib.vd3d_detect_black_bars(ctx.h, frame.ctypes.data, h, w, _lib.MEM_HOST, C.byref(t), C.byref(b)))
    else:
        import torch
        d = torch.from_numpy(frame).cuda()
        torch.cuda.synchronize()
        ctx.check(ctx.lib.vd3d_detect_black_bars(ctx.h, d.data_ptr(), h, w, _lib.MEM_DEVICE, C.byref(t), C.byref(b)))
    return t.value, b.value


def clip(ctx, rp, frames, infos=False):
    """vd3d_render_clip over [(frame, depth)] -> (outputs, frame infos or None, (top, bottom) per frame)."""
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R
    n = len(frames)
    sh, sw = frames[0][0].shape[:2]
    dch = 1 if frames[0][1].ndim == 2 else 3
    outs = [np.empty(R.output_shape(rp, R.plan_sizes(sw, sh, rp)), dtype=np.uint8) for _ in range(n)]
    fp = (C.c_void_p * n)(*[f.ctypes.data for f, _ in frames])
    dp = (C.c_void_p * n)(*[d.ctypes.data for _, d in frames])
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    inf = (_lib.FrameInfo * n)() if infos else None
    ctx.check(ctx.lib.vd3d_render_clip(ctx.h, n, fp, dp, dch, sh, sw, C.byref(rp), op, _lib.MEM_HOST, inf))
    crops = []
    if rp.auto_crop_black_bars:
        tb = (C.c_int32 * (2 * n))()
        ctx.check(ctx.lib.vd3d_last_crops(ctx.h, tb, n))
        crops = [(tb[2 * i], tb[2 * i + 1]) for i in range(n)]
    return outs, inf, crops


def _bars_frame(rng, h, w):
    """Dark rows (gray <= 6) around bright content rows, plus rows on the mean-10 edge."""
    f = rng.integers(0, 7, (h, w, 3), dtype=np.uint8)
    t, b = sorted(int(v) for v in rng.integers(0, h, 2))
    if rng.random() < 0.9:
        f[t:b + 1] = rng.integers(0, 256, (b + 1 - t, w, 3), dtype=np.uint8)
    if rng.random() < 0.5:
        y = int(rng.integers(0, h))
        f[y] = 10
        if rng.random() < 0.5:
            f[y, int(rng.integers(0, w))] = 11
    return f


@pytest.mark.parametrize("mem", ["host", "device"])
def test_detect_black_bars_matches_oracle(ctx, mem):
    rng = np.random.default_rng(12)
    sizes = [(1, 1), (23, 37), (180, 321), (31, 16), (90, 160), (17, 1001), (1080, 1920), (2160, 3840)]
    for h, w in sizes:
        for _ in range(6 if h * w < 10 ** 6 else 2):
            f = _bars_frame(rng, h, w)
            assert detect(ctx, f, mem) == A.detect_black_bars(f), (h, w)
    for i in range(8):
        f, _ = synth_frame(i, W, H, "letterbox")
        assert detect(ctx, f, mem) == A.detect_black_bars(f), i


@pytest.mark.parametrize("name", sorted(AUTOCROP_CASES))
@pytest.mark.parametrize("mode", MODES)
def test_loop_goldens(ctx, golden_dir, name, mode):
    n, kw = AUTOCROP_CASES[name]
    g = np.load(os.path.join(golden_dir, name))
    step = int(g["rows"])
    probe, _ = synth_frame(0, W, H, "letterbox")
    assert detect(ctx, probe) == tuple(g["crops"][0])
    orp = oracle_params(kw, probe)
    rp = _rp(orp)
    ctx.set_exact(mode == "exact")
    ctx.reset()
    frames = [synth_frame(i, W, H, "letterbox") for i in range(1, n)]
    outs, infos, crops = clip(ctx, rp, frames, infos=True)
    assert crops == [tuple(int(v) for v in c) for c in g["crops"][1:]]
    assert [(f.crop_top, f.crop_bottom) for f in infos] == crops
    gs, cs = O.GlobalState(), O.ClipState()
    for j, (fr, dp) in enumerate(frames):
        ref = A.render_frame(gs, cs, fr, dp, orp)
        if mode == "exact":
            assert np.array_equal(outs[j], ref), (name, j)
        else:  # tests/test_dibr_gpu.py _tol("fast", "natural"): packed frames against the oracle
            mx, f0, f1 = u8_diff(outs[j], ref)
            assert mx <= 16 and f1 <= 0.012 and f0 <= 0.05, (name, j, mx, f0, f1)
        # against the reference: the oracle's own gate (tests/test_autocrop_cpu.py), widened by the fast path's
        mx, f0, f1 = u8_diff(outs[j][::step], g[f"final{j}"])
        assert mx <= (12 if mode == "exact" else 16) and f1 <= 0.03 + (0 if mode == "exact" else 0.012), \
            (name, mode, j, mx, f0, f1)


def test_realistic_scope_in_1080p_exact(ctx):
    """2.39:1 content letterboxed in 1920x1080 (138 + 138 dark rows), Half-SBS 1080p: bit for bit with the oracle."""
    rp, orp = _params(output_width=1920, output_height=1080)
    ctx.set_exact(True)
    ctx.reset()
    rng = np.random.default_rng(5)
    frames = []
    for i in range(1, 4):
        f, d = synth_frame(i, 1920, 1080, "natural")
        f[:138] = rng.integers(0, 7, (138, 1920, 3), dtype=np.uint8)
        f[1080 - 138:] = rng.integers(0, 7, (138, 1920, 3), dtype=np.uint8)
        frames.append((f, d))
    outs, _, crops = clip(ctx, rp, frames)
    assert crops == [(138, 138)] * 3
    gs, cs = O.GlobalState(), O.ClipState()
    for j, (f, d) in enumerate(frames):
        assert np.array_equal(outs[j], A.render_frame(gs, cs, f, d, orp)), j


@pytest.mark.parametrize("fmt", ["Half-SBS", "Full-SBS"])
def test_frames_without_bars_unchanged_exact(ctx, fmt):
    """No bars: the crop is the plain aspect crop and bilinear at scale 1 is an exact identity, so the output equals
    the option turned off -- including Full-SBS at source size, which samples the u8 frame directly when it is off."""
    ctx.set_exact(True)
    frames = [synth_frame(i, W, H, "natural") for i in range(1, 5)]
    res = []
    for on in (False, True):
        rp, _ = _params(output_format=fmt, preserve_original_aspect=fmt == "Full-SBS", auto_crop_black_bars=on)
        ctx.reset()
        res.append(clip(ctx, rp, frames)[0])
    for a, b in zip(*res):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("mode", MODES)
def test_graphs_pipelining_and_counts(ctx, mode):
    """Graphs on / off give the same bytes and launch counts; a 20-frame clip (staging slots reused) equals the frames
    rendered one by one."""
    from visiondepth3d_b200 import render_3d as R
    ctx.set_exact(mode == "exact")
    rp, _ = _params()
    frames = [synth_frame(i, W, H, "letterbox") for i in range(20)]
    res = []
    for graphs in (0, 1):
        ctx.check(ctx.lib.vd3d_set_graphs(ctx.h, graphs))
        ctx.reset()
        l0 = ctx.launches
        outs, _, crops = clip(ctx, rp, frames)
        res.append((outs, crops, ctx.launches - l0))
        assert ctx.lib.vd3d_graphs_active(ctx.h) == graphs
    assert res[0][1] == res[1][1] == [A.detect_black_bars(f) for f, _ in frames]
    assert res[0][2] == res[1][2]
    ctx.reset()
    for j, (f, d) in enumerate(frames):
        one, info = R.render_frame(f, d, rp, want_info=True, ctx=ctx)
        assert (info.crop_top, info.crop_bottom) == res[0][1][j]
        assert np.array_equal(one, res[0][0][j]) and np.array_equal(one, res[1][0][j]), j


def test_clip_depth_equals_clip_on_inferred_depth(ctx):
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import hf_config
    torch.manual_seed(0)
    eng = DepthEngine("vits", 70, 126, ctx=ctx)
    try:
        eng.load_state_dict(DepthAnythingForDepthEstimation(hf_config("vits")).eval().state_dict())
        rp, _ = _params()
        frames = [synth_frame(i, W, H, "letterbox")[0] for i in range(11)]
        depths = [eng.infer(f, check_size=False)[1] for f in frames]
        ctx.reset()
        ref, _, ref_crops = clip(ctx, rp, list(zip(frames, depths)))
        n = len(frames)
        outs = [np.empty_like(ref[0]) for _ in range(n)]
        fp = (C.c_void_p * n)(*[f.ctypes.data for f in frames])
        op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
        ctx.reset()
        ctx.check(ctx.lib.vd3d_render_clip_depth(ctx.h, eng.h, n, fp, H, W, C.byref(rp), op, _lib.MEM_HOST))
        tb = (C.c_int32 * (2 * n))()
        ctx.check(ctx.lib.vd3d_last_crops(ctx.h, tb, n))
        assert [(tb[2 * i], tb[2 * i + 1]) for i in range(n)] == ref_crops
        for i in range(n):
            assert np.array_equal(outs[i], ref[i]), i
    finally:
        eng.close()


def test_last_crops_needs_an_auto_cropped_clip(ctx):
    rp, _ = _params(auto_crop_black_bars=False)
    clip(ctx, rp, [synth_frame(i, W, H, "letterbox") for i in range(2)])
    tb = (C.c_int32 * 4)()
    assert ctx.lib.vd3d_last_crops(ctx.h, tb, 2) != 0


def test_sharded_state_chain_exact():
    """advance_state on one context, export, import into a second, render there == one context rendering throughout."""
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R
    rp, _ = _params()
    frames = [synth_frame(i, W, H, "letterbox") for i in range(8)]
    a, b = _lib.Context(), _lib.Context()
    try:
        for c in (a, b):
            c.set_exact(True)
            c.reset()
        ref = [R.render_frame(f, d, rp, ctx=a) for f, d in frames]
        c1 = _lib.Context()
        c1.set_exact(True)
        c1.reset()
        for f, d in frames[:5]:
            R.advance_state(f, d, rp, ctx=c1)
        b.import_state(c1.export_state())
        c1.close()
        for j in range(5, 8):
            assert np.array_equal(R.render_frame(*frames[j], rp, ctx=b), ref[j]), j
    finally:
        a.close()
        b.close()


# launches per frame with auto-crop on: the paths of tests/test_launch_sequence_gpu.py plus k_black_bars
LAUNCHES = {"half_sbs": (dict(), {"fast": 6, "exact": 42}),
            "full_sbs": (dict(output_format="Full-SBS", preserve_original_aspect=True), {"fast": 6, "exact": 41})}
ADVANCE = {"fast": 4, "exact": 38}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(LAUNCHES))
def test_launch_counts(ctx, case, mode):
    from visiondepth3d_b200 import render_3d as R
    kw, want = LAUNCHES[case]
    ctx.set_exact(mode == "exact")
    rp, _ = _params(**kw)
    for graphs in (0, 1):
        ctx.check(ctx.lib.vd3d_set_graphs(ctx.h, graphs))
        ctx.reset()
        counts = []
        for first in (0, 4):
            l0 = ctx.launches
            clip(ctx, rp, [synth_frame(first + i, W, H, "letterbox") for i in range(4)])
            counts.append(ctx.launches - l0)
        assert counts[1] == 4 * want[mode], (graphs, counts)
    rp, _ = _params()
    for f, d in (synth_frame(i, W, H, "letterbox") for i in range(2)):
        l0 = ctx.launches
        R.advance_state(f, d, rp, ctx=ctx)
        assert ctx.launches - l0 == ADVANCE[mode]


class _Var:
    def __init__(self, v):
        self.v = v

    def get(self):
        return self.v


@pytest.mark.parametrize("fmt", ["Half-SBS", "Full-SBS"])
def test_render_sbs_3d_auto_crop(tmp_path, capsys, monkeypatch, fmt):
    """render_sbs_3d(auto_crop_black_bars=True) on an MJPG letterbox clip: the reference's lines, the cropped probe size
    for preserve_original_aspect, and, byte for byte, the frames of the loop run by hand on the decoded inputs (what
    reaches the writer is recorded; the file itself must hold every frame)."""
    import cv2
    from visiondepth3d_b200 import render_3d as R
    w, h, n = W, H, 12
    # Full-SBS: the clip starts at schedule frame 5, whose cropped height (180 - 35 - 13) is even as MJPG needs
    first = 5 if fmt == "Full-SBS" else 0
    rgb, dep, out = str(tmp_path / "rgb.avi"), str(tmp_path / "depth.avi"), str(tmp_path / "out.avi")
    fourcc = cv2.VideoWriter_fourcc(*"MJPG")
    wr, wd = cv2.VideoWriter(rgb, fourcc, 24.0, (w, h)), cv2.VideoWriter(dep, fourcc, 24.0, (w, h))
    for i in range(first, first + n):
        f, d = synth_frame(i, w, h, "letterbox")
        wr.write(f)
        wd.write(d)
    wr.release()
    wd.release()
    written, sizes = [], []

    class Recording(R._FrameSink):
        def __init__(self, path, size, *a):
            sizes.append(size)
            super().__init__(path, size, *a)

        def write(self, frame):
            written.append(np.array(frame))
            super().write(frame)

    monkeypatch.setattr(R, "_FrameSink", Recording)
    preserve = fmt == "Full-SBS"
    R.reset_temporal_state()
    R.render_sbs_3d(rgb, dep, out, "MJPG", 24.0, w, h, 4.5, -1.5, -6.0, 0.2, fmt, _Var("Default (16:9)"),
                    R.aspect_ratios, 0.0, feather_strength=10.0, blur_ksize=9, use_subject_tracking=True,
                    use_floating_window=True, suspend_flag=threading.Event(), cancel_flag=threading.Event(),
                    zero_parallax_strength=0.01, auto_crop_black_bars=True, preserve_original_aspect=preserve)
    lines = capsys.readouterr().out.splitlines()
    ca, cb = cv2.VideoCapture(rgb), cv2.VideoCapture(dep)
    decoded = []
    while True:
        ok1, f = ca.read()
        ok2, d = cb.read()
        if not (ok1 and ok2):
            break
        decoded.append((f, d))
    t0, b0 = A.detect_black_bars(decoded[0][0])
    assert f"Auto-crop: Top {t0}px | Bottom {b0}px" in lines
    per = [ln for ln in lines if ln.startswith("🔪")]
    assert per == [f"🔪 Cropping top: {t}px, bottom: {b}px" for t, b in (A.detect_black_bars(f) for f, _ in decoded[1:])]
    ow, oh = (w, h - t0 - b0) if preserve else (None, None)
    assert sizes == [(2 * w, h - t0 - b0) if preserve else (w, h)]
    rp = R.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, fmt, 16 / 9, 0.0, 10.0, 9, True, True,
                              zero_parallax_strength=0.01, preserve_original_aspect=preserve, original_video_width=ow,
                              original_video_height=oh, auto_crop_black_bars=True)
    R.reset_temporal_state()  # the render started from fresh module singletons too
    expected = [R.render_frame(f, d, rp) for f, d in decoded[1:]]
    R.reset_temporal_state()  # leave the process-wide context as a fresh process has it
    assert len(written) == len(expected) == n - 1
    for k, (a, b) in enumerate(zip(written, expected)):
        assert np.array_equal(a, b), k
    cap = cv2.VideoCapture(out)
    frames = 0
    while cap.read()[0]:
        frames += 1
    assert frames == n - 1
