"""GPU: kernel launches per frame of every frame path, pinned.

Context.launches (vd3d_launch_count) is what bench.py reports as gpu_launches.  The counts below are the kernels each
path enqueues per frame; a change that adds or drops a launch, or counts one it does not make, shows up here.  Every
count must also be the same whether the frame is launched eagerly or replayed from a CUDA graph.
"""
import ctypes as C

import numpy as np
import pytest

from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu

W, H = 320, 180
N = 4  # frames per measured vd3d_render_clip call
MODES = ["fast", "exact"]

# render parameters of each configuration -> launches per frame, by arithmetic mode.  k_render takes odd box sizes up
# to 9 only: an even blur_ksize runs the exact path's kernels in both modes.
CLIP = {
    "half_sbs": (dict(output_format="Half-SBS"), {"fast": 5, "exact": 41}),
    "full_sbs": (dict(output_format="Full-SBS", preserve_original_aspect=True), {"fast": 5, "exact": 40}),
    "anaglyph": (dict(output_format="Red-Cyan Anaglyph"), {"fast": 6, "exact": 40}),
    "dof": (dict(dof_strength=2.0), {"fast": 7, "exact": 42}),
    "even_ksize": (dict(blur_ksize=8), {"fast": 41, "exact": 41}),
}
ADVANCE = {"fast": 3, "exact": 37}
PIXEL_SHIFT = {"fast": 5, "exact": 23}
# vd3d_render_clip_depth over CLIP_DEPTH_FRAMES frames: (context launches, depth engine launches) by depth batch
CLIP_DEPTH_FRAMES = 8
CLIP_DEPTH = {1: (40, 1128), 4: (40, 624)}
# one eager infer_batch of the small random-init model of each depth family (the family tests' models): depth engine
# launches by batch size, pre- and post-process included
FAMILY_BATCH = {
    "da-v2": {1: 141, 4: 312},
    "da-metric": {1: 141, 4: 312},
    "dpt": {1: 93, 4: 252},
    "dpt-hybrid": {1: 240, 4: 858},
    "dpt-beit": {1: 93, 4: 252},
    "zoedepth-2": {1: 123, 4: 372},
    "zoedepth-1": {1: 122, 4: 368},
}


@pytest.fixture
def ctx():
    from visiondepth3d_b200 import _lib
    c = _lib.Context()
    yield c
    c.close()


def render_params(**kw):
    from visiondepth3d_b200 import render_3d as R
    a = dict(output_format="Half-SBS", dof_strength=0.0, blur_ksize=9)
    a.update(kw)
    return R.make_render_params(W, H, 4.5, -1.5, -6.0, 0.2, a.pop("output_format"), 16 / 9, a.pop("dof_strength"),
                                10.0, a.pop("blur_ksize"), True, True, zero_parallax_strength=0.01, **a)


def _outs(rp, n):
    from visiondepth3d_b200 import render_3d as R
    shape = R.output_shape(rp, R.plan_sizes(W, H, rp))
    outs = [np.empty(shape, dtype=np.uint8) for _ in range(n)]
    return outs, (C.c_void_p * n)(*[o.ctypes.data for o in outs])


def _set_graphs(ctx, graphs):
    ctx.check(ctx.lib.vd3d_set_graphs(ctx.h, graphs))


def clip_launches(ctx, rp, graphs):
    """Launches per frame of vd3d_render_clip, measured after a warm-up call (with graphs: captured and replayed)."""
    from visiondepth3d_b200 import _lib
    _set_graphs(ctx, graphs)
    ctx.reset()
    counts = []
    for first in (0, N):
        frames = [synth_frame(first + i, W, H, "natural") for i in range(N)]
        fp = (C.c_void_p * N)(*[f.ctypes.data for f, _ in frames])
        dp = (C.c_void_p * N)(*[d.ctypes.data for _, d in frames])
        outs, op = _outs(rp, N)
        l0 = ctx.launches
        ctx.check(ctx.lib.vd3d_render_clip(ctx.h, N, fp, dp, 3, H, W, C.byref(rp), op, _lib.MEM_HOST, None))
        counts.append(ctx.launches - l0)
    assert ctx.lib.vd3d_graphs_active(ctx.h) == graphs
    assert counts[1] % N == 0, counts
    return counts[1] // N


def advance_launches(ctx):
    """Launches of two consecutive vd3d_advance_state calls."""
    from visiondepth3d_b200 import render_3d as R
    rp = render_params()
    out = []
    for i in range(2):
        f, d = synth_frame(i, W, H, "natural")
        l0 = ctx.launches
        R.advance_state(f, d, rp, ctx=ctx)
        out.append(ctx.launches - l0)
    return out


def pixel_shift_launches(ctx):
    """Launches of two consecutive vd3d_pixel_shift calls."""
    from oracle import dibr as O
    from visiondepth3d_b200 import _lib
    f, d = synth_frame(0, W, H, "natural")
    rgb = np.ascontiguousarray(O.bgr_to_rgb01(f), dtype=np.float32)
    dep = np.ascontiguousarray(O.depth_bgr_to_01(d), dtype=np.float32)
    p = _lib.ShiftParams(4.5, -1.5, -6.0, 9, 10.0, 0.02, 0.8, 0.01, 1, 1, 1, 1, 0.0, 1, 0.85, 0.5, 0.05, 0.95, 1.2,
                         1.1, 1.0)
    left, right = np.empty((H, W, 3), np.uint8), np.empty((H, W, 3), np.uint8)
    out = []
    for _ in range(2):
        l0 = ctx.launches
        ctx.check(ctx.lib.vd3d_pixel_shift(ctx.h, rgb.ctypes.data, dep.ctypes.data, H, W, W, H, C.byref(p),
                                           left.ctypes.data, right.ctypes.data, None, _lib.MEM_HOST, None))
        out.append(ctx.launches - l0)
    return out


def depth_engine(ctx):
    """Small random-init Depth-Anything-V2-Small engine on ctx."""
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import hf_config
    torch.manual_seed(0)
    eng = DepthEngine("vits", 70, 126, ctx=ctx)
    eng.load_state_dict(DepthAnythingForDepthEstimation(hf_config("vits")).eval().state_dict())
    return eng


def clip_depth_launches(ctx, eng, batch, graphs):
    """(context, depth engine) launches of one vd3d_render_clip_depth call, after warm-up calls that take both engine
    instances through their eager batches and the frames through their eager, then captured, passes."""
    from visiondepth3d_b200 import _lib
    n = CLIP_DEPTH_FRAMES
    rp = render_params()
    frames = [synth_frame(i, W, H, "natural")[0] for i in range(n)]
    fp = (C.c_void_p * n)(*[f.ctypes.data for f in frames])
    outs, op = _outs(rp, n)
    ctx.check(ctx.lib.vd3d_set_depth_batch(ctx.h, batch))
    _set_graphs(ctx, graphs)
    for _ in range(4):
        ctx.reset()
        l0, d0 = ctx.launches, eng.launches
        ctx.check(ctx.lib.vd3d_render_clip_depth(ctx.h, eng.h, n, fp, H, W, C.byref(rp), op, _lib.MEM_HOST))
    assert ctx.lib.vd3d_graphs_active(ctx.h) == graphs
    return ctx.launches - l0, eng.launches - d0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(CLIP))
def test_render_clip_launches(ctx, case, mode):
    kw, want = CLIP[case]
    ctx.set_exact(mode == "exact")
    rp = render_params(**kw)
    assert clip_launches(ctx, rp, 0) == want[mode]
    assert clip_launches(ctx, rp, 1) == want[mode]


@pytest.mark.parametrize("mode", MODES)
def test_advance_state_launches(ctx, mode):
    ctx.set_exact(mode == "exact")
    assert advance_launches(ctx) == [ADVANCE[mode]] * 2


@pytest.mark.parametrize("mode", MODES)
def test_pixel_shift_launches(ctx, mode):
    ctx.set_exact(mode == "exact")
    assert pixel_shift_launches(ctx) == [PIXEL_SHIFT[mode]] * 2


@pytest.mark.parametrize("batch", [1, 4])
def test_render_clip_depth_launches(ctx, batch):
    eng = depth_engine(ctx)
    try:
        assert clip_depth_launches(ctx, eng, batch, 0) == CLIP_DEPTH[batch]
        assert clip_depth_launches(ctx, eng, batch, 1) == CLIP_DEPTH[batch]
    finally:
        eng.close()


def family_engine(name):
    """The small random-init model of a depth family on an engine of the size its family tests use."""
    from tests import da_family_oracle as DO
    from tests import dpt_beit_oracle as OB
    from tests import dpt_hybrid_oracle as OH
    from tests import dpt_oracle as OD
    from tests import zoedepth_oracle as ZO
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import da_spec
    proc128 = dict(size=(128, 128), resample=3, mean=(0.5,) * 3, std=(0.5,) * 3)
    if name == "da-v2":
        return depth_engine(None)
    if name == "da-metric":
        sd, spec = DO.random_model(da_spec("vits", head="metric", max_depth=20.0), seed=5)
        e = DepthEngine(spec, 70, 98)
    elif name == "dpt":
        sd, cfg = OD.random_model(small=True)
        e = DepthEngine(cfg, family="dpt", processor=proc128)
    elif name == "dpt-hybrid":
        sd, cfg = OH.random_model(small=True)
        e = DepthEngine(cfg, family="dpt-hybrid", processor=proc128)
    elif name == "dpt-beit":
        sd, cfg = OB.random_model(small=True, seed=3)
        e = DepthEngine(cfg, 64, 96, family="dpt-beit")
    else:
        sd, cfg = ZO.random_model(multi=name == "zoedepth-2", seed=3 if name == "zoedepth-2" else 4)
        e = DepthEngine(cfg, 64, 96, family="zoedepth")
    e.load_state_dict(sd)
    return e


@pytest.mark.parametrize("family", list(FAMILY_BATCH))
def test_depth_family_batch_launches(family):
    """Launches of one eager vd3d_depth_infer_batch per family and batch size, after a warm-up call."""
    e = family_engine(family)
    try:
        for batch, want in FAMILY_BATCH[family].items():
            frames = [synth_frame(i, W, H, "natural")[0] for i in range(batch)]
            e.infer_batch(frames, check_size=False)
            l0 = e.launches
            e.infer_batch(frames, check_size=False)
            assert e.launches - l0 == want, (family, batch)
    finally:
        e.close()
