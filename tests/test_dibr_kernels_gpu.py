"""GPU: each kernel of the fast DIBR path (csrc/dibr_fast.cu: k_stats, k_shift_fast, k_render) on its own, against
the float64 restatements of tests/dibr_kernel_refs.py (pinned to oracle/dibr.py in tests/test_dibr_kernel_refs_cpu.py).

After a frame, vd3d_get_buffer reads back the buffers of the render context and ONE kernel is recomputed from the
inputs the device itself stored for it, so the error budget is one kernel's:
  * k_stats: the ingest resizes (tdf's input, rgb_s, frameB) from the u8 frame, the temporal filter from the previous
    frame's tdf and DevState, the normalisation from tdf and the FrameScalars, the pop shaping from the d0 plane (rebuilt
    bit for bit from dn / the input depth: k_stats shapes it in place), and the radix-select percentiles: the
    interpolated quantiles must be torch.lerp of the exact order statistics of the device's own plane (np.partition).
  * k_shift_fast: the shift map and edge-mask suppression from d and the FrameScalars.
  * k_render: the eyes / the packed SBS frame from shift, d, the linspace axes and the colour source.
Floats are gated by the bounds dibr_kernel_refs derives (printed as "observed / bound", 1.0 = at the bound); bytes by
intervals: exact where the float64 value is farther than its bound from a byte boundary, else either neighbour
("ambiguous"), carried through the colour grade, bars, sharpen and 2:1 INTER_AREA.  The ambiguous fraction is printed
and gated so that a loose bound cannot make a check vacuous.  The gates are not derived: they were set per shape from the
first H100 runs.  Measured there: 0.04 % at the 1080p Half-SBS bench shape, 5.9 % at 4K (a smoother field: longer runs
of equal pixels), up to 15.1 % on the small natural frames and 5.3 % on noise.  The natural set's u8 fields hold runs of equal pixels, and the warped value between equal pixels,
blended with an equal original, is exactly k / 255: a byte boundary, where only the last bit of the blend weight decides.
A feather_strength of 1000 scales the mask's error 1000-fold: that case checks k_shift_fast and is not gated.

Reachable k_render instances (K, SRC, FUSE), K in {0, 1, 3, 5, 7, 9} (0 = feathering off); SRC 0 u8 frame, 1 RGBx
float4 plane, 2 planar f32; FUSE 0 eyes, 1 identity-fit SBS pack, 2 2:1 Half-SBS pack:
    FUSE 0, SRC 2   pixel_shift_cuda
    FUSE 0, SRC 0   frame loop, eyes left for the post kernel (anaglyph / interlaced / DOF), frame used as is
    FUSE 0, SRC 1   the same with a resized (or cropped) frame
    FUSE 1, SRC 0   Full-SBS whose eyes are the frame's size (identity ingest)
    FUSE 1, SRC 1   Full-SBS with a resized / cropped frame
    FUSE 2, SRC 1   Half-SBS (the eye is always half the warp width, so never the identity ingest)
Each case asserts the triple the dispatch recorded for its launch; test_every_instance_is_covered checks that the case
table reaches all 36.

The quantiled planes include ones that are flat (clamp01(tdf) constant: pct_flat; d0 saturated at 1: st_flat) and ones
tied at the selected rank (two-valued depth; d0 clamped to exactly 0 / 1 over more than 5 % of the pixels); each case
asserts the flatness flags and tie counts it was built for.

At 4K the frame-loop case recomputes every kernel with graph replay (the frame bench.py times); eagerly it recomputes
k_stats and k_shift_fast only (the float64 k_render recomputation alone takes over a minute at 4K)."""
import ctypes as C

import numpy as np
import pytest

from tests import dibr_kernel_refs as K
from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu

KS = [0, 1, 3, 5, 7, 9]
AMBIGUOUS = {"natural": 0.16, "noise": 0.06}   # small frames; the bench shapes carry their own gate
F32 = np.float32

FS = np.dtype([("q_lo", "f4"), ("q_hi", "f4"), ("pct_flat", "i4"), ("n_lo", "f4"), ("n_den", "f4"),
               ("sum", "f8"), ("sumsq", "f8"), ("mad_sum", "f8"), ("dyn", "f8"), ("fg", "f8"), ("mg", "f8"),
               ("bg", "f8"), ("motion", "f8"), ("focal", "f8"), ("subj_norm", "f4"), ("stable_zero", "f8"),
               ("bar_width", "i4"), ("bar_side", "i4"), ("subj_raw", "f4"), ("st_lo", "f4"), ("st_hi", "f4"),
               ("st_den", "f4"), ("st_subj", "f4"), ("st_flat", "i4"), ("subj", "f4"), ("zpo", "f8")]
              + [(n, "f4") for n in ("c_fg", "c_fgm", "c_mg", "c_bg", "c_bgm", "c_pb", "c_half", "c_mid", "c_gamma",
                                     "c_zpo", "c_max", "c_conv", "c_m1", "c_m2")]
              + [("use_zpo", "i4"), ("use_conv", "i4"), ("bars", "u4", (2,))], align=True)
ST = np.dtype([("pct_lo", "f4"), ("pct_hi", "f4"), ("pct_init", "i4"), ("conv_val", "f8"), ("conv_init", "i4"),
               ("fw_prev", "f8"), ("fw_count", "i4"), ("bar_prev", "i4"), ("tdf_init", "i4"), ("sm_fg", "f8"),
               ("sm_mg", "f8"), ("sm_bg", "f8"), ("sm_init", "i4"), ("focal", "f8"), ("focal_alpha", "f8"),
               ("focal_init", "i4"), ("have_prev_depth", "i4"), ("dn_cur", "i4")], align=True)


@pytest.fixture(scope="module")
def ctx():
    from visiondepth3d_b200 import _lib
    c = _lib.Context()
    yield c
    c.close()


def buf(ctx, name, shape, dtype=np.float32):
    out = np.empty(shape, dtype)
    ctx.check(ctx.lib.vd3d_get_buffer(ctx.h, name.encode(), out.ctypes.data, out.nbytes))
    return out


def rec(ctx, name, dt):
    r = np.zeros(1, dt)
    ctx.check(ctx.lib.vd3d_get_buffer(ctx.h, name.encode(), r.ctypes.data, dt.itemsize))
    return {k: (r[k][0] if r[k].ndim == 1 else r[k][0].copy()) for k in dt.names}


def triple(ctx):
    return tuple(int(v) for v in buf(ctx, "render", (3,), np.int32))


def report(what, dev, ref, bound):
    err = np.abs(K.f64(dev) - ref)
    r = err / (bound * (1 + 2.0 ** -20) + 1e-300)   # a bound of one rounding may be met exactly
    i = int(np.argmax(r))
    print(f"[dibr-kernels] {what}: observed / bound = {r.flat[i]:.3f} (worst abs err {err.flat[i]:.3e})")
    assert np.isfinite(r.flat[i]) and r.flat[i] <= 1.0, (what, float(r.flat[i]), np.unravel_index(i, r.shape))


def exact_quantile(dev, plane, q, what):
    """the device's interpolated quantile is torch.lerp (same fp32 op sequence, -fmad=false) of the exact order
    statistics of its own plane: bit for bit.  Returns how many elements tie with the selected value."""
    ref = K.quantile32(plane, q)[0]
    ties = K.ties_at(plane, q)
    print(f"[dibr-kernels] {what}: device {float(dev)!r} reference {float(ref)!r}, {ties} elements tied at the rank")
    assert np.asarray(dev, F32).view(np.int32) == np.asarray(ref, F32).view(np.int32), what
    return ties


def bytes_in(dev, lo, hi, what):
    dev = dev.astype(np.int64)
    bad = (dev < lo) | (dev > hi)
    amb = float((hi > lo).mean())
    print(f"[dibr-kernels] {what}: bytes outside their interval {int(bad.sum())} of {dev.size}, ambiguous {amb:.5f}")
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:5].tolist())
    return amb


# ----------------------------------------------------------------------------------------------------------------------
def check_stats_tail(ctx, core, H, W, fs, mid=0.5, gamma=0.85, tag="", st_flat=0, min_ties=1):
    """d0 quantiles, pop shaping; returns d (device)"""
    xs, ys = buf(ctx, "xs", (W,)), buf(ctx, "ys", (H,))
    d0 = K.d0_plane(core, H, W, xs, ys)
    for q, key in ((0.05, "st_lo"), (0.95, "st_hi")):
        ties = exact_quantile(fs[key], d0, q, f"{tag} k_stats quantile {q} of d0")
        assert ties >= min_ties, (tag, q, ties)
    assert fs["st_flat"] == st_flat, tag
    d = buf(ctx, "d", (H, W))
    ref, b = K.pop_shape(d0, fs["st_flat"], fs["st_lo"], fs["st_den"], fs["st_subj"], mid, gamma)
    report(f"{tag} k_stats pop shaping d", d, ref, b)
    return xs, ys, d


def check_shift(ctx, d, H, W, fs, edge, feather, tag=""):
    shift = buf(ctx, "shift", (H, W))
    ref, b = K.shift_map(d, fs, edge, feather)
    report(f"{tag} k_shift_fast shift", shift, ref, b)
    return shift


def eye_intervals(src, xs, ys, shift, d, k, feather, grade=None):
    """[2][3, H, W] RGB byte intervals of the two eyes"""
    out = []
    for sign in (1, -1):
        v, b, ex = K.eye_float(src, xs, ys, shift, d, k, feather, sign)
        lo, hi = K.trunc_interval(v, b, ex)
        if grade is not None:
            lo, hi = K.grade_interval(lo, hi, *grade)
        out.append((lo, hi))
    return out


def to_bgr(a):
    return a[::-1].transpose(1, 2, 0)


# ----------------------------------------------------------------------------------------------------------------------
# the frame loop: k_stats (loop mode) -> k_shift_fast -> k_render
# ----------------------------------------------------------------------------------------------------------------------
def loop_case(name, sw, sh, fmt, aspect, k, kind="natural", shifts=(4.5, -1.5, -6.0), grade=(1.2, 0.9, 0.03),
              sharp=0.2, out_h=None, depth="synth", bar_side=None, gate=None):
    """depth: "synth" (the content's own), "flat" (one gray level: clamp01(tdf) constant, pct_flat) or "two-valued"
    (two gray levels, each on more than 2 % of the pixels: clamp01(tdf) tied at the 0.02 / 0.98 ranks).  bar_side: the
    floating-window side the shifts are chosen to produce (1 right, 2 left)."""
    return pytest.param(dict(sw=sw, sh=sh, fmt=fmt, aspect=aspect, k=k, kind=kind, shifts=shifts, grade=grade,
                             sharp=sharp, out_h=out_h, depth=depth, bar_side=bar_side,
                             gate=gate if gate is not None else AMBIGUOUS[kind]), id=f"{name}-K{k}")


LOOP = []
for i, k in enumerate(KS):
    LOOP.append(loop_case("halfsbs-322x180", 322, 180, "Half-SBS", 322 / 180, k, sharp=[0.0, 0.2, 1.0][i % 3]))
    LOOP.append(loop_case("fullsbs-ident-65x33", 65, 33, "Full-SBS", 65 / 33, k, kind=["natural", "noise"][i % 2]))
    LOOP.append(loop_case("fullsbs-crop-63x31", 63, 31, "Full-SBS", 16 / 9, k))
    LOOP.append(loop_case("anaglyph-ident-321x180", 321, 180, "Red-Cyan Anaglyph", 321 / 180, k))
    LOOP.append(loop_case("anaglyph-crop-320x240", 320, 240, "Red-Cyan Anaglyph", 16 / 9, k, kind="noise"))
LOOP += [
    loop_case("bars-right-320x180", 320, 180, "Half-SBS", 16 / 9, 5, shifts=(-30.0, 10.0, 40.0), bar_side=1),
    loop_case("bars-left-320x180", 320, 180, "Half-SBS", 16 / 9, 3, shifts=(45.0, -15.0, -60.0), bar_side=2),
    loop_case("flat-depth-322x180", 322, 180, "Half-SBS", 322 / 180, 5, depth="flat"),
    loop_case("two-valued-depth-322x180", 322, 180, "Half-SBS", 322 / 180, 5, depth="two-valued"),
    loop_case("two-valued-depth-65x33", 65, 33, "Full-SBS", 65 / 33, 9, depth="two-valued"),
    loop_case("halfsbs-1080p", 1920, 1080, "Half-SBS", 16 / 9, 9, out_h=1080, gate=0.002),
    loop_case("fullsbs-4k", 3840, 2160, "Full-SBS", 16 / 9, 9, grade=(1.0, 1.0, 0.0), gate=0.08),
]


def loop_params(c):
    from visiondepth3d_b200 import render_3d as R
    k = c["k"]
    out_h = c["out_h"] or c["sh"]
    return R.make_render_params(out_h * 16 // 9, out_h, *c["shifts"], c["sharp"], c["fmt"], c["aspect"], 0.0,
                                10.0, k if k else 1, True, True, preserve_original_aspect=c["out_h"] is None,
                                zero_parallax_strength=0.01, enable_feathering=k > 0, color_saturation=c["grade"][0],
                                color_contrast=c["grade"][1], color_brightness=c["grade"][2])


def loop_expected(c):
    """(K, SRC, FUSE) a frame-loop case must launch: the u8 frame itself when the ingest is the identity"""
    from visiondepth3d_b200 import render_3d as R
    pl = R.plan_sizes(c["sw"], c["sh"], loop_params(c))
    ident = (pl.target_eye_w, pl.target_eye_h) == (pl.crop_w, pl.crop_h) == (pl.resized_width, pl.resized_height)
    return c["k"], 0 if ident else 1, {"Half-SBS": 2, "Full-SBS": 1}.get(c["fmt"], 0)


def loop_frame(i, c):
    fr, dp = synth_frame(i, c["sw"], c["sh"], c["kind"])
    if c["depth"] == "flat":
        dp = np.full_like(dp, 128)
    elif c["depth"] == "two-valued":
        y, x = np.mgrid[0:c["sh"], 0:c["sw"]]
        dp = np.ascontiguousarray(np.repeat(np.where((x // 5 + y // 3) % 3 == 0, 40, 200).astype(np.uint8)[..., None],
                                            3, axis=2))
    return fr, dp


def run_clip(ctx, rp, frames, sh, sw):
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R
    n = len(frames)
    pl = R.plan_sizes(sw, sh, rp)
    outs = [np.empty(R.output_shape(rp, pl), np.uint8) for _ in range(n)]
    fp = (C.c_void_p * n)(*[f.ctypes.data for f, _ in frames])
    dp = (C.c_void_p * n)(*[d.ctypes.data for _, d in frames])
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    ctx.check(ctx.lib.vd3d_render_clip(ctx.h, n, fp, dp, 3, sh, sw, C.byref(rp), op, _lib.MEM_HOST, None))
    return outs, pl


@pytest.mark.parametrize("graphs", [0, 1])
@pytest.mark.parametrize("case", LOOP)
def test_frame_loop_kernels(ctx, case, graphs):
    from visiondepth3d_b200 import render_3d as R
    c = case
    sw, sh, k = c["sw"], c["sh"], c["k"]
    rp = loop_params(c)
    ctx.check(ctx.lib.vd3d_set_graphs(ctx.h, graphs))
    ctx.reset()
    frames = [loop_frame(i, c) for i in range(4)]
    run_clip(ctx, rp, frames[:3], sh, sw)                     # the first three frames run eagerly either way
    pl = R.plan_sizes(sw, sh, rp)
    tw, th, W, H = pl.target_eye_w, pl.target_eye_h, pl.resized_width, pl.resized_height
    st0 = rec(ctx, "st", ST)
    tdf_prev = buf(ctx, "tdf", (th, tw))
    outs, _ = run_clip(ctx, rp, frames[3:], sh, sw)           # with graphs on: replayed from the captured graph
    out = outs[0]
    fr, dp = frames[3]
    fs, st = rec(ctx, "fs", FS), rec(ctx, "st", ST)
    tri = triple(ctx)
    tag = f"{sw}x{sh} {c['fmt']} {c['depth']} depth K={k} graphs={graphs}"
    assert tri == loop_expected(c), (tag, tri)
    _, src_kind, fuse = tri
    ident = src_kind == 0

    # ---- k_stats: ingest + TemporalDepthFilter
    crop = (pl.crop_x0, pl.crop_y0, pl.crop_w, pl.crop_h)
    (cur, cb), (rgb, rb) = K.ingest(fr, dp, crop, tw, th)
    tdf = buf(ctx, "tdf", (th, tw))
    ref, b = K.temporal(tdf_prev, cur, cb, st0["tdf_init"])
    assert st0["tdf_init"] == 1
    report(f"{tag} k_stats temporal filter tdf", tdf, ref, b)
    src = None
    if not ident:
        rgb_s = buf(ctx, "rgb_s", (th, tw, 4))
        report(f"{tag} k_stats ingest rgb_s", rgb_s[..., :3].transpose(2, 0, 1), rgb, rb)
        src = rgb_s[..., :3].transpose(2, 0, 1)
        if (W, H) != (tw, th):
            frameB = buf(ctx, "frameB", (H, W, 4))
            ref, b = K.resize_bilinear(src, H, W)
            report(f"{tag} k_stats resize frameB", frameB[..., :3].transpose(2, 0, 1), ref, b)
            src = frameB[..., :3].transpose(2, 0, 1)
    else:
        src = K.lut(fr[pl.crop_y0:pl.crop_y0 + H, pl.crop_x0:pl.crop_x0 + W, ::-1].transpose(2, 0, 1))
    # ---- k_stats: percentiles of clamp01(tdf), normalisation
    ties = [exact_quantile(fs[key], np.clip(tdf, 0, 1), q, f"{tag} k_stats quantile {q} of tdf")
            for q, key in ((0.02, "q_lo"), (0.98, "q_hi"))]
    if c["depth"] != "synth":   # the plane is flat / tied at the rank, as built
        assert min(ties) > 0.02 * tdf.size, (tag, ties)
    # DepthPercentileEMA from the previous frame's DevState and the exact quantiles
    flat, n_lo, n_den, plo, phi = K.pct_scalars(fs["q_lo"], fs["q_hi"], st0["pct_init"], st0["pct_lo"], st0["pct_hi"])
    assert flat == (c["depth"] == "flat") and fs["pct_flat"] == flat, tag
    assert (fs["n_lo"], fs["n_den"], st["pct_lo"], st["pct_hi"]) == (n_lo, n_den, plo, phi), tag
    dn = buf(ctx, "dn", (th, tw))
    ref, b = K.normalize(tdf, flat, n_lo, n_den)
    report(f"{tag} k_stats normalised depth dn", dn, ref, b)
    # ---- k_stats: d0 quantiles + pop shaping; k_shift_fast
    xs, ys, d = check_stats_tail(ctx, dn, H, W, fs, tag=tag)
    shift = check_shift(ctx, d, H, W, fs, True, 10.0, tag=tag)
    if sw == 3840 and not graphs:
        return   # see the module docstring: k_render at 4K is recomputed on the graph-replayed frame
    # ---- k_render
    eyes = eye_intervals(src, xs, ys, shift, d, k, 10.0, grade=c["grade"])
    amb = 0.0
    if fuse == 0:
        for (lo, hi), name in zip(eyes, ("eyeL", "eyeR")):
            amb = max(amb, bytes_in(buf(ctx, name, (H, W, 3), np.uint8), to_bgr(lo), to_bgr(hi), f"{tag} k_render {name}"))
    else:
        side, bw = int(fs["bar_side"]), int(fs["bar_width"])
        if c["bar_side"]:
            assert side == c["bar_side"] and bw > 1, (tag, side, bw)
        pw = pl.per_eye_w
        for e, (lo, hi) in enumerate(eyes):
            amb = max(amb, float((hi > lo).mean()))
            lo, hi = K.bars(to_bgr(lo), side, bw), K.bars(to_bgr(hi), side, bw)
            lo, hi = K.sharpen_interval(lo, hi, c["sharp"])
            if fuse == 2:
                lo, hi = K.area2_interval(lo, hi)
            got = out[:, e * pw:(e + 1) * pw]
            bytes_in(got, lo, hi, f"{tag} k_render packed eye {e}")
            if bw > 1:   # columns whose whole sharpen (and 2:1) footprint lies in the bar are exactly 0
                f = 1 if fuse == 1 else 2
                cols = np.arange(pw)
                inbar = (cols * f - 1 >= W - bw) & (cols * f + f <= W) if side == 1 else (cols * f + f < bw)
                assert inbar.any() and not got[:, inbar].any(), (tag, side, bw)
    print(f"[dibr-kernels] {tag}: ambiguous eye bytes {amb:.5f} (gate {c['gate']})")
    assert amb <= c["gate"], (tag, amb)


# ----------------------------------------------------------------------------------------------------------------------
# pixel_shift_cuda: k_stats (from d0) -> k_shift_fast -> k_render<K, 2, 0>
# ----------------------------------------------------------------------------------------------------------------------
def depth_plane(kind, h, w):
    """natural: the synthetic depth; saturated: 1.5 everywhere, so d0 = clamp01(d + curvature) is 1 everywhere and flat
    (st_flat); binary: 0 / 1 in stripes, so d0 clamps to exactly 0 (outside the unit ellipse) and to exactly 1 (inside)
    on far more than 5 % of the pixels each: the 0.05 and 0.95 selects are tied at their ranks."""
    fr, dp = synth_frame(1, w, h, "natural")
    g = dp[..., 0].astype(np.float32) / np.float32(255)
    if kind == "saturated":
        g[:] = np.float32(1.5)
    elif kind == "binary":
        g = np.where((np.arange(w)[None] // 3 + np.arange(h)[:, None] // 2) % 2 == 0, np.float32(0), np.float32(1))
    return np.ascontiguousarray(g[None].astype(np.float32))


PS = []
for i, k in enumerate(KS):
    PS.append(pytest.param(dict(w=[65, 63, 321][i % 3], h=[33, 31, 180][i % 3], k=k, depth="natural", kw={}),
                           id=f"K{k}"))
PS += [
    pytest.param(dict(w=64, h=48, k=9, depth="natural", kw=dict(enable_edge_masking=False)), id="edge-off"),
    pytest.param(dict(w=64, h=48, k=5, depth="natural", kw=dict(use_subject_tracking=False)), id="zpo-off"),
    pytest.param(dict(w=64, h=48, k=5, depth="natural", kw=dict(convergence_strength=0.4)), id="conv-dyn"),
    pytest.param(dict(w=64, h=48, k=5, depth="natural",
                      kw=dict(convergence_strength=0.3, enable_dynamic_convergence=False)), id="conv-fixed"),
    pytest.param(dict(w=64, h=48, k=3, depth="natural", kw=dict(max_pixel_shift_percent=0.001)), id="clamp"),
    pytest.param(dict(w=200, h=120, k=7, depth="natural", kw=dict(feather_strength=1000.0)), id="feather-overflow"),
    pytest.param(dict(w=160, h=90, k=3, depth="natural", kw={}, iw=100, ih=60), id="resized-input"),
    pytest.param(dict(w=96, h=54, k=9, depth="saturated", kw={}), id="saturated-flat"),
    pytest.param(dict(w=96, h=54, k=9, depth="binary", kw={}), id="binary-tied"),
    pytest.param(dict(w=321, h=180, k=5, depth="binary", kw={}), id="binary-tied-321x180"),
]


@pytest.mark.parametrize("case", PS)
def test_pixel_shift_kernels(ctx, case):
    from oracle import dibr as O
    w, h, k = case["w"], case["h"], case["k"]
    iw, ih = case.get("iw", w), case.get("ih", h)
    fr, _ = synth_frame(2, iw, ih, "natural")
    ft = O.bgr_to_rgb01(fr)
    dt = depth_plane(case["depth"], ih, iw)
    kw = dict(blur_ksize=k if k else 1, enable_feathering=k > 0, feather_strength=10.0, zero_parallax_strength=0.01)
    kw.update(case["kw"])
    ctx.reset()
    from visiondepth3d_b200 import _lib
    p = _lib.ShiftParams(4.5, -1.5, -6.0, kw["blur_ksize"], kw["feather_strength"], kw.get("max_pixel_shift_percent", 0.02),
                         0.8, kw["zero_parallax_strength"], int(kw.get("use_subject_tracking", True)), 1,
                         int(kw["enable_feathering"]), int(kw.get("enable_edge_masking", True)),
                         kw.get("convergence_strength", 0.0), int(kw.get("enable_dynamic_convergence", True)),
                         0.85, 0.5, 0.05, 0.95, 1.2, 1.1, 1.0)
    left = np.empty((h, w, 3), np.uint8)
    right = np.empty_like(left)
    info = _lib.FrameInfo()
    ctx.check(ctx.lib.vd3d_pixel_shift(ctx.h, ft.ctypes.data, dt.ctypes.data, ih, iw, w, h, C.byref(p),
                                       left.ctypes.data, right.ctypes.data, None, _lib.MEM_HOST, C.byref(info)))
    tri = triple(ctx)
    tag = f"pixel_shift {w}x{h} {case['depth']} K={k} {case['kw']}"
    assert tri == (k, 2, 0), (tag, tri)
    fs = rec(ctx, "fs", FS)
    flat = case["depth"] == "saturated"
    min_ties = {"saturated": w * h, "binary": w * h // 20}.get(case["depth"], 1)
    xs, ys, d = check_stats_tail(ctx, dt[0], h, w, fs, tag=tag, st_flat=int(flat), min_ties=min_ties)
    shift = check_shift(ctx, d, h, w, fs, p.enable_edge_masking, p.feather_strength, tag=tag)
    if case["kw"].get("max_pixel_shift_percent"):   # the +-c_max clamp acted: without it the map would differ
        free = dict(fs, c_max=1e30)
        assert not np.allclose(K.shift_map(d, free, p.enable_edge_masking, p.feather_strength)[0], shift), tag
    src = ft if (ih, iw) == (h, w) else buf(ctx, "frameB", (3, h, w))
    eyes = eye_intervals(src, xs, ys, shift, d, k, p.feather_strength)
    amb = max(bytes_in(left, to_bgr(eyes[0][0]), to_bgr(eyes[0][1]), f"{tag} k_render left"),
              bytes_in(right, to_bgr(eyes[1][0]), to_bgr(eyes[1][1]), f"{tag} k_render right"))
    print(f"[dibr-kernels] {tag}: ambiguous eye bytes {amb:.5f}")
    if case["depth"] == "natural" and p.feather_strength <= 10:
        assert amb <= AMBIGUOUS["natural"], (tag, amb)


def test_every_instance_is_covered():
    """the case table reaches the (K, SRC, FUSE) table of the module docstring, all 36 (each case asserts the triple
    its own launch recorded): pixel_shift_cuda always launches SRC 2, FUSE 0"""
    want = {(k, s, f) for k in KS for s, f in ((2, 0), (0, 0), (1, 0), (0, 1), (1, 1), (1, 2))}
    got = {loop_expected(p.values[0]) for p in LOOP} | {(p.values[0]["k"], 2, 0) for p in PS}
    assert got == want, sorted(want ^ got)
