"""CPU: the float64 restatements of tests/dibr_kernel_refs.py against oracle/dibr.py.  Each restatement is fed the
oracle's intermediates and must reproduce the oracle's next intermediate: floats within the bound it states (which
covers the fp32 roundings of the oracle as well), u8 outputs inside their byte intervals, and those intervals a single
byte except where the float64 value lies within 1e-6 of a byte boundary."""
import numpy as np
import pytest

from oracle import dibr as O
from tests import dibr_kernel_refs as K
from visiondepth3d_b200.synth import synth_frame

F32 = np.float32


def _ps(w, h, kind, i=1, **kw):
    fr, dp = synth_frame(i, w, h, kind)
    ft, dt = O.bgr_to_rgb01(fr), O.depth_bgr_to_01(dp)
    p = O.ShiftParams(**kw)
    gs = O.GlobalState()
    left, right, final, parts = O.pixel_shift(gs, ft, dt, w, h, p, return_parts=True)
    return ft, dt, p, left, right, final, parts


def within(ref, bound, got, what, slack=4.0):
    err = np.abs(K.f64(got) - ref)
    tol = slack * bound + 4 * K.U * np.abs(ref) + 1e-30
    r = float((err / tol).max())
    print(f"[dibr-refs] {what}: worst err / tol = {r:.3f}")
    assert r <= 1.0, (what, r)


def inside(lo, hi, got, ref, what):
    """got inside [lo, hi]; and equal to the truncation of the float64 value except within 1e-6 of a byte boundary"""
    got = got.astype(np.int64)
    assert ((got >= lo) & (got <= hi)).all(), (what, int(((got < lo) | (got > hi)).sum()))
    t = np.clip(ref, 0, 1) * 255
    near = np.abs(t - np.rint(t)) < 255e-6
    off = (got != np.floor(t).astype(np.int64)) & ~near
    print(f"[dibr-refs] {what}: interval width > 0 on {float((hi > lo).mean()):.5f}, mismatches {int(off.sum())}")
    assert not off.any(), (what, int(off.sum()))


@pytest.mark.parametrize("kind", ["natural", "smooth"])
def test_ingest_temporal_normalize(kind):
    fr, dp = synth_frame(2, 200, 120, kind)
    (cur, cb), (rgb, rb) = K.ingest(fr, dp, (10, 6, 180, 100), 96, 54)
    dt = O.depth_bgr_to_01(dp)[:, 6:106, 10:190]
    ft = O.bgr_to_rgb01(fr)[:, 6:106, 10:190]
    ocur = O.resize_bilinear(dt, 54, 96)[0]
    within(cur, cb, ocur, "ingest depth resize")
    within(rgb, rb, O.resize_bilinear(ft, 54, 96), "ingest rgb resize")
    cs = O.ClipState()
    t0 = O.temporal_smooth(cs, ocur[None], 0.5)[0].copy()
    v, b = K.temporal(None, K.f64(ocur), np.zeros_like(cb), False)
    within(v, b, t0, "temporal, first frame")
    nxt = (ocur * F32(0.7)).astype(F32)
    t1 = O.temporal_smooth(cs, nxt[None], 0.5)[0]
    v, b = K.temporal(t0, K.f64(nxt), np.zeros_like(cb), True)
    within(v, b, t1, "temporal")
    gs = O.GlobalState()
    dn = O.percentile_normalize(gs, t1[None])[0]
    lo, _ = K.quantile32(np.clip(t1, 0, 1), 0.02)
    hi, _ = K.quantile32(np.clip(t1, 0, 1), 0.98)
    assert lo == O.quantile32(np.clip(t1, 0, 1), 0.02) and hi == O.quantile32(np.clip(t1, 0, 1), 0.98)
    flat, n_lo, den, plo, phi = K.pct_scalars(lo, hi, 0, 0, 0)
    assert (flat, plo, phi) == (0, gs.pct_lo, gs.pct_hi)
    v, b = K.normalize(t1, 0, n_lo, den)
    within(v, b, dn, "normalize")
    t2 = (t1 * F32(0.9)).astype(F32)   # the EMA step of a second frame
    O.percentile_normalize(gs, t2[None])
    lo2, hi2 = K.quantile32(np.clip(t2, 0, 1), 0.02)[0], K.quantile32(np.clip(t2, 0, 1), 0.98)[0]
    flat, n_lo, den, plo, phi = K.pct_scalars(lo2, hi2, 1, plo, phi)
    assert (flat, plo, phi) == (0, gs.pct_lo, gs.pct_hi)
    assert K.pct_scalars(F32(0.5), F32(0.5), 1, plo, phi)[0] == 1


@pytest.mark.parametrize("gamma", [0.85, 0.5, 1.3])
def test_pop_shape_and_quantiles(gamma):
    ft, dt, p, *_ = _ps(160, 90, "natural", depth_pop_gamma=gamma)
    d = O.resize_bilinear(dt, 90, 160)
    d0 = np.clip(O.curvature(d, 0.08), F32(0), F32(1)).astype(F32)
    xs, ys = O.linspace32(160), O.linspace32(90)
    assert np.array_equal(K.d0_plane(dt[0], 90, 160, xs, ys), d0[0])
    subj = O.subject_depth(d0)
    shaped, lo, hi = O.shape_for_pop(d0, subj, p)
    qlo, (a, b, w) = K.quantile32(d0, p.depth_stretch_lo)
    qhi, _ = K.quantile32(d0, p.depth_stretch_hi)
    assert qlo == lo and qhi == hi
    assert a == np.sort(d0.ravel())[K.quantile_rank(p.depth_stretch_lo, d0.size)[0]]
    den = F32(F32(hi - lo) + F32(1e-6))
    ss = F32(min(max(F32(F32(F32(min(max(subj, 0), 1)) - lo) / den), F32(0)), F32(1)))
    v, bnd = K.pop_shape(d0[0], 0, lo, den, ss, p.depth_pop_mid, gamma)
    within(v, bnd, shaped[0], f"pop shaping gamma {gamma}")


@pytest.mark.parametrize("kw", [dict(), dict(enable_edge_masking=False), dict(use_subject_tracking=False),
                                dict(convergence_strength=0.4), dict(max_pixel_shift_percent=0.002),
                                dict(feather_strength=40.0)])
def test_shift_map(kw):
    ft, dt, p, left, right, final, parts = _ps(160, 90, "natural", **kw)
    d = parts["d_shaped"][0]
    half = 80.0
    fs = dict(c_fg=p.fg_shift, c_fgm=p.fg_pop_multiplier, c_mg=p.mg_shift, c_bg=p.bg_shift, c_bgm=p.bg_push_multiplier,
              c_mid=p.depth_pop_mid, c_pb=p.parallax_balance, c_half=half, use_zpo=int(p.use_subject_tracking),
              c_zpo=parts["zpo"], c_max=(160 * p.max_pixel_shift_percent) / half,
              use_conv=int(p.convergence_strength != 0.0), c_conv=0.0)
    if fs["use_conv"]:
        conv = float(F32(O.subject_depth(parts["d_shaped"]) * F32(p.convergence_strength)))
        fs["c_conv"] = conv / half
    ms = float(np.clip(p.feather_strength / 10.0, 0.05, 0.3))
    fs["c_m1"], fs["c_m2"] = 1.0 - ms, ms
    v, b = K.shift_map(d, fs, p.enable_edge_masking, p.feather_strength)
    within(v, b, final[0], f"shift map {kw}")


@pytest.mark.parametrize("k", [0, 1, 3, 5, 7, 9])
@pytest.mark.parametrize("kind", ["natural", "noise"])
def test_render_eyes(k, kind):
    kw = dict(blur_ksize=k, enable_feathering=k > 0, feather_strength=10.0)
    if not k:
        kw["blur_ksize"] = 1
    ft, dt, p, left, right, final, parts = _ps(128, 72, kind, **kw)
    xs, ys = O.linspace32(128), O.linspace32(72)
    for sign, bgr, f in ((1, left, parts["left_f"]), (-1, right, parts["right_f"])):
        v, b, ex = K.eye_float(ft, xs, ys, final[0], parts["d_shaped"][0], k, p.feather_strength, sign)
        within(v, b, f, f"eye K={k} sign {sign}")
        known = ~np.isnan(ex)
        assert np.array_equal(ex[known], K.f64(f)[known]), f"eye K={k}: fp32 restatement"
        lo, hi = K.trunc_interval(v, b, ex)
        inside(lo, hi, bgr[..., ::-1].transpose(2, 0, 1), v, f"eye bytes K={k} sign {sign}")


@pytest.mark.parametrize("sat,con,bri", [(1.0, 1.0, 0.0), (1.3, 0.8, 0.05), (0.6, 1.2, -0.04)])
def test_grade(sat, con, bri):
    rng = np.random.default_rng(3)
    eye = rng.integers(0, 256, (3, 64, 80)).astype(np.int64)
    lo, hi = K.grade_interval(eye, eye, sat, con, bri)
    ref = O.color_grade(O.bgr_to_rgb01(eye.transpose(1, 2, 0)[..., ::-1].astype(np.uint8)), sat, con, bri)
    got = O.rgb01_to_bgr8(ref)[..., ::-1].transpose(2, 0, 1)
    v = K.grade(K.lut(eye), sat, con, bri)
    inside(lo, hi, got, np.clip(v, 0, 1), f"grade {sat} {con} {bri}")


@pytest.mark.parametrize("factor", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("side", [1, 2])
def test_bars_sharpen_area(factor, side):
    rng = np.random.default_rng(5)
    eye = rng.integers(0, 256, (40, 66, 3)).astype(np.uint8)
    barred = K.bars(eye, side, 7)
    assert np.array_equal(barred, O.side_mask(eye, "right" if side == 1 else "left", 7))
    lo, hi = K.sharpen_interval(barred, barred, factor)
    ref = O.sharpen(barred, factor)
    assert ((ref >= lo) & (ref <= hi)).all()
    assert (lo == hi).mean() >= 0.999, factor
    a, b = K.area2_interval(ref, ref)
    assert np.array_equal(a, b) and np.array_equal(a, O.resize_area_int(ref, 33, 40))

