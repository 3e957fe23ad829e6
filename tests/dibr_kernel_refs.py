"""TEST INFRASTRUCTURE: float64 restatements of what the fast DIBR kernels of csrc/dibr_fast.cu compute (k_stats,
k_shift_fast, k_render), following oracle/dibr.py op for op, each with the bound on how far the kernel's fp32 result may
lie from the float64 value when it is given the same fp32 inputs.

tests/test_dibr_kernel_refs_cpu.py pins every function here to oracle/dibr.py; tests/test_dibr_kernels_gpu.py compares
each kernel with them, fed the buffers the device itself stored for it (vd3d_get_buffer).

Error model.  U = 2^-24 is the unit roundoff of fp32: one correctly rounded op on a value v errs by at most U |v|.  The
kernels also use hardware approximations whose documented accuracy enters the bounds:
  * sqrt.approx.f32 (k_shift_fast): PTX ISA, "sqrt": max relative error 2^-23; taken as 2^-22 here (conservative).
  * __expf(x) (k_shift_fast): CUDA C++ Programming Guide, "Intrinsic Functions": 2 + floor(|1.173 x|) ulp; taken as
    (2 + 1.2 |x|) ulp.
  * __fdividef(x, y) (k_shift_fast): same table, 2 ulp for 2^-126 <= |y| <= 2^126 (and 0 above 2^126).
  * __log2f(x) (k_stats pop shaping): same table, 2^-22 absolute on [0.5, 2], else 2 ulp; taken as 2^-21 max(1, |L|)
    absolute (conservative: covers both ranges).
  * exp2f (k_stats pop shaping): Programming Guide, single-precision standard functions: 2 ulp.
u8 outputs are carried as intervals [lo, hi] of the bytes the kernel may produce: a float64 value farther than its
bound from a byte boundary gives one byte, otherwise both neighbours are accepted (the byte is "ambiguous"); intervals go
through the colour grade, the sharpen and the 2:1 INTER_AREA by interval arithmetic.  Stages whose inputs are bytes or
exactly known fp32 values (the grade, the sharpen, an unfeathered sample) are restated in fp32 op for op instead, since
their float64 value can sit exactly on a byte boundary (an identity grade of k / 255, a sample between equal pixels)."""
import numpy as np

from oracle import dibr as O

U = 2.0 ** -24
F32 = np.float32
SQRT_APPROX = 2.0 ** -22
FDIV_APPROX = 2.0 * 2.0 ** -23
EXP2F = 2.0 * 2.0 ** -23
TINY = 2.0 ** -120          # flush-to-zero / overflow-to-one slack of the approximate sigmoid


def f64(a):
    return np.asarray(a, dtype=np.float64)


def c32(v):
    """an fp32 constant or scalar coefficient, as the kernel holds it, in float64"""
    return float(np.float32(v))


# ----------------------------------------------------------------------------------------------------------------------
# exact fp32 restatements (only where a plane has to be rebuilt bit for bit: the d0 plane k_stats quantiles in place)
# ----------------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """correctly rounded fp32 fma: the fp64 product of two fp32 is exact; the fp64 sum p + c is corrected by its exact
    TwoSum error when it lands on an fp32 rounding tie, so that the result is never double-rounded."""
    a, b, c = f64(a), f64(b), f64(c)
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    bits = np.asarray(s).view(np.uint64)
    tie = ((bits & np.uint64(0x1FFFFFFF)) == np.uint64(0x10000000)) & (err != 0)
    s = np.where(tie, np.nextafter(s, s + err), s)
    return s.astype(F32)


def resize_bilinear32(src, oh, ow):
    """rs_axis / rs_combine of dibr_device.cuh on a [h, w] fp32 plane, bit for bit (identity at scale 1)."""
    h, w = src.shape
    if (h, w) == (oh, ow):
        return src.astype(F32)
    y0, y1, ly0, ly1 = O._resize_idx(h, oh)
    x0, x1, lx0, lx1 = O._resize_idx(w, ow)

    def row(r):
        return fma32(src[r][:, x0], lx0[None], (src[r][:, x1] * lx1[None]).astype(F32))

    r0, r1 = row(y0), row(y1)
    return fma32(r0, ly0[:, None], (r1 * ly1[:, None]).astype(F32))


def d0_plane(core32, H, W, xs, ys):
    """k_stats d0 = clamp01(resize(core) + (1 - (x^2 + y^2)) * 0.08) with -fmad=false rounding, bit for bit."""
    d = resize_bilinear32(core32, H, W)
    r2 = ((xs[None] * xs[None]).astype(F32) + (ys[:, None] * ys[:, None]).astype(F32)).astype(F32)
    curv = (F32(1) - r2).astype(F32)
    return np.clip((d + (curv * F32(0.08)).astype(F32)).astype(F32), F32(0), F32(1)).astype(F32)


def torch_lerp32(a, b, w):
    a, b, w = F32(a), F32(b), F32(w)
    diff = F32(b - a)
    return F32(a + F32(w * diff)) if abs(w) < 0.5 else F32(b - F32(diff * F32(F32(1) - w)))


def quantile_rank(q, n):
    """vd3d_api.cu quantile_rank: ranks floor / ceil of fp32(q) * fp32(n - 1) and the fp32 weight."""
    rank = F32(F32(q) * F32(n - 1))
    lo, hi = int(np.floor(rank)), int(np.ceil(rank))
    return lo, hi, F32(rank - F32(lo))


def order_stats(plane, ranks):
    """exact order statistics of an fp32 plane (np.partition), as fp32"""
    flat = np.asarray(plane, F32).reshape(-1)
    part = np.partition(flat, sorted(set(ranks)))
    return [F32(part[r]) for r in ranks]


def quantile32(plane, q):
    """torch.quantile as k_stats computes it: the selected order statistics, then torch.lerp by quantile_rank's weight"""
    lo, hi, w = quantile_rank(q, np.asarray(plane).size)
    a, b = order_stats(plane, [lo, hi])
    return torch_lerp32(a, b, w), (a, b, w)


def ties_at(plane, q):
    """how many elements of the plane equal the lower order statistic quantile q selects"""
    lo, _, _ = quantile_rank(q, np.asarray(plane).size)
    v = order_stats(plane, [lo])[0]
    return int((np.asarray(plane, F32) == v).sum())


def pct_scalars(lo, hi, pct_init, pct_lo, pct_hi, alpha=0.92):
    """DepthPercentileEMA.normalize's state update from this frame's quantiles (fin_pct_core, fp32 op for op):
    (pct_flat, n_lo, n_den, new pct_lo, new pct_hi)"""
    lo, hi = F32(lo), F32(hi)
    if F32(hi - lo) < F32(1e-5):
        return 1, F32(0), F32(1), F32(pct_lo), F32(pct_hi)
    if not pct_init:
        nlo, nhi = lo, hi
    else:
        a, b = F32(alpha), F32(1 - alpha)
        nlo = F32(F32(a * F32(pct_lo)) + F32(b * lo))
        nhi = F32(F32(a * F32(pct_hi)) + F32(b * hi))
    return 0, nlo, F32(F32(nhi - nlo) + F32(1e-6)), nlo, nhi


# ----------------------------------------------------------------------------------------------------------------------
# k_stats
# ----------------------------------------------------------------------------------------------------------------------
def lut(u8):
    """frame_to_tensor / depth_to_tensor: u8 / 255 rounded to fp32 (the kernels' 256-entry table), as float64"""
    return f64((np.arange(256, dtype=F32) / F32(255)).astype(F32))[u8]


def resize_bilinear(src, oh, ow):
    """F.interpolate(bilinear, align_corners=False) of [..., h, w] in float64 with the kernels' fp32 axis weights.
    Bound: the four roundings of rs_combine (two products, two fmas) with convex weights, 4 U max|tap|."""
    src = f64(src)
    h, w = src.shape[-2:]
    if (h, w) == (oh, ow):
        return src.copy(), np.zeros_like(src)
    y0, y1, ly0, ly1 = O._resize_idx(h, oh)
    x0, x1, lx0, lx1 = O._resize_idx(w, ow)
    lx0, lx1, ly0, ly1 = f64(lx0), f64(lx1), f64(ly0), f64(ly1)
    a, b = src[..., y0, :][..., x0], src[..., y0, :][..., x1]
    c, d = src[..., y1, :][..., x0], src[..., y1, :][..., x1]
    v = (a * lx0 + b * lx1) * ly0[:, None] + (c * lx0 + d * lx1) * ly1[:, None]
    m = np.maximum(np.maximum(np.abs(a), np.abs(b)), np.maximum(np.abs(c), np.abs(d)))
    return v, 4 * U * m


def gray_u8(depth):
    return depth if depth.ndim == 2 else O.bgr_to_gray_u8(depth)


def ingest(frame_bgr, depth, crop, tw, th):
    """k_stats ingest: (depth value of the target_eye plane, its bound), (RGB [3, th, tw], bound) of the crop
    {x0, y0, w, h} of the u8 frame / depth resized to (th, tw)."""
    x0, y0, w, h = crop
    g = lut(gray_u8(depth)[y0:y0 + h, x0:x0 + w])
    cur, cb = resize_bilinear(g, th, tw)
    rgb = lut(frame_bgr[y0:y0 + h, x0:x0 + w, ::-1].transpose(2, 0, 1))
    rs, rb = resize_bilinear(rgb, th, tw)
    return (cur, cb), (rs, rb)


def temporal(prev32, cur, cur_b, init):
    """TemporalDepthFilter(alpha=0.5): alpha * prev + (1 - alpha) * cur; the first frame's prev is cur itself (exact)."""
    if not init:
        return cur.copy(), cur_b.copy()
    v = 0.5 * f64(prev32) + 0.5 * cur
    return v, 0.5 * cur_b + U * np.abs(v)


def normalize(tdf32, pct_flat, n_lo, n_den):
    """DepthPercentileEMA.normalize on clamp01(tdf) with the frame's n_lo / n_den: a subtraction and a division."""
    d = np.clip(f64(tdf32), 0, 1)
    if pct_flat:
        return d, np.zeros_like(d)
    q = (d - c32(n_lo)) / c32(n_den)
    return np.clip(q, 0, 1), 2 * U * np.abs(q)


def pop_shape(d0_32, st_flat, st_lo, st_den, st_subj, mid, gamma):
    """shape_depth_for_pop on the d0 plane with the frame's stretch scalars: sign(x) |x|^gamma + mid, x = ds - subj.
    Bound: the roundings of ds, centered and x (x errs by ex); |x|^gamma is gamma-Hoelder, so the exact power of the
    device's x is within 2 ex^gamma (gamma <= 1; gamma ex |x|^(gamma - 1) above); __log2f, the product gamma L and
    exp2f err relatively by ln2 (gamma eL + U |gamma L|) + 2 ulp; one rounding of the final sum."""
    v = f64(d0_32)
    mid, gamma = c32(mid), c32(gamma)
    if st_flat:
        ds, eds = v, np.zeros_like(v)
    else:
        q = (v - c32(st_lo)) / c32(st_den)
        ds, eds = np.clip(q, 0, 1), 2 * U * np.abs(q)
    x = ds - c32(st_subj)
    centered = x + mid
    ex = eds + U * (2 * np.abs(x) + np.abs(centered))
    ax = np.abs(x)
    pw = ax ** gamma if gamma != 0 else np.ones_like(ax)
    out = np.clip(np.sign(x) * pw + mid, 0, 1)
    if gamma <= 1:
        hold = 2 * ex ** gamma
    else:
        hold = gamma * (ax + ex) ** (gamma - 1) * ex
    axu = ax + ex
    with np.errstate(divide="ignore"):
        L = np.where(axu > 0, np.log2(np.maximum(axu, 1e-300)), 0.0)
    eL = 2.0 ** -21 * np.maximum(1.0, np.abs(L))
    rel = np.log(2.0) * (abs(gamma) * eL + U * np.abs(gamma * L)) * 1.01 + EXP2F
    pwu = axu ** gamma if gamma != 0 else np.ones_like(ax)
    return out, hold + rel * pwu + U * (np.abs(out) + 1e-30)


# ----------------------------------------------------------------------------------------------------------------------
# k_shift_fast
# ----------------------------------------------------------------------------------------------------------------------
def edge_mask_sigmoid(d32, feather):
    """1 - sigmoid(5 feather (|grad d| - 0.02)) per pixel (backward differences, 0 in row / column 0) and its bound:
    g errs by (3 U + sqrt.approx) g, z = (g - 0.02) f5 by f5 (eg + U |g - 0.02|) + U |z|, __expf relatively by
    (2 + 1.2 |z|) ulp, 1 + t and __fdividef by U + 2 ulp; m(1 - m) carries an error of z / of log t into m."""
    d = f64(d32)
    dx = np.zeros_like(d)
    dy = np.zeros_like(d)
    dx[:, 1:] = d[:, 1:] - d[:, :-1]
    dy[1:, :] = d[1:, :] - d[:-1, :]
    g = np.sqrt(dx * dx + dy * dy)
    f5 = c32(F32(F32(feather) * F32(5)))
    gm = g - c32(0.02)
    z = gm * f5
    with np.errstate(over="ignore"):
        m = 1.0 / (1.0 + np.exp(z))
    eg = g * (3 * U + SQRT_APPROX)
    ez = f5 * (eg + U * np.abs(gm)) + U * np.abs(z)
    eexp = (2 + 1.2 * np.abs(z)) * 2.0 ** -23
    em = m * (1 - m) * (ez + eexp) * 1.01 + m * (U + FDIV_APPROX) + TINY
    return m, em


def box_sum(x, k):
    """sum over the k x k window centred on each pixel, zero outside the plane (k odd)"""
    p = k // 2
    h, w = x.shape
    xp = np.zeros((h + 2 * p, w + 2 * p))
    xp[p:p + h, p:p + w] = x
    c = np.zeros((h + 2 * p + 1, w + 2 * p + 1))
    c[1:, 1:] = xp.cumsum(0).cumsum(1)
    return c[k:k + h, k:k + w] - c[:h, k:k + w] - c[k:k + h, :w] + c[:h, :w]


def shift_map(d32, fs, edge_mask, feather):
    """k_shift_fast: pixel_shift_cuda's shift map (weights fg (1 - d)^1.5, mg, bg; balance / half; zero-parallax
    offset; +-c_max clamp; convergence) and suppress_artifacts_with_edge_mask (5 x 5 zero-padded mean of the mask).
    fs: dict of the FrameScalars fields.  Returns (value, bound)."""
    v = f64(d32)
    c_fg = c32(F32(F32(fs["c_fg"]) * F32(fs["c_fgm"])))
    c_bg = c32(F32(F32(fs["c_bg"]) * F32(fs["c_bgm"])))
    c_mg, c_mid = c32(fs["c_mg"]), c32(fs["c_mid"])
    o1 = 1 - v
    fgw = np.clip(np.abs(o1) ** 1.5 * np.sign(o1), 0, 1)
    efg = np.abs(fgw) * (2.5 * U + SQRT_APPROX) + TINY
    a = np.abs(v - c_mid) * 3
    mgw = np.clip(1 - a, 0, 1)
    emg = U * (2 * a + np.abs(1 - a))
    bgw = np.clip(v, 0, 1)
    t1, t2, t3 = fgw * c_fg, mgw * c_mg, bgw * c_bg
    raw = t1 + t2 + t3
    er = efg * abs(c_fg) + emg * abs(c_mg) + U * (np.abs(t1) + np.abs(t2) + np.abs(t3)) \
        + U * (np.abs(t1 + t2) + np.abs(raw))
    k = c32(fs["c_pb"]) / c32(fs["c_half"])
    total = raw * k
    et = er * abs(k) + 2 * U * np.abs(total)
    if fs["use_zpo"]:
        total = total - c32(fs["c_zpo"])
        et = et + U * np.abs(total)
    cm = c32(fs["c_max"])
    total = np.clip(total, -cm, cm)
    if fs["use_conv"]:
        total = total - c32(fs["c_conv"])
        et = et + U * np.abs(total)
    if not edge_mask:
        return total, et
    m, em = edge_mask_sigmoid(d32, feather)
    acc = box_sum(m, 5)
    ea = box_sum(em, 5) + 8 * U * acc
    sup = total * acc / 25.0
    esup = np.abs(total) * ea / 25.0 + et * acc / 25.0 + 3 * U * np.abs(sup)
    m1, m2 = c32(fs["c_m1"]), c32(fs["c_m2"])
    fin = m1 * total + m2 * sup
    efin = abs(m1) * et + abs(m2) * esup + U * (np.abs(m1 * total) + np.abs(m2 * sup)) + U * np.abs(fin)
    return fin, efin


# ----------------------------------------------------------------------------------------------------------------------
# k_render
# ----------------------------------------------------------------------------------------------------------------------
class Tap:
    """make_tap (F.grid_sample bilinear / border / align_corners=True) for every pixel.  The source coordinate and the
    four weights are index arithmetic: restated in fp32 op for op (grid xs[x] +- shift, ys[y]), so the kernel and this
    restatement pick the same taps with the same weights; the weighted sum is taken in float64."""

    def __init__(self, xs, ys, shift, sign):
        H, W = shift.shape
        shift = np.asarray(shift, F32)
        gx = (np.asarray(xs, F32)[None] + shift if sign > 0 else np.asarray(xs, F32)[None] - shift).astype(F32)
        gy = np.broadcast_to(np.asarray(ys, F32)[:, None], (H, W))
        ix = ((gx + F32(1)).astype(F32) * (F32(W - 1) / F32(2))).astype(F32)
        iy = ((gy + F32(1)).astype(F32) * (F32(H - 1) / F32(2))).astype(F32)
        ix = np.minimum(F32(W - 1), np.maximum(ix, F32(0)))
        iy = np.minimum(F32(H - 1), np.maximum(iy, F32(0)))
        fx, fy = np.floor(ix), np.floor(iy)
        wx, ny = (ix - fx).astype(F32), (iy - fy).astype(F32)
        ex, sy = (F32(1) - wx).astype(F32), (F32(1) - ny).astype(F32)
        self.x0, self.y0 = fx.astype(np.int64), fy.astype(np.int64)
        self.x1 = np.minimum(self.x0 + 1, W - 1)
        self.y1 = np.minimum(self.y0 + 1, H - 1)
        self.w = tuple(f64((p * q).astype(F32)) for p, q in ((sy, ex), (sy, wx), (ny, ex), (ny, wx)))

    def sample(self, plane):
        """(value, bound) of the bilinear sample of `plane` [H, W]: tap_apply's product and three fmas, 4 U max|tap|
        (the fp32 weights sum to 1 within a few U)"""
        p = f64(plane)
        a, b = p[self.y0, self.x0], p[self.y0, self.x1]
        c, d = p[self.y1, self.x0], p[self.y1, self.x1]
        v = self.w[0] * a + self.w[1] * b + self.w[2] * c + self.w[3] * d
        m = np.maximum(np.maximum(np.abs(a), np.abs(b)), np.maximum(np.abs(c), np.abs(d)))
        return v, 4.1 * U * m

    def sample32(self, plane):
        """tap_apply's fp32 product and fma chain (NW first), bit for bit: the value the kernel holds when nothing else
        follows (no feathering), used where the float64 value sits on a byte boundary"""
        p = np.asarray(plane, F32)
        w = [x.astype(F32) for x in self.w]
        o = (p[self.y0, self.x0] * w[0]).astype(F32)
        o = fma32(p[self.y0, self.x1], w[1], o)
        o = fma32(p[self.y1, self.x0], w[2], o)
        return fma32(p[self.y1, self.x1], w[3], o)


def feather_mask(wd, wdb, feather):
    """feather_shift_edges' e = clamp01(|grad warped depth| feather) (backward differences, 0 at row / column 0)"""
    dx = np.zeros_like(wd)
    dy = np.zeros_like(wd)
    edx = np.zeros_like(wd)
    edy = np.zeros_like(wd)
    dx[:, 1:] = wd[:, 1:] - wd[:, :-1]
    dy[1:, :] = wd[1:, :] - wd[:-1, :]
    edx[:, 1:] = wdb[:, 1:] + wdb[:, :-1] + U * np.abs(dx[:, 1:])
    edy[1:, :] = wdb[1:, :] + wdb[:-1, :] + U * np.abs(dy[1:, :])
    g = np.sqrt(dx * dx + dy * dy)
    fs = c32(feather)
    e = np.clip(g * fs, 0, 1)
    return e, fs * (edx + edy + 3 * U * g) + U * e


def eye_float(src, xs, ys, shift, d, k, feather, sign):
    """One eye of k_render before truncation: bilinear gather of the RGB source [3, H, W] (fp32 values) at the parallax
    tap, blended with the unshifted source by the K x K mean of the warped-depth edge mask (K = 0: no feathering).
    Returns (value [3, H, W], bound, exact): `exact` holds the kernel's fp32 value bit for bit where it is known without
    rounding doubt (NaN elsewhere): every sample without feathering, and the source itself where the whole K x K window
    of the mask is 1 beyond its bound (then the blend weight is exactly 1 and s (1 - b) + o b = o exactly)."""
    src32 = np.asarray(src, F32)
    src = f64(src32)
    t = Tap(xs, ys, shift, sign)
    s = np.empty_like(src)
    sb = np.empty_like(src)
    for ch in range(3):
        s[ch], sb[ch] = t.sample(src[ch])
    if not k:
        return s, sb, f64(np.stack([t.sample32(src32[ch]) for ch in range(3)]))
    wd, wdb = t.sample(d)
    e, eb = feather_mask(wd, wdb, feather)
    b = box_sum(e, k) / (k * k)
    bb = box_sum(eb, k) / (k * k) + (2 * (k - 1) * U) * box_sum(e, k) / (k * k) + U * b
    out = s * (1 - b) + src * b
    ob = sb * (1 - b) + np.abs(s - src) * bb + 5 * U * np.maximum(np.abs(s), np.abs(src))
    ones = box_sum((e - eb >= 1).astype(np.float64), k) >= k * k - 0.5
    exact = np.where(ones[None], np.clip(src, 0, 1), np.nan)
    return np.clip(out, 0, 1), ob, exact


def trunc_interval(v, b, exact=None):
    """tensor_to_frame's (v * 255).astype(uint8) of a value within b of v: the [lo, hi] bytes.  A value clamped to
    exactly 0 or 1 on both sides of the interval is exact, and so is a value given in `exact` (fp32 bit for bit: the
    kernel's own fp32 product with 255 is restated)."""
    lo, hi = np.clip(v - b, 0, 1), np.clip(v + b, 0, 1)
    same = lo == hi
    tlo = np.where(same, lo * 255, lo * 255 * (1 - U))
    thi = np.where(same, hi * 255, hi * 255 * (1 + U))
    lo8 = np.clip(np.floor(tlo), 0, 255).astype(np.int64)
    hi8 = np.clip(np.floor(thi), 0, 255).astype(np.int64)
    if exact is not None:
        known = ~np.isnan(exact)
        t = np.floor((np.nan_to_num(exact).astype(F32) * F32(255)).astype(F32)).astype(np.int64)
        t = np.clip(t, 0, 255)
        lo8, hi8 = np.where(known, t, lo8), np.where(known, t, hi8)
    return lo8, hi8


def grade(rgb, sat, con, bri):
    """apply_color_grade in float64 with the kernel's fp32 constants; rgb [3, ...]"""
    r, g, b = rgb
    luma = c32(0.2126) * r + c32(0.7152) * g + c32(0.0722) * b
    out = []
    for c in (r, g, b):
        s = luma + (c - luma) * c32(sat)
        s = c32(0.5) + (s - c32(0.5)) * c32(con)
        out.append(s + c32(bri))
    return np.stack(out)


def grade_interval(lo, hi, sat, con, bri):
    """frame_to_tensor -> apply_color_grade -> tensor_to_frame of eye bytes known to lie in [lo, hi] ([3, ...] RGB).
    Bytes in, bytes out, and the grade's fp32 op order is oracle/dibr.py's (grade_px): restated exactly (the float64
    value of an identity grade sits exactly on a byte boundary, so only the kernel's own roundings decide the byte) at
    every corner of the input intervals, whose extremes bound the output (the grade is affine in each channel)."""
    L = np.arange(256, dtype=F32) / F32(255)
    out_lo = out_hi = None
    for m in range(8):
        sel = np.stack([hi[c] if (m >> c) & 1 else lo[c] for c in range(3)])
        g = O.color_grade(L[sel].astype(F32), sat, con, bri)
        b8 = (g * F32(255)).astype(F32).astype(np.int64)
        out_lo = b8 if out_lo is None else np.minimum(out_lo, b8)
        out_hi = b8 if out_hi is None else np.maximum(out_hi, b8)
    return out_lo, out_hi


def bars(img, side, width):
    """apply_side_mask on an [H, W, ...] array: side 1 = right bar, 2 = left bar (FrameScalars.bar_side)"""
    out = img.copy()
    w = img.shape[1]
    if side == 1 and width > 0:
        out[:, w - width:] = 0
    elif side == 2 and width > 0:
        out[:, :width] = 0
    return out


def sharpen_coeffs(factor):
    c = F32(5.0 + factor)
    ks = F32(c - F32(4))
    if ks == 0:
        return float(c), -1.0
    return float(F32(c / ks)), float(F32(F32(-1) / ks))


def _reflect101(i, n):
    i = np.abs(i)
    return np.where(i >= n, 2 * n - 2 - i, i)


def sharpen_interval(lo, hi, factor):
    """apply_sharpening (cv2.filter2D, REFLECT_101, round half to even) of u8 [H, W, C] bytes known to lie in [lo, hi].
    Bytes in, bytes out: the kernel's fp32 fma chain (up, left, centre, right, down) is restated exactly.  The centre
    weight is positive and the cross negative and every rounding is monotone, so the chain's extremes are the centre's
    lo with the neighbours' hi and vice versa."""
    kc, ke = sharpen_coeffs(factor)
    H, W = lo.shape[:2]
    yy, xx = np.arange(H), np.arange(W)
    ym, yp = _reflect101(yy - 1, H), _reflect101(yy + 1, H)
    xm, xp = _reflect101(xx - 1, W), _reflect101(xx + 1, W)

    def chain(c, n):
        f = (n[ym].astype(F32) * F32(ke)).astype(F32)
        f = fma32(n[:, xm].astype(F32), F32(ke), f)
        f = fma32(c.astype(F32), F32(kc), f)
        f = fma32(n[:, xp].astype(F32), F32(ke), f)
        f = fma32(n[yp].astype(F32), F32(ke), f)
        return np.clip(np.rint(f), 0, 255).astype(np.int64)

    return chain(lo, hi), chain(hi, lo)


def area2_interval(lo, hi):
    """cv2.resize INTER_AREA 2:1 horizontal (scale 0.5, round half to even) of bytes in [lo, hi]: exact and monotone"""
    def f(a):
        s = a[:, 0::2].astype(np.int64) + a[:, 1::2]
        return np.clip(np.rint(s * 0.5), 0, 255).astype(np.int64)
    return f(lo), f(hi)
