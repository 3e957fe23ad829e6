"""TEST INFRASTRUCTURE: float64 restatements of the operations the Real-ESRGAN network kernels compute, on the layouts
the SR engine documents (depth_engine.cu: sr_network, rrdb_network; merged_pipeline.pack_rrdb), exact numpy-float32
restatements of the three byte kernels, the conv tile choice, and generators of stress weights.

tests/test_sr_kernel_refs_cpu.py pins every function here to torch ops, oracle/sr.py and tests/rrdb_oracle.py;
tests/test_sr_kernels_gpu.py compares each CUDA kernel with them, from the inputs the device itself stored.

Layouts: feature maps are NHWC [H, W, C]; 3x3 conv weights are [Cout, 9 * Cin] (tap-major, tap = 3 * ky + kx), as in
tests/depth_kernel_refs.py, whose conv and f16 helpers are reused here."""
import math

import numpy as np

from tests.depth_kernel_refs import F16_EPS, F32_EPS, conv_transpose_scatter, f16_ulp, f64  # noqa: F401
from tests.test_depth_kernels_gpu import ACC  # noqa: F401  (the fp32 accumulation error model of the wgmma GEMMs)

# pick_tile's candidates (depth_engine.cu): spatial tiles of 128 output pixels, tw x th
TILES = ((128, 1), (64, 2), (32, 4), (16, 8))
NUM_SMS = 132

# (w, h) of the GPU checks and the pick_tile case each stands for (tests/test_sr_kernel_refs_cpu.py asserts the cases)
SIZES = [(128, 8), (250, 8), (100, 9), (64, 48), (130, 9), (32, 12), (96, 54), (48, 16), (67, 45), (8, 8), (320, 180)]


def pick_tile(w, h):
    """depth_engine.cu pick_tile: the candidate whose whole tiles cover the fewest pixels, the first on a tie."""
    best = None
    for tw, th in TILES:
        cover = -(-w // tw) * tw * -(-h // th) * th
        if best is None or cover < best[0]:
            best = (cover, tw, th)
    return best[1], best[2]


def tile_case(w, h):
    """(tw, th, exact, tiles): the tile of a w x h map, whether it covers the map exactly, and how many tiles."""
    tw, th = pick_tile(w, h)
    return tw, th, w % tw == 0 and h % th == 0, -(-w // tw) * -(-h // th)


def pack3x3(w):
    """torch conv weight [Cout, Cin, 3, 3] -> [Cout, 9 * Cin] tap-major (the restatement's layout)."""
    w = f64(w)
    return w.transpose(0, 2, 3, 1).reshape(w.shape[0], 9 * w.shape[1])


# ---------------------------------------------------------------------------------------------------------------------
def _shifted(x, idx, axis):
    """x taken at integer positions idx along axis, zero where idx lies outside (the conv's zero padding)."""
    n = x.shape[axis]
    ok = (idx >= 0) & (idx < n)
    out = np.take(x, np.clip(idx, 0, n - 1), axis=axis)
    shape = [1] * out.ndim
    shape[axis] = len(idx)
    return out * ok.reshape(shape)


def conv3x3_at(x, w, bias=None, rows=None, cols=None):
    """conv3x3 (stride 1, zero padding 1) of NHWC x [H, W, Cin] with w [Cout, 9 * Cin], evaluated only at the output
    pixels rows x cols (all by default) -> [len(rows), len(cols), Cout] in float64."""
    H, W, C = x.shape
    rows = np.arange(H) if rows is None else np.asarray(rows)
    cols = np.arange(W) if cols is None else np.asarray(cols)
    wt = f64(w).reshape(-1, 9, C)
    out = np.zeros((len(rows), len(cols), wt.shape[0]))
    for ky in range(3):
        xr = f64(_shifted(x, rows + ky - 1, 0))
        for kx in range(3):
            out += _shifted(xr, cols + kx - 1, 1) @ wt[:, 3 * ky + kx].T
    return out if bias is None else out + f64(bias)


def conv3x3_at_abs(x, w, bias=None, rows=None, cols=None):
    """sum of |x| |w| (+ |bias|) of the same conv: the scale of its accumulation error."""
    return conv3x3_at(np.abs(f64(x)), np.abs(f64(w)), None if bias is None else np.abs(f64(bias)), rows, cols)


def prelu(x, slopes):
    """PReLU with one slope per channel (the last axis)."""
    x = f64(x)
    return np.where(x > 0, x, x * f64(slopes))


def lrelu(x):
    """LeakyReLU(0.2)."""
    x = f64(x)
    return np.where(x > 0, x, 0.2 * x)


def sr_residual(a, res=None, rs=0.0, res2=None, rs2=0.0):
    """the residual chain of the EPI_SR epilogue before its activation: a = res + rs a, then a = res2 + rs2 a."""
    a = f64(a)
    if res is not None:
        a = f64(res) + rs * a
    if res2 is not None:
        a = f64(res2) + rs2 * a
    return a


def phase_conv(x, wp, bias=None, rows=None, cols=None):
    """nearest x2 + 3x3 conv as the engine runs it: four phase convs on the low-resolution map x [h, w, Cin] with the
    packed weights wp [4 * Cout, 9 * Cin], row (py * 2 + px) * Cout + co, scattered to [2 h, 2 w, Cout]: output pixel
    (2 y + py, 2 x + px) is phase (py, px) at (y, x).  rows / cols select low-resolution pixels."""
    y = conv3x3_at(x, wp, bias, rows, cols)
    return conv_transpose_scatter(y.reshape(-1, y.shape[-1]), y.shape[0], y.shape[1], 2, wp.shape[0] // 4)


def phase_weights(w):
    """the combined phase weights of nearest x2 + conv w [Cout, Cin, 3, 3], restated: output (2 y + py) reads
    upsampled row 2 y + py + dy - 1, which is low-resolution row y + floor((py + dy - 1) / 2); taps landing on one
    low-resolution pixel add up.  -> float64 [4 * Cout, 9 * Cin] in the packed row order."""
    w = f64(w)
    co = w.shape[0]
    ph = np.zeros((2, 2) + w.shape)
    for py in range(2):
        for px in range(2):
            for ky in range(3):
                for kx in range(3):
                    ph[py, px, :, :, (py + ky - 1) // 2 + 1, (px + kx - 1) // 2 + 1] += w[:, :, ky, kx]
    return pack3x3(ph.reshape((4 * co,) + w.shape[1:]))


def nearest2(x):
    """nearest x2 upsample of NHWC x."""
    return np.repeat(np.repeat(x, 2, axis=0), 2, axis=1)


def lrelu_f16(x):
    """an identity conv with LeakyReLU in EPI_SR, on f16 x: a = x (exact), 0.2f * a in fp32, rounded to f16."""
    a = np.asarray(x, dtype=np.float16).astype(np.float32)
    return np.where(a > 0, a, np.float32(0.2) * a).astype(np.float16)


def dense_cols(k):
    """channels of a [.., 320] dense buffer conv k of an RDB reads: x (0..63), then growth slice s at 64 s .. 64 s + 31."""
    return list(range(64)) + [64 * (s + 1) + c for s in range(k - 1) for c in range(32)]


# ---------------------------------------------------------------------------------------------------------------------
# the byte kernels, exactly (numpy float32 performs the same IEEE operations in the same order)
def sr_in(bgr):
    """k_sr_in: BGR u8 [h, w, 3] -> f16 [h, w, 64], channel c < 3 = f16(q_rgb[c] / 255f), channels 3..63 zero."""
    q = np.asarray(bgr, dtype=np.uint8)
    out = np.zeros(q.shape[:2] + (64,), dtype=np.float16)
    out[..., :3] = (q[..., ::-1].astype(np.float32) / np.float32(255.0)).astype(np.float16)
    return out


def sr_out(cv, bgr):
    """k_sr_out: last conv f32 [h, w, 48] and input BGR u8 [h, w, 3] -> BGR u8 [4 h, 4 w, 3]: PixelShuffle(4) channel
    c * 16 + (Y & 3) * 4 + (X & 3) of pixel (Y >> 2, X >> 2), plus the input's channel / 255f, clamped to [0, 1], x 255f,
    truncated, RGB -> BGR."""
    cv = np.asarray(cv, dtype=np.float32)
    h, w = cv.shape[:2]
    Y, X = np.arange(4 * h), np.arange(4 * w)
    out = np.empty((4 * h, 4 * w, 3), dtype=np.uint8)
    for c in range(3):
        ch = c * 16 + (Y[:, None] & 3) * 4 + (X[None, :] & 3)
        v = cv[Y[:, None] >> 2, X[None, :] >> 2, ch]
        base = np.asarray(bgr, dtype=np.uint8)[..., 2 - c].astype(np.float32) / np.float32(255.0)
        v = v + base[Y[:, None] >> 2, X[None, :] >> 2]
        out[..., 2 - c] = (np.minimum(np.maximum(v, np.float32(0)), np.float32(1)) * np.float32(255.0)).astype(np.uint8)
    return out


def rrdb_out(rgb):
    """k_rrdb_out: RRDBNet output f32 [H, W, >= 3] (RGB in channels 0..2) -> BGR u8: clamped to [0, 1], x 255f,
    truncated."""
    v = np.asarray(rgb, dtype=np.float32)[..., 2::-1]
    return (np.minimum(np.maximum(v, np.float32(0)), np.float32(1)) * np.float32(255.0)).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# stress weights: every value representable in f16 (the engine's f16 packing is then exact), every indexing slip visible
def _f16(a):
    return np.asarray(a, dtype=np.float16).astype(np.float32)


def _distinct(rng, n, lo, hi):
    """n values spread over [lo, hi], one per channel in shuffled order, no two equal."""
    return rng.permutation(np.linspace(lo, hi, n))


def stress_slopes(rng, n=64):
    """PReLU slopes distinct per channel over [-0.5, 1.5], one of them exactly 0."""
    s = _distinct(rng, n, -0.5, 1.5)
    s[np.argmin(np.abs(s))] = 0.0
    return _f16(s)


def stress_srvgg_state_dict(num_conv, seed=0):
    """SRVGGNetCompact in the upstream naming: He-scale convs (the last one too, not scaled down), biases distinct per
    output channel over [-0.5, 0.5], stress_slopes."""
    rng = np.random.default_rng(seed)
    chans = [(3, 64)] + [(64, 64)] * num_conv + [(64, 48)]
    sd = {}
    for i, (ci, co) in enumerate(chans):
        sd[f"body.{2 * i}.weight"] = _f16(rng.standard_normal((co, ci, 3, 3)) * math.sqrt(1.0 / (9 * ci)))
        sd[f"body.{2 * i}.bias"] = _f16(_distinct(rng, co, -0.5, 0.5))
        if i < len(chans) - 1:
            sd[f"body.{2 * i + 1}.weight"] = stress_slopes(rng, co)
    return sd


def stress_rrdb_state_dict(nb, scale, seed=0):
    """RRDBNet in the basicsr naming: every conv at He scale for LeakyReLU(0.2), biases distinct per output channel
    over [-0.5, 0.5]; conv_last, whose output is the image, at a tenth of He scale with biases around 0.5, so that
    most of it lands inside [0, 1] and not on the clamps."""
    rng = np.random.default_rng(seed)
    gain = 2.0 / (1.0 + 0.2 ** 2)
    sd = {}

    def conv(name, co, ci, mult=1.0, lo=-0.5, hi=0.5):
        sd[name + ".weight"] = _f16(rng.standard_normal((co, ci, 3, 3)) * mult * math.sqrt(gain / (9 * ci)))
        sd[name + ".bias"] = _f16(_distinct(rng, co, lo, hi))

    conv("conv_first", 64, 3)
    for i in range(nb):
        for j in range(1, 4):
            for k in range(1, 6):
                conv(f"body.{i}.rdb{j}.conv{k}", 32 if k < 5 else 64, 64 + 32 * (k - 1))
    conv("conv_body", 64, 64)
    for u in range(1, 2 if scale == 2 else 3):
        conv(f"conv_up{u}", 64, 64)
    conv("conv_hr", 64, 64)
    conv("conv_last", 3, 64, 0.1, 0.35, 0.65)
    return sd


def identity_conv(c=64):
    """(weight, bias) of a 3x3 conv c -> c that passes its input through: 1.0 on the centre tap, zero bias."""
    w = np.zeros((c, c, 3, 3), np.float32)
    w[np.arange(c), np.arange(c), 1, 1] = 1.0
    return w, np.zeros(c, np.float32)


def sample(n, tile, limit):
    """output rows (or columns) to check on a map of n: all when n <= limit, else both borders, both sides of the
    first limit / 4 tile boundaries and of the last one, and limit / 2 evenly spread others."""
    if n <= limit:
        return np.arange(n)
    bounds = list(range(tile, n, tile))
    bounds = bounds[:limit // 4] + bounds[-1:]
    edges = [0, 1, n - 2, n - 1] + [v for t in bounds for v in (t - 1, t)]
    return np.unique(np.concatenate([edges, np.linspace(0, n - 1, limit // 2).astype(int)]))
