"""Restatement of Pillow's bicubic resize of 8-bit images (Image.resize(size, Image.BICUBIC) on "RGB" / "L"), the
resize the depth pipe applies for an inference size (visiondepth3d_b200/render_depth.py hf_batch_safe_pipe).

Pillow resamples separably, horizontal pass first; a pass whose axis keeps its size is skipped.  Each output index
has a window of input indices and filter weights (bicubic, a = -0.5, support 2, widened by the scale factor when
shrinking), normalised in double and stored as fixed point with 22 fractional bits, rounded away from zero.  A pass
sums u8 * weight in int32 from 1 << 21, shifts right by 22 and clips to 0..255; the intermediate image is u8.
The CUDA kernel (k_resize_pil_u8) applies the same tables, which the library builds on the host
(vd3d_pil_bicubic_table); tests pin both to Pillow bit for bit."""
import math

import numpy as np

PRECISION_BITS = 22


def _bicubic(x):
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coeffs(in_size, out_size):
    """(xmin [out], count [out], fixed-point weights [out, ksize]) of one axis, all int32."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    xmin_a = np.zeros(out_size, np.int32)
    cnt_a = np.zeros(out_size, np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x in range(xmax):
            k = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + k * (1 << PRECISION_BITS)) if k < 0 else int(0.5 + k * (1 << PRECISION_BITS))
        xmin_a[xx], cnt_a[xx] = xmin, xmax
    return xmin_a, cnt_a, kk


def _pass(img, axis, out_size):
    """One separable pass over axis 0 (rows) or 1 (columns) of a u8 [h, w, c] image."""
    xmin, cnt, kk = coeffs(img.shape[axis], out_size)
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full((out_size,) + src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(kk.shape[1]):
        live = t < cnt
        idx = np.where(live, xmin + t, 0)
        w = np.where(live, kk[:, t], 0).astype(np.int64)
        acc += src[idx] * w.reshape((-1,) + (1,) * (src.ndim - 1))
    assert np.abs(acc).max() < 2 ** 31  # Pillow accumulates in int32
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(img, size):
    """PIL.Image.fromarray(img).resize(size, Image.BICUBIC) on a u8 [h, w] or [h, w, c] array; size = (W, H)."""
    a = np.asarray(img, dtype=np.uint8)
    squeeze = a.ndim == 2
    if squeeze:
        a = a[:, :, None]
    ow, oh = int(size[0]), int(size[1])
    if ow != a.shape[1]:
        a = _pass(a, 1, ow)
    if oh != a.shape[0]:
        a = _pass(a, 0, oh)
    a = np.ascontiguousarray(a)
    return a[:, :, 0] if squeeze else a
