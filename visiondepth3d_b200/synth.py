"""Deterministic synthetic clips (SURVEY.md section 8(d)); numpy only.

smooth set: ramps + moving disc (parity gate);  noise set: white-noise RGB
(throughput / adversarial LSB case).  Frame i uses default_rng(1000+i).
letterbox set: the natural content inside top / bottom black bars whose heights change per frame, with the edge cases
of render_sbs_3d's black-bar detection (auto_crop_black_bars) on a fixed eight-frame schedule (_letterbox).
natural set: band-limited random colour / depth fields with fine texture, translating 3 px per frame (temporally
coherent like footage).  Sub-pixel warps of such content land on generic values, not on the k/255 truncation
boundaries the ramps of the smooth set sit on, so it is the set the 1-LSB gate against the reference is meant for.
"""
import numpy as np


def _field(rng, h, w, cell, ch):
    """Bilinear interpolation (float64, numpy only) of a coarse random grid: a band-limited field in [0, 1]."""
    gh, gw = h // cell + 2, w // cell + 2
    g = rng.random((gh, gw, ch))
    yy = np.arange(h, dtype=np.float64) / cell
    xx = np.arange(w, dtype=np.float64) / cell
    y0, x0 = yy.astype(np.int64), xx.astype(np.int64)
    fy, fx = (yy - y0)[:, None, None], (xx - x0)[None, :, None]
    a = g[y0][:, x0] * (1 - fx) + g[y0][:, x0 + 1] * fx
    b = g[y0 + 1][:, x0] * (1 - fx) + g[y0 + 1][:, x0 + 1] * fx
    return a * (1 - fy) + b * fy


def _natural(i, w, h):
    rng = np.random.default_rng(777)           # one scene; frame i is a translated view of it
    pad = 3 * 64                               # room for the 3 px / frame pan
    big_w = w + pad
    col = 0.15 + 0.7 * _field(rng, h, big_w, max(8, h // 12), 3)
    col += 0.10 * (_field(rng, h, big_w, 3, 3) - 0.5)       # fine texture
    dep = 0.1 + 0.8 * _field(rng, h, big_w, max(12, h // 6), 1)[..., 0]
    dep += 0.04 * (_field(rng, h, big_w, 5, 1)[..., 0] - 0.5)
    off = (3 * i) % pad
    rgb = np.clip(col[:, off:off + w] * 255.0, 0, 255).astype(np.uint8)
    d = np.clip(dep[:, off:off + w] * 255.0, 0, 255).astype(np.uint8)
    return rgb, d


def _letterbox(i, w, h, rgb):
    """Bars of the letterbox set on a natural frame, in place.  Bar rows hold dark noise (cv2 gray <= 6).  Frame i % 8:
    0 bars of h/8 and h/8 + 3 rows; 1 no bars; 2 all black; 3 bars with a uniform gray-10 row (mean exactly 10: still a
    bar) next to the picture; 4 the same with one pixel at 11 (mean just above 10: picture); 5 a bright subtitle-like
    line inside the bottom bar; 6 bars with a bright first row; 7 bars with a bright last row."""
    rng = np.random.default_rng(4000 + i)
    k = i % 8
    if k == 1:
        return rgb
    if k == 2:
        rgb[:] = 0
        return rgb
    top, bot = (h // 8, h // 8 + 3) if k == 0 else (h // 6 + k, h // 10 + 2 * k)
    for rows in (slice(0, top), slice(h - bot, h)):
        n = rgb[rows].shape[0]
        rgb[rows] = rng.integers(0, 7, (n, w, 3), dtype=np.uint8)
    if k in (3, 4):
        rgb[top - 1] = 10
        if k == 4:
            rgb[top - 1, w // 3] = 11
    elif k == 5:
        y = h - bot // 2
        rgb[y] = rng.integers(0, 7, (w, 3), dtype=np.uint8)
        rgb[y, w // 4:3 * w // 4] = 220
    elif k == 6:
        rgb[0] = 200
    elif k == 7:
        rgb[h - 1] = 200
    return rgb


def synth_frame(i: int, w: int, h: int, kind: str = "smooth"):
    """Return (frame_bgr u8 [h,w,3], depth_bgr u8 [h,w,3]) for frame index i."""
    rng = np.random.default_rng(1000 + i)
    y, x = np.mgrid[0:h, 0:w]
    cx = (w // 4 + 20 * i) % w
    cy = h // 2
    disc = (x - cx) ** 2 + (y - cy) ** 2 <= (h // 6) ** 2
    if kind in ("natural", "letterbox"):
        rgb, d = _natural(i, w, h)
        d = d.copy()
        d[disc] = 230
        rgb = rgb.copy()
        rgb[disc] = (rgb[disc].astype(np.int32) * 2 // 3 + 60).astype(np.uint8)
        if kind == "letterbox":
            rgb = _letterbox(i, w, h, rgb)
        return np.ascontiguousarray(rgb), np.ascontiguousarray(np.repeat(d[..., None], 3, axis=2))
    if kind == "noise":
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    else:
        rgb = np.empty((h, w, 3), dtype=np.uint8)
        rgb[..., 0] = (x * 255 // max(w - 1, 1)).astype(np.uint8)
        rgb[..., 1] = (y * 255 // max(h - 1, 1)).astype(np.uint8)
        rgb[..., 2] = ((x + y + 8 * i) % 256).astype(np.uint8)
        rgb[disc] = (200, 60, 30)
    d = 255.0 * (0.6 * (0.5 + 0.5 * np.sin(2 * np.pi * x / w)) + 0.4 * y / h)
    d = np.clip(d, 0, 255).astype(np.uint8)
    d[disc] = 230
    depth = np.repeat(d[..., None], 3, axis=2)
    return np.ascontiguousarray(rgb), np.ascontiguousarray(depth)
