"""Deterministic synthetic clips (SURVEY.md section 8(d)); numpy only.

smooth set: ramps + moving disc (parity gate);  noise set: white-noise RGB
(throughput / adversarial LSB case).  Frame i uses default_rng(1000+i).
letterbox set: the natural content inside top / bottom black bars whose heights change per frame, with the edge cases
of render_sbs_3d's black-bar detection (auto_crop_black_bars) on a fixed eight-frame schedule (_letterbox).
letterbox_track / letterbox_track_nobars sets: clips for the depth-video letterbox tracker at a small fps (2: a
six-frame bootstrap window and cooldown), on the schedule of _TRACK / _TRACK_NOBARS.
natural set: band-limited random colour / depth fields with fine texture, translating 3 px per frame (temporally
coherent like footage).  Sub-pixel warps of such content land on generic values, not on the k/255 truncation
boundaries the ramps of the smooth set sit on, so it is the set the 1-LSB gate against the reference is meant for.
"""
import os

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


# (scene, top, bottom, bar content) per frame.  Scenes 0 and 1 differ in brightness, so a switch between them is a
# scene cut by mean absolute difference; consecutive frames of one scene are not cuts.  "black" is all black, "fade"
# near-black; "flat" is scene 0 squeezed to 15 % contrast around its mean (a cut by histogram correlation alone).
# Bar content: "zero" black, "noise" gray noise (fails the variance gate only), "blue" dark saturated blue (saturation
# gate only), "gray40" (luma gate only), "edge" black with one gray-24 row, which puts Canny edges on a black row
# (edge gate only).  Bars of b rows are detected as b - 2 rows (the two rows next to the picture carry its edges).
_TRACK = (
    [(0, 22, 22, "zero")] * 6                                    # 0-5: bootstrap window, locks (20, 20)
    + [("black", 0, 0, "zero"), (1, 22, 22, "zero")]             # 6 near-black; 7 cut, change below min_change
    + [(0, 31, 31, "zero"), (1, 31, 31, "zero"), (0, 31, 31, "zero")]  # 8-10 odd bars -> (30, 30), confirmed at 3
    + [(1, 12, 12, "zero"), (1, 12, 12, "zero"), (0, 12, 12, "zero"), (0, 12, 12, "zero"), (0, 12, 12, "zero")]
    #                                                              11-15 cuts inside the cooldown: ignored
    + [(1, 16, 16, "zero"), (0, 16, 16, "zero"), (1, 31, 31, "zero")]  # 16-18 candidate (14, 14) breaks off after 2
    + [(0, 27, 31, "zero")]                                      # 19 (26, 30): change 4, below min_change
    + [(1, 42, 42, "zero"), (0, 42, 42, "zero"), (1, 42, 42, "zero")]  # 20-22 (40, 40) > max_total_frac -> (0, 0)
    + [(0, 31, 31, "noise"), (1, 31, 31, "blue"), (0, 31, 31, "gray40"), (1, 31, 31, "edge")]  # 23-26 gates
    + [(1, 0, 0, "zero"), (1, 0, 0, "zero"), (0, 0, 0, "zero"), (0, 0, 0, "zero"), ("flat", 0, 0, "zero")]
    #                                                              27-31: 31 is a histogram-only cut
    + [("fade", 0, 0, "zero"), (0, 22, 22, "zero"), (1, 22, 22, "zero"), (0, 22, 22, "zero")]  # 32 fade; 33-35
    #                                                              locked_zero -> bars (20, 20), confirmed at 3
    + [(0, 22, 22, "zero")]                                      # 36
)
_TRACK_NOBARS = [(0, 0, 0, "zero")] * 6 + [(1, 0, 0, "zero"), (0, 0, 0, "zero")]


def _track_frame(i, w, h, sched):
    scene, top, bot, bar = sched[i]
    if scene == "black":
        return np.zeros((h, w, 3), np.uint8)
    base = _natural(i, w, h)[0][..., ::-1].astype(np.float64)
    if scene == "fade":
        f = base * 0.05
    elif scene == "flat":
        f = base * 0.45
        f = (f - f.mean()) * 0.15 + f.mean()
    else:
        f = base * 0.45 if scene == 0 else base * 0.6 + 90
    f = np.clip(f, 0, 255).astype(np.uint8)
    rng = np.random.default_rng(6000 + i)
    for rows, inner in ((slice(0, top), 1), (slice(h - bot, h), h - 2)):
        n = f[rows].shape[0]
        if n == 0:
            continue
        f[rows] = 0
        if bar == "noise":
            f[rows] = rng.integers(0, 14, (n, w, 1), dtype=np.uint8)
        elif bar == "blue":
            f[rows] = (30, 0, 0)
        elif bar == "gray40":
            f[rows] = 40
        elif bar == "edge":
            f[inner + (1 if inner == 1 else -1)] = 24
    return np.ascontiguousarray(f)


def synth_frame(i: int, w: int, h: int, kind: str = "smooth"):
    """Return (frame_bgr u8 [h,w,3], depth_bgr u8 [h,w,3]) for frame index i."""
    if kind in ("letterbox_track", "letterbox_track_nobars"):
        f = _track_frame(i, w, h, _TRACK if kind == "letterbox_track" else _TRACK_NOBARS)
        return f, np.ascontiguousarray(np.repeat(f[..., 1:2], 3, axis=2))
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


# the frames folder of the merged_pipeline fixtures (tools/gen_golden.py merged): numbered PNGs (frame_9 before
# frame_10 only under the number sort), an upper-case .JPG, a name without digits (sorts last), one corrupt PNG (skipped
# by the loader), and files the extension filter drops
MERGED_FOLDER = (("frame_10.png", 0), ("frame_9.png", 1), ("frame_2.JPG", 2), ("shot_b.png", 3), ("frame_11.png", 4),
                 ("frame_1.png", 5))
MERGED_DECOYS = {"notes.txt": b"not a frame", "frame_5.png": b"\x89PNG corrupt", "frame_3.bmp": None}


def merged_frames_folder(path, w=128, h=72):
    """Write the fixture folder into `path` (created) and return it."""
    import cv2
    os.makedirs(path, exist_ok=True)
    for name, seed in MERGED_FOLDER:
        ext = os.path.splitext(name)[1].lower()
        with open(os.path.join(path, name), "wb") as f:
            f.write(cv2.imencode(ext, synth_frame(seed, w, h, "natural")[0])[1].tobytes())
    for name, data in MERGED_DECOYS.items():
        with open(os.path.join(path, name), "wb") as f:
            f.write(data if data is not None else cv2.imencode(".bmp", synth_frame(7, w, h, "natural")[0])[1].tobytes())
    return path


# the photo folder of the image-depth fixtures (tools/gen_golden.py images): two landscape sizes of one processed size
# (640x480 PNG, 1024x768 upper-case .JPG), a portrait and an odd size, and files the extension filter drops
IMAGE_FOLDER = (("a_room.png", 640, 480, 11), ("b_street.JPG", 1024, 768, 12), ("c_portrait.png", 480, 854, 13),
                ("d_odd.jpeg", 333, 517, 14))
IMAGE_DECOYS = {"notes.txt": b"not an image", "scan.bmp": None}


def image_folder(path):
    """Write the photo fixture folder into `path` (created; Pillow encoders, default quality) and return it."""
    from PIL import Image
    os.makedirs(path, exist_ok=True)
    for name, w, h, seed in IMAGE_FOLDER:
        rgb = synth_frame(seed, w, h, "natural")[0][..., ::-1]
        Image.fromarray(np.ascontiguousarray(rgb)).save(os.path.join(path, name), format="JPEG" if name.lower().endswith(
            (".jpg", ".jpeg")) else "PNG")
    for name, data in IMAGE_DECOYS.items():
        p = os.path.join(path, name)
        if data is None:
            Image.fromarray(synth_frame(15, 64, 48, "natural")[0]).save(p, format="BMP")
        else:
            with open(p, "wb") as f:
                f.write(data)
    return path
