"""numpy / cv2 statement of the letterbox tracker of the depth-video pass (the reference's LetterboxTracker and its
helpers, core/render_depth.py:273-573) and of the depth re-pad (1919-1933).  Everything here works on pixels on the
host, so the GPU statistics and the package's host-side decisions can both be checked against it."""
from types import SimpleNamespace

import cv2
import numpy as np

CANNY = (30, 90)


def luma(frame):
    f = frame.astype(np.float32)
    return 0.2126 * f[..., 2] + 0.7152 * f[..., 1] + 0.0722 * f[..., 0]


def saturation(frame):
    return cv2.cvtColor(frame, cv2.COLOR_BGR2HSV)[..., 1].astype(np.float32)


def gray_of(frame):
    return cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY)


def canny(gray, low=CANNY[0], high=CANNY[1]):
    return cv2.Canny(gray, low, high, apertureSize=3, L2gradient=True)


def hist64(gray):
    return cv2.calcHist([gray], [0], None, [64], [0, 256])


def frame_stats(frame, prev_gray=None):
    """The records vd3d_letterbox_stats returns for one frame, from numpy / cv2."""
    y, s, g = luma(frame), saturation(frame), gray_of(frame)
    e = canny(g)
    return SimpleNamespace(
        h=frame.shape[0], w=frame.shape[1], y_mean=y.mean(axis=1), y_var=y.var(axis=1), s_mean=s.mean(axis=1),
        edges=(e > 0).sum(axis=1).astype(np.int32), frame_y_mean=np.float32(y.mean()),
        hist=hist64(g).ravel().astype(np.uint32), gray=g,
        absdiff=None if prev_gray is None else int(np.abs(g.astype(np.int32) - prev_gray.astype(np.int32)).sum()))


def edge_density(gray):
    return canny(gray).mean(axis=1) / 255.0


def scene_cut(prev_gray, gray, mad_thresh=28.0, corr_thresh=0.60):
    if prev_gray is None or gray is None:
        return False
    if prev_gray.shape != gray.shape:
        return True
    if float(np.mean(np.abs(prev_gray.astype(np.int16) - gray.astype(np.int16)))) > mad_thresh:
        return True
    a, b = hist64(prev_gray), hist64(gray)
    cv2.normalize(a, a)
    cv2.normalize(b, b)
    return float(cv2.compareHist(a, b, cv2.HISTCMP_CORREL)) < corr_thresh


def near_black(frame, mean_thresh=18, edge_thresh=0.02):
    return float(luma(frame).mean()) < mean_thresh and edge_density(gray_of(frame)).mean() < edge_thresh


def bars_of_frame(frame, y_thresh=16, var_thresh=3.0, sat_thresh=6.0, max_scan_frac=0.25, min_band_frac=0.06,
                  edge_max=0.04):
    """Single-frame (top, bottom): the run of dark, flat, unsaturated, edge-free rows from each side within the
    first max_scan_frac of the height; runs below min_band_frac of the height drop to 0, odd runs lose a row, and a
    total of 60 % of the height or more is rejected."""
    h, w = frame.shape[:2]
    if h < 64 or w < 64:
        return 0, 0
    y, s = luma(frame), saturation(frame)
    ym, yv, sm = y.mean(axis=1), y.var(axis=1), s.mean(axis=1)
    ed = edge_density(gray_of(frame))
    is_bar = (ym < y_thresh) & (yv < var_thresh) & (sm < sat_thresh) & (ed <= edge_max)
    depth = int(h * max_scan_frac)

    def run_len(flags):
        n = 0
        while n < depth and flags[n]:
            n += 1
        n = 0 if n < int(h * min_band_frac) else n
        return n - (n % 2)

    t, b = run_len(is_bar), run_len(is_bar[::-1])
    return (0, 0) if t + b >= h * 0.6 else (t, b)


def bootstrap(frames, h, fps, max_seconds=3, samples=9):
    """((top, bottom), confidence) from evenly spaced frames of the first max_seconds (frames: the whole clip)."""
    window = max(min(len(frames), int((fps if fps and fps > 0 else 30) * max_seconds)), 1)
    tops, bots, prev = [], [], None
    for i in np.linspace(0, max(0, window - 1), num=min(samples, window), dtype=int):
        fr = frames[int(i)]
        g = gray_of(fr)
        if not (near_black(fr) or scene_cut(prev, g)):
            t, b = bars_of_frame(fr)
            if 0 <= t < h and 0 <= b < h and t + b < h:
                tops.append(t)
                bots.append(b)
        prev = g
    if not tops:
        return (0, 0), 0.0
    t, b = int(np.median(tops)), int(np.median(bots))
    t, b = max(t - t % 2, 0), max(b - b % 2, 0)
    if t + b >= h * 0.6:
        return (0, 0), 0.0
    ok = sum(abs(x - t) <= 4 and abs(y - b) <= 4 for x, y in zip(tops, bots))
    return (t, b), float(ok / max(1, len(tops)))


class Tracker:
    """Bars frozen between scene cuts; a re-check after the cooldown needs confirm consecutive equal candidates that
    differ from the current bars by at least min_change rows."""

    def __init__(self, h, fps, min_change=8, confirm=3, max_total_frac=0.35, conf_enable=0.7, cooldown_sec=3.0):
        self.h = int(h)
        fps = float(fps) if fps and fps > 0 else 30.0
        self.fps, self.min_change, self.confirm = fps, min_change, confirm
        self.max_total, self.conf_enable = int(self.h * max_total_frac), conf_enable
        self.cooldown_frames = int(fps * cooldown_sec)
        self.bars, self.has_bars = (0, 0), False
        self.cand, self.streak, self.cooldown, self.prev = (0, 0), 0, 0, None

    def bootstrap(self, frames):
        bars, conf = bootstrap(frames, self.h, self.fps)
        self.has_bars = conf >= self.conf_enable and sum(bars) > 0
        self.bars = bars if self.has_bars else (0, 0)
        self.cooldown = self.cooldown_frames
        return self.bars, (self.has_bars, not self.has_bars), conf

    def update(self, frame):
        self.cooldown = max(self.cooldown - 1, 0) if self.cooldown > 0 else self.cooldown
        g = gray_of(frame)
        prev, self.prev = self.prev, g
        if near_black(frame) or not scene_cut(prev, g) or self.cooldown > 0:
            return self.bars
        t, b = bars_of_frame(frame)
        if t + b > self.max_total:
            t, b = 0, 0
        t, b = max(t - t % 2, 0), max(b - b % 2, 0)
        if abs(t - self.bars[0]) + abs(b - self.bars[1]) < self.min_change:
            self.streak, self.cand = 0, self.bars
            return self.bars
        self.streak = self.streak + 1 if (t, b) == self.cand else 1
        self.cand = (t, b)
        if self.streak >= self.confirm and (self.has_bars or t + b > 0):
            self.bars, self.has_bars = (t, b), t + b > 0
            self.cooldown = self.cooldown_frames
        return self.bars


def repad(depth_u8, top, bottom):
    """Depth re-pad: INTER_CUBIC resize into rows [top, h - bottom), bar rows at int(np.median(core))."""
    h, w = depth_u8.shape
    if not (top or bottom):
        return depth_u8.copy()
    core_h = h - top - bottom
    if core_h <= 0:
        return depth_u8.copy()
    core = cv2.resize(depth_u8, (w, core_h), interpolation=cv2.INTER_CUBIC)
    out = np.full((h, w), int(np.median(core)), dtype=np.uint8)
    out[top:top + core_h] = core
    return out


def track_frames(kind="letterbox_track"):
    from visiondepth3d_b200 import synth
    n = len(synth._TRACK if kind == "letterbox_track" else synth._TRACK_NOBARS)
    return [synth.synth_frame(i, 320, 180, kind)[0] for i in range(n)]


def stub_depth_u8(frame):
    """The u8 depth of the fixtures' stub pipe (depth = 0.5 * green + row), min-max normalised and truncated."""
    g = frame[..., 1].astype(np.float32)
    d = 0.5 * g + np.arange(g.shape[0], dtype=np.float32)[:, None]
    lo, hi = np.min(d), np.max(d)
    return ((d - lo) / (hi - lo + 1e-6) * 255).astype(np.uint8)


def written_frames(frames, per_frame_bars, batch_size):
    """The planes the depth-video pass writes: each frame of a batch re-padded with the bars after its last frame."""
    out = []
    for i, f in enumerate(frames):
        last = min(len(frames), (i // batch_size + 1) * batch_size) - 1
        out.append(repad(stub_depth_u8(f), *per_frame_bars[last]))
    return out
