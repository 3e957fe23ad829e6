"""numpy restatement of render_sbs_3d's auto_crop_black_bars (core/render_3d.py:293-326, 1065-1070, 1086-1090,
1238-1248), built on oracle/dibr.py: the tests of the option (tests/test_autocrop_*.py) drive it."""
from dataclasses import dataclass

import numpy as np

from oracle import dibr as O


def detect_black_bars(frame_bgr: np.ndarray, threshold=10):
    """detect_black_bars (core/render_3d.py:293-316) -> (top, bottom) in rows.  A row is bright when the np.mean of its
    cv2 gray values exceeds `threshold`; np.mean of u8 sums exactly in float64 and divides once, so that is exactly the
    integer test sum(gray[i]) > threshold * W.  top = first bright row, bottom = H-1-last bright row, (0, 0) when no
    row is bright."""
    gray = O.bgr_to_gray_u8(frame_bgr).astype(np.int64)
    h, w = gray.shape
    bright = np.nonzero(gray.sum(axis=1) > threshold * w)[0]
    if bright.size == 0:
        return 0, 0
    return int(bright[0]), int(h - 1 - bright[-1])


def crop_rows(h: int, top: int, bottom: int):
    """crop_black_bars_torch (core/render_3d.py:318-326): the rows [top, h - bottom) kept, or all of them when
    top + bottom >= h -> (first row, row count)."""
    if top + bottom >= h:
        return 0, h
    return top, h - top - bottom


@dataclass
class RenderParams(O.RenderParams):
    auto_crop_black_bars: bool = False


def probe_original_size(probe_bgr: np.ndarray, rp: RenderParams):
    """render_sbs_3d's preserve_original_aspect fallback (core/render_3d.py:1065-1070, 1086-1090): original_video_*
    left at None take the size of the probe frame (the dropped first pair) after its black bars are cropped when
    auto_crop_black_bars is set.  Returns (width, height) for RenderParams.original_video_width / _height."""
    if rp.original_video_width is not None and rp.original_video_height is not None:
        return rp.original_video_width, rp.original_video_height
    h, w = probe_bgr.shape[:2]
    if rp.auto_crop_black_bars:
        _, h = crop_rows(h, *detect_black_bars(probe_bgr))
    return w, h


def render_frame(gs: O.GlobalState, cs: O.ClipState, frame_bgr: np.ndarray, depth_bgr: np.ndarray, rp: RenderParams,
                 return_parts=False):
    """One iteration of the render_sbs_3d loop body with auto_crop_black_bars (1238-1248): the frame and the depth map
    lose the black-bar rows detected on the frame, then oracle.dibr.render_frame runs on what is left -- its aspect
    crop then works on the cropped size, as the reference's does.  Per-frame sizes do not change, so a
    preserve_original_aspect render needs original_video_* resolved (probe_original_size) beforehand."""
    if not rp.auto_crop_black_bars:
        return O.render_frame(gs, cs, frame_bgr, depth_bgr, rp, return_parts)
    if rp.preserve_original_aspect and (rp.original_video_width is None or rp.original_video_height is None):
        raise ValueError("resolve original_video_* with probe_original_size first")
    bars = detect_black_bars(frame_bgr)
    y0, rows = crop_rows(frame_bgr.shape[0], *bars)
    out = O.render_frame(gs, cs, frame_bgr[y0:y0 + rows], depth_bgr[y0:y0 + rows], rp, return_parts)
    if return_parts:
        out[1]["crop"] = bars
    return out
