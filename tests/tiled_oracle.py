"""numpy / cv2 restatement of the reference's tiled depth path (core/render_depth.py:62-194): the tile plan, the crops,
the Hann blend, np.percentile's linear method in float32 and _normalize_to_u8.  The CPU tests pin it against the
fixtures of `tools/gen_golden.py tiled`; the GPU tests hold libvd3d to it."""
import cv2
import numpy as np

KEYS = ("y0", "y1", "x0", "x1", "yp0", "yp1", "xp0", "xp1", "rh", "rw")


def r14(v):
    return ((int(v) + 13) // 14) * 14


def plan(w, h, tile, pad):
    """[(y0, y1, x0, x1, yp0, yp1, xp0, xp1, rh, rw)], row-major."""
    core = max(1, int(tile) - 2 * int(pad))
    out = []
    for y0 in range(0, h, core):
        for x0 in range(0, w, core):
            y1, x1 = min(y0 + tile, h), min(x0 + tile, w)
            yp0, xp0, yp1, xp1 = max(0, y0 - pad), max(0, x0 - pad), min(h, y1 + pad), min(w, x1 + pad)
            out.append((y0, y1, x0, x1, yp0, yp1, xp0, xp1, r14(yp1 - yp0), r14(xp1 - xp0)))
    return out


def outer_resize(rgb, inference_size):
    h, w = rgb.shape[:2]
    tw, th = inference_size or (w, h)
    interp = cv2.INTER_AREA if (tw < w or th < h) else cv2.INTER_CUBIC
    return cv2.resize(rgb[:, :, ::-1], (tw, th), interpolation=interp)[:, :, ::-1]


def crops(img, tiles):
    out = []
    for y0, y1, x0, x1, yp0, yp1, xp0, xp1, rh, rw in tiles:
        c = img[yp0:yp1, xp0:xp1, :]
        if c.shape[:2] != (rh, rw):
            c = cv2.resize(c, (rw, rh), interpolation=cv2.INTER_CUBIC)
        out.append(np.ascontiguousarray(c))
    return out


def hann2d(h, w):
    m = np.outer(np.hanning(max(2, h)), np.hanning(max(2, w))).astype(np.float32)
    return m / (float(m.max()) + 1e-8)


def weights(ch, cw, tile, pad):
    core = max(1, int(tile) - 2 * int(pad))
    wm = hann2d(core, core)
    if wm.shape != (ch, cw):
        wm = cv2.resize(wm, (cw, ch), interpolation=cv2.INTER_CUBIC)
    return wm


def blend(preds, tiles, w, h, tile, pad):
    """float32 accumulation in plan order, divided by max(w_acc, 1e-8)."""
    acc = np.zeros((h, w), np.float32)
    wacc = np.zeros((h, w), np.float32)
    for p, (y0, y1, x0, x1, yp0, yp1, xp0, xp1, rh, rw) in zip(preds, tiles):
        assert p.shape == (rh, rw) and rh >= yp1 - yp0 and rw >= xp1 - xp0
        center = p[y0 - yp0:y0 - yp0 + (y1 - y0), x0 - xp0:x0 - xp0 + (x1 - x0)]
        wm = weights(y1 - y0, x1 - x0, tile, pad)
        acc[y0:y1, x0:x1] += center * wm
        wacc[y0:y1, x0:x1] += wm
    return acc / np.maximum(wacc, 1e-8)


def percentile(d, p):
    """np.percentile(d, p) of a float32 array (numpy 2.x linear method) restated: q = float32(p) / float32(100), virtual
    index float32(n - 1) * q, the two neighbouring order statistics, numpy's _lerp in float32 with its t >= 0.5 branch."""
    a = np.asarray(d, np.float32).ravel()
    n = a.size
    q = np.float32(p) / np.float32(100)
    nm1 = np.float32(n - 1)
    v = np.float32(nm1 * q)
    if v >= nm1:
        k0 = k1 = n - 1
        g = np.float32(np.float64(v) + 1.0)
    else:
        fl = np.floor(v)
        k0, k1 = int(fl), min(int(fl) + 1, n - 1)
        g = np.float32(v - fl)
    part = np.partition(a, [k0, k1])
    lo, hi = part[k0], part[k1]
    diff = np.float32(hi - lo)
    if g >= 0.5:
        return np.float32(hi - np.float32(diff * np.float32(np.float32(1) - g)))
    return np.float32(lo + np.float32(diff * g))


def normalize_u8(depth, out_size, invert=False, pclip=(1.0, 99.0), resize=None):
    """_normalize_to_u8 restated with percentile().  resize(u8, ow, oh): the final INTER_CUBIC (cv2 by default)."""
    d = np.asarray(depth, np.float32)
    d = np.nan_to_num(d, nan=0.0, posinf=0.0, neginf=0.0)
    lo, hi = percentile(d, pclip[0]), percentile(d, pclip[1])
    if hi - lo < np.float32(1e-6):
        mn, mx = float(d.min()), float(d.max())
        if mx - mn < 1e-6:
            u8 = np.full(d.shape, 128, np.uint8)
        else:
            u8 = (((d - np.float32(mn)) / np.float32(mx - mn + 1e-6)) * np.float32(255.0)).astype(np.uint8)
    else:
        u8 = (np.clip((d - lo) / (hi - lo), np.float32(0), np.float32(1)) * np.float32(255.0)).astype(np.uint8)
    if invert:
        u8 = 255 - u8
    if resize is not None:
        return u8 if u8.shape == (out_size[1], out_size[0]) else resize(u8, *out_size)
    return cv2.resize(u8, tuple(out_size), interpolation=cv2.INTER_CUBIC)


def prediction(crop_rgb, kind):
    """tools/gen_golden.py tiled_prediction: the stand-in depth the fixtures were recorded with."""
    h, w = crop_rgb.shape[:2]
    if kind == "flat":
        return np.full((h, w), 7.0, np.float32)
    if kind == "outliers":
        d = np.full((h, w), 5.0, np.float32)
        d[::5, :2] = 3.0
        return d
    c = crop_rgb.astype(np.float32)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    return c[..., 0] + 2.0 * c[..., 1] + c[..., 2] + xx + 2.0 * yy


def infer(rgb, inference_size, tile, pad, predict):
    """infer_depth_tile restated: predict(crop_rgb) -> float32 [rh, rw] for each crop in plan order."""
    img = outer_resize(rgb, inference_size)
    h, w = img.shape[:2]
    tiles = plan(w, h, tile, pad)
    cs = crops(img, tiles)
    return blend([predict(c) for c in cs], tiles, w, h, tile, pad), tiles, cs


def debug_lines(tiles):
    return [f"[tile] ({y0}:{y1},{x0}:{x1}) crop={(rh, rw)} center={(y1 - y0, x1 - x0)} acc={(y1 - y0, x1 - x0)}"
            for y0, y1, x0, x1, _a, _b, _c, _d, rh, rw in tiles]


def video_frames(frames, per_frame_bars, batch_size, tile, pad, invert, predict, resize=None):
    """The planes process_video2's tiled branch writes: each frame's tiled depth through normalize_u8 at the frame
    size, re-padded with the bars the tracker holds after its batch's last frame.  Also returns the blended depths."""
    from tests.letterbox_oracle import repad
    out, depths = [], []
    for i, f in enumerate(frames):
        h, w = f.shape[:2]
        last = min(len(frames), (i // batch_size + 1) * batch_size) - 1
        depth, _, _ = infer(np.ascontiguousarray(f[..., ::-1]), None, tile, pad, predict)
        depths.append(depth)
        out.append(repad(normalize_u8(depth, (w, h), invert, resize=resize), *per_frame_bars[last]))
    return out, depths
