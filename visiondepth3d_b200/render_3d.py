"""Drop-in for the hot-path surface of the reference's core/render_3d.py, backed by
libvd3d.so (hand-written sm_90a CUDA).  Same names, argument meaning, return types and
error behaviour as the reference (file:line cited per function); no Tk, no ONNXRuntime,
no CPU fallback.

    from visiondepth3d_b200 import render_3d as core_render_3d
    left, right, shift = core_render_3d.pixel_shift_cuda(frame_t, depth_t, W, H, 4.5, -1.5, -6.0)
"""
import ctypes as C
import threading
import time

import numpy as np

from . import _lib
from ._lib import FrameInfo, RenderParams, ShiftParams, SizePlan

try:  # torch is plumbing only (device tensors in / out); numpy works too
    import torch
except Exception:  # pragma: no cover
    torch = None

# module-level names the reference's callers import (core/render_3d.py:33-47)
suspend_flag = threading.Event()
cancel_flag = threading.Event()
aspect_ratios = {
    "Default (16:9)": 16 / 9,
    "CinemaScope (2.39:1)": 2.39,
    "21:9 UltraWide": 21 / 9,
    "4:3 (Classic Films)": 4 / 3,
    "1:1 (Square)": 1 / 1,
    "2.35:1 (Classic Cinematic)": 2.35,
    "2.76:1 (Ultra-Panavision)": 2.76,
}

torch_device = None
if torch is not None:
    torch_device = torch.device("cuda" if torch.cuda.is_available() else "cpu")


def _ctx():
    dev = 0
    if torch is not None and torch.cuda.is_available():
        dev = torch.cuda.current_device()
    return _lib.default_context(dev)


def reset_temporal_state(global_state=True, clip_state=True):
    """Reset what the reference keeps in module singletons (core/render_3d.py:284-285,500,511)
    and in per-render objects (1174-1182)."""
    which = (_lib.STATE_GLOBAL if global_state else 0) | (_lib.STATE_CLIP if clip_state else 0)
    _ctx().reset(which)


# ---------------------------------------------------------------------------
# converters (core/render_3d.py:135-143, 289-291) -- host-side glue the reference's callers use
# ---------------------------------------------------------------------------
def frame_to_tensor(frame):
    """BGR u8 HWC -> RGB f32 CHW /255 on torch_device (core/render_3d.py:135-138)."""
    t = torch.from_numpy(np.ascontiguousarray(frame[..., ::-1])).to(torch_device)
    return t.float().permute(2, 0, 1) / 255.0


def depth_to_tensor(depth_frame):
    """cv2 BGR2GRAY (fixed point) then /255 (core/render_3d.py:140-143)."""
    d = depth_frame.astype(np.int64)
    g = ((d[..., 0] * 3735 + d[..., 1] * 19235 + d[..., 2] * 9798 + (1 << 14)) >> 15).astype(np.uint8)
    return (torch.from_numpy(g).to(torch_device).float().unsqueeze(0)) / 255.0


def tensor_to_frame(tensor):
    """RGB f32 CHW -> BGR u8 HWC, truncating (core/render_3d.py:289-291)."""
    a = (tensor.permute(1, 2, 0).cpu().numpy() * 255).astype(np.uint8)
    return np.ascontiguousarray(a[..., ::-1])


def _ptr_and_mem(x):
    """(address, mem kind, keepalive) for a torch tensor or numpy array."""
    if torch is not None and isinstance(x, torch.Tensor):
        x = x.contiguous()
        if x.is_cuda:
            return x.data_ptr(), _lib.MEM_DEVICE, x
        a = x.numpy()
        return a.ctypes.data, _lib.MEM_HOST, a
    a = np.ascontiguousarray(x)
    return a.ctypes.data, _lib.MEM_HOST, a


def pixel_shift_cuda(
    frame_tensor, depth_tensor, width, height, fg_shift, mg_shift, bg_shift,
    blur_ksize=9, feather_strength=10.0, max_pixel_shift_percent=0.02, parallax_balance=0.8,
    zero_parallax_strength=0.0, use_subject_tracking=True, enable_floating_window=True,
    return_shift_map=True, enable_feathering=True, enable_edge_masking=True, dof_strength=2.0,
    convergence_strength=0.0, enable_dynamic_convergence=True, depth_pop_gamma=0.85,
    depth_pop_mid=0.50, depth_stretch_lo=0.05, depth_stretch_hi=0.95, fg_pop_multiplier=1.20,
    bg_push_multiplier=1.10, subject_lock_strength=1.00, _info=None,
):
    """core/render_3d.py:561-712.  frame_tensor f32 RGB [3,h,w] in 0..1, depth_tensor f32
    [1,h,w]; returns (left_bgr_u8, right_bgr_u8[, final_shift cpu f32 [1,H,W]]).
    `dof_strength` is accepted and unused, as in the reference."""
    width, height = int(width), int(height)
    ctx = _ctx()
    fp, fmem, fk = _ptr_and_mem(frame_tensor if frame_tensor.dtype in (np.float32, getattr(torch, "float32", None))
                                else frame_tensor.float())
    dp, dmem, dk = _ptr_and_mem(depth_tensor if depth_tensor.dtype in (np.float32, getattr(torch, "float32", None))
                                else depth_tensor.float())
    in_h, in_w = int(frame_tensor.shape[1]), int(frame_tensor.shape[2])
    assert tuple(depth_tensor.shape[-2:]) == (in_h, in_w), "Shape mismatch"
    if fmem != dmem:
        raise ValueError("frame and depth must live on the same device")
    p = ShiftParams(
        float(fg_shift), float(mg_shift), float(bg_shift), int(blur_ksize), float(feather_strength),
        float(max_pixel_shift_percent), float(parallax_balance), float(zero_parallax_strength),
        int(bool(use_subject_tracking)), int(bool(enable_floating_window)), int(bool(enable_feathering)),
        int(bool(enable_edge_masking)), float(convergence_strength), int(bool(enable_dynamic_convergence)),
        float(depth_pop_gamma), float(depth_pop_mid), float(depth_stretch_lo), float(depth_stretch_hi),
        float(fg_pop_multiplier), float(bg_push_multiplier), float(subject_lock_strength))
    info = FrameInfo()
    if fmem == _lib.MEM_DEVICE:
        left_t = torch.empty((height, width, 3), dtype=torch.uint8, device=frame_tensor.device)
        right_t = torch.empty_like(left_t)
        shift_t = torch.empty((1, height, width), dtype=torch.float32, device=frame_tensor.device) \
            if return_shift_map else None
        torch.cuda.current_stream().synchronize()
        ctx.check(ctx.lib.vd3d_pixel_shift(
            ctx.h, fp, dp, in_h, in_w, width, height, C.byref(p), left_t.data_ptr(), right_t.data_ptr(),
            shift_t.data_ptr() if shift_t is not None else None, _lib.MEM_DEVICE, C.byref(info)))
        left, right = left_t.cpu().numpy(), right_t.cpu().numpy()
        shift = shift_t.cpu() if shift_t is not None else None
    else:
        left = np.empty((height, width, 3), dtype=np.uint8)
        right = np.empty_like(left)
        sh = np.empty((1, height, width), dtype=np.float32) if return_shift_map else None
        ctx.check(ctx.lib.vd3d_pixel_shift(
            ctx.h, fp, dp, in_h, in_w, width, height, C.byref(p), left.ctypes.data, right.ctypes.data,
            sh.ctypes.data if sh is not None else None, _lib.MEM_HOST, C.byref(info)))
        shift = (torch.from_numpy(sh) if torch is not None else sh) if sh is not None else None
    if _info is not None:
        _info.append(info)
    if return_shift_map:
        return left, right, shift
    return left, right


# ---------------------------------------------------------------------------
# stage functions (same kernels as the fused frame path)
# ---------------------------------------------------------------------------
def apply_sharpening(frame, factor=1.0):
    """core/render_3d.py:717-732 (cv2.filter2D u8 semantics)."""
    ctx = _ctx()
    src = np.ascontiguousarray(frame, dtype=np.uint8)
    out = np.empty_like(src)
    ctx.check(ctx.lib.vd3d_sharpen(ctx.h, src.ctypes.data, src.shape[0], src.shape[1], float(factor),
                                   out.ctypes.data, _lib.MEM_HOST))
    return out


def apply_color_grade(rgb_tensor, saturation=1.0, contrast=1.0, brightness=0.0):
    """core/render_3d.py:734-767: f32 RGB [3,H,W] in 0..1 -> graded, clamped tensor of the same kind (torch tensor on
    its device, or numpy)."""
    assert rgb_tensor.ndim == 3 and rgb_tensor.shape[0] == 3
    ctx = _ctx()
    h, w = int(rgb_tensor.shape[1]), int(rgb_tensor.shape[2])
    is_t = torch is not None and isinstance(rgb_tensor, torch.Tensor)
    if is_t and rgb_tensor.is_cuda:
        src = rgb_tensor.contiguous().float()
        out = torch.empty_like(src)
        torch.cuda.current_stream().synchronize()
        ctx.check(ctx.lib.vd3d_color_grade(ctx.h, src.data_ptr(), h, w, float(saturation), float(contrast),
                                           float(brightness), out.data_ptr(), _lib.MEM_DEVICE))
        return out
    src = np.ascontiguousarray(rgb_tensor.detach().cpu().numpy() if is_t else rgb_tensor, dtype=np.float32)
    out = np.empty_like(src)
    ctx.check(ctx.lib.vd3d_color_grade(ctx.h, src.ctypes.data, h, w, float(saturation), float(contrast),
                                       float(brightness), out.ctypes.data, _lib.MEM_HOST))
    return torch.from_numpy(out) if is_t else out


def dof_grade_frame(frame_bgr, depth01, focal_depth, max_sigma=2.0, saturation=1.0, contrast=1.0,
                    brightness=0.0):
    """frame_to_tensor -> apply_dof_cuda -> apply_color_grade -> tensor_to_frame on a u8 eye
    (core/render_3d.py:1342-1369); max_sigma <= 0 skips DOF (1373-1386)."""
    ctx = _ctx()
    src = np.ascontiguousarray(frame_bgr, dtype=np.uint8)
    out = np.empty_like(src)
    d = None
    dh = dw = 0
    if depth01 is not None:
        d = np.ascontiguousarray(np.asarray(depth01, dtype=np.float32).reshape(depth01.shape[-2:]))
        dh, dw = d.shape
    ctx.check(ctx.lib.vd3d_dof_grade(
        ctx.h, src.ctypes.data, src.shape[0], src.shape[1], d.ctypes.data if d is not None else None, dh, dw,
        float(focal_depth), float(max_sigma), float(saturation), float(contrast), float(brightness),
        out.ctypes.data, _lib.MEM_HOST))
    return out


def heal_missing_pixels(warped_frame, warped_depth, original_frame, edge_mask, heal_strength=0.5):
    """core/render_3d.py:431-459 (`warped_depth` is unused there too).  f32 [3,H,W] tensors / arrays in,
    same type out."""
    ctx = _ctx()
    is_t = torch is not None and isinstance(warped_frame, torch.Tensor)
    wf = np.ascontiguousarray((warped_frame.detach().cpu().numpy() if is_t else warped_frame), dtype=np.float32)
    of = original_frame.detach().cpu().numpy() if (torch is not None and isinstance(original_frame, torch.Tensor)) \
        else original_frame
    of = np.ascontiguousarray(of, dtype=np.float32)
    em = None
    if edge_mask is not None:
        em = edge_mask.detach().cpu().numpy() if (torch is not None and isinstance(edge_mask, torch.Tensor)) else edge_mask
        em = np.ascontiguousarray(np.asarray(em, dtype=np.float32).reshape(wf.shape[1:]))
    out = np.empty_like(wf)
    ctx.check(ctx.lib.vd3d_heal(ctx.h, wf.ctypes.data, of.ctypes.data, em.ctypes.data if em is not None else None,
                                wf.shape[1], wf.shape[2], float(heal_strength), out.ctypes.data, _lib.MEM_HOST))
    return torch.from_numpy(out).to(warped_frame.device) if is_t else out


def _fit_eye(image, target_width, target_height, keep_aspect):
    ctx = _ctx()
    img = np.ascontiguousarray(image, dtype=np.uint8)
    assert img.ndim == 3 and img.shape[2] == 3, "expected a BGR u8 image"
    h, w = img.shape[:2]
    out = np.empty((int(target_height), int(target_width), 3), dtype=np.uint8)
    ctx.check(ctx.lib.vd3d_fit_eye(ctx.h, img.ctypes.data, h, w, int(target_width), int(target_height),
                                   int(bool(keep_aspect)), out.ctypes.data, _lib.MEM_HOST))
    return out


def pad_to_aspect_ratio(image, target_width, target_height, bg_color=(0, 0, 0)):
    """core/render_3d.py:101-131 on the GPU (vd3d_fit_eye): aspect-preserving cv2 INTER_AREA shrink (identity, integer
    or fractional factors) centred on a black canvas.  Enlarging fits raise (cv2 changes algorithm there)."""
    if tuple(int(c) for c in bg_color) != (0, 0, 0):
        raise NotImplementedError("pad_to_aspect_ratio: only the black canvas the render loop uses is supported")
    return _fit_eye(image, target_width, target_height, True)


def resize_area(image, width, height):
    """cv2.resize(image, (width, height), interpolation=cv2.INTER_AREA) as in the Half-SBS eye fit
    (core/render_3d.py:1413-1414), shrinking only."""
    return _fit_eye(image, width, height, False)


def _pack(left, right, fmt):
    """format_3d_output on the GPU (vd3d_pack): SBS hstack, Dubois anaglyph, row interlace."""
    ctx = _ctx()
    l = np.ascontiguousarray(left, dtype=np.uint8)
    r = np.ascontiguousarray(right, dtype=np.uint8)
    assert l.shape == r.shape and l.ndim == 3 and l.shape[2] == 3, "Shape mismatch"
    h, w = l.shape[:2]
    code = _lib.FMT[fmt]
    out = np.empty((h, 2 * w, 3) if code in (0, 1, 4) else (h, w, 3), dtype=np.uint8)
    ctx.check(ctx.lib.vd3d_pack(ctx.h, l.ctypes.data, r.ctypes.data, h, w, code, out.ctypes.data, _lib.MEM_HOST))
    return out


def generate_anaglyph_3d(left_frame, right_frame):
    """core/render_3d.py:862-883 (Dubois matrix on channel indices 0,1,2 as written there)."""
    return _pack(left_frame, right_frame, "Red-Cyan Anaglyph")


def format_3d_output(left, right, fmt):
    """core/render_3d.py:837-860."""
    if fmt == "VR" and tuple(left.shape[:2]) != (1600, 1440):
        # the render loop always hands 1440x1600 eyes (pad_to_aspect_ratio) where the reference's cv2.resize is the identity
        raise NotImplementedError("VR pack of eyes that are not 1440x1600 (cv2 INTER_LINEAR resize) is outside the hot path")
    if fmt not in ("Half-SBS", "Full-SBS", "Red-Cyan Anaglyph", "Passive Interlaced", "VR"):
        fmt = "Half-SBS"  # the reference falls back to hstack (860)
    return _pack(left, right, fmt)


# ---------------------------------------------------------------------------
# frame loop
# ---------------------------------------------------------------------------
def make_render_params(output_width, output_height, fg_shift, mg_shift, bg_shift, sharpness_factor,
                       output_format, aspect_ratio, dof_strength, feather_strength=0.0, blur_ksize=1,
                       use_subject_tracking=False, use_floating_window=False, max_pixel_shift_percent=0.02,
                       preserve_original_aspect=False, zero_parallax_strength=0.0, enable_edge_masking=True,
                       enable_feathering=True, original_video_width=None, original_video_height=None,
                       convergence_strength=0.0, enable_dynamic_convergence=True, ipd_factor=1.0,
                       color_saturation=1.0, color_contrast=1.0, color_brightness=0.0, auto_crop_black_bars=False):
    """vd3d_render_params from render_sbs_3d's arguments (core/render_3d.py:933-985)."""
    if output_format not in _lib.FMT:
        output_format = "Half-SBS"  # format_3d_output's fallback is hstack (860)
    return RenderParams(
        int(output_width), int(output_height), float(fg_shift), float(mg_shift), float(bg_shift),
        float(sharpness_factor), _lib.FMT[output_format], float(aspect_ratio), float(dof_strength),
        float(feather_strength), int(blur_ksize), int(bool(use_subject_tracking)),
        int(bool(use_floating_window)), float(max_pixel_shift_percent), int(bool(preserve_original_aspect)),
        float(zero_parallax_strength), int(bool(enable_edge_masking)), int(bool(enable_feathering)),
        int(original_video_width or 0), int(original_video_height or 0), float(convergence_strength),
        int(bool(enable_dynamic_convergence)), float(ipd_factor), float(color_saturation),
        float(color_contrast), float(color_brightness), int(bool(auto_crop_black_bars)))


def plan_sizes(src_w, src_h, rp):
    pl = SizePlan()
    rc = _lib.load().vd3d_plan_sizes(int(src_w), int(src_h), C.byref(rp), C.byref(pl))
    if rc != 0:
        raise _lib.Vd3dError(f"vd3d_plan_sizes: unsupported configuration ({rc})")
    return pl


def output_shape(rp, pl):
    """Shape of the packed frame (format_3d_output, core/render_3d.py:837-860): anaglyph / interlaced are one eye wide,
    the SBS family is the hstack of the two fitted eyes (2 * per_eye_w: one less than plan.out_width for an odd
    preserve-aspect Half-SBS width)."""
    if rp.output_format in (_lib.FMT["Red-Cyan Anaglyph"], _lib.FMT["Passive Interlaced"]):
        return (pl.per_eye_h, pl.per_eye_w, 3)
    return (pl.per_eye_h, 2 * pl.per_eye_w, 3)


def render_frame(frame_bgr, depth_bgr, rp, want_info=False, ctx=None):
    """One iteration of the render_sbs_3d loop body (core/render_3d.py:1227-1419) on host
    uint8 frames; returns the packed BGR frame (and vd3d_frame_info)."""
    ctx = ctx or _ctx()
    f = np.ascontiguousarray(frame_bgr, dtype=np.uint8)
    d = np.ascontiguousarray(depth_bgr, dtype=np.uint8)
    dch = 1 if d.ndim == 2 else d.shape[2]
    sh, sw = f.shape[:2]
    pl = plan_sizes(sw, sh, rp)
    out = np.empty(output_shape(rp, pl), dtype=np.uint8)
    info = FrameInfo()
    ctx.check(ctx.lib.vd3d_render_frame(ctx.h, f.ctypes.data, d.ctypes.data, dch, sh, sw, C.byref(rp),
                                        out.ctypes.data, _lib.MEM_HOST, C.byref(info) if want_info else None))
    return (out, info) if want_info else out


def advance_state(frame_bgr, depth_bgr, rp, ctx=None):
    """One loop iteration without rendering (temporal state only): the building block of exact
    multi-GPU frame sharding (visiondepth3d_b200/sharding.py)."""
    ctx = ctx or _ctx()
    f = np.ascontiguousarray(frame_bgr, dtype=np.uint8)
    d = np.ascontiguousarray(depth_bgr, dtype=np.uint8)
    dch = 1 if d.ndim == 2 else d.shape[2]
    ctx.check(ctx.lib.vd3d_advance_state(ctx.h, f.ctypes.data, d.ctypes.data, dch, f.shape[0], f.shape[1],
                                         C.byref(rp), _lib.MEM_HOST))


class _ClipWindow:
    """Frame-index arithmetic of render_sbs_3d's optional clip window (core/render_3d.py:986-1030): times are clamped
    to the clip, converted to frame indices by rounding, and a window shorter than half a millisecond is empty.
    `budget` is the number of loop iterations (the whole clip when the window has no frames of its own)."""

    def __init__(self, n_frames, fps, start_s, end_s):
        length_ms = (n_frames / max(fps, 1e-6)) * 1000.0
        t0 = max(0.0, (start_s or 0.0) * 1000.0)
        t1 = length_ms if end_s is None else min(length_ms, end_s * 1000.0)
        self.empty = t0 >= t1 - 0.5
        self.first = int(round(t0 / 1000.0 * fps))
        self.stop = int(round(t1 / 1000.0 * fps))
        span = max(0, self.stop - self.first)
        self.budget = span if span > 0 else n_frames
        self.bounded = end_s is not None


class _PinnedRing:
    """n page-locked host buffers of `shape` u8 (cudaMallocHost through the C ABI) viewed as numpy arrays."""

    def __init__(self, lib, n, shape):
        self.lib, self.ptrs, self.arrays = lib, [], []
        nbytes = int(np.prod(shape))
        for _ in range(n):
            p = lib.vd3d_host_alloc(nbytes)
            if not p:
                self.close()
                raise MemoryError("vd3d_host_alloc failed")
            self.ptrs.append(p)
            self.arrays.append(np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p)).reshape(shape))

    def close(self):
        self.arrays = []
        for p in self.ptrs:
            self.lib.vd3d_host_free(p)
        self.ptrs = []


class _FrameSink:
    """Where packed frames go: raw bgr24 into an ffmpeg stdin pipe (core/render_3d.py:1143-1163, 1422-1427) or a
    cv2.VideoWriter (1164-1169)."""

    def __init__(self, path, size, fps, fourcc, use_ffmpeg, ffmpeg_codec, crf):
        import cv2
        self.proc = self.writer = None
        w, h = size
        if use_ffmpeg:
            import subprocess
            cmd = ["ffmpeg", "-y", "-f", "rawvideo", "-vcodec", "rawvideo", "-pix_fmt", "bgr24", "-s", f"{w}x{h}",
                   "-r", str(fps), "-i", "-", "-an", "-c:v", str(ffmpeg_codec), "-preset", "slow", "-pix_fmt", "yuv420p"]
            if str(ffmpeg_codec).startswith("libx"):
                cmd += ["-crf", str(crf)]
            elif "nvenc" in str(ffmpeg_codec):
                cmd += ["-cq", str(crf), "-b:v", "0"]
            self.proc = subprocess.Popen(cmd + [path], stdin=subprocess.PIPE)
        else:
            self.writer = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*fourcc), fps, (w, h))

    def ok(self):
        return self.proc is not None or (self.writer is not None and self.writer.isOpened())

    def write(self, frame):
        if self.proc is not None:
            self.proc.stdin.write(memoryview(frame).cast("B"))
        else:
            self.writer.write(frame)

    def close(self):
        if self.proc is not None:
            try:
                self.proc.stdin.close()
                self.proc.wait()
            except Exception:
                pass
        if self.writer is not None:
            try:
                self.writer.release()
            except Exception:
                pass


_BATCH = 8  # frames per vd3d_render_clip call of the video loop (3 of them in flight on the device)
_LOOKAHEAD = 3  # runs of up to _RUN pairs in flight between the reader and the two stream workers of render_sbs_3d
_RUN = 4


def render_sbs_3d(
    input_path, depth_path, output_path, selected_codec, fps, output_width, output_height,
    fg_shift, mg_shift, bg_shift, sharpness_factor, output_format, selected_aspect_ratio,
    aspect_ratios, dof_strength, feather_strength=0.0, blur_ksize=1, use_ffmpeg=False,
    selected_ffmpeg_codec=None, crf_value=23, use_subject_tracking=False, use_floating_window=False,
    max_pixel_shift_percent=0.02, progress=None, progress_label=None, suspend_flag=None,
    cancel_flag=None, auto_crop_black_bars=False, parallax_balance=0.8,
    preserve_original_aspect=False, zero_parallax_strength=0.0, enable_edge_masking=True,
    enable_feathering=True, skip_blank_frames=False, original_video_width=None,
    original_video_height=None, convergence_strength=0.0, enable_dynamic_convergence=True,
    ipd_factor=1.0, depth_pop_gamma=0.85, depth_pop_mid=0.50, depth_stretch_lo=0.05,
    depth_stretch_hi=0.95, fg_pop_multiplier=1.20, bg_push_multiplier=1.10,
    subject_lock_strength=1.00, color_saturation=1.0, color_contrast=1.0, color_brightness=0.0,
    start_s=None, end_s=None,
):
    """core/render_3d.py:933-1504: video in -> video out.

    Three stages run concurrently: reader threads decode the colour and the depth stream in parallel (cv2) into a
    ring of page-locked buffers, the calling thread hands batches of them to vd3d_render_clip (H2D | kernels | D2H pipelined over three
    streams, CUDA-graph replay), and a writer thread pushes the packed frames of the previous batch as raw bgr24 into
    an ffmpeg pipe (use_ffmpeg, when the binary exists) or a cv2.VideoWriter.  Sequencing follows the reference:
    first pair of the window dropped, pop controls and parallax_balance not forwarded (1284-1331), no exception
    escapes (1477-1478).  auto_crop_black_bars detects and crops the black bars of every frame on the GPU
    (vd3d_detect_black_bars on the dropped first frame, then per frame inside vd3d_render_clip) and prints the
    reference's lines; skip_blank_frames (an external ffmpeg blackdetect pass) is outside the hot path: refused with a
    message before any file is created."""
    import queue
    import shutil
    import cv2
    if skip_blank_frames:
        print("⚠️ skip_blank_frames (ffmpeg blackdetect) is outside the GPU hot path")
        return
    if use_ffmpeg and shutil.which("ffmpeg") is None:
        print("⚠️ ffmpeg binary not found: writing through cv2.VideoWriter instead")
        use_ffmpeg = False
    cap, dcap = cv2.VideoCapture(input_path), cv2.VideoCapture(depth_path)
    if not cap.isOpened() or not dcap.isOpened():
        return
    n_frames = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
    fps = cap.get(cv2.CAP_PROP_FPS) or fps or 30.0        # the container's rate wins over the argument (993)
    win = _ClipWindow(n_frames, fps, start_s, end_s)
    sink = ring_in = ring_out = free_in = None
    stop = threading.Event()
    threads = []
    try:
        if win.empty:
            print("⚠️ Invalid clip window; nothing to render.")
            return
        cap.set(cv2.CAP_PROP_POS_FRAMES, win.first)
        dcap.set(cv2.CAP_PROP_POS_FRAMES, win.first)
        ok_a, probe = cap.read()
        ok_b, probe_d = dcap.read()
        if not (ok_a and ok_b):
            return
        suspend_flag = suspend_flag or globals()["suspend_flag"]
        cancel_flag = cancel_flag or globals()["cancel_flag"]
        ratio = aspect_ratios.get(selected_aspect_ratio.get(), 16 / 9)
        sh, sw = probe.shape[:2]
        ctx = _ctx()
        if auto_crop_black_bars:  # detected on the first pair, the one the loop drops (1065-1070)
            top, bottom = C.c_int(), C.c_int()
            probe = np.ascontiguousarray(probe)
            ctx.check(ctx.lib.vd3d_detect_black_bars(ctx.h, probe.ctypes.data, sh, sw, _lib.MEM_HOST, C.byref(top),
                                                     C.byref(bottom)))
            print(f"Auto-crop: Top {top.value}px | Bottom {bottom.value}px")
            if preserve_original_aspect and (original_video_width is None or original_video_height is None):
                # the output size falls back to the cropped first frame (1086-1090)
                original_video_width = sw
                original_video_height = sh - top.value - bottom.value if top.value + bottom.value < sh else sh
        rp = make_render_params(
            output_width, output_height, fg_shift, mg_shift, bg_shift, sharpness_factor, output_format, ratio,
            dof_strength, feather_strength, blur_ksize, use_subject_tracking, use_floating_window,
            max_pixel_shift_percent, preserve_original_aspect, zero_parallax_strength, enable_edge_masking,
            enable_feathering, original_video_width, original_video_height, convergence_strength,
            enable_dynamic_convergence, ipd_factor, color_saturation, color_contrast, color_brightness,
            auto_crop_black_bars)
        dch = 1 if probe_d.ndim == 2 else probe_d.shape[2]
        pl = plan_sizes(sw, sh, rp)                     # raises before any output file exists
        oshape = output_shape(rp, pl)
        ctx.check(ctx.lib.vd3d_check_config(ctx.h, sh, sw, C.byref(rp)))   # eye fit / DOF limits, still no file
        sink = _FrameSink(output_path, (oshape[1], oshape[0]), fps, selected_codec, use_ffmpeg, selected_ffmpeg_codec,
                          crf_value)
        if not sink.ok():
            print("❌ OpenCV VideoWriter failed to open. Check codec/fourcc and path.")
            return
        ctx.reset(_lib.STATE_CLIP)  # ShiftSmoother / TemporalDepthFilter / FocalDepthTracker are per render (1174-1182)
        ring_in = (_PinnedRing(ctx.lib, 3 * _BATCH, (sh, sw, 3)), _PinnedRing(ctx.lib, 3 * _BATCH, probe_d.shape))
        ring_out = _PinnedRing(ctx.lib, 2 * _BATCH, oshape)
        free_in, ready = queue.Queue(), queue.Queue(maxsize=3 * _BATCH)
        for k in range(3 * _BATCH):
            free_in.put(k)
        to_write, free_out = queue.Queue(), queue.Queue()
        free_out.put(0)
        free_out.put(1)
        errors = []

        # the colour and the depth stream are decoded (cv2 releases the GIL) and copied into the pinned ring by one
        # worker thread each; `reader` sequences them exactly like the reference's loop consumes pairs
        q_jobs = (queue.Queue(), queue.Queue())
        q_done = (queue.Queue(), queue.Queue())

        def stream_worker(which, src):
            while True:
                ks = q_jobs[which].get()
                if ks is None:
                    return
                n_ok = 0
                try:
                    for k in ks:                        # a run of ring slots (-1: read and drop)
                        ok, img = src.read()
                        if not ok:
                            break
                        if k >= 0:
                            np.copyto(ring_in[which].arrays[k], img)
                        n_ok += 1
                except Exception as e:
                    errors.append(e)
                q_done[which].put(n_ok)

        def collect_run():
            """Pairs of the oldest run that both streams delivered (a decoder that stalls for a minute counts as a failed
            read; the reference would block forever)."""
            try:
                return min(q_done[0].get(timeout=60), q_done[1].get(timeout=60))
            except queue.Empty:
                return 0

        def issue_run(ks):
            q_jobs[0].put(ks)
            q_jobs[1].put(ks)

        def reader():
            # Runs of up to _RUN pairs are handed to the two stream workers, _LOOKAHEAD runs ahead of the one being
            # collected, so the decoders / copies of both streams work back to back instead of meeting at a barrier after
            # every frame (and the queue traffic is per run, not per frame); pairs are still published in order.  A
            # bounded window stops after the pair that reaches its last frame (the reference checks
            # CAP_PROP_POS_FRAMES >= stop after each read, 1196-1199): counted here, because the decoders run ahead of
            # the published position.
            import collections
            try:
                cap.set(cv2.CAP_PROP_POS_FRAMES, win.first)
                dcap.set(cv2.CAP_PROP_POS_FRAMES, win.first)
                issue_run([-1])                         # the first pair of the window is read and dropped (1184-1188)
                limit = max(win.budget - 1, 1) if win.bounded else win.budget
                inflight, issued, closed = collections.deque(), 0, collect_run() != 1
                while True:
                    while not closed and issued < limit and len(inflight) < _LOOKAHEAD:
                        while suspend_flag.is_set() and not cancel_flag.is_set():
                            time.sleep(0.2)
                        if cancel_flag.is_set():
                            closed = True
                            break
                        ks = []
                        try:
                            while len(ks) < min(_RUN, limit - issued):
                                k = free_in.get() if not (inflight or ks) else free_in.get_nowait()
                                if stop.is_set() or k < 0:
                                    closed = True
                                    break
                                ks.append(k)
                        except queue.Empty:
                            pass                        # no more free slots right now
                        if not ks:
                            break                       # collect a finished run first
                        issue_run(ks)
                        inflight.append(ks)
                        issued += len(ks)
                    if not inflight:
                        break
                    ks = inflight.popleft()
                    n_ok = collect_run()
                    for k in ks[:n_ok]:
                        ready.put(k)
                    if n_ok < len(ks):
                        break                           # end of either stream (or a failed read): nothing after it counts
            except Exception as e:  # surfaced by the main thread
                errors.append(e)
            q_jobs[0].put(None)
            q_jobs[1].put(None)
            ready.put(None)

        def writer():
            while True:
                item = to_write.get()
                if item is None:
                    return
                half, n = item
                try:
                    for j in range(n):
                        sink.write(ring_out.arrays[half * _BATCH + j])
                except Exception as e:
                    print(f"❌ FFmpeg write error: {e}" if use_ffmpeg else f"❌ write error: {e}")
                    errors.append(e)
                free_out.put(half)

        th_r = threading.Thread(target=reader, daemon=True)
        th_w = threading.Thread(target=writer, daemon=True)
        threads += [threading.Thread(target=stream_worker, args=(which, src), daemon=True)
                    for which, src in enumerate((cap, dcap))] + [th_r]
        for t in threads:
            t.start()
        th_w.start()
        n_done, t0, eof = 0, time.time(), False
        while not eof and not errors:
            slots = []
            while len(slots) < _BATCH:
                k = ready.get(timeout=180)
                if k is None:
                    eof = True
                    break
                slots.append(k)
            if not slots:
                break
            half = free_out.get()
            n = len(slots)
            fp = (C.c_void_p * n)(*[ring_in[0].ptrs[k] for k in slots])
            dp = (C.c_void_p * n)(*[ring_in[1].ptrs[k] for k in slots])
            op = (C.c_void_p * n)(*[ring_out.ptrs[half * _BATCH + j] for j in range(n)])
            ctx.check(ctx.lib.vd3d_render_clip(ctx.h, n, fp, dp, dch, sh, sw, C.byref(rp), op, _lib.MEM_HOST, None))
            if auto_crop_black_bars:  # the reference prints one line per frame (1238-1240)
                tb = (C.c_int32 * (2 * n))()
                ctx.check(ctx.lib.vd3d_last_crops(ctx.h, tb, n))
                for j in range(n):
                    print(f"🔪 Cropping top: {tb[2 * j]}px, bottom: {tb[2 * j + 1]}px")
            for k in slots:
                free_in.put(k)
            to_write.put((half, n))
            n_done += n
            frac = min(n_done / max(win.budget, 1), 1.0) * 100.0
            if progress:
                progress["value"] = frac
                progress.update()
            if progress_label:
                el = time.time() - t0
                rate = n_done / max(el, 1e-9)
                eta = (win.budget - n_done) / rate if rate > 0 else 0
                progress_label.config(text=f"{frac:.2f}% | FPS: {rate:.2f} | Elapsed: "
                                           f"{time.strftime('%H:%M:%S', time.gmtime(el))} | ETA: "
                                           f"{time.strftime('%H:%M:%S', time.gmtime(max(eta, 0)))}")
        to_write.put(None)
        th_w.join()
        if progress and not cancel_flag.is_set():
            progress["value"] = 100
            progress.update()
    except Exception as e:  # the reference prints and returns None (1477-1478)
        print(f"❌ Render crashed: {e}")
    finally:
        stop.set()
        if free_in is not None:
            free_in.put(-1)   # wake a reader that waits for a free slot
        for t in threads:     # nobody may still be inside cap.read() / the pinned ring when they go away
            t.join(timeout=5.0)
        cap.release()
        dcap.release()
        if sink is not None:
            sink.close()
        try:
            if ring_in is not None:
                _ctx().check(_ctx().lib.vd3d_sync(_ctx().h))
                ring_in[0].close()
                ring_in[1].close()
            if ring_out is not None:
                ring_out.close()
        except Exception:
            pass


# ---------------------------------------------------------------------------
# GUI-facing entry points the reference's callers import (VisionDepth3D.py:25-38).  The dialogs themselves are Tk and
# outside the hot path; the functions keep the reference's call shape so the import list resolves.
# ---------------------------------------------------------------------------
# the GUI's encoder vocabulary -> ffmpeg encoder names (interface constants, core/render_3d.py:49-73)
FFMPEG_CODEC_MAP = {
    "H.264 / AVC (libx264 - CPU)": "libx264", "H.265 / HEVC (libx265 - CPU)": "libx265",
    "AV1 (libaom - CPU)": "libaom-av1", "AV1 (SVT - CPU, faster)": "libsvtav1",
    "MPEG-4 (mp4v - CPU)": "mp4v", "XviD (AVI - CPU)": "XVID", "DivX (AVI - CPU)": "DIVX",
    "H.264 / AVC (NVENC - NVIDIA GPU)": "h264_nvenc", "H.265 / HEVC (NVENC - NVIDIA GPU)": "hevc_nvenc",
    "AV1 (NVENC - NVIDIA RTX 40+ GPU)": "av1_nvenc",
    "H.264 / AVC (AMF - AMD GPU)": "h264_amf", "H.265 / HEVC (AMF - AMD GPU)": "hevc_amf",
    "AV1 (AMF - AMD RDNA3+)": "av1_amf",
    "H.264 / AVC (QSV - Intel GPU)": "h264_qsv", "H.265 / HEVC (QSV - Intel GPU)": "hevc_qsv",
    "VP9 (QSV - Intel GPU)": "vp9_qsv", "AV1 (QSV - Intel ARC / Gen11+)": "av1_qsv",
}
original_video_width = None
original_video_height = None


def _val(v):
    return v.get() if hasattr(v, "get") else v


def process_video(
    input_video_path, selected_depth_map, output_sbs_video_path, selected_codec, fg_shift, mg_shift, bg_shift,
    sharpness_factor, output_format, selected_aspect_ratio, aspect_ratios, feather_strength, blur_ksize, progress,
    progress_label, suspend_flag, cancel_flag, use_ffmpeg, selected_ffmpeg_codec, crf_value, use_subject_tracking,
    use_floating_window, max_pixel_shift, auto_crop_black_bars, parallax_balance, preserve_original_aspect,
    zero_parallax_strength, enable_edge_masking, enable_feathering, skip_blank_frames, dof_strength,
    convergence_strength, enable_dynamic_convergence, depth_pop_gamma, depth_pop_mid, depth_stretch_lo,
    depth_stretch_hi, fg_pop_multiplier, bg_push_multiplier, subject_lock_strength, color_saturation,
    color_contrast, color_brightness, ipd_value=0.0, start_s=None, end_s=None,
):
    """core/render_3d.py:1594-1753: unwrap the GUI variables (anything with .get()), derive the output size from the
    source video and the format, and run render_sbs_3d for the four SBS-family formats (VR is not dispatched by the
    reference either).  Errors the reference reports through message boxes are printed."""
    global original_video_width, original_video_height
    import cv2
    src, dep, dst = _val(input_video_path), _val(selected_depth_map), _val(output_sbs_video_path)
    if not src or not dst or not dep:
        print("Error: Please select input video, depth map, and output path.")
        return
    probe = cv2.VideoCapture(src)
    width = int(probe.get(cv2.CAP_PROP_FRAME_WIDTH))
    height = int(probe.get(cv2.CAP_PROP_FRAME_HEIGHT))
    rate = probe.get(cv2.CAP_PROP_FPS)
    probe.release()
    if rate <= 0:
        print("Error: Unable to retrieve FPS from the input video.")
        return
    original_video_width, original_video_height = width, height
    ratio = aspect_ratios.get(_val(selected_aspect_ratio), 16 / 9)
    fmt = _val(output_format)
    if _val(preserve_original_aspect) or fmt == "Half-SBS":
        out_w, out_h = width, height
    elif fmt == "Full-SBS":
        out_w, out_h = width * 2, height
    elif fmt == "VR":
        out_w, out_h = 4096, int(4096 / ratio)
    else:
        out_w, out_h = width, int(width / ratio)
    if progress is not None:
        progress["value"] = 0
        progress.update()
    if progress_label is not None:
        progress_label.config(text="0%")
    if fmt not in ("Full-SBS", "Half-SBS", "Red-Cyan Anaglyph", "Passive Interlaced"):
        return
    codec_name = _val(selected_ffmpeg_codec)
    render_sbs_3d(
        src, dep, dst, _val(selected_codec), rate, out_w, out_h, _val(fg_shift), _val(mg_shift), _val(bg_shift),
        _val(sharpness_factor), fmt, selected_aspect_ratio, aspect_ratios,
        feather_strength=_val(feather_strength), blur_ksize=_val(blur_ksize), use_ffmpeg=_val(use_ffmpeg),
        selected_ffmpeg_codec=FFMPEG_CODEC_MAP.get(codec_name, codec_name), crf_value=_val(crf_value),
        use_subject_tracking=_val(use_subject_tracking), use_floating_window=_val(use_floating_window),
        max_pixel_shift_percent=_val(max_pixel_shift), progress=progress, progress_label=progress_label,
        suspend_flag=suspend_flag, cancel_flag=cancel_flag, auto_crop_black_bars=_val(auto_crop_black_bars),
        parallax_balance=_val(parallax_balance), preserve_original_aspect=_val(preserve_original_aspect),
        zero_parallax_strength=_val(zero_parallax_strength), enable_edge_masking=_val(enable_edge_masking),
        enable_feathering=_val(enable_feathering), skip_blank_frames=_val(skip_blank_frames),
        dof_strength=_val(dof_strength), original_video_width=width, original_video_height=height,
        convergence_strength=_val(convergence_strength), enable_dynamic_convergence=_val(enable_dynamic_convergence),
        ipd_factor=ipd_value, depth_pop_gamma=_val(depth_pop_gamma), depth_pop_mid=_val(depth_pop_mid),
        depth_stretch_lo=_val(depth_stretch_lo), depth_stretch_hi=_val(depth_stretch_hi),
        fg_pop_multiplier=_val(fg_pop_multiplier), bg_push_multiplier=_val(bg_push_multiplier),
        subject_lock_strength=_val(subject_lock_strength), color_saturation=_val(color_saturation),
        color_contrast=_val(color_contrast), color_brightness=_val(color_brightness), start_s=start_s, end_s=end_s)


def _dialog(kind, **kw):
    try:
        from tkinter import filedialog
    except Exception as e:  # headless box: the dialogs are GUI-only
        raise RuntimeError("file dialogs need tkinter (GUI helper, outside the GPU hot path)") from e
    return getattr(filedialog, kind)(**kw)


_VIDEO_TYPES = [("Video files", "*.mp4 *.avi *.mkv")]


def select_input_video(input_video_path, video_thumbnail_label, video_specs_label, update_aspect_preview,
                       original_video_width, original_video_height):
    """core/render_3d.py:1507-1556 without the thumbnail: pick a file, publish its size / fps to the GUI variables."""
    import cv2
    path = _dialog("askopenfilename", filetypes=_VIDEO_TYPES)
    if not path:
        return
    input_video_path.set(path)
    cap = cv2.VideoCapture(path)
    if not cap.isOpened():
        print("Error: Unable to open video file.")
        return
    w, h = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
    rate = cap.get(cv2.CAP_PROP_FPS)
    cap.release()
    original_video_width.set(w)
    original_video_height.set(h)
    if video_specs_label is not None:
        video_specs_label.config(text=f"Video Info:\nResolution: {w}x{h}\nFPS: {rate:.2f}")
    if update_aspect_preview is not None:
        update_aspect_preview()


def select_output_video(output_sbs_video_path):
    """core/render_3d.py:1568-1578."""
    output_sbs_video_path.set(_dialog("asksaveasfilename", defaultextension=".mp4",
                                      filetypes=[("MP4 files", "*.mp4"), ("MKV files", "*.mkv"), ("AVI files", "*.avi")]))


def select_depth_map(selected_depth_map, depth_map_label):
    """core/render_3d.py:1581-1591."""
    import os
    path = _dialog("askopenfilename", filetypes=_VIDEO_TYPES)
    if not path:
        return
    selected_depth_map.set(path)
    if depth_map_label is not None:
        depth_map_label.config(text=f"Selected Depth Map:\n{os.path.basename(path)}")
