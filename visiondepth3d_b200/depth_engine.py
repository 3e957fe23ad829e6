"""ctypes wrapper of the libvd3d depth engine (include/vd3d.h, "depth forward")."""
import ctypes as C
import sys as _sys

import numpy as np

from . import _lib
from .depth_weights import CONFIGS, prepare


def processed_size(width, height, target=518, multiple=14):
    """(h, w) the DPT image processor resizes a (width, height) image to: keep the aspect ratio, scale the side
    that is closer to `target`, round both to multiples of 14 (transformers image_processing_dpt.py,
    get_resize_output_image_size with keep_aspect_ratio=True, ensure_multiple_of=14)."""
    sh, sw = target / height, target / width
    if abs(1 - sw) < abs(1 - sh):
        sh = sw
    else:
        sw = sh
    rnd = lambda v: max(multiple, int(round(v / multiple) * multiple))  # noqa: E731
    return rnd(sh * height), rnd(sw * width)


class DepthConfig(C.Structure):
    _fields_ = [("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32), ("taps", C.c_int32 * 4),
                ("neck", C.c_int32 * 4), ("fusion", C.c_int32), ("image_h", C.c_int32), ("image_w", C.c_int32)]


def _bind(lib):
    if getattr(lib, "_depth_bound", False):
        return
    vp, i = C.c_void_p, C.c_int
    lib.vd3d_depth_create.argtypes = [C.POINTER(DepthConfig), vp, C.POINTER(vp)]
    lib.vd3d_depth_create.restype = i
    lib.vd3d_depth_destroy.argtypes = [vp]
    lib.vd3d_depth_destroy.restype = None
    lib.vd3d_depth_last_error.argtypes = [vp]
    lib.vd3d_depth_last_error.restype = C.c_char_p
    lib.vd3d_depth_launch_count.argtypes = [vp]
    lib.vd3d_depth_launch_count.restype = C.c_uint64
    lib.vd3d_depth_set_tensor.argtypes = [vp, C.c_char_p, vp, C.c_size_t]
    lib.vd3d_depth_set_tensor.restype = i
    lib.vd3d_depth_forward.argtypes = [vp, vp, vp, i]
    lib.vd3d_depth_forward.restype = i
    lib.vd3d_depth_get_buffer.argtypes = [vp, C.c_char_p, vp, C.c_size_t]
    lib.vd3d_depth_get_buffer.restype = i
    lib.vd3d_gemm_f16.argtypes = [vp, vp, vp, i, i, i, vp, i]
    lib.vd3d_gemm_f16.restype = i
    lib.vd3d_gemm_bench.argtypes = [vp, i, i, i, i, i, i, i, C.POINTER(C.c_float)]
    lib.vd3d_gemm_bench.restype = i
    lib.vd3d_conv_f16.argtypes = [vp, vp, i, i, i, vp, i, i, vp, i, vp]
    lib.vd3d_conv_f16.restype = i
    lib.vd3d_depth_infer.argtypes = [vp, vp, i, i, vp, vp, i]
    lib.vd3d_depth_infer.restype = i
    lib.vd3d_depth_infer_device.argtypes = [vp, vp, i, i, vp, vp, i]
    lib.vd3d_depth_infer_device.restype = i
    lib.vd3d_depth_infer_batch.argtypes = [vp, i, C.POINTER(vp), i, i, C.POINTER(vp), C.POINTER(vp), i]
    lib.vd3d_depth_infer_batch.restype = i
    lib.vd3d_depth_infer_batch_device.argtypes = [vp, i, C.POINTER(vp), i, i, C.POINTER(vp), C.POINTER(vp), i]
    lib.vd3d_depth_infer_batch_device.restype = i
    lib.vd3d_depth_profile.argtypes = [vp, i]
    lib.vd3d_depth_profile.restype = i
    lib.vd3d_depth_profile_collect.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(i), C.POINTER(C.c_double)]
    lib.vd3d_depth_profile_collect.restype = i
    lib.vd3d_depth_profile_spans.argtypes = [vp, C.c_char_p, C.c_size_t]
    lib.vd3d_depth_profile_spans.restype = i
    lib._depth_bound = True


class DepthEngine:
    """Depth-Anything-V2 forward on wgmma tensor cores.  `cfg` is a key of CONFIGS or a dict."""

    def __init__(self, cfg="vits", image_h=518, image_w=924, ctx=None, device=0):
        self.lib = _lib.load()
        _bind(self.lib)
        self.ctx = ctx or _lib.default_context(device)
        self.cfg = dict(CONFIGS[cfg]) if isinstance(cfg, str) else dict(cfg)
        self.image_h, self.image_w = int(image_h), int(image_w)
        c = self.cfg
        dc = DepthConfig(c["hidden"], c["layers"], c["heads"], (C.c_int32 * 4)(*c["taps"]),
                         (C.c_int32 * 4)(*c["neck"]), c["fusion"], self.image_h, self.image_w)
        h = C.c_void_p()
        rc = self.lib.vd3d_depth_create(C.byref(dc), self.lib.vd3d_stream(self.ctx.h), C.byref(h))
        if rc != 0:
            raise _lib.Vd3dError(f"vd3d_depth_create failed ({rc})")
        self.h = h

    def check(self, rc):
        if rc != 0:
            raise _lib.Vd3dError(f"libvd3d depth error {rc}: {self.lib.vd3d_depth_last_error(self.h).decode()}")

    def load_state_dict(self, sd):
        for name, arr in prepare(sd, self.cfg, self.image_h, self.image_w).items():
            arr = np.ascontiguousarray(arr)
            self.check(self.lib.vd3d_depth_set_tensor(self.h, name.encode(), arr.ctypes.data, arr.nbytes))

    def forward(self, pixel_values):
        """pixel_values: f32 [3, image_h, image_w] numpy (host) or CUDA torch tensor -> depth f32 [H, W]."""
        try:
            import torch
        except Exception:  # pragma: no cover
            torch = None
        if torch is not None and isinstance(pixel_values, torch.Tensor) and pixel_values.is_cuda:
            pv = pixel_values.contiguous().float()
            out = torch.empty((self.image_h, self.image_w), dtype=torch.float32, device=pv.device)
            torch.cuda.current_stream().synchronize()
            self.check(self.lib.vd3d_depth_forward(self.h, pv.data_ptr(), out.data_ptr(), _lib.MEM_DEVICE))
            self.ctx.check(self.lib.vd3d_sync(self.ctx.h))
            return out
        pv = np.ascontiguousarray(np.asarray(pixel_values, dtype=np.float32))
        out = np.empty((self.image_h, self.image_w), dtype=np.float32)
        self.check(self.lib.vd3d_depth_forward(self.h, pv.ctypes.data, out.ctypes.data, _lib.MEM_HOST))
        return out

    def infer(self, frame_bgr, invert=False, check_size=True):
        """BGR u8 [h,w,3] -> (predicted_depth f32 [h,w] resized to the frame, min-max u8 [h,w]).
        check_size: refuse frames whose DPT processed size differs from the one this engine was built for (the HF
        processor would pick another keep-aspect /14 size, so the depth would differ from the reference's)."""
        f = np.ascontiguousarray(frame_bgr, dtype=np.uint8)
        h, w = f.shape[:2]
        if check_size and processed_size(w, h) != (self.image_h, self.image_w):
            raise ValueError(f"engine built for processed size {(self.image_h, self.image_w)}, a {w}x{h} frame needs "
                             f"{processed_size(w, h)}")
        d32 = np.empty((h, w), dtype=np.float32)
        d8 = np.empty((h, w), dtype=np.uint8)
        self.check(self.lib.vd3d_depth_infer(self.h, f.ctypes.data, h, w, d32.ctypes.data, d8.ctypes.data,
                                             int(bool(invert))))
        return d32, d8

    def infer_batch(self, frames_bgr, invert=False, check_size=True):
        """List of same-shape BGR frames -> list of (predicted_depth f32, min-max u8), up to 8 frames per batched
        forward (the token-wise GEMMs run on the stacked token matrix of the batch)."""
        frames = [np.ascontiguousarray(f, dtype=np.uint8) for f in frames_bgr]
        if not frames:
            return []
        h, w = frames[0].shape[:2]
        if any(f.shape[:2] != (h, w) for f in frames):
            raise ValueError("infer_batch needs frames of one shape")
        if check_size and processed_size(w, h) != (self.image_h, self.image_w):
            raise ValueError(f"engine built for processed size {(self.image_h, self.image_w)}, a {w}x{h} frame needs "
                             f"{processed_size(w, h)}")
        out = []
        for i0 in range(0, len(frames), 8):
            chunk = frames[i0:i0 + 8]
            n = len(chunk)
            d32 = [np.empty((h, w), dtype=np.float32) for _ in range(n)]
            d8 = [np.empty((h, w), dtype=np.uint8) for _ in range(n)]
            fp = (C.c_void_p * n)(*[f.ctypes.data for f in chunk])
            p32 = (C.c_void_p * n)(*[a.ctypes.data for a in d32])
            p8 = (C.c_void_p * n)(*[a.ctypes.data for a in d8])
            self.check(self.lib.vd3d_depth_infer_batch(self.h, n, fp, h, w, p32, p8, int(bool(invert))))
            out += list(zip(d32, d8))
        return out

    def infer_batch_u8_device(self, frame_ptrs, h, w, u8_ptrs, invert=False):
        """Device form of infer_batch: up to 8 BGR frames [h,w,3] at device pointers -> min-max u8 depth [h,w] at
        device pointers.  Enqueued on the context's stream; no synchronisation."""
        n = len(frame_ptrs)
        if not 1 <= n <= 8 or len(u8_ptrs) != n:
            raise ValueError("infer_batch_u8_device takes 1..8 frames and one output per frame")
        if processed_size(w, h) != (self.image_h, self.image_w):
            raise ValueError(f"engine built for processed size {(self.image_h, self.image_w)}, a {w}x{h} frame needs "
                             f"{processed_size(w, h)}")
        fp = (C.c_void_p * n)(*frame_ptrs)
        p8 = (C.c_void_p * n)(*u8_ptrs)
        self.check(self.lib.vd3d_depth_infer_batch_device(self.h, n, fp, h, w, p8, None, int(bool(invert))))

    def get_buffer(self, name, shape, dtype):
        out = np.empty(shape, dtype=dtype)
        self.check(self.lib.vd3d_depth_get_buffer(self.h, name.encode(), out.ctypes.data, out.nbytes))
        return out

    def gemm(self, A, B, bn=0):
        A = np.ascontiguousarray(A, dtype=np.float16)
        B = np.ascontiguousarray(B, dtype=np.float16)
        M, K = A.shape
        N = B.shape[0]
        Cc = np.empty((M, N), dtype=np.float32)
        self.check(self.lib.vd3d_gemm_f16(self.h, A.ctypes.data, B.ctypes.data, M, N, K, Cc.ctypes.data, bn))
        return Cc

    def gemm_bench(self, M, N, K, variant=0, dbg=0, act=0, iters=20):
        """Average launch time (ms) of one GEMM shape on device operands (tuning hook, see include/vd3d.h)."""
        ms = C.c_float(0)
        self.check(self.lib.vd3d_gemm_bench(self.h, M, N, K, variant, dbg, act, iters, C.byref(ms)))
        return ms.value

    def conv(self, x_nhwc, w, bias=None, k3=True, relu=False):
        x = np.ascontiguousarray(x_nhwc, dtype=np.float16)
        w = np.ascontiguousarray(w, dtype=np.float16)
        H, W_, cin = x.shape
        cout = w.shape[0]
        out = np.empty((H, W_, cout), dtype=np.float32)
        b = np.ascontiguousarray(bias, dtype=np.float32) if bias is not None else None
        self.check(self.lib.vd3d_conv_f16(self.h, x.ctypes.data, H, W_, cin, w.ctypes.data, cout, int(k3),
                                          b.ctypes.data if b is not None else None, int(relu), out.ctypes.data))
        return out

    @property
    def launches(self):
        return int(self.lib.vd3d_depth_launch_count(self.h))

    def close(self):
        if getattr(self, "h", None):
            if getattr(self.ctx, "h", None):
                self.lib.vd3d_release_depth(self.ctx.h, self.h)
            self.lib.vd3d_depth_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            if _sys is None or _sys.is_finalizing():
                return
            self.close()
        except BaseException:
            pass
