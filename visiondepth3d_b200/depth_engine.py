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
    lib.vd3d_depth_infer_images.argtypes = [vp, i, C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(vp), C.POINTER(vp), i,
                                            i]
    lib.vd3d_depth_infer_images.restype = i
    lib.vd3d_depth_resize_pil.argtypes = [vp, vp, i, i, vp, i, i, i]
    lib.vd3d_depth_resize_pil.restype = i
    lib.vd3d_pil_bicubic_table.argtypes = [i, i, vp, vp, i]
    lib.vd3d_pil_bicubic_table.restype = i
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

    def infer_images(self, images_rgb, input_sizes=None, invert=False, want_f32=False):
        """vd3d_depth_infer_images: up to 8 RGB u8 images [h,w,3] of their own sizes -> list of (min-max u8 depth at
        the image's size, predicted_depth f32 at its input size or None), with one batched forward.  input_sizes: one
        (W, H) or None (the image's own size) per image; every input size must map to this engine's processed size.
        images_rgb: host arrays, or CUDA uint8 tensors (the results are then CUDA tensors)."""
        import torch
        n = len(images_rgb)
        if not 1 <= n <= 8:
            raise ValueError("infer_images takes 1..8 images")
        input_sizes = list(input_sizes) if input_sizes is not None else [None] * n
        if len(input_sizes) != n:
            raise ValueError("one input size (or None) per image")
        device = isinstance(images_rgb[0], torch.Tensor) and images_rgb[0].is_cuda
        if device:
            imgs = [t.contiguous() for t in images_rgb]
            if any(t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3 or not t.is_cuda for t in imgs):
                raise ValueError("expected CUDA uint8 tensors [h, w, 3]")
        else:
            imgs = [np.ascontiguousarray(a, dtype=np.uint8) for a in images_rgb]
            if any(a.ndim != 3 or a.shape[2] != 3 for a in imgs):
                raise ValueError("expected RGB uint8 arrays [h, w, 3]")
        sizes = np.empty((n, 4), np.int32)
        for k, (img, ins) in enumerate(zip(imgs, input_sizes)):
            sh, sw = int(img.shape[0]), int(img.shape[1])
            iw, ih = (sw, sh) if ins is None else (int(ins[0]), int(ins[1]))
            if processed_size(iw, ih) != (self.image_h, self.image_w):
                raise ValueError(f"engine built for processed size {(self.image_h, self.image_w)}, a {iw}x{ih} input "
                                 f"needs {processed_size(iw, ih)}")
            sizes[k] = sh, sw, ih, iw
        if device:
            dev = imgs[0].device
            u8 = [torch.empty((int(s[0]), int(s[1])), dtype=torch.uint8, device=dev) for s in sizes]
            f32 = [torch.empty((int(s[2]), int(s[3])), dtype=torch.float32, device=dev) for s in sizes] if want_f32 else None
            ptr, mem = (lambda t: t.data_ptr()), _lib.MEM_DEVICE
            torch.cuda.current_stream().synchronize()  # the images may come from work queued on torch's stream
        else:
            u8 = [np.empty((int(s[0]), int(s[1])), np.uint8) for s in sizes]
            f32 = [np.empty((int(s[2]), int(s[3])), np.float32) for s in sizes] if want_f32 else None
            ptr, mem = (lambda a: a.ctypes.data), _lib.MEM_HOST
        vp = C.c_void_p
        self.check(self.lib.vd3d_depth_infer_images(
            self.h, n, (vp * n)(*[ptr(a) for a in imgs]), sizes.ctypes.data_as(C.POINTER(C.c_int32)),
            (vp * n)(*[ptr(a) for a in u8]), (vp * n)(*[ptr(a) for a in f32]) if want_f32 else None,
            int(bool(invert)), mem))
        if device:
            self.ctx.check(self.lib.vd3d_sync(self.ctx.h))
        return list(zip(u8, f32 if want_f32 else [None] * n))

    def resize_pil(self, rgb, width, height):
        """vd3d_depth_resize_pil: Image.fromarray(rgb).resize((width, height), Image.BICUBIC) on a host RGB u8
        [h,w,3] array, on the GPU."""
        src = np.ascontiguousarray(rgb, dtype=np.uint8)
        if src.ndim != 3 or src.shape[2] != 3:
            raise ValueError("expected an RGB uint8 array [h, w, 3]")
        out = np.empty((int(height), int(width), 3), np.uint8)
        self.check(self.lib.vd3d_depth_resize_pil(self.h, src.ctypes.data, src.shape[0], src.shape[1], out.ctypes.data,
                                                  int(height), int(width), _lib.MEM_HOST))
        return out

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
