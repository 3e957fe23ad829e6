"""Drop-in for the Real-ESRGAN upscale stage of the reference's core/merged_pipeline.py (run_esrgan and its helpers,
lines 221-284), backed by libvd3d.so: the SRVGGNetCompact network on wgmma implicit-GEMM convolutions, cv2's INTER_AREA
/ INTER_CUBIC resizes and addWeighted as CUDA kernels.  RIFE interpolation, the image-folder driver and the ffmpeg
writer of that module are outside the hot path.

The reference loads `weights/RealESR_Gx4_fp16.onnx` through ONNXRuntime (VisionDepth3D.py:1094-1100); here the model is
an upstream-format state_dict (`body.{i}.weight` ...: realesr-general-x4v3 / realesr-animevideov3 .pth files) handed to
load_esrgan(); without one a random-init model is built (no checkpoints offline).
"""
import ctypes as C

import numpy as np

from . import _lib

esrgan_session = None  # the reference's module global: truthy once a model is loaded


class SrEngine:
    """SRVGGNetCompact (num_feat 64, x4) forward on the GPU: BGR u8 [h,w,3] -> BGR u8 [4h,4w,3]."""

    def __init__(self, state_dict, ctx=None, device=0):
        self.lib = _lib.load()
        self.ctx = ctx or _lib.default_context(device)
        h = C.c_void_p()
        rc = self.lib.vd3d_sr_create(self.lib.vd3d_stream(self.ctx.h), C.byref(h))
        if rc != 0:
            raise _lib.Vd3dError(f"vd3d_sr_create failed ({rc})")
        self.h = h
        self.lib.vd3d_depth_set_tensor.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
        self.lib.vd3d_depth_set_tensor.restype = C.c_int
        self.lib.vd3d_depth_last_error.argtypes = [C.c_void_p]
        self.lib.vd3d_depth_last_error.restype = C.c_char_p
        self.lib.vd3d_depth_destroy.argtypes = [C.c_void_p]
        self.lib.vd3d_depth_destroy.restype = None
        n_conv_total = len([k for k in state_dict if k.endswith(".bias")])
        self.num_conv = n_conv_total - 2
        for i in range(n_conv_total):
            w = np.asarray(state_dict[f"body.{2 * i}.weight"], dtype=np.float32)      # [Cout, Cin, 3, 3]
            co, ci = w.shape[:2]
            if ci > 64 or co > 64:
                raise ValueError("SRVGGNetCompact with num_feat 64 expected")
            packed = np.zeros((co, 9, 64), dtype=np.float32)                          # tap-major, channel-minor
            packed[:, :, :ci] = w.transpose(0, 2, 3, 1).reshape(co, 9, ci)
            self._set(f"sr.c{i}.w", packed.reshape(co, 9 * 64).astype(np.float16))
            self._set(f"sr.c{i}.b", np.asarray(state_dict[f"body.{2 * i}.bias"], dtype=np.float32))
            if i < n_conv_total - 1:
                self._set(f"sr.a{i}", np.asarray(state_dict[f"body.{2 * i + 1}.weight"], dtype=np.float32).reshape(-1))

    def _set(self, name, arr):
        arr = np.ascontiguousarray(arr)
        self.check(self.lib.vd3d_depth_set_tensor(self.h, name.encode(), arr.ctypes.data, arr.nbytes))

    def check(self, rc):
        if rc != 0:
            raise _lib.Vd3dError(f"libvd3d sr error {rc}: {self.lib.vd3d_depth_last_error(self.h).decode()}")

    def upscale(self, frame_bgr):
        f = np.ascontiguousarray(frame_bgr, dtype=np.uint8)
        h, w = f.shape[:2]
        out = np.empty((4 * h, 4 * w, 3), dtype=np.uint8)
        self.check(self.lib.vd3d_sr_forward(self.h, f.ctypes.data, h, w, self.num_conv, out.ctypes.data, _lib.MEM_HOST))
        return out

    def close(self):
        if getattr(self, "h", None):
            self.lib.vd3d_depth_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            import sys
            if sys is None or sys.is_finalizing():
                return
            self.close()
        except BaseException:
            pass


def random_srvgg_state_dict(num_conv=32, seed=0, num_feat=64):
    """Random-init SRVGGNetCompact weights in the upstream naming (He init for PReLU(0.25), small last layer), for
    benchmarks and tests: there are no checkpoints offline."""
    rng = np.random.default_rng(seed)
    sd = {}
    chans = [(3, num_feat)] + [(num_feat, num_feat)] * num_conv + [(num_feat, 48)]
    for i, (ci, co) in enumerate(chans):
        std = (2.0 / (1.0 + 0.25 ** 2) / (9 * ci)) ** 0.5 * (0.1 if i == len(chans) - 1 else 1.0)
        sd[f"body.{2 * i}.weight"] = (rng.standard_normal((co, ci, 3, 3)) * std).astype(np.float32)
        sd[f"body.{2 * i}.bias"] = (rng.standard_normal(co) * 0.02).astype(np.float32)
        if i < len(chans) - 1:
            sd[f"body.{2 * i + 1}.weight"] = (0.25 + 0.1 * rng.random(co)).astype(np.float32)
    return sd


def load_esrgan(state_dict=None, num_conv=32, seed=0):
    """Make run_esrgan serve a model: an upstream SRVGGNetCompact state_dict (tensors or arrays), or random-init."""
    global esrgan_session
    if state_dict is None:
        state_dict = random_srvgg_state_dict(num_conv, seed)
    sd = {k: (v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)) for k, v in state_dict.items()}
    esrgan_session = SrEngine(sd)
    return esrgan_session


def preprocess_esr(frame):
    """core/merged_pipeline.py:221-225 (host helper; run_esrgan does this inside vd3d_sr_forward)."""
    img = frame[..., ::-1].astype(np.float32) / np.float32(255.0)
    return np.ascontiguousarray(np.transpose(img, (2, 0, 1))[None]).astype(np.float32)


def postprocess_esr(tensor):
    """core/merged_pipeline.py:227-231 (host helper)."""
    t = np.clip(np.transpose(np.squeeze(tensor, axis=0), (1, 2, 0)), 0, 1) * np.float32(255.0)
    return np.ascontiguousarray(t.astype(np.uint8)[..., ::-1])


def _resize_cubic(img, w, h):
    ctx = _lib.default_context(0)
    src = np.ascontiguousarray(img, dtype=np.uint8)
    out = np.empty((int(h), int(w), src.shape[2]), dtype=np.uint8)
    ctx.check(ctx.lib.vd3d_resize_cubic(ctx.h, src.ctypes.data, src.shape[0], src.shape[1], src.shape[2], out.ctypes.data,
                                        int(h), int(w), _lib.MEM_HOST))
    return out


def blend_images(original, upscaled, mode="OFF"):
    """core/merged_pipeline.py:233-238: cv2.addWeighted(upscaled, alpha, original, 1 - alpha, 0) on the GPU."""
    if mode == "OFF":
        return upscaled
    alpha = {"LOW": 0.85, "MEDIUM": 0.5, "HIGH": 0.25}.get(mode.upper(), 1.0)
    ctx = _lib.default_context(0)
    a = np.ascontiguousarray(upscaled, dtype=np.uint8)
    b = np.ascontiguousarray(original, dtype=np.uint8)
    assert a.shape == b.shape
    out = np.empty_like(a)
    ctx.check(ctx.lib.vd3d_add_weighted(ctx.h, a.ctypes.data, float(alpha), b.ctypes.data, float(1 - alpha), a.size,
                                        out.ctypes.data, _lib.MEM_HOST))
    return out


def _esrgan_tiled(img, tile, pad):
    """core/merged_pipeline.py:269-284: tile the frame with `pad` pixels of context and keep the tile centres.  The
    reference writes the 4x tile output into a canvas of the INPUT size (so the tiles are cropped, not placed at 4x);
    reproduced as written."""
    h, w = img.shape[:2]
    out = np.zeros_like(img)
    for y in range(0, h, tile):
        for x in range(0, w, tile):
            y0, x0 = max(0, y - pad), max(0, x - pad)
            y1, x1 = min(h, y + tile + pad), min(w, x + tile + pad)
            up = esrgan_session.upscale(img[y0:y1, x0:x1])
            yc0, xc0 = y - y0, x - x0
            th, tw = min(tile, h - y), min(tile, w - x)
            out[y:y + th, x:x + tw] = up[yc0:yc0 + th, xc0:xc0 + tw]
    return out


def run_esrgan(frame, blend_mode="OFF", input_res_pct=100, model_name="RealESR_Gx4_fp16", target_size=None, tile=None,
               tile_pad=8):
    """core/merged_pipeline.py:240-267.  Returns the input frame when no model is loaded or the engine fails, like the
    reference."""
    if not esrgan_session:
        return frame
    from . import render_3d as R
    original = frame
    if input_res_pct != 100:
        h, w = frame.shape[:2]
        nw, nh = int(w * input_res_pct / 100), int(h * input_res_pct / 100)
        frame = R.resize_area(frame, nw, nh) if input_res_pct < 100 else _resize_cubic(frame, nw, nh)
    try:
        upscaled = _esrgan_tiled(frame, tile, tile_pad) if tile else esrgan_session.upscale(frame)
    except Exception as e:
        print(f"❌ ESRGAN failed: {e}")
        return original
    scale = 2 if "x2" in model_name.lower() else 4
    upscaled = _resize_cubic(upscaled, frame.shape[1] * scale, frame.shape[0] * scale)
    upscaled = _resize_cubic(upscaled, original.shape[1], original.shape[0])
    if target_size:
        upscaled = _resize_cubic(upscaled, target_size[0], target_size[1])
    return blend_images(original, upscaled, mode=blend_mode)
