"""ctypes binding of libvd3d.so (include/vd3d.h).  No CPU fallback: importing this
module without the built library, or creating a context without a CUDA device,
raises."""
import ctypes as C
import sys as _sys
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvd3d.so")

MEM_HOST, MEM_DEVICE = 0, 1
FMT = {"Half-SBS": 0, "Full-SBS": 1, "Red-Cyan Anaglyph": 2, "Passive Interlaced": 3, "VR": 4}
STATE_GLOBAL, STATE_CLIP = 1, 2


class ShiftParams(C.Structure):
    _fields_ = [
        ("fg_shift", C.c_double), ("mg_shift", C.c_double), ("bg_shift", C.c_double),
        ("blur_ksize", C.c_int32),
        ("feather_strength", C.c_double),
        ("max_pixel_shift_percent", C.c_double),
        ("parallax_balance", C.c_double),
        ("zero_parallax_strength", C.c_double),
        ("use_subject_tracking", C.c_int32),
        ("enable_floating_window", C.c_int32),
        ("enable_feathering", C.c_int32),
        ("enable_edge_masking", C.c_int32),
        ("convergence_strength", C.c_double),
        ("enable_dynamic_convergence", C.c_int32),
        ("depth_pop_gamma", C.c_double), ("depth_pop_mid", C.c_double),
        ("depth_stretch_lo", C.c_double), ("depth_stretch_hi", C.c_double),
        ("fg_pop_multiplier", C.c_double), ("bg_push_multiplier", C.c_double),
        ("subject_lock_strength", C.c_double),
    ]


class RenderParams(C.Structure):
    _fields_ = [
        ("output_width", C.c_int32), ("output_height", C.c_int32),
        ("fg_shift", C.c_double), ("mg_shift", C.c_double), ("bg_shift", C.c_double),
        ("sharpness_factor", C.c_double),
        ("output_format", C.c_int32),
        ("aspect_ratio", C.c_double),
        ("dof_strength", C.c_double),
        ("feather_strength", C.c_double),
        ("blur_ksize", C.c_int32),
        ("use_subject_tracking", C.c_int32), ("use_floating_window", C.c_int32),
        ("max_pixel_shift_percent", C.c_double),
        ("preserve_original_aspect", C.c_int32),
        ("zero_parallax_strength", C.c_double),
        ("enable_edge_masking", C.c_int32), ("enable_feathering", C.c_int32),
        ("original_video_width", C.c_int32), ("original_video_height", C.c_int32),
        ("convergence_strength", C.c_double),
        ("enable_dynamic_convergence", C.c_int32),
        ("ipd_factor", C.c_double),
        ("color_saturation", C.c_double), ("color_contrast", C.c_double), ("color_brightness", C.c_double),
        ("auto_crop_black_bars", C.c_int32),
    ]


class SizePlan(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "crop_x0", "crop_y0", "crop_w", "crop_h", "target_eye_w", "target_eye_h",
        "resized_width", "resized_height", "per_eye_w", "per_eye_h", "out_width", "out_height")]


class FrameInfo(C.Structure):
    _fields_ = [
        ("pct_lo", C.c_float), ("pct_hi", C.c_float),
        ("subj_raw", C.c_float), ("stretch_lo", C.c_float), ("stretch_hi", C.c_float),
        ("subj_shaped", C.c_float), ("subj_norm", C.c_float),
        ("dyn_scale", C.c_double), ("fg", C.c_double), ("mg", C.c_double), ("bg", C.c_double),
        ("zero_parallax_offset", C.c_double),
        ("focal_depth", C.c_double), ("motion_metric", C.c_double),
        ("stable_zero", C.c_double),
        ("bar_width", C.c_int32), ("bar_side", C.c_int32),
        ("crop_top", C.c_int32), ("crop_bottom", C.c_int32),
    ]


class UpscaleParams(C.Structure):
    _fields_ = [
        ("input_res_pct", C.c_double),
        ("scale", C.c_int32),
        ("target_w", C.c_int32), ("target_h", C.c_int32),
        ("blend_alpha", C.c_double),
    ]


class Tile(C.Structure):
    """vd3d_tile: one tile of infer_depth_tile's plan (core rect, padded crop, crop size rounded to 14, engine class)."""
    _fields_ = [(n, C.c_int32) for n in ("y0", "y1", "x0", "x1", "yp0", "yp1", "xp0", "xp1", "rh", "rw", "cls")]


# every symbol declared in include/vd3d.h (tests/test_abi.py checks the header against this)
SYMBOLS = [
    "vd3d_create", "vd3d_destroy", "vd3d_last_error", "vd3d_reset_state", "vd3d_host_alloc",
    "vd3d_host_free", "vd3d_stream", "vd3d_sync", "vd3d_launch_count", "vd3d_set_graphs",
    "vd3d_set_exact", "vd3d_get_exact", "vd3d_graphs_active", "vd3d_get_buffer",
    "vd3d_pixel_shift", "vd3d_plan_sizes", "vd3d_render_frame", "vd3d_render_clip",
    "vd3d_sharpen", "vd3d_dof_grade", "vd3d_struct_size", "vd3d_pack", "vd3d_fit_eye", "vd3d_area_table", "vd3d_area_linear_table", "vd3d_heal",
    "vd3d_profile", "vd3d_profile_collect", "vd3d_check_config", "vd3d_color_grade", "vd3d_resize_cubic", "vd3d_add_weighted",
    "vd3d_sr_create", "vd3d_sr_forward", "vd3d_sr_upscale", "vd3d_sr_set_rrdb",
    # depth forward (bound in depth_engine.py)
    "vd3d_depth_create", "vd3d_depth_create_ex", "vd3d_depth_set_fit", "vd3d_depth_set_zoe", "vd3d_depth_destroy", "vd3d_depth_last_error", "vd3d_depth_launch_count",
    "vd3d_depth_set_tensor", "vd3d_depth_forward", "vd3d_depth_get_buffer", "vd3d_gemm_f16", "vd3d_conv_f16",
    "vd3d_bit_kernel", "vd3d_zoe_kernel",
    "vd3d_depth_infer_batch", "vd3d_depth_infer_batch_device",
    "vd3d_set_depth_batch", "vd3d_get_depth_batch", "vd3d_render_clip_depth", "vd3d_depth_add_launches", "vd3d_depth_clone", "vd3d_release_depth",
    "vd3d_depth_profile", "vd3d_depth_profile_collect", "vd3d_depth_profile_spans",
    "vd3d_advance_state", "vd3d_state_bytes", "vd3d_export_state", "vd3d_import_state",
    "vd3d_last_crops", "vd3d_detect_black_bars",
    "vd3d_letterbox_stats", "vd3d_canny_u8", "vd3d_letterbox_repad",
    "vd3d_tile_crops", "vd3d_tile_blend", "vd3d_normalize_u8", "vd3d_depth_tiled",
    "vd3d_depth_resize_pil", "vd3d_pil_bicubic_table", "vd3d_depth_infer_images",
]

_lib = None


def load():
    """Load libvd3d.so (raises OSError with a build hint when it is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise OSError(
            f"{LIB_PATH} not found: build it with `python -m visiondepth3d_b200.build` "
            "(or __graft_entry__.build()). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i, u8p, fp = C.c_void_p, C.c_int, C.c_void_p, C.c_void_p
    lib.vd3d_struct_size.argtypes = [i]
    lib.vd3d_struct_size.restype = i
    for which, st in enumerate((ShiftParams, RenderParams, SizePlan, FrameInfo, UpscaleParams, Tile)):
        if lib.vd3d_struct_size(which) != C.sizeof(st):
            raise OSError(f"libvd3d ABI mismatch for {st.__name__}: "
                          f"{lib.vd3d_struct_size(which)} != {C.sizeof(st)}")
    lib.vd3d_create.argtypes = [i, C.POINTER(vp)]
    lib.vd3d_create.restype = i
    lib.vd3d_destroy.argtypes = [vp]
    lib.vd3d_destroy.restype = None
    lib.vd3d_last_error.argtypes = [vp]
    lib.vd3d_last_error.restype = C.c_char_p
    lib.vd3d_reset_state.argtypes = [vp, C.c_uint32]
    lib.vd3d_reset_state.restype = i
    lib.vd3d_host_alloc.argtypes = [C.c_size_t]
    lib.vd3d_host_alloc.restype = vp
    lib.vd3d_host_free.argtypes = [vp]
    lib.vd3d_host_free.restype = None
    lib.vd3d_stream.argtypes = [vp]
    lib.vd3d_stream.restype = vp
    lib.vd3d_sync.argtypes = [vp]
    lib.vd3d_sync.restype = i
    lib.vd3d_launch_count.argtypes = [vp]
    lib.vd3d_launch_count.restype = C.c_uint64
    lib.vd3d_profile.argtypes = [vp, i]
    lib.vd3d_profile.restype = i
    lib.vd3d_profile_collect.argtypes = [vp, i, C.POINTER(C.c_double), C.POINTER(C.c_int)]
    lib.vd3d_profile_collect.restype = i
    lib.vd3d_set_graphs.argtypes = [vp, i]
    lib.vd3d_set_graphs.restype = i
    lib.vd3d_set_exact.argtypes = [vp, i]
    lib.vd3d_set_exact.restype = i
    lib.vd3d_set_depth_batch.argtypes = [vp, i]
    lib.vd3d_set_depth_batch.restype = i
    lib.vd3d_get_depth_batch.argtypes = [vp]
    lib.vd3d_get_depth_batch.restype = i
    lib.vd3d_get_exact.argtypes = [vp]
    lib.vd3d_get_exact.restype = i
    lib.vd3d_graphs_active.argtypes = [vp]
    lib.vd3d_graphs_active.restype = i
    lib.vd3d_get_buffer.argtypes = [vp, C.c_char_p, vp, C.c_size_t]
    lib.vd3d_get_buffer.restype = i
    lib.vd3d_pixel_shift.argtypes = [vp, fp, fp, i, i, i, i, C.POINTER(ShiftParams), u8p, u8p, fp, i,
                                     C.POINTER(FrameInfo)]
    lib.vd3d_pixel_shift.restype = i
    lib.vd3d_plan_sizes.argtypes = [i, i, C.POINTER(RenderParams), C.POINTER(SizePlan)]
    lib.vd3d_plan_sizes.restype = i
    lib.vd3d_render_frame.argtypes = [vp, u8p, u8p, i, i, i, C.POINTER(RenderParams), u8p, i,
                                      C.POINTER(FrameInfo)]
    lib.vd3d_render_frame.restype = i
    lib.vd3d_render_clip.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), i, i, i, C.POINTER(RenderParams),
                                     C.POINTER(vp), i, C.POINTER(FrameInfo)]
    lib.vd3d_render_clip.restype = i
    lib.vd3d_render_clip_depth.argtypes = [vp, vp, i, C.POINTER(vp), i, i, C.POINTER(RenderParams), C.POINTER(vp), i]
    lib.vd3d_render_clip_depth.restype = i
    lib.vd3d_last_crops.argtypes = [vp, C.POINTER(C.c_int32), i]
    lib.vd3d_last_crops.restype = i
    lib.vd3d_detect_black_bars.argtypes = [vp, u8p, i, i, i, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.vd3d_detect_black_bars.restype = i
    lib.vd3d_letterbox_stats.argtypes = [vp, i, u8p, i, i, u8p, i, fp, fp, fp, vp, fp, vp, vp, u8p]
    lib.vd3d_letterbox_stats.restype = i
    lib.vd3d_canny_u8.argtypes = [vp, u8p, i, i, C.c_double, C.c_double, u8p, i]
    lib.vd3d_canny_u8.restype = i
    lib.vd3d_letterbox_repad.argtypes = [vp, u8p, i, i, i, i, u8p, i]
    lib.vd3d_letterbox_repad.restype = i
    tp = C.POINTER(Tile)
    lib.vd3d_tile_crops.argtypes = [vp, u8p, i, i, i, i, tp, i, u8p, i]
    lib.vd3d_tile_crops.restype = i
    lib.vd3d_tile_blend.argtypes = [vp, i, i, i, i, tp, i, C.POINTER(vp), C.POINTER(vp), fp, fp, i]
    lib.vd3d_tile_blend.restype = i
    lib.vd3d_normalize_u8.argtypes = [vp, fp, i, i, C.c_double, C.c_double, i, u8p, i, i, fp, i]
    lib.vd3d_normalize_u8.restype = i
    lib.vd3d_depth_tiled.argtypes = [vp, C.POINTER(vp), i, i, C.POINTER(vp), i, i, i, i, tp, i, C.POINTER(vp), i, i, i,
                                     C.POINTER(vp), C.POINTER(vp), fp, i]
    lib.vd3d_depth_tiled.restype = i
    lib.vd3d_heal.argtypes = [vp, fp, fp, fp, i, i, C.c_double, fp, i]
    lib.vd3d_heal.restype = i
    lib.vd3d_pack.argtypes = [vp, u8p, u8p, i, i, i, u8p, i]
    lib.vd3d_pack.restype = i
    lib.vd3d_fit_eye.argtypes = [vp, u8p, i, i, i, i, i, u8p, i]
    lib.vd3d_fit_eye.restype = i
    lib.vd3d_area_table.argtypes = [i, i, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_float), i]
    lib.vd3d_area_table.restype = i
    lib.vd3d_area_linear_table.argtypes = [i, i, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.vd3d_area_linear_table.restype = i
    lib.vd3d_advance_state.argtypes = [vp, u8p, u8p, i, i, i, C.POINTER(RenderParams), i]
    lib.vd3d_advance_state.restype = i
    lib.vd3d_state_bytes.argtypes = [vp]
    lib.vd3d_state_bytes.restype = C.c_size_t
    lib.vd3d_export_state.argtypes = [vp, vp, C.c_size_t, i]
    lib.vd3d_export_state.restype = i
    lib.vd3d_import_state.argtypes = [vp, vp, C.c_size_t, i]
    lib.vd3d_import_state.restype = i
    lib.vd3d_release_depth.argtypes = [vp, vp]
    lib.vd3d_release_depth.restype = i
    lib.vd3d_check_config.argtypes = [vp, i, i, C.POINTER(RenderParams)]
    lib.vd3d_check_config.restype = i
    lib.vd3d_resize_cubic.argtypes = [vp, u8p, i, i, i, u8p, i, i, i]
    lib.vd3d_resize_cubic.restype = i
    lib.vd3d_add_weighted.argtypes = [vp, u8p, C.c_double, u8p, C.c_double, C.c_size_t, u8p, i]
    lib.vd3d_add_weighted.restype = i
    lib.vd3d_sr_create.argtypes = [vp, C.POINTER(vp)]
    lib.vd3d_sr_create.restype = i
    lib.vd3d_sr_forward.argtypes = [vp, u8p, i, i, i, u8p, i]
    lib.vd3d_sr_forward.restype = i
    lib.vd3d_sr_upscale.argtypes = [vp, vp, i, C.POINTER(vp), i, i, i, C.POINTER(UpscaleParams), C.POINTER(vp), i]
    lib.vd3d_sr_upscale.restype = i
    lib.vd3d_sr_set_rrdb.argtypes = [vp, i, i]
    lib.vd3d_sr_set_rrdb.restype = i
    lib.vd3d_color_grade.argtypes = [vp, fp, i, i, C.c_double, C.c_double, C.c_double, fp, i]
    lib.vd3d_color_grade.restype = i
    lib.vd3d_sharpen.argtypes = [vp, u8p, i, i, C.c_double, u8p, i]
    lib.vd3d_sharpen.restype = i
    lib.vd3d_dof_grade.argtypes = [vp, u8p, i, i, fp, i, i, C.c_double, C.c_double, C.c_double, C.c_double,
                                   C.c_double, u8p, i]
    lib.vd3d_dof_grade.restype = i
    _lib = lib
    return lib


class Vd3dError(RuntimeError):
    pass


class Context:
    """Owns one vd3d_ctx (one per GPU / per process)."""

    def __init__(self, device=0):
        self.lib = load()
        h = C.c_void_p()
        rc = self.lib.vd3d_create(int(device), C.byref(h))
        if rc != 0:
            raise Vd3dError(f"vd3d_create failed ({rc}): {self.lib.vd3d_last_error(None).decode()}")
        self.h = h
        self.device = int(device)

    def check(self, rc):
        if rc != 0:
            raise Vd3dError(f"libvd3d error {rc}: {self.lib.vd3d_last_error(self.h).decode()}")

    def reset(self, which=STATE_GLOBAL | STATE_CLIP):
        self.check(self.lib.vd3d_reset_state(self.h, which))

    def set_exact(self, enable=True):
        """DIBR arithmetic mode (include/vd3d.h: vd3d_set_exact): True = bit-for-bit with the oracle."""
        self.check(self.lib.vd3d_set_exact(self.h, int(bool(enable))))

    def export_state(self):
        """Temporal state after the last frame as a uint8 numpy blob (SURVEY 8(e) exact sharding)."""
        import numpy as np
        n = int(self.lib.vd3d_state_bytes(self.h))
        buf = np.empty(n, dtype=np.uint8)
        self.check(self.lib.vd3d_export_state(self.h, buf.ctypes.data, n, MEM_HOST))
        return buf

    def import_state(self, blob):
        import numpy as np
        b = np.ascontiguousarray(blob, dtype=np.uint8)
        self.check(self.lib.vd3d_import_state(self.h, b.ctypes.data, b.nbytes, MEM_HOST))

    def close(self):
        if getattr(self, "h", None):
            self.lib.vd3d_destroy(self.h)
            self.h = None

    def __del__(self):
        try:  # the CUDA runtime may already be torn down at interpreter exit: leave it to the OS then
            if _sys is None or _sys.is_finalizing():
                return
            self.close()
        except BaseException:
            pass

    @property
    def launches(self):
        return int(self.lib.vd3d_launch_count(self.h))


_default_ctx = {}


def default_context(device=0):
    """Process-wide context: the counterpart of the reference's module singletons."""
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]
