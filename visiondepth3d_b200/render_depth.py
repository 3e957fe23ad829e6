"""Drop-in for the hot-path surface of the reference's core/render_depth.py: the `pipe`
callable protocol and the depth -> uint8 normalisation, backed by the libvd3d depth engine
(Depth-Anything-V2 on wgmma tensor cores), and the letterbox tracker of the depth-video pass with its pixel work on
the GPU (letterbox.cu), and the still-image drivers of the Depth tab (depth_images, vd3d_depth_infer_images).  GUI,
ONNX, Marigold and DepthCrafter are outside the GPU hot path (SURVEY.md section 2).

Protocol kept (core/render_depth.py:1113-1119, consumers 201-268 and 1894-1917):
    pipe(images: list[PIL.Image], inference_size: (W, H) | None) -> list[{"predicted_depth": Tensor[h, w]}]
with `predicted_depth` already resized (bicubic) to the PIL image size, as
transformers' DepthEstimationPipeline.postprocess does.
"""
import os
import re
import threading
import time
from ctypes import c_void_p as C_void_p

import numpy as np

from .depth_engine import FAMILY_DA_V2, FAMILY_DPT, DepthEngine, processed_size as _processed_size
from .depth_weights import (CONFIGS, DPT_CONFIGS, DPT_PROCESSOR, da_arch, da_config_from_json, da_processor_from_json,
                            da_spec, dpt_config_from_json, dpt_processed_size, dpt_processor_from_json, hf_config,
                            hf_dpt_config, is_plain_v2)
from .render_3d import _dialog, _val

try:
    import torch
    torch.set_grad_enabled(False)  # the reference does this at import (core/render_depth.py:42)
except Exception:  # pragma: no cover
    torch = None

# module globals the reference's callers read (core/render_depth.py:34-36, 992)
pipe = None
pipe_type = None
_engine = None

# the checkpoints of the hot path (core/render_depth.py:689-712): the Depth-Anything family (V2, V1, Distill-Any-Depth,
# the V2 metric models) and DPT-Large.  label -> (checkpoint id, backbone size)
supported_models = {
    "Distil-Any-Depth-Large": ("xingyang1/Distill-Any-Depth-Large-hf", "vitl"),
    "Distil-Any-Depth-Small": ("xingyang1/Distill-Any-Depth-Small-hf", "vits"),
    "keetrap-Distil-Any-Depth-Large": ("keetrap/Distil-Any-Depth-Large-hf", "vitl"),
    "keetrap-Distil-Any-Depth-Small": ("keetrap/Distill-Any-Depth-Small-hf", "vits"),
    "Depth Anything V2 Large": ("depth-anything/Depth-Anything-V2-Large-hf", "vitl"),
    "Depth Anything V2 Base": ("depth-anything/Depth-Anything-V2-Base-hf", "vitb"),
    "Depth Anything V2 Small": ("depth-anything/Depth-Anything-V2-Small-hf", "vits"),
    "Depth Anything V1 Large": ("LiheYoung/depth-anything-large-hf", "vitl"),
    "Depth Anything V1 Base": ("LiheYoung/depth-anything-base-hf", "vitb"),
    "Depth Anything V1 Small": ("LiheYoung/depth-anything-small-hf", "vits"),
    "V2-Metric-Indoor-Large": ("depth-anything/Depth-Anything-V2-Metric-Indoor-Large-hf", "vitl"),
    "V2-Metric-Outdoor-Large": ("depth-anything/Depth-Anything-V2-Metric-Outdoor-Large-hf", "vitl"),
    "DPT-Large": ("Intel/dpt-large", "dpt-large"),
    "Manojb - DPT-Large": ("Manojb/dpt-large", "dpt-large"),
}
# the Depth-Anything checkpoints other than V2's: their taps and head are only in config.json (the tensors have V2's
# shapes), so they load only with it, and with Depth-Anything's preprocessor_config.json when one is present
DA_CONFIG_REQUIRED = frozenset(v[0] for k, v in supported_models.items()
                               if v[1] != "dpt-large" and not k.startswith("Depth Anything V2"))


def _family_of(arch):
    return FAMILY_DPT if arch in DPT_CONFIGS else FAMILY_DA_V2


def _load_dpt_checkpoint(sd, cfg_path):
    """arch of a DPT state dict (dpt.* keys): DPT-Large when its shapes (and config.json, when present) say so."""
    import json
    c = DPT_CONFIGS["dpt-large"]
    if os.path.exists(cfg_path):
        with open(cfg_path) as f:
            got = dpt_config_from_json(json.load(f))
        if got != c:
            raise ValueError(f"config.json {got} does not match the built-in dpt-large configuration {c}")
    hidden = sd["dpt.embeddings.cls_token"].shape[-1]
    layers = len({k.split(".")[3] for k in sd if k.startswith("dpt.encoder.layer.")})
    return "dpt-large" if (hidden, layers) == (c["hidden"], c["layers"]) else None


def _check_da_state_dict(sd, spec):
    """ValueError when a Depth-Anything state dict does not have the shapes of `spec` (config.json)."""
    got = dict(hidden=sd["backbone.embeddings.cls_token"].shape[-1],
               layers=len({k.split(".")[3] for k in sd if k.startswith("backbone.encoder.layer.")}),
               neck=[sd[f"neck.reassemble_stage.layers.{i}.projection.weight"].shape[0] for i in range(4)],
               fusion=sd["neck.convs.0.weight"].shape[0])
    want = {k: spec[k] for k in got}
    if got != want:
        raise ValueError(f"state dict {got} does not match its config.json {want}")


def load_checkpoint(path):
    """HF-format checkpoint (model.safetensors / pytorch_model.bin of a DepthAnythingForDepthEstimation or
    Intel/dpt-large model) -> (arch, state_dict), arch None for another model.  Depth-Anything: with a config.json next
    to it, the model is what da_config_from_json reads there (ValueError for what the engine does not serve): arch is
    the size key of depth_weights.CONFIGS for a plain V2 model, else the spec dict (V1 taps, a metric head); without
    one, the V2 size of the hidden width.  DPT: cross-checked against DPT_CONFIGS."""
    import json
    import os
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path)
    else:
        sd = torch.load(path, map_location="cpu")
    if "dpt.embeddings.cls_token" in sd:
        return _load_dpt_checkpoint(sd, os.path.join(os.path.dirname(path), "config.json")), sd
    if "backbone.embeddings.cls_token" not in sd:
        return None, sd
    cfg_path = os.path.join(os.path.dirname(path), "config.json")
    if os.path.exists(cfg_path):
        with open(cfg_path) as f:
            spec = da_config_from_json(json.load(f))
        _check_da_state_dict(sd, spec)
        return (da_arch(spec) if is_plain_v2(spec) else spec), sd
    arch = None
    hidden = sd["backbone.embeddings.cls_token"].shape[-1]
    for name, c in CONFIGS.items():
        if c["hidden"] == hidden:
            arch = name
    return arch, sd


_state_dict = None      # weights of the loaded model (HF naming): engines for other processed sizes are built from it
_arch = None            # "vits" / "vitb" / "vitl" (the Depth-Anything backbone size) or "dpt-large"
_spec = None            # Depth-Anything: the spec (taps, head, max_depth; depth_weights.da_spec) every engine is built with
_processor = None       # DPT: the image processor's settings (depth_weights.DPT_PROCESSOR or preprocessor_config.json)
_engines = {}           # (processed_h, processed_w) -> DepthEngine, all sharing _state_dict
cancel_requested = threading.Event()   # core/render_depth.py:38 (the GUI's cancel flag for depth jobs)


def _weights_dir():
    """<project root>/weights, where the reference keeps its checkpoints (core/render_depth.py:615-626)."""
    return os.path.join(os.path.abspath(os.path.join(os.path.dirname(__file__), "..")), "weights")


local_model_dir = _weights_dir()


def model_processed_size(width, height):
    """(h, w) the loaded model's image processor resizes a (width, height) image to: Depth-Anything-V2 keeps the
    aspect at multiples of 14 near 518, DPT-Large resizes every image to its processor's fixed size."""
    if _family_of(_arch) == FAMILY_DPT:
        return dpt_processed_size(_processor)
    return _processed_size(width, height)


def _check_tiled_supported():
    if USE_TILED_DEPTH and _family_of(_arch) == FAMILY_DPT:
        raise ValueError("USE_TILED_DEPTH is served for Depth-Anything-V2 models only, not for DPT-Large")


def _engine_for(width, height):
    """The engine whose processed size fits a (width, height) image; built on first use from the loaded weights
    (the DA processor picks a keep-aspect multiple-of-14 size per image, so one model serves every aspect)."""
    global _engine
    if _state_dict is None:
        raise RuntimeError("no depth model loaded: call load_depth_model() / update_pipeline() first")
    key = model_processed_size(width, height)
    eng = _engines.get(key)
    if eng is None:
        dpt = _family_of(_arch) == FAMILY_DPT
        eng = DepthEngine(_arch if dpt else _spec, key[0], key[1], family=_family_of(_arch), processor=_processor)
        eng.load_state_dict(_state_dict)
        _engines[key] = eng
    _engine = eng
    return eng


def load_depth_model(arch="vits", state_dict=None, width=1920, height=1080, seed=0, processor=None):
    """Make `pipe` serve a Depth-Anything model or DPT-Large ("dpt-large").  arch: a Depth-Anything-V2 size ("vits" /
    "vitb" / "vitl") or a Depth-Anything spec dict (depth_weights.da_spec / da_config_from_json: V1's taps, a metric
    head with its max_depth), which every engine built from these weights then carries.
    `state_dict` uses HF DepthAnythingForDepthEstimation / DPTForDepthEstimation naming (e.g. from a local
    safetensors checkpoint); without one a random-init model (torch.manual_seed(seed)) is used -- there is no network
    here and the reference ships no weights.  processor (DPT only): the image processor's settings
    (dpt_processor_from_json of the checkpoint's preprocessor_config.json; default DPTImageProcessor's).  (width,
    height) only pre-builds the engine for that frame shape; other shapes get their own engine on first use."""
    global pipe, pipe_type, _state_dict, _arch, _spec, _processor
    spec = None
    if isinstance(arch, dict):
        spec = da_spec(arch)
        arch = da_arch(spec)
        if arch is None:
            raise ValueError(f"unknown depth model {spec!r}")
    dpt = _family_of(arch) == FAMILY_DPT
    if not dpt and arch not in CONFIGS:
        raise ValueError(f"unknown depth model {arch!r}")
    if not dpt and spec is None:
        spec = da_spec(arch)
    if dpt:
        processor = dict(processor or DPT_PROCESSOR)
        dpt_processed_size(processor)  # refuse an unserved processor before anything is built
    if state_dict is None:
        torch.manual_seed(seed)
        if dpt:
            from transformers import DPTForDepthEstimation
            state_dict = DPTForDepthEstimation(hf_dpt_config(arch)).eval().state_dict()
        else:
            from transformers import DepthAnythingForDepthEstimation
            state_dict = DepthAnythingForDepthEstimation(hf_config(spec)).eval().state_dict()
    for e in _engines.values():
        e.close()
    _engines.clear()
    _state_dict, _arch, _spec, _processor = state_dict, arch, spec, (processor if dpt else None)
    eng = _engine_for(width, height)
    pipe = hf_batch_safe_pipe
    pipe_type = "hf"
    return pipe, {"arch": arch, "processed_size": (eng.image_h, eng.image_w),
                  "config": DPT_CONFIGS[arch] if dpt else dict(spec)}


def hf_batch_safe_pipe(images, inference_size=None):
    """The `pipe` protocol of core/render_depth.py:1113-1119: list of PIL images (optionally resized to
    inference_size with PIL bicubic first) -> list of {"predicted_depth": tensor [h, w]} at each image's own size.
    Images of one shape go through the engine as one batch."""
    if not isinstance(images, (list, tuple)):
        images = [images]
    frames = []
    for img in images:
        if inference_size is not None:
            from PIL import Image
            img = img.resize(tuple(inference_size), Image.BICUBIC)
        rgb = np.asarray(img.convert("RGB"), dtype=np.uint8)
        frames.append(np.ascontiguousarray(rgb[..., ::-1]))
    out = [None] * len(frames)
    by_shape = {}
    for k, f in enumerate(frames):
        by_shape.setdefault(f.shape[:2], []).append(k)
    for (h, w), idxs in by_shape.items():
        eng = _engine_for(w, h)
        for k, (d32, _) in zip(idxs, eng.infer_batch([frames[k] for k in idxs])):
            out[k] = {"predicted_depth": torch.from_numpy(d32) if torch is not None else d32}
    return out


def depth_u8_from_frame(frame_bgr, invert=False):
    """frame -> pipe -> convert_depth_to_grayscale in one GPU pass (u8 [h, w])."""
    h, w = frame_bgr.shape[:2]
    return _engine_for(w, h).infer(frame_bgr, invert=invert)[1]


def _depth_plane(depth):
    """Whatever a depth backend returns -> one float32 plane.  Accepted: PIL image, torch tensor, ndarray; ranks 2 or
    3; a leading or trailing axis of 1 or 3 channels is reduced (single channel taken, three averaged)."""
    if torch is not None and isinstance(depth, torch.Tensor):
        plane = depth.detach().cpu().float().numpy()
    elif isinstance(depth, np.ndarray):
        plane = depth.astype(np.float32)
    else:
        try:
            from PIL import Image
        except Exception:  # pragma: no cover
            Image = None
        if Image is None or not isinstance(depth, Image.Image):
            raise TypeError(f"depth must be a PIL image, a torch tensor or an ndarray, got {type(depth).__name__}")
        plane = np.array(depth).astype(np.float32)
    if plane.ndim == 2:
        return plane
    if plane.ndim != 3:
        raise ValueError(f"depth must have 2 or 3 dimensions, got shape {plane.shape}")
    for axis in (0, 2):
        c = plane.shape[axis]
        if c == 1:
            return np.take(plane, 0, axis=axis)
        if c == 3:
            return plane.mean(axis=axis)
    return plane  # an unexpected channel count is passed through, as the reference does (core/render_depth.py:597-601)


def convert_depth_to_grayscale(depth):
    """core/render_depth.py:585-611: per-frame min-max normalisation to uint8 with truncation.  A frame with NaNs or
    with less than 1e-6 of range comes back all zero.  Host helper for callers that hold CPU data, like the
    reference's; the frame path does the same on the GPU (k_depth_upsample_minmax + k_depth_to_u8)."""
    plane = _depth_plane(depth)
    lo, hi = np.min(plane), np.max(plane)
    usable = not (np.isnan(lo) or np.isnan(hi)) and (hi - lo) >= 1e-6
    if not usable:
        print("⚠️ depth frame has no usable range (NaN or flat): writing zeros")
        return np.zeros_like(plane, dtype=np.uint8)
    return ((plane - lo) / (hi - lo + 1e-6) * 255).astype(np.uint8)


def resize_cubic_u8(plane, width, height):
    """cv2.resize(u8 plane, (width, height), interpolation=cv2.INTER_CUBIC) on the GPU (vd3d_resize_cubic, one
    channel): the resize the reference's depth writer applies to the u8 depth (core/render_depth.py:1917, 193)."""
    from . import _lib
    ctx = _lib.default_context(0)
    src = np.ascontiguousarray(plane, dtype=np.uint8)
    assert src.ndim == 2
    out = np.empty((int(height), int(width)), dtype=np.uint8)
    ctx.check(ctx.lib.vd3d_resize_cubic(ctx.h, src.ctypes.data, src.shape[0], src.shape[1], 1, out.ctypes.data,
                                        int(height), int(width), _lib.MEM_HOST))
    return out


def _normalize_to_u8(depth_f, out_size, invert=False, pclip=(1.0, 99.0)):
    """core/render_depth.py:173-194 (the ndarray / tiled-depth front end) on the GPU (vd3d_normalize_u8): non-finite
    values -> 0, clip to the [p1, p99] percentiles (np.percentile, linear, float32), fall back to min-max when they
    coincide and to flat 128 when the frame is flat, truncate to u8, optional inversion, INTER_CUBIC resize to
    out_size = (W, H)."""
    from . import _lib
    ctx = _lib.default_context(0)
    d = np.ascontiguousarray(depth_f, dtype=np.float32)
    if d.ndim != 2:
        raise ValueError(f"depth must be a 2D plane, got shape {d.shape}")
    ow, oh = int(out_size[0]), int(out_size[1])
    out = np.empty((oh, ow), dtype=np.uint8)
    ctx.check(ctx.lib.vd3d_normalize_u8(ctx.h, d.ctypes.data, d.shape[0], d.shape[1], float(pclip[0]), float(pclip[1]),
                                        int(bool(invert)), out.ctypes.data, oh, ow, None, _lib.MEM_HOST))
    return out


# ---------------------------------------------------------------------------
# tiled depth inference (core/render_depth.py:46-51, 62-268): the tile crops, the batched per-tile forwards, the Hann
# blend and the percentile normalisation run on the GPU in one call (vd3d_depth_tiled)
# ---------------------------------------------------------------------------
USE_TILED_DEPTH = False   # read at call time by _run_pipe_or_tile and the depth-video pass
TILE_SIZE = 512
TILE_PAD = 32
TILE_DEBUG = False        # print one line per tile

assert TILE_SIZE > 2 * TILE_PAD, "TILE_SIZE must be larger than 2*TILE_PAD"


def _hann2d(h, w):
    """core/render_depth.py:62-66: outer product of two np.hanning windows, divided by (max + 1e-8), float32."""
    wy = np.hanning(max(2, h))
    wx = np.hanning(max(2, w))
    m = np.outer(wy, wx).astype(np.float32)
    mmax = float(m.max()) if m.size else 1.0
    return m / (mmax + 1e-8)


def _ensure_depth_np(pred):
    """core/render_depth.py:68-100: a prediction (tensor / ndarray, optionally in a dict or list) -> float32 [H, W]."""
    if isinstance(pred, list):
        pred = pred[0]
    if isinstance(pred, dict) and "predicted_depth" in pred:
        pred = pred["predicted_depth"]
    if torch is not None and isinstance(pred, torch.Tensor):
        arr = pred.detach().cpu().float().numpy()
    elif isinstance(pred, np.ndarray):
        arr = pred.astype(np.float32, copy=False)
    else:
        raise TypeError(f"Unexpected depth type: {type(pred)}")
    if arr.ndim == 3:
        if arr.shape[0] in (1, 3):
            arr = arr[0] if arr.shape[0] == 1 else arr.mean(axis=0)
        elif arr.shape[2] in (1, 3):
            arr = arr[..., 0] if arr.shape[2] == 1 else arr.mean(axis=-1)
        else:
            arr = np.squeeze(arr)
    elif arr.ndim > 2:
        arr = np.squeeze(arr)
    if arr.ndim != 2:
        raise ValueError(f"Depth must be 2D after squeeze; got shape {arr.shape}")
    return arr.astype(np.float32, copy=False)


def tile_plan(width, height, tile=TILE_SIZE, pad=TILE_PAD):
    """infer_depth_tile's loop over a (width, height) image: [(y0, y1, x0, x1, yp0, yp1, xp0, xp1, rh, rw)] in
    row-major order -- core rect, padded crop, and the crop size rounded up to multiples of 14."""
    core = max(1, int(tile) - 2 * int(pad))
    r14 = lambda v: ((int(v) + 13) // 14) * 14  # noqa: E731
    out = []
    for y0 in range(0, height, core):
        for x0 in range(0, width, core):
            y1, x1 = min(y0 + tile, height), min(x0 + tile, width)
            yp0, xp0 = max(0, y0 - pad), max(0, x0 - pad)
            yp1, xp1 = min(height, y1 + pad), min(width, x1 + pad)
            out.append((y0, y1, x0, x1, yp0, yp1, xp0, xp1, r14(yp1 - yp0), r14(xp1 - xp0)))
    return out


def tile_weights(ch, cw, tile=TILE_SIZE, pad=TILE_PAD):
    """The Hann weights of a tile whose core rect is ch x cw, as infer_depth_tile builds them (cv2 INTER_CUBIC from
    the core x core window when the shapes differ)."""
    import cv2
    core = max(1, int(tile) - 2 * int(pad))
    w = _hann2d(core, core)
    if w.shape != (ch, cw):
        w = cv2.resize(w, (cw, ch), interpolation=cv2.INTER_CUBIC)
    return np.ascontiguousarray(w, dtype=np.float32)


class _TilePlan:
    """Set-up of one (width, height, tile, pad): the tiles (vd3d_tile array), one class per rounded crop size (in order
    of first use), and the Hann weights uploaded once, one map per core-rect shape."""

    def __init__(self, width, height, tile, pad):
        from . import _lib
        self.width, self.height, self.tile, self.pad = width, height, tile, pad
        self.rects = tile_plan(width, height, tile, pad)
        self.classes = []
        for r in self.rects:
            if (r[8], r[9]) not in self.classes:
                self.classes.append((r[8], r[9]))
        self.tiles = (_lib.Tile * len(self.rects))()
        maps = {}
        self._weights = []  # keeps the CUDA tensors alive
        for k, r in enumerate(self.rects):
            self.tiles[k] = _lib.Tile(*r, self.classes.index((r[8], r[9])))
            shape = (r[1] - r[0], r[3] - r[2])
            if shape not in maps:
                maps[shape] = torch.from_numpy(tile_weights(*shape, tile, pad)).cuda()
                self._weights.append(maps[shape])
        self.weight_ptrs = (C_void_p * len(self.rects))(*[maps[(r[1] - r[0], r[3] - r[2])].data_ptr()
                                                           for r in self.rects])
        torch.cuda.current_stream().synchronize()

    def engines(self):
        """The engine of each class (through _engine_for, so they follow the loaded model)."""
        return [_engine_for(rw, rh) for rh, rw in self.classes]

    def debug_lines(self):
        return [f"[tile] ({y0}:{y1},{x0}:{x1}) crop={(rh, rw)} center={(y1 - y0, x1 - x0)} acc={(y1 - y0, x1 - x0)}"
                for y0, y1, x0, x1, _a, _b, _c, _d, rh, rw in self.rects]


_tile_plans = {}  # (width, height, tile, pad) -> _TilePlan


def _plan_for(width, height, tile, pad):
    key = (int(width), int(height), int(tile), int(pad))
    plan = _tile_plans.get(key)
    if plan is None:
        plan = _tile_plans[key] = _TilePlan(*key)
    return plan


def depth_tiled(frames, width, height, out_size, invert=False, tile=None, pad=None, want_f32=False):
    """vd3d_depth_tiled on n same-shape u8 BGR frames [height, width, 3]: the tiled depth of each frame, normalised
    by _normalize_to_u8 to out_size = (W, H).  frames: a list of host frames or a CUDA uint8 tensor [n, h, w, 3] (the
    results are then CUDA tensors).  Returns (u8 planes, float32 depth planes or None, [(min, max)] per frame)."""
    from . import _lib
    _check_tiled_supported()
    tile = TILE_SIZE if tile is None else int(tile)
    pad = TILE_PAD if pad is None else int(pad)
    ctx = _lib.default_context(0)
    plan = _plan_for(width, height, tile, pad)
    engines = plan.engines()
    ow, oh = int(out_size[0]), int(out_size[1])
    device = _is_cuda_tensor(frames)
    if device:
        fr = frames.contiguous()
        n = int(fr.shape[0])
        u8 = torch.empty((n, oh, ow), dtype=torch.uint8, device=fr.device)
        f32 = torch.empty((n, height, width), dtype=torch.float32, device=fr.device) if want_f32 else None
        fptr = [fr[k].data_ptr() for k in range(n)]
        uptr = [u8[k].data_ptr() for k in range(n)]
        dptr = [f32[k].data_ptr() for k in range(n)] if want_f32 else None
        mem = _lib.MEM_DEVICE
        torch.cuda.current_stream().synchronize()  # the frames may come from work queued on torch's stream
    else:
        fr = [np.ascontiguousarray(f, dtype=np.uint8) for f in frames]
        n = len(fr)
        u8 = [np.empty((oh, ow), np.uint8) for _ in range(n)]
        f32 = [np.empty((height, width), np.float32) for _ in range(n)] if want_f32 else None
        fptr = [f.ctypes.data for f in fr]
        uptr = [u.ctypes.data for u in u8]
        dptr = [d.ctypes.data for d in f32] if want_f32 else None
        mem = _lib.MEM_HOST
    mm = np.empty((n, 2), np.float32)
    vp = C_void_p
    ctx.check(ctx.lib.vd3d_depth_tiled(
        ctx.h, (vp * len(engines))(*[e.h for e in engines]), len(engines), n, (vp * n)(*fptr), height, width, tile,
        pad, plan.tiles, len(plan.rects), plan.weight_ptrs, int(bool(invert)), oh, ow, (vp * n)(*uptr),
        (vp * n)(*dptr) if want_f32 else None, mm.ctypes.data, mem))
    return u8, f32, [(float(a), float(b)) for a, b in mm]


def _print_tile_log(width, height, ranges):
    """What _run_pipe_or_tile prints per image, image after image: the TILE_DEBUG lines of the plan, then the range."""
    for lo, hi in ranges:
        if TILE_DEBUG:
            for line in _plan_for(width, height, TILE_SIZE, TILE_PAD).debug_lines():
                print(line)
        print(f"[tile] range min={lo:.6f} max={hi:.6f}")


def _outer_resize(rgb, tgt_w, tgt_h):
    """infer_depth_tile's first step on the GPU: cv2 INTER_AREA when the image shrinks (vd3d_fit_eye), INTER_CUBIC when
    it grows (vd3d_resize_cubic), a copy at the same size; returns BGR.  One axis shrinking while the other grows is
    refused: cv2 takes neither path there."""
    from . import _lib
    h, w = rgb.shape[:2]
    bgr = np.ascontiguousarray(rgb[:, :, ::-1])
    if (tgt_w, tgt_h) == (w, h):
        return bgr
    ctx = _lib.default_context(0)
    out = np.empty((tgt_h, tgt_w, 3), np.uint8)
    if tgt_w <= w and tgt_h <= h:
        ctx.check(ctx.lib.vd3d_fit_eye(ctx.h, bgr.ctypes.data, h, w, tgt_w, tgt_h, 0, out.ctypes.data, _lib.MEM_HOST))
    elif tgt_w >= w and tgt_h >= h:
        ctx.check(ctx.lib.vd3d_resize_cubic(ctx.h, bgr.ctypes.data, h, w, 3, out.ctypes.data, tgt_h, tgt_w,
                                            _lib.MEM_HOST))
    else:
        raise ValueError(f"inference_size {(tgt_w, tgt_h)} shrinks one axis of a {w}x{h} image and enlarges the other: "
                         "cv2's INTER_AREA takes no area path there, which the GPU path does not reproduce")
    return out


def infer_depth_tile(model_call, rgb_np, inference_size, tile=TILE_SIZE, pad=TILE_PAD):
    """core/render_depth.py:102-170 for this module's `pipe`: resize to inference_size, tile with `pad` of context,
    run every tile crop through the depth engine (batched per crop size), blend the predictions with Hann weights.
    Returns float32 [tgtH, tgtW].  Other model callables are refused: the tiles never leave the GPU."""
    if model_call is not hf_batch_safe_pipe:
        raise TypeError("infer_depth_tile runs this module's depth pipe on the GPU (vd3d_depth_tiled); load a model with "
                        "load_depth_model() / update_pipeline() and pass render_depth.pipe")
    if rgb_np.dtype != np.uint8:
        rgb_np = rgb_np.astype(np.uint8, copy=False)
    H, W = rgb_np.shape[:2]
    tgt_w, tgt_h = (inference_size or (W, H))
    bgr = _outer_resize(rgb_np, int(tgt_w), int(tgt_h))
    _u8, f32, _mm = depth_tiled([bgr], int(tgt_w), int(tgt_h), (int(tgt_w), int(tgt_h)), tile=tile, pad=pad,
                                want_f32=True)
    if TILE_DEBUG:
        for line in _plan_for(int(tgt_w), int(tgt_h), tile, pad).debug_lines():
            print(line)
    return f32[0]


def _run_pipe_or_tile(images_pil, inference_size):
    """core/render_depth.py:201-268 for the HF pipe: with USE_TILED_DEPTH each image goes through infer_depth_tile
    (one "[tile] range" line per image), otherwise the whole list through pipe."""
    if USE_TILED_DEPTH:
        _check_tiled_supported()
        preds = []
        for img in images_pil:
            rgb = np.array(img.convert("RGB"))
            dep = infer_depth_tile(pipe, rgb, inference_size, tile=TILE_SIZE, pad=TILE_PAD)
            dep_min, dep_max = float(np.nanmin(dep)), float(np.nanmax(dep))
            print(f"[tile] range min={dep_min:.6f} max={dep_max:.6f}")
            preds.append({"predicted_depth": dep})
        return preds
    try:
        res = pipe(images_pil, inference_size=inference_size)
        if isinstance(res, list):
            return res
        elif isinstance(res, dict):
            return [res]
        else:
            return [{"predicted_depth": res}]
    except TypeError:
        outs = []
        for img in images_pil:
            r = pipe(img, inference_size=inference_size)
            if isinstance(r, list):
                r = r[0]
            outs.append(r if isinstance(r, dict) else {"predicted_depth": r})
        return outs


# ---------------------------------------------------------------------------
# model loading entry points (core/render_depth.py:728-829, 973-1140) for the Depth-Anything and DPT checkpoints of the hot path
# ---------------------------------------------------------------------------
def _find_checkpoint_file(folder):
    for root, _dirs, files in os.walk(folder):
        for name in ("model.safetensors", "pytorch_model.bin"):
            if name in files:
                return os.path.join(root, name)
    return None


def ensure_model_downloaded(checkpoint):
    """Resolve a checkpoint id to (model, metadata) like core/render_depth.py:728-829 does for HF ids and local
    folders.  No network is assumed: an HF id is looked up in the reference's cache layout
    (weights/<org>_<name>/...), a directory is searched for model.safetensors / pytorch_model.bin.  Returns
    (state_dict, {"arch", "is_b200": True}) or (None, None) with a message, as the reference does on failure."""
    if not isinstance(checkpoint, str):
        print(f"❌ Unsupported checkpoint: {checkpoint!r}")
        return None, None
    folder = checkpoint if os.path.isdir(checkpoint) else os.path.join(local_model_dir, checkpoint.replace("/", "_"))
    path = _find_checkpoint_file(folder) if os.path.isdir(folder) else None
    if path is None:
        print(f"❌ No local weights for {checkpoint} under {folder} (no network: place model.safetensors there)")
        return None, None
    import json
    ckdir = os.path.dirname(path)
    needs_config = checkpoint in DA_CONFIG_REQUIRED
    if needs_config and not os.path.exists(os.path.join(ckdir, "config.json")):
        print(f"❌ {checkpoint}: no config.json next to {path} (its taps and head are only there)")
        return None, None
    try:
        arch, sd = load_checkpoint(path)
    except Exception as e:
        print(f"❌ Failed to load {path}: {e}")
        return None, None
    if arch is None:
        print(f"❌ {path} is not a Depth-Anything (V2, V1, Distill-Any-Depth, V2-Metric) or DPT-Large checkpoint")
        return None, None
    spec = None
    if isinstance(arch, dict):
        spec, arch = arch, da_arch(arch)
    elif _family_of(arch) == FAMILY_DA_V2:
        spec = da_spec(arch)
    meta = {"arch": arch, "is_b200": True, "path": path}
    if spec is not None:
        meta["spec"] = spec
        pp = os.path.join(ckdir, "preprocessor_config.json")
        if (needs_config or not is_plain_v2(spec)) and os.path.exists(pp):
            try:
                with open(pp) as f:
                    da_processor_from_json(json.load(f))
            except ValueError as e:
                print(f"❌ {pp}: {e}")
                return None, None
    if _family_of(arch) == FAMILY_DPT:
        pp = os.path.join(ckdir, "preprocessor_config.json")
        try:
            if os.path.exists(pp):
                with open(pp) as f:
                    meta["processor"] = dpt_processor_from_json(json.load(f))
            else:
                meta["processor"] = dict(DPT_PROCESSOR)
            dpt_processed_size(meta["processor"])
        except ValueError as e:
            print(f"❌ {pp}: {e}")
            return None, None
    return sd, meta


def _notify(widget, text):
    """Status text to a Tk-like label (config / after) or stdout."""
    if widget is None:
        print(text)
        return
    try:
        if hasattr(widget, "after"):
            widget.after(0, lambda: widget.config(text=text))
        else:
            widget.config(text=text)
    except Exception:
        print(text)


def update_pipeline(selected_model_var, status_label_widget, inference_res_var, offload_mode_dropdown, *args):
    """core/render_depth.py:973-1140: load the model named by the GUI variable on a worker thread, publish it as the
    module globals `pipe` / `pipe_type`, warm it up with one dummy frame, report through the status label.
    Returns the thread (the reference returns None; callers ignore the value)."""
    name = selected_model_var.get() if hasattr(selected_model_var, "get") else selected_model_var
    entry = supported_models.get(name)
    checkpoint = entry[0] if entry else name

    def work():
        try:
            sd, meta = ensure_model_downloaded(checkpoint)
            if sd is None:
                _notify(status_label_widget, f"❌ Failed to load model: {name}")
                return
            _notify(status_label_widget, "🔄 Warming up H100 depth engine...")
            load_depth_model(meta.get("spec") or meta["arch"], sd, 384, 384, processor=meta.get("processor"))
            from PIL import Image
            pipe([Image.new("RGB", (384, 384), (127, 127, 127))])
            _notify(status_label_widget, f"✅ Depth model loaded: {name} (libvd3d, sm_90a)")
        except Exception as e:
            _notify(status_label_widget, f"💥 Init error: {e}")

    t = threading.Thread(target=work, daemon=True)
    t.start()
    return t


def update_progress(processed, total, fps, eta, progress_bar, status_label):
    """core/render_depth.py:1342-1351."""
    progress_bar.config(value=processed)
    eta_txt = time.strftime("%H:%M:%S", time.gmtime(eta)) if eta > 0 else "--:--:--"
    status_label.config(text=f"📸 Processed: {processed}/{total} | {fps:.2f} FPS | ETA: {eta_txt}")


def choose_output_directory(output_label_widget, output_dir_var):
    """core/render_depth.py:1200-1204 (Tk directory dialog; GUI helper)."""
    from tkinter import filedialog
    d = filedialog.askdirectory()
    if d:
        output_dir_var.set(d)
        output_label_widget.config(text=f"📁 {d}")


# ---------------------------------------------------------------------------
# depth video in the reference's handoff format (core/render_depth.py:1736-1763, 1894-1935): per-frame min-max u8
# depth as XVID BGR .mkv + <name>.letterbox.json sidecar -- what render_sbs_3d's depth_path expects
# ---------------------------------------------------------------------------
def write_letterbox_sidecar(video_path, top, bottom, orig_w, orig_h):
    import json
    side = os.path.splitext(video_path)[0] + ".letterbox.json"
    with open(side, "w", encoding="utf-8") as f:
        json.dump({"top": int(top), "bottom": int(bottom), "orig_w": int(orig_w), "orig_h": int(orig_h)}, f, indent=2)
    return side


def read_letterbox_sidecar(video_path):
    import json
    side = os.path.splitext(video_path)[0] + ".letterbox.json"
    if not os.path.exists(side):
        return None
    with open(side, encoding="utf-8") as f:
        return json.load(f)


# ---------------------------------------------------------------------------
# letterbox tracker (core/render_depth.py:273-573): the pixel statistics come from the GPU (vd3d_letterbox_stats, one
# small record per frame); the scan, the gates, the bootstrap median and the hysteresis are host scalar logic
# ---------------------------------------------------------------------------
class _FrameStats:
    """GPU statistics of one u8 BGR frame: what the reference's helpers compute from its pixels.  has_prev: a
    previous gray plane was compared (absdiff is meaningful); prev_shape_differs: the previous plane had another
    shape, which is_scene_cut counts as a cut."""
    __slots__ = ("h", "w", "y_mean", "y_var", "s_mean", "edges", "frame_y_mean", "hist", "absdiff", "has_prev",
                 "prev_shape_differs")

    def row_edge_density(self):
        # _horizontal_edge_density: edges.mean(axis=1) / 255.0 on the 0/255 Canny map, built as numpy builds it
        return (self.edges.astype(np.float64) * 255.0) / np.intp(self.w) / 255.0


def _is_cuda_tensor(x):
    return torch is not None and isinstance(x, torch.Tensor) and x.is_cuda


def letterbox_stats(frames, prev_gray=None):
    """Statistics of same-shape u8 BGR frames in one GPU pass -> (list of _FrameStats, gray plane of the last frame).
    frames: a list of host frames [h,w,3], or a CUDA uint8 tensor [n,h,w,3] (the statistics then read device memory and
    the returned gray plane is a CUDA tensor).  prev_gray: the gray plane before the first frame (host array or CUDA
    tensor), or None.  Only the per-row / per-frame records come back to the host, in one copy."""
    from . import _lib
    ctx = _lib.default_context(0)
    device = _is_cuda_tensor(frames)
    if device:
        fr = frames.contiguous()
        if fr.dtype != torch.uint8 or fr.dim() != 4 or fr.shape[3] != 3:
            raise ValueError("Expected a uint8 CUDA tensor [n, h, w, 3] of BGR frames")
        n, h, w = (int(v) for v in fr.shape[:3])
    else:
        fr = np.ascontiguousarray(np.stack([np.asarray(f, dtype=np.uint8) for f in frames]))
        if fr.ndim != 4 or fr.shape[3] != 3:
            raise ValueError("Expected BGR uint8 image with 3 channels")
        n, h, w = fr.shape[:3]
    ym = np.empty((n, h), np.float32)
    yv = np.empty((n, h), np.float32)
    sm = np.empty((n, h), np.float32)
    ed = np.empty((n, h), np.int32)
    fm = np.empty(n, np.float32)
    hist = np.empty((n, 64), np.uint32)
    ad = np.empty(n, np.uint64)
    pg = None
    shape_differs = prev_gray is not None and tuple(prev_gray.shape) != (h, w)
    if prev_gray is not None and not shape_differs:
        if device:
            pg = (prev_gray if _is_cuda_tensor(prev_gray) else torch.from_numpy(np.asarray(prev_gray))).to(
                fr.device, torch.uint8).contiguous()
        else:
            pg = np.ascontiguousarray(prev_gray.cpu().numpy() if _is_cuda_tensor(prev_gray) else prev_gray,
                                      dtype=np.uint8)
    if device:
        last = torch.empty((h, w), dtype=torch.uint8, device=fr.device)
        torch.cuda.current_stream().synchronize()  # the frames may come from work queued on torch's stream
        fp, pp, lp, mem = fr.data_ptr(), pg.data_ptr() if pg is not None else None, last.data_ptr(), _lib.MEM_DEVICE
    else:
        last = np.empty((h, w), np.uint8)
        fp, pp, lp, mem = fr.ctypes.data, pg.ctypes.data if pg is not None else None, last.ctypes.data, _lib.MEM_HOST
    ctx.check(ctx.lib.vd3d_letterbox_stats(ctx.h, n, fp, h, w, pp, mem, ym.ctypes.data, yv.ctypes.data,
                                           sm.ctypes.data, ed.ctypes.data, fm.ctypes.data, hist.ctypes.data,
                                           ad.ctypes.data, lp))
    out = []
    for i in range(n):
        st = _FrameStats()
        st.h, st.w = h, w
        st.y_mean, st.y_var, st.s_mean, st.edges = ym[i], yv[i], sm[i], ed[i]
        st.frame_y_mean, st.hist, st.absdiff = fm[i], hist[i], int(ad[i])
        st.has_prev = i > 0 or pg is not None
        st.prev_shape_differs = i == 0 and shape_differs
        out.append(st)
    return out, last


def _stats1(frame_bgr):
    if frame_bgr is None or frame_bgr.ndim != 3 or frame_bgr.shape[2] != 3:
        raise ValueError("Expected BGR uint8 image with 3 channels")
    return letterbox_stats([frame_bgr])[0][0]


def _scene_cut_from_stats(st, prev_hist, mad_thresh=28.0, corr_thresh=0.60):
    import cv2
    if st.prev_shape_differs:
        return True
    if not st.has_prev:
        return False
    mad = float(np.float64(st.absdiff) / np.intp(st.h * st.w))
    if mad > mad_thresh:
        return True
    h1 = prev_hist.astype(np.float32).reshape(64, 1)
    h2 = st.hist.astype(np.float32).reshape(64, 1)
    cv2.normalize(h1, h1)
    cv2.normalize(h2, h2)
    return float(cv2.compareHist(h1, h2, cv2.HISTCMP_CORREL)) < corr_thresh


def _near_black_from_stats(st, mean_thresh=18, edge_thresh=0.02):
    return float(st.frame_y_mean) < mean_thresh and st.row_edge_density().mean() < edge_thresh


def _strict_robust_from_stats(st, y_thresh=16, var_thresh=3.0, sat_thresh=6.0, max_scan_frac=0.25,
                              min_band_frac=0.06, edge_max=0.04):
    h, w = st.h, st.w
    if h < 64 or w < 64:
        return 0, 0
    y_mean, y_var, s_mean, row_edge = st.y_mean, st.y_var, st.s_mean, st.row_edge_density()

    def scan(rows):
        run = 0
        for i in rows:
            if y_mean[i] < y_thresh and y_var[i] < var_thresh and s_mean[i] < sat_thresh and row_edge[i] <= edge_max:
                run += 1
            else:
                break
        if run < int(h * min_band_frac):
            run = 0
        if run % 2 == 1:
            run -= 1
        return max(run, 0)

    H = int(h * max_scan_frac)
    top = scan(range(0, H))
    bot = scan(range(h - 1, h - 1 - H, -1))
    if top + bot >= h * 0.6:  # absurd
        return 0, 0
    return int(top), int(bot)


def is_scene_cut(prev_gray, gray, mad_thresh=28.0, corr_thresh=0.60):
    """core/render_depth.py:295-319 on two gray planes: MAD above mad_thresh, else 64-bin histogram correlation below
    corr_thresh."""
    import cv2
    if prev_gray is None or gray is None:
        return False
    if prev_gray.shape != gray.shape:
        return True
    mad = float(np.mean(np.abs(prev_gray.astype(np.int16) - gray.astype(np.int16))))
    if mad > mad_thresh:
        return True
    h1 = cv2.calcHist([prev_gray], [0], None, [64], [0, 256])
    h2 = cv2.calcHist([gray], [0], None, [64], [0, 256])
    cv2.normalize(h1, h1)
    cv2.normalize(h2, h2)
    return float(cv2.compareHist(h1, h2, cv2.HISTCMP_CORREL)) < corr_thresh


def detect_letterbox_strict_robust(frame_bgr, y_thresh=16, var_thresh=3.0, sat_thresh=6.0, max_scan_frac=0.25,
                                   min_band_frac=0.06, edge_max=0.04):
    """core/render_depth.py:336-385: (top, bottom) bar rows of one frame, or (0, 0)."""
    h, w = frame_bgr.shape[:2]
    if h < 64 or w < 64:
        return 0, 0
    return _strict_robust_from_stats(_stats1(frame_bgr), y_thresh, var_thresh, sat_thresh, max_scan_frac,
                                     min_band_frac, edge_max)


def is_near_black_frame(frame_bgr, mean_thresh=18, edge_thresh=0.02):
    """core/render_depth.py:387-392: dark (luma mean) and nearly edge-free."""
    return _near_black_from_stats(_stats1(frame_bgr), mean_thresh, edge_thresh)


def detect_letterbox_multiframe_confidence(cap, original_height, fps, max_seconds=3, samples=9):
    """core/render_depth.py:394-455: ((top, bottom), confidence) from up to `samples` frames of the first
    max_seconds, skipping near-black frames and scene cuts; the capture position is restored."""
    import cv2
    try:
        total = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
    except Exception:
        total = 0
    window = max(min(total, int((fps if fps and fps > 0 else 30) * max_seconds)), 1)
    tops, bottoms = [], []
    prev_gray, prev_hist = None, None
    pos_backup = cap.get(cv2.CAP_PROP_POS_FRAMES)
    for i in np.linspace(0, max(0, window - 1), num=min(samples, window), dtype=int):
        cap.set(cv2.CAP_PROP_POS_FRAMES, int(i))
        ok, frame = cap.read()
        if not ok:
            continue
        (st,), gray = letterbox_stats([frame], prev_gray)
        if not (_near_black_from_stats(st) or _scene_cut_from_stats(st, prev_hist)):
            t, b = _strict_robust_from_stats(st)
            if 0 <= t < original_height and 0 <= b < original_height and (t + b) < original_height:
                tops.append(t)
                bottoms.append(b)
        prev_gray, prev_hist = gray, st.hist
    cap.set(cv2.CAP_PROP_POS_FRAMES, pos_backup or 0)
    if not tops:
        return (0, 0), 0.0
    t_med, b_med = int(np.median(tops)), int(np.median(bottoms))
    if t_med % 2:
        t_med -= 1
    if b_med % 2:
        b_med -= 1
    t_med, b_med = max(t_med, 0), max(b_med, 0)
    if t_med + b_med >= original_height * 0.6:
        return (0, 0), 0.0
    agree = sum(1 for t, b in zip(tops, bottoms) if abs(t - t_med) <= 4 and abs(b - b_med) <= 4)
    return (t_med, b_med), float(agree / max(1, len(tops)))


class LetterboxTracker:
    """core/render_depth.py:458-573: tracks and freezes letterbox bars, re-checking only at scene cuts on non-black
    frames, with a cooldown and confirm_needed-fold hysteresis.  States: locked_zero (no bars) and locked_bars.
    update() takes one frame; update_batch() takes a batch in one GPU pass with the same result frame by frame."""

    def __init__(self, h, fps, min_change=8, confirm_needed=3, max_total_frac=0.35, conf_enable=0.7,
                 conf_disable=0.6, cooldown_sec=3.0):
        self.h = int(h)
        self.fps = float(fps) if fps and fps > 0 else 30.0
        self.min_change = int(min_change)
        self.confirm_needed = int(confirm_needed)
        self.max_total_frac = float(max_total_frac)
        self.conf_enable = float(conf_enable)
        self.conf_disable = float(conf_disable)
        self.cooldown_frames = int(self.fps * cooldown_sec)
        self.top = 0
        self.bot = 0
        self.locked_zero = True
        self.locked_bars = False
        self._cand = (0, 0)
        self._streak = 0
        self._cooldown = 0
        self.prev_gray = None
        self._prev_hist = None

    def bootstrap(self, cap):
        (t, b), conf = detect_letterbox_multiframe_confidence(cap, self.h, self.fps)
        if conf >= self.conf_enable and (t + b) > 0:
            self.top, self.bot = t, b
            self.locked_bars, self.locked_zero = True, False
        else:
            self.top, self.bot = 0, 0
            self.locked_zero, self.locked_bars = True, False
        self._cooldown = self.cooldown_frames
        return self.top, self.bot, (self.locked_bars, self.locked_zero)

    def should_recheck(self, frame_idx):
        return self._cooldown <= 0

    def update(self, frame_bgr, frame_idx):
        return self.update_batch([frame_bgr], frame_idx)[-1]

    def update_batch(self, frames_bgr, first_idx=0):
        """update() on each frame in order (indices first_idx, first_idx + 1, ...) -> list of (top, bottom).  frames_bgr:
        a list of host frames or a CUDA uint8 tensor [n, h, w, 3] (the previous gray plane then stays on the device)."""
        stats, gray = letterbox_stats(frames_bgr, self.prev_gray)
        out = []
        for k, st in enumerate(stats):
            out.append(self._step(st, first_idx + k))
            self._prev_hist = st.hist
        self.prev_gray = gray
        return out

    def _step(self, st, frame_idx):
        if self._cooldown > 0:
            self._cooldown -= 1
        if _near_black_from_stats(st):
            return self.top, self.bot
        if not _scene_cut_from_stats(st, self._prev_hist):
            return self.top, self.bot
        if not self.should_recheck(frame_idx):
            return self.top, self.bot
        mt, mb = _strict_robust_from_stats(st)
        if (mt + mb) > int(self.h * self.max_total_frac):
            mt, mb = 0, 0
        if mt % 2:
            mt -= 1
        if mb % 2:
            mb -= 1
        mt, mb = max(mt, 0), max(mb, 0)
        if abs(mt - self.top) + abs(mb - self.bot) < self.min_change:
            self._streak = 0
            self._cand = (self.top, self.bot)
            return self.top, self.bot
        cand = (mt, mb)
        if cand == self._cand:
            self._streak += 1
        else:
            self._cand = cand
            self._streak = 1
        if self._streak >= self.confirm_needed:
            if self.locked_zero and (mt + mb) > 0:
                self.top, self.bot = mt, mb
                self.locked_zero, self.locked_bars = False, True
                self._cooldown = self.cooldown_frames
            elif self.locked_bars:
                self.top, self.bot = mt, mb
                self.locked_zero = (mt + mb) == 0
                self.locked_bars = (mt + mb) > 0
                self._cooldown = self.cooldown_frames
        return self.top, self.bot


def crop_by_bars(frame_bgr, top, bottom):
    """core/render_depth.py:577-583: drop the bar rows, unless that would leave nothing."""
    h = frame_bgr.shape[0]
    top, bottom = max(int(top), 0), max(int(bottom), 0)
    if top + bottom >= h:
        return frame_bgr
    return frame_bgr[top:h - bottom, :]


def letterbox_repad(depth_u8, top, bottom):
    """process_video2's re-pad of a u8 depth plane (core/render_depth.py:1919-1933) on the GPU
    (vd3d_letterbox_repad): INTER_CUBIC resize into the core rows, bar rows filled with the core's median."""
    from . import _lib
    ctx = _lib.default_context(0)
    src = np.ascontiguousarray(depth_u8, dtype=np.uint8)
    out = np.empty_like(src)
    ctx.check(ctx.lib.vd3d_letterbox_repad(ctx.h, src.ctypes.data, src.shape[0], src.shape[1], int(top), int(bottom),
                                           out.ctypes.data, _lib.MEM_HOST))
    return out


def _repad_device(src, top, bottom, dst):
    """vd3d_letterbox_repad on CUDA planes (src, dst: uint8 tensors [h, w], distinct)."""
    from . import _lib
    ctx = _lib.default_context(0)
    h, w = (int(v) for v in src.shape)
    ctx.check(ctx.lib.vd3d_letterbox_repad(ctx.h, src.data_ptr(), h, w, int(top), int(bottom), dst.data_ptr(),
                                           _lib.MEM_DEVICE))


_staging = {}  # (n, H, W) -> pinned host tensor [n, H, W, 3]: the upload buffer of the depth-video pass


def iter_depth_frames(cap, W, H, invert=False, inference_size=None, batch_size=8, max_frames=None, tracker=None,
                      status=None):
    """The u8 depth planes depth_video_from_video writes, in order, from the frames cap.read() returns.  With a
    bootstrapped `tracker` (ignore_letterbox_bars), every frame read goes through tracker.update and each frame of a
    batch is re-padded with the bars the tracker holds after the batch's last frame, as process_video2 does.
    Each batch goes to the GPU in one pinned upload; the tracker's statistics and the depth read that copy, the re-pad
    works on the device depth, and the planes come back in one download."""
    from . import _lib
    _check_tiled_supported()
    n, batch = 0, []
    tiled = USE_TILED_DEPTH

    def flush():
        k = len(batch)
        host = _staging.get((k, H, W))
        if host is None:
            host = _staging[(k, H, W)] = torch.empty((k, H, W, 3), dtype=torch.uint8).pin_memory()
        hn = host.numpy()
        for i, f in enumerate(batch):
            hn[i] = f
        batch.clear()
        dev = host.to("cuda", non_blocking=True)
        torch.cuda.current_stream().synchronize()  # the library reads `dev` on its own stream
        bars = tracker.update_batch(dev, n + 1)[-1] if tracker is not None else (0, 0)
        if tiled:
            # process_video2's tiled branch: _run_pipe_or_tile -> infer_depth_tile on each (Pillow-resized) frame,
            # then _normalize_to_u8 to the frame size, in one vd3d_depth_tiled call
            frames, tw, th = dev, W, H
            if inference_size is not None:
                tw, th = int(inference_size[0]), int(inference_size[1])
                eng = _plan_for(tw, th, TILE_SIZE, TILE_PAD).engines()[0]  # the resize needs no weights: any engine
                frames = torch.stack([eng.resize_pil(f, tw, th) for f in dev])
            d8, _, ranges = depth_tiled(frames, tw, th, (W, H), invert)
            _print_tile_log(tw, th, ranges)
        elif inference_size is None:
            eng = _engine_for(W, H)
            d8 = torch.empty((k, H, W), dtype=torch.uint8, device=dev.device)
            for i0 in range(0, k, 8):
                idx = range(i0, min(k, i0 + 8))
                eng.infer_batch_u8_device([dev[i].data_ptr() for i in idx], H, W, [d8[i].data_ptr() for i in idx],
                                          invert)
        else:
            # hf_batch_safe_pipe at inference_size -> convert_depth_to_grayscale -> invert -> INTER_CUBIC back to the
            # frame size: the composition vd3d_depth_infer_images computes for RGB images
            eng = _engine_for(*inference_size)
            rgb = dev.flip(-1)
            planes = []
            for i0 in range(0, k, 8):
                chunk = list(rgb[i0:i0 + 8])
                planes += [u8 for u8, _ in eng.infer_images(chunk, [inference_size] * len(chunk), invert)]
            d8 = torch.stack(planes)
            torch.cuda.current_stream().synchronize()  # stacked on torch's stream; the re-pad reads it on the library's
        if bars[0] or bars[1]:
            out = torch.empty_like(d8)
            for i in range(k):
                _repad_device(d8[i], bars[0], bars[1], out[i])
            d8 = out
        ctx = _lib.default_context(0)
        ctx.check(ctx.lib.vd3d_sync(ctx.h))
        return list(d8.cpu().numpy())

    while not cancel_requested.is_set():
        ok, frame = cap.read()
        if not ok or (max_frames is not None and n + len(batch) >= max_frames):
            break
        batch.append(frame)
        if len(batch) >= batch_size:
            for d8 in flush():
                n += 1
                yield d8
            if status is not None:
                _notify(status, f"📸 Processed: {n}")
    if batch and not cancel_requested.is_set():
        for d8 in flush():
            n += 1
            yield d8
        if status is not None:
            _notify(status, f"📸 Processed: {n}")


def depth_video_from_video(input_path, output_path, invert=False, inference_size=None, batch_size=8,
                           status=None, max_frames=None, ignore_letterbox_bars=False):
    """Frames of `input_path` -> depth video `output_path` in the reference's format (process_video2's `hf` branch):
    each frame through the depth engine, min-max u8 (convert_depth_to_grayscale), optional inversion, INTER_CUBIC
    resize back when inference_size was given, grey -> BGR, XVID.  Returns the number of frames written.
    ignore_letterbox_bars=False writes bars 0/0 to the sidecar.  True runs the reference's letterbox tracker: a
    bootstrap on the first int(fps * 3) frames decides the sidecar's bars, every frame updates the tracker, and each
    depth frame is re-padded to the tracked bars (iter_depth_frames)."""
    import cv2
    _check_tiled_supported()
    cap = cv2.VideoCapture(input_path)
    if not cap.isOpened():
        print(f"❌ Cannot open {input_path}")
        return 0
    raw_fps = cap.get(cv2.CAP_PROP_FPS)
    fps = raw_fps or 24.0
    W, H = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
    tracker = None
    top = bottom = 0
    if ignore_letterbox_bars:
        tracker = LetterboxTracker(H, raw_fps)
        top, bottom, (locked_bars, locked_zero) = tracker.bootstrap(cap)
        print(f"[VD3D] Bootstrap bars: top={top} bottom={bottom} | locked_bars={locked_bars} locked_zero={locked_zero}")
    write_letterbox_sidecar(output_path, top, bottom, W, H)
    out = cv2.VideoWriter(output_path, cv2.VideoWriter_fourcc(*"XVID"), fps, (W, H))
    if not out.isOpened():
        print(f"❌ Failed to open video writer for {os.path.basename(output_path)}")
        cap.release()
        return 0
    n = 0
    try:
        for d8 in iter_depth_frames(cap, W, H, invert, inference_size, batch_size, max_frames, tracker, status):
            out.write(cv2.cvtColor(d8, cv2.COLOR_GRAY2BGR))
            n += 1
    finally:
        cap.release()
        out.release()
    return n


# ---------------------------------------------------------------------------
# still images (core/render_depth.py:1196-1213, 1215-1340, 1353-1515): the drivers of the Depth tab's image modes.  The
# pixel work of the `pipe` path -- the inference-size resize, the DPT processor, one batched forward per processed
# size, the bicubic post-resize, min-max u8 and the resize back -- runs on the GPU in one call per batch
# (vd3d_depth_infer_images)
# ---------------------------------------------------------------------------
IMAGE_EXTENSIONS = (".jpeg", ".jpg", ".png")
_RESOLUTION = re.compile(r"^\s*(\d+)\s*x\s*(\d+)")


def parse_inference_resolution(res_string, fallback=(384, 384)):
    """core/render_depth.py:1196-1197: the (W, H) of a resolution choice of the Depth tab, read from its "<W>x<H>"
    prefix ("910x518 (Depth Anything)" -> (910, 518)); "Original" -> None (each image at its own size); anything
    else -> fallback."""
    s = res_string.strip()
    if s == "Original":
        return None
    m = _RESOLUTION.match(s)
    return (int(m.group(1)), int(m.group(2))) if m else fallback


def get_dynamic_batch_size(base=4, scale_factor=1.0, max_limit=32, reserve_vram_gb=1.0):
    """core/render_depth.py:1206-1213: base images per GB of device memory beyond reserve_vram_gb, capped at
    max_limit; base without a GPU."""
    if torch is not None and torch.cuda.is_available():
        total = torch.cuda.get_device_properties(0).total_memory / (1024 ** 3)
        return min(int(base * max(0, total - reserve_vram_gb) * scale_factor), max_limit)
    return base


def _rgb_array(img):
    if isinstance(img, np.ndarray):
        if img.ndim != 3 or img.shape[2] != 3:
            raise ValueError(f"expected an RGB array [h, w, 3], got shape {img.shape}")
        return np.ascontiguousarray(img, dtype=np.uint8)
    return np.asarray(img.convert("RGB"), dtype=np.uint8)


def depth_images(images, inference_size=None, invert=False):
    """Still images -> u8 depth planes, each at its image's own size: what _run_pipe_or_tile + the image drivers'
    min-max normalisation, inversion and cv2 INTER_CUBIC resize back compute for the `pipe` path.  images: PIL
    images or RGB u8 arrays.  Images whose input size (inference_size, or their own size) maps to the same DPT
    processed size share one batched forward (up to 8 per forward), whatever their source sizes."""
    rgbs = [_rgb_array(img) for img in images]
    groups = {}
    for k, a in enumerate(rgbs):
        iw, ih = inference_size if inference_size is not None else (a.shape[1], a.shape[0])
        groups.setdefault(model_processed_size(int(iw), int(ih)), []).append(k)
    out = [None] * len(rgbs)
    for (ph, pw), idxs in groups.items():
        iw, ih = inference_size if inference_size is not None else (rgbs[idxs[0]].shape[1], rgbs[idxs[0]].shape[0])
        eng = _engine_for(int(iw), int(ih))
        for i0 in range(0, len(idxs), 8):
            chunk = idxs[i0:i0 + 8]
            ins = [inference_size] * len(chunk)
            for k, (d8, _) in zip(chunk, eng.infer_images([rgbs[k] for k in chunk], ins, invert=invert)):
                out[k] = d8
    return out


def _progress(bar, **kw):
    if bar is not None:
        bar.config(**kw)


def _grayscale_image(depth_u8, colormap_name):
    """The written image: grayscale ("L").  Colour maps come from matplotlib in the reference, which this package
    does not use: any other name falls back to grayscale with the reference's message."""
    from PIL import Image
    if colormap_name != "default":
        print(f"⚠️ Unknown colormap '{colormap_name}', defaulting to grayscale.")
    return Image.fromarray(np.ascontiguousarray(depth_u8, dtype=np.uint8))  # 2-D u8 -> mode "L"


def _ensure_output_dir(output_dir, status_label):
    """The output-directory checks of the image drivers: True when output_dir exists or was created."""
    if not output_dir:
        print("⚠️ Please select an output directory before processing.")
        _notify(status_label, "❌ Output directory not selected.")
        return False
    if not os.path.exists(output_dir):
        try:
            os.makedirs(output_dir)
        except Exception as e:
            print(f"❌ Could not create output directory:\n{e}")
            _notify(status_label, "❌ Failed to create output directory.")
            return False
    return True


def _depth_output_path(output_dir, file_path):
    return os.path.join(output_dir, f"{os.path.splitext(os.path.basename(file_path))[0]}_depth.png")


def process_images_in_folder(folder_path, batch_size_widget, output_dir_var, inference_res_var, status_label,
                             progress_bar, root, invert_var):
    """core/render_depth.py:1229-1340: every .jpeg / .jpg / .png of folder_path (os.listdir order) -> <stem>_depth.png
    (u8 grayscale, the image's size) in the output directory, in chunks of the batch size.  GUI variables may be Tk
    variables or plain values; status text goes to status_label (or stdout), root is not used.  With USE_TILED_DEPTH
    each image goes through infer_depth_tile and _normalize_to_u8, otherwise through depth_images."""
    _check_tiled_supported()
    output_dir = str(_val(output_dir_var) or "").strip()
    if not _ensure_output_dir(output_dir, status_label):
        return
    inference_size = parse_inference_resolution(_val(inference_res_var))
    try:
        user_value = str(_val(batch_size_widget) or "").strip()
        batch_size = int(user_value) if user_value else get_dynamic_batch_size()
        if batch_size <= 0:
            raise ValueError
    except Exception:
        batch_size = get_dynamic_batch_size()
        _notify(status_label, f"⚠️ Invalid batch size. Using dynamic batch size: {batch_size}")
    image_files = [os.path.join(folder_path, f) for f in os.listdir(folder_path) if f.lower().endswith(IMAGE_EXTENSIONS)]
    if not image_files:
        _notify(status_label, "⚠️ No image files found.")
        return
    total = len(image_files)
    invert = bool(_val(invert_var))
    _notify(status_label, f"📂 Processing {total} images...")
    _progress(progress_bar, maximum=total, value=0)
    from PIL import Image
    start = time.time()
    for i in range(0, total, batch_size):
        if cancel_requested.is_set():
            _notify(status_label, "❌ Cancelled by user.")
            return
        batch_files = image_files[i:i + batch_size]
        images = [Image.open(f).convert("RGB") for f in batch_files]
        print(f"🚀 Running batch of {len(images)} images at {inference_size}")
        if USE_TILED_DEPTH:
            planes = [p["predicted_depth"] for p in _run_pipe_or_tile(images, inference_size)]
        else:
            planes = depth_images(images, inference_size, invert)
        for j, plane in enumerate(planes):
            if cancel_requested.is_set():
                _notify(status_label, "❌ Cancelled during batch.")
                return
            file_path = batch_files[j]
            try:
                d8 = _normalize_to_u8(plane, images[j].size, invert=invert) if USE_TILED_DEPTH else plane
                _grayscale_image(d8, "default").save(_depth_output_path(output_dir, file_path))
            except Exception as e:
                print(f"❌ Error processing {file_path}: {e}")
                continue
            done = i + j + 1
            elapsed = time.time() - start
            fps = done / elapsed if elapsed > 0 else 0
            eta = (total - done) / fps if fps > 0 else 0
            if progress_bar is not None and status_label is not None:
                update_progress(done, total, fps, eta, progress_bar, status_label)
    _notify(status_label, "✅ All images processed successfully!")
    _progress(progress_bar, value=total)


def process_image(file_path, colormap_var, invert_var, output_dir_var, inference_res_var, input_label, output_label,
                  status_label, progress_bar, folder=False):
    """core/render_depth.py:1353-1477: one image -> <stem>_depth.png in the output directory, the same file the folder
    driver writes for it.  The Tk previews (input_label / output_label thumbnails) are not produced; colour maps fall
    back to grayscale."""
    from PIL import Image
    _check_tiled_supported()
    image = Image.open(file_path).convert("RGB")
    inference_size = parse_inference_resolution(_val(inference_res_var))
    print("📏 Using inference size:", inference_size)
    invert = bool(_val(invert_var))
    colormap_name = str(_val(colormap_var)).strip().lower()
    if USE_TILED_DEPTH:
        dep = _run_pipe_or_tile([image], inference_size)[0]["predicted_depth"]
    else:
        dep = depth_images([image], inference_size, invert)[0]
    try:
        d8 = _normalize_to_u8(dep, image.size, invert=invert) if USE_TILED_DEPTH else dep
        depth_image = _grayscale_image(d8, colormap_name)
    except Exception as e:
        print(f"❌ Error extracting depth: {e}")
        return
    output_dir = str(_val(output_dir_var) or "").strip()
    if not _ensure_output_dir(output_dir, status_label):
        return
    path = _depth_output_path(output_dir, file_path)
    depth_image.save(path)
    if not folder:
        cancel_requested.clear()
        _notify(status_label, f"✅ Image saved: {path}")
        _progress(progress_bar, value=100)
        if progress_bar is not None and hasattr(progress_bar, "stop"):
            progress_bar.stop()


def open_image(status_label_widget, progress_bar_widget, colormap_var, invert_var, output_dir_var, inference_res_var,
               input_label_widget, output_label_widget):
    """core/render_depth.py:1480-1514: pick an image (Tk file dialog) and run process_image on a worker thread.
    Returns the thread, or None when no file was picked."""
    file_path = _dialog("askopenfilename", filetypes=[("Image Files", "*.jpeg;*.jpg;*.png")])
    if not file_path:
        return None
    cancel_requested.clear()
    _notify(status_label_widget, "🔄 Processing image...")
    if progress_bar_widget is not None and hasattr(progress_bar_widget, "start"):
        progress_bar_widget.start(10)

    def work():
        process_image(file_path, colormap_var, invert_var, output_dir_var, inference_res_var, input_label_widget,
                      output_label_widget, status_label_widget, progress_bar_widget)
        if progress_bar_widget is not None and hasattr(progress_bar_widget, "stop"):
            progress_bar_widget.stop()

    t = threading.Thread(target=work, daemon=True)
    t.start()
    return t


def process_image_folder(batch_size_widget, output_dir_var, inference_res_var, status_label, progress_bar, invert_var,
                         root):
    """core/render_depth.py:1215-1226: pick a folder (Tk directory dialog) and run process_images_in_folder on a
    worker thread.  Returns the thread, or None when no folder was picked."""
    folder_path = _dialog("askdirectory", title="Select Folder Containing Images")
    if not folder_path:
        cancel_requested.clear()
        _notify(status_label, "⚠️ No folder selected.")
        return None
    t = threading.Thread(target=process_images_in_folder, args=(folder_path, batch_size_widget, output_dir_var,
                                                                 inference_res_var, status_label, progress_bar, root,
                                                                 invert_var), daemon=True)
    t.start()
    return t


def _gui_only(name):
    def f(*_a, **_k):
        raise RuntimeError(f"{name} is a Tk GUI driver of the reference (core/render_depth.py); on the GPU path use "
                           "depth_video_from_video() / hf_batch_safe_pipe() instead")
    f.__name__ = name
    return f


# GUI batch drivers the reference's main window imports (VisionDepth3D.py:41-53); the import list must resolve
open_video = _gui_only("open_video")
process_video_folder = _gui_only("process_video_folder")
process_videos_in_folder = _gui_only("process_videos_in_folder")
