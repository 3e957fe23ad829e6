"""Drop-in for the hot-path surface of the reference's core/render_depth.py: the `pipe`
callable protocol and the depth -> uint8 normalisation, backed by the libvd3d depth engine
(Depth-Anything-V2 on wgmma tensor cores).  GUI, ONNX, Marigold, DepthCrafter and the
letterbox tracker are outside the GPU hot path (SURVEY.md section 2).

Protocol kept (core/render_depth.py:1113-1119, consumers 201-268 and 1894-1917):
    pipe(images: list[PIL.Image], inference_size: (W, H) | None) -> list[{"predicted_depth": Tensor[h, w]}]
with `predicted_depth` already resized (bicubic) to the PIL image size, as
transformers' DepthEstimationPipeline.postprocess does.
"""
import os
import threading
import time

import numpy as np

from .depth_engine import DepthEngine, processed_size as _processed_size
from .depth_weights import CONFIGS, hf_config

try:
    import torch
    torch.set_grad_enabled(False)  # the reference does this at import (core/render_depth.py:42)
except Exception:  # pragma: no cover
    torch = None

# module globals the reference's callers read (core/render_depth.py:34-36, 992)
pipe = None
pipe_type = None
_engine = None

# the three checkpoints of the hot path (core/render_depth.py:695-697)
supported_models = {
    "Depth Anything V2 Small": ("depth-anything/Depth-Anything-V2-Small-hf", "vits"),
    "Depth Anything V2 Base": ("depth-anything/Depth-Anything-V2-Base-hf", "vitb"),
    "Depth Anything V2 Large": ("depth-anything/Depth-Anything-V2-Large-hf", "vitl"),
}


def load_checkpoint(path):
    """HF-format checkpoint (model.safetensors / pytorch_model.bin of
    depth-anything/Depth-Anything-V2-{Small,Base,Large}-hf) -> state_dict.  If a config.json sits next
    to it, the architecture is cross-checked against depth_weights.CONFIGS."""
    import json
    import os
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path)
    else:
        sd = torch.load(path, map_location="cpu")
    arch = None
    hidden = sd["backbone.embeddings.cls_token"].shape[-1]
    for name, c in CONFIGS.items():
        if c["hidden"] == hidden:
            arch = name
    cfg_path = os.path.join(os.path.dirname(path), "config.json")
    if arch and os.path.exists(cfg_path):
        cj = json.load(open(cfg_path))
        c = CONFIGS[arch]
        got = (cj.get("neck_hidden_sizes"), cj.get("fusion_hidden_size"),
               cj.get("backbone_config", {}).get("out_indices"))
        want = (c["neck"], c["fusion"], c["taps"])
        if any(g is not None and list(g) != list(w) if isinstance(w, list) else (g is not None and g != w)
               for g, w in zip(got, want)):
            raise ValueError(f"config.json {got} does not match the built-in {arch} configuration {want}")
    return arch, sd


_state_dict = None      # weights of the loaded model (HF naming): engines for other processed sizes are built from it
_arch = None
_engines = {}           # (processed_h, processed_w) -> DepthEngine, all sharing _state_dict
cancel_requested = threading.Event()   # core/render_depth.py:38 (the GUI's cancel flag for depth jobs)


def _weights_dir():
    """<project root>/weights, where the reference keeps its checkpoints (core/render_depth.py:615-626)."""
    return os.path.join(os.path.abspath(os.path.join(os.path.dirname(__file__), "..")), "weights")


local_model_dir = _weights_dir()


def _engine_for(width, height):
    """The engine whose DPT processed size fits a (width, height) image; built on first use from the loaded weights
    (the HF processor picks a keep-aspect multiple-of-14 size per image, so one model serves every aspect)."""
    global _engine
    if _state_dict is None:
        raise RuntimeError("no depth model loaded: call load_depth_model() / update_pipeline() first")
    key = _processed_size(width, height)
    eng = _engines.get(key)
    if eng is None:
        eng = DepthEngine(_arch, key[0], key[1])
        eng.load_state_dict(_state_dict)
        _engines[key] = eng
    _engine = eng
    return eng


def load_depth_model(arch="vits", state_dict=None, width=1920, height=1080, seed=0):
    """Make `pipe` serve a Depth-Anything-V2 model.  `state_dict` uses HF DepthAnythingForDepthEstimation naming
    (e.g. from a local safetensors checkpoint); without one a random-init model (torch.manual_seed(seed)) is used --
    there is no network here and the reference ships no weights.  (width, height) only pre-builds the engine for that
    frame shape; other shapes get their own engine on first use."""
    global pipe, pipe_type, _state_dict, _arch
    if state_dict is None:
        from transformers import DepthAnythingForDepthEstimation
        torch.manual_seed(seed)
        state_dict = DepthAnythingForDepthEstimation(hf_config(arch)).eval().state_dict()
    for e in _engines.values():
        e.close()
    _engines.clear()
    _state_dict, _arch = state_dict, arch
    eng = _engine_for(width, height)
    pipe = hf_batch_safe_pipe
    pipe_type = "hf"
    return pipe, {"arch": arch, "processed_size": (eng.image_h, eng.image_w), "config": CONFIGS[arch]}


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
    """cv2.resize(u8 plane, (width, height), interpolation=cv2.INTER_CUBIC) on the GPU (vd3d_resize_cubic_u8): the
    resize the reference's depth writer applies to the u8 depth (core/render_depth.py:1917, 193)."""
    from . import _lib
    ctx = _lib.default_context(0)
    src = np.ascontiguousarray(plane, dtype=np.uint8)
    assert src.ndim == 2
    out = np.empty((int(height), int(width)), dtype=np.uint8)
    ctx.check(ctx.lib.vd3d_resize_cubic_u8(ctx.h, src.ctypes.data, src.shape[0], src.shape[1], out.ctypes.data,
                                           int(height), int(width), _lib.MEM_HOST))
    return out


def _normalize_to_u8(depth_f, out_size, invert=False, pclip=(1.0, 99.0)):
    """core/render_depth.py:173-194 (the ndarray / tiled-depth front end): non-finite values -> 0, clip to the
    [p1, p99] percentiles (np.percentile, linear), fall back to min-max when they coincide and to flat 128 when the
    frame is flat, truncate to u8, optional inversion, INTER_CUBIC resize to out_size = (W, H) on the GPU.  The
    percentile front end is a host helper: the HF tensor path of the hot loop never takes it (1907-1917)."""
    d = np.asarray(depth_f, dtype=np.float32)
    if not np.isfinite(d).all():
        d = np.nan_to_num(d, nan=0.0, posinf=0.0, neginf=0.0)
    lo, hi = np.percentile(d, pclip[0]), np.percentile(d, pclip[1])
    if hi - lo >= 1e-6:
        u8 = (np.clip((d - lo) / (hi - lo), 0.0, 1.0) * 255.0).astype(np.uint8)
    else:
        mn, mx = float(d.min()), float(d.max())
        if mx - mn >= 1e-6:
            u8 = (((d - mn) / (mx - mn + 1e-6)) * 255.0).astype(np.uint8)
        else:
            u8 = np.full_like(d, 128, dtype=np.uint8)
    if invert:
        u8 = 255 - u8
    return resize_cubic_u8(u8, out_size[0], out_size[1])


# ---------------------------------------------------------------------------
# model loading entry points (core/render_depth.py:728-829, 973-1140) for the three DA-V2 checkpoints of the hot path
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
    try:
        arch, sd = load_checkpoint(path)
    except Exception as e:
        print(f"❌ Failed to load {path}: {e}")
        return None, None
    if arch is None:
        print(f"❌ {path} is not a Depth-Anything-V2 Small / Base / Large checkpoint")
        return None, None
    return sd, {"arch": arch, "is_b200": True, "path": path}


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
            load_depth_model(meta["arch"], sd, 384, 384)
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


def depth_video_from_video(input_path, output_path, invert=False, inference_size=None, batch_size=8,
                           status=None, max_frames=None):
    """Frames of `input_path` -> depth video `output_path` in the reference's format (process_video2's `hf` branch
    without the letterbox tracker, i.e. bars 0/0 in the sidecar): each frame through the depth engine, min-max u8
    (convert_depth_to_grayscale), optional inversion, INTER_CUBIC resize back when inference_size was given, grey ->
    BGR, XVID.  Returns the number of frames written."""
    import cv2
    from PIL import Image
    cap = cv2.VideoCapture(input_path)
    if not cap.isOpened():
        print(f"❌ Cannot open {input_path}")
        return 0
    fps = cap.get(cv2.CAP_PROP_FPS) or 24.0
    W, H = int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
    write_letterbox_sidecar(output_path, 0, 0, W, H)
    out = cv2.VideoWriter(output_path, cv2.VideoWriter_fourcc(*"XVID"), fps, (W, H))
    if not out.isOpened():
        print(f"❌ Failed to open video writer for {os.path.basename(output_path)}")
        cap.release()
        return 0
    n, batch = 0, []

    def flush():
        nonlocal n
        if inference_size is None:
            eng = _engine_for(W, H)
            for _, d8 in eng.infer_batch(batch, invert=invert):
                out.write(cv2.cvtColor(d8, cv2.COLOR_GRAY2BGR))
                n += 1
        else:
            pil = [Image.fromarray(f[..., ::-1].copy()) for f in batch]
            for res in hf_batch_safe_pipe(pil, inference_size):
                d8 = convert_depth_to_grayscale(res["predicted_depth"])
                if invert:
                    d8 = 255 - d8
                d8 = resize_cubic_u8(d8, W, H)
                out.write(cv2.cvtColor(d8, cv2.COLOR_GRAY2BGR))
                n += 1
        batch.clear()
        if status is not None:
            _notify(status, f"📸 Processed: {n}")

    try:
        while not cancel_requested.is_set():
            ok, frame = cap.read()
            if not ok or (max_frames is not None and n + len(batch) >= max_frames):
                break
            batch.append(frame)
            if len(batch) >= batch_size:
                flush()
        if batch and not cancel_requested.is_set():
            flush()
    finally:
        cap.release()
        out.release()
    return n


def _gui_only(name):
    def f(*_a, **_k):
        raise RuntimeError(f"{name} is a Tk GUI driver of the reference (core/render_depth.py); on the GPU path use "
                           "depth_video_from_video() / hf_batch_safe_pipe() instead")
    f.__name__ = name
    return f


# GUI batch drivers the reference's main window imports (VisionDepth3D.py:41-53); the import list must resolve
open_image = _gui_only("open_image")
open_video = _gui_only("open_video")
process_image = _gui_only("process_image")
process_image_folder = _gui_only("process_image_folder")
process_images_in_folder = _gui_only("process_images_in_folder")
process_video_folder = _gui_only("process_video_folder")
process_videos_in_folder = _gui_only("process_videos_in_folder")
