"""Drop-in for the reference's core/merged_pipeline.py, backed by libvd3d.so: the SRVGGNetCompact network on wgmma
implicit-GEMM convolutions, and run_esrgan's whole untiled chain (input resize, network, INTER_CUBIC resizes,
addWeighted) as one device call, vd3d_sr_upscale.  start_merged_pipeline drives an image folder through it into ffmpeg.

    from visiondepth3d_b200 import merged_pipeline as core_merged_pipeline
    core_merged_pipeline.start_merged_pipeline(settings, progress_bar, status_label)

The reference loads `weights/RealESR_Gx4_fp16.onnx` through ONNXRuntime (VisionDepth3D.py:1094-1100).  ONNX files are
not read here: the model is an upstream-format state_dict, either handed to load_esrgan() or found as `<stem>.pth` /
`<stem>.safetensors` next to the settings' model_path.  Two architectures are served, told apart by the keys:
SRVGGNetCompact (`body.{i}.weight` ...: realesr-general-x4v3 / realesr-animevideov3) and RRDBNet (RealESRGAN_x4plus,
BSRGAN x4 / x2: `conv_first`, `body.{i}.rdb{j}.conv{k}` ... or the old-ESRGAN `RRDB_trunk.{i}.RDB{j}.conv{k}` ...).  RIFE frame interpolation is not built: its network is not part of the reference (it loads a
`RIFE_fp32.onnx` it does not ship), so rife_session stays None and run_rife returns [] -- what the reference does
without that file.
"""
import ctypes as C
import os
import re
import threading
import time

import numpy as np

from . import _lib

esrgan_session = None  # the reference's module global: truthy once a model is loaded
rife_session = None    # RIFE is not built (see the module docstring)
suspend_flag = threading.Event()
cancel_flag = threading.Event()
progress_bar = None
status_label = None


# old-ESRGAN / BSRGAN key names -> the basicsr names of the same RRDBNet tensors
_RRDB_RENAMES = [(re.compile(r"^RRDB_trunk\.(\d+)\.RDB(\d)\.conv(\d)\."), r"body.\1.rdb\2.conv\3."),
                 (re.compile(r"^trunk_conv\."), "conv_body."), (re.compile(r"^upconv1\."), "conv_up1."),
                 (re.compile(r"^upconv2\."), "conv_up2."), (re.compile(r"^HRconv\."), "conv_hr.")]


def is_rrdb_state_dict(sd):
    """True for RRDBNet keys (either naming), False for SRVGGNetCompact's."""
    return any(k.startswith(("conv_first.", "RRDB_trunk.")) for k in sd)


def rrdb_layout(sd):
    """(state dict in the basicsr naming as float32 arrays, nb, net scale) of an RRDBNet state dict in either naming;
    ValueError unless it is exactly an RRDBNet with num_feat 64, growth 32, 3 input / output channels and one or two
    up-convs (basicsr's pixel-unshuffle x2 / x1 variants take 12 / 48 input channels and are refused)."""
    canon = {}
    for k, v in sd.items():
        for pat, new in _RRDB_RENAMES:
            k = pat.sub(new, k)
        canon[k] = np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, dtype=np.float32)
    w = canon.get("conv_first.weight")
    if w is None or w.ndim != 4:
        raise ValueError("not an RRDBNet state dict: no conv_first weight")
    if w.shape[1] != 3:
        raise ValueError(f"RRDBNet conv_first takes {w.shape[1]} input channels: only the 3-channel x4 / x2 models are "
                         "served (not the pixel-unshuffle variants)")
    nb = 0
    while f"body.{nb}.rdb1.conv1.weight" in canon:
        nb += 1
    scale = 4 if "conv_up2.weight" in canon else 2
    shapes = {"conv_first": (64, 3), "conv_body": (64, 64), "conv_up1": (64, 64), "conv_hr": (64, 64),
              "conv_last": (3, 64)}
    if scale == 4:
        shapes["conv_up2"] = (64, 64)
    for i in range(nb):
        for j in range(1, 4):
            for k in range(1, 6):
                shapes[f"body.{i}.rdb{j}.conv{k}"] = (32 if k < 5 else 64, 64 + 32 * (k - 1))
    want = {f"{n}.weight": (co, ci, 3, 3) for n, (co, ci) in shapes.items()}
    want.update({f"{n}.bias": (co,) for n, (co, _) in shapes.items()})
    bad = sorted(k for k in set(want) | set(canon) if k not in canon or k not in want or canon[k].shape != want[k])
    if nb < 1 or bad:
        raise ValueError(f"not an RRDBNet state dict (num_feat 64, growth 32): {nb} blocks, mismatched keys {bad[:4]}")
    return canon, nb, scale


def _pack3x3(w, cols, cin_pad, rows=None):
    """Conv weight [Cout, Cin, 3, 3] -> f16 [rows or Cout, 9 * cin_pad], tap-major, input channel c at column cols[c]."""
    co, ci = w.shape[:2]
    out = np.zeros((rows or co, 9, cin_pad), dtype=np.float32)
    out[:co, :, cols] = w.transpose(0, 2, 3, 1).reshape(co, 9, ci)
    return out.reshape(-1, 9 * cin_pad).astype(np.float16)


def _phase_weights(w):
    """nearest x2 followed by a 3x3 conv (pad 1) as four 3x3 convs on the low-resolution map, one per output phase
    (py, px): output (2y + py, 2x + px) reads upsampled row 2y + py + dy = low row y + (py + dy) // 2, so the taps that
    land on one low-resolution pixel add up.  [4 * Cout, Cin, 3, 3], rows (py * 2 + px) * Cout + co."""
    co = w.shape[0]
    ph = np.zeros((2, 2) + w.shape, dtype=np.float32)
    for py in range(2):
        for px in range(2):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    ph[py, px, :, :, (py + dy) // 2 + 1, (px + dx) // 2 + 1] += w[:, :, dy + 1, dx + 1]
    return ph.reshape((4 * co,) + w.shape[1:])


def pack_rrdb(sd):
    """(nb, net scale, {engine tensor name: array}) of an RRDBNet state dict in either naming (vd3d_sr_set_rrdb's
    layouts: dense-block inputs with each 32-channel growth slice padded to 64 channels)."""
    sd, nb, scale = rrdb_layout(sd)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    t = {"rr.first.w": _pack3x3(sd["conv_first.weight"], [0, 1, 2], 64), "rr.first.b": f32(sd["conv_first.bias"])}
    for i in range(nb):
        for j in range(3):
            for k in range(1, 6):
                cols = list(range(64)) + [64 * (s + 1) + c for s in range(k - 1) for c in range(32)]
                n = f"body.{i}.rdb{j + 1}.conv{k}"
                t[f"rr.{i}.{j}.{k}.w"] = _pack3x3(sd[n + ".weight"], cols, 64 * k)
                t[f"rr.{i}.{j}.{k}.b"] = f32(sd[n + ".bias"])
    t["rr.body.w"], t["rr.body.b"] = _pack3x3(sd["conv_body.weight"], list(range(64)), 64), f32(sd["conv_body.bias"])
    for u in range(1, 2 if scale == 2 else 3):
        t[f"rr.up{u}.w"] = _pack3x3(_phase_weights(sd[f"conv_up{u}.weight"]), list(range(64)), 64)
        t[f"rr.up{u}.b"] = f32(np.tile(sd[f"conv_up{u}.bias"], 4))
    t["rr.hr.w"], t["rr.hr.b"] = _pack3x3(sd["conv_hr.weight"], list(range(64)), 64), f32(sd["conv_hr.bias"])
    t["rr.last.w"] = _pack3x3(sd["conv_last.weight"], list(range(64)), 64, rows=32)
    t["rr.last.b"] = f32(np.pad(sd["conv_last.bias"], (0, 29)))
    return nb, scale, t


class SrEngine:
    """Real-ESRGAN network forward on the GPU: SRVGGNetCompact (num_feat 64, x4) or RRDBNet (x4 or x2, chosen by the
    state dict's keys): BGR u8 [h,w,3] -> BGR u8 [s h, s w, 3], s = net_scale."""

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
        self.net_scale = 4
        if is_rrdb_state_dict(state_dict):
            nb, self.net_scale, tensors = pack_rrdb(state_dict)
            for name, arr in tensors.items():
                self._set(name, arr)
            self.check(self.lib.vd3d_sr_set_rrdb(self.h, nb, self.net_scale))
            self.num_conv = 0  # ignored by RRDBNet engines
            return
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
        out = np.empty((self.net_scale * h, self.net_scale * w, 3), dtype=np.uint8)
        self.check(self.lib.vd3d_sr_forward(self.h, f.ctypes.data, h, w, self.num_conv, out.ctypes.data, _lib.MEM_HOST))
        return out

    def upscale_ptrs(self, frames, h, w, params, outs, mem):
        """vd3d_sr_upscale on len(frames) frames BGR u8 [h,w,3] given as addresses in `mem` (host / device) memory."""
        n = len(frames)
        fp = (C.c_void_p * n)(*frames)
        op = (C.c_void_p * n)(*outs)
        self.ctx.check(self.lib.vd3d_sr_upscale(self.ctx.h, self.h, n, fp, int(h), int(w), self.num_conv,
                                                C.byref(params), op, mem))

    def upscale_chain(self, frames, params, out_size):
        """run_esrgan's untiled chain on a list of same-size host frames; returns new arrays of out_size (w, h)."""
        fr = [np.ascontiguousarray(f, dtype=np.uint8) for f in frames]
        h, w = fr[0].shape[:2]
        outs = [np.empty((out_size[1], out_size[0], 3), dtype=np.uint8) for _ in fr]
        self.upscale_ptrs([f.ctypes.data for f in fr], h, w, params, [o.ctypes.data for o in outs], _lib.MEM_HOST)
        return outs

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


def random_rrdb_state_dict(nb=23, scale=4, seed=0, naming="basicsr"):
    """Random-init RRDBNet weights (num_feat 64, growth 32) in the basicsr naming or, with naming="esrgan", the
    old-ESRGAN / BSRGAN one, for benchmarks and tests.  He init (LeakyReLU 0.2) on conv_first and the upsampling tail;
    the dense blocks at a tenth of it, so that the trunk stays a modest residual over conv_first's features as in a
    trained model; conv_last small with a 0.5 bias, so that a natural frame maps to an image with spread in [0, 1] and
    little clipping (not a constant or saturated image against which any kernel output would pass)."""
    rng = np.random.default_rng(seed)
    gain = 2.0 / (1.0 + 0.2 ** 2)
    sd = {}

    def conv(name, co, ci, mult, bias_std=0.01):
        sd[name + ".weight"] = (rng.standard_normal((co, ci, 3, 3)) * mult * (gain / (9 * ci)) ** 0.5).astype(np.float32)
        sd[name + ".bias"] = (rng.standard_normal(co) * bias_std).astype(np.float32)

    conv("conv_first", 64, 3, 1.0)
    for i in range(nb):
        for j in range(1, 4):
            for k in range(1, 6):
                conv(f"body.{i}.rdb{j}.conv{k}", 32 if k < 5 else 64, 64 + 32 * (k - 1), 0.1)
    conv("conv_body", 64, 64, 0.1)
    for u in range(1, 2 if scale == 2 else 3):
        conv(f"conv_up{u}", 64, 64, 1.0)
    conv("conv_hr", 64, 64, 1.0)
    conv("conv_last", 3, 64, 0.035)
    sd["conv_last.bias"] = np.full(3, 0.5, np.float32)
    if naming == "esrgan":
        old = {"conv_body.": "trunk_conv.", "conv_up1.": "upconv1.", "conv_up2.": "upconv2.", "conv_hr.": "HRconv."}
        out = {}
        for k, v in sd.items():
            m = re.match(r"body\.(\d+)\.rdb(\d)\.conv(\d)\.(.*)", k)
            if m:
                k = f"RRDB_trunk.{m.group(1)}.RDB{m.group(2)}.conv{m.group(3)}.{m.group(4)}"
            for a, b in old.items():
                if k.startswith(a):
                    k = b + k[len(a):]
            out[k] = v
        sd = out
    elif naming != "basicsr":
        raise ValueError(f"naming must be 'basicsr' or 'esrgan', not {naming!r}")
    return sd


def load_esrgan(state_dict=None, num_conv=32, seed=0):
    """Make run_esrgan serve a model: an upstream SRVGGNetCompact or RRDBNet state_dict (tensors or arrays), or
    random-init SRVGGNetCompact."""
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


_BLEND_ALPHA = {"LOW": 0.85, "MEDIUM": 0.5, "HIGH": 0.25}


def upscale_params(blend_mode="OFF", input_res_pct=100, model_name="RealESR_Gx4_fp16", target_size=None):
    """vd3d_upscale_params of a run_esrgan call: blend_images' alpha (exactly "OFF": none; an unknown mode: 1.0),
    the x2 model-name quirk, target_size (w, h) or None."""
    tw, th = (int(target_size[0]), int(target_size[1])) if target_size else (0, 0)
    alpha = -1.0 if blend_mode == "OFF" else _BLEND_ALPHA.get(blend_mode.upper(), 1.0)
    return _lib.UpscaleParams(float(input_res_pct), 2 if "x2" in model_name.lower() else 4, tw, th, float(alpha))


def run_esrgan(frame, blend_mode="OFF", input_res_pct=100, model_name="RealESR_Gx4_fp16", target_size=None, tile=None,
               tile_pad=8):
    """core/merged_pipeline.py:240-267.  Untiled: one vd3d_sr_upscale call (one upload, one download).  Returns the
    input frame when no model is loaded or the engine fails, like the reference."""
    if not esrgan_session:
        return frame
    if not tile:
        h, w = frame.shape[:2]
        p = upscale_params(blend_mode, input_res_pct, model_name, target_size)
        size = (p.target_w, p.target_h) if target_size else (w, h)
        if blend_mode != "OFF":
            assert size == (w, h)  # blend_images: cv2.addWeighted raises on two different sizes
        # the caller's sizes raise here, as the reference's cv2.resize calls do; only the engine takes the fallback
        nw, nh = int(w * input_res_pct / 100), int(h * input_res_pct / 100)
        if nw < 1 or nh < 1 or size[0] < 1 or size[1] < 1:
            raise ValueError(f"run_esrgan: empty size (input {nw}x{nh}, output {size[0]}x{size[1]})")
        try:
            return esrgan_session.upscale_chain([frame], p, size)[0]
        except _lib.Vd3dError as e:
            print(f"❌ ESRGAN failed: {e}")
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


# ---------------------------------------------------------------------------
# RIFE (core/merged_pipeline.py:196-219): the helpers as the reference defines them; without a RIFE network
# rife_session is None and run_rife interpolates nothing
# ---------------------------------------------------------------------------
def concatenate_images(frame1, frame2):
    """Both frames as float32 / 255, stacked on the channel axis."""
    return np.concatenate([frame1.astype(np.float32) / 255.0, frame2.astype(np.float32) / 255.0], axis=2)


def preprocess_rife(frame):
    """HWC -> NCHW float32 with a batch axis of one."""
    return np.expand_dims(np.transpose(frame, (2, 0, 1)), 0).astype(np.float32)


def run_rife(frame1, frame2, multiplier):
    """multiplier - 1 frames between frame1 and frame2 from rife_session, or [] without one (or when it fails)."""
    if not rife_session:
        return []
    batch = np.repeat(preprocess_rife(concatenate_images(frame1, frame2)), multiplier - 1, axis=0)
    try:
        out = rife_session.run(None, {rife_session.get_inputs()[0].name: batch})[0]
    except Exception as e:
        print(f"❌ RIFE inference error: {e}")
        return []
    return [(f * 255).astype(np.uint8) for f in np.transpose(np.clip(out, 0, 1), (0, 2, 3, 1))]


# ---------------------------------------------------------------------------
# folder helpers and progress (core/merged_pipeline.py:64-80, 189-194)
# ---------------------------------------------------------------------------
def extract_frame_number(filename):
    """The first run of digits in the basename as an int; inf when there is none (such names sort last)."""
    m = re.search(r"\d+", os.path.basename(filename))
    return float("inf") if m is None else int(m.group(0))


def natural_sort(files):
    """Stable sort on extract_frame_number."""
    return sorted(files, key=extract_frame_number)


def update_progress(done, total, start):
    """Progress bar value and "Progress: done/total | FPS | ETA" on the status label, marshalled with .after(0, ...);
    nothing without both widgets."""
    if not progress_bar or not status_label:
        return
    el = time.time() - start
    rate = done / el if el > 0 else 0
    eta = (total - done) / rate if rate > 0 else float("inf")
    eta_s = "--:--" if eta == float("inf") else time.strftime("%H:%M:%S", time.gmtime(eta))
    pct = done / total * 100 if total else 0
    try:
        progress_bar.after(0, lambda: progress_bar.configure(value=pct))
        status_label.after(0, lambda: status_label.configure(
            text=f"Progress: {done}/{total} | FPS: {rate:.2f} | ETA: {eta_s}"))
    except Exception:
        pass


def _gui_only(name):
    def f(*_a, **_k):
        raise RuntimeError(f"{name} is a Tk GUI helper of the reference (core/merged_pipeline.py); pass paths to "
                           "start_merged_pipeline's settings instead")
    f.__name__ = name
    return f


# Tk dialogs the reference's main window imports (VisionDepth3D.py:55-61); the import list must resolve
select_video_and_generate_frames = _gui_only("select_video_and_generate_frames")
select_output_file = _gui_only("select_output_file")
select_frames_folder = _gui_only("select_frames_folder")


def _encoder_args(codec):
    if "nvenc" in (codec or "").lower():
        return ["-c:v", "h264_nvenc", "-preset", "p4", "-tune", "hq", "-rc", "vbr", "-cq", "19", "-rc-lookahead", "20",
                "-bf:v", "3", "-b_ref_mode", "middle", "-pix_fmt", "yuv420p"]
    return ["-c:v", "libx264", "-preset", "medium", "-crf", "18", "-pix_fmt", "yuv420p"]


def start_ffmpeg_writer(output_path, width, height, fps, codec):
    """core/merged_pipeline.py:390-426: an ffmpeg process reading raw bgr24 frames of width x height on stdin."""
    import subprocess
    cmd = ["ffmpeg", "-y", "-f", "rawvideo", "-vcodec", "rawvideo", "-pix_fmt", "bgr24", "-s", f"{width}x{height}",
           "-r", str(fps), "-i", "-"] + _encoder_args(codec) + [output_path]
    return subprocess.Popen(cmd, stdin=subprocess.PIPE)


# ---------------------------------------------------------------------------
# model loading
# ---------------------------------------------------------------------------
def _read_state_dict(path):
    if path.lower().endswith(".safetensors"):
        from safetensors.numpy import load_file
        sd = load_file(path)
    else:
        import torch
        sd = torch.load(path, map_location="cpu", weights_only=True)
    for key in ("params_ema", "params"):  # upstream Real-ESRGAN checkpoints wrap the state dict
        if isinstance(sd, dict) and key in sd and isinstance(sd[key], dict):
            sd = sd[key]
            break
    sd = {k: (v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)) for k, v in sd.items()}
    if is_rrdb_state_dict(sd):
        try:
            rrdb_layout(sd)
        except ValueError as e:
            raise ValueError(f"{path}: {e}") from None
        return sd
    n = len([k for k in sd if k.startswith("body.") and k.endswith(".bias")])
    ok = n >= 3
    for i in range(n if ok else 0):
        w = sd.get(f"body.{2 * i}.weight")
        ci, co = (3 if i == 0 else 64), (48 if i == n - 1 else 64)
        ok = ok and w is not None and tuple(w.shape) == (co, ci, 3, 3) and (i == n - 1 or f"body.{2 * i + 1}.weight" in sd)
    if not ok:
        raise ValueError(f"{path}: not an SRVGGNetCompact x4 state dict (num_feat 64)")
    return sd


def _model_files(model_path):
    stem, ext = os.path.splitext(model_path)
    if ext.lower() in (".pth", ".safetensors"):
        return [model_path]
    return [stem + ".pth", stem + ".safetensors"]


def load_esrgan_from(model_path):
    """The settings' model_path: the path itself when it is a .pth / .safetensors file, else <stem>.pth or
    <stem>.safetensors next to it (the ONNX file is not read).  None, with the reference's message, when there is
    none; a state dict that is neither SRVGGNetCompact nor RRDBNet raises."""
    global esrgan_session
    for f in _model_files(model_path):
        if os.path.exists(f):
            return load_esrgan(_read_state_dict(f))
    print(f"❌ ESRGAN model missing: {model_path}")
    esrgan_session = None
    return None


# ---------------------------------------------------------------------------
# the image-folder driver (core/merged_pipeline.py:85-104, 287-386)
# ---------------------------------------------------------------------------
_SR_BATCH = 4  # frames per vd3d_sr_upscale call


class _MergedPlan:
    def __init__(self, settings):
        self.frames_dir = settings["frames_folder"]
        self.output_path = settings["output_file"]
        self.codec = settings["codec"]
        self.width, self.height = int(settings["width"]), int(settings["height"])
        self.fps = settings["fps"]
        self.fps_mult = settings["fps_multiplier"]
        self.enable_rife = settings["enable_rife"]
        self.enable_upscale = settings["enable_upscale"]
        self.blend_mode = settings.get("blend_mode", "OFF")
        self.input_res_pct = settings.get("input_res_pct", 100)
        self.model_path = settings.get("model_path", "weights/RealESR_Gx4_fp16.onnx")
        self.output_fps = self.fps * self.fps_mult if self.enable_rife else self.fps
        self.files = []

    def prepare(self):
        """Model (before any file is listed or written) and the frame list; False when there are no frames."""
        if self.enable_upscale:
            load_esrgan_from(self.model_path)
        self.files = natural_sort([os.path.join(self.frames_dir, f) for f in os.listdir(self.frames_dir)
                                   if f.lower().endswith((".jpg", ".jpeg", ".png"))])
        if not self.files:
            print("❌ No frames found in selected folder.")
            return False
        return True


def _prefetch(files, ring, free, out_q, stop):
    """Reader thread: decode each file (unreadable ones are skipped), copy it into a free slot of the pinned ring when
    it has the ring's shape, and queue (slot, None) or (None, array); None ends the stream."""
    import cv2
    try:
        for fp in files:
            if stop.is_set():
                break
            img = cv2.imread(fp, cv2.IMREAD_COLOR)
            if img is None:
                continue
            if ring is not None and img.shape == ring.arrays[0].shape:
                k = free.get()
                if k is None:
                    break
                np.copyto(ring.arrays[k], img)
                out_q.put((k, None))
            else:
                out_q.put((None, img))
    finally:
        out_q.put(None)


def _close_rings(pinned):
    while pinned:
        pinned.pop().close()


def _merged_batches(plan, stop, pinned):
    """Frames for the writer, in order, as (list of frames, release) pairs: release() returns pinned output slots.
    The pinned rings are appended to `pinned` instead of being freed here: the frames handed out are views into them,
    and whoever consumes those views (a writer thread may still be writing them after this generator has finished)
    frees the rings with _close_rings once it is done with every frame.
    Upscaling on with a model: batches of up to _SR_BATCH same-size frames through vd3d_sr_upscale (target size
    (width, height), scale 4, the settings' blend and input_res_pct).  Upscaling on without a model: the source
    frames.  Upscaling off: the loader's resize to (width, height) on the GPU (INTER_AREA when the source is wider than
    the target, else INTER_CUBIC).  cancel_flag is read once per source frame after the first."""
    import cv2
    import queue
    from . import render_3d as R
    sr = esrgan_session if plan.enable_upscale else None
    target = (plan.width, plan.height)
    probe, i0 = None, 0
    for i0, fp in enumerate(plan.files):  # the ring is shaped by the first readable frame, which goes in first
        probe = cv2.imread(fp, cv2.IMREAD_COLOR)
        if probe is not None:
            break
    if probe is None:
        print("❌ No readable frames.")
        return
    lib = _lib.load()
    ring = outs = None
    if sr:
        ring = R._PinnedRing(lib, 3 * _SR_BATCH, probe.shape)
        pinned.append(ring)
        outs = R._PinnedRing(lib, 2 * _SR_BATCH, (plan.height, plan.width, 3))
        pinned.append(outs)
    params = upscale_params(plan.blend_mode, plan.input_res_pct, target_size=target) if sr else None
    free, free_out, q = queue.Queue(), queue.Queue(), queue.Queue(maxsize=3 * _SR_BATCH)
    for k in range(3 * _SR_BATCH if sr else 0):
        free.put(k)
    free_out.put(0)
    free_out.put(1)
    if sr:
        k = free.get()
        np.copyto(ring.arrays[k], probe)
        q.put((k, None))
    else:
        q.put((None, probe))
    th = threading.Thread(target=_prefetch, args=(plan.files[i0 + 1:], ring, free, q, stop), daemon=True)
    th.start()
    try:
        n_src, pending, done = 0, None, False
        while not done:
            batch = [pending] if pending is not None else []
            pending = None
            while len(batch) < (_SR_BATCH if sr else 1):
                if batch and q.empty():
                    break  # hand over what is there rather than wait for a full batch
                item = q.get()
                if item is None:
                    done = True
                    break
                if n_src > 0 and cancel_flag.is_set():
                    done = True
                    break
                n_src += 1
                if batch and (item[0] is None or batch[0][0] is None):  # arrays travel alone
                    pending = item
                    break
                batch.append(item)
            if not batch:
                break
            if not sr:
                frames = [img for _, img in batch]
                if not plan.enable_upscale:
                    frames = [R.resize_area(f, *target) if f.shape[1] > target[0] else _resize_cubic(f, *target)
                              for f in frames]
                yield frames, (lambda: None)
                continue
            if batch[0][0] is None:  # a frame of another size than the first one: host memory, alone
                yield sr.upscale_chain([batch[0][1]], params, target), (lambda: None)
                continue
            half = free_out.get()
            ks = [k for k, _ in batch]
            optrs = [outs.ptrs[half * _SR_BATCH + j] for j in range(len(ks))]
            sr.upscale_ptrs([ring.ptrs[k] for k in ks], probe.shape[0], probe.shape[1], params, optrs, _lib.MEM_HOST)
            for k in ks:
                free.put(k)
            yield ([outs.arrays[half * _SR_BATCH + j] for j in range(len(ks))],
                   (lambda h=half: free_out.put(h)))
    finally:
        stop.set()
        free.put(None)
        while th.is_alive():  # unblock a reader waiting on a full queue
            try:
                q.get(timeout=0.05)
            except queue.Empty:
                pass
        th.join()


def _merged_stream(plan, stop, pinned):
    """(frame, release, is_source_frame) in writer order, with the reference's sequencing: the first frame, then for every further
    source frame run_rife(prev, curr)'s frames (when enable_rife) followed by the frame itself."""
    prev = None
    for frames, release in _merged_batches(plan, stop, pinned):
        for j, f in enumerate(frames):
            last = j == len(frames) - 1
            if prev is not None and plan.enable_rife:
                for g in run_rife(prev, f, plan.fps_mult):
                    yield g, None, False
            prev = f
            yield f, (release if last else None), True


def iter_merged_frames(settings):
    """Every frame start_merged_pipeline hands its writer, in order (copies), without a codec: for tests and for
    callers that encode themselves."""
    plan = _MergedPlan(settings)
    if not plan.prepare():
        return
    stop, pinned = threading.Event(), []
    gen = _merged_stream(plan, stop, pinned)
    try:
        for f, release, _ in gen:
            out = np.array(f, copy=True)
            if release:
                release()
            yield out
    finally:
        gen.close()
        _close_rings(pinned)


class _PipeWriter:
    def __init__(self, proc):
        self.proc = proc

    def write(self, frame):
        self.proc.stdin.write(memoryview(np.ascontiguousarray(frame)).cast("B"))

    def close(self):
        try:
            self.proc.stdin.close()
        except Exception:
            pass
        self.proc.wait()


def start_merged_pipeline(settings, progress_widget, status_label_widget):
    """core/merged_pipeline.py:287-386: an image folder -> (RIFE) -> Real-ESRGAN -> video.

    A reader thread decodes the frames into a pinned ring, the calling thread hands batches to vd3d_sr_upscale (or the
    GPU resize when upscaling is off), and a writer thread pipes bgr24 into start_ffmpeg_writer's process -- or, where
    the ffmpeg binary is missing, a cv2.VideoWriter (mp4v).  The writer is opened at (width, height) and output fps
    fps * fps_multiplier whenever enable_rife, as in the reference."""
    global progress_bar, status_label
    import queue
    import shutil
    from . import render_3d as R
    progress_bar, status_label = progress_widget, status_label_widget
    plan = _MergedPlan(settings)
    print("⚠️ RIFE interpolation is not built: no frames are interpolated")
    if not plan.prepare():
        return
    if shutil.which("ffmpeg") is not None:
        sink = _PipeWriter(start_ffmpeg_writer(plan.output_path, plan.width, plan.height, plan.output_fps, plan.codec))
    else:
        print("⚠️ ffmpeg binary not found: writing through cv2.VideoWriter instead")
        sink = R._FrameSink(plan.output_path, (plan.width, plan.height), plan.output_fps, "mp4v", False, None, 0)
    to_write, errors = queue.Queue(maxsize=4 * _SR_BATCH), []

    def writer():
        while True:
            item = to_write.get()
            if item is None:
                return
            f, release = item
            try:
                if not errors:
                    sink.write(f)
            except Exception as e:
                print(f"❌ write error: {e}")
                errors.append(e)
            if release:
                release()

    th = threading.Thread(target=writer, daemon=True)
    th.start()
    stop, pinned = threading.Event(), []
    start = time.time()
    total = len(plan.files) if not plan.enable_rife else len(plan.files) - 1
    n = 0
    gen = _merged_stream(plan, stop, pinned)
    try:
        for f, release, src in gen:
            to_write.put((f, release))
            n += src
            if src and n > 1:  # progress per source frame after the first
                update_progress(n, total, start)
    finally:
        gen.close()
        to_write.put(None)
        th.join()          # every queued frame is written (or dropped after a write error) ...
        _close_rings(pinned)  # ... before the pinned buffers they point into are freed
        sink.close()
    update_progress(total, total, start)
    try:
        status_label.after(0, lambda: status_label.configure(text="✅ Processing Complete!"))
    except Exception:
        pass
