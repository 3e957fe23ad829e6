"""Generate tests/golden/*.npz by running the UNMODIFIED reference (CPU, via
tools/refshim.py) on seeded synthetic inputs.  Build-container only.

    python tools/gen_golden.py

Golden files hold outputs only (inputs are regenerated from the seed by
visiondepth3d_b200.synth), plus versions of the third-party libs used.
"""
import os
import sys
import threading

import numpy as np

sys.path.insert(0, os.path.dirname(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import refshim  # noqa: E402
from visiondepth3d_b200.synth import synth_frame  # noqa: E402

OUT = os.path.join(os.path.dirname(__file__), "..", "tests", "golden")


class Var:
    def __init__(self, v):
        self.v = v

    def get(self):
        return self.v


def run_pixel_shift(r3d, torch, w, h, iw, ih, n_frames, kind, **kw):
    """pixel_shift_cuda on n_frames consecutive frames (floating-window state carries)."""
    refshim.reset_singletons(r3d)
    out = {}
    for i in range(n_frames):
        fr, dp = synth_frame(i, iw, ih, kind)
        ft = r3d.frame_to_tensor(fr)
        dt = r3d.depth_to_tensor(dp)
        l, r, s = r3d.pixel_shift_cuda(ft, dt, w, h, 4.5, -1.5, -6.0, return_shift_map=True, **kw)
        out[f"left{i}"] = l
        out[f"right{i}"] = r
        out[f"shift{i}"] = s.numpy().astype(np.float16 if False else np.float32)
    return out


def every_row(g, step):
    """Every step-th row of the stored eyes (tests/util.py `rows`): keeps a fixture under 1 MB."""
    return {k: (v[::step] if k.startswith(("left", "right")) else v) for k, v in g.items()}


def run_loop(r3d, torch, cv2, src_w, src_h, n_frames, kind, rp):
    """Drive the body of render_sbs_3d in memory by writing lossless-ish input is not
    possible (codecs are lossy) -> we run the real render_sbs_3d with cv2 capture
    monkey-patched to an in-memory frame source and the writer to a collector."""
    refshim.reset_singletons(r3d)
    frames = [synth_frame(i, src_w, src_h, kind) for i in range(n_frames)]

    class Cap:
        def __init__(self, which):
            self.which = which
            self.pos = 0

        def isOpened(self):
            return True

        def get(self, prop):
            if prop == cv2.CAP_PROP_FRAME_COUNT:
                return float(n_frames)
            if prop == cv2.CAP_PROP_FPS:
                return 24.0
            if prop == cv2.CAP_PROP_POS_FRAMES:
                return float(self.pos)
            return 0.0

        def set(self, prop, v):
            if prop == cv2.CAP_PROP_POS_FRAMES:
                self.pos = int(v)
            return True

        def read(self):
            if self.pos >= n_frames:
                return False, None
            f = frames[self.pos][self.which].copy()
            self.pos += 1
            return True, f

        def release(self):
            pass

    collected = []

    class Writer:
        def __init__(self, *a, **k):
            pass

        def isOpened(self):
            return True

        def write(self, f):
            collected.append(f.copy())

        def release(self):
            pass

    real_cap, real_wr = cv2.VideoCapture, cv2.VideoWriter
    cv2.VideoCapture = lambda path: Cap(0 if path == "rgb" else 1)
    cv2.VideoWriter = Writer
    try:
        r3d.render_sbs_3d(
            "rgb", "depth", "out.avi", "XVID", 24.0, rp["output_width"], rp["output_height"],
            4.5, -1.5, -6.0, rp["sharpness_factor"], rp["output_format"], Var(rp.get("aspect_name", "Default (16:9)")),
            r3d.aspect_ratios, rp["dof_strength"],
            feather_strength=rp["feather_strength"], blur_ksize=rp["blur_ksize"],
            use_subject_tracking=rp["use_subject_tracking"],
            use_floating_window=rp["use_floating_window"],
            max_pixel_shift_percent=0.02, suspend_flag=threading.Event(),
            cancel_flag=threading.Event(),
            preserve_original_aspect=rp["preserve_original_aspect"],
            zero_parallax_strength=rp["zero_parallax_strength"],
            color_saturation=rp.get("color_saturation", 1.0),
            color_contrast=rp.get("color_contrast", 1.0),
            color_brightness=rp.get("color_brightness", 0.0),
            **{k: rp[k] for k in ("enable_edge_masking", "enable_feathering",
                                  "convergence_strength", "enable_dynamic_convergence", "ipd_factor",
                                  "parallax_balance", "depth_pop_gamma", "fg_pop_multiplier", "auto_crop_black_bars")
               if k in rp},
        )
    finally:
        cv2.VideoCapture, cv2.VideoWriter = real_cap, real_wr
    return {f"final{i}": f for i, f in enumerate(collected)}


def main():
    mods = refshim.load_reference(("render_3d",))
    r3d = mods["render_3d"]
    import cv2
    import torch
    import torchvision
    torch.set_num_threads(os.cpu_count())
    os.makedirs(OUT, exist_ok=True)
    meta = dict(torch=torch.__version__, torchvision=torchvision.__version__, cv2=cv2.__version__,
                numpy=np.__version__)

    # A. pixel_shift_cuda, identity resize, GUI-style params, 3 consecutive frames
    g = run_pixel_shift(r3d, torch, 320, 180, 320, 180, 3, "smooth",
                        blur_ksize=9, feather_strength=10.0, zero_parallax_strength=0.01)
    np.savez_compressed(os.path.join(OUT, "ps_smooth_320x180.npz"), **every_row(g, 2), **meta)
    # B. 2x upsample inside pixel_shift (Half-SBS style), no floating window
    g = run_pixel_shift(r3d, torch, 320, 180, 160, 90, 2, "smooth",
                        blur_ksize=5, feather_strength=4.0, enable_floating_window=False,
                        convergence_strength=0.5)
    np.savez_compressed(os.path.join(OUT, "ps_up2_320x180.npz"), **g, **meta)
    # C. noise content (adversarial LSB), edge masking off, even blur ksize
    g = run_pixel_shift(r3d, torch, 192, 108, 192, 108, 1, "noise",
                        blur_ksize=4, feather_strength=10.0, enable_edge_masking=False,
                        use_subject_tracking=False)
    np.savez_compressed(os.path.join(OUT, "ps_noise_192x108.npz"), **g, **meta)

    # D. full loop, Half-SBS (config-2 shape scaled down 6x: 320x180 source)
    base = dict(output_width=320, output_height=180, sharpness_factor=0.2, output_format="Half-SBS",
                dof_strength=0.0, feather_strength=10.0, blur_ksize=9, use_subject_tracking=True,
                use_floating_window=True, preserve_original_aspect=False, zero_parallax_strength=0.01)
    g = run_loop(r3d, torch, cv2, 320, 180, 6, "smooth", base)
    np.savez_compressed(os.path.join(OUT, "loop_halfsbs_320x180.npz"), **g, **meta)
    # E. full loop, Full-SBS preserve aspect (config-3 shape scaled down), DOF on + colour grade
    rp = dict(base, output_format="Full-SBS", preserve_original_aspect=True, dof_strength=2.0,
              color_saturation=1.1, color_contrast=1.05, color_brightness=0.02)
    g = run_loop(r3d, torch, cv2, 320, 180, 5, "smooth", rp)
    np.savez_compressed(os.path.join(OUT, "loop_fullsbs_dof_320x180.npz"), **g, **meta)
    # F. anaglyph + interlaced formats, render defaults (no tracking)
    rp = dict(base, output_format="Red-Cyan Anaglyph", preserve_original_aspect=True,
              use_subject_tracking=False, use_floating_window=False, feather_strength=0.0, blur_ksize=1)
    g = run_loop(r3d, torch, cv2, 256, 144, 3, "smooth", rp)
    np.savez_compressed(os.path.join(OUT, "loop_anaglyph_256x144.npz"), **g, **meta)
    rp = dict(rp, output_format="Passive Interlaced")
    g = run_loop(r3d, torch, cv2, 256, 144, 3, "smooth", rp)
    np.savez_compressed(os.path.join(OUT, "loop_interlaced_256x144.npz"), **g, **meta)
    # G. heal_missing_pixels (dead code in the reference's loop, named by north_star): standalone op
    rng = np.random.default_rng(21)
    H, W = 90, 160
    yy, xx = np.mgrid[0:H, 0:W]
    warped = np.stack([(xx / W), (yy / H), ((xx + yy) % 32) / 32.0]).astype(np.float32)
    warped[:, 30:60, 50:90] = rng.random((3, 30, 40), dtype=np.float32)
    orig = np.clip(warped + 0.1 * rng.standard_normal(warped.shape).astype(np.float32), 0, 1).astype(np.float32)
    edge = (rng.random((1, H, W), dtype=np.float32) > 0.9).astype(np.float32)
    outs = {}
    for name, em in (("none", None), ("edge", edge)):
        outs["heal_" + name] = r3d.heal_missing_pixels(
            torch.from_numpy(warped), None, torch.from_numpy(orig),
            torch.from_numpy(em) if em is not None else None, 0.5).numpy()
    np.savez_compressed(os.path.join(OUT, "heal_160x90.npz"), warped=warped, orig=orig, edge=edge, **outs)
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


def gen_vr():
    """H. VR format: 1600x900 eyes -> pad_to_aspect_ratio(1440, 1600) = non-integer INTER_AREA (x1.111) + black
    bars, hstack to 2880x1600.  Separate entry (`python tools/gen_golden.py vr`) so the earlier fixtures stay
    byte-identical.  Stored per frame: every 3rd row / column of the image band (the rest of the 2880x1600 frame is
    black), the band position, and a sha256 of the whole frame."""
    import hashlib
    mods = refshim.load_reference(("render_3d",))
    r3d = mods["render_3d"]
    import cv2
    import torch
    import torchvision
    torch.set_num_threads(os.cpu_count())
    meta = dict(torch=torch.__version__, torchvision=torchvision.__version__, cv2=cv2.__version__,
                numpy=np.__version__)
    rp = dict(output_width=1600, output_height=900, sharpness_factor=0.2, output_format="VR",
              dof_strength=0.0, feather_strength=10.0, blur_ksize=9, use_subject_tracking=True,
              use_floating_window=True, preserve_original_aspect=False, zero_parallax_strength=0.01)
    g = run_loop(r3d, torch, cv2, 320, 180, 3, "smooth", rp)
    out = {}
    for k, f in g.items():
        assert f.shape == (1600, 2880, 3), f.shape
        rows = np.nonzero(f.reshape(1600, -1).any(axis=1))[0]
        y0, y1 = int(rows.min()), int(rows.max()) + 1
        out[k + "_band"] = f[y0:y1:3, ::3]
        out[k + "_y0"] = np.int32(y0)
        out[k + "_y1"] = np.int32(y1)
        out[k + "_sha256"] = np.frombuffer(hashlib.sha256(f.tobytes()).digest(), dtype=np.uint8)
    p = os.path.join(OUT, "loop_vr_320x180.npz")
    np.savez_compressed(p, **out, **meta)
    print(p, os.path.getsize(p), {k: v.shape for k, v in out.items() if k.endswith("_band")})


def gen_extra():
    """I-K. loop cases that pin the crop / aspect / fractional-fit branches of render_sbs_3d
    (`python tools/gen_golden.py extra`; the earlier fixtures stay byte-identical)."""
    mods = refshim.load_reference(("render_3d",))
    r3d = mods["render_3d"]
    import cv2
    import torch
    import torchvision
    torch.set_num_threads(os.cpu_count())
    meta = dict(torch=torch.__version__, torchvision=torchvision.__version__, cv2=cv2.__version__,
                numpy=np.__version__)
    base = dict(output_width=320, output_height=180, sharpness_factor=0.2, output_format="Half-SBS",
                dof_strength=0.0, feather_strength=10.0, blur_ksize=9, use_subject_tracking=True,
                use_floating_window=True, preserve_original_aspect=False, zero_parallax_strength=0.01)
    # I. 4:3 source against the 16:9 target: centre crop of the height (1244-1248)
    g = run_loop(r3d, torch, cv2, 320, 240, 3, "smooth", base)
    np.savez_compressed(os.path.join(OUT, "loop_crop43_320x240.npz"), **g, **meta)
    # J. CinemaScope 2.39:1 target on a 16:9 source: crop + 430x180 warp + 215x180 eyes
    g = run_loop(r3d, torch, cv2, 320, 180, 3, "smooth", dict(base, aspect_name="CinemaScope (2.39:1)"))
    np.savez_compressed(os.path.join(OUT, "loop_scope239_320x180.npz"), **g, **meta)
    # K. preserve_original_aspect with an odd width: 321 -> 160 per eye = fractional INTER_AREA (x2.00625)
    g = run_loop(r3d, torch, cv2, 321, 180, 3, "smooth", dict(base, preserve_original_aspect=True))
    np.savez_compressed(os.path.join(OUT, "loop_halfsbs_odd_321x180.npz"), **g, **meta)
    # L. the remaining loop-level controls: IPD factor, fixed convergence, edge masking off, sharpness factor 0 (still a
    #    5/-1 kernel), and the parallax/pop controls the loop accepts but does not forward to pixel_shift_cuda
    g = run_loop(r3d, torch, cv2, 320, 180, 4, "smooth",
                 dict(base, sharpness_factor=0.0, ipd_factor=0.8, convergence_strength=0.3,
                      enable_dynamic_convergence=False, enable_edge_masking=False, parallax_balance=0.6,
                      depth_pop_gamma=0.7, fg_pop_multiplier=1.4))
    np.savez_compressed(os.path.join(OUT, "loop_controls_320x180.npz"), **g, **meta)
    # M. DOF on the Half-SBS path: the normalised depth (160x90) is upsampled to the eye size for apply_dof_cuda
    g = run_loop(r3d, torch, cv2, 320, 180, 3, "smooth", dict(base, dof_strength=1.5))
    np.savez_compressed(os.path.join(OUT, "loop_dof_halfsbs_320x180.npz"), **g, **meta)
    # N. pixel_shift_cuda with every shaping / balance control off its default (the preview path passes them)
    g = run_pixel_shift(r3d, torch, 256, 144, 256, 144, 2, "smooth",
                        blur_ksize=5, feather_strength=20.0, convergence_strength=0.3, enable_dynamic_convergence=False,
                        depth_pop_gamma=0.7, depth_pop_mid=0.4, depth_stretch_lo=0.1, depth_stretch_hi=0.9,
                        fg_pop_multiplier=1.5, bg_push_multiplier=0.9, subject_lock_strength=0.5,
                        parallax_balance=0.6, max_pixel_shift_percent=0.03, zero_parallax_strength=0.02)
    np.savez_compressed(os.path.join(OUT, "ps_controls_256x144.npz"), **g, **meta)
    print("ps_controls_256x144.npz", os.path.getsize(os.path.join(OUT, "ps_controls_256x144.npz")))
    for f in ("loop_crop43_320x240.npz", "loop_scope239_320x180.npz", "loop_halfsbs_odd_321x180.npz",
              "loop_controls_320x180.npz", "loop_dof_halfsbs_320x180.npz"):
        z = np.load(os.path.join(OUT, f))
        print(f, os.path.getsize(os.path.join(OUT, f)), {k: z[k].shape for k in z.files if k.startswith("final")})


def _sparse(f, step):
    import hashlib
    return f[::step, ::step].copy(), np.frombuffer(hashlib.sha256(f.tobytes()).digest(), dtype=np.uint8)


def gen_natural():
    """Q. the "natural" synthetic set (visiondepth3d_b200/synth.py: band-limited fields + texture, values off the
    k/255 truncation grid) through pixel_shift_cuda and the full loop with sharpening on, plus the two BASELINE sizes
    (1080p Half-SBS, 4K Full-SBS) stored as every 7th / 16th row and column + sha256 of the full frame
    (`python tools/gen_golden.py natural`)."""
    mods = refshim.load_reference(("render_3d",))
    r3d = mods["render_3d"]
    import cv2
    import torch
    import torchvision
    torch.set_num_threads(os.cpu_count())
    meta = dict(torch=torch.__version__, torchvision=torchvision.__version__, cv2=cv2.__version__,
                numpy=np.__version__)
    base = dict(output_width=320, output_height=180, sharpness_factor=0.2, output_format="Half-SBS",
                dof_strength=0.0, feather_strength=10.0, blur_ksize=9, use_subject_tracking=True,
                use_floating_window=True, preserve_original_aspect=False, zero_parallax_strength=0.01)
    g = run_pixel_shift(r3d, torch, 320, 180, 320, 180, 3, "natural",
                        blur_ksize=9, feather_strength=10.0, zero_parallax_strength=0.01)
    np.savez_compressed(os.path.join(OUT, "ps_natural_320x180.npz"), **every_row(g, 4), **meta)
    g = run_loop(r3d, torch, cv2, 320, 180, 5, "natural", base)
    np.savez_compressed(os.path.join(OUT, "loop_natural_halfsbs_320x180.npz"), **g, **meta)
    g = run_loop(r3d, torch, cv2, 320, 180, 4, "natural", dict(base, output_format="Full-SBS", preserve_original_aspect=True))
    np.savez_compressed(os.path.join(OUT, "loop_natural_fullsbs_320x180.npz"), **g, **meta)
    # BASELINE sizes
    g = run_loop(r3d, torch, cv2, 1920, 1080, 3, "natural", dict(base, output_width=1920, output_height=1080))
    out = {}
    for k, f in g.items():
        assert f.shape == (1080, 1920, 3), f.shape
        out[k + "_s7"], out[k + "_sha256"] = _sparse(f, 7)
    np.savez_compressed(os.path.join(OUT, "loop_natural_1080p_halfsbs.npz"), **out, **meta)
    g = run_loop(r3d, torch, cv2, 3840, 2160, 2, "natural",
                 dict(base, output_width=3840, output_height=2160, output_format="Full-SBS", preserve_original_aspect=True))
    out = {}
    for k, f in g.items():
        assert f.shape == (2160, 7680, 3), f.shape
        out[k + "_s16"], out[k + "_sha256"] = _sparse(f, 16)
    np.savez_compressed(os.path.join(OUT, "loop_natural_4k_fullsbs.npz"), **out, **meta)
    for f in ("ps_natural_320x180.npz", "loop_natural_halfsbs_320x180.npz", "loop_natural_fullsbs_320x180.npz",
              "loop_natural_1080p_halfsbs.npz", "loop_natural_4k_fullsbs.npz"):
        print(f, os.path.getsize(os.path.join(OUT, f)))


def gen_depth_gray():
    """O. convert_depth_to_grayscale (core/render_depth.py:585-611) on the input kinds it accepts
    (`python tools/gen_golden.py depthgray`): tensor / ndarray, 2-D, [C,H,W], [H,W,C], flat and NaN frames."""
    # core/render_depth.py drags in diffusers / DepthCrafter at import; run just this (unmodified) function by
    # compiling its definition out of the reference file at generation time -- nothing is copied into the repo
    import ast
    import types
    import torch
    from PIL import Image
    path = os.path.join(refshim.REF_ROOT, "core", "render_depth.py")
    tree = ast.parse(open(path).read(), filename=path)
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "convert_depth_to_grayscale"]
    ns = {"np": np, "torch": torch, "Image": Image}
    exec(compile(ast.Module(body=fn, type_ignores=[]), path, "exec"), ns)
    rd = types.SimpleNamespace(convert_depth_to_grayscale=ns["convert_depth_to_grayscale"])
    rng = np.random.default_rng(77)
    base = (rng.standard_normal((24, 32)) * 3.0 + 5.0).astype(np.float32)
    inputs = {
        "hw": base,
        "chw1": base[None],
        "chw3": np.stack([base, base * 0.5, base + 1.0]).astype(np.float32),
        "hwc1": base[..., None],
        "hwc3": np.stack([base, base * 0.5, base + 1.0], axis=-1).astype(np.float32),
        "flat": np.full((24, 32), 2.5, dtype=np.float32),
        "nan": np.where(rng.random((24, 32)) < 0.05, np.nan, base).astype(np.float32),
        "f64": base.astype(np.float64) * 1e-3,
        "neg": -base,
    }
    out = {}
    for k, v in inputs.items():
        out["in_" + k] = v
        out["np_" + k] = rd.convert_depth_to_grayscale(v.copy())
        out["pt_" + k] = rd.convert_depth_to_grayscale(torch.from_numpy(v.copy()))
    p = os.path.join(OUT, "depth_gray.npz")
    np.savez_compressed(p, **out)
    print(p, os.path.getsize(p))


def gen_signatures():
    """P. the call surface of the boundary (SURVEY 8(b)): parameter names, order and defaults of the reference's
    hot-path functions (`python tools/gen_golden.py signatures`) -> tests/golden/signatures.json."""
    import inspect
    import json
    mods = refshim.load_reference(("render_3d",))
    r3d = mods["render_3d"]
    names = ["pixel_shift_cuda", "render_sbs_3d", "format_3d_output", "generate_anaglyph_3d", "apply_sharpening",
             "pad_to_aspect_ratio", "frame_to_tensor", "depth_to_tensor", "tensor_to_frame", "heal_missing_pixels"]
    out = {}
    for n in names:
        sig = inspect.signature(getattr(r3d, n))
        out[n] = [[p.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
                  for p in sig.parameters.values()]
    out["aspect_ratios"] = {k: float(v) for k, v in r3d.aspect_ratios.items()}
    p = os.path.join(OUT, "signatures.json")
    json.dump(out, open(p, "w"), indent=1, sort_keys=True)
    print(p, os.path.getsize(p))


def gen_autocrop():
    """R. auto_crop_black_bars on the letterbox set (visiondepth3d_b200/synth.py), `python tools/gen_golden.py autocrop`.
    The reference's detect_black_bars is wrapped so that each fixture also records every (top, bottom) it returned, the
    probe frame's first (`crops` [n, 2]).  Final frames keep every `rows`-th row to stay under 1 MB."""
    mods = refshim.load_reference(("render_3d",))
    r3d = mods["render_3d"]
    import cv2
    import torch
    import torchvision
    torch.set_num_threads(os.cpu_count())
    meta = dict(torch=torch.__version__, torchvision=torchvision.__version__, cv2=cv2.__version__,
                numpy=np.__version__)
    base = dict(output_width=320, output_height=180, sharpness_factor=0.2, output_format="Half-SBS",
                dof_strength=0.0, feather_strength=10.0, blur_ksize=9, use_subject_tracking=True,
                use_floating_window=True, preserve_original_aspect=False, zero_parallax_strength=0.01,
                auto_crop_black_bars=True)
    real = r3d.detect_black_bars
    cases = (
        # Half-SBS: the fused k_render path; all eight frames of the schedule (the first is the probe)
        ("loop_autocrop_halfsbs_320x180.npz", 8, base, 1),
        # Full-SBS, preserve_original_aspect, original_video_* None: the output size comes from the cropped probe frame
        ("loop_autocrop_fullsbs_320x180.npz", 6, dict(base, output_format="Full-SBS", preserve_original_aspect=True), 2),
        # DOF on the Half-SBS path: the non-fused post chain
        ("loop_autocrop_dof_halfsbs_320x180.npz", 6, dict(base, dof_strength=1.5), 2),
    )
    for name, n, rp, step in cases:
        crops = []

        def wrapped(frame_tensor, threshold=10):
            tb = real(frame_tensor, threshold)
            crops.append(tb)
            return tb

        r3d.detect_black_bars = wrapped
        try:
            g = run_loop(r3d, torch, cv2, 320, 180, n, "letterbox", rp)
        finally:
            r3d.detect_black_bars = real
        assert len(crops) == n and len(g) == n - 1, (len(crops), len(g))
        out = {k: v[::step] for k, v in g.items()}
        p = os.path.join(OUT, name)
        np.savez_compressed(p, **out, crops=np.array(crops, dtype=np.int32), rows=np.int32(step), **meta)
        print(name, os.path.getsize(p), crops, {k: v.shape for k, v in g.items()})


def gen_letterbox():
    """S. the depth-video letterbox tracker: the unmodified process_video2 with ignore_letterbox_bars=True on the
    letterbox_track sets (visiondepth3d_b200/synth.py), `python tools/gen_golden.py letterbox`.  An in-memory capture
    (frame count, fps 2, size, POS_FRAMES seeks) feeds it, a recording writer collects the u8 frames it writes, and
    `pipe` is a deterministic stub (pipe_type "hf", tensor output: depth = 0.5 * green + row) that the tests
    reproduce.  LetterboxTracker.bootstrap / update and detect_letterbox_multiframe_confidence are wrapped to record
    the bootstrap (bars, confidence, locks) and every per-frame (top, bottom).  Batches of 4 frames: neither clip
    length is a multiple of 4."""
    import json
    import tempfile
    import types
    import cv2
    import torch
    from PIL import Image
    for n in ("diffusers.configuration_utils", "core.unet", "core.depthcrafter_adapter"):
        refshim._stub(n)
    rd = refshim.load_reference(("render_depth",))["render_depth"]
    from visiondepth3d_b200 import synth
    meta = dict(torch=torch.__version__, cv2=cv2.__version__, numpy=np.__version__)

    def stub_pipe(images, inference_size=None):
        out = []
        for img in images:
            g = np.asarray(img.convert("RGB"), dtype=np.float32)[..., 1]
            out.append({"predicted_depth": torch.from_numpy(0.5 * g + np.arange(g.shape[0], dtype=np.float32)[:, None])})
        return out

    for kind, sched in (("letterbox_track", synth._TRACK), ("letterbox_track_nobars", synth._TRACK_NOBARS)):
        n_frames = len(sched)
        frames = [synth_frame(i, 320, 180, kind)[0] for i in range(n_frames)]

        class Cap:
            def __init__(self, *a):
                self.pos = 0

            def isOpened(self):
                return True

            def get(self, prop):
                return float({cv2.CAP_PROP_FRAME_COUNT: n_frames, cv2.CAP_PROP_FPS: 2.0, cv2.CAP_PROP_FRAME_WIDTH: 320,
                              cv2.CAP_PROP_FRAME_HEIGHT: 180, cv2.CAP_PROP_POS_FRAMES: self.pos}.get(prop, 0.0))

            def set(self, prop, v):
                if prop == cv2.CAP_PROP_POS_FRAMES:
                    self.pos = int(v)
                return True

            def read(self):
                if self.pos >= n_frames:
                    return False, None
                self.pos += 1
                return True, frames[self.pos - 1].copy()

            def release(self):
                pass

        written = []

        class Writer:
            def __init__(self, *a, **k):
                pass

            def isOpened(self):
                return True

            def write(self, f):
                written.append(f[..., 0].copy())

            def release(self):
                pass

        rec = {"boot": None, "conf": None, "bars": []}
        real_boot, real_upd = rd.LetterboxTracker.bootstrap, rd.LetterboxTracker.update
        real_conf = rd.detect_letterbox_multiframe_confidence

        def conf(*a, **k):
            r = real_conf(*a, **k)
            rec["conf"] = r[1]
            return r

        def boot(self, cap):
            r = real_boot(self, cap)
            rec["boot"] = (r[0], r[1], bool(r[2][0]), bool(r[2][1]))
            return r

        def upd(self, frame, idx):
            r = real_upd(self, frame, idx)
            rec["bars"].append(r)
            return r

        real_cap, real_wr = cv2.VideoCapture, cv2.VideoWriter
        rd.detect_letterbox_multiframe_confidence = conf
        rd.LetterboxTracker.bootstrap, rd.LetterboxTracker.update = boot, upd
        cv2.VideoCapture, cv2.VideoWriter = Cap, Writer
        rd.pipe, rd.pipe_type = stub_pipe, "hf"
        status = types.SimpleNamespace(config=lambda **k: None, update_idletasks=lambda: None)
        try:
            with tempfile.TemporaryDirectory() as td:
                rd.process_video2(os.path.join(td, kind + ".mkv"), n_frames, 0, 4, Var(td), Var("Original"), status,
                                  {}, threading.Event(), Var(False), ignore_letterbox_bars=True)
                side = json.load(open(os.path.join(td, kind + "_depth.letterbox.json")))
        finally:
            cv2.VideoCapture, cv2.VideoWriter = real_cap, real_wr
            rd.detect_letterbox_multiframe_confidence = real_conf
            rd.LetterboxTracker.bootstrap, rd.LetterboxTracker.update = real_boot, real_upd
        assert len(written) == n_frames and len(rec["bars"]) == n_frames, (len(written), len(rec["bars"]))
        p = os.path.join(OUT, kind.replace("letterbox_track", "letterbox") + "_320x180.npz")
        np.savez_compressed(p, kind=kind, batch_size=np.int32(4), fps=np.float64(2.0),
                            boot_bars=np.array(rec["boot"][:2], np.int32), boot_locks=np.array(rec["boot"][2:], bool),
                            boot_conf=np.float64(rec["conf"]), bars=np.array(rec["bars"], np.int32),
                            sidecar=json.dumps(side, sort_keys=True), written=np.stack(written), **meta)
        print(p, os.path.getsize(p), rec["boot"], rec["conf"], side)


def gen_merged():
    """The unmodified start_merged_pipeline (core/merged_pipeline.py:287-386) on the synth frames folder,
    `python tools/gen_golden.py merged`.  Stand-ins: an onnxruntime module whose InferenceSession raises for the RIFE
    file (the reference then runs without RIFE) and runs oracle/sr.py's srvgg_forward for the ESRGAN file;
    start_ffmpeg_writer replaced by a recorder of (width, height, fps, codec) and every frame written;
    natural_sort wrapped to record the file order."""
    import importlib.machinery
    import json
    import tempfile
    import types
    import cv2
    import torch
    from oracle import sr as S
    from tests.merged_oracle import MERGED_BASE, MERGED_CASES, MERGED_SR
    from visiondepth3d_b200 import synth
    sd = S.srvgg_state_dict(**MERGED_SR)

    class Session:
        def __init__(self, path, sess_options=None, providers=None):
            if "RIFE" in os.path.basename(path):
                raise FileNotFoundError(path)

        def get_inputs(self):
            return [types.SimpleNamespace(name="input")]

        def run(self, _outputs, feeds):
            with torch.no_grad():
                return [S.srvgg_forward(sd, torch.from_numpy(feeds["input"])).numpy()]

    ort = types.ModuleType("onnxruntime")
    ort.__spec__ = importlib.machinery.ModuleSpec("onnxruntime", None)
    ort.SessionOptions = type("SessionOptions", (), {})
    ort.GraphOptimizationLevel = types.SimpleNamespace(ORT_ENABLE_ALL=99)
    ort.get_available_providers = lambda: ["CPUExecutionProvider"]
    ort.InferenceSession = Session
    sys.modules["onnxruntime"] = ort
    mp = refshim.load_reference(("merged_pipeline",))["merged_pipeline"]
    meta = dict(torch=torch.__version__, cv2=cv2.__version__, numpy=np.__version__)
    real_sort = mp.natural_sort
    for name, case in MERGED_CASES.items():
        rec = {"frames": []}

        class Proc:
            class stdin:  # noqa: N801
                write = staticmethod(lambda b: rec["frames"].append(bytes(b)))
                close = staticmethod(lambda: None)

            def wait(self):
                return 0

        def writer(path, w, h, fps, codec):
            rec["args"] = (w, h, fps, codec)
            return Proc()

        def sort(files):
            out = real_sort(files)
            rec["files"] = [os.path.basename(f) for f in out]
            return out

        mp.start_ffmpeg_writer, mp.natural_sort = writer, sort
        with tempfile.TemporaryDirectory() as td:
            folder = synth.merged_frames_folder(os.path.join(td, "frames"))
            model = os.path.join(td, "weights", "RealESR_Gx4_fp16.onnx")
            if case.get("model") != "missing":
                os.makedirs(os.path.dirname(model))
                open(model, "wb").close()
            settings = dict(MERGED_BASE, frames_folder=folder, output_file=os.path.join(td, "out.mp4"), model_path=model)
            settings.update({k: v for k, v in case.items() if k != "model"})
            mp.start_merged_pipeline(settings, None, None)
        w, h = rec["args"][:2]
        frames = np.stack([np.frombuffer(b, np.uint8).reshape((h, w, 3) if len(b) == w * h * 3 else (72, 128, 3))
                           for b in rec["frames"]])
        p = os.path.join(OUT, name)
        np.savez_compressed(p, frames=frames, writer_size=np.array(rec["args"][:2], np.int32),
                            writer_fps=np.float64(rec["args"][2]), codec=rec["args"][3], files=json.dumps(rec["files"]),
                            settings=json.dumps({k: v for k, v in case.items()}), **meta)
        print(p, os.path.getsize(p), frames.shape, rec["args"], rec["files"])
    mp.natural_sort = real_sort

TILED_CASES = [  # name, frame (w, h), inference_size, tile, pad, invert, prediction
    ("256x144_t96p16", (256, 144), None, 96, 16, False, "ramp"),
    ("odd_203x117_t96p16_inv", (203, 117), None, 96, 16, True, "ramp"),
    ("small_80x60_t96p16", (80, 60), None, 96, 16, False, "ramp"),
    ("bigpad_100x64_t64p24", (100, 64), None, 64, 24, False, "ramp"),
    ("shrink_256x144_to_200x112", (256, 144), (200, 112), 96, 16, False, "ramp"),
    ("grow_160x90_to_208x117", (160, 90), (208, 117), 96, 16, True, "ramp"),
    ("flat_128x96_t64p16", (128, 96), None, 64, 16, False, "flat"),
    ("outliers_200x120_t96p16", (200, 120), None, 96, 16, False, "outliers"),
]


def tiled_prediction(crop_rgb, kind):
    """The stand-in depth of a tile crop (RGB u8 [h, w, 3]): integer-valued float32 arithmetic, exact in any order.
    ramp: R + 2G + B + x + 2y (tile seams stay visible); flat: 7; outliers: 5 everywhere but 3 (the first of every
    fifth row's first two columns), so p1 == p99 while the range is not flat."""
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


def gen_tiled():
    """T. tiled depth: the unmodified infer_depth_tile, _run_pipe_or_tile and _normalize_to_u8 with the module's
    USE_TILED_DEPTH / TILE_* set as attributes, `python tools/gen_golden.py tiled`.  `pipe` is a recording stand-in
    whose prediction is tiled_prediction of the crop; the fixtures hold the crops it was handed, the blended float32
    depth, its percentiles, the written u8 frame and the printed lines."""
    import contextlib
    import io
    import cv2
    import torch
    for n in ("diffusers.configuration_utils", "core.unet", "core.depthcrafter_adapter"):
        refshim._stub(n)
    rd = refshim.load_reference(("render_depth",))["render_depth"]
    from PIL import Image
    meta = dict(torch=torch.__version__, cv2=cv2.__version__, numpy=np.__version__)
    for name, (w, h), inf, tile, pad, invert, kind in TILED_CASES:
        rng = np.random.default_rng(len(name) * 7919 + w * 31 + h)
        rgb = np.clip(rng.normal(128, 60, (h, w, 3)), 0, 255).astype(np.uint8)
        crops, sizes = [], []

        def stub_pipe(images, inference_size=None):
            out = []
            for img in images:
                a = np.asarray(img.convert("RGB"))
                assert inference_size == (a.shape[1], a.shape[0])
                crops.append(a.copy())
                sizes.append(inference_size)
                out.append({"predicted_depth": torch.from_numpy(tiled_prediction(a, kind))})
            return out

        rd.pipe, rd.pipe_type = stub_pipe, "hf"
        rd.USE_TILED_DEPTH, rd.TILE_SIZE, rd.TILE_PAD, rd.TILE_DEBUG = True, tile, pad, True
        # the tile defaults are bound at import: pass them as _run_pipe_or_tile does, through the attributes above
        rd.infer_depth_tile.__defaults__ = (tile, pad)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            res = rd._run_pipe_or_tile([Image.fromarray(rgb)], inf)
        depth = res[0]["predicted_depth"]
        assert depth.dtype == np.float32
        u8 = rd._normalize_to_u8(depth, (w, h), invert=invert)
        dn = np.nan_to_num(depth, nan=0.0, posinf=0.0, neginf=0.0)
        pct = np.array([np.percentile(dn, 1.0), np.percentile(dn, 99.0)], np.float32)
        p = os.path.join(OUT, f"tiled_{name}.npz")
        np.savez_compressed(p, rgb=rgb, size=np.array([w, h], np.int32),
                            inference_size=np.array(inf if inf else (0, 0), np.int32), tile=np.int32(tile),
                            pad=np.int32(pad), invert=np.bool_(invert), kind=kind,
                            crop_sizes=np.array(sizes, np.int32), crops=np.concatenate([c.ravel() for c in crops]),
                            depth=depth, pct=pct, u8=u8, log=buf.getvalue(), **meta)
        print(p, os.path.getsize(p), len(crops), "tiles")
    gen_tiled_video(rd, torch, cv2, meta)


def gen_tiled_video(rd, torch, cv2, meta):
    """The tiled branch of the unmodified process_video2 (USE_TILED_DEPTH, tile 96, pad 16) on the first 13 frames of
    the letterbox_track clip at 2 fps, in batches of 4, with and without ignore_letterbox_bars: an in-memory capture
    and a recording writer as in gen_letterbox, the stand-in pipe's "ramp" prediction.  Records every per-frame
    (top, bottom), every written frame and the printed [tile] lines."""
    import contextlib
    import io
    import json
    import tempfile
    import types
    n_frames = 13
    frames = [synth_frame(i, 320, 180, "letterbox_track")[0] for i in range(n_frames)]

    def stub_pipe(images, inference_size=None):
        return [{"predicted_depth": torch.from_numpy(tiled_prediction(np.asarray(img.convert("RGB")), "ramp"))}
                for img in images]

    for ignore in (True, False):
        class Cap:
            def __init__(self, *a):
                self.pos = 0

            def isOpened(self):
                return True

            def get(self, prop):
                return float({cv2.CAP_PROP_FRAME_COUNT: n_frames, cv2.CAP_PROP_FPS: 2.0, cv2.CAP_PROP_FRAME_WIDTH: 320,
                              cv2.CAP_PROP_FRAME_HEIGHT: 180, cv2.CAP_PROP_POS_FRAMES: self.pos}.get(prop, 0.0))

            def set(self, prop, v):
                if prop == cv2.CAP_PROP_POS_FRAMES:
                    self.pos = int(v)
                return True

            def read(self):
                if self.pos >= n_frames:
                    return False, None
                self.pos += 1
                return True, frames[self.pos - 1].copy()

            def release(self):
                pass

        written, bars = [], []

        class Writer:
            def __init__(self, *a, **k):
                pass

            def isOpened(self):
                return True

            def write(self, f):
                written.append(f[..., 0].copy())

            def release(self):
                pass

        real_upd = rd.LetterboxTracker.update

        def upd(self, frame, idx):
            r = real_upd(self, frame, idx)
            bars.append(r)
            return r

        real_cap, real_wr = cv2.VideoCapture, cv2.VideoWriter
        rd.LetterboxTracker.update = upd
        cv2.VideoCapture, cv2.VideoWriter = Cap, Writer
        rd.pipe, rd.pipe_type = stub_pipe, "hf"
        rd.USE_TILED_DEPTH, rd.TILE_SIZE, rd.TILE_PAD, rd.TILE_DEBUG = True, 96, 16, False
        rd.infer_depth_tile.__defaults__ = (96, 16)
        status = types.SimpleNamespace(config=lambda **k: None, update_idletasks=lambda: None)
        buf = io.StringIO()
        try:
            with tempfile.TemporaryDirectory() as td, contextlib.redirect_stdout(buf):
                rd.process_video2(os.path.join(td, "clip.mkv"), n_frames, 0, 4, Var(td), Var("Original"), status,
                                  {}, threading.Event(), Var(False), ignore_letterbox_bars=ignore)
                side = json.load(open(os.path.join(td, "clip_depth.letterbox.json")))
        finally:
            cv2.VideoCapture, cv2.VideoWriter = real_cap, real_wr
            rd.LetterboxTracker.update = real_upd
        assert len(written) == n_frames, len(written)
        if not ignore:
            bars = [(0, 0)] * n_frames
        ranges = [ln for ln in buf.getvalue().splitlines() if ln.startswith("[tile] range")]
        p = os.path.join(OUT, "tiled_video_%s_320x180.npz" % ("bars" if ignore else "nobars"))
        np.savez_compressed(p, batch_size=np.int32(4), tile=np.int32(96), pad=np.int32(16),
                            ignore_letterbox_bars=np.bool_(ignore), bars=np.array(bars, np.int32),
                            sidecar=json.dumps(side, sort_keys=True), written=np.stack(written),
                            ranges="\n".join(ranges), **meta)
        print(p, os.path.getsize(p), side, sorted(set(map(tuple, bars))))


IMAGE_VARIANTS = (("original", "Original", False), ("384x384", "384x384", False), ("invert", "Original", True))


def image_depth_weights():
    """The random-init Depth-Anything-V2-Small of the depth tests (seed 0; the head's last 1x1 conv made non-negative
    so that its output does not cancel, tests/test_depth_gpu.py _model)."""
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200.depth_weights import hf_config
    torch.manual_seed(0)
    sd = DepthAnythingForDepthEstimation(hf_config("vits")).eval().state_dict()
    sd["head.conv3.weight"] = sd["head.conv3.weight"].abs() + 0.02
    sd["head.conv3.bias"] = torch.zeros_like(sd["head.conv3.bias"])
    return sd


def gen_images():
    """I. still images: the unmodified process_images_in_folder and process_image on the photo folder of
    visiondepth3d_b200.synth.image_folder, for Original, "384x384" and invert (`python tools/gen_golden.py images`).
    `pipe` is the reference's HF branch: a transformers depth-estimation pipeline over image_depth_weights() and the
    DA-V2 image processor, behind the pipe protocol (PIL bicubic to the inference size first).  Records the written
    file names and their u8 arrays and modes."""
    import contextlib
    import io
    import tempfile
    import zlib
    import torch
    from PIL import Image
    from transformers import DepthAnythingForDepthEstimation, pipeline
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    from visiondepth3d_b200.depth_weights import hf_config
    from visiondepth3d_b200.synth import IMAGE_FOLDER, image_folder
    for n in ("diffusers.configuration_utils", "core.unet", "core.depthcrafter_adapter"):
        refshim._stub(n)
    rd = refshim.load_reference(("render_depth",))["render_depth"]
    model = DepthAnythingForDepthEstimation(hf_config("vits")).eval()
    model.load_state_dict(image_depth_weights())
    proc = DPTImageProcessor(do_resize=True, size={"height": 518, "width": 518}, keep_aspect_ratio=True,
                             ensure_multiple_of=14, resample=3, do_rescale=True, do_normalize=True,
                             image_mean=[0.485, 0.456, 0.406], image_std=[0.229, 0.224, 0.225], do_pad=False)
    raw = pipeline("depth-estimation", model=model, image_processor=proc, device=-1)

    def hf_pipe(images, inference_size=None):  # the pipe protocol of the reference's HF branch
        if inference_size:
            images = [img.resize(inference_size, Image.BICUBIC) for img in images]
        return raw(images) if isinstance(images, list) else [raw(images)]

    class Widget:
        def __init__(self):
            self.kw = {}

        def after(self, _ms, fn):
            fn()

        def config(self, **kw):
            self.kw.update(kw)

        def __getitem__(self, k):
            return self.kw.get(k)

        def start(self, *_a):
            pass

        def stop(self):
            pass

    rd.pipe, rd.pipe_type, rd.USE_TILED_DEPTH = hf_pipe, "hf", False
    import json
    p = os.path.join(OUT, "images_resolutions.json")  # the choices parse_inference_resolution must read as it does
    json.dump({k: (list(v) if v else None) for k, v in rd.INFERENCE_RESOLUTIONS.items()}, open(p, "w"), indent=1)
    meta = dict(torch=torch.__version__, numpy=np.__version__, pillow=Image.__version__)
    with tempfile.TemporaryDirectory() as tmp:
        src = image_folder(os.path.join(tmp, "in"))
        inputs = {name: np.asarray(Image.open(os.path.join(src, name)).convert("RGB")) for name, *_ in IMAGE_FOLDER}
        crc = np.array([zlib.crc32(inputs[name].tobytes()) for name, *_ in IMAGE_FOLDER], np.uint32)
        for tag, res, invert in IMAGE_VARIANTS:
            out = {}
            for mode in ("folder", "single"):
                dst = os.path.join(tmp, f"{tag}_{mode}")
                log = io.StringIO()
                with torch.no_grad(), contextlib.redirect_stdout(log):
                    if mode == "folder":
                        rd.process_images_in_folder(src, Var("4"), Var(dst), Var(res), Widget(), Widget(), Widget(),
                                                    Var(invert))
                    else:
                        for name, *_ in IMAGE_FOLDER:
                            rd.process_image(os.path.join(src, name), Var("Default"), Var(invert), Var(dst), Var(res),
                                             Widget(), Widget(), Widget(), Widget())
                names = sorted(os.listdir(dst))
                out[f"{mode}_names"] = np.array(names)
                for n in names:
                    im = Image.open(os.path.join(dst, n))
                    out[f"{mode}_mode_{n}"] = im.mode
                    out[f"{mode}_{n}"] = np.asarray(im)
            # every 4th row and column of the folder outputs (keeps the fixture small); process_image wrote the same
            for n in out["folder_names"]:
                full = out.pop(f"folder_{n}")
                assert np.array_equal(out.pop(f"single_{n}"), full) and out.pop(f"single_mode_{n}") == "L"
                out[f"shape_{n}"] = np.array(full.shape, np.int32)
                out[f"u8_{n}"] = full[::4, ::4]
            p = os.path.join(OUT, f"images_{tag}.npz")
            np.savez_compressed(p, resolution=res, invert=np.bool_(invert), input_crc=crc, **out, **meta)
            print(p, os.path.getsize(p), list(out["folder_names"]))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "signatures":
        gen_signatures()
    elif len(sys.argv) > 1 and sys.argv[1] == "depthgray":
        gen_depth_gray()
    elif len(sys.argv) > 1 and sys.argv[1] == "extra":
        gen_extra()
    elif len(sys.argv) > 1 and sys.argv[1] == "vr":
        gen_vr()
    elif len(sys.argv) > 1 and sys.argv[1] == "natural":
        gen_natural()
    elif len(sys.argv) > 1 and sys.argv[1] == "autocrop":
        gen_autocrop()
    elif len(sys.argv) > 1 and sys.argv[1] == "letterbox":
        gen_letterbox()
    elif len(sys.argv) > 1 and sys.argv[1] == "merged":
        gen_merged()
    elif len(sys.argv) > 1 and sys.argv[1] == "tiled":
        gen_tiled()
    elif len(sys.argv) > 1 and sys.argv[1] == "images":
        gen_images()
    else:
        main()
