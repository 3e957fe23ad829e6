"""The image-folder driver of core/merged_pipeline.py (start_merged_pipeline, 287-386) restated in numpy / cv2 on top
of oracle/sr.py: which files are read and in what order, what each frame goes through, and what the writer is opened
with.  RIFE interpolates nothing (no RIFE network), so the writer receives exactly one frame per readable source frame.
TEST INFRASTRUCTURE ONLY."""
import os
import re


def frame_number(name):
    m = re.search(r"\d+", os.path.basename(name))
    return int(m.group(0)) if m else float("inf")


def frame_files(folder):
    """.jpg / .jpeg / .png after lower(), stably sorted on the first number of the basename (none: last)."""
    names = [f for f in os.listdir(folder) if f.lower().endswith((".jpg", ".jpeg", ".png"))]
    return sorted((os.path.join(folder, f) for f in names), key=frame_number)


def writer_args(settings):
    """(width, height, fps, codec) of the writer: fps x fps_multiplier whenever enable_rife."""
    fps = settings["fps"] * settings["fps_multiplier"] if settings["enable_rife"] else settings["fps"]
    return settings["width"], settings["height"], fps, settings["codec"]


def loader_resize(img, target):
    """The loader's resize when upscaling is off: INTER_AREA iff the source is wider than the target."""
    import cv2
    return cv2.resize(img, target, interpolation=cv2.INTER_AREA if img.shape[1] > target[0] else cv2.INTER_CUBIC)


def merged_frames(settings, state_dict=None):
    """Frames handed to the writer.  state_dict: the SRVGGNetCompact model (torch tensors), None when the model file is
    missing (frames then stay at source size)."""
    import cv2
    from oracle import sr as S
    target = (settings["width"], settings["height"])
    out = []
    for f in frame_files(settings["frames_folder"]):
        img = cv2.imread(f, cv2.IMREAD_COLOR)
        if img is None:
            continue
        if not settings["enable_upscale"]:
            out.append(loader_resize(img, target))
        elif state_dict is None:
            out.append(img)
        else:  # run_esrgan with the default model name (scale 4) and target_size = (width, height)
            out.append(S.run_esrgan(state_dict, img, settings.get("blend_mode", "OFF"),
                                    settings.get("input_res_pct", 100), target))
    return out


def blend_alpha(mode):
    """blend_images' alpha: None for exactly "OFF"; LOW / MEDIUM / HIGH after upper(); 1.0 for anything else."""
    if mode == "OFF":
        return None
    return {"LOW": 0.85, "MEDIUM": 0.5, "HIGH": 0.25}.get(mode.upper(), 1.0)


# the fixture cases (tools/gen_golden.py merged -> tests/golden/<name>): the settings of each case on top of
# MERGED_BASE; the frames folder is synth.merged_frames_folder (128x72 frames); the ESRGAN model is
# oracle.sr.srvgg_state_dict(**MERGED_SR)
MERGED_SR = dict(num_conv=4, seed=7)
MERGED_BASE = dict(codec="libx264", fps=24, fps_multiplier=2, input_res_pct=100, blend_mode="OFF")
MERGED_CASES = {
    "merged_area_rife.npz": dict(enable_upscale=False, enable_rife=True, width=96, height=54),
    "merged_cubic_rife.npz": dict(enable_upscale=False, enable_rife=True, width=200, height=112),
    "merged_sr_pct50_x2target.npz": dict(enable_upscale=True, enable_rife=False, width=256, height=144,
                                         input_res_pct=50, blend_mode="OFF"),
    "merged_sr_medium.npz": dict(enable_upscale=True, enable_rife=True, width=128, height=72, blend_mode="MEDIUM"),
    "merged_sr_nomodel.npz": dict(enable_upscale=True, enable_rife=False, width=96, height=54, model="missing"),
}
