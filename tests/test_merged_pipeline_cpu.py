"""CPU: the host side of the merged_pipeline drop-in -- the reference's import list, frame listing and sorting quirks,
writer arguments, model loading, run_esrgan's parameters as vd3d_upscale_params, RIFE without a network -- against
tests/merged_oracle.py (no GPU needed)."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import merged_oracle as MO
from visiondepth3d_b200 import _lib
from visiondepth3d_b200 import merged_pipeline as MP


@pytest.fixture
def folder(tmp_path):
    import cv2
    d = tmp_path / "frames"
    d.mkdir()
    img = np.zeros((18, 32, 3), np.uint8)
    for i, name in enumerate(("frame_10.png", "frame_9.png", "frame_2.jpeg", "shot.png", "frame_1.JPG", "Frame_7.PNG",
                              "last_b.png", "frame_3.bmp")):
        ext = os.path.splitext(name)[1].lower().replace("jpeg", "jpg")
        (d / name).write_bytes(cv2.imencode(ext, img + i)[1].tobytes())
    (d / "notes.txt").write_text("x")
    (d / "frame_5.png").write_bytes(b"corrupt")
    return d


def _settings(d, tmp_path, **kw):
    s = dict(frames_folder=str(d), output_file=str(tmp_path / "o.mp4"), codec="libx264", width=64, height=36, fps=24,
             fps_multiplier=3, enable_rife=True, enable_upscale=False, blend_mode="OFF", input_res_pct=100,
             model_path=str(tmp_path / "RealESR_Gx4_fp16.onnx"))
    s.update(kw)
    return s


def test_callers_import_lists_resolve():
    """VisionDepth3D.py:55-61 and core/__init__.py:21-26 import these from core.merged_pipeline."""
    from visiondepth3d_b200.merged_pipeline import (  # noqa: F401
        start_merged_pipeline, select_video_and_generate_frames, select_output_file, select_frames_folder,
        start_ffmpeg_writer)
    assert MP.rife_session is None and MP.esrgan_session is None
    assert MP.progress_bar is None and MP.status_label is None
    assert hasattr(MP.suspend_flag, "is_set") and hasattr(MP.cancel_flag, "is_set")
    for name in ("select_video_and_generate_frames", "select_output_file", "select_frames_folder"):
        with pytest.raises(RuntimeError, match="GUI"):
            getattr(MP, name)(None)


def test_upscale_params_struct_matches_library():
    lib = _lib.load()
    assert lib.vd3d_struct_size(4) == C.sizeof(_lib.UpscaleParams) == 32


def test_frame_listing_and_natural_sort(folder, tmp_path):
    """Extension filter after lower(); the first number of the basename orders the files (frame_9 before frame_10);
    names without a number go last in listing order (stable)."""
    plan = MP._MergedPlan(_settings(folder, tmp_path))
    assert plan.prepare()
    got = [os.path.basename(f) for f in plan.files]
    assert got == [os.path.basename(f) for f in MO.frame_files(str(folder))]
    assert got[:6] == ["frame_1.JPG", "frame_2.jpeg", "frame_5.png", "Frame_7.PNG", "frame_9.png", "frame_10.png"]
    assert set(got[6:]) == {"shot.png", "last_b.png"} and "frame_3.bmp" not in got and "notes.txt" not in got
    assert MP.extract_frame_number("/a/b7/x_12_3.png") == 12 and MP.extract_frame_number("abc.png") == float("inf")
    names = ["b.png", "a.png", "c2.png"]
    assert MP.natural_sort(names) == ["c2.png", "b.png", "a.png"]


def test_empty_folder_prints_and_writes_nothing(tmp_path, capsys):
    d = tmp_path / "empty"
    d.mkdir()
    (d / "readme.txt").write_text("x")
    MP.start_merged_pipeline(_settings(d, tmp_path), None, None)
    out = capsys.readouterr().out
    assert "RIFE interpolation is not built" in out and "No frames found" in out
    assert not os.path.exists(tmp_path / "o.mp4")


def test_writer_fps_and_command_line(monkeypatch, tmp_path, folder):
    for rife, exp in ((True, 72), (False, 24)):
        plan = MP._MergedPlan(_settings(folder, tmp_path, enable_rife=rife))
        assert plan.output_fps == exp == MO.writer_args(_settings(folder, tmp_path, enable_rife=rife))[2]
    seen = {}
    import subprocess
    monkeypatch.setattr(subprocess, "Popen", lambda cmd, stdin=None: seen.setdefault("cmd", cmd))
    MP.start_ffmpeg_writer("o.mp4", 64, 36, 72, "libx264")
    assert seen["cmd"] == ["ffmpeg", "-y", "-f", "rawvideo", "-vcodec", "rawvideo", "-pix_fmt", "bgr24", "-s", "64x36",
                           "-r", "72", "-i", "-", "-c:v", "libx264", "-preset", "medium", "-crf", "18", "-pix_fmt",
                           "yuv420p", "o.mp4"]
    seen.clear()
    MP.start_ffmpeg_writer("o.mp4", 64, 36, 24.0, "H264_NVENC")
    assert seen["cmd"][14:17] ==["-c:v", "h264_nvenc", "-preset"] and seen["cmd"][-1] == "o.mp4"


def test_model_loading(tmp_path, capsys):
    import torch
    onnx = str(tmp_path / "RealESR_Gx4_fp16.onnx")
    assert MP._model_files(onnx) == [str(tmp_path / "RealESR_Gx4_fp16.pth"), str(tmp_path / "RealESR_Gx4_fp16.safetensors")]
    assert MP._model_files("m.PTH") == ["m.PTH"]
    assert MP.load_esrgan_from(onnx) is None and MP.esrgan_session is None
    assert f"❌ ESRGAN model missing: {onnx}" in capsys.readouterr().out
    sd = MP.random_srvgg_state_dict(2, seed=0)
    torch.save({"params_ema": {k: torch.from_numpy(v) for k, v in sd.items()}}, str(tmp_path / "a.pth"))
    got = MP._read_state_dict(str(tmp_path / "a.pth"))
    assert sorted(got) == sorted(sd) and all(np.array_equal(got[k], sd[k]) for k in sd)
    from safetensors.numpy import save_file
    save_file(sd, str(tmp_path / "b.safetensors"))
    assert all(np.array_equal(MP._read_state_dict(str(tmp_path / "b.safetensors"))[k], sd[k]) for k in sd)
    bad = dict(sd)
    bad["body.0.weight"] = np.zeros((32, 3, 3, 3), np.float32)  # num_feat 32: not the network vd3d serves
    torch.save({"params": {k: torch.from_numpy(v) for k, v in bad.items()}}, str(tmp_path / "c.pth"))
    with pytest.raises(ValueError, match="SRVGGNetCompact"):
        MP._read_state_dict(str(tmp_path / "c.pth"))


def test_bad_model_raises_before_any_output(tmp_path, folder):
    import torch
    torch.save({"params": {"conv_first.weight": torch.zeros(64, 3, 3, 3)}}, str(tmp_path / "RealESR_Gx4_fp16.pth"))
    with pytest.raises(ValueError):
        MP.start_merged_pipeline(_settings(folder, tmp_path, enable_upscale=True), None, None)
    assert not os.path.exists(tmp_path / "o.mp4")


def test_upscale_params_follow_blend_images_and_model_name():
    for mode in ("OFF", "LOW", "MEDIUM", "HIGH", "low", "off", "Sharp", ""):
        p = MP.upscale_params(mode)
        exp = MO.blend_alpha(mode)
        assert (p.blend_alpha < 0) if exp is None else (p.blend_alpha == exp), mode
    assert MP.upscale_params(model_name="RealESR_Gx4_fp16").scale == 4
    assert MP.upscale_params(model_name="RealESRGAN_X2plus").scale == 2
    p = MP.upscale_params("OFF", 50, target_size=(7680, 2160))
    assert (p.input_res_pct, p.target_w, p.target_h) == (50.0, 7680, 2160)
    assert (MP.upscale_params().target_w, MP.upscale_params().target_h) == (0, 0)


def test_run_rife_without_network_and_helpers():
    a = np.full((4, 6, 3), 255, np.uint8)
    b = np.zeros((4, 6, 3), np.uint8)
    assert MP.run_rife(a, b, 2) == []
    cat = MP.concatenate_images(a, b)
    assert cat.shape == (4, 6, 6) and cat.dtype == np.float32 and cat[..., :3].max() == 1.0
    t = MP.preprocess_rife(cat)
    assert t.shape == (1, 6, 4, 6) and t.dtype == np.float32


def test_update_progress_marshals_to_widgets(monkeypatch):
    calls = []

    class W:
        def after(self, ms, fn):
            calls.append(ms)
            fn()

        def configure(self, **kw):
            calls.append(kw)

    monkeypatch.setattr(MP, "progress_bar", W())
    monkeypatch.setattr(MP, "status_label", W())
    MP.update_progress(5, 10, 0.0)
    assert calls[0] == 0 and calls[1] == {"value": 50.0} and calls[3]["text"].startswith("Progress: 5/10 | FPS: ")
    monkeypatch.setattr(MP, "status_label", None)
    calls.clear()
    MP.update_progress(5, 10, 0.0)
    assert not calls


def test_prefetch_skips_unreadable_frames_silently(folder, tmp_path, capsys):
    import queue
    import threading
    plan = MP._MergedPlan(_settings(folder, tmp_path))
    assert plan.prepare()
    q = queue.Queue()
    MP._prefetch(plan.files, None, queue.Queue(), q, threading.Event())
    items = []
    while True:
        it = q.get_nowait()
        if it is None:
            break
        items.append(it[1])
    assert len(items) == len(plan.files) - 1 == 7  # frame_5.png is not an image
    assert capsys.readouterr().out == ""
    import cv2
    readable = [cv2.imread(f) for f in plan.files]
    assert all(np.array_equal(a, b) for a, b in zip(items, [r for r in readable if r is not None]))


# ---------------------------------------------------------------------------
# against the unmodified reference driver (tests/golden/merged_*.npz, tools/gen_golden.py merged)
# ---------------------------------------------------------------------------
def fixture_settings(name, tmp_path):
    """The settings a fixture was recorded with, on a freshly written copy of its frames folder."""
    from tests.merged_oracle import MERGED_BASE, MERGED_CASES
    from visiondepth3d_b200 import synth
    case = dict(MERGED_CASES[name])
    folder = synth.merged_frames_folder(str(tmp_path / "frames"))
    model = tmp_path / "weights" / "RealESR_Gx4_fp16.onnx"
    s = dict(MERGED_BASE, frames_folder=folder, output_file=str(tmp_path / "out.mp4"), model_path=str(model))
    s.update({k: v for k, v in case.items() if k != "model"})
    return s, case.get("model") != "missing"


@pytest.mark.parametrize("name", ["merged_area_rife.npz", "merged_cubic_rife.npz", "merged_sr_pct50_x2target.npz",
                                  "merged_sr_medium.npz", "merged_sr_nomodel.npz"])
def test_merged_oracle_and_dropin_host_side_match_reference(name, tmp_path, golden_dir):
    """merged_oracle reproduces every frame the reference driver wrote and its writer arguments (exact where the path
    is INTER_AREA or the source frame, <= 1 LSB / < 0.2 % where it is cv2's INTER_CUBIC); the drop-in's frame list and
    writer arguments are the reference's."""
    import json
    from oracle import sr as S
    from tests.merged_oracle import MERGED_SR
    from tests.util import u8_diff
    g = np.load(os.path.join(golden_dir, name))
    s, has_model = fixture_settings(name, tmp_path)
    files = json.loads(str(g["files"]))
    # quirks: .jpg/.jpeg/.png after lower() (the upper-case .JPG is in, .bmp / .txt are out), first number of the
    # basename (frame_9 before frame_10), no number last, the corrupt PNG listed but skipped by the loader
    assert files == ["frame_1.png", "frame_2.JPG", "frame_5.png", "frame_9.png", "frame_10.png", "frame_11.png",
                     "shot_b.png"]
    assert [os.path.basename(f) for f in MO.frame_files(s["frames_folder"])] == files
    plan = MP._MergedPlan(s)
    plan.enable_upscale = False  # the listing only: no model load on the CPU
    assert plan.prepare() and [os.path.basename(f) for f in plan.files] == files
    w, h, fps, codec = MO.writer_args(s)
    assert (w, h) == tuple(g["writer_size"]) and fps == float(g["writer_fps"]) and codec == str(g["codec"])
    assert (plan.width, plan.height, plan.output_fps, plan.codec) == (w, h, fps, codec)
    assert fps == (48 if s["enable_rife"] else 24)  # fps x multiplier with RIFE on, though nothing is interpolated
    sd = S.srvgg_state_dict(**MERGED_SR) if has_model else None
    ref = MO.merged_frames(s, sd)
    frames = g["frames"]
    assert len(ref) == len(frames) == len(files) - 1  # one frame per readable source, the first one included
    if s["enable_upscale"] and not has_model:          # no model: frames at source size, writer still at (w, h)
        assert frames.shape[1:3] == (72, 128) and (w, h) == (96, 54)
    exact = (not s["enable_upscale"] and 128 > w) or not has_model
    for a, b in zip(ref, frames):
        mx, f0, _ = u8_diff(a, b)
        assert a.shape == b.shape, (name, a.shape, b.shape)
        assert (mx == 0) if exact else (mx <= 1 and f0 < 0.002), (name, mx, f0)


def test_driver_frees_pinned_rings_only_after_the_writer(monkeypatch, tmp_path, folder):
    """A slow writer: every frame start_merged_pipeline pipes out is read while its pinned buffer is still alive (the
    rings are freed after the writer thread is done), and every byte is the frame computed for it."""
    import shutil
    import threading
    import time
    from visiondepth3d_b200 import render_3d as R
    live = {}

    class Ring:  # R._PinnedRing stand-in: "addresses" index numpy arrays; close() poisons them
        def __init__(self, lib, n, shape):
            self.arrays = [np.zeros(shape, np.uint8) for _ in range(n)]
            self.ptrs = [id(a) for a in self.arrays]
            live.update(zip(self.ptrs, self.arrays))

        def close(self):
            for a in self.arrays:
                a.fill(0xEE)
            self.arrays = []

    class Engine:  # the SR call stand-in: out = 255 - frame (target = source size here)
        def upscale_ptrs(self, frames, h, w, params, outs, mem):
            for f, o in zip(frames, outs):
                np.subtract(255, live[f], out=live[o])

        def upscale_chain(self, frames, params, size):
            return [255 - f for f in frames]

    import cv2
    d = tmp_path / "many"
    d.mkdir()
    srcs = [np.full((18, 32, 3), 10 + 9 * i, np.uint8) for i in range(11)]
    for i, f in enumerate(srcs):
        cv2.imwrite(str(d / f"f_{i}.png"), f)
    written, lock = [], threading.Lock()

    class SlowProc:
        class stdin:  # noqa: N801
            @staticmethod
            def write(b):
                time.sleep(0.03)  # slower than the "GPU": batches queue up behind the writer
                with lock:
                    written.append(bytes(b))

            @staticmethod
            def close():
                pass

        def wait(self):
            return 0

    monkeypatch.setattr(R, "_PinnedRing", Ring)
    monkeypatch.setattr(MP, "load_esrgan_from", lambda path: setattr(MP, "esrgan_session", Engine()))
    monkeypatch.setattr(MP, "start_ffmpeg_writer", lambda *a: SlowProc())
    monkeypatch.setattr(shutil, "which", lambda name: "/usr/bin/ffmpeg")
    try:
        MP.start_merged_pipeline(_settings(d, tmp_path, width=32, height=18, enable_upscale=True), None, None)
    finally:
        MP.esrgan_session = None
    exp = [(255 - f).tobytes() for f in sorted(srcs, key=lambda a: int(a[0, 0, 0]))]
    assert len(written) == 11 and written == exp
