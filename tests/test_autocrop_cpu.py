"""CPU: auto_crop_black_bars of render_sbs_3d.  The oracle (tests/autocrop_oracle.py) against the unmodified
reference on the letterbox set (tools/gen_golden.py autocrop: every (top, bottom) the reference detected, and the final
frames), the edge cases of detect_black_bars, and the drop-in's host logic (probe line, per-frame lines, writer size,
refusals) against a stub of the C ABI."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from oracle import dibr as O
from tests import autocrop_oracle as A
from tests.util import u8_diff
from visiondepth3d_b200.synth import synth_frame

_BASE = dict(output_width=320, output_height=180, sharpness_factor=0.2, output_format="Half-SBS",
             dof_strength=0.0, feather_strength=10.0, blur_ksize=9, use_subject_tracking=True,
             use_floating_window=True, preserve_original_aspect=False, zero_parallax_strength=0.01,
             auto_crop_black_bars=True)
# fixture -> (frames incl. the dropped probe, render params); shared with tests/test_autocrop_gpu.py
AUTOCROP_CASES = {
    "loop_autocrop_halfsbs_320x180.npz": (8, dict(_BASE)),
    "loop_autocrop_fullsbs_320x180.npz": (6, dict(_BASE, output_format="Full-SBS", preserve_original_aspect=True)),
    "loop_autocrop_dof_halfsbs_320x180.npz": (6, dict(_BASE, dof_strength=1.5)),
}


def oracle_params(rp_kw, probe):
    """RenderParams as render_sbs_3d resolves them: original_video_* from the cropped probe frame when left at None."""
    rp = A.RenderParams(**rp_kw)
    if rp.preserve_original_aspect:
        rp.original_video_width, rp.original_video_height = A.probe_original_size(probe, rp)
    return rp


@pytest.mark.parametrize("name", sorted(AUTOCROP_CASES))
def test_autocrop_loop_vs_reference(golden_dir, name):
    n, kw = AUTOCROP_CASES[name]
    g = np.load(os.path.join(golden_dir, name))
    step = int(g["rows"])
    crops = [tuple(int(v) for v in c) for c in g["crops"]]
    assert len(crops) == n
    probe, _ = synth_frame(0, 320, 180, "letterbox")
    assert A.detect_black_bars(probe) == crops[0]
    rp = oracle_params(kw, probe)
    gs, cs = O.GlobalState(), O.ClipState()
    for j, i in enumerate(range(1, n)):  # the reference drops the first frame of a clip
        fr, dp = synth_frame(i, 320, 180, "letterbox")
        f, parts = A.render_frame(gs, cs, fr, dp, rp, return_parts=True)
        assert parts["crop"] == crops[i], (name, i)
        ref = g[f"final{j}"]
        assert f[::step].shape == ref.shape
        mx, f0, f1 = u8_diff(f[::step], ref)
        assert mx <= 12 and f1 <= 0.03, (name, j, mx, f0, f1)
    assert len([k for k in g.files if k.startswith("final")]) == n - 1


def test_detect_black_bars_edge_cases():
    import cv2

    def ref(fr, threshold=10):  # core/render_3d.py:293-316 on the u8 frame
        gray = cv2.cvtColor(fr, cv2.COLOR_BGR2GRAY)
        h = gray.shape[0]
        top = bottom = 0
        for i in range(h):
            if np.mean(gray[i]) > threshold:
                top = i
                break
        for i in range(h - 1, -1, -1):
            if np.mean(gray[i]) > threshold:
                bottom = h - i - 1
                break
        return top, bottom

    w, h = 37, 20
    fr = np.zeros((h, w, 3), dtype=np.uint8)
    assert A.detect_black_bars(fr) == ref(fr) == (0, 0)          # all black
    fr[:] = 10
    assert A.detect_black_bars(fr) == ref(fr) == (0, 0)          # mean exactly 10 is not bright
    fr[7, 5] = 11
    assert A.detect_black_bars(fr) == ref(fr) == (7, 12)         # one pixel above: 1-row content
    fr[0] = 200
    assert A.detect_black_bars(fr) == ref(fr) == (0, 12)         # bright first row
    fr[h - 1] = 200
    assert A.detect_black_bars(fr) == ref(fr) == (0, 0)          # bright last row
    rng = np.random.default_rng(3)
    for _ in range(40):
        fr = rng.integers(0, 12, (h, w, 3), dtype=np.uint8)
        fr[rng.integers(0, h)] = rng.integers(0, 40, (w, 3), dtype=np.uint8)
        assert A.detect_black_bars(fr) == ref(fr)
    assert A.crop_rows(20, 7, 12) == (7, 1) and A.crop_rows(20, 10, 10) == (0, 20)


def test_probe_size_rule():
    probe, _ = synth_frame(0, 320, 180, "letterbox")
    rp = A.RenderParams(output_format="Full-SBS", preserve_original_aspect=True, auto_crop_black_bars=True)
    assert A.probe_original_size(probe, rp) == (320, 180 - 22 - 25)
    rp.auto_crop_black_bars = False
    assert A.probe_original_size(probe, rp) == (320, 180)
    rp.original_video_width, rp.original_video_height = 640, 360
    assert A.probe_original_size(probe, rp) == (640, 360)


# ---------------------------------------------------------------------------------------------------------------------
# drop-in host logic against a stub library
# ---------------------------------------------------------------------------------------------------------------------
class _Var:
    def __init__(self, v):
        self.v = v

    def get(self):
        return self.v


class _StubLib:
    """vd3d_render_clip 'renders' by copying each frame's first byte; vd3d_last_crops reports (tag, tag + 1) per frame of
    the last call; vd3d_detect_black_bars reports (3, 5)."""

    def __init__(self, real):
        self.real = real
        self.last = []
        self.detect_calls = 0
        self.rps = []
        self._keep = []

    def vd3d_plan_sizes(self, *a):
        return self.real.vd3d_plan_sizes(*a)

    def vd3d_check_config(self, h, sh, sw, rp):
        self.rps.append((rp._obj.original_video_width, rp._obj.original_video_height, rp._obj.auto_crop_black_bars))
        return 0

    def vd3d_sync(self, *a):
        return 0

    def vd3d_host_alloc(self, n):
        buf = (C.c_uint8 * int(n))()
        self._keep.append(buf)
        return C.addressof(buf)

    def vd3d_host_free(self, p):
        return None

    def vd3d_detect_black_bars(self, h, frame, fh, fw, mem, top, bottom):
        self.detect_calls += 1
        top._obj.value, bottom._obj.value = 3, 5
        return 0

    def vd3d_render_clip(self, h, n, fp, dp, dch, sh, sw, rp, op, mem, infos):
        self.last = []
        for i in range(n):
            tag = C.cast(fp[i], C.POINTER(C.c_uint8))[0]
            C.cast(op[i], C.POINTER(C.c_uint8))[0] = tag
            self.last.append(tag)
        return 0

    def vd3d_last_crops(self, h, out, n):
        assert n == len(self.last)
        for i, t in enumerate(self.last):
            out[2 * i], out[2 * i + 1] = t, t + 1
        return 0


class _NoCropLib(_StubLib):
    """The library surface before auto-crop existed: a render without the option must not need more."""

    def __getattribute__(self, name):
        if name in ("vd3d_detect_black_bars", "vd3d_last_crops"):
            raise AttributeError(name)
        return object.__getattribute__(self, name)


class _StubCtx:
    def __init__(self, lib):
        self.lib, self.h = lib, C.c_void_p(1)

    def check(self, rc):
        assert rc == 0

    def reset(self, which=3):
        pass


@pytest.fixture
def dropin(monkeypatch):
    import cv2
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R
    state = {"n": 20, "lib": _StubLib(_lib.load())}
    monkeypatch.setattr(R, "_ctx", lambda: _StubCtx(state["lib"]))

    class Cap:
        def __init__(self, path):
            self.pos = 0

        def isOpened(self):
            return True

        def get(self, prop):
            return {cv2.CAP_PROP_FRAME_COUNT: float(state["n"]), cv2.CAP_PROP_FPS: 24.0,
                    cv2.CAP_PROP_POS_FRAMES: float(self.pos)}.get(prop, 0.0)

        def set(self, prop, v):
            if prop == cv2.CAP_PROP_POS_FRAMES:
                self.pos = int(v)
            return True

        def read(self):
            if self.pos >= state["n"]:
                return False, None
            f = np.full((36, 64, 3), self.pos % 256, dtype=np.uint8)
            self.pos += 1
            return True, f

        def release(self):
            pass

    written, sizes = [], []

    class Sink:
        def __init__(self, path, size, *a):
            sizes.append(size)

        def ok(self):
            return True

        def write(self, frame):
            written.append(int(frame.flat[0]))

        def close(self):
            pass

    monkeypatch.setattr(cv2, "VideoCapture", Cap)
    monkeypatch.setattr(R, "_FrameSink", Sink)

    def run(fmt="Half-SBS", **kw):
        written.clear()
        sizes.clear()
        R.render_sbs_3d("rgb", "depth", "out.mp4", "mp4v", 24.0, 64, 36, 4.5, -1.5, -6.0, 0.2, fmt,
                        _Var("Default (16:9)"), R.aspect_ratios, 0.0, suspend_flag=threading.Event(),
                        cancel_flag=threading.Event(), **kw)
        return list(written), list(sizes)
    return run, state


def test_dropin_prints_probe_and_per_frame_crops(dropin, capsys):
    run, state = dropin
    out, sizes = run(auto_crop_black_bars=True)
    lines = capsys.readouterr().out.splitlines()
    assert out == list(range(1, 20)) and sizes == [(64, 36)]
    assert state["lib"].detect_calls == 1
    assert lines.count("Auto-crop: Top 3px | Bottom 5px") == 1
    per_frame = [ln for ln in lines if ln.startswith("🔪")]
    assert per_frame == [f"🔪 Cropping top: {t}px, bottom: {t + 1}px" for t in range(1, 20)]  # frame order, 3 batches
    assert lines.index("Auto-crop: Top 3px | Bottom 5px") < lines.index(per_frame[0])


def test_dropin_probe_size_fallback(dropin):
    run, state = dropin
    # preserve_original_aspect with original_video_* None: the writer gets the cropped probe size (W, H - 3 - 5)
    _, sizes = run(fmt="Full-SBS", preserve_original_aspect=True, auto_crop_black_bars=True)
    assert sizes == [(2 * 64, 36 - 8)] and state["lib"].rps[-1] == (64, 28, 1)
    # explicit sizes win, as in the reference
    _, sizes = run(fmt="Full-SBS", preserve_original_aspect=True, auto_crop_black_bars=True,
                   original_video_width=64, original_video_height=36)
    assert sizes == [(128, 36)] and state["lib"].rps[-1] == (64, 36, 1)


def test_dropin_without_autocrop_needs_no_new_entry_points(dropin, capsys):
    from visiondepth3d_b200 import _lib
    run, state = dropin
    state["lib"] = _NoCropLib(_lib.load())
    out, sizes = run(fmt="Full-SBS", preserve_original_aspect=True)
    assert out == list(range(1, 20)) and sizes == [(128, 36)] and state["lib"].rps[-1] == (0, 0, 0)
    assert "Cropping" not in capsys.readouterr().out


def test_dropin_still_refuses_skip_blank_frames(dropin, capsys):
    run, state = dropin
    assert run(skip_blank_frames=True) == ([], [])
    assert run(skip_blank_frames=True, auto_crop_black_bars=True) == ([], [])
    assert "skip_blank_frames" in capsys.readouterr().out and state["lib"].detect_calls == 0
