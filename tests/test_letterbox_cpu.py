"""CPU: the oracle against the fixtures recorded from the unmodified reference (tests/golden/letterbox_*.npz), the
scenarios of the tracker clip, and the package's host-side tracker decisions fed with numpy / cv2 statistics."""
import json
import os

import cv2
import numpy as np
import pytest

from tests import letterbox_oracle as L
from visiondepth3d_b200 import render_depth as RD


def _host_stats(frames, prev_gray=None):
    out, prev = [], prev_gray
    for i, f in enumerate(frames):
        o = L.frame_stats(f, prev)
        st = RD._FrameStats()
        st.h, st.w = o.h, o.w
        st.y_mean, st.y_var, st.s_mean, st.edges = o.y_mean, o.y_var, o.s_mean, o.edges
        st.frame_y_mean, st.hist = o.frame_y_mean, o.hist
        st.absdiff, st.has_prev, st.prev_shape_differs = o.absdiff or 0, prev is not None, False
        out.append(st)
        prev = o.gray
    return out, prev


class _Cap:
    """In-memory cv2.VideoCapture: frame count, fps, size and POS_FRAMES seeks."""

    def __init__(self, frames, fps):
        import cv2
        self.frames, self.fps, self.pos = frames, fps, 0
        self.props = {cv2.CAP_PROP_FRAME_COUNT: len(frames), cv2.CAP_PROP_FPS: fps,
                      cv2.CAP_PROP_FRAME_WIDTH: frames[0].shape[1], cv2.CAP_PROP_FRAME_HEIGHT: frames[0].shape[0]}

    def get(self, prop):
        import cv2
        return float(self.pos) if prop == cv2.CAP_PROP_POS_FRAMES else float(self.props.get(prop, 0))

    def set(self, prop, v):
        self.pos = int(v)
        return True

    def read(self):
        if self.pos >= len(self.frames):
            return False, None
        self.pos += 1
        return True, self.frames[self.pos - 1].copy()


@pytest.fixture
def host_stats(monkeypatch):
    monkeypatch.setattr(RD, "letterbox_stats", _host_stats)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KINDS = {"letterbox_track": "letterbox_320x180.npz", "letterbox_track_nobars": "letterbox_nobars_320x180.npz"}


def golden(kind):
    return np.load(os.path.join(GOLDEN, KINDS[kind]))


@pytest.mark.parametrize("kind", list(KINDS))
def test_oracle_reproduces_reference_fixture(kind):
    g = golden(kind)
    frames = L.track_frames(kind)
    o = L.Tracker(180, float(g["fps"]))
    bars, locks, conf = o.bootstrap(frames)
    assert bars == tuple(g["boot_bars"]) and locks == tuple(g["boot_locks"]) and conf == float(g["boot_conf"])
    per = [o.update(f) for f in frames]
    assert per == [tuple(b) for b in g["bars"]]
    assert json.loads(str(g["sidecar"])) == {"top": bars[0], "bottom": bars[1], "orig_w": 320, "orig_h": 180}
    written = L.written_frames(frames, per, int(g["batch_size"]))
    assert len(written) == len(g["written"])
    for a, b in zip(written, g["written"]):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("kind", list(KINDS))
def test_package_tracker_reproduces_reference_fixture(host_stats, kind):
    g = golden(kind)
    frames = L.track_frames(kind)
    t = RD.LetterboxTracker(180, float(g["fps"]))
    cap = _Cap(frames, float(g["fps"]))
    top, bot, locks = t.bootstrap(cap)
    assert (top, bot) == tuple(g["boot_bars"]) and locks == tuple(g["boot_locks"]) and cap.pos == 0
    assert [t.update(f, i + 1) for i, f in enumerate(frames)] == [tuple(b) for b in g["bars"]]


def test_track_clip_exercises_every_scenario():
    frames = L.track_frames()
    o = L.Tracker(180, 2)
    assert o.bootstrap(frames)[1] == (True, False)
    assert L.Tracker(180, 2).bootstrap(L.track_frames("letterbox_track_nobars"))[1] == (False, True)
    log, prev = [], None
    for f in frames:
        g = L.gray_of(f)
        cut = L.scene_cut(prev, g)
        mad = None if prev is None else float(np.mean(np.abs(prev.astype(np.int16) - g.astype(np.int16))))
        cd_before = o.cooldown
        bars_before, has_before = o.bars, o.has_bars
        o.update(f)
        log.append(dict(cut=cut, mad=mad, black=L.near_black(f), cd=cd_before, streak=o.streak, bars=o.bars,
                        before=bars_before, had=has_before, det=L.bars_of_frame(f), prev=prev, gray=g))
        prev = g
    assert log[6]["black"] and log[32]["black"] and frames[32].max() > 0          # black and fade frames
    e = log[31]                                                                    # histogram-only cut
    a, b = L.hist64(e["prev"]), L.hist64(e["gray"])
    cv2.normalize(a, a)
    cv2.normalize(b, b)
    assert e["cut"] and e["mad"] <= 28 and cv2.compareHist(a, b, cv2.HISTCMP_CORREL) < 0.6
    assert [x["streak"] for x in log[8:11]] == [1, 2, 3] and log[10]["bars"] == (30, 30)   # confirmed at 3
    assert log[10]["before"] == (20, 20) and 31 % 2 == 1 and log[8]["det"] == (30, 30)     # odd bars, even rule
    assert all(x["bars"] == (30, 30) for x in log[11:16]) and log[11]["cut"] and log[11]["det"] != (30, 30)  # cooldown
    assert [x["streak"] for x in log[16:19]] == [1, 2, 0] and log[18]["bars"] == (30, 30)  # breaks off after 2
    assert log[19]["cut"] and log[19]["det"] == (26, 30) and log[19]["streak"] == 0        # below min_change
    assert log[20]["det"] == (40, 40) and sum(log[20]["det"]) > int(180 * 0.35)            # above max_total_frac
    assert log[22]["before"] == (30, 30) and log[22]["bars"] == (0, 0)                    # locked_bars -> zero
    assert log[35]["had"] is False and log[35]["bars"] == (20, 20)                       # locked_zero -> bars
    for i, gate in zip(range(23, 27), ("var", "sat", "luma", "edge")):               # one gate fails per bar kind
        f = frames[i]
        y, s = L.luma(f), L.saturation(f)
        flags = dict(luma=y.mean(1) < 16, var=y.var(1) < 3.0, sat=s.mean(1) < 6.0,
                     edge=L.edge_density(L.gray_of(f)) <= 0.04)
        row = next(r for r in range(45) if not all(flags[k][r] for k in flags))
        assert [k for k in flags if not flags[k][row]] == [gate], (i, gate)


def test_batched_update_equals_frame_by_frame(host_stats):
    frames = L.track_frames()
    a, b = RD.LetterboxTracker(180, 2), RD.LetterboxTracker(180, 2)
    a.bootstrap(_Cap(frames, 2))
    b.bootstrap(_Cap(frames, 2))
    one = [a.update(f, i) for i, f in enumerate(frames)]
    batched = []
    for i in range(0, len(frames), 4):
        batched += b.update_batch(frames[i:i + 4], i)
    assert one == batched


def test_single_frame_helpers_match_oracle(host_stats):
    frames = L.track_frames()
    for f in frames:
        assert RD.detect_letterbox_strict_robust(f) == L.bars_of_frame(f)
        assert RD.is_near_black_frame(f) == L.near_black(f)
    g = [L.gray_of(f) for f in frames]
    for a, b in zip(g, g[1:]):
        assert RD.is_scene_cut(a, b) == L.scene_cut(a, b)
    assert RD.is_scene_cut(None, g[0]) is False


def test_crop_by_bars():
    f = np.arange(100 * 4 * 3, dtype=np.uint8).reshape(100, 4, 3)
    assert RD.crop_by_bars(f, 10, 20).shape == (70, 4, 3)
    assert RD.crop_by_bars(f, 60, 40) is f


def test_synth_track_kinds_are_deterministic():
    from visiondepth3d_b200.synth import synth_frame
    for kind in KINDS:
        for i in (0, 7):
            a, b = synth_frame(i, 320, 180, kind), synth_frame(i, 320, 180, kind)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
