"""GPU: the eye-fit stage beyond integer factors -- cv2's general INTER_AREA shrink (ResizeArea_ tables built on the
host exactly as cv2 does, applied inside k_post) through vd3d_fit_eye and through the VR render loop.

Gates: the fit is the same fp32 arithmetic as the oracle (which equals cv2 bit-for-bit on CPU,
tests/test_oracle_golden.py::test_inter_area_matches_cv2) -> exact; the VR loop like every other full frame."""
import os

import numpy as np
import pytest

from oracle import dibr as O
from tests.test_dibr_gpu import _rp
from tests.util import VR_CASE, u8_diff
from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    from visiondepth3d_b200 import render_3d
    return render_3d


@pytest.mark.parametrize("case", [(480, 270, 360, 400), (640, 360, 427, 240), (500, 350, 333, 233), (400, 300, 399, 299),
                                  (1600, 900, 1440, 1600), (96, 54, 48, 27), (96, 54, 96, 54), (480, 270, 240, 203)])
def test_fit_eye_matches_oracle(R, case):
    w, h, tw, th = case
    rng = np.random.default_rng(w * 31 + th)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    assert np.array_equal(R.pad_to_aspect_ratio(img, tw, th), O.pad_to_aspect(img, tw, th)), case
    if tw <= w and th <= h:
        assert np.array_equal(R.resize_area(img, tw, th), O.resize_area(img, tw, th)), case


@pytest.mark.parametrize("case", [(1280, 720, 1920, 1080), (160, 90, 1440, 1600), (100, 70, 133, 91), (100, 70, 80, 140)])
def test_fit_eye_enlarge_matches_oracle(R, case):
    """cv2 INTER_AREA with an enlarged axis = fixed-point bilinear emulation; integer arithmetic, exact."""
    w, h, tw, th = case
    rng = np.random.default_rng(w * 17 + th)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    assert np.array_equal(R.pad_to_aspect_ratio(img, tw, th), O.pad_to_aspect(img, tw, th)), case
    assert np.array_equal(R.resize_area(img, tw, th), O.resize_area(img, tw, th)), case


def test_vr_loop_vs_oracle_and_golden(R, golden_dir):
    c = VR_CASE
    g = np.load(os.path.join(golden_dir, c["file"]))
    rp, orp = _rp(R, c["rp"], c["sw"], c["sh"])
    R.reset_temporal_state()
    gs, cs = O.GlobalState(), O.ClipState()
    for j, i in enumerate(range(1, c["n"])):
        fr, dp = synth_frame(i, c["sw"], c["sh"], c["kind"])
        out = R.render_frame(fr, dp, rp)
        ref = O.render_frame(gs, cs, fr, dp, orp)
        assert out.shape == ref.shape == (1600, 2880, 3)
        mx, f0, f1 = u8_diff(out, ref)
        assert mx <= 16 and f1 <= 0.10 and f0 <= 0.30, (j, mx, f0, f1)   # default (fast) arithmetic on ramp content: see tests/test_dibr_gpu.py::_tol
        y0, y1 = int(g[f"final{j}_y0"]), int(g[f"final{j}_y1"])
        assert not out[:y0].any() and not out[y1:].any()
        mx, f0, f1 = u8_diff(out[y0:y1:3, ::3], g[f"final{j}_band"])  # vs the real reference
        assert mx <= 12 and f1 <= 0.03, (j, mx, f0, f1)
    l = np.full((1600, 1440, 3), 7, dtype=np.uint8)
    assert np.array_equal(R.format_3d_output(l, l + 1, "VR"), np.hstack((l, l + 1)))


def test_resize_cubic_u8_matches_oracle():
    """resize_cubic_u8 (vd3d_resize_cubic on one channel: the depth writer's cv2 INTER_CUBIC) against the cv2-pinned
    oracle: same float32 arithmetic, exact."""
    from visiondepth3d_b200 import render_depth as RD
    rng = np.random.default_rng(9)
    for (w, h, ow, oh) in ((924, 518, 1920, 1080), (100, 70, 133, 91), (640, 360, 320, 180), (37, 23, 80, 50), (64, 48, 64, 48)):
        img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        assert np.array_equal(RD.resize_cubic_u8(img, ow, oh), O.resize_cubic_u8(img, ow, oh)), (w, h, ow, oh)
    d = rng.random((70, 100)).astype(np.float32)
    u = RD._normalize_to_u8(d, (133, 91), invert=True)
    lo, hi = np.percentile(d, 1.0), np.percentile(d, 99.0)
    ref = 255 - (np.clip((d - lo) / (hi - lo), 0.0, 1.0) * 255.0).astype(np.uint8)
    assert np.array_equal(u, O.resize_cubic_u8(ref, 133, 91))
