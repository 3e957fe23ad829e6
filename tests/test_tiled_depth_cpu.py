"""CPU: the restatement of the reference's tiled depth path (tests/tiled_oracle.py) reproduces every tiled_* fixture
exactly, its percentile equals np.percentile on adversarial arrays, and render_depth exposes the reference's names."""
import glob
import inspect
import os

import numpy as np
import pytest

from tests import tiled_oracle as T

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FIXTURES = sorted(p for p in glob.glob(os.path.join(GOLDEN, "tiled_*.npz")) if "tiled_video_" not in p)


def test_fixtures_present():
    assert len(FIXTURES) == 8


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[6:-4] for p in FIXTURES])
def test_restatement_reproduces_fixture(path):
    g = np.load(path)
    w, h = (int(v) for v in g["size"])
    inf = tuple(int(v) for v in g["inference_size"])
    inf = None if inf == (0, 0) else inf
    tile, pad, kind = int(g["tile"]), int(g["pad"]), str(g["kind"])
    depth, tiles, crops = T.infer(g["rgb"], inf, tile, pad, lambda c: T.prediction(c, kind))
    # plan and crops handed to the pipe
    assert [tuple(c) for c in g["crop_sizes"]] == [(t[9], t[8]) for t in tiles]
    assert np.array_equal(np.concatenate([c.ravel() for c in crops]), g["crops"])
    # blended float32 depth, bit for bit (border pixels included)
    assert depth.dtype == np.float32
    assert np.array_equal(depth.view(np.uint32), g["depth"].view(np.uint32))
    # percentiles and the written frame
    assert np.array_equal(np.array([T.percentile(depth, 1.0), T.percentile(depth, 99.0)], np.float32), g["pct"])
    assert np.array_equal(T.normalize_u8(depth, (w, h), bool(g["invert"])), g["u8"])
    # the reference's TILE_DEBUG lines and range line
    lines = str(g["log"]).splitlines()
    assert lines[:-1] == T.debug_lines(tiles)
    assert lines[-1] == f"[tile] range min={float(np.nanmin(depth)):.6f} max={float(np.nanmax(depth)):.6f}"


def test_fixtures_cover_the_cases():
    by = {os.path.basename(p)[6:-4]: np.load(p) for p in FIXTURES}
    # more than 2 x 2 tiles cover a pixel when the pad is large against the tile
    g = by["bigpad_100x64_t64p24"]
    tiles = T.plan(100, 64, 64, 24)
    cover = np.zeros((64, 100), int)
    for y0, y1, x0, x1, *_ in tiles:
        cover[y0:y1, x0:x1] += 1
    assert cover.max() > 4
    # a last column narrower than the pad
    assert any(t[3] - t[2] < 16 for t in T.plan(203, 117, 96, 16))
    # a frame smaller than one tile
    assert all(v < 96 for v in by["small_80x60_t96p16"]["size"])
    # border pixels covered only by cubic Hann tails: weights <= 0 occur
    assert min(T.weights(t[1] - t[0], t[3] - t[2], 96, 16).min() for t in T.plan(256, 144, 96, 16)) <= 0
    assert g["depth"].min() < -1e6  # divided by the 1e-8 floor


ADVERSARIAL = [
    np.array([3.5], np.float32),
    np.array([2.0, -1.0], np.float32),
    np.array([1.0, 1.0, 1.0, 2.0], np.float32),
    np.array([-3e30, 1e30, 5e30, -1e31, 0.0, 7.0], np.float32),
    np.repeat(np.array([-2.0, 0.5, 0.5, 9.0], np.float32), 37),
    np.array([0.0, -0.0, 1e-7, -1e-7, 1e38, -1e38], np.float32),
]


def test_percentile_matches_numpy():
    rng = np.random.default_rng(3)
    arrays = list(ADVERSARIAL)
    for n in (1, 2, 3, 99, 100, 101, 1000, 12345):
        arrays.append((rng.standard_normal(n) * 10.0 ** rng.integers(-8, 30)).astype(np.float32))
        arrays.append(rng.integers(-3, 3, n).astype(np.float32))
    bad = rng.standard_normal(500).astype(np.float32)
    bad[::7], bad[3::11], bad[5::13] = np.nan, np.inf, -np.inf
    arrays.append(np.nan_to_num(bad, nan=0.0, posinf=0.0, neginf=0.0))
    for a in arrays:
        for p in (1.0, 99.0, 0.0, 100.0, 50.0, 25.0):
            got, want = T.percentile(a, p), np.percentile(a, p)
            assert got.dtype == np.float32 and want.dtype == np.float32
            assert got == want or (got == 0 and want == 0), (a[:8], p, got, want)


def test_normalize_branches():
    # percentile clip, min-max fallback (p1 == p99 with a range), flat 128
    d = np.full((40, 50), 5.0, np.float32)
    d[0, :3] = 3.0
    u = T.normalize_u8(d, (50, 40))
    assert u.max() == 254 and u.min() == 0  # min-max branch: the + 1e-6 keeps the top below 255
    assert np.array_equal(T.normalize_u8(np.full((9, 9), 2.0, np.float32), (9, 9)), np.full((9, 9), 128, np.uint8))


def test_public_names_have_reference_signatures():
    from visiondepth3d_b200 import render_depth as R
    assert (R.USE_TILED_DEPTH, R.TILE_SIZE, R.TILE_PAD, R.TILE_DEBUG) == (False, 512, 32, False)
    assert str(inspect.signature(R.infer_depth_tile)) == "(model_call, rgb_np, inference_size, tile=512, pad=32)"
    assert str(inspect.signature(R._run_pipe_or_tile)) == "(images_pil, inference_size)"
    assert str(inspect.signature(R._hann2d)) == "(h, w)"
    assert str(inspect.signature(R._ensure_depth_np)) == "(pred)"
    assert str(inspect.signature(R._normalize_to_u8)) == "(depth_f, out_size, invert=False, pclip=(1.0, 99.0))"
    for hw in ((448, 448), (2, 2), (1, 5)):
        assert np.array_equal(R._hann2d(*hw), T.hann2d(*hw))
    assert R.tile_plan(203, 117, 96, 16) == T.plan(203, 117, 96, 16)
    assert len(R.tile_plan(1920, 1080)) == 15 and len(R.tile_plan(3840, 2160)) == 45


def test_ensure_depth_np_forms():
    from visiondepth3d_b200 import render_depth as R
    a = np.arange(20, dtype=np.float64).reshape(4, 5)
    assert R._ensure_depth_np([{"predicted_depth": a}]).dtype == np.float32
    assert R._ensure_depth_np(a[None]).shape == (4, 5)
    assert np.array_equal(R._ensure_depth_np(np.stack([a, a + 3, a + 6], -1)), (a + 3).astype(np.float32))
    with pytest.raises(TypeError):
        R._ensure_depth_np("x")


def test_infer_depth_tile_refuses_other_callables():
    from visiondepth3d_b200 import render_depth as R
    with pytest.raises(TypeError):
        R.infer_depth_tile(lambda imgs, inference_size=None: None, np.zeros((32, 32, 3), np.uint8), None)


@pytest.mark.parametrize("which", ["bars", "nobars"])
def test_restatement_reproduces_video_branch(which):
    """process_video2's tiled branch (recorded from the reference, 13 frames in batches of 4, with and without
    ignore_letterbox_bars): every written frame and every printed range line."""
    from visiondepth3d_b200.synth import synth_frame
    g = np.load(os.path.join(GOLDEN, f"tiled_video_{which}_320x180.npz"))
    frames = [synth_frame(i, 320, 180, "letterbox_track")[0] for i in range(len(g["written"]))]
    bars = [tuple(b) for b in g["bars"]]
    assert (len(set(bars)) > 1) == (which == "bars")  # the bars change inside the clip, so the re-pad follows them
    out, depths = T.video_frames(frames, bars, int(g["batch_size"]), int(g["tile"]), int(g["pad"]), False,
                                 lambda c: T.prediction(c, "ramp"))
    for k, (a, b) in enumerate(zip(out, g["written"])):
        assert np.array_equal(a, b), k
    assert str(g["ranges"]).splitlines() == [
        f"[tile] range min={float(np.nanmin(d)):.6f} max={float(np.nanmax(d)):.6f}" for d in depths]
