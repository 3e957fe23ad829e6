"""GPU: the letterbox kernels (letterbox.cu) against numpy / cv2, and the GPU-backed tracker and tracked depth video
against the oracle (tests/letterbox_oracle.py)."""
import json
import os

import numpy as np
import pytest

from tests import letterbox_oracle as L

pytestmark = pytest.mark.gpu


def _ctx():
    from visiondepth3d_b200 import _lib
    return _lib.default_context(0)


def _canny_gpu(gray, low=30, high=90):
    from visiondepth3d_b200 import _lib
    ctx = _ctx()
    g = np.ascontiguousarray(gray)
    out = np.empty_like(g)
    ctx.check(ctx.lib.vd3d_canny_u8(ctx.h, g.ctypes.data, g.shape[0], g.shape[1], float(low), float(high),
                                    out.ctypes.data, _lib.MEM_HOST))
    return out


def _blurred_noise(h, w, seed):
    import cv2
    rng = np.random.default_rng(seed)
    return cv2.GaussianBlur(rng.integers(0, 256, (h, w), dtype=np.uint8), (0, 0), 1.5)


def _spiral(n=512):
    """A one-pixel weak-edge spiral over many tiles with a single strong pixel at its outer end."""
    g = np.full((n, n), 100, np.uint8)
    y, x, d, step, k = n // 2, n // 2, 0, 1, 0
    dirs = [(0, 1), (1, 0), (0, -1), (-1, 0)]
    pts = []
    while 4 < y < n - 4 and 4 < x < n - 4:
        for _ in range(step):
            pts.append((y, x))
            y, x = y + dirs[d][0] * 1, x + dirs[d][1] * 1
        d = (d + 1) % 4
        k += 1
        if k % 2 == 0:
            step += 6
    for py, px in pts:
        g[py, px] = 112  # a gradient between the thresholds
    g[pts[-1]] = 255      # the one strong pixel
    return g


def _canny_cases():
    from visiondepth3d_b200.synth import synth_frame
    cases = {f"noise{h}x{w}": _blurred_noise(h, w, h + w) for h, w in ((180, 320), (181, 321), (1080, 1920),
                                                                      (2160, 3840))}
    cases["natural"] = L.gray_of(synth_frame(3, 320, 180, "natural")[0])
    cases["letterbox"] = L.gray_of(synth_frame(5, 320, 180, "letterbox")[0])
    cases["flat"] = np.full((90, 160), 77, np.uint8)
    cases["small64"] = _blurred_noise(64, 64, 7)
    b = np.zeros((120, 200), np.uint8)
    b[0, :], b[-1, :], b[:, 0], b[:, -1] = 255, 200, 180, 255
    b[40:80, 60:140] = 150
    cases["borders"] = b
    cases["spiral"] = _spiral()
    return cases


@pytest.mark.parametrize("name", list(_canny_cases()))
def test_canny_matches_cv2(name):
    g = _canny_cases()[name]
    assert np.array_equal(_canny_gpu(g), L.canny(g)), name
    if name in ("noise180x320", "spiral", "natural"):
        import cv2
        assert np.array_equal(_canny_gpu(g, 50, 150), cv2.Canny(g, 50, 150, apertureSize=3, L2gradient=True))


def _stats(frames, prev=None, device=False):
    from visiondepth3d_b200 import _lib
    ctx = _ctx()
    fr = np.ascontiguousarray(np.stack(frames))
    n, h, w = fr.shape[:3]
    rec = dict(ym=np.empty((n, h), np.float32), yv=np.empty((n, h), np.float32), sm=np.empty((n, h), np.float32),
               ed=np.empty((n, h), np.int32), fm=np.empty(n, np.float32), hist=np.empty((n, 64), np.uint32),
               ad=np.empty(n, np.uint64))
    if device:
        import torch
        f_t = torch.from_numpy(fr).cuda()
        p_t = torch.from_numpy(np.ascontiguousarray(prev)).cuda() if prev is not None else None
        last_t = torch.empty((h, w), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        fp, pp, lp, mem = f_t.data_ptr(), p_t.data_ptr() if p_t is not None else None, last_t.data_ptr(), _lib.MEM_DEVICE
    else:
        last = np.empty((h, w), np.uint8)
        pv = np.ascontiguousarray(prev) if prev is not None else None
        fp, pp, lp, mem = fr.ctypes.data, pv.ctypes.data if pv is not None else None, last.ctypes.data, _lib.MEM_HOST
    ctx.check(ctx.lib.vd3d_letterbox_stats(ctx.h, n, fp, h, w, pp, mem, *(rec[k].ctypes.data for k in
                                                                         ("ym", "yv", "sm", "ed", "fm", "hist", "ad")),
                                           lp))
    rec["last"] = last_t.cpu().numpy() if device else last
    return rec


@pytest.mark.parametrize("w", [5, 7, 13, 100, 128, 129, 333, 3840])
@pytest.mark.parametrize("device", [False, True])
def test_stats_equal_numpy_bit_for_bit(w, device):
    rng = np.random.default_rng(w)
    h, n = 70, 3
    frames = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(n)]
    frames[1][: h // 3] = rng.integers(0, 8, (h // 3, w, 3), dtype=np.uint8)  # a dark band
    for prev in (None, rng.integers(0, 256, (h, w), dtype=np.uint8)):
        r = _stats(frames, prev, device)
        p = prev
        for i, f in enumerate(frames):
            o = L.frame_stats(f, p)
            assert np.array_equal(r["ym"][i], o.y_mean) and np.array_equal(r["yv"][i], o.y_var)
            assert np.array_equal(r["sm"][i], o.s_mean)
            assert r["fm"][i].tobytes() == np.float32(o.frame_y_mean).tobytes()
            assert np.array_equal(r["ed"][i], o.edges) and np.array_equal(r["hist"][i], o.hist)
            assert int(r["ad"][i]) == (o.absdiff or 0)
            p = o.gray
        assert np.array_equal(r["last"], L.gray_of(frames[-1]))


def test_stats_frame_mean_at_4k():
    from visiondepth3d_b200.synth import synth_frame
    f = synth_frame(2, 3840, 2160, "natural")[0]
    r = _stats([f, f[::-1].copy()])
    for i, x in enumerate((f, f[::-1])):
        assert r["fm"][i] == L.luma(x).mean()
        assert np.array_equal(r["ym"][i], L.luma(x).mean(axis=1)) and np.array_equal(r["yv"][i], L.luma(x).var(axis=1))


@pytest.mark.parametrize("kind", ["letterbox_track", "letterbox_track_nobars"])
def test_gpu_tracker_matches_reference_fixture(kind):
    from visiondepth3d_b200 import render_depth as RD
    from tests.test_letterbox_cpu import _Cap, golden
    g = golden(kind)
    clip = L.track_frames(kind)
    want = [tuple(b) for b in g["bars"]]
    t = RD.LetterboxTracker(180, 2)
    top, bot, locks = t.bootstrap(_Cap(clip, 2))
    assert (top, bot) == tuple(g["boot_bars"]) and locks == tuple(g["boot_locks"])
    assert [t.update(f, i + 1) for i, f in enumerate(clip)] == want
    import torch
    b = RD.LetterboxTracker(180, 2)
    b.bootstrap(_Cap(clip, 2))
    got = []
    for i in range(0, len(clip), 4):  # device-resident batches, as the depth-video pass runs them
        got += b.update_batch(torch.from_numpy(np.stack(clip[i:i + 4])).cuda(), i + 1)
    assert got == want


def test_gpu_repad_of_fixture_depth_matches_reference_writes():
    from visiondepth3d_b200 import render_depth as RD
    from tests.test_letterbox_cpu import golden
    g = golden("letterbox_track")
    clip = L.track_frames()
    bars = [tuple(b) for b in g["bars"]]
    for i, f in enumerate(clip):
        top, bot = bars[min(len(clip), (i // 4 + 1) * 4) - 1]
        got, ref = RD.letterbox_repad(L.stub_depth_u8(f), top, bot), g["written"][i]
        core_h = 180 - top - bot
        assert (got[:top] == ref[:top]).all() and (got[top + core_h:] == ref[top + core_h:]).all()
        d = np.abs(got.astype(int) - ref.astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 0.002


def test_repad_matches_oracle():
    from visiondepth3d_b200 import render_depth as RD
    rng = np.random.default_rng(5)
    for h, w, t, b in ((180, 320, 20, 24), (181, 321, 30, 0), (1080, 1920, 138, 138), (64, 64, 0, 0), (90, 90, 50, 50)):
        d = (np.linspace(0, 255, h)[:, None] + rng.integers(0, 40, (h, w))).clip(0, 255).astype(np.uint8)
        got, want = RD.letterbox_repad(d, t, b), L.repad(d, t, b)
        core_h = h - t - b
        if (t or b) and core_h > 0:
            core = RD.resize_cubic_u8(d, w, core_h)
            exact = np.full((h, w), int(np.median(core)), np.uint8)
            exact[t:t + core_h] = core
            assert np.array_equal(got, exact)
            assert (got[:t] == want[:t]).all() and (got[t + core_h:] == want[t + core_h:]).all()
            diff = np.abs(got.astype(int) - want.astype(int))
            assert diff.max() <= 1 and (diff > 0).mean() < 0.002
        else:
            assert np.array_equal(got, d)


def test_repad_device_memory():
    import torch
    from visiondepth3d_b200 import _lib, render_depth as RD
    d = np.random.default_rng(1).integers(0, 256, (180, 320), dtype=np.uint8)
    src, dst = torch.from_numpy(d).cuda(), torch.empty((180, 320), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx = _ctx()
    ctx.check(ctx.lib.vd3d_letterbox_repad(ctx.h, src.data_ptr(), 180, 320, 16, 22, dst.data_ptr(), _lib.MEM_DEVICE))
    assert np.array_equal(dst.cpu().numpy(), RD.letterbox_repad(d, 16, 22))


@pytest.fixture(scope="module")
def depth_model():
    from visiondepth3d_b200 import render_depth as RD
    RD.load_depth_model("vits", width=320, height=180, seed=0)
    return RD


def test_tracked_depth_frames_equal_repad_of_plain_depth(depth_model):
    RD = depth_model
    from tests.test_letterbox_cpu import _Cap, golden
    frames = L.track_frames()
    bars = [tuple(b) for b in golden("letterbox_track")["bars"]]
    t = RD.LetterboxTracker(180, 2)
    cap = _Cap(frames, 2)
    t.bootstrap(cap)
    got = list(RD.iter_depth_frames(cap, 320, 180, batch_size=4, tracker=t))
    plain = list(RD.iter_depth_frames(_Cap(frames, 2), 320, 180, batch_size=4))
    assert len(got) == len(frames) == len(plain)
    for i in range(len(frames)):
        b = bars[min(len(frames), (i // 4 + 1) * 4) - 1]  # the state after the batch's last frame
        assert np.array_equal(got[i], RD.letterbox_repad(plain[i], *b))
        if b != (0, 0):
            assert (got[i][: b[0]] == got[i][0, 0]).all()


class _Bars:
    """Stand-in tracker: fixed bars after every batch; records the index of each batch's first frame."""

    def __init__(self, bars):
        self.bars, self.first = bars, []

    def update_batch(self, frames, first_idx=0):
        self.first.append(first_idx)
        return [self.bars] * len(frames)


@pytest.mark.parametrize("inf,bars,invert", [((224, 126), None, False), ((224, 126), (12, 10), True),
                                             ((448, 252), None, True), ((448, 252), (12, 10), False)])
def test_depth_frames_with_inference_size_equal_host_composition(depth_model, inf, bars, invert):
    """process_video2 with an inference size: each frame through hf_batch_safe_pipe at that size (Pillow resize in
    the pipe), convert_depth_to_grayscale, inversion, INTER_CUBIC back to the frame size and the re-pad to the
    tracked bars."""
    from PIL import Image
    from tests.test_letterbox_cpu import _Cap
    RD = depth_model
    frames = L.track_frames()[:10]
    tracker = _Bars(bars) if bars else None
    got = list(RD.iter_depth_frames(_Cap(frames, 2), 320, 180, invert, inf, batch_size=4, tracker=tracker))
    assert len(got) == len(frames)
    if tracker:
        assert tracker.first == [1, 5, 9]
    for f, g in zip(frames, got):
        d = RD.hf_batch_safe_pipe([Image.fromarray(f[..., ::-1].copy())], inf)[0]["predicted_depth"]
        want = RD.convert_depth_to_grayscale(d)
        if invert:
            want = 255 - want
        want = RD.resize_cubic_u8(want, 320, 180)
        if bars:
            want = RD.letterbox_repad(want, *bars)
        assert np.array_equal(g, want)


def test_depth_video_end_to_end(depth_model, tmp_path):
    import cv2
    RD = depth_model
    frames = L.track_frames()[:20]
    src = str(tmp_path / "clip.avi")
    wr = cv2.VideoWriter(src, cv2.VideoWriter_fourcc(*"FFV1"), 2.0, (320, 180))
    for f in frames:
        wr.write(f)
    wr.release()
    cap = cv2.VideoCapture(src)
    decoded = [cap.read()[1] for _ in frames]
    cap.release()
    on, off = str(tmp_path / "on_depth.mkv"), str(tmp_path / "off_depth.mkv")
    assert RD.depth_video_from_video(src, on, batch_size=3, ignore_letterbox_bars=True) == len(frames)
    assert RD.depth_video_from_video(src, off, batch_size=3) == len(frames)
    (t, b), conf = L.bootstrap(decoded, 180, 2.0)
    want_bars = (t, b) if conf >= 0.7 and t + b > 0 else (0, 0)
    side = json.load(open(os.path.splitext(on)[0] + ".letterbox.json"))
    assert side == {"top": want_bars[0], "bottom": want_bars[1], "orig_w": 320, "orig_h": 180}
    assert json.load(open(os.path.splitext(off)[0] + ".letterbox.json")) == {"top": 0, "bottom": 0, "orig_w": 320,
                                                                               "orig_h": 180}
    cap = cv2.VideoCapture(on)
    first = cap.read()[1][..., 0]
    n = 1 + sum(1 for _ in iter(lambda: cap.read()[0], False))
    cap.release()
    assert n == len(frames)
    if want_bars[0] > 4:
        bar = first[: want_bars[0] - 4].astype(int)
        assert bar.max() - bar.min() <= 3  # XVID keeps a flat bar flat up to coding noise
