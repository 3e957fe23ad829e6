"""GPU: dpt-beit-large-512 (MiDaS v3.1 BEiT-L 512) on the depth engine -- the attention with relative position bias
(k_umma_attention<true>) against float64 on the engine's own q / k / v^T buffers, the forward against
tests/dpt_beit_oracle.py (fp32), a batch against single forwards, the family's argument checks, and the image / video
drivers of render_depth with a model written by save_pretrained.  Every model here has its bias tables filled
(transformers initialises them to zeros, which would leave the bias path untested)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from tests import depth_kernel_refs as R
from tests import dpt_beit_oracle as OB
from tests.test_depth_kernels_gpu import ACC, stored_f16

pytestmark = pytest.mark.gpu


def _depth_u8(d):
    d = d.astype(np.float32)
    return ((d - d.min()) / (d.max() - d.min() + np.float32(1e-6)) * 255).astype(np.uint8)


def _engine(sd, cfg, h, w, processor=None):
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine(cfg, h, w, family="dpt-beit", processor=processor)
    e.load_state_dict(sd)
    return e


@pytest.fixture(scope="module")
def small():
    return OB.random_model(small=True, seed=3)


@pytest.fixture(scope="module")
def large():
    return OB.random_model(seed=1)


# ---------------------------------------------------------------------------------------------------------------------
# the attention with relative position bias, isolated: the last layer's attention of a forward, recomputed in float64
# from the q, k, v^T the device stored and the layer's prepared (grid-resampled) table
# ---------------------------------------------------------------------------------------------------------------------
class BiasRig:
    def __init__(self, sd, cfg, h, w):
        from visiondepth3d_b200.depth_weights import prepare_dpt_beit
        self.cfg, self.h, self.w = cfg, h, w
        self.ph, self.pw = h // 16, w // 16
        self.NT = self.ph * self.pw + 1
        self.NP = (self.NT + 127) // 128 * 128
        self.D, self.H, self.L = cfg["hidden"], cfg["heads"], cfg["layers"] - 1
        self.eng = _engine(sd, cfg, h, w)
        self.table = prepare_dpt_beit(sd, cfg, h, w)[f"l{self.L}.rpb"].copy()
        self.idx = OB.rel_index(self.ph, self.pw).numpy()

    def set_table(self, t):
        t = np.ascontiguousarray(t, np.float32)
        assert t.shape == self.table.shape
        self.eng.check(self.eng.lib.vd3d_depth_set_tensor(self.eng.h, f"l{self.L}.rpb".encode(), t.ctypes.data, t.nbytes))
        self.table = t

    def run(self, B, seed=0):
        rng = np.random.default_rng(seed)
        self.B = B
        self.eng.infer_batch([rng.integers(0, 256, (self.h, self.w, 3), dtype=np.uint8) for _ in range(B)],
                             check_size=False)

    def check(self, what):
        """attn against float64 softmax(q k^T + bias) v; returns (logits without bias, bias) of every image / head."""
        B, H, NT, NP, D = self.B, self.H, self.NT, self.NP, self.D
        q = self.eng.get_buffer("q", (B, H, NP, 64), np.float16)
        k = self.eng.get_buffer("k", (B, H, NP, 64), np.float16)
        vt = self.eng.get_buffer("vt", (B, H, 64, NP), np.float16)
        dev = self.eng.get_buffer("attn", (B * NP, D), np.float16).reshape(B, NP, D)
        ref = np.zeros((B, NT, D))
        slack = np.zeros((B, NT, D))
        out_s, out_b = [], []
        for b in range(B):
            for h in range(H):
                qh, kh = R.f64(q[b, h, :NT]), R.f64(k[b, h, :NT])
                v = R.f64(vt[b, h, :, :NT]).T
                s = qh @ kh.T  # q is stored pre-scaled by 1/8
                bias = self.table[h].astype(np.float64)[self.idx]
                lg = s + bias
                p = np.exp(lg - lg.max(axis=1, keepdims=True))
                p /= p.sum(axis=1, keepdims=True)
                ref[b, :, 64 * h:64 * h + 64] = p @ v
                mag = p @ np.abs(v)
                sabs = float((np.abs(qh) @ np.abs(kh).T).max())
                babs = float(np.abs(bias).max())
                # f16 probabilities, the fp32 logits (QK^T on the tensor core, + bias rounded once) and P V's sums
                rel = (2 * R.F16_EPS + 2 * ACC(64) * sabs + 4 * R.F32_EPS * (sabs + babs)
                       + (NT / 16 + NP / 128 + 8) * 2 * R.F32_EPS)
                slack[b, :, 64 * h:64 * h + 64] = rel * mag + NT * 2.0 ** -32 * float(np.abs(v).max())
                out_s.append(s)
                out_b.append(bias)
        stored_f16(dev[:, :NT], ref, slack, what)
        assert not dev[-1, NT:].any()  # query rows that do not exist are never written
        return out_s, out_b

    def close(self):
        self.eng.close()


GRIDS = [(64, 96), (192, 192), (256, 192), (192, 256), (512, 896)]


@pytest.mark.parametrize("hw", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_attention_bias_against_float64(small, hw):
    """Square and rectangular grids; NT = 25, 145, 193 (one key tile, tails of 17 and 65 keys, a last query block
    of one row) and 1793 (the 1080p processed size: 15 key tiles, 10 query blocks).  The tables differ per head and
    reach +-8: CLS rows and columns take their own entries."""
    sd, cfg = small
    rig = BiasRig(sd, cfg, *hw)
    try:
        rig.run(1, seed=hw[0] + hw[1])
        s, b = rig.check(f"BEiT attention {hw[0]}x{hw[1]} (NT {rig.NT})")
        assert np.abs(b[0]).max() >= 4 and not np.array_equal(b[0], b[1])
    finally:
        rig.close()


def test_attention_bias_dominated_logits_move_the_argmax(small):
    """The table scaled up to a standard deviation of ~11 logits: the bias, not q k^T, picks each row's maximum."""
    sd, cfg = small
    rig = BiasRig(sd, cfg, 256, 192)
    try:
        rig.set_table(rig.table * 8.0)
        rig.run(1, seed=5)
        s, b = rig.check("BEiT attention, bias-dominated logits")
        moved = np.mean([(si.argmax(1) != (si + bi).argmax(1)).mean() for si, bi in zip(s, b)])
        print("rows whose argmax the bias moves", moved)
        assert moved > 0.5
    finally:
        rig.close()


def test_attention_bias_cls_entries_batch_of_three(small):
    """B = 3 images (the image index of grid.y) with distinct tables per head, and the three CLS entries made
    decisive: head 0's CLS column (num - 2) +30 pulls every patch row to the CLS key; head 1's CLS-to-CLS (num - 1)
    +20 over a CLS row (num - 3) of -20 keeps the CLS row on itself; head 2's CLS column -30 shuts the CLS key out."""
    sd, cfg = small
    rig = BiasRig(sd, cfg, 192, 256)
    try:
        t = rig.table.copy()
        n = t.shape[1]
        t[0, n - 2] = 30.0
        t[1, n - 1], t[1, n - 3] = 20.0, -20.0
        t[2, n - 2] = -30.0
        rig.set_table(t)
        rig.run(3, seed=9)
        s, b = rig.check("BEiT attention B=3, decisive CLS entries")
        H = rig.H
        for img in range(3):
            lg = [s[img * H + h] + b[img * H + h] for h in range(H)]
            assert (lg[0][1:].argmax(1) == 0).all()
            assert lg[1][0].argmax() == 0
            assert (lg[2][1:].argmax(1) != 0).all()
    finally:
        rig.close()


# ---------------------------------------------------------------------------------------------------------------------
# the forward against the fp32 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _forward_err(sd, cfg, h, w, seed):
    import torch
    e = _engine(sd, cfg, h, w)
    px = torch.randn(3, h, w, generator=torch.Generator().manual_seed(seed))
    with torch.no_grad():
        ref = OB.forward(sd, cfg, px).numpy()
    out = e.forward(px.numpy())
    e.close()
    err = float(np.abs(out - ref).max() / (ref.max() - ref.min()))
    lsb = int(np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int)).max())
    return err, lsb


@pytest.mark.parametrize("hw", [(64, 64), (64, 96), (128, 192)])
def test_forward_matches_oracle_small(small, hw):
    sd, cfg = small
    err, lsb = _forward_err(sd, cfg, *hw, seed=7)
    print(f"DPT-BEiT small {hw} max-abs error / range {err:.3e}, u8 max diff {lsb}")
    assert err <= 1.5e-3 and lsb <= 1


def test_forward_matches_oracle_large_1080p_size(large):
    """BEiT-L/16 at 512 x 896, the processed size of a 1920 x 1080 frame (1793 tokens)."""
    sd, cfg = large
    err, lsb = _forward_err(sd, cfg, 512, 896, seed=11)
    print(f"DPT-BEiT-L 512x896 max-abs error / range {err:.3e}, u8 max diff {lsb}")
    assert err <= 1.5e-3 and lsb <= 1


def test_batch_of_four_equals_single_forwards(large):
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = large
    e = _engine(sd, cfg, 512, 896)
    frames = [synth_frame(i, 1920, 1080, k)[0] for i, k in ((1, "natural"), (2, "noise"), (3, "smooth"), (4, "natural"))]
    batch = e.infer_batch(frames)
    for f, (d32, d8) in zip(frames, batch):
        s32, s8 = e.infer(f)
        assert np.array_equal(d32, s32) and np.array_equal(d8, s8)
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
# the family's argument checks
# ---------------------------------------------------------------------------------------------------------------------
def test_create_ex_arguments():
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200.depth_engine import DepthConfig, DepthConfigEx, _bind
    lib = _lib.load()
    _bind(lib)
    ctx = _lib.default_context(0)

    def make(size=(512, 896), family=3, patch=16, head=0, fit=None):
        dc = DepthConfig(1024, 24, 16, (C.c_int32 * 4)(6, 12, 18, 24), (C.c_int32 * 4)(256, 512, 1024, 1024), 256,
                         *size)
        dx = DepthConfigEx(dc, family, patch, 1e-12, 3, (C.c_float * 3)(0.5, 0.5, 0.5), (C.c_float * 3)(0.5, 0.5, 0.5),
                           head, 1.0 if head == 0 else 10.0)
        h = C.c_void_p()
        rc = lib.vd3d_depth_create_ex(C.byref(dx), lib.vd3d_stream(ctx.h), C.byref(h))
        if rc == 0 and fit is not None:
            rc = lib.vd3d_depth_set_fit(h, *fit)
        if h.value:
            lib.vd3d_depth_destroy(h)
        return rc
    assert make() == 0 and make((896, 512)) == 0 and make(fit=(512, 512, 32)) == 0 and make(fit=(0, 0, 0)) == 0
    assert make((512, 880)) == -2 and make((496, 896)) == -2     # sides must be multiples of 32
    assert make(patch=14, size=(448, 896)) == -2 and make(head=1) == -2
    assert make(fit=(512, 512, 14)) == -2 and make(fit=(16, 512, 32)) == -2
    assert make((512, 32000)) == -2   # a 63 x 3999 table does not fit the attention's shared memory
    assert make((512, 896), family=1) == -2 and make((384, 384), family=1, fit=(512, 512, 32)) == -2


# ---------------------------------------------------------------------------------------------------------------------
# the drivers with a model written by save_pretrained (BEiT-L: config.json must be the served configuration)
# ---------------------------------------------------------------------------------------------------------------------
PREPROC = dict(do_resize=True, size={"height": 512, "width": 512}, keep_aspect_ratio=True, ensure_multiple_of=32,
               resample=3, do_rescale=True, rescale_factor=1 / 255, do_normalize=True, image_mean=[0.5] * 3,
               image_std=[0.5] * 3, do_pad=False)


class Var:
    def __init__(self, v):
        self.v = v

    def get(self):
        return self.v


@pytest.fixture(scope="module")
def beit(large, tmp_path_factory):
    from visiondepth3d_b200 import render_depth as RD
    sd, _ = large
    root = tmp_path_factory.mktemp("w")
    model = OB.hf_model(sd)
    folder = root / "weights" / "Intel_dpt-beit-large-512"
    model.save_pretrained(str(folder))
    with open(folder / "preprocessor_config.json", "w") as f:
        json.dump(dict(PREPROC, image_processor_type="DPTImageProcessor"), f)
    old = RD.local_model_dir
    RD.local_model_dir = str(root / "weights")
    RD.update_pipeline("dpt-beit-large-512", None, None, None).join()
    yield RD, model, folder
    RD.local_model_dir = old
    RD.USE_TILED_DEPTH = False


def test_update_pipeline_publishes_pipe(beit):
    RD, _, folder = beit
    assert {"model.safetensors", "config.json", "preprocessor_config.json"} <= set(os.listdir(folder))
    assert RD._arch == "dpt-beit-large-512" and RD.pipe is not None and RD.pipe_type == "hf"
    assert RD.model_processed_size(1920, 1080) == (512, 896) and RD.model_processed_size(1080, 1920) == (896, 512)


def test_process_image_matches_transformers_pipeline(beit, tmp_path):
    """A 1920 x 1080 image through process_image against transformers' pipeline("depth-estimation") on the same
    weights and processor on the CPU, then the min-max u8 of convert_depth_to_grayscale."""
    import torch
    from PIL import Image
    from transformers import pipeline
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    from visiondepth3d_b200.synth import synth_frame
    RD, model, _ = beit
    fr, _ = synth_frame(5, 1920, 1080, "natural")
    img = Image.fromarray(fr[..., ::-1].copy())
    src = tmp_path / "in.png"
    img.save(src)
    RD.process_image(str(src), Var("default"), Var(False), Var(str(tmp_path / "o")), Var("Original"), None, None, None,
                     None)
    got = np.array(Image.open(tmp_path / "o" / "in_depth.png"))
    assert got.shape == (1080, 1920)
    proc = DPTImageProcessor(**{k: v for k, v in PREPROC.items()})
    pipe = pipeline("depth-estimation", model=model, image_processor=proc, device="cpu")
    with torch.no_grad():
        d = pipe(img)["predicted_depth"]
    want = RD.convert_depth_to_grayscale(d)
    if want.shape != got.shape:
        want = RD.resize_cubic_u8(want, 1920, 1080)
    diff = np.abs(got.astype(int) - want.astype(int))
    print("process_image vs transformers pipeline: max LSB", int(diff.max()), "share > 0", float((diff > 0).mean()))
    assert diff.max() <= 1


def test_folder_of_mixed_sizes(beit, tmp_path, monkeypatch):
    """Images whose processed sizes differ (16:9, portrait, 2.39:1, square) go through one forward per processed size;
    each output equals the pipe's own depth of that image within 1 LSB."""
    from PIL import Image
    from visiondepth3d_b200.depth_engine import DepthEngine
    RD, _, _ = beit
    src = tmp_path / "in"
    src.mkdir()
    rng = np.random.default_rng(2)
    sizes = [(1280, 720), (720, 1280), (956, 400), (384, 384), (1920, 1080)]
    for k, (w, h) in enumerate(sizes):
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(src / f"im{k}.png")
    calls = []
    orig = DepthEngine.infer_images

    def spy(self, images, *a, **kw):
        calls.append((self.image_h, self.image_w, len(images)))
        return orig(self, images, *a, **kw)
    monkeypatch.setattr(DepthEngine, "infer_images", spy)
    out = tmp_path / "out"
    RD.process_images_in_folder(str(src), 8, str(out), "Original", None, None, None, False)
    assert [RD.model_processed_size(w, h) for w, h in sizes] == [(512, 896), (896, 512), (512, 1216), (512, 512),
                                                                 (512, 896)]
    assert sorted(calls) == sorted([(512, 896, 2), (896, 512, 1), (512, 1216, 1), (512, 512, 1)])
    for k, (w, h) in enumerate(sizes):
        got = np.array(Image.open(out / f"im{k}_depth.png"))
        img = Image.open(src / f"im{k}.png")
        want = RD.convert_depth_to_grayscale(RD.hf_batch_safe_pipe([img])[0]["predicted_depth"])
        assert got.shape == (h, w) and np.abs(got.astype(int) - want.astype(int)).max() <= 1


def test_depth_video_clip(beit, tmp_path):
    import cv2
    from tests import letterbox_oracle as L
    from tests.test_letterbox_cpu import _Cap
    RD, _, _ = beit
    frames = L.track_frames()[:6]
    h, w = frames[0].shape[:2]
    got = list(RD.iter_depth_frames(_Cap(frames, 2), w, h, False, None, batch_size=4))
    assert len(got) == len(frames)
    for f, g in zip(frames, got):
        want = RD.depth_u8_from_frame(f)
        assert np.abs(g.astype(int) - want.astype(int)).max() <= 1
    src = str(tmp_path / "clip.avi")
    wr = cv2.VideoWriter(src, cv2.VideoWriter_fourcc(*"MJPG"), 24.0, (w, h))
    for f in frames:
        wr.write(f)
    wr.release()
    dst = str(tmp_path / "depth.avi")
    assert RD.depth_video_from_video(src, dst) == len(frames)
    cap = cv2.VideoCapture(dst)
    n = 0
    while cap.read()[0]:
        n += 1
    cap.release()
    assert n == len(frames)


def test_tiled_depth_is_refused_before_files_exist(beit, tmp_path):
    RD, _, _ = beit
    RD.USE_TILED_DEPTH = True
    try:
        with pytest.raises(ValueError, match="USE_TILED_DEPTH"):
            RD.depth_video_from_video(str(tmp_path / "missing.mp4"), str(tmp_path / "o.mkv"))
        with pytest.raises(ValueError, match="USE_TILED_DEPTH"):
            RD.process_images_in_folder(str(tmp_path), 2, str(tmp_path / "out"), "Original", None, None, None, False)
        assert os.listdir(tmp_path) == []
    finally:
        RD.USE_TILED_DEPTH = False


def test_clip_depth_and_tiled_depth_refuse_beit(small):
    """The joined depth -> stereo path and the tiled path serve Depth-Anything-V2 engines only: VD3D_ERR_UNSUPPORTED,
    as for DPT-Large."""
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R3
    from visiondepth3d_b200.render_depth import _plan_for
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = small
    e = _engine(sd, cfg, 64, 96)
    w, h = 320, 180
    rp = R3.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, "Half-SBS", 16 / 9, 0.0, 10.0, 9, True, True)
    frames = [synth_frame(i, w, h, "smooth")[0] for i in range(2)]
    outs = [np.empty((h, w, 3), np.uint8) for _ in frames]
    vp = C.c_void_p
    ctx = e.ctx
    assert ctx.lib.vd3d_render_clip_depth(ctx.h, e.h, 2, (vp * 2)(*[f.ctypes.data for f in frames]), h, w,
                                          C.byref(rp), (vp * 2)(*[o.ctypes.data for o in outs]), _lib.MEM_HOST) == -3
    plan = _plan_for(60, 50, 96, 16)
    frame = np.zeros((50, 60, 3), np.uint8)
    u8 = np.empty((50, 60), np.uint8)
    rc = ctx.lib.vd3d_depth_tiled(ctx.h, (vp * 1)(e.h), 1, 1, (vp * 1)(frame.ctypes.data), 50, 60, 96, 16, plan.tiles,
                                  len(plan.rects), plan.weight_ptrs, 0, 50, 60, (vp * 1)(u8.ctypes.data), None, None,
                                  _lib.MEM_HOST)
    assert rc == -3 and b"Depth-Anything-V2" in ctx.lib.vd3d_last_error(ctx.h)
    e.close()
