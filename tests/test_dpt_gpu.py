"""GPU: DPT-Large on the depth engine -- the forward against tests/dpt_oracle.py (fp32), the readout GEMM and the
un-normalised tap copy against float64 on the engine's own buffers, processor parity with DPTImageProcessor, and the
image / video drivers of render_depth with a DPT model."""
import json
import os

import numpy as np
import pytest

from tests import dpt_oracle as OD

pytestmark = pytest.mark.gpu


def _depth_u8(d):
    d = d.astype(np.float32)
    return ((d - d.min()) / (d.max() - d.min() + np.float32(1e-6)) * 255).astype(np.uint8)


def _engine(sd, cfg, processor=None):
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine(cfg, family="dpt", processor=processor)
    e.load_state_dict(sd)
    return e


@pytest.fixture(scope="module")
def large():
    return OD.random_model()


def _f16(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float64)


def test_forward_matches_oracle_b1(large):
    import torch
    sd, cfg = large
    e = _engine(sd, cfg)
    assert (e.image_h, e.image_w) == (384, 384)
    torch.manual_seed(3)
    px = torch.randn(3, 384, 384)
    with torch.no_grad():
        ref = OD.forward(sd, cfg, px).numpy()
    out = e.forward(px.numpy())
    err = np.abs(out - ref).max() / float(ref.max() - ref.min())
    print("DPT-Large B=1 max-abs error / range", err)
    # f16 storage of the weights and pixels alone moves this random-init model's depth by 7.2e-4 of its range (spread
    # over every stage, computed on the CPU with the oracle); the engine's f16 activations add the rest
    assert err <= 1.5e-3, err
    assert np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int)).max() <= 1
    e.close()


def test_batch_of_four_equals_single_forwards(large):
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = large
    e = _engine(sd, cfg)
    frames = [synth_frame(i, 640, 360, k)[0] for i, k in ((1, "natural"), (2, "noise"), (3, "smooth"), (4, "natural"))]
    batch = e.infer_batch(frames)
    for f, (d32, d8) in zip(frames, batch):
        s32, s8 = e.infer(f)
        assert np.array_equal(d32, s32) and np.array_equal(d8, s8)
    e.close()


def test_forward_massive_activation_channels(large):
    """Four channels of the residual stream at |x| ~ 1e2 .. 1e3: the taps are not normalised, so they reach the
    readout GEMM's f16 operand as they are."""
    import torch
    sd, cfg = OD.random_model(stress=True)
    e = _engine(sd, cfg)
    torch.manual_seed(4)
    px = torch.randn(3, 384, 384)
    with torch.no_grad():
        ref, parts = OD.forward(sd, cfg, px, return_parts=True)
    ref = ref.numpy()
    assert float(max(t.abs().max() for t in parts["taps"])) > 100.0
    out = e.forward(px.numpy())
    assert np.isfinite(out).all()
    err = np.abs(out - ref).max() / float(ref.max() - ref.min())
    print("DPT-Large stress max-abs error / range", err)
    assert err <= 2e-3, err
    assert np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int)).max() <= 1
    e.close()


@pytest.mark.parametrize("stress", [False, True])
def test_readout_and_tap_copy_against_float64(stress):
    """After a forward: the last tap (taken after the last layer, so the final residual stream "x" is its source)
    is f16(x) row for row; the CLS term c = Wc cls + b and the readout GELU(Wt tok + c) against float64 on the f16
    operands the engine stored, within half an f16 ulp plus the fp32 accumulation."""
    import torch
    from visiondepth3d_b200.depth_weights import prepare_dpt
    sd, cfg = OD.random_model(small=True, stress=stress)
    e = _engine(sd, cfg, processor=dict(size=(128, 128), resample=3, mean=(0.5,) * 3, std=(0.5,) * 3))
    torch.manual_seed(5)
    e.forward(torch.randn(3, 128, 128).numpy())
    D, N = cfg["hidden"], 8 * 8
    w = prepare_dpt(sd, cfg, 128, 128)
    x = e.get_buffer("x", (N + 1, D), np.float32).astype(np.float64)
    tap = e.get_buffer("tap3", (N, D), np.float16).astype(np.float64)
    assert np.array_equal(tap, _f16(np.clip(x[1:], -65504, 65504)))
    if stress:
        assert np.abs(x).max() > 100.0
    wc, wt, b = (w["ro3.wc"].astype(np.float64), w["ro3.wt"].astype(np.float64), w["ro3.b"].astype(np.float64))
    c = e.get_buffer("ro3.c", (1, D), np.float32).astype(np.float64)[0]
    c_ref = wc @ x[0] + b
    eps32 = 2.0 ** -24
    assert (np.abs(c - c_ref) <= 2 * D * eps32 * (np.abs(wc) @ np.abs(x[0]) + np.abs(b)) + 1e-30).all()
    ro = e.get_buffer("ro3", (N, D), np.float16).astype(np.float64)
    from scipy.special import erf
    pre = tap @ wt.T + c[None, :]
    ref = 0.5 * pre * (1 + erf(pre / np.sqrt(2)))
    acc = 2 * D * eps32 * (np.abs(tap) @ np.abs(wt).T + np.abs(c)[None, :])  # fp32 accumulation, GELU slope <= 1.13
    tol = 1.13 * acc + 2.0 ** -11 * np.abs(ref) + 2.0 ** -25 + 1e-6 * np.abs(pre)
    assert (np.abs(ro - ref) <= tol).all(), float((np.abs(ro - ref) / tol).max())
    e.close()


@pytest.mark.parametrize("resample", [3, 2])
def test_processor_parity_with_dpt_image_processor(large, resample):
    from PIL import Image
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    from visiondepth3d_b200.depth_weights import dpt_processor_from_json
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = large
    proc = DPTImageProcessor(resample=resample)
    e = _engine(sd, cfg, processor=dpt_processor_from_json(proc.to_dict()))
    for (w, h, kind) in ((1280, 720, "smooth"), (1920, 1080, "noise")):
        fr, _ = synth_frame(3, w, h, kind)
        pv = proc(images=Image.fromarray(fr[..., ::-1].copy()), return_tensors="pt")["pixel_values"][0].numpy()
        e.infer(fr)
        px = e.get_buffer("px", (3, 384, 384), np.float32)
        dpx = np.abs(px - pv) * 0.5 * 255  # in u8 LSB of the resized image
        # float weights here vs ATen's fixed-point uint8 path.  At DPT's 3.3x / 5x shrink of a smooth gradient the
        # fixed-point sums round up where the float ones round down on ~6 % of the pixels (1 LSB, one direction;
        # H100: 5.0 % bicubic, 5.9 % bilinear); on textured frames below 1 %, as for Depth-Anything's processor
        share = 0.07 if kind == "smooth" else 0.01
        assert dpx.max() <= 2.01 and (dpx > 0.5).mean() <= share, (w, kind, dpx.max(), (dpx > 0.5).mean())
    e.close()


@pytest.fixture(scope="module")
def dpt_model(large):
    from visiondepth3d_b200 import render_depth as RD
    sd, _ = large
    RD.load_depth_model("dpt-large", sd, 320, 180)
    yield RD
    RD.USE_TILED_DEPTH = False


def test_update_pipeline_from_saved_folder(large, tmp_path, monkeypatch):
    import torch
    from PIL import Image
    from transformers import DPTForDepthEstimation
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    from visiondepth3d_b200 import render_depth as RD
    from visiondepth3d_b200.depth_weights import hf_dpt_config
    sd, _ = large
    model = DPTForDepthEstimation(hf_dpt_config()).eval()
    model.load_state_dict(sd)
    folder = tmp_path / "weights" / "Intel_dpt-large"
    model.save_pretrained(str(folder))
    DPTImageProcessor(resample=2).save_pretrained(str(folder))
    assert {"model.safetensors", "config.json", "preprocessor_config.json"} <= set(os.listdir(folder))
    monkeypatch.setattr(RD, "local_model_dir", str(tmp_path / "weights"))
    RD.update_pipeline("DPT-Large", None, None, None).join()
    assert RD._arch == "dpt-large" and RD._processor["resample"] == 2
    img = Image.fromarray(np.random.default_rng(1).integers(0, 256, (300, 500, 3), dtype=np.uint8))
    got = RD.pipe([img])[0]["predicted_depth"].numpy()
    RD.load_depth_model("dpt-large", sd, 384, 384, processor=dict(RD.DPT_PROCESSOR, resample=2))
    want = RD.pipe([img])[0]["predicted_depth"].numpy()
    assert np.array_equal(got, want)
    # a config.json of another architecture is refused, before anything is loaded
    cj = json.load(open(folder / "config.json"))
    cj["num_hidden_layers"] = 12
    json.dump(cj, open(folder / "config.json", "w"))
    assert RD.ensure_model_downloaded("Intel/dpt-large") == (None, None)


def test_folder_of_mixed_sizes_runs_one_forward(dpt_model, tmp_path, monkeypatch):
    from PIL import Image
    from visiondepth3d_b200.depth_engine import DepthEngine
    RD = dpt_model
    src = tmp_path / "in"
    src.mkdir()
    rng = np.random.default_rng(2)
    sizes = [(640, 360), (333, 500), (384, 384), (1021, 767)]
    for k, (w, h) in enumerate(sizes):
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(src / f"im{k}.png")
    calls = []
    orig = DepthEngine.infer_images

    def spy(self, images, *a, **kw):
        calls.append(len(images))
        return orig(self, images, *a, **kw)
    monkeypatch.setattr(DepthEngine, "infer_images", spy)
    out = tmp_path / "out"
    RD.process_images_in_folder(str(src), 8, str(out), "Original", None, None, None, False)
    assert calls == [len(sizes)]
    for k, (w, h) in enumerate(sizes):
        got = np.array(Image.open(out / f"im{k}_depth.png"))
        img = Image.open(src / f"im{k}.png")
        want = RD.convert_depth_to_grayscale(RD.hf_batch_safe_pipe([img])[0]["predicted_depth"])
        assert got.shape == (h, w) and np.abs(got.astype(int) - want.astype(int)).max() <= 1


def test_tiled_depth_is_refused_before_files_exist(dpt_model, tmp_path):
    RD = dpt_model
    RD.USE_TILED_DEPTH = True
    try:
        with pytest.raises(ValueError, match="USE_TILED_DEPTH"):
            RD.depth_video_from_video(str(tmp_path / "missing.mp4"), str(tmp_path / "o.mkv"))
        with pytest.raises(ValueError, match="USE_TILED_DEPTH"):
            RD.process_images_in_folder(str(tmp_path), 2, str(tmp_path / "out"), "Original", None, None, None, False)
        assert os.listdir(tmp_path) == []
    finally:
        RD.USE_TILED_DEPTH = False


class _Bars:
    def __init__(self, bars):
        self.bars = bars

    def update_batch(self, frames, first_idx=0):
        return [self.bars] * len(frames)


@pytest.mark.parametrize("inf,bars,invert", [(None, None, False), (None, (12, 10), True), ((224, 126), None, True),
                                             ((448, 252), (12, 10), False)])
def test_depth_frames_equal_host_composition(dpt_model, inf, bars, invert):
    from PIL import Image
    from tests import letterbox_oracle as L
    from tests.test_letterbox_cpu import _Cap
    RD = dpt_model
    frames = L.track_frames()[:10]
    got = list(RD.iter_depth_frames(_Cap(frames, 2), 320, 180, invert, inf, batch_size=4,
                                    tracker=_Bars(bars) if bars else None))
    assert len(got) == len(frames)
    for f, g in zip(frames, got):
        d = RD.hf_batch_safe_pipe([Image.fromarray(f[..., ::-1].copy())], inf)[0]["predicted_depth"]
        want = RD.convert_depth_to_grayscale(d)
        if invert:
            want = 255 - want
        want = RD.resize_cubic_u8(want, 320, 180)
        if bars:
            want = RD.letterbox_repad(want, *bars)
        assert np.abs(g.astype(int) - want.astype(int)).max() <= 1
