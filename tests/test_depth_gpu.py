"""GPU: the wgmma GEMM / implicit-GEMM conv kernels and the Depth-Anything-V2 forward
against fp32 references (numpy matmul, torch conv2d, oracle/depth.py).

Tolerances: GEMM/conv operands are f16 (10-bit mantissa) with fp32 accumulation, so unit
kernels are compared with the SAME f16-rounded operands (error = accumulation order only,
<= 2e-3 relative to the result scale); the full forward is gated at <= 1e-3 max-abs on the
depth normalised to [0, 1] (north_star tolerance for float intermediates; asserted as 1e-3 in
test_forward_matches_oracle on a model whose head does not cancel) and <= 1 LSB after
the reference's min-max -> u8 quantisation (core/render_depth.py:605-611)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from visiondepth3d_b200.depth_engine import DepthEngine
    return DepthEngine("vits", 70, 98)


@pytest.mark.parametrize("shape", [(128, 128, 64), (128, 128, 128), (256, 384, 768), (2443, 1152, 384),
                                   (100, 200, 72), (2442, 48 + 16, 384), (300, 32, 576), (129, 130, 8),
                                   (2443, 768, 3072), (2443, 2304, 768)])
def test_gemm_matches_numpy(eng, shape):
    M, N, K = shape
    rng = np.random.default_rng(M * 7 + N)
    A = (rng.standard_normal((M, K)) * 0.5).astype(np.float16)
    B = (rng.standard_normal((N, K)) * 0.5).astype(np.float16)
    ref = A.astype(np.float32) @ B.astype(np.float32).T
    for bn in ((0,) if N < 64 else (0, 64, 32)):
        out = eng.gemm(A, B, bn)
        assert np.abs(out - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), (shape, bn)


@pytest.mark.parametrize("case", [(37, 66, 64, 64, True), (74, 132, 128, 64, True), (19, 33, 64, 128, True),
                                  (148, 264, 64, 64, True), (40, 50, 64, 32, True), (37, 66, 128, 64, False)])
def test_conv_matches_torch(eng, case):
    import torch
    import torch.nn.functional as F
    H, W, cin, cout, k3 = case
    rng = np.random.default_rng(H * W)
    x = (rng.standard_normal((H, W, cin)) * 0.5).astype(np.float16)
    w = (rng.standard_normal((cout, cin, 3, 3) if k3 else (cout, cin, 1, 1)) * 0.1).astype(np.float16)
    b = rng.standard_normal(cout).astype(np.float32)
    xt = torch.from_numpy(x.astype(np.float32)).permute(2, 0, 1)[None]
    ref = F.conv2d(xt, torch.from_numpy(w.astype(np.float32)), torch.from_numpy(b), padding=1 if k3 else 0)
    ref = torch.relu(ref)[0].permute(1, 2, 0).numpy()
    wk = w.transpose(0, 2, 3, 1).reshape(cout, -1)  # [Cout, tap, Cin]
    out = eng.conv(x, wk, b, k3=k3, relu=True)
    assert np.abs(out - ref).max() <= 3e-3 * max(1.0, np.abs(ref).max()), case


def _model(name, head="positive", stress=False):
    """Random-init Depth-Anything-V2 (no checkpoints offline) made to behave like a trained one where it matters
    for a parity gate:
    * head="positive": the DPT head's last 1x1 conv (32 -> 1) gets non-negative weights.  PyTorch's symmetric init
      makes that projection cancel to an output range of ~1e-4 of its terms, so a range-normalised error measures
      the cancellation, not the kernels; trained heads (ReLU features -> positive depth) do not cancel.
    * stress=True: DINOv2-style statistics -- LayerScale spread over two decades, a few "massive activation"
      channels (large LayerNorm gains / fc2 biases / pos-embed offsets), so that f16 operand storage sees values
      far from O(1).
    """
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200.depth_weights import hf_config
    torch.manual_seed(0)
    sd = DepthAnythingForDepthEstimation(hf_config(name)).eval().state_dict()
    g = torch.Generator().manual_seed(1)
    if head == "positive":
        sd["head.conv3.weight"] = sd["head.conv3.weight"].abs() + 0.02
        sd["head.conv3.bias"] = torch.zeros_like(sd["head.conv3.bias"])
    if stress:
        D = sd["backbone.layernorm.weight"].numel()
        hot = torch.randperm(D, generator=g)[:4]
        for k in list(sd):
            if k.endswith("layer_scale1.lambda1") or k.endswith("layer_scale2.lambda1"):
                sd[k] = torch.exp(torch.empty(D).uniform_(-4.6, 0.7, generator=g))      # 0.01 .. 2
            if k.endswith("norm1.weight") or k.endswith("norm2.weight"):
                w = sd[k].clone()
                w[hot] = 8.0
                sd[k] = w
            if k.endswith("mlp.fc2.bias"):
                b = sd[k].clone()
                b[hot] = torch.tensor([60.0, -45.0, 30.0, 80.0])
                sd[k] = b
        pe = sd["backbone.embeddings.position_embeddings"].clone()
        pe[..., hot] += 25.0
        sd["backbone.embeddings.position_embeddings"] = pe
    return sd


def _depth_u8(d):
    """convert_depth_to_grayscale tensor path (core/render_depth.py:605-611)."""
    d = d.astype(np.float32)
    return ((d - d.min()) / (d.max() - d.min() + np.float32(1e-6)) * 255).astype(np.uint8)


@pytest.mark.parametrize("name,h,w", [("vits", 70, 98), ("vits", 518, 924), ("vitb", 518, 924), ("vitl", 518, 924)])
def test_forward_matches_oracle(name, h, w):
    """predicted_depth <= 1e-3 max-abs of its range (north_star) against the fp32 oracle, <= 1 LSB after the
    reference's min-max u8 quantisation; every tap / neck feature / fused map <= 2e-3 of its own max."""
    import torch
    from oracle import depth as OD
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import CONFIGS
    sd = _model(name)
    e = DepthEngine(name, h, w)
    e.load_state_dict(sd)
    torch.manual_seed(2)
    px = torch.randn(3, h, w)
    with torch.no_grad():
        ref = OD.forward(sd, CONFIGS[name], px).numpy()
    out = e.forward(px.numpy())
    scale = float(ref.max() - ref.min())
    assert scale > 1e-2 * float(np.abs(ref).max()), "degenerate test model: output range cancels"
    err = np.abs(out - ref).max() / scale
    assert err <= 1e-3, (name, h, w, err)
    du = np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int))
    assert du.max() <= 1
    e.close()


def test_forward_random_head_u8():
    """The symmetric random head (output range ~1e-4 of its terms): only the u8 handoff is meaningful there."""
    import torch
    from oracle import depth as OD
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import CONFIGS
    sd = _model("vits", head="random")
    e = DepthEngine("vits", 518, 924)
    e.load_state_dict(sd)
    torch.manual_seed(2)
    px = torch.randn(3, 518, 924)
    with torch.no_grad():
        ref = OD.forward(sd, CONFIGS["vits"], px).numpy()
    out = e.forward(px.numpy())
    assert np.abs(out - ref).max() / float(ref.max() - ref.min()) <= 3e-3
    assert np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int)).max() <= 1
    e.close()


@pytest.mark.parametrize("name", ["vits", "vitb"])
def test_forward_outlier_channels_no_f16_overflow(name):
    """DINOv2-like statistics: LayerScale over two decades, four massive-activation channels (|x| ~ 1e2 in the
    residual stream, LayerNorm gain 8).  The f16 operand stores must neither overflow nor lose the gate."""
    import torch
    from oracle import depth as OD
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import CONFIGS
    sd = _model(name, stress=True)
    e = DepthEngine(name, 518, 924)
    e.load_state_dict(sd)
    torch.manual_seed(3)
    px = torch.randn(3, 518, 924)
    with torch.no_grad():
        ref, parts = OD.forward(sd, CONFIGS[name], px, return_parts=True)
    ref = ref.numpy()
    assert float(parts["x"].abs().max()) > 50.0          # the stress really produced outliers
    out = e.forward(px.numpy())
    assert np.isfinite(out).all()
    err = np.abs(out - ref).max() / float(ref.max() - ref.min())
    assert err <= 2e-3, (name, err)   # outlier channels cost f16 mantissa in the neck's inputs; u8 handoff still exact:
    assert np.abs(_depth_u8(out).astype(int) - _depth_u8(ref).astype(int)).max() <= 1
    e.close()


def test_infer_matches_hf_pipeline_stages():
    """frame -> DPT image processor -> forward -> bicubic back -> min-max u8, against the
    transformers processor + the fp32 oracle + F.interpolate (what hf_batch_safe_pipe and
    convert_depth_to_grayscale compute, core/render_depth.py:1113-1119, 605-611)."""
    import torch
    import torch.nn.functional as F
    from PIL import Image
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    from oracle import depth as OD
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import CONFIGS
    from visiondepth3d_b200.synth import synth_frame
    sd = _model("vits")
    e = DepthEngine("vits", 518, 924)
    e.load_state_dict(sd)
    proc = DPTImageProcessor(do_resize=True, size={"height": 518, "width": 518}, keep_aspect_ratio=True,
                             ensure_multiple_of=14, resample=3, do_rescale=True, do_normalize=True,
                             image_mean=[0.485, 0.456, 0.406], image_std=[0.229, 0.224, 0.225], do_pad=False)
    for (w, h, kind) in ((1280, 720, "smooth"), (1920, 1080, "noise")):
        fr, _ = synth_frame(3, w, h, kind)
        pv = proc(images=Image.fromarray(fr[..., ::-1].copy()), return_tensors="pt")["pixel_values"][0]
        assert tuple(pv.shape) == (3, 518, 924)
        # processor parity: our pixel_values (from the engine's "px" buffer) vs HF's
        d32, d8 = e.infer(fr)
        px = e.get_buffer("px", (3, 518, 924), np.float32)
        dpx = np.abs(px - pv.numpy()) * 0.225 * 255  # in u8 LSB of the resized image
        # float weights here vs ATen's int16 fixed-point uint8 path: >99 % identical, rare 1-2 LSB
        assert dpx.max() <= 2.01 and (dpx > 0.5).mean() <= 0.01, (dpx.max(), (dpx > 0.5).mean())
        # forward + bicubic resize to the frame + min-max u8 from OUR pixel_values (the rare 1-2 LSB processor
        # differences above are an input difference, measured separately): north-star gates
        with torch.no_grad():
            ref = OD.forward(sd, CONFIGS["vits"], torch.from_numpy(px.copy()))
            ref = F.interpolate(ref[None, None], size=(h, w), mode="bicubic", align_corners=False)[0, 0].numpy()
        scale = float(ref.max() - ref.min())
        assert np.abs(d32 - ref).max() / scale <= 1e-3
        du = np.abs(d8.astype(int) - _depth_u8(ref).astype(int))
        assert du.max() <= 1, (du.max(), (du > 0).mean())
        # and end to end from HF's pixel_values: bounded by the processor difference
        with torch.no_grad():
            ref2 = OD.forward(sd, CONFIGS["vits"], pv)
            ref2 = F.interpolate(ref2[None, None], size=(h, w), mode="bicubic", align_corners=False)[0, 0].numpy()
        assert np.abs(d32 - ref2).max() / scale <= 2e-2
    e.close()


def test_infer_batch_equals_single_frames():
    """One batched forward (stacked token matrix, attention with grid.y = images * heads) against frame-by-frame
    inference: rows of a GEMM do not depend on the other rows, so the results are the same bits."""
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.synth import synth_frame
    sd = _model("vits")
    e = DepthEngine("vits", 518, 924)
    e.load_state_dict(sd)
    frames = [synth_frame(i, 1280, 720, "natural")[0] for i in range(5)]
    single = [e.infer(f) for f in frames]
    for nb in (2, 3, 5):
        batch = e.infer_batch(frames[:nb])
        for k in range(nb):
            assert np.array_equal(batch[k][1], single[k][1]), (nb, k)
            assert np.abs(batch[k][0] - single[k][0]).max() <= 1e-6 * np.abs(single[k][0]).max(), (nb, k)
    e.close()


def test_clip_depth_pipeline_equals_stagewise():
    """vd3d_render_clip_depth (two depth streams + graphs + in-HBM u8 handoff) must equal
    depth inference followed by vd3d_render_frame with that u8 depth, frame by frame."""
    import ctypes as C
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.synth import synth_frame
    sd = _model("vits")
    w, h = 640, 360
    e = DepthEngine("vits", 364, 644)  # DPT size for a 16:9 frame of height 360: round(360*518/360 ...) -> any /14 size works
    e.load_state_dict(sd)
    rp = R.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, "Half-SBS", 16 / 9, 0.0, 10.0, 9, True, True,
                              zero_parallax_strength=0.01)
    frames = [synth_frame(i, w, h, "smooth")[0] for i in range(11)]   # 3 + 3 + 3 + 2: two engine instances, a tail batch
    ctx = e.ctx
    ctx.reset()
    ref = []
    for f in frames:
        _, d8 = e.infer(f, check_size=False)
        ref.append(R.render_frame(f, d8, rp, ctx=ctx))
    ctx.reset()
    n = len(frames)
    outs = [np.empty_like(ref[0]) for _ in range(n)]
    fp = (C.c_void_p * n)(*[f.ctypes.data for f in frames])
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    ctx.check(ctx.lib.vd3d_render_clip_depth(ctx.h, e.h, n, fp, h, w, C.byref(rp), op, _lib.MEM_HOST))
    for i, (a, b) in enumerate(zip(ref, outs)):
        assert np.array_equal(a, b), i
    e.close()
