"""CPU: pin tests/dpt_oracle.py against the installed transformers DPTForDepthEstimation (random-init weights), and
the DPT weight preparation, checkpoint checks and processed-size rule of the engine."""
import numpy as np
import pytest
import torch

from tests import dpt_oracle as OD
from visiondepth3d_b200 import depth_weights as DW


def _compare(model, sd, cfg, px):
    with torch.no_grad():
        out = model(pixel_values=px[None], output_hidden_states=True)
        mine, parts = OD.forward(sd, cfg, px, return_parts=True)
    ref = out.predicted_depth[0]
    assert mine.shape == ref.shape
    scale = float(ref.max() - ref.min())
    assert scale > 0
    assert float((mine - ref).abs().max()) / scale <= 1e-4
    # per stage: the taps are hidden_states[1:] at backbone_out_indices, raw (no final LayerNorm)
    hs = out.hidden_states
    for t, i in zip(parts["taps"], cfg["taps"]):
        assert torch.allclose(t, hs[i], atol=1e-4 * float(hs[i].abs().max()), rtol=0)
    with torch.no_grad():
        feats = model.neck.reassemble_stage([hs[i] for i in cfg["taps"]])
        necks = [model.neck.convs[i](f) for i, f in enumerate(feats)]
        fused = model.neck.fusion_stage(necks)
    for a, b in zip(parts["feats"], necks):
        assert float((a - b).abs().max()) <= 1e-4 * float(b.abs().max())
    for a, b in zip(parts["fused"], fused):
        assert float((a - b).abs().max()) <= 1e-4 * float(b.abs().max())
    # the readout output is the input of the reassemble projection
    with torch.no_grad():
        for i, ro in enumerate(parts["readouts"]):
            g = int(round(ro.shape[0] ** 0.5))
            m = ro.reshape(1, g, g, -1).permute(0, 3, 1, 2)
            assert torch.allclose(model.neck.reassemble_stage.layers[i](m), feats[i], atol=1e-4 * float(feats[i].abs().max()))


def test_oracle_matches_transformers_dpt_large_384():
    from transformers import DPTForDepthEstimation
    sd, cfg = OD.random_model()
    model = DPTForDepthEstimation(DW.hf_dpt_config()).eval()
    model.load_state_dict(sd)
    torch.manual_seed(1)
    _compare(model, sd, cfg, torch.randn(3, 384, 384))


@pytest.mark.parametrize("side", [64, 128])
def test_oracle_matches_transformers_small_config(side):
    from transformers import DPTForDepthEstimation
    sd, cfg = OD.random_model(small=True)
    model = DPTForDepthEstimation(DW.hf_dpt_config("dpt-large", **OD.SMALL)).eval()
    model.load_state_dict(sd)
    torch.manual_seed(2)
    _compare(model, sd, cfg, torch.randn(3, side, side))


def test_hf_dpt_config_equals_dpt_large():
    c = DW.hf_dpt_config()
    assert (c.hidden_size, c.num_hidden_layers, c.num_attention_heads, c.intermediate_size) == (1024, 24, 16, 4096)
    assert list(c.backbone_out_indices) == [5, 11, 17, 23] and list(c.neck_hidden_sizes) == [256, 512, 1024, 1024]
    assert (c.patch_size, c.image_size, c.layer_norm_eps, c.readout_type) == (16, 384, 1e-12, "project")
    assert DW.dpt_config_from_json(c.to_dict()) == DW.DPT_CONFIGS["dpt-large"]


def test_prepare_dpt_shapes_and_keys():
    sd, cfg = OD.random_model(small=True)
    w = DW.prepare_dpt(sd, cfg, 128, 128)
    D = cfg["hidden"]
    assert w["pe.w"].shape == (D, 768) and w["pe.w"].dtype == np.float16
    assert w["pos"].shape == (8 * 8 + 1, D)
    assert w["l0.qkv.w"].shape == (3 * D, D) and (w["l0.ls1"] == 1).all() and (w["l3.ls2"] == 1).all()
    assert w["ro0.wt"].shape == (D, D) and w["ro0.wc"].shape == (D, D) and w["ro3.b"].shape == (D,)
    W0 = sd["neck.reassemble_stage.readout_projects.0.0.weight"].numpy().astype(np.float16)
    assert (w["ro0.wt"] == W0[:, :D]).all() and (w["ro0.wc"] == W0[:, D:]).all()
    assert w["r0.proj.w"].shape == (64, D) and w["r0.up.w"].shape == (16 * 64, 64) and w["r3.down.w"].shape == (256, 9 * 256)
    assert w["h.c1.w"].shape == (64, 9 * 64) and w["h.c2.w"].shape == (32, 9 * 64) and w["h.c3.w"].shape == (32,)
    assert "norm.g" not in w and "f0.rl2.c1.w" in w
    # position embeddings at the checkpoint's own grid are the checkpoint's (bilinear resize is the identity)
    w64 = DW.prepare_dpt(sd, cfg, 64, 64)
    assert np.array_equal(w64["pos"], sd["dpt.embeddings.position_embeddings"][0].numpy())


def test_prepare_dpt_names_missing_and_misshaped_keys():
    sd, cfg = OD.random_model(small=True)
    needed = DW.dpt_keys(cfg)
    unused = [k for k in sd if k not in needed]
    assert set(unused) == {"dpt.layernorm.weight", "dpt.layernorm.bias"} | {
        k for k in sd if k.startswith("neck.fusion_stage.layers.0.residual_layer1.")}
    extra = dict(sd)
    extra["dpt.pooler.dense.weight"] = torch.zeros(4, 4)
    del extra["dpt.layernorm.weight"]
    DW.prepare_dpt(extra, cfg, 64, 64)  # unused keys are accepted either way
    for k in ("dpt.encoder.layer.2.output.dense.bias", "neck.reassemble_stage.readout_projects.1.0.weight",
              "head.head.4.weight"):
        bad = dict(sd)
        del bad[k]
        with pytest.raises(ValueError, match="missing key " + k.replace(".", r"\.")):
            DW.prepare_dpt(bad, cfg, 64, 64)
    bad = dict(sd)
    bad["neck.convs.2.weight"] = torch.zeros(64, 128, 3, 3)
    with pytest.raises(ValueError, match=r"neck\.convs\.2\.weight has shape"):
        DW.prepare_dpt(bad, cfg, 64, 64)


@pytest.mark.parametrize("resample", [2, 3])
def test_processed_size_agrees_with_dpt_image_processor(resample):
    from PIL import Image
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    p = DW.dpt_processor_from_json(DPTImageProcessor(resample=resample).to_dict())
    assert p["resample"] == resample and p["mean"] == (0.5,) * 3 and p["std"] == (0.5,) * 3
    proc = DPTImageProcessor(resample=resample)
    rng = np.random.default_rng(0)
    for w, h in ((1280, 720), (1920, 1080), (641, 359), (333, 500), (384, 384), (97, 1001)):
        img = Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        pv = proc(images=img, return_tensors="pt")["pixel_values"]
        assert tuple(pv.shape[2:]) == DW.dpt_processed_size(p)


def test_unserved_dpt_configurations_are_refused():
    base = dict(DW.DPT_PROCESSOR)
    for size in ((384, 512), (400, 400), (360, 360)):
        with pytest.raises(ValueError, match="square"):
            DW.dpt_processed_size(dict(base, size=size))
    assert DW.dpt_processed_size(dict(base, size=(512, 512))) == (512, 512)
    for pj in ({"keep_aspect_ratio": True}, {"ensure_multiple_of": 32}, {"resample": 1}, {"resample": 0},
               {"do_pad": True}, {"do_normalize": False}):
        with pytest.raises(ValueError):
            DW.dpt_processor_from_json(pj)
    c = DW.hf_dpt_config().to_dict()
    for k, v in (("readout_type", "add"), ("is_hybrid", True), ("add_projection", True),
                 ("reassemble_factors", [4, 2, 1, 1])):
        with pytest.raises(ValueError):
            DW.dpt_config_from_json(dict(c, **{k: v}))
