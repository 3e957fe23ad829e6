"""CPU: the DPT-Hybrid (MiDaS 3.0) oracle pinned to transformers, the load-time weight standardisation, the SAME pads,
the config.json / state-dict checks, the menu entry and checkpoint loading, and the f16 floors of the engine's
precision policy that the GPU gates rest on."""
import json
import os

import numpy as np
import pytest
import torch

from tests import dpt_hybrid_oracle as OH
from visiondepth3d_b200 import depth_weights as DW


@pytest.fixture(scope="module", autouse=True)
def _no_grad():
    with torch.no_grad():
        yield


@pytest.fixture(scope="module")
def default_model():
    return OH.random_model()


@pytest.mark.parametrize("small", [True, False])
def test_oracle_equals_transformers(small, default_model):
    sd, cfg = OH.random_model(small=True) if small else default_model
    S = cfg["image_size"]
    px = torch.randn(3, S, S, generator=torch.Generator().manual_seed(3))
    m = OH.hf_model(sd, small)
    out = m(pixel_values=px[None], output_hidden_states=True)
    ref = out.predicted_depth[0]
    got, parts = OH.forward(sd, cfg, px, return_parts=True)
    rng = float(ref.max() - ref.min())
    assert float((got - ref).abs().max()) <= 1e-5 * rng
    # the stage maps are the backbone's feature maps; the taps the ViT's hidden states after layers taps[2:]
    bb = m.dpt.embeddings.backbone(px[None]).feature_maps
    for a, b in zip(parts["stages"], bb):
        assert a.shape == b.shape and float((a - b).abs().max()) <= 1e-4 * float(b.abs().max())
    assert [t.shape[1] for t in parts["taps"]] == [(S // 16) ** 2 + 1] * 2
    for t, k in zip(parts["taps"], cfg["taps"][2:]):
        h = out.hidden_states[k]
        assert float((t - h).abs().max()) <= 1e-4 * float(h.abs().max())


def test_weight_standardisation_equals_transformers():
    """prepare_dpt_hybrid's float64 standardisation against WeightStandardizedConv2d's batch_norm, run in float64."""
    import torch.nn.functional as F
    from transformers.models.bit.modeling_bit import WeightStandardizedConv2d
    g = torch.Generator().manual_seed(1)
    for shape in ((64, 3, 7, 7), (256, 64, 1, 1), (128, 128, 3, 3)):
        conv = WeightStandardizedConv2d(shape[1], shape[0], shape[2], eps=1e-8).double()
        conv.weight.data = torch.randn(shape, generator=g, dtype=torch.float64) * 0.05 + 0.01
        hf = F.batch_norm(conv.weight.reshape(1, shape[0], -1), None, None, training=True, momentum=0.0,
                          eps=conv.eps).reshape_as(conv.weight)
        ours = DW.standardize_weight(conv.weight.data)
        assert torch.allclose(ours, hf, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("S", [64, 128, 384, 512])
def test_same_pads(S):
    """The pads the kernels hard-code: stem 2 / 3, max-pool and stride-2 3x3 0 / 1, stride-2 1x1 none, stride-1 3x3
    symmetric 1 -- the TF SAME rule of transformers' DynamicPad2d at every stage size."""
    from transformers.models.bit.modeling_bit import DynamicPad2d
    assert OH.same_pad(S, 7, 2) == (2, 3)
    assert OH.same_pad(S // 2, 3, 2) == (0, 1)
    for s in (S // 4, S // 8):
        assert OH.same_pad(s, 3, 2) == (0, 1)
        assert OH.same_pad(s, 1, 2) == (0, 0)
    x = torch.ones(1, 1, S, S)
    assert DynamicPad2d(7, 2, 1)(x).shape[-1] == S + 5
    assert DynamicPad2d(3, 2, 1)(x[..., : S // 2, : S // 2]).shape[-1] == S // 2 + 1


def _hybrid_json():
    return DW.hf_dpt_hybrid_config().to_dict()


def test_config_from_json_accepts_hybrid():
    assert DW.dpt_hybrid_config_from_json(_hybrid_json()) == DW.DPT_HYBRID_CONFIGS["dpt-hybrid-midas"]
    cj = json.loads(json.dumps(_hybrid_json()))  # through JSON, as read from config.json
    assert DW.dpt_hybrid_config_from_json(cj) == DW.DPT_HYBRID_CONFIGS["dpt-hybrid-midas"]


@pytest.mark.parametrize("field,value", [
    ("backbone_config.layer_type", "preactivation"), ("backbone_config.global_padding", None),
    ("backbone_config.depths", [3, 4, 6]), ("backbone_config.hidden_sizes", [256, 512, 768, 2048]),
    ("backbone_config.num_groups", 16), ("readout_type", "ignore"), ("reassemble_factors", [4, 2, 1, 0.5]),
    ("neck_hidden_sizes", [96, 192, 384, 768]), ("add_projection", True), ("use_batch_norm_in_fusion_residual", True),
    ("is_hybrid", False), ("patch_size", 14), ("backbone_out_indices", [2, 5, 11, 8])])
def test_config_from_json_refuses(field, value):
    cj = _hybrid_json()
    d = cj
    keys = field.split(".")
    for k in keys[:-1]:
        d = d[k]
    d[keys[-1]] = value
    with pytest.raises(ValueError, match=keys[-1]):
        DW.dpt_hybrid_config_from_json(cj)


def test_dpt_config_from_json_still_refuses_hybrid():
    with pytest.raises(ValueError):
        DW.dpt_config_from_json(_hybrid_json())


def test_state_dict_check_names_key(default_model):
    sd, cfg = default_model
    DW.check_dpt_hybrid_state_dict(sd, cfg)
    assert "neck.reassemble_stage.readout_projects.0.0.weight" not in DW.dpt_hybrid_keys(cfg)
    k = "dpt.embeddings.backbone.bit.encoder.stages.1.layers.0.downsample.conv.weight"
    bad = dict(sd)
    del bad[k]
    with pytest.raises(ValueError, match="missing key " + k):
        DW.check_dpt_hybrid_state_dict(bad, cfg)
    bad = dict(sd, **{k: torch.zeros(512, 128, 1, 1)})
    with pytest.raises(ValueError, match=r"has shape \(512, 128, 1, 1\), expected \(512, 256, 1, 1\)"):
        DW.check_dpt_hybrid_state_dict(bad, cfg)


def test_prepared_layouts(default_model):
    sd, cfg = default_model
    w = DW.prepare_dpt_hybrid(sd, cfg, 384, 384)
    assert w["bit.stem.w"].shape == (64, 147) and w["bit.stem.w"].dtype == np.float32
    assert w["bit.s1.b0.c2.w"].shape == (128, 9 * 128) and w["bit.s1.b0.c2.w"].dtype == np.float16
    assert w["bit.s2.b8.c3.w"].shape == (1024, 256) and "bit.s2.b1.ds.w" not in w
    assert w["pe.w"].shape == (768, 1024) and w["pos"].shape == (577, 768)
    assert {"ro2.wt", "ro3.wt"} <= set(w) and "ro0.wt" not in w and "r0.proj.w" not in w
    assert w["n0.conv.w"].shape == (256, 9 * 256) and w["n1.conv.w"].shape == (256, 9 * 512)
    # tap-major conv2: column tap * C + c
    c2 = DW.standardize_weight(sd[OH.BIT + "encoder.stages.0.layers.1.conv2.weight"])
    assert np.array_equal(w["bit.s0.b1.c2.w"].reshape(64, 9, 64)[:, 4, :],
                          c2[:, :, 1, 1].float().numpy().astype(np.float16))


def test_menu_entry():
    from visiondepth3d_b200 import render_depth as RD
    assert RD.supported_models["MiDaS 3.0"] == ("Intel/dpt-hybrid-midas", "dpt-hybrid-midas")
    assert "Intel/dpt-hybrid-midas" not in RD.DA_CONFIG_REQUIRED
    assert RD._family_of("dpt-hybrid-midas") == "dpt-hybrid"


def test_load_checkpoint_from_saved_folder(default_model, tmp_path, monkeypatch, capsys):
    from visiondepth3d_b200 import render_depth as RD
    sd, _ = default_model
    folder = tmp_path / "weights" / "Intel_dpt-hybrid-midas"
    OH.hf_model(sd).save_pretrained(str(folder))
    arch, got = RD.load_checkpoint(str(folder / "model.safetensors"))
    assert arch == "dpt-hybrid-midas" and set(got) == set(sd)
    monkeypatch.setattr(RD, "local_model_dir", str(tmp_path / "weights"))
    sdl, meta = RD.ensure_model_downloaded("Intel/dpt-hybrid-midas")
    assert meta["arch"] == "dpt-hybrid-midas" and meta["processor"] == RD.DPT_PROCESSOR
    # without config.json: refused (the backbone is described only there)
    os.remove(folder / "config.json")
    assert RD.ensure_model_downloaded("Intel/dpt-hybrid-midas") == (None, None)
    assert "config.json" in capsys.readouterr().out
    with pytest.raises(ValueError, match="config.json"):
        RD.load_checkpoint(str(folder / "model.safetensors"))


@pytest.mark.parametrize("gamma3,gate", [(0.25, 1.5e-3), (1.0, 5e-3)])
def test_f16_emulation_floor(gamma3, gate):
    """The engine's storage precision emulated on the oracle (f16 backbone conv operands and block outputs, f16 ViT,
    projection, neck and head weights; the stem conv in f32): the error it alone causes stays well inside the GPU
    gates.  Measured: 1.03e-3 (gamma3 0.25) and 2.65e-3 (gamma3 1) of the depth range."""
    sd, cfg = OH.random_model(gamma3=gamma3)
    px = torch.randn(3, 384, 384, generator=torch.Generator().manual_seed(3))
    ref = OH.forward(sd, cfg, px)
    em = OH.forward(sd, cfg, px, emulate=True)
    err = float((em - ref).abs().max() / (ref.max() - ref.min()))
    print("f16 emulation floor, gamma3", gamma3, err)
    assert err <= 0.8 * gate
