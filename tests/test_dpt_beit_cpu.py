"""CPU: pin tests/dpt_beit_oracle.py against the installed transformers DPTForDepthEstimation with a BEiT backbone
(random-init weights, bias tables filled), and the DPT-BEiT weight preparation, config and processor parsing,
checkpoint routing, processed-size rule and refusals of the engine's drivers."""
import json
import os

import numpy as np
import pytest
import torch

from tests import dpt_beit_oracle as OB
from visiondepth3d_b200 import depth_weights as DW


@pytest.fixture(scope="module")
def small():
    sd, cfg = OB.random_model(small=True)
    return sd, cfg, OB.hf_model(sd, small=True)


def _compare(model, sd, cfg, px, tol=1e-4):
    with torch.no_grad():
        out = model(pixel_values=px[None], output_hidden_states=True)
        mine, parts = OB.forward(sd, cfg, px, return_parts=True)
    ref = out.predicted_depth[0]
    assert mine.shape == ref.shape == px.shape[1:]
    scale = float(ref.max() - ref.min())
    assert scale > 0
    err = float((mine - ref).abs().max()) / scale
    print("oracle vs transformers, max-abs / range", tuple(px.shape[1:]), err)
    assert err <= tol
    hs = out.hidden_states  # BeitBackbone's hidden states: the embeddings, then one per layer
    for t, i in zip(parts["taps"], cfg["taps"]):
        assert torch.allclose(t, hs[i], atol=tol * float(hs[i].abs().max()), rtol=0)


def test_oracle_matches_transformers_small_square_at_pretrained_window(small):
    sd, cfg, model = small
    _compare(model, sd, cfg, torch.randn(3, 64, 64, generator=torch.Generator().manual_seed(1)))


@pytest.mark.parametrize("hw", [(64, 96), (96, 64)])
def test_oracle_matches_transformers_small_rectangular(small, hw):
    sd, cfg, model = small
    _compare(model, sd, cfg, torch.randn(3, *hw, generator=torch.Generator().manual_seed(2)))


def test_oracle_matches_transformers_large_512():
    sd, cfg = OB.random_model()
    model = OB.hf_model(sd)
    _compare(model, sd, cfg, torch.randn(3, 512, 512, generator=torch.Generator().manual_seed(3)))


def test_tables_fill_every_layer_and_head(small):
    sd, cfg, _ = small
    tabs = [v for k, v in sd.items() if k.endswith("relative_position_bias_table")]
    assert len(tabs) == cfg["layers"]
    assert all(t.abs().max() >= 8.0 for t in tabs)
    assert not torch.equal(tabs[0], tabs[1]) and not torch.equal(tabs[0][:, 0], tabs[0][:, 1])


@pytest.mark.parametrize("hw", [(64, 64), (64, 96), (96, 64), (32, 128)])
def test_prepared_tables_bit_identical_to_transformers(small, hw):
    """l{i}.rpb gathered with the kernel's index rule equals BeitRelativePositionBias.forward bit for bit, at the
    pretrained window and at resampled ones."""
    sd, cfg, model = small
    ph, pw = hw[0] // 16, hw[1] // 16
    w = DW.prepare_dpt_beit(sd, cfg, *hw)
    idx = OB.rel_index(ph, pw)
    for i, layer in enumerate(model.backbone.encoder.layer):
        with torch.no_grad():
            ref = layer.attention.attention.relative_position_bias((ph, pw))[0]  # [1, heads, N + 1, N + 1]
        t = torch.from_numpy(w[f"l{i}.rpb"])
        assert t.shape == (cfg["heads"], (2 * ph - 1) * (2 * pw - 1) + 3)
        assert torch.equal(t[:, idx], ref), (i, hw)


def test_kernel_index_factorisation():
    """The kernel's A(m) - B(n) (umma_attention.cuh) equals the patch-to-patch index, and stays in [0, num - 4]."""
    for ph, pw in ((4, 4), (3, 7), (32, 56), (1, 5), (6, 1)):
        idx = OB.rel_index(ph, pw)
        p = torch.arange(ph * pw)
        b = p + (p // pw) * (pw - 1)
        bmax = (ph - 1) * (2 * pw - 1) + pw - 1
        fact = (b + bmax)[:, None] - b[None, :]
        assert torch.equal(fact, idx[1:, 1:])
        assert int(fact.min()) == 0 and int(fact.max()) == (2 * ph - 1) * (2 * pw - 1) - 1


def test_prepared_layouts(small):
    sd, cfg, _ = small
    D = cfg["hidden"]
    w = DW.prepare_dpt_beit(sd, cfg, 64, 96)
    assert w["pe.w"].shape == (D, 768) and w["pos"].shape == (4 * 6 + 1, D) and not w["pos"].any()
    a = "backbone.encoder.layer.0.attention.attention."
    assert not w["l0.qkv.b"][D:2 * D].any()  # the key projection has no bias
    assert np.array_equal(w["l0.qkv.b"][:D], sd[a + "query.bias"].numpy())
    assert np.array_equal(w["l0.qkv.b"][2 * D:], sd[a + "value.bias"].numpy())
    assert np.array_equal(w["l2.ls1"], sd["backbone.encoder.layer.2.lambda_1"].numpy())
    assert np.array_equal(w["l3.ls2"], sd["backbone.encoder.layer.3.lambda_2"].numpy())
    assert {f"ro{i}.wt" for i in range(4)} <= set(w) and w["l1.rpb"].dtype == np.float32


def test_no_layer_scale_means_ones():
    from transformers import DPTForDepthEstimation
    cfg = dict(DW.DPT_BEIT_CONFIGS["dpt-beit-large-512"], **OB.SMALL, layer_scale=False)
    sd = DPTForDepthEstimation(DW.hf_dpt_beit_config(**OB.SMALL, layer_scale=False)).state_dict()
    assert not any("lambda" in k for k in sd)
    w = DW.prepare_dpt_beit(sd, cfg, 64, 64)
    assert (w["l0.ls1"] == 1).all() and (w["l3.ls2"] == 1).all()
    cj = DW.hf_dpt_beit_config(**OB.SMALL, layer_scale=False).to_dict()
    assert DW.dpt_beit_config_from_json(cj)["layer_scale"] is False


def test_state_dict_check(small):
    sd, cfg, _ = small
    DW.check_dpt_beit_state_dict(dict(sd, **{"backbone.encoder.layer.0.attention.attention.relative_position_index":
                                             torch.zeros(17, 17, dtype=torch.long),
                                             "backbone.embeddings.mask_token": torch.zeros(1, 1, 256)}), cfg)
    k = "backbone.encoder.layer.1.attention.attention.relative_position_bias.relative_position_bias_table"
    bad = dict(sd)
    del bad[k]
    with pytest.raises(ValueError, match="missing key " + k):
        DW.check_dpt_beit_state_dict(bad, cfg)
    with pytest.raises(ValueError, match=r"expected \(52, 4\)"):
        DW.check_dpt_beit_state_dict(dict(sd, **{k: torch.zeros(40, 4)}), cfg)


def _beit_json():
    return json.loads(json.dumps(DW.hf_dpt_beit_config().to_dict()))


def test_config_from_json_accepts_the_checkpoint_config():
    assert DW.dpt_beit_config_from_json(_beit_json()) == DW.DPT_BEIT_CONFIGS["dpt-beit-large-512"]
    cj = _beit_json()
    del cj["backbone_config"]["out_indices"]
    cj["backbone_config"]["out_features"] = ["stage6", "stage12", "stage18", "stage24"]
    assert DW.dpt_beit_config_from_json(cj)["taps"] == [6, 12, 18, 24]


@pytest.mark.parametrize("field,value", [
    ("backbone_config.use_absolute_position_embeddings", True),
    ("backbone_config.use_shared_relative_position_bias", True),
    ("backbone_config.use_relative_position_bias", False), ("backbone_config.reshape_hidden_states", True),
    ("backbone_config.add_fpn", True), ("backbone_config.patch_size", 14),
    ("backbone_config.num_attention_heads", 8), ("backbone_config.hidden_act", "gelu_new"),
    ("backbone_config.out_indices", [6, 12, 24, 18]), ("backbone_config.out_indices", [6, 12, 18]),
    ("backbone_config.out_indices", [0, 12, 18, 24]), ("readout_type", "ignore"),
    ("reassemble_factors", [1, 1, 1, 0.5]), ("add_projection", True), ("use_batch_norm_in_fusion_residual", True),
    ("use_bias_in_fusion_residual", False), ("head_in_index", 0), ("fusion_hidden_size", 100),
    ("neck_hidden_sizes", [256, 512, 1024])])
def test_config_from_json_refuses(field, value):
    cj = _beit_json()
    d = cj
    keys = field.split(".")
    for k in keys[:-1]:
        d = d[k]
    d[keys[-1]] = value
    with pytest.raises(ValueError, match=keys[-1]):
        DW.dpt_beit_config_from_json(cj)


def test_config_from_json_names_every_refused_field():
    cj = _beit_json()
    cj["backbone_config"]["add_fpn"] = True
    cj["readout_type"] = "add"
    with pytest.raises(ValueError, match="add_fpn.*readout_type"):
        DW.dpt_beit_config_from_json(cj)
    del cj["backbone_config"]["use_relative_position_bias"]  # BeitConfig's default: False
    with pytest.raises(ValueError, match="use_relative_position_bias"):
        DW.dpt_beit_config_from_json(cj)


def test_other_parsers_refuse_beit():
    with pytest.raises(ValueError):
        DW.dpt_config_from_json(_beit_json())
    with pytest.raises(ValueError):
        DW.dpt_hybrid_config_from_json(_beit_json())


SWEEP = [(1920, 1080), (3840, 2160), (1920, 804), (1080, 1920), (1280, 720), (720, 480), (640, 640), (512, 512),
         (4096, 1716), (2560, 1080), (1440, 1080), (768, 1024), (1000, 333), (333, 1000), (300, 200), (7680, 4320)]


@pytest.mark.parametrize("wh", SWEEP, ids=[f"{w}x{h}" for w, h in SWEEP])
def test_processed_size_matches_dpt_image_processor(wh):
    from PIL import Image
    from transformers import DPTImageProcessor
    w, h = wh
    proc = DPTImageProcessor(size={"height": 512, "width": 512}, keep_aspect_ratio=True, ensure_multiple_of=32)
    got = proc(Image.new("RGB", (w, h)), return_tensors="np")["pixel_values"].shape[2:]
    assert DW.dpt_beit_processed_size(w, h) == tuple(got)
    if wh == (1920, 1080):
        assert tuple(got) == (512, 896)


def test_processor_parser():
    pj = dict(do_resize=True, size={"height": 512, "width": 512}, keep_aspect_ratio=True, ensure_multiple_of=32,
              resample=3, do_rescale=True, rescale_factor=1 / 255, do_normalize=True, image_mean=[0.5] * 3,
              image_std=[0.5] * 3, do_pad=False)
    assert DW.dpt_beit_processor_from_json(pj) == DW.DPT_BEIT_PROCESSOR
    fixed = DW.dpt_beit_processor_from_json(dict(pj, keep_aspect_ratio=False, size={"height": 384, "width": 640}))
    assert fixed["keep_aspect"] is False and DW.dpt_beit_processed_size(1920, 1080, fixed) == (384, 640)
    for bad in (dict(ensure_multiple_of=14), dict(keep_aspect_ratio=False, size={"height": 500, "width": 500}),
                dict(do_pad=True), dict(resample=0), dict(rescale_factor=1.0), dict(do_normalize=False)):
        with pytest.raises(ValueError):
            DW.dpt_beit_processor_from_json(dict(pj, **bad))


def test_menu_entry_and_families():
    from visiondepth3d_b200 import render_depth as RD
    assert RD.supported_models["dpt-beit-large-512"] == ("Intel/dpt-beit-large-512", "dpt-beit-large-512")
    assert RD._family_of("dpt-beit-large-512") == "dpt-beit" and RD._dpt_like("dpt-beit-large-512")
    assert "Intel/dpt-beit-large-512" in RD.DPT_BEIT_FILES_REQUIRED
    assert "Intel/dpt-beit-large-512" not in RD.DA_CONFIG_REQUIRED


def _save(folder, sd, config):
    from safetensors.torch import save_file
    os.makedirs(folder, exist_ok=True)
    save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(folder, "model.safetensors"))
    if config is not None:
        with open(os.path.join(folder, "config.json"), "w") as f:
            json.dump(config, f)


def test_checkpoint_routing(small, tmp_path):
    """A state dict with relative_position_bias_table keys goes to DPT-BEiT before the backbone.embeddings.cls_token
    test that sends Depth-Anything state dicts to Depth-Anything; a DA folder still routes to DA."""
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200 import render_depth as RD
    sd, _, _ = small
    assert "backbone.embeddings.cls_token" in sd
    beit = str(tmp_path / "beit")
    _save(beit, sd, _beit_json())
    arch, got = RD.load_checkpoint(os.path.join(beit, "model.safetensors"))
    assert arch == "dpt-beit-large-512" and set(got) == set(sd)
    _save(beit, sd, DW.hf_dpt_beit_config(**OB.SMALL).to_dict())
    with pytest.raises(ValueError, match="does not match the built-in dpt-beit-large-512"):
        RD.load_checkpoint(os.path.join(beit, "model.safetensors"))
    os.remove(os.path.join(beit, "config.json"))
    with pytest.raises(ValueError, match="needs its config.json"):
        RD.load_checkpoint(os.path.join(beit, "model.safetensors"))
    torch.manual_seed(0)
    da = str(tmp_path / "da")
    _save(da, DepthAnythingForDepthEstimation(DW.hf_config("vits")).state_dict(), None)
    assert RD.load_checkpoint(os.path.join(da, "model.safetensors"))[0] == "vits"


def test_required_files_messages(small, tmp_path, monkeypatch, capsys):
    from visiondepth3d_b200 import render_depth as RD
    sd, _, _ = small
    folder = str(tmp_path / "weights" / "Intel_dpt-beit-large-512")
    _save(folder, sd, _beit_json())
    monkeypatch.setattr(RD, "local_model_dir", str(tmp_path / "weights"))
    assert RD.ensure_model_downloaded("Intel/dpt-beit-large-512") == (None, None)
    assert "no preprocessor_config.json" in capsys.readouterr().out
    with open(os.path.join(folder, "preprocessor_config.json"), "w") as f:
        json.dump(dict(size={"height": 512, "width": 512}, keep_aspect_ratio=True, ensure_multiple_of=32,
                       image_mean=[0.5] * 3, image_std=[0.5] * 3), f)
    got, meta = RD.ensure_model_downloaded("Intel/dpt-beit-large-512")
    assert meta["arch"] == "dpt-beit-large-512" and meta["processor"] == DW.DPT_BEIT_PROCESSOR
    os.remove(os.path.join(folder, "config.json"))
    assert RD.ensure_model_downloaded("Intel/dpt-beit-large-512") == (None, None)
    assert "no config.json" in capsys.readouterr().out


def test_tiled_depth_refused_before_any_output(tmp_path, monkeypatch):
    from PIL import Image
    from visiondepth3d_b200 import render_depth as RD
    monkeypatch.setattr(RD, "_arch", "dpt-beit-large-512")
    monkeypatch.setattr(RD, "_state_dict", {})
    monkeypatch.setattr(RD, "USE_TILED_DEPTH", True)
    src = tmp_path / "in.png"
    Image.new("RGB", (64, 48)).save(src)
    out = tmp_path / "out"
    out.mkdir()
    with pytest.raises(ValueError, match="dpt-beit-large-512"):
        RD.process_image(str(src), None, False, str(out), None, None, None, None, None)
    assert not any(out.iterdir())
    with pytest.raises(ValueError, match="USE_TILED_DEPTH"):
        RD.depth_video_from_video(str(tmp_path / "none.mp4"), str(out / "d.mp4"))
    assert not any(out.iterdir())
