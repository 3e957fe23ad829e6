"""ZoeDepth on the CPU: the fp32 oracle (tests/zoedepth_oracle.py) against transformers' ZoeDepthForDepthEstimation
and ZoeDepthImageProcessor, the quirks of transformers' head the engine reproduces, the config / processor parsers and
their refusals, the weight packing, and load_checkpoint's routing."""
import json

import numpy as np
import pytest
import torch

from tests import zoedepth_oracle as ZO
from visiondepth3d_b200 import depth_weights as DW


def _force_route(sd, route, margin=50.0):
    sd = dict(sd)
    b = torch.zeros(2)
    b[route] = margin
    sd[ZO.M + "mlp_classifier.linear2.bias"] = b
    return sd


@pytest.mark.parametrize("multi,route,hw", [(True, None, (64, 96)), (True, 0, (96, 64)), (True, 1, (64, 64)),
                                            (False, None, (64, 128))])
def test_oracle_matches_transformers(multi, route, hw):
    sd, cfg = ZO.random_model(multi=multi)
    if route is not None:
        sd = _force_route(sd, route)
    m = ZO.hf_model(sd, "zoedepth-nyu-kitti" if multi else "zoedepth-nyu")
    torch.manual_seed(3)
    px = torch.randn(3, *hw)
    with torch.no_grad():
        out = m(pixel_values=px[None])
        ref = out.predicted_depth[0]
        d, parts = ZO.forward(sd, cfg, px, return_parts=True)
    if route is not None:
        assert parts["route"] == route
        assert int(torch.argmax(out.domain_logits.sum(0))) == route
    err = float((d - ref).abs().max() / (ref.max() - ref.min()))
    assert err < 1e-5, err
    assert float(ref.max() - ref.min()) > 1e-3


@pytest.mark.parametrize("w,h", [(1920, 1080), (1080, 1920), (641, 479), (16, 16), (333, 97)])
def test_processor_matches_transformers(w, h):
    from transformers import ZoeDepthImageProcessor
    proc = ZoeDepthImageProcessor(ensure_multiple_of=32, keep_aspect_ratio=True, size={"height": 384, "width": 512})
    rng = np.random.default_rng(w * 7 + h)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    ref = proc(images=img, return_tensors="pt")["pixel_values"][0]
    out = ZO.processor(img)
    assert tuple(out.shape) == tuple(ref.shape)
    assert tuple(ref.shape[1:]) == DW.zoedepth_processed_size(w, h) == ZO.processed_size(w, h)
    assert float((out - ref).abs().max()) < 1e-5


def test_processed_sizes_of_the_issue():
    assert DW.zoedepth_processed_size(1920, 1080) == (384, 672)
    assert DW.zoedepth_processed_size(1080, 1920) == (896, 512)
    assert (DW.zoedepth_pad(1080), DW.zoedepth_pad(1920)) == (69, 92)


def test_post_process_matches_transformers():
    from transformers import ZoeDepthImageProcessor
    from transformers.models.zoedepth.modeling_zoedepth import ZoeDepthDepthEstimatorOutput
    proc = ZoeDepthImageProcessor()
    torch.manual_seed(0)
    d = torch.rand(384, 672) * 10
    ref = proc.post_process_depth_estimation(ZoeDepthDepthEstimatorOutput(predicted_depth=d[None]),
                                             source_sizes=[(1080, 1920)])[0]["predicted_depth"]
    out = ZO.post_process(d, (1080, 1920))
    assert out.shape == ref.shape == (1080, 1920)
    assert float((out - ref).abs().max()) < 1e-5


def test_quirks_of_the_head():
    """inv_attractor runs with 300 / 2 whatever attractor_alpha / _gamma say; the two-configuration head has 16
    attractors per layer (num_attractors lands in the unused n_bins); the unnormed layer adds no 1e-3, sorts nothing and
    clips nothing."""
    from transformers.models.zoedepth.modeling_zoedepth import ZoeDepthAttractorLayerUnnormed
    sd, cfg = ZO.random_model(multi=True)
    assert DW.zoedepth_attractors(sd, cfg) == [16, 16, 16, 16]
    sd1, cfg1 = ZO.random_model(multi=False)
    assert DW.zoedepth_attractors(sd1, cfg1) == [16, 8, 4, 1]
    hc = DW.hf_zoedepth_config("zoedepth-nyu-kitti", **ZO.SMALL)
    assert hc.attractor_alpha == 1000
    layer = ZoeDepthAttractorLayerUnnormed(hc, n_bins=64, n_attractors=4).eval()
    torch.manual_seed(1)
    x = torch.randn(1, 128, 3, 5)
    prev = torch.rand(1, 64, 2, 3) * 5 - 1  # negative and unsorted bins stay so
    with torch.no_grad():
        got, _ = layer(x, prev, None, interpolate=True)
        a = torch.nn.functional.softplus(layer.conv2(torch.relu(layer.conv1(x))))
    ref = ZO.attractor(a, prev, 4)
    assert torch.equal(got, ref)
    assert float(got.min()) < 0


def test_config_and_processor_from_json_roundtrip():
    hc = DW.hf_zoedepth_config("zoedepth-nyu-kitti")
    cfg = DW.zoedepth_config_from_json(json.loads(hc.to_json_string()))
    want = DW.ZOEDEPTH_CONFIGS["zoedepth-nyu-kitti"]
    for k in ("hidden", "layers", "heads", "taps", "neck", "fusion", "patch", "image_size", "attractors", "bottleneck"):
        assert cfg[k] == want[k], k
    assert [b["max_depth"] for b in cfg["bins"]] == [10.0, 80.0]
    pj = dict(do_resize=True, do_rescale=True, do_normalize=True, do_pad=True, keep_aspect_ratio=True,
              ensure_multiple_of=32, size={"height": 384, "width": 512}, resample=2, image_mean=[0.5] * 3,
              image_std=[0.5] * 3, rescale_factor=1 / 255)
    assert DW.zoedepth_processor_from_json(pj) == DW.ZOEDEPTH_PROCESSOR


@pytest.mark.parametrize("field,value", [("bin_centers_type", "normed"), ("attractor_kind", "sum"),
                                         ("add_projection", True), ("use_batch_norm_in_fusion_residual", True),
                                         ("bin_configurations", [{"n_bins": 64, "min_depth": 0.1, "max_depth": 1}] * 3),
                                         ("num_relative_features", 16), ("bin_embedding_dim", 64)])
def test_config_refusals_name_the_field(field, value):
    cj = json.loads(DW.hf_zoedepth_config("zoedepth-nyu-kitti").to_json_string())
    cj[field] = value
    with pytest.raises(ValueError, match=field):
        DW.zoedepth_config_from_json(cj)


def test_config_refuses_a_non_beit_backbone():
    cj = json.loads(DW.hf_zoedepth_config("zoedepth-nyu-kitti").to_json_string())
    cj["backbone_config"]["model_type"] = "dinov2"
    with pytest.raises(ValueError, match="BEiT"):
        DW.zoedepth_config_from_json(cj)


@pytest.mark.parametrize("field,value", [("ensure_multiple_of", 1 / 32), ("do_pad", False), ("resample", 3),
                                         ("keep_aspect_ratio", False)])
def test_processor_refusals_name_the_field(field, value):
    pj = dict(do_resize=True, do_rescale=True, do_normalize=True, do_pad=True, keep_aspect_ratio=True,
              ensure_multiple_of=32, size={"height": 384, "width": 512}, resample=2)
    pj[field] = value
    with pytest.raises(ValueError, match=field):
        DW.zoedepth_processor_from_json(pj)


def test_state_dict_check_and_packing():
    sd, cfg = ZO.random_model(multi=True)
    out = DW.prepare_zoedepth(sd, cfg, 64, 96)
    assert out["z.s2.w"].shape == (128, 128) and not out["z.s2.w"][:64, 64:].any()
    assert out["z.a0.1.w"].shape == (256, 128) and out["z.a0.2.w"].shape == (2, 16, 128)
    assert out["z.lb"].size == 2 * (160 * 40 + 5 * 40 + 4)
    nb = 2 * 3  # the 4 x 6 grid's bottleneck after the stride-2 reassemble
    assert out["z.r.pe"].shape == (nb + 1, 128)
    bad = dict(sd)
    del bad[ZO.M + "attractors.kitti.2.conv2.weight"]
    with pytest.raises(ValueError, match="attractors.kitti.2.conv2.weight"):
        DW.prepare_zoedepth(bad, cfg, 64, 96)


def test_position_code_matches_transformers():
    from transformers.models.zoedepth.modeling_zoedepth import ZoeDepthPatchTransformerEncoder
    enc = ZoeDepthPatchTransformerEncoder(DW.hf_zoedepth_config("zoedepth-nyu-kitti", **ZO.SMALL))
    ref = enc.positional_encoding_1d(1, 253, 128)[0]
    assert torch.equal(DW.zoedepth_position_code(253), ref)


def test_f16_emulation_floor():
    """The engine's operands are f16 where the GPU runs them on the tensor cores: rounding every weight of the head to
    f16 moves the oracle's metric depth by far less than the GPU gate (1.5e-3 of the range)."""
    sd, cfg = ZO.random_model(multi=True)
    sd16 = {k: (v.half().float() if v.is_floating_point() else v) for k, v in sd.items()}
    torch.manual_seed(5)
    px = torch.randn(3, 64, 96)
    with torch.no_grad():
        d = ZO.forward(sd, cfg, px)
        d16 = ZO.forward(sd16, cfg, px)
    floor = float((d - d16).abs().max() / (d.max() - d.min()))
    assert floor < 1.5e-3, floor


def _save(folder, sd, config):
    import os
    from safetensors.torch import save_file
    os.makedirs(folder, exist_ok=True)
    save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(folder, "model.safetensors"))
    if config is not None:
        with open(os.path.join(folder, "config.json"), "w") as f:
            json.dump(config, f)


def test_menu_entry_and_family():
    from visiondepth3d_b200 import render_depth as RD
    assert RD.supported_models["ZoeDepth"] == ("Intel/zoedepth-nyu-kitti", "zoedepth-nyu-kitti")
    assert RD._family_of("zoedepth-nyu-kitti") == "zoedepth" and RD._dpt_like("zoedepth-nyu-kitti")
    assert "Intel/zoedepth-nyu-kitti" in RD.ZOEDEPTH_FILES_REQUIRED


def test_checkpoint_routing(tmp_path):
    """ZoeDepth state dicts (metric_head.* keys) route to ZoeDepth before the relative_position_bias_table test that
    sends BEiT state dicts to dpt-beit; single-configuration folders load through the same code; a dpt-beit and a
    Depth-Anything folder route as before."""
    import os
    from transformers import DepthAnythingForDepthEstimation
    from tests import dpt_beit_oracle as OB
    from visiondepth3d_b200 import render_depth as RD
    sd, _ = ZO.random_model(multi=True)
    assert any(k.endswith("relative_position_bias_table") for k in sd)
    zoe = str(tmp_path / "zoe")
    _save(zoe, sd, json.loads(DW.hf_zoedepth_config("zoedepth-nyu-kitti").to_json_string()))
    arch, got = RD.load_checkpoint(os.path.join(zoe, "model.safetensors"))
    assert arch == "zoedepth-nyu-kitti" and set(got) == set(sd)
    for name in ("zoedepth-nyu", "zoedepth-kitti"):
        _save(zoe, sd, json.loads(DW.hf_zoedepth_config(name).to_json_string()))
        assert RD.load_checkpoint(os.path.join(zoe, "model.safetensors"))[0] == name
    os.remove(os.path.join(zoe, "config.json"))
    with pytest.raises(ValueError, match="needs its config.json"):
        RD.load_checkpoint(os.path.join(zoe, "model.safetensors"))
    bsd, _ = OB.random_model(small=True)
    beit = str(tmp_path / "beit")
    _save(beit, bsd, json.loads(DW.hf_dpt_beit_config().to_json_string()))
    assert RD.load_checkpoint(os.path.join(beit, "model.safetensors"))[0] == "dpt-beit-large-512"
    torch.manual_seed(0)
    da = str(tmp_path / "da")
    _save(da, DepthAnythingForDepthEstimation(DW.hf_config("vits")).state_dict(), None)
    assert RD.load_checkpoint(os.path.join(da, "model.safetensors"))[0] == "vits"


def test_required_files_and_tiled_refusal(tmp_path, monkeypatch, capsys):
    import os
    from visiondepth3d_b200 import render_depth as RD
    sd, _ = ZO.random_model(multi=True)
    folder = str(tmp_path / "weights" / "Intel_zoedepth-nyu-kitti")
    _save(folder, sd, json.loads(DW.hf_zoedepth_config("zoedepth-nyu-kitti").to_json_string()))
    monkeypatch.setattr(RD, "local_model_dir", str(tmp_path / "weights"))
    assert RD.ensure_model_downloaded("Intel/zoedepth-nyu-kitti") == (None, None)
    assert "no preprocessor_config.json" in capsys.readouterr().out
    with open(os.path.join(folder, "preprocessor_config.json"), "w") as f:
        json.dump(dict(do_resize=True, do_rescale=True, do_normalize=True, do_pad=True, keep_aspect_ratio=True,
                       ensure_multiple_of=32, size={"height": 384, "width": 512}, resample=2, image_mean=[0.5] * 3,
                       image_std=[0.5] * 3), f)
    got, meta = RD.ensure_model_downloaded("Intel/zoedepth-nyu-kitti")
    assert meta["arch"] == "zoedepth-nyu-kitti" and meta["processor"] == DW.ZOEDEPTH_PROCESSOR
    monkeypatch.setattr(RD, "_arch", "zoedepth-nyu-kitti")
    monkeypatch.setattr(RD, "_processor", DW.ZOEDEPTH_PROCESSOR)
    assert RD.model_processed_size(1920, 1080) == (384, 672)
    monkeypatch.setattr(RD, "USE_TILED_DEPTH", True)
    with pytest.raises(ValueError, match="ZoeDepth"):
        RD._check_tiled_supported()
