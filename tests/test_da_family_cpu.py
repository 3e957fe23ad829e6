"""CPU: the Depth-Anything family beyond V2 -- Depth Anything V1 (the last four layers as taps), Distill-Any-Depth and
the V2 metric models (max_depth * sigmoid head): the fp32 oracle against transformers, config.json / preprocessor
parsing, the menu, and checkpoint folders resolved to their spec."""
import json

import numpy as np
import pytest
import torch

from tests import da_family_oracle as DO
from visiondepth3d_b200 import depth_weights as DW

V1 = {k: DW.da_spec(k, taps=DW.V1_TAPS[k]) for k in ("vits", "vitb", "vitl")}
V2 = {k: DW.da_spec(k) for k in ("vits", "vitb", "vitl")}
METRIC = {"indoor": DW.da_spec("vitl", head="metric", max_depth=20.0),
          "outdoor": DW.da_spec("vitl", head="metric", max_depth=80.0)}


def _hf_depth(sd, spec, px):
    from transformers import DepthAnythingForDepthEstimation
    m = DepthAnythingForDepthEstimation(DW.hf_config(spec)).eval()
    m.load_state_dict(sd)
    with torch.no_grad():
        return m(pixel_values=px[None]).predicted_depth[0]


@pytest.mark.parametrize("case", ["v1-s", "v1-l", "metric-20", "metric-80"])
def test_oracle_matches_transformers(case):
    spec = {"v1-s": V1["vits"], "v1-l": V1["vitl"], "metric-20": DW.da_spec("vits", head="metric", max_depth=20.0),
            "metric-80": DW.da_spec("vits", head="metric", max_depth=80.0)}[case]
    px = torch.randn(3, 70, 98, generator=torch.Generator().manual_seed(7))
    sd, spec = DO.random_model(spec, calib=px)
    with torch.no_grad():
        ref, pre = DO.forward(sd, spec, px, return_pre=True)
    got = _hf_depth(sd, spec, px)
    if spec["head"] == "metric":  # the scaled head reaches both flat tails and the steep middle of the sigmoid
        assert float(pre.min()) < -3.9 and float(pre.max()) > 3.9
        assert float(ref.min()) < 0.03 * spec["max_depth"] and float(ref.max()) > 0.97 * spec["max_depth"]
    assert float((ref - got).abs().max()) <= 1e-4 * float(ref.abs().max()), case


def test_taps_change_the_depth():
    """V1 and V2 tensors have the same shapes: the taps only come from config.json, and they matter."""
    px = torch.randn(3, 70, 98, generator=torch.Generator().manual_seed(3))
    sd, _ = DO.random_model(V1["vits"])
    with torch.no_grad():
        a, b = DO.forward(sd, V1["vits"], px), DO.forward(sd, V2["vits"], px)
    assert float((a - b).abs().max()) > 1e-2 * float(a.max() - a.min())


def _saved_config(tmp_path, spec):
    DW.hf_config(spec).save_pretrained(str(tmp_path))
    return json.load(open(tmp_path / "config.json"))


@pytest.mark.parametrize("name", ["v1-vits", "v1-vitb", "v1-vitl", "v2-vits", "v2-vitb", "v2-vitl", "indoor",
                                  "outdoor"])
def test_config_from_saved_json(tmp_path, name):
    spec = METRIC.get(name) or (V1 if name.startswith("v1") else V2)[name[3:]]
    got = DW.da_config_from_json(_saved_config(tmp_path, spec))
    assert got == spec
    assert DW.is_plain_v2(got) == name.startswith("v2")


def test_config_defaults_are_v1_small():
    from transformers import DepthAnythingConfig
    assert DW.da_config_from_json(DepthAnythingConfig().to_dict()) == V1["vits"]


UNSERVED = [
    ("backbone_config.model_type", lambda c: c["backbone_config"].update(model_type="vit")),
    ("backbone_config.patch_size", lambda c: c["backbone_config"].update(patch_size=16)),
    ("patch_size", lambda c: c.update(patch_size=16)),
    ("num_hidden_layers", lambda c: c["backbone_config"].update(num_hidden_layers=18)),
    ("hidden_size", lambda c: c["backbone_config"].update(hidden_size=512)),
    ("num_attention_heads", lambda c: c["backbone_config"].update(num_attention_heads=8)),
    ("use_swiglu_ffn", lambda c: c["backbone_config"].update(use_swiglu_ffn=True)),
    ("layer_norm_eps", lambda c: c["backbone_config"].update(layer_norm_eps=1e-5)),
    ("hidden_act", lambda c: c["backbone_config"].update(hidden_act="relu")),
    ("apply_layernorm", lambda c: c["backbone_config"].update(apply_layernorm=False)),
    ("reshape_hidden_states", lambda c: c["backbone_config"].update(reshape_hidden_states=True)),
    ("reassemble_hidden_size", lambda c: c.update(reassemble_hidden_size=256)),
    ("reassemble_factors", lambda c: c.update(reassemble_factors=[4, 2, 1, 1])),
    ("head_hidden_size", lambda c: c.update(head_hidden_size=64)),
    ("head_in_index", lambda c: c.update(head_in_index=2)),
    ("out_indices", lambda c: c["backbone_config"].update(out_indices=[3, 6, 9])),
    ("out_indices", lambda c: c["backbone_config"].update(out_indices=[3, 9, 6, 12])),
    ("out_indices", lambda c: c["backbone_config"].update(out_indices=[3, 6, 9, 13])),
    ("out_indices", lambda c: c["backbone_config"].update(out_indices=[0, 6, 9, 12])),
    ("depth_estimation_type", lambda c: c.update(depth_estimation_type="disparity")),
    ("max_depth", lambda c: c.update(depth_estimation_type="metric", max_depth=-5)),
    ("max_depth", lambda c: c.update(max_depth=20)),  # a relative head scaled by max_depth
    ("fusion_hidden_size", lambda c: c.update(fusion_hidden_size=96)),
]


@pytest.mark.parametrize("field,edit", UNSERVED, ids=[f"{f}-{i}" for i, (f, _) in enumerate(UNSERVED)])
def test_unserved_config_refused(tmp_path, field, edit):
    cj = _saved_config(tmp_path, V2["vits"])
    edit(cj)
    with pytest.raises(ValueError, match=field.split(".")[-1]):
        DW.da_config_from_json(cj)


def _processor(**kw):
    from transformers.models.dpt.image_processing_dpt import DPTImageProcessor
    args = dict(keep_aspect_ratio=True, ensure_multiple_of=14, size={"height": 518, "width": 518}, resample=3,
                image_mean=[0.485, 0.456, 0.406], image_std=[0.229, 0.224, 0.225])
    args.update(kw)
    return DPTImageProcessor(**args)


def _saved_processor(tmp_path, proc):
    proc.save_pretrained(str(tmp_path))
    return json.load(open(tmp_path / "preprocessor_config.json"))


def test_processor_accepted(tmp_path):
    assert DW.da_processor_from_json(_saved_processor(tmp_path, _processor())) == DW.DA_PROCESSOR


@pytest.mark.parametrize("kw", [dict(keep_aspect_ratio=False), dict(ensure_multiple_of=1), dict(ensure_multiple_of=32),
                                dict(size={"height": 384, "width": 384}), dict(resample=2), dict(rescale_factor=1 / 127.5),
                                dict(image_mean=[0.5, 0.5, 0.5]), dict(image_std=[0.5, 0.5, 0.5]), dict(do_pad=True),
                                dict(do_resize=False), dict(do_rescale=False), dict(do_normalize=False)],
                         ids=lambda kw: next(iter(kw)))
def test_processor_variants_refused(tmp_path, kw):
    pj = _saved_processor(tmp_path, _processor(**kw))
    with pytest.raises(ValueError, match=next(iter(kw))):
        DW.da_processor_from_json(pj)


def test_menu_has_the_family():
    from visiondepth3d_b200 import render_depth as RD
    want = {
        "Depth Anything V1 Small": "LiheYoung/depth-anything-small-hf",
        "Depth Anything V1 Base": "LiheYoung/depth-anything-base-hf",
        "Depth Anything V1 Large": "LiheYoung/depth-anything-large-hf",
        "Distil-Any-Depth-Large": "xingyang1/Distill-Any-Depth-Large-hf",
        "Distil-Any-Depth-Small": "xingyang1/Distill-Any-Depth-Small-hf",
        "keetrap-Distil-Any-Depth-Large": "keetrap/Distil-Any-Depth-Large-hf",
        "keetrap-Distil-Any-Depth-Small": "keetrap/Distill-Any-Depth-Small-hf",
        "V2-Metric-Indoor-Large": "depth-anything/Depth-Anything-V2-Metric-Indoor-Large-hf",
        "V2-Metric-Outdoor-Large": "depth-anything/Depth-Anything-V2-Metric-Outdoor-Large-hf",
    }
    for label, ck in want.items():
        assert RD.supported_models[label][0] == ck
        assert ck in RD.DA_CONFIG_REQUIRED
    assert "vitl14" not in RD.supported_models


def _folder(tmp_path, name, spec, processor=True):
    """A checkpoint folder in the reference's cache layout (weights/<org>_<name>) written by save_pretrained."""
    from transformers import DepthAnythingForDepthEstimation
    torch.manual_seed(0)
    model = DepthAnythingForDepthEstimation(DW.hf_config(spec)).eval()
    folder = tmp_path / "weights" / name.replace("/", "_")
    model.save_pretrained(str(folder))
    if processor:
        _processor().save_pretrained(str(folder))
    return folder, model.state_dict()


@pytest.mark.parametrize("ck,spec", [("LiheYoung/depth-anything-small-hf", V1["vits"]),
                                     ("xingyang1/Distill-Any-Depth-Small-hf", V2["vits"]),
                                     ("depth-anything/Depth-Anything-V2-Metric-Indoor-Large-hf", METRIC["indoor"])])
def test_checkpoint_folder_resolves_to_its_spec(tmp_path, monkeypatch, ck, spec):
    from visiondepth3d_b200 import render_depth as RD
    folder, sd = _folder(tmp_path, ck, spec)
    monkeypatch.setattr(RD, "local_model_dir", str(tmp_path / "weights"))
    got, meta = RD.ensure_model_downloaded(ck)
    assert meta["spec"] == spec and meta["arch"] == DW.da_arch(spec) and set(got) == set(sd)
    # a tampered config.json / preprocessor_config.json is refused
    cfg = json.load(open(folder / "config.json"))
    bad = json.loads(json.dumps(cfg))
    bad["backbone_config"]["use_swiglu_ffn"] = True
    json.dump(bad, open(folder / "config.json", "w"))
    assert RD.ensure_model_downloaded(ck) == (None, None)
    json.dump(cfg, open(folder / "config.json", "w"))
    pj = json.load(open(folder / "preprocessor_config.json"))
    json.dump(dict(pj, ensure_multiple_of=32), open(folder / "preprocessor_config.json", "w"))
    assert RD.ensure_model_downloaded(ck) == (None, None)
    # without its config.json the checkpoint does not load (its taps and head are only there)
    (folder / "preprocessor_config.json").unlink()
    assert RD.ensure_model_downloaded(ck)[1]["spec"] == spec  # the processor file is optional
    (folder / "config.json").unlink()
    assert RD.ensure_model_downloaded(ck) == (None, None)


def test_v2_folder_loads_as_before(tmp_path, monkeypatch):
    """Plain V2 keeps its loader: without config.json the size comes from the hidden width; with one it is parsed."""
    from visiondepth3d_b200 import render_depth as RD
    ck = "depth-anything/Depth-Anything-V2-Base-hf"
    folder, _ = _folder(tmp_path, ck, V2["vitb"], processor=False)
    monkeypatch.setattr(RD, "local_model_dir", str(tmp_path / "weights"))
    got, meta = RD.ensure_model_downloaded(ck)
    assert meta["arch"] == "vitb" and meta["spec"] == V2["vitb"]
    (folder / "config.json").unlink()
    got, meta = RD.ensure_model_downloaded(ck)
    assert meta["arch"] == "vitb" and meta["spec"] == V2["vitb"]


def test_state_dict_must_match_its_config(tmp_path, monkeypatch):
    from visiondepth3d_b200 import render_depth as RD
    ck = "LiheYoung/depth-anything-small-hf"
    folder, _ = _folder(tmp_path, ck, V1["vits"])
    DW.hf_config(V1["vitb"]).save_pretrained(str(folder))  # a Base config next to Small weights
    monkeypatch.setattr(RD, "local_model_dir", str(tmp_path / "weights"))
    assert RD.ensure_model_downloaded(ck) == (None, None)


def test_depth_config_ex_mirror():
    import ctypes as C
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200.depth_engine import DepthConfigEx, _bind
    lib = _lib.load()
    _bind(lib)
    assert lib.vd3d_struct_size(6) == C.sizeof(DepthConfigEx)
    assert [f[0] for f in DepthConfigEx._fields_][-2:] == ["head", "max_depth"]
    assert np.isclose(DW.DA_PROCESSOR["std"][0], 0.229)
