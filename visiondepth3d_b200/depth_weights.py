"""Prepare Depth-Anything-V2 weights (HF state_dict naming, transformers 5.5
DepthAnythingForDepthEstimation) for the libvd3d depth engine: f16 K-major GEMM operands,
3x3 conv kernels as [Cout, tap, Cin_pad], ConvTranspose as pixel-shuffle GEMMs, position
embeddings interpolated for the processed size.  Pure set-up code (runs once per model)."""
import numpy as np
import torch
import torch.nn.functional as F

CONFIGS = {  # SURVEY section 8(c); verify against config.json when real checkpoints are supplied
    "vits": dict(hidden=384, layers=12, heads=6, taps=[3, 6, 9, 12], neck=[48, 96, 192, 384], fusion=64),
    "vitb": dict(hidden=768, layers=12, heads=12, taps=[3, 6, 9, 12], neck=[96, 192, 384, 768], fusion=128),
    "vitl": dict(hidden=1024, layers=24, heads=16, taps=[5, 12, 18, 24], neck=[256, 512, 1024, 1024], fusion=256),
}


# Depth Anything V1 (LiheYoung/depth-anything-{small,base,large}-hf) taps the last four layers of the backbone
V1_TAPS = {"vits": [9, 10, 11, 12], "vitb": [9, 10, 11, 12], "vitl": [21, 22, 23, 24]}
HEADS = ("relative", "metric")


def da_spec(cfg, taps=None, head=None, max_depth=None):
    """The full engine spec of a Depth-Anything model: `cfg` (a key of CONFIGS or a dict) with the head kind and
    max_depth filled in (relative, 1.0 by default) and any of taps / head / max_depth overridden."""
    c = dict(CONFIGS[cfg]) if isinstance(cfg, str) else dict(cfg)
    c["taps"] = [int(t) for t in (taps if taps is not None else c["taps"])]
    c["head"] = head if head is not None else c.get("head", "relative")
    c["max_depth"] = float(max_depth if max_depth is not None else c.get("max_depth", 1.0))
    if c["head"] not in HEADS:
        raise ValueError(f"unknown depth head {c['head']!r}")
    return c


def da_arch(cfg):
    """The CONFIGS key of a Depth-Anything spec's backbone size ("vits" / "vitb" / "vitl"), or None."""
    for name, c in CONFIGS.items():
        if (c["hidden"], c["layers"], c["heads"]) == (cfg["hidden"], cfg["layers"], cfg["heads"]):
            return name
    return None


def is_plain_v2(cfg):
    """True when a spec is exactly one of the three Depth-Anything-V2 sizes with the relative head."""
    arch = da_arch(cfg)
    s = da_spec(cfg)
    return arch is not None and s == da_spec(arch)


def hf_config(name):
    """transformers config objects equivalent to depth-anything/Depth-Anything-V2-{Small,Base,Large}-hf; `name` may
    also be a spec dict (da_spec / da_config_from_json): V1 taps, a metric head with its max_depth."""
    from transformers import DepthAnythingConfig, Dinov2Config
    c = da_spec(name)
    bc = Dinov2Config(hidden_size=c["hidden"], num_hidden_layers=c["layers"], num_attention_heads=c["heads"],
                      image_size=518, patch_size=14, out_indices=c["taps"], apply_layernorm=True,
                      reshape_hidden_states=False)
    return DepthAnythingConfig(backbone_config=bc, reassemble_hidden_size=c["hidden"],
                               neck_hidden_sizes=c["neck"], fusion_hidden_size=c["fusion"], head_hidden_size=32,
                               patch_size=14, reassemble_factors=[4, 2, 1, 0.5], depth_estimation_type=c["head"],
                               max_depth=int(c["max_depth"]) if c["max_depth"].is_integer() else c["max_depth"])


def da_config_from_json(cj):
    """The engine spec (hidden, layers, heads, taps, neck, fusion, head, max_depth) of a DepthAnythingForDepthEstimation
    config.json (dict), or ValueError naming the field this engine does not serve.  Missing fields take transformers'
    defaults (DepthAnythingConfig: the V1-Small model; Dinov2Config for the backbone's own fields)."""
    import math

    def bad(field, value):
        raise ValueError(f"config.json: {field} = {value!r} is not served (Depth-Anything on a DINOv2 ViT-S/B/L "
                         "backbone with the DPT neck and head)")
    if cj.get("model_type", "depth_anything") != "depth_anything":
        bad("model_type", cj.get("model_type"))
    bj = cj.get("backbone_config")
    if bj is None:
        bj = dict(model_type="dinov2", hidden_size=384, num_hidden_layers=12, num_attention_heads=6,
                  reshape_hidden_states=False, out_indices=[9, 10, 11, 12])
    if not isinstance(bj, dict):
        bad("backbone_config", bj)
    if bj.get("model_type") != "dinov2":
        bad("backbone_config.model_type", bj.get("model_type"))
    for field, want in (("patch_size", 14), ("mlp_ratio", 4), ("num_channels", 3)):
        if bj.get(field, want) != want:
            bad(f"backbone_config.{field}", bj.get(field))
    if cj.get("patch_size", 14) != 14:
        bad("patch_size", cj.get("patch_size"))
    hidden, layers, heads = (int(bj.get("hidden_size", 768)), int(bj.get("num_hidden_layers", 12)),
                             int(bj.get("num_attention_heads", 12)))
    arch = da_arch(dict(hidden=hidden, layers=layers, heads=heads))
    if arch is None:
        bad("backbone_config.hidden_size / num_hidden_layers / num_attention_heads", (hidden, layers, heads))
    if bj.get("use_swiglu_ffn", False):
        bad("backbone_config.use_swiglu_ffn", bj.get("use_swiglu_ffn"))
    eps = bj.get("layer_norm_eps", 1e-6)
    if not isinstance(eps, (int, float)) or abs(float(eps) - 1e-6) > 1e-12:
        bad("backbone_config.layer_norm_eps", eps)
    if bj.get("hidden_act", "gelu") != "gelu":
        bad("backbone_config.hidden_act", bj.get("hidden_act"))
    if bj.get("qkv_bias", True) is not True:
        bad("backbone_config.qkv_bias", bj.get("qkv_bias"))
    if bj.get("apply_layernorm", True) is not True:
        bad("backbone_config.apply_layernorm", bj.get("apply_layernorm"))
    if bj.get("reshape_hidden_states", True) is not False:
        bad("backbone_config.reshape_hidden_states", bj.get("reshape_hidden_states", True))
    taps = bj.get("out_indices")
    if (not isinstance(taps, (list, tuple)) or len(taps) != 4 or any(type(t) is not int for t in taps)
            or not 1 <= taps[0] < taps[1] < taps[2] < taps[3] <= layers):
        bad("backbone_config.out_indices", taps)
    if cj.get("reassemble_hidden_size", 384) != hidden:
        bad("reassemble_hidden_size", cj.get("reassemble_hidden_size", 384))
    if [float(f) for f in cj.get("reassemble_factors", [4, 2, 1, 0.5])] != [4.0, 2.0, 1.0, 0.5]:
        bad("reassemble_factors", cj.get("reassemble_factors"))
    neck = cj.get("neck_hidden_sizes", [48, 96, 192, 384])
    if not isinstance(neck, (list, tuple)) or len(neck) != 4 or any(type(v) is not int or v < 1 for v in neck):
        bad("neck_hidden_sizes", neck)
    fusion = cj.get("fusion_hidden_size", 64)
    if type(fusion) is not int or fusion < 64 or fusion % 64:
        bad("fusion_hidden_size", fusion)
    if cj.get("head_hidden_size", 32) != 32:
        bad("head_hidden_size", cj.get("head_hidden_size"))
    if cj.get("head_in_index", -1) != -1:
        bad("head_in_index", cj.get("head_in_index"))
    head = cj.get("depth_estimation_type", "relative")
    if head not in HEADS:
        bad("depth_estimation_type", head)
    md = cj.get("max_depth") or 1  # DepthAnythingConfig: max_depth if max_depth else 1
    if not isinstance(md, (int, float)) or not math.isfinite(md) or md <= 0 or (head == "relative" and md != 1):
        bad("max_depth", cj.get("max_depth"))
    return dict(hidden=hidden, layers=layers, heads=heads, taps=list(taps), neck=list(neck), fusion=fusion,
                head=head, max_depth=float(md))


# DPTImageProcessor as Depth-Anything's checkpoints configure it: keep the aspect ratio, sides multiples of 14 near
# 518, bicubic, ImageNet mean / std, no padding
DA_PROCESSOR = dict(size=(518, 518), resample=3, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))


def da_processor_from_json(pj):
    """DA_PROCESSOR when a preprocessor_config.json (dict) is Depth-Anything's processor, else ValueError naming the
    field that differs: the engine's processor does exactly that resize and normalisation."""
    def bad(field, value):
        raise ValueError(f"preprocessor_config.json: {field} = {value!r} is not served (Depth-Anything's processor: "
                         "keep_aspect_ratio, ensure_multiple_of 14, 518 x 518, bicubic, 1/255, ImageNet mean / std)")
    for field in ("do_resize", "do_rescale", "do_normalize", "keep_aspect_ratio"):
        if pj.get(field, True) is not True:
            bad(field, pj.get(field))
    if "keep_aspect_ratio" not in pj:
        bad("keep_aspect_ratio", None)
    if pj.get("ensure_multiple_of") != 14:
        bad("ensure_multiple_of", pj.get("ensure_multiple_of"))
    size = pj.get("size")
    if size != {"height": 518, "width": 518}:
        bad("size", size)
    if pj.get("resample", 3) != 3:
        bad("resample", pj.get("resample"))
    rf = pj.get("rescale_factor", 1 / 255)
    if not isinstance(rf, (int, float)) or abs(rf - 1 / 255) > 1e-9:
        bad("rescale_factor", rf)
    for field, want in (("image_mean", DA_PROCESSOR["mean"]), ("image_std", DA_PROCESSOR["std"])):
        v = pj.get(field)
        if (not isinstance(v, (list, tuple)) or len(v) != 3
                or any(not isinstance(x, (int, float)) or abs(x - w) > 1e-6 for x, w in zip(v, want))):
            bad(field, v)
    if pj.get("do_pad", False):
        bad("do_pad", pj.get("do_pad"))
    return dict(DA_PROCESSOR)


def _up(v, m):
    return (v + m - 1) // m * m


def _f16(t):
    return np.ascontiguousarray(t.detach().to(torch.float32).cpu().numpy().astype(np.float16))


def _f32(t):
    return np.ascontiguousarray(t.detach().to(torch.float32).cpu().numpy())


def _conv3(w, cin_pad, cout_pad=None):
    """[Cout, Cin, 3, 3] -> [Cout_pad, 9 * cin_pad] (tap-major, channel-minor), zero padded."""
    co, ci = w.shape[0], w.shape[1]
    cout_pad = cout_pad or co
    out = torch.zeros(cout_pad, 9, cin_pad, dtype=torch.float32)
    out[:co, :, :ci] = w.detach().float().permute(0, 2, 3, 1).reshape(co, 9, ci)
    return _f16(out.reshape(cout_pad, 9 * cin_pad))


def _pad_vec(b, n):
    out = torch.zeros(n, dtype=torch.float32)
    out[: b.numel()] = b.detach().float().reshape(-1)
    return _f32(out)


def prepare(sd, cfg, image_h, image_w):
    """state_dict -> {name: np.ndarray} in the layouts depth_engine.cu expects."""
    D, L = cfg["hidden"], cfg["layers"]
    ph, pw = image_h // 14, image_w // 14
    out = {}
    e = "backbone.embeddings."
    w = torch.zeros(D, 592)
    w[:, :588] = sd[e + "patch_embeddings.projection.weight"].float().reshape(D, 588)
    out["pe.w"] = _f16(w)
    out["pe.b"] = _f32(sd[e + "patch_embeddings.projection.bias"])
    out["cls"] = _f32(sd[e + "cls_token"].reshape(D))
    pos = sd[e + "position_embeddings"].float()
    npos = pos.shape[1] - 1
    g = int(round(npos ** 0.5))
    if not (ph == g and pw == g):
        pp = pos[:, 1:].reshape(1, g, g, D).permute(0, 3, 1, 2)
        pp = F.interpolate(pp, size=(ph, pw), mode="bicubic", align_corners=False)  # Dinov2Embeddings.interpolate_pos_encoding
        pos = torch.cat((pos[:, :1], pp.permute(0, 2, 3, 1).reshape(1, -1, D)), dim=1)
    out["pos"] = _f32(pos.reshape(-1, D))
    for i in range(L):
        p = f"backbone.encoder.layer.{i}."
        a = p + "attention.attention."
        out[f"l{i}.ln1.g"] = _f32(sd[p + "norm1.weight"])
        out[f"l{i}.ln1.b"] = _f32(sd[p + "norm1.bias"])
        out[f"l{i}.qkv.w"] = _f16(torch.cat([sd[a + "query.weight"], sd[a + "key.weight"], sd[a + "value.weight"]], 0))
        out[f"l{i}.qkv.b"] = _f32(torch.cat([sd[a + "query.bias"], sd[a + "key.bias"], sd[a + "value.bias"]], 0))
        out[f"l{i}.proj.w"] = _f16(sd[p + "attention.output.dense.weight"])
        out[f"l{i}.proj.b"] = _f32(sd[p + "attention.output.dense.bias"])
        out[f"l{i}.ls1"] = _f32(sd[p + "layer_scale1.lambda1"])
        out[f"l{i}.ln2.g"] = _f32(sd[p + "norm2.weight"])
        out[f"l{i}.ln2.b"] = _f32(sd[p + "norm2.bias"])
        out[f"l{i}.fc1.w"] = _f16(sd[p + "mlp.fc1.weight"])
        out[f"l{i}.fc1.b"] = _f32(sd[p + "mlp.fc1.bias"])
        out[f"l{i}.fc2.w"] = _f16(sd[p + "mlp.fc2.weight"])
        out[f"l{i}.fc2.b"] = _f32(sd[p + "mlp.fc2.bias"])
        out[f"l{i}.ls2"] = _f32(sd[p + "layer_scale2.lambda1"])
    out["norm.g"] = _f32(sd["backbone.layernorm.weight"])
    out["norm.b"] = _f32(sd["backbone.layernorm.bias"])
    out.update(_prepare_tail(sd, cfg))
    return out


def _prepare_tail(sd, cfg):
    """The reassemble layers, neck convs, fusion stage and head (HF names of DepthAnythingForDepthEstimation) in the
    engine's layouts: shared by Depth-Anything and DPT.  Fusion layer 0 never runs its residual_layer1; it is packed
    when the state dict has it."""
    D, Fz = cfg["hidden"], cfg["fusion"]
    out = {}
    for i, C in enumerate(cfg["neck"]):
        CP = _up(C, 64)
        r = f"neck.reassemble_stage.layers.{i}."
        pw_ = torch.zeros(CP, D)
        pw_[:C] = sd[r + "projection.weight"].float().reshape(C, D)
        out[f"r{i}.proj.w"] = _f16(pw_)
        out[f"r{i}.proj.b"] = _pad_vec(sd[r + "projection.bias"], CP)
        if i < 2:  # ConvTranspose2d [Cin, Cout, k, k] -> rows n = (dy*k+dx)*CP + co, cols ci
            k = 4 if i == 0 else 2
            wt = sd[r + "resize.weight"].float()
            uw = torch.zeros(k * k, CP, CP)
            uw[:, :C, :C] = wt.permute(2, 3, 1, 0).reshape(k * k, C, C)
            out[f"r{i}.up.w"] = _f16(uw.reshape(k * k * CP, CP))
            ub = torch.zeros(k * k, CP)
            ub[:, :C] = sd[r + "resize.bias"].float()[None, :]
            out[f"r{i}.up.b"] = _f32(ub.reshape(-1))
        elif i == 3:
            out["r3.down.w"] = _conv3(sd[r + "resize.weight"], CP, CP)
            out["r3.down.b"] = _pad_vec(sd[r + "resize.bias"], CP)
        out[f"n{i}.conv.w"] = _conv3(sd[f"neck.convs.{i}.weight"], CP)
    for j in range(4):
        f = f"neck.fusion_stage.layers.{j}."
        for unit, hf in (("rl1", "residual_layer1"), ("rl2", "residual_layer2")):
            if f + hf + ".convolution1.weight" not in sd and j == 0 and unit == "rl1":
                continue
            for c, hc in (("c1", "convolution1"), ("c2", "convolution2")):
                out[f"f{j}.{unit}.{c}.w"] = _conv3(sd[f + hf + "." + hc + ".weight"], Fz)
                out[f"f{j}.{unit}.{c}.b"] = _f32(sd[f + hf + "." + hc + ".bias"])
        out[f"f{j}.proj.w"] = _f16(sd[f + "projection.weight"].reshape(Fz, Fz))
        out[f"f{j}.proj.b"] = _f32(sd[f + "projection.bias"])
    F2 = _up(Fz // 2, 64)
    out["h.c1.w"] = _conv3(sd["head.conv1.weight"], Fz, F2)
    out["h.c1.b"] = _pad_vec(sd["head.conv1.bias"], F2)
    out["h.c2.w"] = _conv3(sd["head.conv2.weight"], F2)
    out["h.c2.b"] = _f32(sd["head.conv2.bias"])
    out["h.c3.w"] = _f32(sd["head.conv3.weight"].reshape(-1))
    out["h.c3.b"] = _f32(sd["head.conv3.bias"].reshape(-1))
    return out


# ---------------------------------------------------------------------------
# DPT-Large (Intel/dpt-large; transformers 5.5 DPTForDepthEstimation): ViT-L/16 without LayerScale, LayerNorm eps
# 1e-12, taps = the raw residual stream after layers 6 / 12 / 18 / 24 (backbone_out_indices [5, 11, 17, 23] over
# hidden_states[1:]), project readout GELU(Linear_{2D -> D}(cat(tok, cls))) per tap, then the neck and head of
# Depth-Anything with the head's upsample x2 (= patch x grid).
# ---------------------------------------------------------------------------
DPT_CONFIGS = {
    "dpt-large": dict(hidden=1024, layers=24, heads=16, taps=[6, 12, 18, 24], neck=[256, 512, 1024, 1024], fusion=256,
                      patch=16, ln_eps=1e-12, image_size=384),
}

# DPTImageProcessor's class defaults, which Intel/dpt-large's preprocessor_config.json repeats: a fixed 384 x 384
# target without keeping the aspect ratio, bicubic, mean = std = 0.5
DPT_PROCESSOR = dict(size=(384, 384), resample=3, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5))


def hf_dpt_config(name="dpt-large", **cfg):
    """transformers DPTConfig equal to the checkpoint's (Intel/dpt-large's config.json); `cfg` overrides entries of
    DPT_CONFIGS[name] (a smaller ViT for tests)."""
    from transformers import DPTConfig
    c = dict(DPT_CONFIGS[name], **cfg)
    return DPTConfig(hidden_size=c["hidden"], num_hidden_layers=c["layers"], num_attention_heads=c["heads"],
                     intermediate_size=4 * c["hidden"], hidden_act="gelu", layer_norm_eps=c["ln_eps"],
                     image_size=c["image_size"], patch_size=c["patch"], num_channels=3, qkv_bias=True,
                     is_hybrid=False, backbone_out_indices=[t - 1 for t in c["taps"]], readout_type="project",
                     reassemble_factors=[4, 2, 1, 0.5], neck_hidden_sizes=c["neck"], fusion_hidden_size=c["fusion"],
                     head_in_index=-1, use_batch_norm_in_fusion_residual=False, use_bias_in_fusion_residual=None,
                     add_projection=False)


def dpt_config_from_json(cj):
    """The engine configuration of a DPT config.json (dict), or ValueError naming what this engine does not serve."""
    def bad(what):
        raise ValueError(f"config.json: {what} is not served (DPT with a ViT backbone and project readout only)")
    if cj.get("is_hybrid") or cj.get("backbone_config"):
        bad("a hybrid / external backbone")
    if cj.get("readout_type", "project") != "project":
        bad(f"readout_type {cj.get('readout_type')!r}")
    if cj.get("add_projection") or cj.get("use_batch_norm_in_fusion_residual"):
        bad("a head projection or batch-norm fusion units")
    if list(cj.get("reassemble_factors", [4, 2, 1, 0.5])) != [4, 2, 1, 0.5]:
        bad(f"reassemble_factors {cj.get('reassemble_factors')}")
    if cj.get("hidden_act", "gelu") != "gelu" or cj.get("use_bias_in_fusion_residual") is False:
        bad("another activation or bias-free fusion units")
    hidden = int(cj.get("hidden_size", 768))
    heads = int(cj.get("num_attention_heads", 12))
    if int(cj.get("intermediate_size", 4 * hidden)) != 4 * hidden or hidden != 64 * heads:
        bad("an MLP width other than 4 x hidden or a head size other than 64")
    return dict(hidden=hidden, layers=int(cj.get("num_hidden_layers", 12)), heads=heads,
                taps=[int(t) + 1 for t in cj.get("backbone_out_indices", [2, 5, 8, 11])],
                neck=[int(v) for v in cj.get("neck_hidden_sizes", [96, 192, 384, 768])],
                fusion=int(cj.get("fusion_hidden_size", 256)), patch=int(cj.get("patch_size", 16)),
                ln_eps=float(cj.get("layer_norm_eps", 1e-12)), image_size=int(cj.get("image_size", 384)))


def dpt_processor_from_json(pj):
    """DPT_PROCESSOR updated from a preprocessor_config.json (dict); ValueError for what the engine's processor does
    not do (keep_aspect_ratio, ensure_multiple_of > 1, padding, a resample other than bicubic / bilinear)."""
    p = dict(DPT_PROCESSOR)
    if pj.get("keep_aspect_ratio") or int(pj.get("ensure_multiple_of", 1)) != 1 or pj.get("do_pad"):
        raise ValueError("preprocessor_config.json: keep_aspect_ratio / ensure_multiple_of / do_pad are not served")
    if pj.get("do_resize", True) is False or pj.get("do_rescale", True) is False or pj.get("do_normalize", True) is False:
        raise ValueError("preprocessor_config.json: the processor must resize, rescale and normalise")
    if abs(float(pj.get("rescale_factor", 1 / 255)) - 1 / 255) > 1e-9:
        raise ValueError("preprocessor_config.json: rescale_factor must be 1/255")
    size = pj.get("size", {"height": 384, "width": 384})
    if isinstance(size, int):
        size = {"height": size, "width": size}
    if "height" not in size or "width" not in size:
        raise ValueError(f"preprocessor_config.json: size {size} is not a height / width pair")
    p["size"] = (int(size["height"]), int(size["width"]))
    p["resample"] = int(pj.get("resample", 3))
    if p["resample"] not in (2, 3):
        raise ValueError(f"preprocessor_config.json: resample {p['resample']} is not served (2 bilinear, 3 bicubic)")
    for k, key in (("mean", "image_mean"), ("std", "image_std")):
        if key in pj:
            v = pj[key]
            p[k] = tuple(float(x) for x in (v if isinstance(v, (list, tuple)) else [v] * 3))
    return p


def dpt_processed_size(processor=None):
    """(h, w) DPTImageProcessor resizes every image to (keep_aspect_ratio False, ensure_multiple_of 1): the fixed
    size, whatever the frame.  ValueError unless it is square with a side that is a multiple of 32: DPT reshapes the
    tokens as a square grid, and an even grid makes each fusion x2 land on the next map."""
    h, w = (processor or DPT_PROCESSOR)["size"]
    if h != w or h % 32 or h < 32:
        raise ValueError(f"DPT processed size {w}x{h} is not served: it must be square with a side that is a "
                         "multiple of 32")
    return h, w


def dpt_keys(cfg):
    """Every state_dict key (and its shape) the DPT depth forward reads."""
    D, L, P = cfg["hidden"], cfg["layers"], cfg["patch"]
    g = cfg["image_size"] // P
    k = {"dpt.embeddings.cls_token": (1, 1, D), "dpt.embeddings.position_embeddings": (1, g * g + 1, D),
         "dpt.embeddings.patch_embeddings.projection.weight": (D, 3, P, P),
         "dpt.embeddings.patch_embeddings.projection.bias": (D,)}
    for i in range(L):
        p = f"dpt.encoder.layer.{i}."
        for n in ("layernorm_before", "layernorm_after"):
            k[p + n + ".weight"] = k[p + n + ".bias"] = (D,)
        for n in ("query", "key", "value"):
            k[p + "attention.attention." + n + ".weight"] = (D, D)
            k[p + "attention.attention." + n + ".bias"] = (D,)
        k[p + "attention.output.dense.weight"], k[p + "attention.output.dense.bias"] = (D, D), (D,)
        k[p + "intermediate.dense.weight"], k[p + "intermediate.dense.bias"] = (4 * D, D), (4 * D,)
        k[p + "output.dense.weight"], k[p + "output.dense.bias"] = (D, 4 * D), (D,)
    Fz = cfg["fusion"]
    for i, C in enumerate(cfg["neck"]):
        r = f"neck.reassemble_stage."
        k[r + f"readout_projects.{i}.0.weight"], k[r + f"readout_projects.{i}.0.bias"] = (D, 2 * D), (D,)
        r += f"layers.{i}."
        k[r + "projection.weight"], k[r + "projection.bias"] = (C, D, 1, 1), (C,)
        if i < 2:
            f = 4 if i == 0 else 2
            k[r + "resize.weight"], k[r + "resize.bias"] = (C, C, f, f), (C,)
        elif i == 3:
            k[r + "resize.weight"], k[r + "resize.bias"] = (C, C, 3, 3), (C,)
        k[f"neck.convs.{i}.weight"] = (Fz, C, 3, 3)
    for j in range(4):
        f = f"neck.fusion_stage.layers.{j}."
        for u in ("residual_layer1", "residual_layer2") if j else ("residual_layer2",):
            for c in ("convolution1", "convolution2"):
                k[f + u + "." + c + ".weight"], k[f + u + "." + c + ".bias"] = (Fz, Fz, 3, 3), (Fz,)
        k[f + "projection.weight"], k[f + "projection.bias"] = (Fz, Fz, 1, 1), (Fz,)
    k["head.head.0.weight"], k["head.head.0.bias"] = (Fz // 2, Fz, 3, 3), (Fz // 2,)
    k["head.head.2.weight"], k["head.head.2.bias"] = (32, Fz // 2, 3, 3), (32,)
    k["head.head.4.weight"], k["head.head.4.bias"] = (1, 32, 1, 1), (1,)
    return k


def check_dpt_state_dict(sd, cfg):
    """ValueError naming the first missing or mis-shaped key the DPT forward reads.  Other keys (the final
    dpt.layernorm, a pooler, fusion layer 0's unused residual_layer1) are ignored."""
    for name, shape in dpt_keys(cfg).items():
        if name not in sd:
            raise ValueError(f"DPT state dict: missing key {name}")
        if tuple(sd[name].shape) != shape:
            raise ValueError(f"DPT state dict: {name} has shape {tuple(sd[name].shape)}, expected {shape}")


def prepare_dpt(sd, cfg, image_h, image_w):
    """DPT state_dict -> {name: np.ndarray} in the layouts depth_engine.cu expects (the tensor names of `prepare`
    where the op is shared; LayerScale as vectors of ones, exact in EPI_RESID_LS; the readout split into its token
    and CLS halves "ro{i}.wt" / "ro{i}.wc")."""
    check_dpt_state_dict(sd, cfg)
    D, P = cfg["hidden"], cfg["patch"]
    ph, pw = image_h // P, image_w // P
    e = "dpt.embeddings."
    out = {"pe.w": _f16(sd[e + "patch_embeddings.projection.weight"].float().reshape(D, 3 * P * P)),
           "pe.b": _f32(sd[e + "patch_embeddings.projection.bias"]),
           "cls": _f32(sd[e + "cls_token"].reshape(D))}
    pos = sd[e + "position_embeddings"].float()
    g = int(round((pos.shape[1] - 1) ** 0.5))
    pp = pos[:, 1:].reshape(1, g, g, D).permute(0, 3, 1, 2)
    pp = F.interpolate(pp, size=(ph, pw), mode="bilinear")  # DPTViTEmbeddings._resize_pos_embed (identity at g x g)
    out["pos"] = _f32(torch.cat((pos[:, :1], pp.permute(0, 2, 3, 1).reshape(1, -1, D)), dim=1).reshape(-1, D))
    ones = np.ones(D, np.float32)
    for i in range(cfg["layers"]):
        p = f"dpt.encoder.layer.{i}."
        a = p + "attention.attention."
        out[f"l{i}.ln1.g"] = _f32(sd[p + "layernorm_before.weight"])
        out[f"l{i}.ln1.b"] = _f32(sd[p + "layernorm_before.bias"])
        out[f"l{i}.qkv.w"] = _f16(torch.cat([sd[a + "query.weight"], sd[a + "key.weight"], sd[a + "value.weight"]], 0))
        out[f"l{i}.qkv.b"] = _f32(torch.cat([sd[a + "query.bias"], sd[a + "key.bias"], sd[a + "value.bias"]], 0))
        out[f"l{i}.proj.w"] = _f16(sd[p + "attention.output.dense.weight"])
        out[f"l{i}.proj.b"] = _f32(sd[p + "attention.output.dense.bias"])
        out[f"l{i}.ls1"] = ones
        out[f"l{i}.ln2.g"] = _f32(sd[p + "layernorm_after.weight"])
        out[f"l{i}.ln2.b"] = _f32(sd[p + "layernorm_after.bias"])
        out[f"l{i}.fc1.w"] = _f16(sd[p + "intermediate.dense.weight"])
        out[f"l{i}.fc1.b"] = _f32(sd[p + "intermediate.dense.bias"])
        out[f"l{i}.fc2.w"] = _f16(sd[p + "output.dense.weight"])
        out[f"l{i}.fc2.b"] = _f32(sd[p + "output.dense.bias"])
        out[f"l{i}.ls2"] = ones
    for i in range(4):
        r = f"neck.reassemble_stage.readout_projects.{i}.0."
        w = sd[r + "weight"].float()
        out[f"ro{i}.wt"] = _f16(w[:, :D])
        out[f"ro{i}.wc"] = _f16(w[:, D:])
        out[f"ro{i}.b"] = _f32(sd[r + "bias"])
    # the neck, fusion and head share Depth-Anything's layouts: rename the head and reuse `prepare`'s code for them
    shared = {k: v for k, v in sd.items() if k.startswith("neck.reassemble_stage.layers.") or k.startswith("neck.convs.")
              or k.startswith("neck.fusion_stage.")}
    for j, n in ((0, "conv1"), (2, "conv2"), (4, "conv3")):
        shared[f"head.{n}.weight"] = sd[f"head.head.{j}.weight"]
        shared[f"head.{n}.bias"] = sd[f"head.head.{j}.bias"]
    out.update(_prepare_tail(shared, cfg))
    return out
