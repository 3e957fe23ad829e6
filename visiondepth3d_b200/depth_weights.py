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


def _prepare_tail(sd, cfg, direct=()):
    """The reassemble layers, neck convs, fusion stage and head (HF names of DepthAnythingForDepthEstimation) in the
    engine's layouts: shared by Depth-Anything and DPT.  Fusion layer 0 never runs its residual_layer1; it is packed
    when the state dict has it.  direct: neck inputs without a reassemble layer (DPT-Hybrid's BiT stages 1 and 2)."""
    D, Fz = cfg["hidden"], cfg["fusion"]
    out = {}
    for i, C in enumerate(cfg["neck"]):
        CP = _up(C, 64)
        if i in direct:
            out[f"n{i}.conv.w"] = _conv3(sd[f"neck.convs.{i}.weight"], CP)
            continue
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
    e = "dpt.embeddings."
    out = {"pe.w": _f16(sd[e + "patch_embeddings.projection.weight"].float().reshape(D, 3 * P * P)),
           "pe.b": _f32(sd[e + "patch_embeddings.projection.bias"])}
    out.update(_prepare_dpt_vit(sd, cfg, image_h, image_w, range(4)))
    return out


def _prepare_dpt_vit(sd, cfg, image_h, image_w, readouts, direct=()):
    """DPT's CLS token, position embeddings, ViT layers, the project readouts `readouts` and the neck, fusion and head
    (shared by DPT-Large and DPT-Hybrid)."""
    D, P = cfg["hidden"], cfg["patch"]
    ph, pw = image_h // P, image_w // P
    e = "dpt.embeddings."
    out = {"cls": _f32(sd[e + "cls_token"].reshape(D))}
    pos = sd[e + "position_embeddings"].float()
    g = int(round((pos.shape[1] - 1) ** 0.5))
    pp = pos[:, 1:].reshape(1, g, g, D).permute(0, 3, 1, 2)
    pp = F.interpolate(pp, size=(ph, pw), mode="bilinear")  # DPTViTEmbeddings._resize_pos_embed (identity at g x g)
    out["pos"] = _f32(torch.cat((pos[:, :1], pp.permute(0, 2, 3, 1).reshape(1, -1, D)), dim=1).reshape(-1, D))
    out.update(_prepare_dpt_layers(sd, cfg, "dpt.encoder.layer."))
    out.update(_prepare_dpt_neck(sd, cfg, readouts, direct))
    return out


def _prepare_dpt_layers(sd, cfg, prefix):
    """The ViT layers of DPT (transformers' DPTViTLayer and BeitLayer share these names) under `prefix`: a missing key
    bias (BEiT's key projection has none) is zero; LayerScale is the lambdas when cfg["layer_scale"], else ones (exact in
    EPI_RESID_LS)."""
    D = cfg["hidden"]
    ones, out = np.ones(D, np.float32), {}
    for i in range(cfg["layers"]):
        p = f"{prefix}{i}."
        a = p + "attention.attention."
        kb = sd[a + "key.bias"] if a + "key.bias" in sd else torch.zeros(D)
        out[f"l{i}.ln1.g"] = _f32(sd[p + "layernorm_before.weight"])
        out[f"l{i}.ln1.b"] = _f32(sd[p + "layernorm_before.bias"])
        out[f"l{i}.qkv.w"] = _f16(torch.cat([sd[a + "query.weight"], sd[a + "key.weight"], sd[a + "value.weight"]], 0))
        out[f"l{i}.qkv.b"] = _f32(torch.cat([sd[a + "query.bias"], kb, sd[a + "value.bias"]], 0))
        out[f"l{i}.proj.w"] = _f16(sd[p + "attention.output.dense.weight"])
        out[f"l{i}.proj.b"] = _f32(sd[p + "attention.output.dense.bias"])
        out[f"l{i}.ls1"] = _f32(sd[p + "lambda_1"]) if cfg.get("layer_scale") else ones
        out[f"l{i}.ln2.g"] = _f32(sd[p + "layernorm_after.weight"])
        out[f"l{i}.ln2.b"] = _f32(sd[p + "layernorm_after.bias"])
        out[f"l{i}.fc1.w"] = _f16(sd[p + "intermediate.dense.weight"])
        out[f"l{i}.fc1.b"] = _f32(sd[p + "intermediate.dense.bias"])
        out[f"l{i}.fc2.w"] = _f16(sd[p + "output.dense.weight"])
        out[f"l{i}.fc2.b"] = _f32(sd[p + "output.dense.bias"])
        out[f"l{i}.ls2"] = _f32(sd[p + "lambda_2"]) if cfg.get("layer_scale") else ones
    return out


def _prepare_dpt_neck(sd, cfg, readouts, direct=()):
    """DPT's project readouts `readouts` (split into their token and CLS halves) and the neck, fusion and head."""
    D = cfg["hidden"]
    out = {}
    for i in readouts:
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
    out.update(_prepare_tail(shared, cfg, direct))
    return out


# ---------------------------------------------------------------------------
# DPT-Hybrid / MiDaS 3.0 (Intel/dpt-hybrid-midas; transformers 5.5 DPTForDepthEstimation with is_hybrid=True): a BiT
# ResNet-50 front end (BitConfig layer_type "bottleneck", global_padding "SAME", depths [3, 4, 9], 32 groups) whose
# stage-3 map, projected 1024 -> hidden by a 1x1 conv, is the ViT-B/16's token grid; the stage-1 and stage-2 maps are
# neck inputs 0 and 1 as they are; the residual stream after layers 9 and 12 (backbone_out_indices[2:]) feeds readouts
# 2 and 3.  From the ViT on it is DPT-Large's path.
# ---------------------------------------------------------------------------
DPT_HYBRID_CONFIGS = {
    "dpt-hybrid-midas": dict(hidden=768, layers=12, heads=12, taps=[3, 6, 9, 12], neck=[256, 512, 768, 768],
                             fusion=256, patch=16, ln_eps=1e-12, image_size=384),
}
BIT_DEPTHS, BIT_WIDTHS, BIT_GROUPS = (3, 4, 9), (256, 512, 1024), 32


def hf_dpt_hybrid_config(name="dpt-hybrid-midas", **cfg):
    """transformers DPTConfig of the hybrid checkpoint (Intel/dpt-hybrid-midas's config.json as far as the engine reads
    it); `cfg` overrides entries of DPT_HYBRID_CONFIGS[name] (a smaller ViT and image for tests)."""
    from transformers import DPTConfig
    c = dict(DPT_HYBRID_CONFIGS[name], **cfg)
    g = c["image_size"] // c["patch"]
    return DPTConfig(hidden_size=c["hidden"], num_hidden_layers=c["layers"], num_attention_heads=c["heads"],
                     intermediate_size=4 * c["hidden"], hidden_act="gelu", layer_norm_eps=c["ln_eps"],
                     image_size=c["image_size"], patch_size=c["patch"], num_channels=3, qkv_bias=True,
                     is_hybrid=True, backbone_out_indices=[t - 1 for t in c["taps"]], readout_type="project",
                     reassemble_factors=[1, 1, 1, 0.5], neck_hidden_sizes=c["neck"], fusion_hidden_size=c["fusion"],
                     head_in_index=-1, use_batch_norm_in_fusion_residual=False, use_bias_in_fusion_residual=None,
                     add_projection=False, backbone_featmap_shape=[1, 1024, g, g],
                     backbone_config=dict(model_type="bit", layer_type="bottleneck", global_padding="same",
                                          embedding_dynamic_padding=True, depths=list(BIT_DEPTHS),
                                          hidden_sizes=[256, 512, 1024, 2048], embedding_size=64,
                                          num_groups=BIT_GROUPS, hidden_act="relu",
                                          out_features=["stage1", "stage2", "stage3"]))


def dpt_hybrid_config_from_json(cj):
    """The engine configuration of a DPT-Hybrid config.json (dict), or ValueError naming the field the engine does not
    serve: the backbone must be BiT's bottleneck ResNet with SAME padding, depths [3, 4, 9], widths 256 / 512 / 1024 and
    32 groups; readout "project", reassemble_factors [1, 1, 1, 0.5], neck_hidden_sizes[:2] [256, 512], no head
    projection or batch-norm fusion units."""
    def bad(field, value):
        raise ValueError(f"config.json: {field} = {value!r} is not served (DPT-Hybrid: BiT ResNet-50 stages 1-3 and a "
                         "ViT with project readout)")
    if cj.get("model_type", "dpt") != "dpt":
        bad("model_type", cj.get("model_type"))
    if cj.get("is_hybrid") is not True:
        bad("is_hybrid", cj.get("is_hybrid"))
    bj = cj.get("backbone_config")
    if not isinstance(bj, dict):
        bad("backbone_config", bj)
    if bj.get("model_type", "bit") != "bit":
        bad("backbone_config.model_type", bj.get("model_type"))
    if bj.get("layer_type") != "bottleneck":
        bad("backbone_config.layer_type", bj.get("layer_type"))
    if str(bj.get("global_padding", "")).upper() != "SAME":
        bad("backbone_config.global_padding", bj.get("global_padding"))
    if bj.get("embedding_dynamic_padding") is not True:
        bad("backbone_config.embedding_dynamic_padding", bj.get("embedding_dynamic_padding"))
    if list(bj.get("depths", [])) != list(BIT_DEPTHS):
        bad("backbone_config.depths", bj.get("depths"))
    hs = bj.get("hidden_sizes", [])
    if list(hs)[:3] != list(BIT_WIDTHS):
        bad("backbone_config.hidden_sizes", hs)
    for field, want in (("num_groups", BIT_GROUPS), ("embedding_size", 64), ("num_channels", 3),
                        ("hidden_act", "relu"), ("width_factor", 1), ("output_stride", 32)):
        if bj.get(field, want) != want:
            bad(f"backbone_config.{field}", bj.get(field))
    if list(bj.get("out_features", ["stage1", "stage2", "stage3"])) != ["stage1", "stage2", "stage3"]:
        bad("backbone_config.out_features", bj.get("out_features"))
    if cj.get("readout_type", "project") != "project":
        bad("readout_type", cj.get("readout_type"))
    if [float(f) for f in cj.get("reassemble_factors", [4, 2, 1, 0.5])] != [1.0, 1.0, 1.0, 0.5]:
        bad("reassemble_factors", cj.get("reassemble_factors"))
    neck = cj.get("neck_hidden_sizes", [96, 192, 384, 768])
    if not isinstance(neck, (list, tuple)) or len(neck) != 4 or list(neck[:2]) != [256, 512]:
        bad("neck_hidden_sizes", neck)
    if cj.get("add_projection"):
        bad("add_projection", cj.get("add_projection"))
    if cj.get("use_batch_norm_in_fusion_residual"):
        bad("use_batch_norm_in_fusion_residual", cj.get("use_batch_norm_in_fusion_residual"))
    if cj.get("use_bias_in_fusion_residual") is False:
        bad("use_bias_in_fusion_residual", False)
    if cj.get("hidden_act", "gelu") != "gelu":
        bad("hidden_act", cj.get("hidden_act"))
    if cj.get("head_in_index", -1) != -1:
        bad("head_in_index", cj.get("head_in_index"))
    hidden = int(cj.get("hidden_size", 768))
    heads = int(cj.get("num_attention_heads", 12))
    if int(cj.get("intermediate_size", 4 * hidden)) != 4 * hidden:
        bad("intermediate_size", cj.get("intermediate_size"))
    if hidden != 64 * heads:
        bad("hidden_size / num_attention_heads", (hidden, heads))
    if int(cj.get("patch_size", 16)) != 16:
        bad("patch_size", cj.get("patch_size"))
    layers = int(cj.get("num_hidden_layers", 12))
    taps = cj.get("backbone_out_indices", [2, 5, 8, 11])
    if (not isinstance(taps, (list, tuple)) or len(taps) != 4 or any(type(t) is not int for t in taps)
            or not 0 <= taps[0] < taps[1] < taps[2] < taps[3] < layers):
        bad("backbone_out_indices", taps)
    size = cj.get("image_size", 384)
    fmap = cj.get("backbone_featmap_shape", [1, 1024, size // 16, size // 16])
    if list(fmap)[1:] != [1024, size // 16, size // 16]:
        bad("backbone_featmap_shape", fmap)
    return dict(hidden=hidden, layers=layers, heads=heads, taps=[int(t) + 1 for t in taps],
                neck=[int(v) for v in neck], fusion=int(cj.get("fusion_hidden_size", 256)), patch=16,
                ln_eps=float(cj.get("layer_norm_eps", 1e-12)), image_size=int(size))


_BIT = "dpt.embeddings.backbone.bit."


def dpt_hybrid_keys(cfg):
    """Every state_dict key (and its shape) the DPT-Hybrid depth forward reads: DPT's keys without the patch embedding,
    readouts 0 / 1 and reassemble layers 0 / 1, plus the BiT stem and stages and the 1x1 projection."""
    k = {n: v for n, v in dpt_keys(cfg).items() if not n.startswith("dpt.embeddings.patch_embeddings.")
         and not any(n.startswith(f"neck.reassemble_stage.{m}.{i}.") for m in ("readout_projects", "layers")
                     for i in (0, 1))}
    k[_BIT + "embedder.convolution.weight"] = (64, 3, 7, 7)
    k[_BIT + "embedder.norm.weight"] = k[_BIT + "embedder.norm.bias"] = (64,)
    cin = 64
    for st, (depth, out_c) in enumerate(zip(BIT_DEPTHS, BIT_WIDTHS)):
        mid = out_c // 4
        for b in range(depth):
            p = f"{_BIT}encoder.stages.{st}.layers.{b}."
            if b == 0:
                k[p + "downsample.conv.weight"] = (out_c, cin, 1, 1)
                k[p + "downsample.norm.weight"] = k[p + "downsample.norm.bias"] = (out_c,)
            k[p + "conv1.weight"] = (mid, cin if b == 0 else out_c, 1, 1)
            k[p + "conv2.weight"] = (mid, mid, 3, 3)
            k[p + "conv3.weight"] = (out_c, mid, 1, 1)
            for n, c in (("norm1", mid), ("norm2", mid), ("norm3", out_c)):
                k[p + n + ".weight"] = k[p + n + ".bias"] = (c,)
        cin = out_c
    k["dpt.embeddings.projection.weight"] = (cfg["hidden"], 1024, 1, 1)
    k["dpt.embeddings.projection.bias"] = (cfg["hidden"],)
    return k


def check_dpt_hybrid_state_dict(sd, cfg):
    """ValueError naming the first missing or mis-shaped key the DPT-Hybrid forward reads."""
    for name, shape in dpt_hybrid_keys(cfg).items():
        if name not in sd:
            raise ValueError(f"DPT-Hybrid state dict: missing key {name}")
        if tuple(sd[name].shape) != shape:
            raise ValueError(f"DPT-Hybrid state dict: {name} has shape {tuple(sd[name].shape)}, expected {shape}")


def standardize_weight(w, eps=1e-8):
    """BiT's weight standardisation (WeightStandardizedConv2d: batch_norm over each output channel's weights, biased
    variance, eps 1e-8) in float64: (w - mean) / sqrt(var + eps)."""
    w = w.detach().double()
    flat = w.reshape(w.shape[0], -1)
    m = flat.mean(dim=1, keepdim=True)
    v = ((flat - m) ** 2).mean(dim=1, keepdim=True)
    return ((flat - m) / torch.sqrt(v + eps)).reshape(w.shape)


def prepare_dpt_hybrid(sd, cfg, image_h, image_w):
    """DPT-Hybrid state_dict -> {name: np.ndarray} in the layouts depth_engine.cu expects: the BiT convs weight-
    standardised in float64 at load time, then f16 ("bit.s{st}.b{k}.c{1,2,3}.w", ".ds.w"; 3x3 kernels tap-major) or
    f32 for the stem conv, which runs in f32 ("bit.stem.w" [64, 147]); GroupNorm affines f32; the 1x1 projection as
    "pe.w" / "pe.b"; the ViT, readouts 2 / 3, neck, fusion and head as for DPT-Large."""
    check_dpt_hybrid_state_dict(sd, cfg)
    D = cfg["hidden"]
    out = {"bit.stem.w": _f32(standardize_weight(sd[_BIT + "embedder.convolution.weight"]).reshape(64, 147)),
           "bit.stem.g": _f32(sd[_BIT + "embedder.norm.weight"]), "bit.stem.b": _f32(sd[_BIT + "embedder.norm.bias"])}
    for st, depth in enumerate(BIT_DEPTHS):
        for b in range(depth):
            p = f"{_BIT}encoder.stages.{st}.layers.{b}."
            q = f"bit.s{st}.b{b}."
            w1 = standardize_weight(sd[p + "conv1.weight"])
            out[q + "c1.w"] = _f16(w1.reshape(w1.shape[0], -1))
            out[q + "c2.w"] = _conv3(standardize_weight(sd[p + "conv2.weight"]), sd[p + "conv2.weight"].shape[1])
            w3 = standardize_weight(sd[p + "conv3.weight"])
            out[q + "c3.w"] = _f16(w3.reshape(w3.shape[0], -1))
            for i in (1, 2, 3):
                out[q + f"n{i}.g"] = _f32(sd[p + f"norm{i}.weight"])
                out[q + f"n{i}.b"] = _f32(sd[p + f"norm{i}.bias"])
            if b == 0:
                wd = standardize_weight(sd[p + "downsample.conv.weight"])
                out[q + "ds.w"] = _f16(wd.reshape(wd.shape[0], -1))
                out[q + "ds.g"] = _f32(sd[p + "downsample.norm.weight"])
                out[q + "ds.b"] = _f32(sd[p + "downsample.norm.bias"])
    out["pe.w"] = _f16(sd["dpt.embeddings.projection.weight"].float().reshape(D, 1024))
    out["pe.b"] = _f32(sd["dpt.embeddings.projection.bias"])
    out.update(_prepare_dpt_vit(sd, cfg, image_h, image_w, (2, 3), direct=(0, 1)))
    return out


# ---------------------------------------------------------------------------
# DPT-BEiT (Intel/dpt-beit-large-512, MiDaS v3.1 BEiT-L 512; transformers 5.5 DPTForDepthEstimation whose backbone is
# BeitBackbone, built by load_backbone, state dict prefix "backbone."): a BEiT-L/16 with LayerScale, no absolute
# position embedding, and a relative position bias per layer (BeitRelativePositionBias: a [(2 W - 1)^2 + 3, heads] table
# for the pretrained W x W window, resampled bilinearly to the input's grid); its key projection has no bias.  Taps =
# the raw hidden states (CLS included) after the out_indices layers; from there on DPT-Large's path.
# ---------------------------------------------------------------------------
DPT_BEIT_CONFIGS = {
    "dpt-beit-large-512": dict(hidden=1024, layers=24, heads=16, taps=[6, 12, 18, 24], neck=[256, 512, 1024, 1024],
                               fusion=256, patch=16, ln_eps=1e-12, image_size=512, layer_scale=True),
}

# DPTImageProcessor as MiDaS v3.1's BEiT checkpoints are expected to configure it: keep the aspect ratio, sides
# multiples of 32 near 512, bicubic, mean = std = 0.5.  The checkpoint's preprocessor_config.json is what the drivers read.
DPT_BEIT_PROCESSOR = dict(size=(512, 512), resample=3, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5), keep_aspect=True,
                          multiple=32)


def hf_dpt_beit_config(name="dpt-beit-large-512", **cfg):
    """transformers DPTConfig with a BeitConfig backbone equal to the checkpoint's as far as the engine reads it; `cfg`
    overrides entries of DPT_BEIT_CONFIGS[name] (a smaller BEiT for tests; layer_scale False: no lambdas)."""
    from transformers import BeitConfig, DPTConfig
    c = dict(DPT_BEIT_CONFIGS[name], **cfg)
    bc = BeitConfig(image_size=c["image_size"], patch_size=c["patch"], num_channels=3, hidden_size=c["hidden"],
                    num_hidden_layers=c["layers"], num_attention_heads=c["heads"], intermediate_size=4 * c["hidden"],
                    hidden_act="gelu", layer_norm_eps=c["ln_eps"], use_mask_token=False,
                    use_absolute_position_embeddings=False, use_relative_position_bias=True,
                    use_shared_relative_position_bias=False, layer_scale_init_value=0.1 if c["layer_scale"] else 0.0,
                    out_indices=list(c["taps"]), reshape_hidden_states=False, add_fpn=False)
    return DPTConfig(backbone_config=bc, hidden_size=c["hidden"], is_hybrid=False, readout_type="project",
                     reassemble_factors=[4, 2, 1, 0.5], neck_hidden_sizes=c["neck"], fusion_hidden_size=c["fusion"],
                     head_in_index=-1, use_batch_norm_in_fusion_residual=False, use_bias_in_fusion_residual=None,
                     add_projection=False)


def dpt_beit_config_from_json(cj):
    """The engine configuration of a DPT config.json (dict) with a BEiT backbone, or ValueError naming every field the
    engine does not compute: absolute position embeddings, a shared relative bias, no relative bias, reshaped hidden
    states, an FPN, a patch other than 16, a head size other than 64, an activation other than GELU, taps that are not
    four increasing layers, a readout other than "project", and the neck / fusion / head options DPT-Large does not
    serve.  layer_scale_init_value 0 means no LayerScale (ones)."""
    bad = []
    if cj.get("model_type", "dpt") != "dpt":
        bad.append(("model_type", cj.get("model_type")))
    if cj.get("is_hybrid"):
        bad.append(("is_hybrid", cj.get("is_hybrid")))
    bj = cj.get("backbone_config")
    if not isinstance(bj, dict) or bj.get("model_type") != "beit":
        raise ValueError(f"config.json: backbone_config = {bj!r} is not a BEiT backbone")
    for field, want in (("use_absolute_position_embeddings", False), ("use_shared_relative_position_bias", False),
                        ("use_relative_position_bias", True), ("reshape_hidden_states", False), ("add_fpn", False)):
        default = {"use_relative_position_bias": False, "reshape_hidden_states": True}.get(field, False)
        if bool(bj.get(field, default)) is not want:
            bad.append((f"backbone_config.{field}", bj.get(field, default)))
    if bj.get("patch_size", 16) != 16:
        bad.append(("backbone_config.patch_size", bj.get("patch_size")))
    if bj.get("num_channels", 3) != 3:
        bad.append(("backbone_config.num_channels", bj.get("num_channels")))
    hidden, layers, heads = (int(bj.get("hidden_size", 768)), int(bj.get("num_hidden_layers", 12)),
                             int(bj.get("num_attention_heads", 12)))
    if hidden != 64 * heads or hidden % 128 or hidden > 1024:
        bad.append(("backbone_config.hidden_size / num_attention_heads", (hidden, heads)))
    if int(bj.get("intermediate_size", 3072)) != 4 * hidden:
        bad.append(("backbone_config.intermediate_size", bj.get("intermediate_size", 3072)))
    if bj.get("hidden_act", "gelu") != "gelu":
        bad.append(("backbone_config.hidden_act", bj.get("hidden_act")))
    taps = bj.get("out_indices")
    if taps is None and isinstance(bj.get("out_features"), (list, tuple)):
        taps = [int(f[5:]) if isinstance(f, str) and f.startswith("stage") and f[5:].isdigit() else f
                for f in bj["out_features"]]
    if (not isinstance(taps, (list, tuple)) or len(taps) != 4 or any(type(t) is not int for t in taps)
            or not 1 <= taps[0] < taps[1] < taps[2] < taps[3] <= layers):
        bad.append(("backbone_config.out_indices", taps))
    if cj.get("readout_type", "project") != "project":
        bad.append(("readout_type", cj.get("readout_type")))
    if [float(f) for f in cj.get("reassemble_factors", [4, 2, 1, 0.5])] != [4.0, 2.0, 1.0, 0.5]:
        bad.append(("reassemble_factors", cj.get("reassemble_factors")))
    neck = cj.get("neck_hidden_sizes", [96, 192, 384, 768])
    if not isinstance(neck, (list, tuple)) or len(neck) != 4 or any(type(v) is not int or v < 1 for v in neck):
        bad.append(("neck_hidden_sizes", neck))
    fusion = cj.get("fusion_hidden_size", 256)
    if type(fusion) is not int or fusion < 64 or fusion % 64:
        bad.append(("fusion_hidden_size", fusion))
    for field, default in (("add_projection", False), ("use_batch_norm_in_fusion_residual", False)):
        if cj.get(field, default):
            bad.append((field, cj.get(field)))
    if cj.get("use_bias_in_fusion_residual") is False:
        bad.append(("use_bias_in_fusion_residual", False))
    if cj.get("head_in_index", -1) != -1:
        bad.append(("head_in_index", cj.get("head_in_index")))
    if bad:
        raise ValueError("config.json: " + ", ".join(f"{f} = {v!r}" for f, v in bad) + " not served (DPT on a BEiT "
                         "backbone with its own relative position bias per layer and the project readout)")
    ls = bj.get("layer_scale_init_value", 0.1)
    return dict(hidden=hidden, layers=layers, heads=heads, taps=list(taps), neck=list(neck), fusion=fusion, patch=16,
                ln_eps=float(bj.get("layer_norm_eps", 1e-12)), image_size=int(bj.get("image_size", 224)),
                layer_scale=bool(ls > 0))


def dpt_beit_processor_from_json(pj):
    """DPT_BEIT_PROCESSOR updated from a preprocessor_config.json (dict), or ValueError: keep_aspect_ratio with
    ensure_multiple_of 32, or a fixed size whose sides are multiples of 32; bicubic or bilinear; 1/255; no padding."""
    def bad(field, value):
        raise ValueError(f"preprocessor_config.json: {field} = {value!r} is not served (DPT processor: keep_aspect_ratio "
                         "with ensure_multiple_of 32, or a fixed size of multiples of 32)")
    for field in ("do_resize", "do_rescale", "do_normalize"):
        if pj.get(field, True) is not True:
            bad(field, pj.get(field))
    if pj.get("do_pad"):
        bad("do_pad", pj.get("do_pad"))
    rf = pj.get("rescale_factor", 1 / 255)
    if not isinstance(rf, (int, float)) or abs(rf - 1 / 255) > 1e-9:
        bad("rescale_factor", rf)
    size = pj.get("size", {"height": 384, "width": 384})
    if isinstance(size, int):
        size = {"height": size, "width": size}
    if not isinstance(size, dict) or type(size.get("height")) is not int or type(size.get("width")) is not int:
        bad("size", size)
    h, w = size["height"], size["width"]
    keep, mult = bool(pj.get("keep_aspect_ratio", False)), pj.get("ensure_multiple_of", 1)
    if keep and mult != 32:
        bad("ensure_multiple_of", mult)
    if not keep and (mult not in (1, 32) or h % 32 or w % 32):
        bad("size / ensure_multiple_of", (size, mult))
    if h < 32 or w < 32:
        bad("size", size)
    p = dict(DPT_BEIT_PROCESSOR, size=(h, w), keep_aspect=keep, multiple=32 if keep else 0)
    p["resample"] = pj.get("resample", 3)
    if p["resample"] not in (2, 3):
        bad("resample", p["resample"])
    for k, key in (("mean", "image_mean"), ("std", "image_std")):
        if key in pj:
            v = pj[key]
            v = v if isinstance(v, (list, tuple)) else [v] * 3
            if len(v) != 3 or any(not isinstance(x, (int, float)) for x in v):
                bad(key, pj[key])
            p[k] = tuple(float(x) for x in v)
    return p


def dpt_beit_processed_size(width, height, processor=None):
    """(h, w) a DPT-BEiT processor resizes a (width, height) image to: DPTImageProcessor's keep-aspect size (the side
    whose scale to the target is closer to 1 sets both, each rounded to a multiple of 32) or its fixed size."""
    p = processor or DPT_BEIT_PROCESSOR
    th, tw = p["size"]
    if not p["keep_aspect"]:
        return th, tw
    sh, sw = th / height, tw / width
    if abs(1 - sw) < abs(1 - sh):
        sh = sw
    else:
        sw = sh
    m = p["multiple"]
    rnd = lambda v: max(m, int(round(v / m) * m))  # noqa: E731
    return rnd(sh * height), rnd(sw * width)


_BEIT = "backbone."


def dpt_beit_keys(cfg):
    """Every state_dict key (and its shape) the DPT-BEiT depth forward reads."""
    D, L, P, H = cfg["hidden"], cfg["layers"], cfg["patch"], cfg["heads"]
    W = cfg["image_size"] // P
    k = {_BEIT + "embeddings.cls_token": (1, 1, D), _BEIT + "embeddings.patch_embeddings.projection.weight": (D, 3, P, P),
         _BEIT + "embeddings.patch_embeddings.projection.bias": (D,)}
    for i in range(L):
        p = f"{_BEIT}encoder.layer.{i}."
        a = p + "attention.attention."
        for n in ("layernorm_before", "layernorm_after"):
            k[p + n + ".weight"] = k[p + n + ".bias"] = (D,)
        for n in ("query", "key", "value"):
            k[a + n + ".weight"] = (D, D)
        k[a + "query.bias"] = k[a + "value.bias"] = (D,)
        k[a + "relative_position_bias.relative_position_bias_table"] = ((2 * W - 1) ** 2 + 3, H)
        if cfg.get("layer_scale"):
            k[p + "lambda_1"] = k[p + "lambda_2"] = (D,)
        k[p + "attention.output.dense.weight"], k[p + "attention.output.dense.bias"] = (D, D), (D,)
        k[p + "intermediate.dense.weight"], k[p + "intermediate.dense.bias"] = (4 * D, D), (4 * D,)
        k[p + "output.dense.weight"], k[p + "output.dense.bias"] = (D, 4 * D), (D,)
    k.update({n: v for n, v in dpt_keys(cfg).items() if not n.startswith("dpt.")})
    return k


def check_dpt_beit_state_dict(sd, cfg):
    """ValueError naming the first missing or mis-shaped key the DPT-BEiT forward reads.  Other keys (the
    relative_position_index buffers, a mask_token, a key bias, which a softmax row does not see) are ignored."""
    for name, shape in dpt_beit_keys(cfg).items():
        if name not in sd:
            raise ValueError(f"DPT-BEiT state dict: missing key {name}")
        if tuple(sd[name].shape) != shape:
            raise ValueError(f"DPT-BEiT state dict: {name} has shape {tuple(sd[name].shape)}, expected {shape}")


def beit_bias_table(table, window, grid):
    """BeitRelativePositionBias.forward's table for a token grid (ph, pw) from the pretrained window's [(2 Wh - 1)
    (2 Ww - 1) + 3, heads] table, with the same torch ops in fp32 on the CPU: the (2 Wh - 1) x (2 Ww - 1) part resampled
    bilinearly (align_corners False) to (2 ph - 1) x (2 pw - 1), the three CLS entries appended as they are."""
    t = table.detach().to(device="cpu", dtype=torch.float32)
    old_h, old_w = 2 * window[0] - 1, 2 * window[1] - 1
    new_h, new_w = 2 * grid[0] - 1, 2 * grid[1] - 1
    n_old = old_h * old_w
    sub = t[:n_old].reshape(1, old_w, old_h, -1).permute(0, 3, 1, 2)
    sub = F.interpolate(sub, size=(new_h, new_w), mode="bilinear")
    sub = sub.permute(0, 2, 3, 1).reshape(new_h * new_w, -1)
    return torch.cat([sub, t[n_old:]])


def prepare_dpt_beit(sd, cfg, image_h, image_w):
    """DPT-BEiT state_dict -> {name: np.ndarray} in the layouts depth_engine.cu expects: DPT-Large's with the lambdas as
    LayerScale, a zero key bias, a zero "pos" (BEiT has no absolute position embedding: EPI_PATCH adds 0, exactly), and
    "l{i}.rpb" f32 [heads, (2 ph - 1)(2 pw - 1) + 3], each layer's table resampled to the image_h x image_w grid."""
    check_dpt_beit_state_dict(sd, cfg)
    D, P = cfg["hidden"], cfg["patch"]
    ph, pw = image_h // P, image_w // P
    W = cfg["image_size"] // P
    e = _BEIT + "embeddings."
    out = {"pe.w": _f16(sd[e + "patch_embeddings.projection.weight"].float().reshape(D, 3 * P * P)),
           "pe.b": _f32(sd[e + "patch_embeddings.projection.bias"]),
           "cls": _f32(sd[e + "cls_token"].reshape(D)), "pos": np.zeros((ph * pw + 1, D), np.float32)}
    out.update(_prepare_dpt_layers(sd, cfg, _BEIT + "encoder.layer."))
    for i in range(cfg["layers"]):
        t = sd[f"{_BEIT}encoder.layer.{i}.attention.attention.relative_position_bias.relative_position_bias_table"]
        out[f"l{i}.rpb"] = _f32(beit_bias_table(t, (W, W), (ph, pw)).t())
    out.update(_prepare_dpt_neck(sd, cfg, range(4)))
    return out


# ---------------------------------------------------------------------------
# ZoeDepth (Intel/zoedepth-nyu-kitti, -nyu, -kitti; transformers 5.5 ZoeDepthForDepthEstimation): dpt-beit-large-512's
# trunk, neck and fusion on a BEiT-L/16 with a 24 x 24 pretraining window, DPT's relative head up to its conv2 + ReLU,
# then the metric-bins head (softplus seed bins, four unnormed attractor layers, the conditional log-binomial).  The
# two-configuration checkpoint routes each image through a patch transformer + MLP classifier.
# ---------------------------------------------------------------------------
ZOEDEPTH_CONFIGS = {
    "zoedepth-nyu-kitti": dict(DPT_BEIT_CONFIGS["dpt-beit-large-512"], image_size=384,
                               bins=[dict(name="nyu", n_bins=64, min_depth=1e-3, max_depth=10.0),
                                     dict(name="kitti", n_bins=64, min_depth=1e-3, max_depth=80.0)],
                               attractors=[16, 8, 4, 1], min_temp=0.0212, max_temp=50.0, bottleneck=256, embed=128),
    "zoedepth-nyu": dict(DPT_BEIT_CONFIGS["dpt-beit-large-512"], image_size=384,
                         bins=[dict(name="nyu", n_bins=64, min_depth=1e-3, max_depth=10.0)],
                         attractors=[16, 8, 4, 1], min_temp=0.0212, max_temp=50.0, bottleneck=256, embed=128),
}
ZOEDEPTH_CONFIGS["zoedepth-kitti"] = dict(ZOEDEPTH_CONFIGS["zoedepth-nyu"],
                                          bins=[dict(name="kitti", n_bins=64, min_depth=1e-3, max_depth=80.0)])

# ZoeDepthImageProcessor as the checkpoints configure it: reflect padding, keep-aspect multiples of 32 near 384 x 512,
# bilinear with align_corners, mean = std = 0.5.  The checkpoint's preprocessor_config.json is what the drivers read.
ZOEDEPTH_PROCESSOR = dict(size=(384, 512), resample=2, mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5), keep_aspect=True,
                          multiple=32)


def hf_zoedepth_config(name="zoedepth-nyu-kitti", **cfg):
    """transformers ZoeDepthConfig equal to the checkpoint's as far as the engine reads it; `cfg` overrides entries of
    ZOEDEPTH_CONFIGS[name] (a smaller BEiT for tests)."""
    from transformers import BeitConfig, ZoeDepthConfig
    c = dict(ZOEDEPTH_CONFIGS[name], **cfg)
    bc = BeitConfig(image_size=c["image_size"], patch_size=c["patch"], num_channels=3, hidden_size=c["hidden"],
                    num_hidden_layers=c["layers"], num_attention_heads=c["heads"], intermediate_size=4 * c["hidden"],
                    hidden_act="gelu", layer_norm_eps=c["ln_eps"], use_mask_token=False,
                    use_absolute_position_embeddings=False, use_relative_position_bias=True,
                    use_shared_relative_position_bias=False, layer_scale_init_value=0.1 if c["layer_scale"] else 0.0,
                    out_indices=list(c["taps"]), reshape_hidden_states=False, add_fpn=False)
    multi = len(c["bins"]) > 1
    return ZoeDepthConfig(backbone_config=bc, readout_type="project", reassemble_factors=[4, 2, 1, 0.5],
                          neck_hidden_sizes=c["neck"], fusion_hidden_size=c["fusion"], head_in_index=-1,
                          use_batch_norm_in_fusion_residual=False, use_bias_in_fusion_residual=None,
                          num_relative_features=32, add_projection=False, bottleneck_features=c["bottleneck"],
                          num_attractors=list(c["attractors"]), bin_embedding_dim=c["embed"], attractor_alpha=1000,
                          attractor_gamma=2, attractor_kind="mean", min_temp=c["min_temp"], max_temp=c["max_temp"],
                          bin_centers_type="softplus", bin_configurations=[dict(b) for b in c["bins"]],
                          num_patch_transformer_layers=4 if multi else None,
                          patch_transformer_hidden_size=128 if multi else None,
                          patch_transformer_intermediate_size=1024 if multi else None,
                          patch_transformer_num_attention_heads=4 if multi else None)


def zoedepth_config_from_json(cj):
    """The engine configuration of a ZoeDepth config.json (dict), or ValueError naming every field the engine does not
    compute: a non-BEiT backbone (and the BEiT fields dpt_beit_config_from_json refuses), a "normed" bin type, an
    attractor kind other than "mean", add_projection, batch norm in fusion, a bin_configurations list of other than 1
    or 2 entries or with n_bins other than 64, a bin embedding other than 128 or a bottleneck other than the fusion
    width, a relative feature count other than 32, and a patch transformer other than 4 layers of 128 / 4 heads / 1024.
    transformers ignores attractor_alpha / attractor_gamma (inv_attractor runs with 300 / 2), and so does the engine."""
    bad = []
    if cj.get("model_type") != "zoedepth":
        bad.append(("model_type", cj.get("model_type")))
    try:
        base = dpt_beit_config_from_json(dict(cj, model_type="dpt"))
    except ValueError as ex:
        bad.append(("backbone / neck", str(ex)))
        base = None
    for field, want in (("bin_centers_type", "softplus"), ("attractor_kind", "mean")):
        if cj.get(field, want) != want:
            bad.append((field, cj.get(field)))
    if cj.get("num_relative_features", 32) != 32:
        bad.append(("num_relative_features", cj.get("num_relative_features")))
    if cj.get("bin_embedding_dim", 128) != 128:
        bad.append(("bin_embedding_dim", cj.get("bin_embedding_dim")))
    fusion = cj.get("fusion_hidden_size", 256)
    if cj.get("bottleneck_features", 256) != fusion:
        bad.append(("bottleneck_features", cj.get("bottleneck_features")))
    bins = cj.get("bin_configurations") or [{"n_bins": 64, "min_depth": 0.001, "max_depth": 10.0}]
    if not isinstance(bins, list) or len(bins) not in (1, 2):
        bad.append(("bin_configurations", bins))
        bins = []
    for b in bins:
        if (not isinstance(b, dict) or b.get("n_bins") != 64
                or not 0 <= float(b.get("min_depth", -1)) < float(b.get("max_depth", -1))):
            bad.append(("bin_configurations", b))
    att = cj.get("num_attractors", [16, 8, 4, 1])
    if not isinstance(att, list) or len(att) != 4 or any(type(a) is not int or not 1 <= a <= 16 for a in att):
        bad.append(("num_attractors", att))
    if len(bins) == 2:
        for field, want in (("num_patch_transformer_layers", 4), ("patch_transformer_hidden_size", 128),
                            ("patch_transformer_intermediate_size", 1024),
                            ("patch_transformer_num_attention_heads", 4)):
            if cj.get(field) != want:
                bad.append((field, cj.get(field)))
    tmin, tmax = cj.get("min_temp", 0.0212), cj.get("max_temp", 50.0)
    if not (isinstance(tmin, (int, float)) and isinstance(tmax, (int, float)) and 0 < tmin < tmax):
        bad.append(("min_temp / max_temp", (tmin, tmax)))
    if bad:
        raise ValueError("config.json: " + ", ".join(f"{f} = {v!r}" for f, v in bad) + " not served (ZoeDepth: BEiT "
                         "trunk, softplus bins with unnormed mean attractors, one or two bin configurations)")
    bj = cj["backbone_config"]
    return dict(base, image_size=int(bj.get("image_size", 384)),
                bins=[dict(name=b.get("name", f"c{i}"), n_bins=64, min_depth=float(b["min_depth"]),
                           max_depth=float(b["max_depth"])) for i, b in enumerate(bins)],
                attractors=list(att), min_temp=float(tmin), max_temp=float(tmax), bottleneck=fusion, embed=128)


def zoedepth_processor_from_json(pj):
    """ZOEDEPTH_PROCESSOR updated from a preprocessor_config.json (dict), or ValueError: padding on, keep_aspect_ratio
    with ensure_multiple_of 32 (the class default 1/32 is not served), bilinear, 1/255."""
    def bad(field, value):
        raise ValueError(f"preprocessor_config.json: {field} = {value!r} is not served (ZoeDepth processor: reflect "
                         "padding, keep_aspect_ratio with ensure_multiple_of 32, bilinear)")
    for field in ("do_resize", "do_rescale", "do_normalize", "do_pad", "keep_aspect_ratio"):
        if field not in pj:
            bad(field, "missing")
        if pj[field] is not True:
            bad(field, pj[field])
    if pj.get("ensure_multiple_of") != 32:
        bad("ensure_multiple_of", pj.get("ensure_multiple_of"))
    rf = pj.get("rescale_factor", 1 / 255)
    if not isinstance(rf, (int, float)) or abs(rf - 1 / 255) > 1e-9:
        bad("rescale_factor", rf)
    if pj.get("resample", 2) != 2:
        bad("resample", pj.get("resample"))
    size = pj.get("size")
    if not isinstance(size, dict) or type(size.get("height")) is not int or type(size.get("width")) is not int \
            or size["height"] < 32 or size["width"] < 32:
        bad("size", size)
    p = dict(ZOEDEPTH_PROCESSOR, size=(size["height"], size["width"]))
    for k, key in (("mean", "image_mean"), ("std", "image_std")):
        if key in pj:
            v = pj[key]
            v = v if isinstance(v, (list, tuple)) else [v] * 3
            if len(v) != 3 or any(not isinstance(x, (int, float)) for x in v):
                bad(key, pj[key])
            p[k] = tuple(float(x) for x in v)
    return p


def zoedepth_pad(n):
    """ZoeDepthImageProcessor's reflect padding of a side of n pixels (post_process_depth_estimation crops the same)."""
    return int(np.sqrt(n / 2) * 3)


def zoedepth_processed_size(width, height, processor=None):
    """(h, w) ZoeDepthImageProcessor resizes a (width, height) image to: DPT's keep-aspect rule on the padded size."""
    return dpt_beit_processed_size(width + 2 * zoedepth_pad(width), height + 2 * zoedepth_pad(height),
                                   processor or ZOEDEPTH_PROCESSOR)


_ZM = "metric_head."


def zoedepth_keys(cfg):
    """Every state_dict key (and its shape) the ZoeDepth forward reads: the BEiT trunk and DPT neck of dpt_beit_keys
    (the relative head named relative_head.conv1..3) and the metric head."""
    F, E = cfg["fusion"], cfg["embed"]
    k = {n: v for n, v in dpt_beit_keys(cfg).items() if not n.startswith("head.")}
    F2 = F // 2
    k["relative_head.conv1.weight"], k["relative_head.conv1.bias"] = (F2, F, 3, 3), (F2,)
    k["relative_head.conv2.weight"], k["relative_head.conv2.bias"] = (32, F2, 3, 3), (32,)
    k["relative_head.conv3.weight"], k["relative_head.conv3.bias"] = (1, 32, 1, 1), (1,)
    multi = len(cfg["bins"]) > 1

    def conv(name, o, i):
        k[_ZM + name + ".weight"], k[_ZM + name + ".bias"] = (o, i, 1, 1), (o,)
    conv("conv2", F, F)
    mlp = E // 2 if multi else 128  # the projectors' hidden width (ZoeDepthProjector's default 128 on one configuration)
    conv("seed_projector.conv1", mlp, F)
    conv("seed_projector.conv2", E, mlp)
    for j in range(4):
        conv(f"projectors.{j}.conv1", mlp, F)
        conv(f"projectors.{j}.conv2", E, mlp)
    if multi:
        for c in cfg["bins"]:
            n = c["name"]
            conv(f"seed_bin_regressors.{n}.conv1", E // 2, F)
            conv(f"seed_bin_regressors.{n}.conv2", 64, E // 2)
            for j in range(4):
                conv(f"attractors.{n}.{j}.conv1", E, E)
                conv(f"attractors.{n}.{j}.conv2", 16, E)  # the constructor's default n_attractors on every layer
            conv(f"conditional_log_binomial.{n}.mlp.0", (32 + E) // 4, 32 + E)
            conv(f"conditional_log_binomial.{n}.mlp.2", 4, (32 + E) // 4)
        p = "patch_transformer."
        conv(p + "embedding_convPxP", 128, F)
        for i in range(4):
            a = f"{_ZM}{p}transformer_encoder.{i}."
            for n in ("query", "key", "value", "out_proj"):
                k[a + f"self_attn.{n}.weight"], k[a + f"self_attn.{n}.bias"] = (128, 128), (128,)
            k[a + "linear1.weight"], k[a + "linear1.bias"] = (1024, 128), (1024,)
            k[a + "linear2.weight"], k[a + "linear2.bias"] = (128, 1024), (128,)
            for n in ("norm1", "norm2"):
                k[a + n + ".weight"] = k[a + n + ".bias"] = (128,)
        for n, o in (("linear1", 128), ("linear2", 2)):
            k[f"{_ZM}mlp_classifier.{n}.weight"], k[f"{_ZM}mlp_classifier.{n}.bias"] = (o, 128), (o,)
    else:
        conv("seed_bin_regressor.conv1", 256, F)
        conv("seed_bin_regressor.conv2", 64, 256)
        for j, na in enumerate(cfg["attractors"]):
            conv(f"attractors.{j}.conv1", E, E)
            conv(f"attractors.{j}.conv2", na, E)
        conv("conditional_log_binomial.mlp.0", (33 + E) // 2, 33 + E)
        conv("conditional_log_binomial.mlp.2", 4, (33 + E) // 2)
    return k


def check_zoedepth_state_dict(sd, cfg):
    """ValueError naming the first missing or mis-shaped key the ZoeDepth forward reads."""
    for name, shape in zoedepth_keys(cfg).items():
        if name not in sd:
            raise ValueError(f"ZoeDepth state dict: missing key {name}")
        if tuple(sd[name].shape) != shape:
            raise ValueError(f"ZoeDepth state dict: {name} has shape {tuple(sd[name].shape)}, expected {shape}")


def zoedepth_attractors(sd, cfg):
    """Attractors per layer as the weights define them: 16 on every layer of the two-configuration head (transformers
    passes num_attractors to the unused n_bins), num_attractors on the single-configuration head."""
    if len(cfg["bins"]) > 1:
        n = cfg["bins"][0]["name"]
        return [int(sd[f"{_ZM}attractors.{n}.{j}.conv2.weight"].shape[0]) for j in range(4)]
    return [int(sd[f"{_ZM}attractors.{j}.conv2.weight"].shape[0]) for j in range(4)]


def zoedepth_position_code(n, dim=128):
    """ZoeDepthPatchTransformerEncoder.positional_encoding_1d for n tokens, with the same torch ops in f32."""
    position = torch.arange(0, n, dtype=torch.float32).unsqueeze(1)
    index = torch.arange(0, dim, 2, dtype=torch.float32).unsqueeze(0)
    div_term = torch.exp(index * (-torch.log(torch.tensor(10000.0)) / dim))
    pe = position * div_term
    return torch.cat([torch.sin(pe), torch.cos(pe)], dim=1)


def prepare_zoedepth(sd, cfg, image_h, image_w):
    """ZoeDepth state_dict -> {name: np.ndarray} in the layouts depth_engine.cu expects: prepare_dpt_beit's trunk, neck
    and relative head, and the metric head's "z.*" tensors (zoe_head in depth_engine.cu)."""
    check_zoedepth_state_dict(sd, cfg)
    sdb = {k: v for k, v in sd.items() if not k.startswith("relative_head.") and not k.startswith(_ZM)}
    for j, n in ((0, "conv1"), (2, "conv2"), (4, "conv3")):
        sdb[f"head.head.{j}.weight"] = sd[f"relative_head.{n}.weight"]
        sdb[f"head.head.{j}.bias"] = sd[f"relative_head.{n}.bias"]
    out = prepare_dpt_beit(sdb, cfg, image_h, image_w)
    names = [c["name"] for c in cfg["bins"]]
    multi = len(names) > 1

    def w2(name):
        return sd[_ZM + name + ".weight"].float().reshape(sd[_ZM + name + ".weight"].shape[0], -1)

    def b(name):
        return sd[_ZM + name + ".bias"].float()

    def put(dst, name):
        out[dst + ".w"], out[dst + ".b"] = _f16(w2(name)), _f32(b(name))
    put("z.bt", "conv2")
    put("z.sp1", "seed_projector.conv1")
    put("z.sp2", "seed_projector.conv2")
    for j in range(4):
        put(f"z.p{j}.1", f"projectors.{j}.conv1")
        put(f"z.p{j}.2", f"projectors.{j}.conv2")
    seed = [f"seed_bin_regressors.{n}" for n in names] if multi else ["seed_bin_regressor"]
    att = [f"attractors.{n}." for n in names] if multi else ["attractors."]
    clb = [f"conditional_log_binomial.{n}" for n in names] if multi else ["conditional_log_binomial"]
    out["z.s1.w"] = _f16(torch.cat([w2(s + ".conv1") for s in seed]))
    out["z.s1.b"] = _f32(torch.cat([b(s + ".conv1") for s in seed]))
    s2 = torch.block_diag(*[w2(s + ".conv2") for s in seed])  # each configuration's conv2 on its own seed columns
    out["z.s2.w"], out["z.s2.b"] = _f16(s2), _f32(torch.cat([b(s + ".conv2") for s in seed]))
    for j in range(4):
        out[f"z.a{j}.1.w"] = _f16(torch.cat([w2(a + f"{j}.conv1") for a in att]))
        out[f"z.a{j}.1.b"] = _f32(torch.cat([b(a + f"{j}.conv1") for a in att]))
        out[f"z.a{j}.2.w"] = _f32(torch.stack([w2(a + f"{j}.conv2") for a in att]))
        out[f"z.a{j}.2.b"] = _f32(torch.stack([b(a + f"{j}.conv2") for a in att]))
    lb = []
    for c in clb:  # per configuration: w1 [cin][hid], b1, w2 [4][hid], b2
        lb += [w2(c + ".mlp.0").t().reshape(-1), b(c + ".mlp.0"), w2(c + ".mlp.2").reshape(-1), b(c + ".mlp.2")]
    out["z.lb"] = _f32(torch.cat(lb))
    if multi:
        p = "patch_transformer."
        blob = [w2(p + "embedding_convPxP").reshape(-1), b(p + "embedding_convPxP")]
        for i in range(4):
            a = f"{_ZM}{p}transformer_encoder.{i}."
            g = lambda n: sd[a + n].float().reshape(-1)  # noqa: E731
            blob += [g("self_attn.query.weight"), g("self_attn.key.weight"), g("self_attn.value.weight"),
                     g("self_attn.query.bias"), g("self_attn.key.bias"), g("self_attn.value.bias"),
                     g("self_attn.out_proj.weight"), g("self_attn.out_proj.bias"), g("norm1.weight"), g("norm1.bias"),
                     g("linear1.weight"), g("linear1.bias"), g("linear2.weight"), g("linear2.bias"),
                     g("norm2.weight"), g("norm2.bias")]
        for n in ("linear1", "linear2"):
            blob += [sd[f"{_ZM}mlp_classifier.{n}.weight"].float().reshape(-1),
                     sd[f"{_ZM}mlp_classifier.{n}.bias"].float()]
        out["z.router"] = _f32(torch.cat(blob))
        P = cfg["patch"]
        nb = ((image_h // P - 1) // 2 + 1) * ((image_w // P - 1) // 2 + 1)
        out["z.r.pe"] = _f32(zoedepth_position_code(nb + 1))
    return out
