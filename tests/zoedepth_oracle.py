"""torch fp32 functional restatement of ZoeDepth's depth forward and image processor (transformers 5.5
models/zoedepth: ZoeDepthForDepthEstimation on a BEiT backbone, ZoeDepthImageProcessor, post_process_depth_estimation),
written on the HF state_dict and pinned against the installed transformers modules in tests/test_zoedepth_cpu.py.
The trunk, neck and fusion are dpt_beit_oracle's; what is new here is the metric-bins head, routed per image.
Test infrastructure: the reference for the GPU engine."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from tests import dpt_beit_oracle as BO

M = "metric_head."


def processor(image_u8, size=(384, 512), mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5)):
    """ZoeDepthImageProcessor on one RGB u8 [h, w, 3] image -> pixel_values f32 [3, H, W]: rescale, reflect-pad,
    keep-aspect multiple-of-32 bilinear resize with align_corners, normalise."""
    x = torch.from_numpy(np.ascontiguousarray(image_u8)).permute(2, 0, 1)[None]
    x = x * (1 / 255)
    h, w = x.shape[-2:]
    ph, pw = int(np.sqrt(h / 2) * 3), int(np.sqrt(w / 2) * 3)
    x = F.pad(x, (pw, pw, ph, ph), mode="reflect")
    oh, ow = processed_size(w, h, size)
    x = F.interpolate(x, (oh, ow), mode="bilinear", align_corners=True)
    m, s = torch.tensor(mean).view(1, 3, 1, 1), torch.tensor(std).view(1, 3, 1, 1)
    return ((x - m) / s)[0]


def processed_size(width, height, size=(384, 512)):
    """(h, w) of ZoeDepthImageProcessor's resize of a (width, height) image (the padded size fitted to `size`)."""
    H, W = height + 2 * int(np.sqrt(height / 2) * 3), width + 2 * int(np.sqrt(width / 2) * 3)
    sh, sw = size[0] / H, size[1] / W
    if abs(1 - sw) < abs(1 - sh):
        sh = sw
    else:
        sw = sh
    return int(np.round(sh * H / 32) * 32), int(np.round(sw * W / 32) * 32)


def post_process(depth, source_hw):
    """post_process_depth_estimation with source_sizes: bicubic (antialias off) to the padded size, crop."""
    h, w = source_hw
    ph, pw = int(np.sqrt(h / 2) * 3), int(np.sqrt(w / 2) * 3)
    d = F.interpolate(depth[None, None], size=(h + 2 * ph, w + 2 * pw), mode="bicubic", align_corners=False)
    return d[0, 0, ph:ph + h, pw:pw + w]


def _conv(sd, name, x, act=None):
    y = F.conv2d(x, sd[M + name + ".weight"], sd[M + name + ".bias"])
    return act(y) if act else y


def up(x, hw):
    return F.interpolate(x, hw, mode="bilinear", align_corners=True)


def attractor(a, prev, n_attr):
    """ZoeDepthAttractorLayerUnnormed's update: the mean over attractors of dx / (1 + 300 dx^2), summed attractor by
    attractor (transformers' memory_efficient loop), no +1e-3, no sort, no clip."""
    c = up(prev, a.shape[-2:])
    dc = torch.zeros_like(c)
    for i in range(n_attr):
        dx = a[:, i:i + 1] - c
        dc += dx.div(1 + 300 * dx.pow(2))
    return c + dc / n_attr


def log_binomial(z4, bins, min_temp, max_temp, n_bins=64):
    """The conditional log-binomial from the MLP's Softplus output z4 [1, 4, H, W] and the bins [1, K, H, W] -> depth."""
    p = z4[:, :2] + 1e-4
    p = p[:, 0] / (p[:, 0] + p[:, 1])
    t = z4[:, 2:] + 1e-4
    t = (t[:, 0] / (t[:, 0] + t[:, 1]))[:, None]
    t = (max_temp - min_temp) * t + min_temp
    k = torch.arange(n_bins).view(1, -1, 1, 1)
    km1 = torch.tensor([n_bins - 1]).view(1, -1, 1, 1)
    q = torch.clamp(1 - p, 1e-4, 1)[:, None]
    p = torch.clamp(p, 1e-4, 1)[:, None]
    n, kk = km1 + 1e-7, k + 1e-7
    lb = n * torch.log(n) - kk * torch.log(kk) - (n - kk) * torch.log(n - kk + 1e-7)
    y = torch.softmax((lb + k * torch.log(p) + (km1 - k) * torch.log(q)) / t, dim=1)
    return torch.sum(y * bins, dim=1, keepdim=True)


def router(sd, x):
    """ZoeDepthPatchTransformerEncoder + ZoeDepthMLPClassifier on one image's bottleneck conv2 x [1, F, h, w] ->
    logits [2]."""
    p = M + "patch_transformer."
    e = F.conv2d(x, sd[p + "embedding_convPxP.weight"], sd[p + "embedding_convPxP.bias"]).flatten(2)
    e = F.pad(e, (1, 0)).permute(0, 2, 1)
    n = e.shape[1]
    pos = torch.arange(0, n, dtype=torch.float32).unsqueeze(1)
    idx = torch.arange(0, 128, 2, dtype=torch.float32).unsqueeze(0)
    pe = pos * torch.exp(idx * (-torch.log(torch.tensor(10000.0)) / 128))
    e = e + torch.cat([torch.sin(pe), torch.cos(pe)], dim=1)[None]
    for i in range(4):
        a = f"{p}transformer_encoder.{i}."
        q, k, v = (F.linear(e, sd[a + f"self_attn.{n}.weight"], sd[a + f"self_attn.{n}.bias"]).view(1, -1, 4, 32)
                   .transpose(1, 2) for n in ("query", "key", "value"))
        s = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(32), dim=-1)
        o = (s @ v).transpose(1, 2).reshape(1, -1, 128)
        o = F.linear(o, sd[a + "self_attn.out_proj.weight"], sd[a + "self_attn.out_proj.bias"])
        e = F.layer_norm(e + o, (128,), sd[a + "norm1.weight"], sd[a + "norm1.bias"], 1e-5)
        h = F.linear(F.relu(F.linear(e, sd[a + "linear1.weight"], sd[a + "linear1.bias"])), sd[a + "linear2.weight"],
                     sd[a + "linear2.bias"])
        e = F.layer_norm(e + h, (128,), sd[a + "norm2.weight"], sd[a + "norm2.bias"], 1e-5)
    c = F.relu(F.linear(e[:, 0], sd[M + "mlp_classifier.linear1.weight"], sd[M + "mlp_classifier.linear1.bias"]))
    return F.linear(c, sd[M + "mlp_classifier.linear2.weight"], sd[M + "mlp_classifier.linear2.bias"])[0]


def metric_head(sd, cfg, act, bottleneck, blocks, rel=None, route=None):
    """The metric head on one image: act [1, 32, H, W] (the relative head's conv2 + ReLU), bottleneck [1, F, h, w],
    blocks: the four fusion outputs, rel [1, 1, H, W] the relative depth (single configuration) -> (depth [H, W],
    logits or None, route).  route forces the configuration (None: the router's argmax, ties to 0)."""
    names = [c["name"] for c in cfg["bins"]]
    multi = len(names) > 1
    x = _conv(sd, "conv2", bottleneck)
    logits = None
    if multi:
        logits = router(sd, x)
        if route is None:
            route = int(torch.argmax(torch.softmax(logits, -1)))
    route = route or 0
    pfx = f"seed_bin_regressors.{names[route]}" if multi else "seed_bin_regressor"
    prev = _conv(sd, pfx + ".conv2", _conv(sd, pfx + ".conv1", x, F.relu), F.softplus)
    prev_emb = _conv(sd, "seed_projector.conv2", _conv(sd, "seed_projector.conv1", x, F.relu))
    for j, blk in enumerate(blocks):
        emb = _conv(sd, f"projectors.{j}.conv2", _conv(sd, f"projectors.{j}.conv1", blk, F.relu))
        a = f"attractors.{names[route]}.{j}" if multi else f"attractors.{j}"
        h = emb + up(prev_emb, blk.shape[-2:])
        att = _conv(sd, a + ".conv2", _conv(sd, a + ".conv1", h, F.relu), F.softplus)
        prev = attractor(att, prev, att.shape[1])
        prev_emb = emb
    last = act if rel is None else torch.cat([act, up(rel, act.shape[-2:])], 1)
    clb = f"conditional_log_binomial.{names[route]}" if multi else "conditional_log_binomial"
    z = _conv(sd, clb + ".mlp.0", torch.cat([last, up(prev_emb, act.shape[-2:])], 1), F.gelu)
    z4 = _conv(sd, clb + ".mlp.2", z, F.softplus)
    bins = up(prev, act.shape[-2:])
    return log_binomial(z4, bins, cfg["min_temp"], cfg["max_temp"])[0, 0], logits, route


def beit_sd(sd):
    """The trunk / neck / relative head of a ZoeDepth state_dict under dpt_beit_oracle's names."""
    out = {k: v for k, v in sd.items() if not k.startswith("relative_head.") and not k.startswith(M)}
    for j, n in ((0, "conv1"), (2, "conv2"), (4, "conv3")):
        out[f"head.head.{j}.weight"] = sd[f"relative_head.{n}.weight"]
        out[f"head.head.{j}.bias"] = sd[f"relative_head.{n}.bias"]
    return out


def forward(sd, cfg, pixel_values, route=None, return_parts=False):
    """sd: ZoeDepthForDepthEstimation state_dict; cfg: a depth_weights.ZOEDEPTH_CONFIGS-style dict; pixel_values
    [3, H, W] f32, H and W multiples of 32 -> metric depth [H, W] (and the parts: logits, route, act)."""
    rel, parts = BO.forward(beit_sd(sd), cfg, pixel_values, return_parts=True)
    h = F.conv2d(parts["fused"][-1], sd["relative_head.conv1.weight"], sd["relative_head.conv1.bias"], padding=1)
    h = F.interpolate(h, scale_factor=2, mode="bilinear", align_corners=True)
    act = F.relu(F.conv2d(h, sd["relative_head.conv2.weight"], sd["relative_head.conv2.bias"], padding=1))
    single = len(cfg["bins"]) == 1
    d, logits, rt = metric_head(sd, cfg, act, parts["feats"][3], parts["fused"], rel[None, None] if single else None,
                                route)
    if return_parts:
        return d, dict(logits=logits, route=rt, act=act, bottleneck=parts["feats"][3], fused=parts["fused"])
    return d


# a 4-layer BEiT with a 4 x 4 pretrained window (64 x 64 pixels), fusion 64, the head's real widths
SMALL = dict(BO.SMALL, bottleneck=64)


def random_model(multi=True, small=True, seed=0, **cfg):
    """(state_dict, cfg) of a random-init transformers ZoeDepthForDepthEstimation (the SMALL BEiT or BEiT-L/16 384) with
    filled bias tables, LayerScale lambdas in [0.05, 0.3], and the bins' seed made positive and spread so that the
    metric depth has a range worth measuring.  cfg overrides entries of the configuration (e.g. the fusion width)."""
    from transformers import ZoeDepthForDepthEstimation
    from visiondepth3d_b200.depth_weights import ZOEDEPTH_CONFIGS, hf_zoedepth_config
    name = "zoedepth-nyu-kitti" if multi else "zoedepth-nyu"
    over = dict(SMALL if small else {}, **cfg)
    cfg = dict(ZOEDEPTH_CONFIGS[name], **over)
    torch.manual_seed(seed)
    sd = ZoeDepthForDepthEstimation(hf_zoedepth_config(name, **over)).eval().state_dict()
    BO.fill_tables(sd, seed)
    g = torch.Generator().manual_seed(seed + 29)
    for k in list(sd):
        if k.endswith("lambda_1") or k.endswith("lambda_2"):
            sd[k] = 0.05 + 0.25 * torch.rand(sd[k].shape, generator=g)
        if k.startswith(M) and k.endswith(".conv2.bias") and ("seed_bin" in k):
            sd[k] = torch.linspace(-2.0, 3.0, sd[k].shape[0])
        # the HF init leaves the fusion outputs and the head's activation near 1e-4: widen the log-binomial's MLP and
        # the relative head so that p and t vary over the image
        # (BEiT-L's activations are ~1e3 times larger already: its head keeps the HF init)
        if small and "conditional_log_binomial" in k and (k.endswith("mlp.0.weight") or k.endswith("mlp.2.weight")):
            sd[k] = sd[k] * 40.0
        if small and k.startswith("relative_head.conv") and k.endswith(".weight"):
            sd[k] = sd[k] * 30.0
    return sd, cfg


def hf_model(sd, cfg_name="zoedepth-nyu-kitti", small=True):
    """transformers' ZoeDepthForDepthEstimation carrying `sd`."""
    from transformers import ZoeDepthForDepthEstimation
    from visiondepth3d_b200.depth_weights import hf_zoedepth_config
    m = ZoeDepthForDepthEstimation(hf_zoedepth_config(cfg_name, **(SMALL if small else {}))).eval()
    m.load_state_dict(sd)
    return m
