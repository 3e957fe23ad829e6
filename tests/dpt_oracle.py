"""torch fp32 functional restatement of DPT's depth forward (transformers 5.5 models/dpt/modeling_dpt.py,
DPTForDepthEstimation with a ViT backbone: DPTViTEmbeddings, DPTViTLayer, DPTReassembleStage with the project
readout, DPTNeck, DPTFeatureFusionStage, DPTDepthEstimationHead), written on the HF state_dict and pinned against the
installed transformers module in tests/test_oracle_dpt.py.  Test infrastructure: the reference for the GPU engine."""
import torch
import torch.nn.functional as F


def forward(sd, cfg, pixel_values, return_parts=False):
    """sd: DPTForDepthEstimation state_dict; cfg: visiondepth3d_b200.depth_weights.DPT_CONFIGS entry (hidden, layers,
    heads, taps as 1-based layer numbers, neck, fusion, patch, ln_eps); pixel_values [3, H, W] f32 with H == W a
    multiple of the patch -> predicted_depth [H, W].  return_parts adds the taps (raw residual stream, CLS included),
    the readout outputs [N, D], the neck features, the fused maps and the final residual stream."""
    D, L, Hh, P, eps = cfg["hidden"], cfg["layers"], cfg["heads"], cfg["patch"], cfg["ln_eps"]
    x = pixel_values[None].float()
    _, _, IH, IW = x.shape
    ph, pw = IH // P, IW // P
    e = "dpt.embeddings."
    t = F.conv2d(x, sd[e + "patch_embeddings.projection.weight"], sd[e + "patch_embeddings.projection.bias"], stride=P)
    t = torch.cat((sd[e + "cls_token"], t.flatten(2).transpose(1, 2)), dim=1)
    pos = sd[e + "position_embeddings"]
    g = int(round((pos.shape[1] - 1) ** 0.5))
    pp = F.interpolate(pos[:, 1:].reshape(1, g, g, D).permute(0, 3, 1, 2), size=(ph, pw), mode="bilinear")
    t = t + torch.cat((pos[:, :1], pp.permute(0, 2, 3, 1).reshape(1, -1, D)), dim=1)
    taps = []
    for i in range(L):
        p = f"dpt.encoder.layer.{i}."
        a = p + "attention.attention."
        h = F.layer_norm(t, (D,), sd[p + "layernorm_before.weight"], sd[p + "layernorm_before.bias"], eps)
        q, k, v = (F.linear(h, sd[a + n + ".weight"], sd[a + n + ".bias"]).view(1, -1, Hh, D // Hh).transpose(1, 2)
                   for n in ("query", "key", "value"))
        s = torch.softmax(q @ k.transpose(-1, -2) / (D // Hh) ** 0.5, dim=-1)
        o = (s @ v).transpose(1, 2).reshape(1, -1, D)
        t = t + F.linear(o, sd[p + "attention.output.dense.weight"], sd[p + "attention.output.dense.bias"])
        h = F.layer_norm(t, (D,), sd[p + "layernorm_after.weight"], sd[p + "layernorm_after.bias"], eps)
        h = F.gelu(F.linear(h, sd[p + "intermediate.dense.weight"], sd[p + "intermediate.dense.bias"]))
        t = t + F.linear(h, sd[p + "output.dense.weight"], sd[p + "output.dense.bias"])
        if (i + 1) in cfg["taps"]:
            taps.append(t)  # hidden_states[i + 1]: no final LayerNorm
    readouts, feats = [], []
    for i, hs in enumerate(taps):
        tok, cls = hs[:, 1:], hs[:, :1].expand(-1, ph * pw, -1)
        r = f"neck.reassemble_stage.readout_projects.{i}.0."
        ro = F.gelu(F.linear(torch.cat((tok, cls), -1), sd[r + "weight"], sd[r + "bias"]))
        readouts.append(ro[0])
        r = f"neck.reassemble_stage.layers.{i}."
        m = ro.reshape(1, ph, pw, D).permute(0, 3, 1, 2)
        m = F.conv2d(m, sd[r + "projection.weight"], sd[r + "projection.bias"])
        if i < 2:
            m = F.conv_transpose2d(m, sd[r + "resize.weight"], sd[r + "resize.bias"], stride=4 if i == 0 else 2)
        elif i == 3:
            m = F.conv2d(m, sd[r + "resize.weight"], sd[r + "resize.bias"], stride=2, padding=1)
        feats.append(F.conv2d(m, sd[f"neck.convs.{i}.weight"], None, padding=1))

    def rl(h, pfx):
        r = h
        h = F.conv2d(F.relu(h), sd[pfx + "convolution1.weight"], sd[pfx + "convolution1.bias"], padding=1)
        h = F.conv2d(F.relu(h), sd[pfx + "convolution2.weight"], sd[pfx + "convolution2.bias"], padding=1)
        return h + r

    fused, fused_all = None, []
    for j, f in enumerate(feats[::-1]):
        pfx = f"neck.fusion_stage.layers.{j}."
        h = f if fused is None else fused + rl(f, pfx + "residual_layer1.")
        h = rl(h, pfx + "residual_layer2.")
        h = F.interpolate(h, scale_factor=2, mode="bilinear", align_corners=True)
        fused = F.conv2d(h, sd[pfx + "projection.weight"], sd[pfx + "projection.bias"])
        fused_all.append(fused)
    d = F.conv2d(fused, sd["head.head.0.weight"], sd["head.head.0.bias"], padding=1)
    d = F.interpolate(d, scale_factor=2, mode="bilinear", align_corners=True)
    d = F.relu(F.conv2d(d, sd["head.head.2.weight"], sd["head.head.2.bias"], padding=1))
    d = F.relu(F.conv2d(d, sd["head.head.4.weight"], sd["head.head.4.bias"]))
    out = d[0, 0]
    if return_parts:
        return out, dict(taps=taps, readouts=readouts, feats=feats, fused=fused_all, x=t)
    return out


SMALL = dict(hidden=256, layers=4, heads=4, taps=[1, 2, 3, 4], neck=[64, 128, 256, 256], fusion=64, image_size=64)


def random_model(small=False, positive_head=True, stress=False, seed=0):
    """(state_dict, engine cfg) of a random-init transformers DPTForDepthEstimation (DPT-Large, or the small test ViT).
    positive_head: non-negative weights on the last 1x1 conv, so that the depth range is not a cancellation residue
    (as a trained head's).  stress: four massive-activation channels in the residual stream (fc2 biases of +-60..80
    in every layer, position-embedding offsets of 25): |x| reaches several hundred, which the un-normalised taps carry
    into the readout GEMM."""
    from transformers import DPTForDepthEstimation
    from visiondepth3d_b200.depth_weights import DPT_CONFIGS, hf_dpt_config
    cfg = dict(DPT_CONFIGS["dpt-large"], **(SMALL if small else {}))
    torch.manual_seed(seed)
    sd = DPTForDepthEstimation(hf_dpt_config("dpt-large", **(SMALL if small else {}))).eval().state_dict()
    if positive_head:
        sd["head.head.4.weight"] = sd["head.head.4.weight"].abs() + 0.02
        sd["head.head.4.bias"] = torch.zeros_like(sd["head.head.4.bias"])
    if stress:
        g = torch.Generator().manual_seed(seed + 1)
        D = cfg["hidden"]
        hot = torch.randperm(D, generator=g)[:4]
        for k in list(sd):
            if k.endswith("output.dense.bias") and "attention" not in k:
                b = sd[k].clone()
                b[hot] = torch.tensor([60.0, -45.0, 30.0, 80.0])
                sd[k] = b
        pe = sd["dpt.embeddings.position_embeddings"].clone()
        pe[..., hot] += 25.0
        sd["dpt.embeddings.position_embeddings"] = pe
    return sd, cfg
