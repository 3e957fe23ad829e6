"""torch fp32 functional restatement of DPT's depth forward on a BEiT backbone (transformers 5.5
models/dpt/modeling_dpt.py DPTForDepthEstimation with backbone_config.model_type "beit": BeitEmbeddings without
absolute positions, BeitLayer with LayerScale, BeitSelfAttention with BeitRelativePositionBias, the raw hidden states
as taps, then DPT-Large's project readout, neck, fusion and head on the input's patch_height x patch_width grid),
written on the HF state_dict and pinned against the installed transformers module in tests/test_dpt_beit_cpu.py.
Test infrastructure: the reference for the GPU engine."""
import torch
import torch.nn.functional as F

B = "backbone."


def rel_index(ph, pw):
    """The relative position index of a ph x pw grid with the CLS token at 0: (qy - ky + ph - 1)(2 pw - 1) + (qx - kx +
    pw - 1) between patches, num - 3 on the CLS row, num - 2 on the CLS column, num - 1 at (0, 0)."""
    num = (2 * ph - 1) * (2 * pw - 1) + 3
    y, x = torch.meshgrid(torch.arange(ph), torch.arange(pw), indexing="ij")
    y, x = y.reshape(-1), x.reshape(-1)
    idx = torch.empty(ph * pw + 1, ph * pw + 1, dtype=torch.long)
    idx[1:, 1:] = (y[:, None] - y[None, :] + ph - 1) * (2 * pw - 1) + (x[:, None] - x[None, :] + pw - 1)
    idx[0, :] = num - 3
    idx[:, 0] = num - 2
    idx[0, 0] = num - 1
    return idx


def grid_table(table, window, ph, pw):
    """[(2 W - 1)^2 + 3, heads] pretrained table -> [(2 ph - 1)(2 pw - 1) + 3, heads] for the grid: the patch part
    resampled bilinearly (align_corners False), the three CLS entries kept."""
    n = (2 * window - 1) ** 2
    sub = table[:n].reshape(1, 2 * window - 1, 2 * window - 1, -1).permute(0, 3, 1, 2)
    sub = F.interpolate(sub, size=(2 * ph - 1, 2 * pw - 1), mode="bilinear", align_corners=False)
    return torch.cat([sub.permute(0, 2, 3, 1).reshape((2 * ph - 1) * (2 * pw - 1), -1), table[n:]])


def forward(sd, cfg, pixel_values, return_parts=False):
    """sd: DPTForDepthEstimation (BEiT backbone) state_dict; cfg: a depth_weights.DPT_BEIT_CONFIGS entry;
    pixel_values [3, H, W] f32, H and W multiples of 32 -> predicted_depth [H, W].  return_parts adds the taps, the
    per-layer bias [heads, N + 1, N + 1], the neck features and the fused maps."""
    D, L, Hh, P, eps = cfg["hidden"], cfg["layers"], cfg["heads"], cfg["patch"], cfg["ln_eps"]
    W0 = cfg["image_size"] // P
    x = pixel_values[None].float()
    _, _, IH, IW = x.shape
    ph, pw = IH // P, IW // P
    e = B + "embeddings."
    t = F.conv2d(x, sd[e + "patch_embeddings.projection.weight"], sd[e + "patch_embeddings.projection.bias"], stride=P)
    t = torch.cat((sd[e + "cls_token"], t.flatten(2).transpose(1, 2)), dim=1)
    idx = rel_index(ph, pw)
    taps, biases = [], []
    for i in range(L):
        p = f"{B}encoder.layer.{i}."
        a = p + "attention.attention."
        h = F.layer_norm(t, (D,), sd[p + "layernorm_before.weight"], sd[p + "layernorm_before.bias"], eps)
        q, k, v = (F.linear(h, sd[a + n + ".weight"], sd.get(a + n + ".bias")).view(1, -1, Hh, 64).transpose(1, 2)
                   for n in ("query", "key", "value"))
        tab = grid_table(sd[a + "relative_position_bias.relative_position_bias_table"].float(), W0, ph, pw)
        bias = tab[idx.reshape(-1)].reshape(idx.shape[0], idx.shape[1], Hh).permute(2, 0, 1)
        biases.append(bias)
        s = torch.softmax(q @ k.transpose(-1, -2) / 8.0 + bias[None], dim=-1)
        o = (s @ v).transpose(1, 2).reshape(1, -1, D)
        o = F.linear(o, sd[p + "attention.output.dense.weight"], sd[p + "attention.output.dense.bias"])
        t = t + (sd[p + "lambda_1"] * o if p + "lambda_1" in sd else o)
        h = F.layer_norm(t, (D,), sd[p + "layernorm_after.weight"], sd[p + "layernorm_after.bias"], eps)
        h = F.gelu(F.linear(h, sd[p + "intermediate.dense.weight"], sd[p + "intermediate.dense.bias"]))
        h = F.linear(h, sd[p + "output.dense.weight"], sd[p + "output.dense.bias"])
        t = t + (sd[p + "lambda_2"] * h if p + "lambda_2" in sd else h)
        if (i + 1) in cfg["taps"]:
            taps.append(t)  # hidden_states[i + 1], CLS included, no LayerNorm
    feats = []
    for i, hs in enumerate(taps):
        tok, cls = hs[:, 1:], hs[:, :1].expand(-1, ph * pw, -1)
        r = f"neck.reassemble_stage.readout_projects.{i}.0."
        ro = F.gelu(F.linear(torch.cat((tok, cls), -1), sd[r + "weight"], sd[r + "bias"]))
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
        return out, dict(taps=taps, bias=biases, feats=feats, fused=fused_all)
    return out


# a 4-layer BEiT with a 4 x 4 pretrained window (64 x 64 pixels)
SMALL = dict(hidden=256, layers=4, heads=4, taps=[1, 2, 3, 4], neck=[64, 128, 256, 256], fusion=64, image_size=64)


def fill_tables(sd, seed=0, std=2.0 ** 0.5, spikes=4, spike=8.0):
    """HF initialises every relative_position_bias_table to zeros, which would leave the bias path untested: N(0, std^2)
    entries, different per layer and head, plus `spikes` entries per head of +-`spike` (the CLS entries included)."""
    g = torch.Generator().manual_seed(seed + 17)
    for k in sorted(sd):
        if k.endswith("relative_position_bias_table"):
            n, H = sd[k].shape
            t = torch.randn(n, H, generator=g) * std
            for h in range(H):
                at = torch.randperm(n - 3, generator=g)[:spikes - 1].tolist() + [n - 3 + h % 3]
                t[at, h] = spike * torch.where(torch.rand(len(at), generator=g) < 0.5, -1.0, 1.0)
            sd[k] = t
    return sd


def random_model(small=False, seed=0, positive_head=True):
    """(state_dict, engine cfg) of a random-init transformers DPTForDepthEstimation with a BEiT backbone (BEiT-L/16 512,
    or the SMALL one) with filled bias tables, LayerScale lambdas drawn from [0.05, 0.3] per channel, and (positive_head)
    non-negative weights on the last 1x1 conv so that the depth range is not a cancellation residue."""
    from transformers import DPTForDepthEstimation
    from visiondepth3d_b200.depth_weights import DPT_BEIT_CONFIGS, hf_dpt_beit_config
    over = SMALL if small else {}
    cfg = dict(DPT_BEIT_CONFIGS["dpt-beit-large-512"], **over)
    torch.manual_seed(seed)
    sd = DPTForDepthEstimation(hf_dpt_beit_config(**over)).eval().state_dict()
    fill_tables(sd, seed)
    g = torch.Generator().manual_seed(seed + 29)
    for k in list(sd):
        if k.endswith("lambda_1") or k.endswith("lambda_2"):
            sd[k] = 0.05 + 0.25 * torch.rand(sd[k].shape, generator=g)
    if positive_head:
        sd["head.head.4.weight"] = sd["head.head.4.weight"].abs() + 0.02
        sd["head.head.4.bias"] = torch.zeros_like(sd["head.head.4.bias"])
    return sd, cfg


def hf_model(sd, small=False):
    """transformers' DPTForDepthEstimation carrying `sd`."""
    from transformers import DPTForDepthEstimation
    from visiondepth3d_b200.depth_weights import hf_dpt_beit_config
    m = DPTForDepthEstimation(hf_dpt_beit_config(**(SMALL if small else {}))).eval()
    m.load_state_dict(sd)
    return m
