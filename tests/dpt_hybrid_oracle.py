"""torch functional restatement of DPT-Hybrid's depth forward (MiDaS 3.0; transformers 5.5 models/dpt/modeling_dpt.py
DPTForDepthEstimation with is_hybrid=True, its BiT backbone models/bit/modeling_bit.py), written on the HF state_dict
and pinned against the installed transformers module in tests/test_oracle_dpt_hybrid.py.  Test infrastructure: the
reference for the GPU engine.  `dtype` float64 gives the float64 references of the kernel tests; `f16` emulates the
engine's storage precision (see emulate_engine)."""
import torch
import torch.nn.functional as F

BIT = "dpt.embeddings.backbone.bit."
DEPTHS, WIDTHS = (3, 4, 9), (256, 512, 1024)


def same_pad(size, k, s):
    """TF "SAME" padding of one axis (DynamicPad2d): (before, after)."""
    total = max((-(-size // s) - 1) * s + k - size, 0)
    return total // 2, total - total // 2


def standardize(w, eps=1e-8):
    """WeightStandardizedConv2d's weights: per output channel (w - mean) / sqrt(biased var + eps)."""
    flat = w.reshape(w.shape[0], -1)
    m = flat.mean(dim=1, keepdim=True)
    v = ((flat - m) ** 2).mean(dim=1, keepdim=True)
    return ((flat - m) / torch.sqrt(v + eps)).reshape(w.shape)


def conv_same(x, w, stride, ws=True, q=None):
    """BiT conv: weight-standardised, SAME padding (static pad (k - 1) / 2 at stride 1, dynamic at stride 2).  q: a
    rounding applied to the standardised weights and to the input (the engine's f16 operands)."""
    k = w.shape[-1]
    w = standardize(w) if ws else w
    if q is not None:
        w, x = q(w), q(x)
    if stride == 1:
        return F.conv2d(x, w, padding=(k - 1) // 2)
    ph, pw = same_pad(x.shape[-2], k, stride), same_pad(x.shape[-1], k, stride)
    return F.conv2d(F.pad(x, (pw[0], pw[1], ph[0], ph[1])), w, stride=stride)


def gn(x, sd, pfx, relu):
    y = F.group_norm(x, 32, sd[pfx + ".weight"], sd[pfx + ".bias"], 1e-5)
    return F.relu(y) if relu else y


def backbone(sd, px, q=None, stem_q=None, return_parts=False):
    """BiT stem + stages 1-3 on pixel_values [1, 3, S, S] -> (stage1, stage2, stage3) NCHW.  q: the rounding of every
    conv operand but the stem's (the engine: f16); stem_q: of the stem's (the engine: none, its stem runs in f32); the
    block outputs, which the engine stores in f16, are rounded with q too.  return_parts adds a dict of the stem's
    conv / GroupNorm / pool outputs and the first block's intermediates."""
    parts = {}
    y = conv_same(px, sd[BIT + "embedder.convolution.weight"], 2, q=stem_q)
    parts["stem_conv"] = y
    y = gn(y, sd, BIT + "embedder.norm", True)
    parts["stem_gn"] = y
    ph, pw = same_pad(y.shape[-2], 3, 2), same_pad(y.shape[-1], 3, 2)
    x = F.max_pool2d(F.pad(y, (pw[0], pw[1], ph[0], ph[1]), value=0.0), 3, 2)
    parts["pool"] = x
    rq = q or (lambda t: t)
    outs = []
    for st, depth in enumerate(DEPTHS):
        for b in range(depth):
            p = f"{BIT}encoder.stages.{st}.layers.{b}."
            s = 2 if (b == 0 and st > 0) else 1
            sc = x
            if b == 0:
                sc = gn(conv_same(x, sd[p + "downsample.conv.weight"], s, q=q), sd, p + "downsample.norm", False)
            h = gn(conv_same(x, sd[p + "conv1.weight"], 1, q=q), sd, p + "norm1", True)
            h = gn(conv_same(h, sd[p + "conv2.weight"], s, q=q), sd, p + "norm2", True)
            h = gn(conv_same(h, sd[p + "conv3.weight"], 1, q=q), sd, p + "norm3", False)
            x = rq(F.relu(h + sc))
        outs.append(x)
    if return_parts:
        return outs, parts
    return outs


def f16(t):
    """Round to f16 and back (the engine's storage precision)."""
    return t.to(torch.float16).to(t.dtype)


def forward(sd, cfg, pixel_values, return_parts=False, dtype=torch.float32, emulate=False):
    """sd: DPTForDepthEstimation (is_hybrid) state_dict; cfg: visiondepth3d_b200.depth_weights.DPT_HYBRID_CONFIGS entry
    (hidden, layers, heads, taps as 1-based layer numbers, neck, fusion, ln_eps); pixel_values [3, S, S] with S a
    multiple of 32 -> predicted_depth [S, S].  return_parts adds the stage maps, the taps (raw residual stream, CLS
    included), the readout outputs [N, D], the neck features and the fused maps.  emulate: round to f16 where the
    engine stores f16 (pixels kept f32 for the f32 stem, every other backbone conv operand and block output, the ViT
    and projection weights, the neck and head weights)."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    q = f16 if emulate else None
    D, L, Hh, P, eps = cfg["hidden"], cfg["layers"], cfg["heads"], cfg["patch"], cfg["ln_eps"]
    x = pixel_values[None].to(dtype)
    S = x.shape[-1]
    g = S // P
    s1, s2, s3 = backbone(sd, x, q=q)
    wq = q or (lambda t: t)
    e = "dpt.embeddings."
    t = F.conv2d(wq(s3), wq(sd[e + "projection.weight"]), sd[e + "projection.bias"]).flatten(2).transpose(1, 2)
    t = torch.cat((sd[e + "cls_token"], t), dim=1)
    pos = sd[e + "position_embeddings"]
    g0 = int(round((pos.shape[1] - 1) ** 0.5))
    pp = F.interpolate(pos[:, 1:].reshape(1, g0, g0, D).permute(0, 3, 1, 2), size=(g, g), mode="bilinear")
    t = t + torch.cat((pos[:, :1], pp.permute(0, 2, 3, 1).reshape(1, -1, D)), dim=1)
    taps = []
    for i in range(L):
        p = f"dpt.encoder.layer.{i}."
        a = p + "attention.attention."
        h = F.layer_norm(t, (D,), sd[p + "layernorm_before.weight"], sd[p + "layernorm_before.bias"], eps)
        qh, kh, vh = (F.linear(h, wq(sd[a + n + ".weight"]), sd[a + n + ".bias"]).view(1, -1, Hh, D // Hh)
                      .transpose(1, 2) for n in ("query", "key", "value"))
        s = torch.softmax(qh @ kh.transpose(-1, -2) / (D // Hh) ** 0.5, dim=-1)
        o = (s @ vh).transpose(1, 2).reshape(1, -1, D)
        t = t + F.linear(o, wq(sd[p + "attention.output.dense.weight"]), sd[p + "attention.output.dense.bias"])
        h = F.layer_norm(t, (D,), sd[p + "layernorm_after.weight"], sd[p + "layernorm_after.bias"], eps)
        h = F.gelu(F.linear(h, wq(sd[p + "intermediate.dense.weight"]), sd[p + "intermediate.dense.bias"]))
        t = t + F.linear(h, wq(sd[p + "output.dense.weight"]), sd[p + "output.dense.bias"])
        if (i + 1) in cfg["taps"][2:]:
            taps.append(t)  # hidden_states[i + 1]: no final LayerNorm
    readouts, feats = [], []
    for i, m in enumerate((s1, s2)):
        feats.append(F.conv2d(m, wq(sd[f"neck.convs.{i}.weight"]), None, padding=1))
    for i, hs in zip((2, 3), taps):
        tok, cls = hs[:, 1:], hs[:, :1].expand(-1, g * g, -1)
        r = f"neck.reassemble_stage.readout_projects.{i}.0."
        ro = F.gelu(F.linear(torch.cat((tok, cls), -1), wq(sd[r + "weight"]), sd[r + "bias"]))
        readouts.append(ro[0])
        r = f"neck.reassemble_stage.layers.{i}."
        m = ro.reshape(1, g, g, D).permute(0, 3, 1, 2)
        m = F.conv2d(m, wq(sd[r + "projection.weight"]), sd[r + "projection.bias"])
        if i == 3:
            m = F.conv2d(m, wq(sd[r + "resize.weight"]), sd[r + "resize.bias"], stride=2, padding=1)
        feats.append(F.conv2d(m, wq(sd[f"neck.convs.{i}.weight"]), None, padding=1))

    def rl(h, pfx):
        r = h
        h = F.conv2d(F.relu(h), wq(sd[pfx + "convolution1.weight"]), sd[pfx + "convolution1.bias"], padding=1)
        h = F.conv2d(F.relu(h), wq(sd[pfx + "convolution2.weight"]), sd[pfx + "convolution2.bias"], padding=1)
        return h + r

    fused, fused_all = None, []
    for j, f in enumerate(feats[::-1]):
        pfx = f"neck.fusion_stage.layers.{j}."
        h = f if fused is None else fused + rl(f, pfx + "residual_layer1.")
        h = rl(h, pfx + "residual_layer2.")
        h = F.interpolate(h, scale_factor=2, mode="bilinear", align_corners=True)
        fused = F.conv2d(h, wq(sd[pfx + "projection.weight"]), sd[pfx + "projection.bias"])
        fused_all.append(fused)
    d = F.conv2d(fused, wq(sd["head.head.0.weight"]), sd["head.head.0.bias"], padding=1)
    d = F.interpolate(d, scale_factor=2, mode="bilinear", align_corners=True)
    d = F.relu(F.conv2d(d, wq(sd["head.head.2.weight"]), sd["head.head.2.bias"], padding=1))
    d = F.relu(F.conv2d(d, sd["head.head.4.weight"], sd["head.head.4.bias"]))
    out = d[0, 0]
    if return_parts:
        return out, dict(stages=[s1, s2, s3], taps=taps, readouts=readouts, feats=feats, fused=fused_all, x=t)
    return out


SMALL = dict(hidden=256, layers=4, heads=4, taps=[1, 2, 3, 4], neck=[256, 512, 256, 256], fusion=64, image_size=128)


def random_model(small=False, gamma3=0.25, seed=0):
    """(state_dict, engine cfg) of a random-init transformers DPTForDepthEstimation(is_hybrid=True) (MiDaS 3.0's
    shapes, or the small test ViT at 128 x 128; the BiT backbone is always the full ResNet-50 stages 1-3).  The last
    1x1 head conv is made non-negative, as in tests/dpt_oracle.random_model.  gamma3 scales every block's norm3.weight:
    a trained ResNet damps its residual branches (initialising that norm at zero is a common recipe), while at HF's
    init (gamma3 = 1) sixteen undamped blocks amplify rounding; gamma3 = 1 is the stress model."""
    from transformers import DPTForDepthEstimation
    from visiondepth3d_b200.depth_weights import DPT_HYBRID_CONFIGS, hf_dpt_hybrid_config
    cfg = dict(DPT_HYBRID_CONFIGS["dpt-hybrid-midas"], **(SMALL if small else {}))
    torch.manual_seed(seed)
    sd = DPTForDepthEstimation(hf_dpt_hybrid_config(**(SMALL if small else {}))).eval().state_dict()
    sd["head.head.4.weight"] = sd["head.head.4.weight"].abs() + 0.02
    sd["head.head.4.bias"] = torch.zeros_like(sd["head.head.4.bias"])
    if gamma3 != 1:
        for k in list(sd):
            if k.startswith(BIT) and k.endswith("norm3.weight"):
                sd[k] = sd[k] * gamma3
    return sd, cfg


def hf_model(sd, small=False):
    """The transformers module carrying `sd` (for the pins against transformers)."""
    from transformers import DPTForDepthEstimation
    from visiondepth3d_b200.depth_weights import hf_dpt_hybrid_config
    m = DPTForDepthEstimation(hf_dpt_hybrid_config(**(SMALL if small else {}))).eval()
    m.load_state_dict(sd)
    return m
