"""TEST INFRASTRUCTURE: plain numpy float64 restatements of what MiDaS 3.0's BiT backbone and ZoeDepth's metric head
run on k_umma_gemm and their own kernels, on the layouts the engine stores (depth_weights.prepare_dpt_hybrid /
prepare_zoedepth; bit_backbone, bit_conv and zoe_head in depth_engine.cu).

tests/test_hybrid_zoe_kernel_refs_cpu.py pins the compositions of these functions to tests/dpt_hybrid_oracle.backbone
and tests/zoedepth_oracle.metric_head; tests/test_hybrid_zoe_kernels_gpu.py and tests/test_zoedepth_gpu.py compare the
CUDA kernels with them, from the inputs the device itself stored.

Layouts: maps are NHWC [H, W, C] or their pixel rows [H * W, C]; 3x3 conv weights are [Cout, 9 * Cin] (tap-major,
tap = 3 * ky + kx); the metric head's packed tensors concatenate the configurations along N (z.s1, z.a{j}.1: config c
in columns [c n, (c + 1) n)), z.s2 is block-diagonal, z.a{j}.2 and z.lb are stacked per configuration."""
import numpy as np

from tests import depth_kernel_refs as R
from tests.dpt_hybrid_oracle import same_pad

f64 = R.f64
BIT_1X1, BIT_3X3, BIT_3X3_S2, BIT_1X1_S2 = range(4)   # vd3d_bit_kernel op 4's kinds
E, NB = 128, 64                                        # ZoeDepth's embedding width and bin count


# ---------------------------------------------------------------------------------------------------------------------
# BiT backbone
# ---------------------------------------------------------------------------------------------------------------------
def same_im2col_s2(x):
    """3x3, stride 2, TF-SAME pads (same_pad: 0 before and 1 after on even sides) on NHWC [H, W, C] ->
    [OH * OW, 9 * C] (tap-major), OH = ceil(H / 2)."""
    x = f64(x)
    H, W, C = x.shape
    (pt, pb), (pl, pr) = same_pad(H, 3, 2), same_pad(W, 3, 2)
    p = np.pad(x, ((pt, pb), (pl, pr), (0, 0)))
    OH, OW = -(-H // 2), -(-W // 2)
    cols = [p[ky: ky + 2 * OH - 1: 2, kx: kx + 2 * OW - 1: 2] for ky in range(3) for kx in range(3)]
    return np.stack(cols, axis=2).reshape(OH * OW, 9 * C)


def bit_conv(x, w, kind):
    """One bias-free BiT conv: x NHWC [H, W, cin], w [cout, cin] or [cout, 9 cin] -> output pixel rows [Ho * Wo, cout]."""
    x = f64(x)
    H, W, C = x.shape
    if kind == BIT_1X1:
        return R.linear(x.reshape(H * W, C), w)
    if kind == BIT_3X3:
        return R.conv3x3(x, w).reshape(H * W, -1)
    if kind == BIT_1X1_S2:
        return R.linear(x[::2, ::2].reshape(-1, C), w)
    assert kind == BIT_3X3_S2
    return R.linear(same_im2col_s2(x), w)


def bit_conv_abs(x, w, kind):
    """sum of |x| |w| of the same conv: the scale of its accumulation error."""
    return bit_conv(np.abs(f64(x)), np.abs(f64(w)), kind)


def group_stats(y, groups=32):
    """float64 mean and biased variance of each of the groups of the channels of y [rows, C]."""
    y = f64(y)
    rows, C = y.shape
    yg = y.reshape(rows, groups, C // groups)
    m = yg.mean(axis=(0, 2))
    return m, ((yg - m[None, :, None]) ** 2).mean(axis=(0, 2))


def groupnorm(y, g, b, groups=32, eps=1e-5):
    """GroupNorm of y [rows, C] with the affine (g, b) -> (out, z): z is the normalised y before the affine."""
    y = f64(y)
    m, v = group_stats(y, groups)
    grp = np.arange(y.shape[1]) // (y.shape[1] // groups)
    z = (y - m[grp]) / np.sqrt(v[grp] + eps)
    return z * f64(g) + f64(b), z


def gn_apply(y, g, b, y2=None, g2=None, b2=None, res=None, relu=True):
    """The engine's GroupNorm apply: GN(y) [+ GN(y2; g2, b2)] [+ res], ReLU -> float64 [rows, C]."""
    out = groupnorm(y, g, b)[0]
    if y2 is not None:
        out = out + groupnorm(y2, g2, b2)[0]
    if res is not None:
        out = out + f64(res)
    return np.maximum(out, 0.0) if relu else out


def bit_stages(P, x, rnd=None, stages=3):
    """BiT stages 1..3 from the max-pool output x NHWC [S/4, S/4, 64] on prepare_dpt_hybrid's tensors P, composed of
    bit_conv and gn_apply as bit_backbone runs them -> [stage maps, NHWC].  rnd: the rounding of every stored activation
    the convs read and of every block output (the engine: f16)."""
    rnd = rnd or (lambda t: t)
    x = rnd(f64(x))
    outs = []
    for st, (depth, width) in enumerate(zip((3, 4, 9), (256, 512, 1024))):
        mid = width // 4
        for k in range(depth):
            q = f"bit.s{st}.b{k}."
            s2 = k == 0 and st > 0
            H = x.shape[0]
            Ho = H // 2 if s2 else H
            cin = x.shape[2]
            t1 = rnd(gn_apply(bit_conv(x, P[q + "c1.w"], BIT_1X1), P[q + "n1.g"], P[q + "n1.b"]))
            t2 = rnd(gn_apply(bit_conv(t1.reshape(H, H, mid), P[q + "c2.w"], BIT_3X3_S2 if s2 else BIT_3X3),
                              P[q + "n2.g"], P[q + "n2.b"]))
            y = bit_conv(t2.reshape(Ho, Ho, mid), P[q + "c3.w"], BIT_1X1)
            if k == 0:
                y2 = bit_conv(x, P[q + "ds.w"], BIT_1X1_S2 if s2 else BIT_1X1)
                out = gn_apply(y, P[q + "n3.g"], P[q + "n3.b"], y2, P[q + "ds.g"], P[q + "ds.b"])
            else:
                out = gn_apply(y, P[q + "n3.g"], P[q + "n3.b"], res=x.reshape(-1, cin))
            x = rnd(out).reshape(Ho, Ho, width)
        outs.append(x)
        if st + 1 == stages:
            break
    return outs


# ---------------------------------------------------------------------------------------------------------------------
# ZoeDepth metric head
# ---------------------------------------------------------------------------------------------------------------------
def softplus(x):
    x = f64(x)
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def lin(P, name, x, relu=False):
    """a packed 1x1 layer "name.w" [N, K] / "name.b" [N] on rows x [M, K]."""
    y = R.linear(x, P[name + ".w"], P[name + ".b"])
    return np.maximum(y, 0.0) if relu else y


def lin_abs(P, name, x):
    return R.linear_abs(x, P[name + ".w"], P[name + ".b"])


def seed_conv2(P, sh, nc):
    """The seed regressors' conv2 of every configuration, each on its own ms columns of sh [M, nc ms] (z.s2 is block-
    diagonal: its off-diagonal blocks are zero) -> raw [M, nc NB], configuration c in columns [c NB, (c + 1) NB)."""
    ms = sh.shape[1] // nc
    w, b = f64(P["z.s2.w"]), f64(P["z.s2.b"])
    return np.concatenate([f64(sh)[:, c * ms:(c + 1) * ms] @ w[c * NB:(c + 1) * NB, c * ms:(c + 1) * ms].T
                           + b[c * NB:(c + 1) * NB] for c in range(nc)], axis=1)


def route_cols(a, route, n):
    """configuration route's n columns of a layout concatenated along N."""
    return a[:, route * n:(route + 1) * n]


def attractor(hid, w2, b2, prev, Hp, Wp, H, W, prev_softplus=False):
    """ZoeDepthAttractorLayerUnnormed on one configuration: hid [H W, E] (its ReLU(conv1)), w2 [na, E], b2 [na], prev
    [Hp Wp, NB] the previous bins (raw seed conv2 when prev_softplus) -> (bins [H W, NB], attractors a [H W, na],
    upsampled previous bins c [H W, NB])."""
    a = softplus(f64(hid) @ f64(w2).T + f64(b2))
    p = softplus(prev) if prev_softplus else f64(prev)
    c = R.upsample_ac(p.reshape(Hp, Wp, -1), H, W).reshape(H * W, -1)
    dx = a[:, :, None] - c[:, None, :]
    return c + (dx / (1 + 300 * dx * dx)).mean(axis=1), a, c


def logbinom_unpack(lb, nc, cin, hid, route):
    """configuration route's (w1 [cin, hid], b1, w2 [4, hid], b2) out of z.lb."""
    per = cin * hid + hid + 4 * hid + 4
    assert f64(lb).size == nc * per
    s = f64(lb)[route * per:(route + 1) * per]
    return (s[:cin * hid].reshape(cin, hid), s[cin * hid:cin * hid + hid],
            s[cin * hid + hid:cin * hid + 5 * hid].reshape(4, hid), s[cin * hid + 5 * hid:])


def log_binomial(act, emb, bins, He, We, H, W, mlp, tmin, tmax, w3=None, b3=None, parts=False):
    """ZoeDepthConditionalLogBinomialSoftmax and the expectation on one configuration: act [H W, 32], emb [He We, E],
    bins [He We, NB], mlp = logbinom_unpack(...), w3 / b3: the relative head's last conv when the relative depth is the
    33rd input -> depth [H W] (and, with parts, a dict of the intermediates the error bound needs)."""
    from scipy.special import erf
    w1, b1, w2, b2 = mlp
    a64 = f64(act)
    cols = [a64]
    rel = None
    if w3 is not None:
        rel = np.maximum(a64 @ f64(w3).reshape(-1) + float(np.asarray(b3).reshape(-1)[0]), 0.0)
        cols.append(rel[:, None])
    ue = R.upsample_ac(f64(emb).reshape(He, We, -1), H, W).reshape(H * W, -1)
    cols.append(ue)
    x = np.concatenate(cols, 1)
    h = x @ w1 + b1
    g = 0.5 * h * (1 + erf(h / np.sqrt(2)))
    o = softplus(g @ w2.T + b2)
    pa, pb = o[:, 0] + 1e-4, o[:, 1] + 1e-4
    p = pa / (pa + pb)
    ta, tb = o[:, 2] + 1e-4, o[:, 3] + 1e-4
    t = (tmax - tmin) * (ta / (ta + tb)) + tmin
    q, p = np.clip(1 - p, 1e-4, 1), np.clip(p, 1e-4, 1)
    k = np.arange(NB, dtype=np.float64)
    n_, kk = NB - 1 + 1e-7, k + 1e-7
    lbk = n_ * np.log(n_) - kk * np.log(kk) - (n_ - kk) * np.log(n_ - kk + 1e-7)
    y = lbk[None] + k[None] * np.log(p)[:, None] + (NB - 1 - k)[None] * np.log(q)[:, None]
    lg = y / t[:, None]
    wgt = np.exp(lg - lg.max(1, keepdims=True))
    wgt /= wgt.sum(1, keepdims=True)
    c = R.upsample_ac(f64(bins).reshape(He, We, -1), H, W).reshape(H * W, -1)
    d = (wgt * c).sum(1)
    if not parts:
        return d
    return d, dict(x=x, h=h, g=g, o=o, p=p, q=q, t=t, ta_tb=ta + tb, pa_pb=pa + pb, y=y, lg=lg, wgt=wgt, c=c, lbk=lbk,
                   rel=rel, ue=ue)


def router64(sd, x):
    """ZoeDepth's router (patch transformer + MLP classifier) in float64 on one image's bottleneck conv2 x [1, F, h, w]
    (torch float64; sd: the metric head's tensors in float64) -> logits [2].  The sinusoid is built in f32 as
    transformers builds it, then widened."""
    import torch
    import torch.nn.functional as F
    from tests.zoedepth_oracle import M
    from visiondepth3d_b200.depth_weights import zoedepth_position_code
    p = M + "patch_transformer."
    e = F.conv2d(x, sd[p + "embedding_convPxP.weight"], sd[p + "embedding_convPxP.bias"]).flatten(2)
    e = F.pad(e, (1, 0)).permute(0, 2, 1)
    e = e + zoedepth_position_code(e.shape[1]).double()[None]
    for i in range(4):
        a = f"{p}transformer_encoder.{i}."
        q, k, v = (F.linear(e, sd[a + f"self_attn.{n}.weight"], sd[a + f"self_attn.{n}.bias"]).view(1, -1, 4, 32)
                   .transpose(1, 2) for n in ("query", "key", "value"))
        s = torch.softmax(q @ k.transpose(-1, -2) / np.sqrt(32), dim=-1)
        o = F.linear((s @ v).transpose(1, 2).reshape(1, -1, 128), sd[a + "self_attn.out_proj.weight"],
                     sd[a + "self_attn.out_proj.bias"])
        e = F.layer_norm(e + o, (128,), sd[a + "norm1.weight"], sd[a + "norm1.bias"], 1e-5)
        h = F.linear(F.relu(F.linear(e, sd[a + "linear1.weight"], sd[a + "linear1.bias"])), sd[a + "linear2.weight"],
                     sd[a + "linear2.bias"])
        e = F.layer_norm(e + h, (128,), sd[a + "norm2.weight"], sd[a + "norm2.bias"], 1e-5)
    c = F.relu(F.linear(e[:, 0], sd[M + "mlp_classifier.linear1.weight"], sd[M + "mlp_classifier.linear1.bias"]))
    return F.linear(c, sd[M + "mlp_classifier.linear2.weight"], sd[M + "mlp_classifier.linear2.bias"])[0]


def metric_head(P, nc, route, bott, bh, bw, blocks, act, H, W, tmin, tmax, cat=False, hid=None):
    """zoe_head composed of the functions above on prepare_zoedepth's tensors P: bott [bh bw, F] (the bottleneck),
    blocks [(map [h w, F], h, w)] the four fusion outputs, act [H W, 32] -> (depth [H W], dict of every intermediate
    under the engine's buffer names)."""
    zb = lin(P, "z.bt", bott)
    sh = lin(P, "z.s1", zb, relu=True)
    seed = seed_conv2(P, sh, nc)
    t1 = lin(P, "z.sp1", zb, relu=True)
    emb = lin(P, "z.sp2", t1)
    T = dict(zb32=zb, sh=sh, seed=seed)
    prev, ph, pw = route_cols(seed, route, NB), bh, bw
    for j, (blk, h, w) in enumerate(blocks):
        t1 = lin(P, f"z.p{j}.1", blk, relu=True)
        cur = lin(P, f"z.p{j}.2", t1)
        up = R.upsample_ac(emb.reshape(ph, pw, E), h, w).reshape(h * w, E)
        x = cur + up
        hb = lin(P, f"z.a{j}.1", x, relu=True)
        bins, _, _ = attractor(route_cols(hb, route, E), f64(P[f"z.a{j}.2.w"])[route], f64(P[f"z.a{j}.2.b"])[route],
                               prev, ph, pw, h, w, prev_softplus=j == 0)
        T.update({f"t1.{j}": t1, f"emb.{j}": cur, f"up.{j}": up, f"x.{j}": x, f"hid.{j}": hb, f"bins.{j}": bins})
        prev, emb, ph, pw = bins, cur, h, w
    cin = 32 + int(cat) + E
    hid = hid or (f64(P["z.lb"]).size // nc - 4) // (cin + 5)
    mlp = logbinom_unpack(P["z.lb"], nc, cin, hid, route)
    d = log_binomial(act, emb, prev, ph, pw, H, W, mlp, tmin, tmax, *((P["h.c3.w"], P["h.c3.b"]) if cat else ()))
    return d, T
