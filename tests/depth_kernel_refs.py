"""TEST INFRASTRUCTURE: plain numpy float64 restatements of the operations the depth-forward kernels compute, on the
layouts the engine documents (include/vd3d.h, depth_weights.prepare), plus a generator of synthetic checkpoints.

tests/test_depth_kernel_refs_cpu.py pins every function here to oracle/depth.py and to torch ops;
tests/test_depth_kernels_gpu.py compares each CUDA kernel with them, from the inputs the device itself stored.

Layouts: token matrices are [rows, channels]; feature maps are NHWC [H, W, C]; 3x3 conv weights are
[Cout, 9 * Cin] (tap-major, tap = 3 * ky + kx); q and k are [image][head][NP][64], v is stored transposed as
[image][head][64][NP], NP = tokens rounded up to 128."""
import math

import numpy as np

F16_EPS = 2.0 ** -11      # half an ulp of f16, relative: the rounding of one f16 store
F32_EPS = 2.0 ** -24


def f64(a):
    return np.asarray(a, dtype=np.float64)


def layernorm(x, gamma, beta, eps=1e-6):
    x = f64(x)
    mu = x.mean(axis=-1, keepdims=True)
    var = ((x - mu) ** 2).mean(axis=-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * f64(gamma) + f64(beta)


def gelu(x):
    """0.5 x (1 + erf(x / sqrt 2)); written as max(x, 0) - 0.5 |x| erfc(|x| / sqrt 2) so that x << 0 does not cancel."""
    import torch
    x = np.ascontiguousarray(f64(x))
    erfc = torch.special.erfc(torch.from_numpy(np.abs(x) / math.sqrt(2.0))).numpy()
    return np.maximum(x, 0.0) - 0.5 * np.abs(x) * erfc


def attention_logits(q, k, nt):
    """q . k over the first nt keys (q holds the 1/sqrt(64) already): [..., nt, nt]."""
    return f64(q)[..., :nt, :] @ np.swapaxes(f64(k)[..., :nt, :], -1, -2)


def attention(q, k, vt, nt, with_abs=False):
    """softmax(q k^T) v of every (image, head): q, k [B, H, NP, 64], vt [B, H, 64, NP] -> [B, nt, H * 64] (head h in
    columns [64 h, 64 h + 64)).  Keys and queries >= nt do not exist.  with_abs: also the same weights applied to |v|
    (the scale of the error a relative perturbation of the weights causes)."""
    B, H = q.shape[:2]
    out = np.empty((B, nt, H * 64))
    mag = np.empty_like(out) if with_abs else None
    for b in range(B):
        for h in range(H):   # one head at a time: the [nt, nt] logits of all heads at once would not fit
            s = attention_logits(q[b, h], k[b, h], nt)
            p = np.exp(s - s.max(axis=-1, keepdims=True))
            p /= p.sum(axis=-1, keepdims=True)
            v = f64(vt[b, h, :, :nt]).T
            out[b, :, 64 * h: 64 * h + 64] = p @ v
            if with_abs:
                mag[b, :, 64 * h: 64 * h + 64] = p @ np.abs(v)
    return (out, mag) if with_abs else out


def qkv_split(y, images, npad, nt, heads, qscale=0.125):
    """y = tokens . Wqkv^T + b, rows image * npad + token, columns [q | k | v] each head-major: -> q (scaled), k
    [images, heads, nt, 64] and v^T [images, heads, 64, nt]."""
    y = f64(y)
    D = heads * 64
    q = np.empty((images, heads, nt, 64))
    k = np.empty((images, heads, nt, 64))
    vt = np.empty((images, heads, 64, nt))
    for b in range(images):
        rows = y[b * npad: b * npad + nt]
        q[b] = rows[:, :D].reshape(nt, heads, 64).transpose(1, 0, 2) * qscale
        k[b] = rows[:, D:2 * D].reshape(nt, heads, 64).transpose(1, 0, 2)
        vt[b] = rows[:, 2 * D:].reshape(nt, heads, 64).transpose(1, 2, 0)
    return q, k, vt


def patch_im2col(px):
    """pixel_values [3, IH, IW] -> [ph * pw, 588], column = c * 196 + dy * 14 + dx."""
    px = f64(px)
    _, IH, IW = px.shape
    ph, pw = IH // 14, IW // 14
    return px.reshape(3, ph, 14, pw, 14).transpose(1, 3, 0, 2, 4).reshape(ph * pw, 588)


def conv_transpose_scatter(y, ph, pw, k, cout):
    """ConvTranspose2d(kernel = stride = k) as a GEMM: y [ph * pw, k * k * cout] with column (dy * k + dx) * cout + co
    -> NHWC [ph * k, pw * k, cout], pixel (k y + dy, k x + dx)."""
    return f64(y).reshape(ph, pw, k, k, cout).transpose(0, 2, 1, 3, 4).reshape(ph * k, pw * k, cout)


def _pad1(x):
    return np.pad(f64(x), ((1, 1), (1, 1), (0, 0)))


def im2col_s2(x):
    """3x3, stride 2, zero padding 1 on NHWC [H, W, C] -> [OH * OW, 9 * C] (tap-major), OH = (H - 1) // 2 + 1."""
    H, W, C = x.shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    p = _pad1(x)
    cols = [p[ky: ky + 2 * OH - 1: 2, kx: kx + 2 * OW - 1: 2] for ky in range(3) for kx in range(3)]
    return np.stack(cols, axis=2).reshape(OH * OW, 9 * C)


def conv3x3(x, w, bias=None):
    """3x3, stride 1, zero padding 1: x NHWC [H, W, Cin], w [Cout, 9 * Cin] -> [H, W, Cout]."""
    H, W, C = x.shape
    p = _pad1(x)
    wt = f64(w).reshape(-1, 9, C)
    out = np.zeros((H, W, wt.shape[0]))
    for ky in range(3):
        for kx in range(3):
            out += p[ky: ky + H, kx: kx + W] @ wt[:, 3 * ky + kx].T
    if bias is not None:
        out = out + f64(bias)
    return out


def conv3x3_abs(x, w, bias=None):
    """sum of |x| |w| (+ |bias|) of the same conv: the scale of its accumulation error."""
    return conv3x3(np.abs(f64(x)), np.abs(f64(w)), None if bias is None else np.abs(f64(bias)))


def linear(x, w, bias=None):
    """x [..., K] . w [N, K]^T + bias (a 1x1 conv on NHWC, or a token GEMM)."""
    out = f64(x) @ f64(w).T
    return out if bias is None else out + f64(bias)


def linear_abs(x, w, bias=None):
    return linear(np.abs(f64(x)), np.abs(f64(w)), None if bias is None else np.abs(f64(bias)))


def upsample_ac(x, OH, OW):
    """bilinear, align_corners=True, NHWC [H, W, C] -> [OH, OW, C]."""
    x = f64(x)
    H, W, _ = x.shape

    def axis(n_in, n_out):
        f = np.arange(n_out) * ((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
        i0 = np.minimum(np.floor(f).astype(int), n_in - 1)
        return i0, np.minimum(i0 + 1, n_in - 1), f - i0

    y0, y1, ly = axis(H, OH)
    x0, x1, lx = axis(W, OW)
    lx = lx[None, :, None]
    top = x[y0][:, x0] * (1 - lx) + x[y0][:, x1] * lx
    bot = x[y1][:, x0] * (1 - lx) + x[y1][:, x1] * lx
    ly = ly[:, None, None]
    return top * (1 - ly) + bot * ly


def head(x, w2, b2, w3, b3):
    """DPT head after the upsample: relu(sum_c relu(conv3x3(x) + b2)[c] * w3[c] + b3) -> [H, W]."""
    t = np.maximum(conv3x3(x, w2, b2), 0.0)
    return np.maximum(t @ f64(w3).reshape(-1) + float(np.asarray(b3).reshape(-1)[0]), 0.0)


def f16_ulp(x):
    """spacing of f16 at |x| (normal range; 2^-24 in the subnormals)."""
    ax = np.maximum(np.abs(f64(x)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(ax)) - 10)


# ---------------------------------------------------------------------------------------------------------------------
def small_config(hidden, neck, fusion, layers=4):
    """A ViT of `layers` blocks whose last four are the taps: what the engine needs at least."""
    return dict(hidden=hidden, layers=layers, heads=hidden // 64, taps=list(range(layers - 3, layers + 1)),
                neck=list(neck), fusion=fusion)


def synth_state_dict(cfg, seed=0, grid=4):
    """A random checkpoint in the HF naming depth_weights.prepare reads, every tensor already representable in f16 (so
    that the prepared f16 operands and an fp32 evaluation of the same dict use the same numbers).  GEMM weights are
    ~ N(0, 1 / fan_in), LayerScale is 1, the head's last projection is non-negative."""
    import torch
    g = torch.Generator().manual_seed(seed)
    D, Fz = cfg["hidden"], cfg["fusion"]

    def rn(*shape, std=1.0):
        return (torch.randn(*shape, generator=g) * std).half().float()

    def lin(n, k, *ks):
        return rn(n, k, *ks, std=1.0 / math.sqrt(k * max(1, int(np.prod(ks)))))

    sd = {}
    e = "backbone.embeddings."
    sd[e + "patch_embeddings.projection.weight"] = lin(D, 3, 14, 14)
    sd[e + "patch_embeddings.projection.bias"] = rn(D, std=0.1)
    sd[e + "cls_token"] = rn(1, 1, D)
    sd[e + "position_embeddings"] = rn(1, 1 + grid * grid, D)
    for i in range(cfg["layers"]):
        p = f"backbone.encoder.layer.{i}."
        a = p + "attention.attention."
        for n in ("norm1", "norm2"):
            sd[p + n + ".weight"] = (1.0 + rn(D, std=0.1)).half().float()
            sd[p + n + ".bias"] = rn(D, std=0.1)
        for n in ("query", "key", "value"):
            sd[a + n + ".weight"] = lin(D, D)
            sd[a + n + ".bias"] = rn(D, std=0.1)
        sd[p + "attention.output.dense.weight"] = lin(D, D)
        sd[p + "attention.output.dense.bias"] = rn(D, std=0.1)
        sd[p + "layer_scale1.lambda1"] = torch.ones(D)
        sd[p + "mlp.fc1.weight"] = lin(4 * D, D)
        sd[p + "mlp.fc1.bias"] = rn(4 * D, std=0.1)
        sd[p + "mlp.fc2.weight"] = lin(D, 4 * D)
        sd[p + "mlp.fc2.bias"] = rn(D, std=0.1)
        sd[p + "layer_scale2.lambda1"] = torch.ones(D)
    sd["backbone.layernorm.weight"] = (1.0 + rn(D, std=0.1)).half().float()
    sd["backbone.layernorm.bias"] = rn(D, std=0.1)
    for i, C in enumerate(cfg["neck"]):
        r = f"neck.reassemble_stage.layers.{i}."
        sd[r + "projection.weight"] = lin(C, D, 1, 1)
        sd[r + "projection.bias"] = rn(C, std=0.1)
        if i < 2:
            kk = 4 if i == 0 else 2
            sd[r + "resize.weight"] = rn(C, C, kk, kk, std=1.0 / math.sqrt(C))
            sd[r + "resize.bias"] = rn(C, std=0.1)
        elif i == 3:
            sd[r + "resize.weight"] = lin(C, C, 3, 3)
            sd[r + "resize.bias"] = rn(C, std=0.1)
        sd[f"neck.convs.{i}.weight"] = lin(Fz, C, 3, 3)
    for j in range(4):
        f = f"neck.fusion_stage.layers.{j}."
        for unit in ("residual_layer1.", "residual_layer2."):
            for c in ("convolution1", "convolution2"):
                sd[f + unit + c + ".weight"] = lin(Fz, Fz, 3, 3)
                sd[f + unit + c + ".bias"] = rn(Fz, std=0.1)
        sd[f + "projection.weight"] = lin(Fz, Fz, 1, 1)
        sd[f + "projection.bias"] = rn(Fz, std=0.1)
    sd["head.conv1.weight"] = lin(Fz // 2, Fz, 3, 3)
    sd["head.conv1.bias"] = rn(Fz // 2, std=0.1)
    sd["head.conv2.weight"] = lin(32, Fz // 2, 3, 3)
    sd["head.conv2.bias"] = rn(32, std=0.1)
    sd["head.conv3.weight"] = (rn(1, 32, 1, 1, std=0.2).abs() + 0.02).half().float()
    sd["head.conv3.bias"] = rn(1, std=0.1)
    return sd
