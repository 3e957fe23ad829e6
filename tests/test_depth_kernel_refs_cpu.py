"""CPU: pin tests/depth_kernel_refs.py -- the float64 restatements tests/test_depth_kernels_gpu.py holds each CUDA
kernel against -- to oracle/depth.py and to torch ops.  The whole forward is composed from the restatements on the
PREPARED weights (depth_weights.prepare: the arrays the engine uploads, in the engine's layouts, channel padding
included) and compared, stage by stage, with the oracle on the checkpoint those weights were prepared from."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import depth as OD
from tests import depth_kernel_refs as R
from visiondepth3d_b200.depth_weights import prepare

CFG = R.small_config(128, neck=[48, 96, 64, 128], fusion=64)


def ref_forward(P, cfg, px):
    """The engine's launch sequence, every step one restatement, all float64."""
    D, Hh, Fz = cfg["hidden"], cfg["heads"], cfg["fusion"]
    _, IH, IW = px.shape
    ph, pw = IH // 14, IW // 14
    NT = ph * pw + 1
    NP = (NT + 127) // 128 * 128
    x = np.empty((NT, D))
    x[0] = R.f64(P["cls"]) + R.f64(P["pos"][0])
    x[1:] = R.linear(R.patch_im2col(px), P["pe.w"][:, :588], P["pe.b"]) + R.f64(P["pos"][1:])
    taps = []
    for i in range(cfg["layers"]):
        w = lambda n: P[f"l{i}.{n}"]  # noqa: E731
        xn = R.layernorm(x, w("ln1.g"), w("ln1.b"))
        y = np.zeros((NP, 3 * D))
        y[:NT] = R.linear(xn, w("qkv.w"), w("qkv.b"))
        q, k, vt = R.qkv_split(y, 1, NP, NT, Hh)
        x = x + R.f64(w("ls1")) * R.linear(R.attention(q, k, vt, NT)[0], w("proj.w"), w("proj.b"))
        h = R.gelu(R.linear(R.layernorm(x, w("ln2.g"), w("ln2.b")), w("fc1.w"), w("fc1.b")))
        x = x + R.f64(w("ls2")) * R.linear(h, w("fc2.w"), w("fc2.b"))
        if (i + 1) in cfg["taps"]:
            taps.append(R.layernorm(x[1:], P["norm.g"], P["norm.b"]))
    feats = []
    for i, C in enumerate(cfg["neck"]):
        CP = (C + 63) // 64 * 64
        p = R.linear(taps[i], P[f"r{i}.proj.w"], P[f"r{i}.proj.b"])
        if i < 2:
            kk = 4 if i == 0 else 2
            s = R.conv_transpose_scatter(R.linear(p, P[f"r{i}.up.w"], P[f"r{i}.up.b"]), ph, pw, kk, CP)
        elif i == 2:
            s = p.reshape(ph, pw, CP)
        else:
            oh, ow = (ph - 1) // 2 + 1, (pw - 1) // 2 + 1
            s = R.linear(R.im2col_s2(p.reshape(ph, pw, CP)), P["r3.down.w"], P["r3.down.b"]).reshape(oh, ow, CP)
        feats.append(R.conv3x3(s, P[f"n{i}.conv.w"]))
    fused, fused_all = None, []
    for j in range(4):
        f = feats[3 - j]

        def unit(v, u):
            mid = np.maximum(R.conv3x3(np.maximum(v, 0), P[f"f{j}.{u}.c1.w"], P[f"f{j}.{u}.c1.b"]), 0)
            return R.conv3x3(mid, P[f"f{j}.{u}.c2.w"], P[f"f{j}.{u}.c2.b"]) + v

        h = f if fused is None else fused + unit(f, "rl1")
        y = unit(h, "rl2")
        OH, OW = feats[2 - j].shape[:2] if j < 3 else (2 * y.shape[0], 2 * y.shape[1])
        fused = R.linear(R.upsample_ac(y, OH, OW), P[f"f{j}.proj.w"], P[f"f{j}.proj.b"])
        fused_all.append(fused)
    h1u = R.upsample_ac(R.conv3x3(fused, P["h.c1.w"], P["h.c1.b"]), IH, IW)
    depth = R.head(h1u, P["h.c2.w"], P["h.c2.b"], P["h.c3.w"], P["h.c3.b"])
    return dict(x=x, taps=taps, feats=feats, fused=fused_all, depth=depth)


@pytest.mark.parametrize("h,w", [(70, 98), (84, 56)])   # 5x7 (odd, odd) and 6x4 (even, even) patches
def test_composed_restatements_match_the_oracle(h, w):
    sd = R.synth_state_dict(CFG, seed=3)
    P = prepare(sd, CFG, h, w)
    torch.manual_seed(4)
    px = torch.randn(3, h, w)
    with torch.no_grad():
        depth, parts = OD.forward(sd, CFG, px, return_parts=True)
    mine = ref_forward(P, CFG, px.numpy())

    def close(a, b, what):   # the oracle is fp32: 1e-4 of the map's scale is its own rounding, far below any layout slip
        b = b.detach().double().numpy()
        assert a.shape == b.shape, what
        assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max(), (what, np.abs(a - b).max(), np.abs(b).max())

    close(mine["x"], parts["x"][0], "x")
    for i in range(4):
        close(mine["taps"][i], parts["taps"][i][0, 1:], f"tap{i}")
        close(mine["feats"][i], parts["feats"][i][0].permute(1, 2, 0), f"feat{i}")
        close(mine["fused"][i], parts["fused"][i][0].permute(1, 2, 0), f"fused{i}")
    close(mine["depth"], depth, "depth")
    assert float(depth.max()) > 0 and float((depth > 0).float().mean()) > 0.5   # the final ReLU is not all there is


def test_attention_ignores_padding_and_matches_torch():
    rng = np.random.default_rng(0)
    B, H, NT, NP = 2, 3, 36, 128
    q = rng.standard_normal((B, H, NP, 64)) * 0.6
    k = rng.standard_normal((B, H, NP, 64)) * 3
    vt = rng.standard_normal((B, H, 64, NP))
    ref = F.scaled_dot_product_attention(torch.from_numpy(q[:, :, :NT]), torch.from_numpy(k[:, :, :NT]),
                                         torch.from_numpy(vt[:, :, :, :NT]).transpose(-1, -2), scale=1.0)
    ref = ref.permute(0, 2, 1, 3).reshape(B, NT, H * 64).numpy()
    out = R.attention(q, k, vt, NT)
    assert np.abs(out - ref).max() <= 1e-12
    q[:, :, NT:] = 1e4
    k[:, :, NT:] = 1e4
    vt[:, :, :, NT:] = -1e4
    assert np.array_equal(R.attention(q, k, vt, NT), out)
    lg = R.attention_logits(q, k, NT)
    assert lg.shape == (B, H, NT, NT) and lg.std() > 5     # a peaked softmax, not a uniform one


def test_qkv_split_places_every_image_head_and_the_transpose():
    B, NP, NT, H = 2, 128, 36, 2
    D = 64 * H
    y = np.arange((B * NP) * 3 * D, dtype=np.float64).reshape(B * NP, 3 * D)
    q, k, vt = R.qkv_split(y, B, NP, NT, H)
    for b, h, t, d in ((0, 0, 0, 0), (1, 1, 35, 63), (1, 0, 7, 5), (0, 1, 20, 40)):
        row = y[b * NP + t]
        assert q[b, h, t, d] == 0.125 * row[h * 64 + d]
        assert k[b, h, t, d] == row[D + h * 64 + d]
        assert vt[b, h, d, t] == row[2 * D + h * 64 + d]


def test_gelu_is_the_erf_form_everywhere():
    x = np.linspace(-8, 8, 4001)
    ref = F.gelu(torch.from_numpy(x)).numpy()
    assert np.abs(R.gelu(x) - ref).max() <= 1e-15
    tanh_form = F.gelu(torch.from_numpy(x), approximate="tanh").numpy()
    assert np.abs(R.gelu(x) - tanh_form).max() > 1e-4       # the two forms are distinguishable where the tests look
    assert R.gelu(np.array([-6.0]))[0] < 0                  # no cancellation to zero in the left tail


@pytest.mark.parametrize("H,W", [(5, 7), (6, 4), (37, 66)])
def test_spatial_restatements_match_torch(H, W):
    rng = np.random.default_rng(H * W)
    C, Co = 8, 5
    x = rng.standard_normal((H, W, C))
    xt = torch.from_numpy(x).permute(2, 0, 1)[None]
    nhwc = lambda t: t[0].permute(1, 2, 0).numpy()  # noqa: E731
    w = rng.standard_normal((Co, C, 3, 3))
    b = rng.standard_normal(Co)
    wk = w.transpose(0, 2, 3, 1).reshape(Co, 9 * C)
    ref = nhwc(F.conv2d(xt, torch.from_numpy(w), torch.from_numpy(b), padding=1))
    assert np.abs(R.conv3x3(x, wk, b) - ref).max() <= 1e-12
    ref = nhwc(F.conv2d(xt, torch.from_numpy(w), torch.from_numpy(b), padding=1, stride=2))
    out = R.linear(R.im2col_s2(x), wk, b).reshape(ref.shape)
    assert np.abs(out - ref).max() <= 1e-12
    for (OH, OW) in ((2 * H, 2 * W), (2 * H - 1, 2 * W + 3), (14 * H, 14 * W)):
        ref = nhwc(F.interpolate(xt, size=(OH, OW), mode="bilinear", align_corners=True))
        assert np.abs(R.upsample_ac(x, OH, OW) - ref).max() <= 1e-12
    for kk in (2, 4):
        wt = rng.standard_normal((C, Co, kk, kk))
        ref = nhwc(F.conv_transpose2d(xt, torch.from_numpy(wt), torch.from_numpy(b), stride=kk))
        wg = wt.transpose(2, 3, 1, 0).reshape(kk * kk * Co, C)           # rows (dy * k + dx) * Cout + co
        y = R.linear(x.reshape(H * W, C), wg, np.tile(b, kk * kk))
        assert np.abs(R.conv_transpose_scatter(y, H, W, kk, Co) - ref).max() <= 1e-12
    px = rng.standard_normal((3, 14 * H, 14 * W))
    wp = rng.standard_normal((Co, 3, 14, 14))
    ref = F.conv2d(torch.from_numpy(px)[None], torch.from_numpy(wp), stride=14)[0].flatten(1).T.numpy()
    assert np.abs(R.linear(R.patch_im2col(px), wp.reshape(Co, 588)) - ref).max() <= 1e-11


def test_layernorm_and_head_match_torch():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((9, 128)) * 5 + 3
    g, b = rng.standard_normal(128), rng.standard_normal(128)
    ref = F.layer_norm(torch.from_numpy(x), (128,), torch.from_numpy(g), torch.from_numpy(b), 1e-6).numpy()
    assert np.abs(R.layernorm(x, g, b) - ref).max() <= 1e-12
    H, W, C = 6, 5, 8
    f = rng.standard_normal((H, W, C))
    w2, b2 = rng.standard_normal((32, C, 3, 3)), rng.standard_normal(32)
    w3, b3 = rng.standard_normal(32), np.array([0.3])
    t = torch.relu(F.conv2d(torch.from_numpy(f).permute(2, 0, 1)[None], torch.from_numpy(w2), torch.from_numpy(b2),
                            padding=1))
    ref = torch.relu(F.conv2d(t, torch.from_numpy(w3).reshape(1, 32, 1, 1), torch.from_numpy(b3)))[0, 0].numpy()
    out = R.head(f, w2.transpose(0, 2, 3, 1).reshape(32, 9 * C), b2, w3, b3)
    assert np.abs(out - ref).max() <= 1e-12 and (ref == 0).any() and (ref > 0).any()


def test_f16_ulp():
    for v in (1.0, 1.5, 0.75, 1000.0, 3e-5):
        a = np.float16(v)
        assert R.f16_ulp(float(a)) == float(np.nextafter(a, np.float16(np.inf))) - float(a)
