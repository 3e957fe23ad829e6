"""GPU: what MiDaS 3.0 (DPT-Hybrid) and ZoeDepth run on k_umma_gemm, layer by layer, against the float64 restatements
of tests/hybrid_zoe_kernel_refs.py (pinned to the oracles in tests/test_hybrid_zoe_kernel_refs_cpu.py), in the method
and with the error model of tests/test_depth_kernels_gpu.py (ACC, stored_f16, report: "observed / bound" per check).

  * Every BiT conv shape of MiDaS 3.0 at 384 x 384 and of the 128 x 128 small model, through vd3d_bit_kernel op 4: the
    very launch path bit_backbone runs (1x1, 3x3 stride 1, 3x3 stride 2 SAME on k_im2col_same, 1x1 stride 2), on
    non-negative inputs and weight-standardised filters (zero mean: the sums cancel; the bound is relative to
    sum |a| |w|, so it holds under cancellation).
  * The hybrid forward's own buffers at B = 1 and 2: the stage-3 shortcut im2col and GEMM, the last block's conv3 and
    its GroupNorm + residual (the scratch buffers hold the last image's), the neck's 3x3 convs on the stage-1 / 2 maps
    of every image, and the token projection of the stage-3 map (EPI_PATCH, CLS row, zero padding rows).
  * ZoeDepth's metric head on its own buffers after a forward, with stress weights (1x1 layers at He scale, biases
    distinct per channel, the configurations drawn independently): bottleneck conv2 (f16 and f32), router, seed
    regressor of both configurations, the last projector with its residual, the attractor conv1 of both
    configurations, the last attractor (route's columns), the relative head's conv2 + ReLU and the log-binomial.
    The j < 3 projector / attractor buffers and the seed-stage attractor are overwritten before the forward ends; the
    vd3d_zoe_kernel hook tests of tests/test_zoedepth_gpu.py keep covering the attractor's seed stage.

Bounds beyond test_depth_kernels_gpu's: a CUDA-core fp32 dot product of n terms is within n 2^-24 sum |a| |w|; the
GroupNorm's fp32 statistics within 64 2^-24 (|mean| + sd) (tests/test_dpt_hybrid_gpu.py measures them directly); the
attractor and the log-binomial carry their input errors through each operation's largest slope (|dx / (1 + 300 dx^2)|'
<= 1, GELU' <= 1.13, Softplus' <= 1, a softmax whose logits move by at most d changes sum w c by at most
(e^(2 d) - 1) sum w |c - mean|)."""
import numpy as np
import pytest
import torch

from tests import depth_kernel_refs as R
from tests import dpt_hybrid_oracle as OH
from tests import hybrid_zoe_kernel_refs as HZ
from tests import zoedepth_oracle as ZO
from tests.test_depth_kernels_gpu import ACC, conv_check, report, stored_f16, up_check
from tests.test_zoedepth_gpu import ROUTER_BOUND

pytestmark = pytest.mark.gpu

EPS32 = R.F32_EPS
PROC128 = dict(size=(128, 128), resample=3, mean=(0.5,) * 3, std=(0.5,) * 3)


def f32_check(dev, ref, absum, K, what, extra=0.0):
    """an f32 GEMM output: ACC(K) of sum |a| |b| (the accumulator is what is stored)"""
    return report(what, np.abs(R.f64(dev) - ref), ACC(K) * absum + extra + 1e-30)


# ---------------------------------------------------------------------------------------------------------------------
# 2. every BiT conv shape through the backbone's own launch (vd3d_bit_kernel op 4)
# ---------------------------------------------------------------------------------------------------------------------
def _shapes(S):
    """(kind, H, cin, cout) of every conv MiDaS 3.0 runs on an S x S image (H: the conv's input side)"""
    a, b, c = S // 4, S // 8, S // 16
    return sorted({(0, a, 64, 64), (0, a, 256, 64), (1, a, 64, 64), (0, a, 64, 256),             # stage 1
                   (0, a, 256, 128), (0, b, 512, 128), (2, a, 128, 128), (1, b, 128, 128),      # stage 2
                   (0, b, 128, 512), (3, a, 256, 512),
                   (0, b, 512, 256), (0, c, 1024, 256), (2, b, 256, 256), (1, c, 256, 256),     # stage 3
                   (0, c, 256, 1024), (3, b, 512, 1024)})


@pytest.fixture(scope="module")
def keng():
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine(OH.SMALL | dict(patch=16, ln_eps=1e-12), family="dpt-hybrid", processor=PROC128)
    yield e
    e.close()


@pytest.mark.parametrize("kind,H,cin,cout", sorted(set(_shapes(384)) | set(_shapes(128))))
def test_bit_conv_against_float64(keng, kind, H, cin, cout):
    from visiondepth3d_b200.depth_weights import _conv3, standardize_weight
    rng = np.random.default_rng(H * 7 + cin + 3 * cout + kind)
    k = 3 if kind in (HZ.BIT_3X3, HZ.BIT_3X3_S2) else 1
    x = np.abs(rng.standard_normal((H, H, cin))).astype(np.float16)
    w = standardize_weight(torch.from_numpy(rng.standard_normal((cout, cin, k, k))))
    w = _conv3(w, cin) if k == 3 else w.reshape(cout, cin).numpy().astype(np.float16)
    Ho = H // 2 if kind >= HZ.BIT_3X3_S2 else H
    out = keng.bit_kernel(4, (H, H, cin, cout, kind), {"t.in": x, "t.w": w}, (Ho * Ho, cout), np.float32)
    ref, absum = HZ.bit_conv(x, w, kind), HZ.bit_conv_abs(x, w, kind)
    assert np.median(np.abs(ref) / absum) < 0.25                # the sums do cancel
    f32_check(out, ref, absum, k * k * cin, f"bit conv kind {kind} {H}^2 {cin} -> {cout}")
    if kind == HZ.BIT_3X3_S2:  # the im2col rows the GEMM read
        col = keng.get_buffer("t.col", (Ho * Ho, 9 * cin), np.float16)
        assert np.array_equal(col.astype(np.float64), HZ.same_im2col_s2(x))


def test_bit_conv_refuses_bad_arguments(keng):
    from visiondepth3d_b200 import _lib
    x = np.zeros((8, 8, 64), np.float16)
    w = np.zeros((64, 9 * 64), np.float16)
    for dims in ((8, 8, 64, 64, 4), (8, 8, 32, 64, 0), (8, 8, 64, 32, 0), (7, 8, 64, 64, 2), (1, 8, 64, 64, 0)):
        with pytest.raises(_lib.Vd3dError):
            keng.bit_kernel(4, dims, {"t.in": x, "t.w": w}, (1,), np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the hybrid forward's own buffers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hybrid():
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import prepare_dpt_hybrid
    sd, cfg = OH.random_model()
    S = cfg["image_size"]
    e = DepthEngine(cfg, family="dpt-hybrid")
    P = prepare_dpt_hybrid(sd, cfg, S, S)
    e.load_state_dict(sd)
    yield e, P, cfg
    e.close()


def _frames(B, S, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (S, S, 3), dtype=np.uint8) for _ in range(B)]


def gn_check(dev, y, g, b, res, what):
    """relu(GN(y) + res) stored f16, y f32 as the device stored it: fp32 statistics (mean off by 64 ulp of |mean| + sd,
    variance by 64 ulp) carried through the affine, the residual add and the rounding"""
    m, v = HZ.group_stats(y)
    grp = np.arange(y.shape[1]) // (y.shape[1] // 32)
    gn, z = HZ.groupnorm(y, g, b)
    rel = 64 * EPS32 * (np.abs(m[grp]) + np.sqrt(v[grp])) / np.sqrt(v[grp] + 1e-5)
    slack = np.abs(R.f64(g)) * (rel * (1 + np.abs(z)) + 8 * EPS32 * np.abs(z)) + 8 * EPS32 * (np.abs(gn) + np.abs(R.f64(res)))
    return stored_f16(dev, np.maximum(gn + R.f64(res), 0), slack, what)


@pytest.mark.parametrize("B", [1, 2])
def test_hybrid_backbone_and_neck_buffers(hybrid, B):
    e, P, cfg = hybrid
    S, F_ = cfg["image_size"], cfg["fusion"]
    a, b2, c = S // 4, S // 8, S // 16
    e.infer_batch(_frames(B, S, B), check_size=False)
    st1 = [e.get_buffer(f"bit.stage1.{i}", (a, a, 256), np.float16) for i in range(B)]
    st2 = [e.get_buffer(f"bit.stage2.{i}", (b2, b2, 512), np.float16) for i in range(B)]
    # the shared scratch buffers hold the last image's stage 3: its first block's shortcut im2col and GEMM ...
    col = e.get_buffer("bit.col", (c * c, 512), np.float16)
    assert np.array_equal(col, st2[-1][::2, ::2].reshape(-1, 512)), "k_im2col_same 1x1 stride 2"
    y2 = e.get_buffer("bit.y2", (c * c, 1024), np.float32)
    w = P["bit.s2.b0.ds.w"]
    f32_check(y2, R.linear(col, w), R.linear_abs(col, w), 512, f"bit.y2 (stage-3 shortcut, K = 512) B={B}")
    # ... and its last block (stage 3 has 9 blocks alternating from bit.xa: the output in bit.xa, its input in bit.xb)
    t2 = e.get_buffer("bit.t2", (c * c, 256), np.float16)
    y = e.get_buffer("bit.y", (c * c, 1024), np.float32)
    w = P["bit.s2.b8.c3.w"]
    f32_check(y, R.linear(t2, w), R.linear_abs(t2, w), 256, f"bit.y (last conv3, K = 256) B={B}")
    xin = e.get_buffer("bit.xb", (c * c, 1024), np.float16)
    out = e.get_buffer("bit.xa", (c * c, 1024), np.float16)
    gn_check(out, y, P["bit.s2.b8.n3.g"], P["bit.s2.b8.n3.b"], xin, f"stage 3 = relu(GN3(bit.y) + input) B={B}")
    # the neck's 3x3 convs read the stage-1 / stage-2 maps of every image directly
    for i in range(B):
        sfx = "" if B == 1 else f"#{i}"
        for n, (m, side) in enumerate(((st1[i], a), (st2[i], b2))):
            f = e.get_buffer(f"f{n}{sfx}", (side, side, F_), np.float16)
            conv_check(f, m, P[f"n{n}.conv.w"], None, f"f{n} (3x3, {m.shape[2]} -> {F_}) B={B} image {i}")


@pytest.mark.parametrize("B", [1, 2])
def test_hybrid_token_projection(hybrid, B):
    """Every LayerScale at zero keeps the residual stream at the embedding: x of image b is EPI_PATCH's stage3 @ pe.w
    + pe.b + pos in rows 1 .. NT - 1 and k_set_cls's cls + pos[0] in row 0."""
    e, P, cfg = hybrid
    S, D, L = cfg["image_size"], cfg["hidden"], cfg["layers"]
    NT = (S // 16) ** 2 + 1
    NP = (NT + 127) // 128 * 128

    def put(name, arr):
        arr = np.ascontiguousarray(arr)
        e.check(e.lib.vd3d_depth_set_tensor(e.h, name.encode(), arr.ctypes.data, arr.nbytes))
    rng = np.random.default_rng(B)
    pos = rng.standard_normal(P["pos"].shape).astype(np.float32)   # the model's rows are equal (zero at init)
    cls = rng.standard_normal(P["cls"].shape).astype(np.float32)
    try:
        for i in range(L):
            put(f"l{i}.ls1", np.zeros(D, np.float32))
            put(f"l{i}.ls2", np.zeros(D, np.float32))
        put("pos", pos)
        put("cls", cls)
        e.infer_batch(_frames(B, S, 10 + B), check_size=False)
        x = e.get_buffer("x", (B, NP, D), np.float32)
        s3 = e.get_buffer("bit.xa", (NT - 1, 1024), np.float16)   # the last image's stage-3 map
    finally:
        for i in range(L):
            put(f"l{i}.ls1", P[f"l{i}.ls1"])
            put(f"l{i}.ls2", P[f"l{i}.ls2"])
        put("pos", P["pos"])
        put("cls", P["cls"])
    P = dict(P, pos=pos, cls=cls)
    cls0 = P["cls"].reshape(-1) + P["pos"][0]
    for b in range(B):
        assert np.array_equal(x[b, 0], cls0), ("k_set_cls", b)
        if b + 1 < B:
            assert not x[b, NT:].any(), ("rows [NT, NP) of an image that is not the last", b)
    ref = R.linear(s3, P["pe.w"], P["pe.b"]) + R.f64(P["pos"][1:NT])
    tol = ACC(1024) * (R.linear_abs(s3, P["pe.w"], P["pe.b"]) + np.abs(R.f64(P["pos"][1:NT]))) + 2 * EPS32 * np.abs(ref)
    report(f"EPI_PATCH stage 3 -> tokens (K = 1024) B={B}", np.abs(R.f64(x[B - 1, 1:NT]) - ref), tol)
    assert np.abs(ref).max() > 1


# ---------------------------------------------------------------------------------------------------------------------
# 4. ZoeDepth's metric head on its own buffers
# ---------------------------------------------------------------------------------------------------------------------
def stress(sd, seed, router=True):
    """the metric head's 1x1 layers (bottleneck conv2 unless not router, seed regressors / projector, projectors,
    attractors) at He scale with biases drawn per output channel, every configuration drawn on its own.  The
    log-binomial MLP keeps HF's init scale, with its temperature pair well away from zero: the temperature
    t = min_t + (max_t - min_t) ta / (ta + tb) turns an error e in ta or tb into (max_t - min_t) e / (ta + tb)"""
    g = torch.Generator().manual_seed(seed)
    sd = dict(sd)
    skip = ("patch_transformer", "mlp_classifier", "conditional_log_binomial") + (() if router else (ZO.M + "conv2",))
    for k, v in list(sd.items()):
        if k.startswith(ZO.M) and "conditional_log_binomial" in k and k.endswith("mlp.2.bias"):
            sd[k] = v.clone()
            sd[k][2:] = 4.0
        if k.startswith(ZO.M) and "conditional_log_binomial" in k and k.endswith(".weight"):
            sd[k] = (torch.randn(v.shape, generator=g) * (1.0 / v.shape[1]) ** 0.5).half().float()
        if not k.startswith(ZO.M) or any(s in k for s in skip) or v.dim() != 4 or v.shape[-1] != 1:
            continue
        fan = v.shape[1]
        sd[k] = (torch.randn(v.shape, generator=g) * (2.0 / fan) ** 0.5).half().float()
        b = k[:-len("weight")] + "bias"
        sd[b] = (torch.rand(v.shape[0], generator=g) - 0.5).half().float()
    return sd


def _route_bias(sd, shift):
    sd = dict(sd)
    b = sd[ZO.M + "mlp_classifier.linear2.bias"].clone()
    b[1] += shift
    sd[ZO.M + "mlp_classifier.linear2.bias"] = b
    return sd


def attractor_check(dev, hid, w2, b2, prev, Hp, Wp, H, W, what):
    ref, a, c = HZ.attractor(hid, w2, b2, prev, Hp, Wp, H, W)
    na, K = w2.shape
    e_a = (K + 1) * EPS32 * (np.abs(R.f64(hid)) @ np.abs(R.f64(w2)).T + np.abs(R.f64(b2))) + 8 * EPS32 * (1 + np.abs(a))
    e_c = (8 + 8 * max(Hp, Wp)) * EPS32 * float(np.abs(R.f64(prev)).max())
    fmax = 0.5 / np.sqrt(300.0)                            # max |dx / (1 + 300 dx^2)|
    tol = (2 * e_c + e_a.mean(1)[:, None] + EPS32 * (np.abs(a).mean(1)[:, None] + np.abs(c))
           + (8 + na) * EPS32 * fmax + 2 * EPS32 * np.abs(ref))
    return report(what, np.abs(R.f64(dev) - ref), tol)


def logbinom_check(dev, act, emb, bins, He, We, H, W, mlp, tmin, tmax, w3, b3, what):
    d, p = HZ.log_binomial(act, emb, bins, He, We, H, W, mlp, tmin, tmax, w3, b3, parts=True)
    w1, b1, w2, b2 = mlp
    cin, hid = w1.shape
    K = HZ.NB
    ex = np.zeros_like(p["x"])
    if w3 is not None:   # the relative depth (an fp32 dot product of 32) and the upsampled embedding (fp32 lerps)
        ex[:, 32] = 34 * EPS32 * (np.abs(R.f64(act)) @ np.abs(R.f64(w3)).reshape(-1) + abs(float(np.ravel(b3)[0])))
    ex[:, -HZ.E:] = (8 + 8 * max(He, We)) * EPS32 * float(np.abs(R.f64(emb)).max())
    e_h = (cin + 1) * EPS32 * (np.abs(p["x"]) @ np.abs(w1) + np.abs(b1)) + ex @ np.abs(w1)
    e_g = 1.13 * e_h + 2.0 ** -21 * np.abs(p["h"]) + 4 * EPS32 * np.abs(p["g"])
    e_o = (hid + 1) * EPS32 * (np.abs(p["g"]) @ np.abs(w2).T + np.abs(b2)) + e_g @ np.abs(w2).T
    # Softplus' = sigmoid = 1 - exp(-softplus), at most e^e_o times larger anywhere within e_o of the pre-activation
    e_s = e_o * -np.expm1(-p["o"]) * np.exp(e_o) + 8 * EPS32 * p["o"]
    dp = (e_s[:, 0] + e_s[:, 1]) / p["pa_pb"] + 4 * EPS32
    t = p["t"]
    dt = (tmax - tmin) * ((e_s[:, 2] + e_s[:, 3]) / p["ta_tb"] + 4 * EPS32) + 2 * EPS32 * t
    lp, lq = np.log(p["p"]), np.log(p["q"])
    e_lp = dp / np.maximum(p["p"] - dp, 1e-4) + 2 * EPS32 * np.abs(lp)
    e_lq = dp / np.maximum(p["q"] - dp, 1e-4) + 2 * EPS32 * np.abs(lq)
    k = np.arange(K, dtype=np.float64)
    n_, kk, nk = K - 1 + 1e-7, k + 1e-7, K - 1 - k

    def tl(v):  # v log v evaluated in fp32 on an fp32 argument (1e-7 lost in the rounding of k + 1e-7)
        v = np.maximum(v, 1e-7)
        return 6 * EPS32 * np.abs(v * np.log(v)) + (np.abs(np.log(v)) + 1) * 2 * EPS32 * v
    e_lb = tl(n_) + tl(kk) + tl(nk + 1e-7) + 2 * EPS32 * np.abs(p["lbk"])
    e_y = (e_lb[None] + k[None] * e_lp[:, None] + nk[None] * e_lq[:, None]
           + 4 * EPS32 * (np.abs(p["lbk"])[None] + k[None] * np.abs(lp)[:, None] + nk[None] * np.abs(lq)[:, None]))
    lg = p["lg"]
    # the device's temperature is at least min_temp: |y / t' - y / t| <= |y| dt / (t max(t - dt, min_temp))
    e_l = e_y / t[:, None] + np.abs(p["y"]) * (dt / (t * np.maximum(t - dt, tmin)))[:, None] + EPS32 * np.abs(lg)
    delta = e_l.max(1) + 2 * EPS32 * (lg.max(1) - lg.min(1))
    wgt, c = p["wgt"], p["c"]
    e_c = (8 + 8 * max(He, We)) * EPS32 * float(np.abs(R.f64(bins)).max())
    rest = e_c + (2 * K + 8) * EPS32 * (wgt * np.abs(c)).sum(1)
    tol = np.expm1(np.minimum(2 * delta, 700.0)) * (wgt * np.abs(c - d[:, None])).sum(1) + rest
    # the depth is a convex combination of the bins whatever the logits: where a near-zero temperature pair makes the
    # propagated bound wider than the bins' spread, the spread is the bound
    cap = c.max(1) - c.min(1) + rest
    tight = float((tol < cap).mean())
    print(f"[depth-kernels] {what}: propagated bound tighter than the bins' spread on {tight:.1%} of the pixels")
    assert tight >= 0.5
    return report(what, np.abs(R.f64(dev).reshape(-1) - d), np.minimum(tol, cap))


def check_zoe(e, P, sd, cfg, B, b, tag, want_route=None):
    """the metric-head chain of image b of the last forward of e, from its z.* buffers"""
    H, W, F_ = e.image_h, e.image_w, cfg["fusion"]
    nc = len(cfg["bins"])
    sfx = "" if B == 1 else f"#{b}"
    g = lambda n, shape, dt=np.float16: e.get_buffer(n + sfx, shape, dt)  # noqa: E731
    bh, bw = H // 32, W // 32
    sizes = [(H // 16, W // 16), (H // 8, W // 8), (H // 4, W // 4), (H // 2, W // 2)]
    nb3, (h2, w2_), (h3, w3_) = bh * bw, sizes[2], sizes[3]
    M3 = h3 * w3_
    ms, mp = P["z.s1.b"].size // nc, P["z.sp1.b"].size
    bott = g("f3", (nb3, F_))
    zb16, zb32 = g("z.zb16", (nb3, F_)), g("z.zb32", (nb3, F_), np.float32)
    f32_check(zb32, HZ.lin(P, "z.bt", bott), HZ.lin_abs(P, "z.bt", bott), F_, f"z.zb32 (bottleneck conv2) {tag}")
    assert np.array_equal(zb16, zb32.astype(np.float16)), "z.zb16 is the same GEMM as z.zb32, rounded"
    route = int(g("z.route", (4,), np.int32)[0])
    if nc == 2:
        lg = g("z.logits", (2,), np.float32)
        sd64 = {k: v.double() for k, v in sd.items() if v.is_floating_point()}
        with torch.no_grad():
            ref = HZ.router64(sd64, torch.from_numpy(zb32.astype(np.float64)).t().reshape(1, F_, bh, bw)).numpy()
        report(f"z.logits (router of z.zb32) {tag}", np.abs(lg - ref), np.full(2, ROUTER_BOUND))
        assert route == int(lg[1] > lg[0])
    else:
        assert route == 0
    if want_route is not None:
        assert route == want_route, (route, want_route)
    sh = g("z.sh", (nb3, nc * ms))
    stored_f16(sh, HZ.lin(P, "z.s1", zb16, relu=True), ACC(F_) * HZ.lin_abs(P, "z.s1", zb16),
               f"z.sh (seed conv1, {nc} configurations) {tag}")
    seed = g("z.seed", (nb3, nc * HZ.NB), np.float32)
    Pabs = {"z.s2.w": np.abs(R.f64(P["z.s2.w"])), "z.s2.b": np.abs(R.f64(P["z.s2.b"]))}
    ref = HZ.seed_conv2(P, sh, nc)
    f32_check(seed, ref, HZ.seed_conv2(Pabs, np.abs(R.f64(sh)), nc), nc * ms,
              f"z.seed (block-diagonal seed conv2, both configurations' columns) {tag}", 2 * EPS32 * np.abs(ref))
    # the last projector (j = 3) and its residual; z.emb0 is the j = 2 embedding the residual upsamples
    fused = g("fused3", (M3, F_))
    t1 = g("z.t1", (M3, mp))
    stored_f16(t1, HZ.lin(P, "z.p3.1", fused, relu=True), ACC(F_) * HZ.lin_abs(P, "z.p3.1", fused),
               f"z.t1 (projector 3 conv1) {tag}")
    emb1, emb0, up = g("z.emb1", (M3, HZ.E)), g("z.emb0", (h2 * w2_, HZ.E)), g("z.up", (h3, w3_, HZ.E))
    stored_f16(emb1, HZ.lin(P, "z.p3.2", t1), ACC(mp) * HZ.lin_abs(P, "z.p3.2", t1), f"z.emb1 (projector 3) {tag}")
    up_check(up, emb0.reshape(h2, w2_, HZ.E), h3, w3_, f"z.up (embedding 2 upsampled) {tag}")
    up = up.reshape(M3, HZ.E)
    x = g("z.x", (M3, HZ.E))
    stored_f16(x, HZ.lin(P, "z.p3.2", t1) + R.f64(up), ACC(mp) * (HZ.lin_abs(P, "z.p3.2", t1) + np.abs(R.f64(up))),
               f"z.x (projector 3 + res_f16) {tag}")
    assert np.abs(R.f64(up)).mean() > 0.1 * np.abs(R.f64(x)).mean()        # the residual matters
    hid = g("z.hid", (M3, nc * HZ.E))
    stored_f16(hid, HZ.lin(P, "z.a3.1", x, relu=True), ACC(HZ.E) * HZ.lin_abs(P, "z.a3.1", x),
               f"z.hid (attractor conv1, {nc} configurations) {tag}")
    bins0, bins1 = g("z.bins0", (h2 * w2_, HZ.NB), np.float32), g("z.bins1", (M3, HZ.NB), np.float32)
    attractor_check(bins1, HZ.route_cols(hid, route, HZ.E), R.f64(P["z.a3.2.w"])[route], R.f64(P["z.a3.2.b"])[route],
                    bins0, h2, w2_, h3, w3_, f"z.bins1 (attractor 3, route {route}) {tag}")
    F2 = (F_ // 2 + 63) // 64 * 64
    h1u, act = g("h1u", (H, W, F2)), g("z.act", (H, W, 32))
    conv_check(act, h1u, P["h.c2.w"], P["h.c2.b"], f"z.act (3x3 + ReLU, N = 32) {tag}", relu=True)
    depth = e.get_buffer("depth" if b == 0 else f"depth.{b}", (H, W), np.float32)
    cat = nc == 1
    cin = 32 + int(cat) + HZ.E
    hidn = (P["z.lb"].size // nc - 4) // (cin + 5)
    mlp = HZ.logbinom_unpack(P["z.lb"], nc, cin, hidn, route)
    logbinom_check(depth, act.reshape(-1, 32), emb1, bins1, h3, w3_, H, W, mlp, cfg["min_temp"], cfg["max_temp"],
                   P["h.c3.w"] if cat else None, P["h.c3.b"] if cat else None, f"depth (log-binomial) {tag}")
    return route


def _zoe(sd, cfg, H, W):
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import prepare_zoedepth
    e = DepthEngine(cfg, H, W, family="zoedepth")
    e.load_state_dict(sd)
    return e, prepare_zoedepth(sd, cfg, H, W)


def _zoe_frames(B, H, W, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(B)]


@pytest.mark.parametrize("multi,route", [(True, 0), (True, 1), (False, None)])
def test_zoe_metric_head_buffers(multi, route):
    sd, cfg = ZO.random_model(multi=multi, seed=3 if multi else 4)
    sd = stress(sd, 21)
    if multi:
        sd = _route_bias(sd, 50.0 if route else -50.0)
    e, P = _zoe(sd, cfg, 64, 96)
    try:
        e.infer_batch(_zoe_frames(1, 64, 96, 1), check_size=False)
        tag = f"{'2 configurations' if multi else '1 configuration'} 64x96"
        check_zoe(e, P, sd, cfg, 1, 0, tag, route if multi else 0)
    finally:
        e.close()


def test_zoe_metric_head_batch_of_two_routes():
    """B = 2 images on different routes (the classifier's bias split between their logit margins): the per-tail
    buffers z.*#b of each image, each on its own route."""
    from visiondepth3d_b200.depth_weights import prepare_zoedepth
    from visiondepth3d_b200.synth import synth_frame
    sd, cfg = ZO.random_model(multi=True, seed=3)
    sd = stress(sd, 22, router=False)   # the router's input keeps the model's scale: logit margins vary by image
    e, P = _zoe(sd, cfg, 384, 672)
    try:
        frames = [synth_frame(i, 1920, 1080, k)[0] for i, k in
                  ((1, "natural"), (2, "noise"), (3, "smooth"), (4, "natural"), (5, "noise"), (6, "smooth"))]
        diffs = []
        for f in frames:
            e.infer_batch([f])
            lg = e.get_buffer("z.logits", (2,), np.float32)
            diffs.append(float(lg[1] - lg[0]))
        lo, hi = int(np.argmin(diffs)), int(np.argmax(diffs))
        assert diffs[hi] > diffs[lo], diffs
        sd = _route_bias(sd, -(diffs[lo] + diffs[hi]) / 2)
        e.load_state_dict(sd)
        P = prepare_zoedepth(sd, cfg, 384, 672)
        e.infer_batch([frames[lo], frames[hi]])
        routes = [check_zoe(e, P, sd, cfg, 2, b, f"B=2 image {b}") for b in range(2)]
        assert routes == [0, 1], routes
    finally:
        e.close()


def test_zoe_metric_head_at_the_real_widths():
    """fusion and bottleneck 256, a 384 x 672 image (a 1080p frame's processed size: bottleneck grid 12 x 21), on the
    small BEiT trunk"""
    sd, cfg = ZO.random_model(multi=True, seed=5, fusion=256, bottleneck=256)
    sd = _route_bias(stress(sd, 23), 50.0)
    e, P = _zoe(sd, cfg, 384, 672)
    try:
        e.infer_batch(_zoe_frames(1, 384, 672, 3), check_size=False)
        check_zoe(e, P, sd, cfg, 1, 0, "fusion 256 384x672", 1)
    finally:
        e.close()
