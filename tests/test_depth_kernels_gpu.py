"""GPU: every kernel of the depth forward on its own, against the float64 restatements of tests/depth_kernel_refs.py
(pinned to oracle/depth.py and torch in tests/test_depth_kernel_refs_cpu.py).

Each check reads the activation buffers of the last forward (DepthEngine.get_buffer) and recomputes ONE kernel in
float64 from the inputs the device itself stored for it, with the prepared (f16-rounded) weights, so the error
budget is one kernel's and not the model's.  The residual epilogues are isolated by running the same input again
with the layer's LayerScale at zero (x += 0 * (...) leaves x exact) and subtracting.

Error model (asserted, printed beside the observed worst case as "observed / bound", 1.0 = at the bound):
  * an f16 store rounds to nearest: half an ulp of the stored value;
  * a GEMM accumulates f16 products in fp32 on the tensor core, which truncates when it adds a k16 product sum: at most
    one fp32 ulp (2^-23) per k16 step inside a group of 256, then one rounding (2^-24) per group added in the FP32
    pipe, relative to sum |a| |b|: ACC(K) = (2 * min(K, 256) / 16 + ceil(K / 256) + 4) * 2^-24;
  * attention: the probabilities are f16 (2^-11 each) in numerator and denominator alike, so the softmax weights move
    by at most 2 * 2^-11, the logits carry ACC(64) of sum |q| |k|, P V accumulates NT / 16 k16 steps.
Models are synthetic (tests/depth_kernel_refs.synth_state_dict), four blocks deep at the real widths."""
import math

import numpy as np
import pytest

from tests import depth_kernel_refs as R

pytestmark = pytest.mark.gpu

REAL = {"vits": (384, [48, 96, 192, 384], 64), "vitb": (768, [96, 192, 384, 768], 128),
        "vitl": (1024, [256, 512, 1024, 1024], 256)}
TINY = (128, [48, 96, 64, 128], 64)


def ACC(K):
    return (2 * min(K, 256) / 16 + math.ceil(K / 256) + 4) * R.F32_EPS


def report(what, err, tol):
    """worst observed error as a fraction of its bound; fails above 1."""
    ratio = np.max(np.asarray(err, dtype=np.float64) / np.asarray(tol, dtype=np.float64))
    i = np.argmax(np.asarray(err, dtype=np.float64) / np.asarray(tol, dtype=np.float64))
    print(f"[depth-kernels] {what}: observed / bound = {ratio:.3f} (worst abs err {np.ravel(err)[i]:.3e})")
    assert np.isfinite(ratio) and ratio <= 1.0, (what, float(ratio))
    return float(ratio)


def stored_f16(dev, ref, slack, what):
    """dev: f16 values the device stored; ref: float64; slack: bound on the error before the store."""
    err = np.abs(R.f64(dev) - ref)
    return report(what, err, 0.5 * R.f16_ulp(np.abs(ref) + slack) + slack)


class Rig:
    """One engine with a synthetic model whose prepared tensors stay on the host: overwrite one, run, restore."""

    def __init__(self, hidden, neck, fusion, h, w, seed=0):
        from visiondepth3d_b200.depth_engine import DepthEngine
        from visiondepth3d_b200.depth_weights import prepare
        self.cfg = R.small_config(hidden, neck, fusion)
        self.h, self.w, self.ph, self.pw = h, w, h // 14, w // 14
        self.D, self.H, self.L = hidden, hidden // 64, self.cfg["layers"] - 1
        self.NT = self.ph * self.pw + 1
        self.NP = (self.NT + 127) // 128 * 128
        self.eng = DepthEngine(self.cfg, h, w)
        self.base = {k: np.ascontiguousarray(v) for k, v in prepare(R.synth_state_dict(self.cfg, seed), self.cfg, h, w).items()}
        rng = np.random.default_rng(seed + 100)
        D, L = self.D, self.L
        for i in range(self.cfg["layers"]):
            self.base[f"l{i}.ls1"] = rng.uniform(0.5, 1.5, D).astype(np.float32)
            self.base[f"l{i}.ls2"] = rng.uniform(0.5, 1.5, D).astype(np.float32)
        # last block: logits with a standard deviation of several units (q and k weights doubled), and a V bias that
        # differs from head to head, so that a head written to another head's slot cannot go unnoticed
        wq = self.base[f"l{L}.qkv.w"].astype(np.float32)
        wq[:2 * D] *= 2.0
        self.base[f"l{L}.qkv.w"] = wq.astype(np.float16)
        bq = self.base[f"l{L}.qkv.b"].copy()
        bq[2 * D:] += 0.5 * np.repeat(np.arange(self.H), 64)
        self.base[f"l{L}.qkv.b"] = bq
        # a head whose last projection has both signs, so that its final ReLU clips about half of the pixels
        w3 = self.base["h.c3.w"].copy()
        w3[::2] *= -1
        self.base["h.c3.w"] = w3
        self.P, self.dirty = {}, set()
        self.restore(*self.base)

    def set(self, name, arr):
        b = self.base[name]
        arr = np.ascontiguousarray(np.broadcast_to(np.asarray(arr, dtype=b.dtype), b.shape))
        self.P[name] = arr
        self.dirty.add(name)
        self.eng.check(self.eng.lib.vd3d_depth_set_tensor(self.eng.h, name.encode(), arr.ctypes.data, arr.nbytes))

    def restore(self, *names):
        """the named tensors, or every overwritten one, back to the model's own"""
        for n in names or sorted(self.dirty):
            self.set(n, self.base[n])
            self.dirty.discard(n)

    def last(self, name):
        return f"l{self.L}.{name}"

    def frames(self, n, seed=0):
        rng = np.random.default_rng(seed)
        return [rng.integers(0, 256, (self.h, self.w, 3), dtype=np.uint8) for _ in range(n)]

    def run(self, frames):
        """one batched forward of BGR frames at the processed size (the resize is then the identity)"""
        self.B = len(frames)
        return self.eng.infer_batch(frames, check_size=False)

    def buf(self, name, shape, dtype=np.float16):
        return self.eng.get_buffer(name, shape, dtype)

    def tok(self, name, cols=None, dtype=np.float16):
        return self.buf(name, (self.B * self.NP, cols or self.D), dtype)

    def qkv(self):
        B, H, NP = self.B, self.H, self.NP
        return self.buf("q", (B, H, NP, 64)), self.buf("k", (B, H, NP, 64)), self.buf("vt", (B, H, 64, NP))

    def rows(self, B):
        """rows of the stacked token matrix of B images that hold tokens"""
        return np.concatenate([b * self.NP + np.arange(self.NT) for b in range(B)])

    def close(self):
        self.eng.close()


_rigs = {}


def rig_for(name):
    if name not in _rigs:
        if name == "tiny":
            _rigs[name] = Rig(*TINY, 70, 98, seed=5)
        else:
            _rigs[name] = Rig(*REAL[name], 518, 924, seed={"vits": 1, "vitb": 2, "vitl": 3}[name])
    return _rigs[name]


@pytest.fixture(scope="module", autouse=True)
def _close_rigs():
    yield
    for r in _rigs.values():
        r.close()
    _rigs.clear()


# ---------------------------------------------------------------------------------------------------------------------
# 1. attention, isolated
# ---------------------------------------------------------------------------------------------------------------------
def check_attention(rig, what, min_std=3.0):
    """attn against float64 softmax(q k^T) v from the q, k, v^T the device stored; returns the logits of head 0."""
    q, k, vt = rig.qkv()
    NT, NP, B = rig.NT, rig.NP, rig.B
    ref, mag = R.attention(q, k, vt, NT, with_abs=True)
    dev = rig.tok("attn").reshape(B, NP, rig.D)
    sabs = max(float((np.abs(R.f64(q[b, h, :NT])) @ np.abs(R.f64(k[b, h, :NT])).T).max())
               for b in range(B) for h in range(rig.H))
    vmax = float(np.abs(R.f64(vt)).max())
    rel = 2 * R.F16_EPS + 2 * ACC(64) * sabs + (NT / 16 + NP / 128 + 8) * 2 * R.F32_EPS
    slack = rel * mag + NT * 2.0 ** -32 * vmax
    stored_f16(dev[:, :NT], ref, slack, what)
    lg = R.attention_logits(q[0, 0], k[0, 0], NT)
    if min_std:
        assert lg.std() >= min_std, ("the fixture no longer gives a peaked softmax", float(lg.std()))
    # query rows that do not exist are skipped by the kernel: they keep the zeros the buffer was allocated with
    assert not dev[-1, NT:].any()
    return lg, dev


class AttnRig(Rig):
    """Two heads, every block but the last switched off and the patch projection small, so that the residual stream
    entering the last block is the position table: one freely chosen vector per token.  Token n is z_n + a_n u with
    z_n random and orthogonal to the fixed direction u; channel 0 of every head's key reads u, channel 0 of every
    query is the constant 1, so key n gets the logit offset gamma * a_n / sqrt(1 + a_n^2) on top of random logits."""
    GAMMA = 128.0

    def __init__(self, h, w):
        super().__init__(*TINY, h, w, seed=7)
        D, L = self.D, self.L
        for i in range(self.cfg["layers"]):
            if i < L:
                self.base[f"l{i}.ls1"] = np.zeros(D, np.float32)
                self.base[f"l{i}.ls2"] = np.zeros(D, np.float32)
        self.base["pe.w"] = (self.base["pe.w"].astype(np.float32) * 0.02).astype(np.float16)
        self.base["pe.b"] = np.zeros(D, np.float32)
        self.base["cls"] = np.zeros(D, np.float32)
        self.base[self.last("ln1.g")] = np.ones(D, np.float32)
        self.base[self.last("ln1.b")] = np.zeros(D, np.float32)
        self.u = np.where(np.arange(D) % 2 == 0, 1.0, -1.0)
        self.restore(*self.base)

    def design(self, offsets, noise):
        """offsets: wanted logit offset per key [NT] (< 0.7 * GAMMA); noise: standard deviation of the random logits."""
        D, H, NT, L = self.D, self.H, self.NT, self.L
        rng = np.random.default_rng(11)
        z = rng.standard_normal((NT, D))
        z -= z.mean(axis=1, keepdims=True)
        z -= np.outer(z @ self.u / D, self.u)
        z /= z.std(axis=1, keepdims=True)
        t = np.asarray(offsets, dtype=np.float64) / self.GAMMA
        a = t / np.sqrt(1 - t * t)
        self.set("pos", (z + a[:, None] * self.u).astype(np.float32))
        s = math.sqrt(noise) if noise else 0.0
        w = rng.standard_normal((3 * D, D)) / math.sqrt(D)
        w[:2 * D] *= s
        b = np.zeros(3 * D)
        b[2 * D:] = rng.standard_normal(D)
        for hd in range(H):
            w[hd * 64] = 0.0
            b[hd * 64] = 8.0 if noise is not None else 0.0         # q channel 0 = 8 * 0.125
            w[D + hd * 64] = self.GAMMA * self.u / D
        if noise is None:                                          # every logit equal: q = 0
            w[:D] = 0.0
        self.set(self.last("qkv.w"), w.astype(np.float16))
        self.set(self.last("qkv.b"), b.astype(np.float32))


GRIDS = [(15, 17), (8, 16), (9, 14), (5, 7), (37, 66)]   # tokens 256, 129, 127, 36, 2443: NT % 128 = 0, 1, 127, 36, 11


@pytest.mark.parametrize("ph,pw", GRIDS)
def test_attention_peaked_softmax_and_key_tile_tails(ph, pw):
    rig = AttnRig(14 * ph, 14 * pw)
    NT, T = rig.NT, (rig.NT + 127) // 128
    fr = rig.frames(1)
    tile = np.arange(NT) // 128

    def gaps(lg):
        top2 = np.sort(lg, axis=1)[:, -2:]
        return top2[:, 1] - top2[:, 0]

    # the row maximum in the first key tile, far above the runner-up
    off = np.zeros(NT)
    off[5] = 88.0
    rig.design(off, 4.0)
    rig.run(fr)
    lg, _ = check_attention(rig, f"attention {ph}x{pw} peak in the first tile")
    assert (lg.argmax(axis=1) == 5).all() and np.median(gaps(lg)) > 60
    # ... in the last tile, on the very last key
    off = np.zeros(NT)
    off[NT - 1] = 88.0
    rig.design(off, 4.0)
    rig.run(fr)
    lg, _ = check_attention(rig, f"attention {ph}x{pw} peak on the last key")
    assert (lg.argmax(axis=1) == NT - 1).all() and np.median(gaps(lg)) > 60
    # ... moving up tile by tile: the running maximum changes, and the accumulator is rescaled, at every step
    step = min(8.0, 80.0 / max(T - 1, 1))
    rig.design(step * tile, 1.0)
    rig.run(fr)
    lg, _ = check_attention(rig, f"attention {ph}x{pw} maximum rising tile by tile", min_std=0)
    if T > 1:
        tmax = np.stack([lg[:, tile == t].max(axis=1) for t in range(T)], axis=1)
        assert (np.diff(tmax, axis=1) > 0).all(axis=1).mean() > 0.9
    # ... and all logits equal: the mean of v over exactly NT keys
    rig.design(np.zeros(NT), None)
    rig.run(fr)
    lg, dev = check_attention(rig, f"attention {ph}x{pw} all logits equal", min_std=0)
    assert not lg.any()
    rig.close()


def test_attention_never_reads_padded_keys_and_batch_index():
    """Rows [NT, NP) of k and v^T of every image but the last are written by the QKV GEMM (they are rows of the stacked
    token matrix, LayerNorm of a zero row is its bias, zero here): their keys are 0.  Every real key is pushed ~57
    logits below that, so one padded key that took part would take all the weight.  The result must be the same bits
    as each image alone."""
    rig = AttnRig(70, 98)
    D, NT, NP = rig.D, rig.NT, rig.NP
    rig.design(np.full(NT, -57.0), 4.0)
    fr = rig.frames(3, seed=4)
    alone = []
    for f in fr:
        rig.run([f])
        alone.append(rig.tok("attn")[:NT].copy())
    assert not np.array_equal(alone[0], alone[1])
    rig.run(fr)
    q, k, vt = rig.qkv()
    assert (q[:, :, :NT, 0] == 1).all() and (k[:, :, :NT, 0] < -45).all() and not k[:, :, NT:].any()
    assert np.abs(vt[0, :, :, NT:]).max() > 1                      # a padded value is there to be picked up
    check_attention(rig, "attention B=3, padded keys 57 logits above the real ones", min_std=0)
    dev = rig.tok("attn").reshape(3, NP, D)
    for i in range(3):
        assert np.array_equal(dev[i, :NT], alone[i]), i
        assert not dev[i, NT:].any(), i
    rig.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. token-stage kernels of the last block, 3. neck and head
# ---------------------------------------------------------------------------------------------------------------------
_stage = {}


def stage(name, B):
    """Three forwards of one input.  A: both LayerScales of the last block zero and its second LayerNorm made equal to
    the first (x is the block's input; xn is the very LayerNorm output the QKV GEMM read).  M: only the second zero (x
    is the state between proj and fc2).  F: the model as it is."""
    key = (name, B)
    if key in _stage:
        return _stage[key]
    rig = rig_for(name)
    fr = rig.frames(B, seed=B)
    g = lambda *n: {k: rig.tok(k, c, t) for k, c, t in n}  # noqa: E731
    D = rig.D
    rig.set(rig.last("ls1"), 0.0)
    rig.set(rig.last("ls2"), 0.0)
    rig.set(rig.last("ln2.g"), rig.P[rig.last("ln1.g")])
    rig.set(rig.last("ln2.b"), rig.P[rig.last("ln1.b")])
    rig.run(fr)
    A = g(("x", D, np.float32), ("xn", D, np.float16), ("attn", D, np.float16), ("h", 4 * D, np.float16))
    A["q"], A["k"], A["vt"] = rig.qkv()
    rig.restore(rig.last("ls1"), rig.last("ln2.g"), rig.last("ln2.b"))
    rig.run(fr)
    M = g(("x", D, np.float32), ("xn", D, np.float16), ("h", 4 * D, np.float16))
    rig.restore(rig.last("ls2"))
    out = rig.run(fr)
    Fd = g(("x", D, np.float32))
    Fd["tail"] = {b: grab_tail(rig, b) for b in sorted({0, B - 1})}
    _stage[key] = (rig, A, M, Fd, out)
    return _stage[key]


def grab_tail(rig, b):
    """every neck / fusion / head buffer of image b of the forward that just ran, in its NHWC shape"""
    cfg, ph, pw, Fz = rig.cfg, rig.ph, rig.pw, rig.cfg["fusion"]
    nm = (lambda n: n) if rig.B == 1 else (lambda n: f"{n}#{b}")
    t = {}
    dims = [(4 * ph, 4 * pw), (2 * ph, 2 * pw), (ph, pw), ((ph - 1) // 2 + 1, (pw - 1) // 2 + 1)]
    for i, C in enumerate(cfg["neck"]):
        CP = (C + 63) // 64 * 64
        t[f"tap{i}"] = rig.buf(f"tap{i}.{b}", (ph * pw, rig.D))
        t[f"r{i}.p"] = rig.buf(nm(f"r{i}.p"), (ph * pw, CP))
        if i < 2:
            t[f"r{i}.s"] = rig.buf(nm(f"r{i}.s"), dims[i] + (CP,))
        if i == 3:
            t["r3.col"] = rig.buf(nm("r3.col"), (dims[3][0] * dims[3][1], 9 * CP))
            t["r3.s"] = rig.buf(nm("r3.s"), dims[3] + (CP,))
        t[f"f{i}"] = rig.buf(nm(f"f{i}"), dims[i] + (Fz,))
    fh, fw = dims[0]
    for n in ("fu.relu", "fu.h", "fu.hrelu", "fu.mid", "fu.y", "fused2"):
        t[n] = rig.buf(nm(n), (fh, fw, Fz))
    F2 = (Fz // 2 + 63) // 64 * 64
    t["fu.up3"] = rig.buf(nm("fu.up3"), (2 * fh, 2 * fw, Fz))
    t["fused3"] = rig.buf(nm("fused3"), (2 * fh, 2 * fw, Fz))
    t["h1"] = rig.buf(nm("h1"), (2 * fh, 2 * fw, F2))
    t["h1u"] = rig.buf(nm("h1u"), (rig.h, rig.w, F2))
    t["depth"] = rig.buf("depth" if b == 0 else f"depth.{b}", (rig.h, rig.w), np.float32)
    return t


CASES = [("vits", 1), ("vitb", 1), ("vitl", 1), ("vits", 4), ("tiny", 2)]


@pytest.mark.parametrize("name,B", CASES)
def test_layernorm(name, B):
    rig, A, M, Fd, _ = stage(name, B)
    P, rows = rig.P, rig.rows(B)

    def check(dev, x, g, b, what):
        ref = R.layernorm(x, g, b).astype(np.float16)          # <= 1 f16 ulp off, and almost never off at all
        d = np.abs(R.f64(dev) - R.f64(ref))
        off = float((d > 0).mean())
        print(f"[depth-kernels] {what}: {off:.2e} of the elements differ from the rounded float64 result, max "
              f"{float((d / R.f16_ulp(ref)).max()):.1f} ulp (bounds 1e-2, 1)")
        assert (d <= R.f16_ulp(ref)).all() and off <= 1e-2, what

    check(A["xn"][rows], A["x"][rows], P[rig.last("ln1.g")], P[rig.last("ln1.b")], f"k_layernorm {name} B={B} ln1")
    check(M["xn"][rows], M["x"][rows], P[rig.last("ln2.g")], P[rig.last("ln2.b")], f"k_layernorm {name} B={B} ln2")
    NPATCH = rig.NT - 1
    assert NPATCH == rig.ph * rig.pw
    for b, t in Fd["tail"].items():      # the tap variant: final norm, CLS row dropped
        check(t["tap3"], Fd["x"][b * rig.NP + 1: b * rig.NP + rig.NT], P["norm.g"], P["norm.b"],
              f"k_layernorm {name} B={B} tap of image {b}")


@pytest.mark.parametrize("name,B", CASES)
def test_qkv_epilogue(name, B):
    rig, A, *_ = stage(name, B)
    W, bias = rig.P[rig.last("qkv.w")], rig.P[rig.last("qkv.b")]
    MT = (B - 1) * rig.NP + rig.NT
    xn = np.zeros((B * rig.NP, rig.D))
    xn[:MT] = A["xn"][:MT]
    y = R.linear(xn, W, bias)
    slack = ACC(rig.D) * R.linear_abs(xn, W, bias)
    q, k, vt = R.qkv_split(y, B, rig.NP, rig.NT, rig.H)
    sq, sk, sv = R.qkv_split(slack, B, rig.NP, rig.NT, rig.H)
    NT = rig.NT
    stored_f16(A["q"][:, :, :NT], q, sq, f"EPI_QKV {name} B={B} q")
    stored_f16(A["k"][:, :, :NT], k, sk, f"EPI_QKV {name} B={B} k")
    stored_f16(A["vt"][:, :, :, :NT], vt, sv, f"EPI_QKV {name} B={B} vT")
    if B > 1:
        assert not np.array_equal(A["q"][0, :, :NT], A["q"][1, :, :NT])     # the images differ: a dropped index shows


@pytest.mark.parametrize("name,B", CASES)
def test_attention_at_model_width(name, B):
    rig, A, *_ = stage(name, B)
    q, k, vt = A["q"], A["k"], A["vt"]
    NT, NP = rig.NT, rig.NP
    ref, mag = R.attention(q, k, vt, NT, with_abs=True)
    sabs = max(float((np.abs(R.f64(q[b, h, :NT])) @ np.abs(R.f64(k[b, h, :NT])).T).max())
               for b in range(B) for h in range(rig.H))
    rel = 2 * R.F16_EPS + 2 * ACC(64) * sabs + (NT / 16 + NP / 128 + 8) * 2 * R.F32_EPS
    slack = rel * mag + NT * 2.0 ** -32 * float(np.abs(R.f64(vt)).max())
    stored_f16(A["attn"].reshape(B, NP, rig.D)[:, :NT], ref, slack, f"attention {name} B={B} ({rig.H} heads)")
    lg = R.attention_logits(q[B - 1, rig.H - 1], k[B - 1, rig.H - 1], NT)
    assert lg.std() >= 3.0, float(lg.std())


@pytest.mark.parametrize("name,B", CASES)
def test_fc1_gelu_epilogue(name, B):
    rig, _, M, *_ = stage(name, B)
    rows = rig.rows(B)
    W, bias = rig.P[rig.last("fc1.w")], rig.P[rig.last("fc1.b")]
    pre = R.linear(M["xn"][rows], W, bias)
    # |gelu'| <= 1.13; the erfc polynomial is within 1.5e-7, times |x| / 2; two approximate MUFU results (2^-22 each)
    slack = 1.13 * ACC(rig.D) * R.linear_abs(M["xn"][rows], W, bias) + 1e-7 * np.abs(pre) + 2.0 ** -21 * np.abs(R.gelu(pre))
    stored_f16(M["h"][rows], R.gelu(pre), slack, f"EPI_F16 + GELU {name} B={B}")


def test_gelu_over_the_whole_range():
    """Pre-activations swept over [-6, 6] by the bias: the left tail, where a tanh form or a cancelling 1 + erf differs."""
    rig = rig_for("vits")
    n = rig.P[rig.last("fc1.b")].size
    rig.set(rig.last("fc1.w"), (rig.base[rig.last("fc1.w")].astype(np.float32) * 0.05).astype(np.float16))
    rig.set(rig.last("fc1.b"), np.linspace(-6, 6, n).astype(np.float32))
    rig.run(rig.frames(1, seed=9))
    xn, h = rig.tok("xn")[:rig.NT], rig.tok("h", 4 * rig.D)[:rig.NT]
    W, bias = rig.P[rig.last("fc1.w")], rig.P[rig.last("fc1.b")]
    pre = R.linear(xn, W, bias)
    assert pre.min() < -5.9 and pre.max() > 5.9
    slack = 1.13 * ACC(rig.D) * R.linear_abs(xn, W, bias) + 1e-7 * np.abs(pre) + 2.0 ** -21 * np.abs(R.gelu(pre))
    stored_f16(h, R.gelu(pre), slack, "EPI_F16 + GELU sweep [-6, 6]")
    left = pre < -3
    assert left.mean() > 0.2 and (h[left] < 0).mean() > 0.9      # the left tail is resolved, not flushed to zero
    rig.restore()


def resid_check(x_after, x_before, a, W, bias, ls, what):
    ref = R.f64(ls) * R.linear(a, W, bias)
    tol = ACC(W.shape[1]) * np.abs(R.f64(ls)) * R.linear_abs(a, W, bias) + 2 * R.F32_EPS * np.abs(R.f64(x_after)) + 1e-30
    return report(what, np.abs(R.f64(x_after) - R.f64(x_before) - ref), tol)


@pytest.mark.parametrize("name,B", CASES)
def test_residual_layerscale_epilogue(name, B):
    rig, A, M, Fd, _ = stage(name, B)
    P, rows = rig.P, rig.rows(B)
    assert np.abs(M["x"][rows] - A["x"][rows]).max() > 0.1
    resid_check(M["x"][rows], A["x"][rows], A["attn"][rows], P[rig.last("proj.w")], P[rig.last("proj.b")],
                P[rig.last("ls1")], f"EPI_RESID_LS {name} B={B} proj (K = {rig.D})")
    resid_check(Fd["x"][rows], M["x"][rows], M["h"][rows], P[rig.last("fc2.w")], P[rig.last("fc2.b")],
                P[rig.last("ls2")], f"EPI_RESID_LS {name} B={B} fc2 (K = {4 * rig.D})")


def test_fc2_long_reduction_with_positive_operands():
    """K = 4096 with every product positive: rounding cannot cancel, and the tensor core's truncation is all of one
    sign.  The bound holds because the accumulator is promoted to an fp32 total every 256."""
    rig = rig_for("vitl")
    fc1w, fc2w = rig.base[rig.last("fc1.w")].astype(np.float32), rig.base[rig.last("fc2.w")].astype(np.float32)
    rng = np.random.default_rng(3)
    rig.set(rig.last("fc1.w"), (fc1w * 0.1).astype(np.float16))
    rig.set(rig.last("fc1.b"), rng.uniform(0.5, 1.5, 4 * rig.D).astype(np.float32))
    rig.set(rig.last("fc2.w"), (np.abs(fc2w) + 2.0 ** -10).astype(np.float16))
    rig.set(rig.last("fc2.b"), np.abs(rig.base[rig.last("fc2.b")]))
    rig.set(rig.last("ls2"), 0.0)
    fr = rig.frames(1, seed=6)
    rig.run(fr)
    x0, h = rig.tok("x", dtype=np.float32)[:rig.NT], rig.tok("h", 4 * rig.D)[:rig.NT]
    assert h.min() > 0
    rig.set(rig.last("ls2"), 1.0)
    rig.run(fr)
    x1 = rig.tok("x", dtype=np.float32)[:rig.NT]
    resid_check(x1, x0, h, rig.P[rig.last("fc2.w")], rig.P[rig.last("fc2.b")], rig.P[rig.last("ls2")],
                "EPI_RESID_LS vitl fc2, positive operands (K = 4096)")
    rig.restore()


@pytest.mark.parametrize("name", ["vits", "tiny"])
def test_patch_embedding(name):
    rig = rig_for(name)
    for i in range(rig.cfg["layers"]):
        rig.set(f"l{i}.ls1", 0.0)
        rig.set(f"l{i}.ls2", 0.0)
    rng = np.random.default_rng(8)
    px = rng.standard_normal((3, rig.h, rig.w)).astype(np.float32)
    rig.B = 1
    rig.eng.forward(px)
    P = rig.P
    x = rig.tok("x", dtype=np.float32)[:rig.NT]
    ape = rig.buf("ape", (rig.NT - 1, 592))
    assert np.array_equal(ape[:, :588], R.patch_im2col(px).astype(np.float16)) and not ape[:, 588:].any()
    assert np.array_equal(x[0], P["cls"] + P["pos"][0])
    ref = R.linear(ape, P["pe.w"], P["pe.b"]) + R.f64(P["pos"][1:])
    tol = ACC(592) * (R.linear_abs(ape, P["pe.w"], P["pe.b"]) + np.abs(P["pos"][1:])) + 2 * R.F32_EPS * np.abs(ref)
    report(f"EPI_PATCH {name}", np.abs(R.f64(x[1:]) - ref), tol)
    rig.restore()


def conv_check(dev, x, w, bias, what, relu=False, res=None):
    ref = R.conv3x3(x, w, bias)
    if res is not None:
        ref = ref + R.f64(res)
    slack = ACC(w.shape[1]) * (R.conv3x3_abs(x, w, bias) + (0 if res is None else np.abs(R.f64(res))))
    if relu:
        ref = np.maximum(ref, 0)
    return stored_f16(dev, ref, slack, what)


def lin_check(dev, x, w, bias, what):
    return stored_f16(dev, R.linear(x, w, bias), ACC(w.shape[1]) * R.linear_abs(x, w, bias), what)


def up_check(dev, x, OH, OW, what):
    H, W, _ = x.shape
    # fp32 source coordinates (a few 2^-24 of the map's size) times the largest step between neighbours, and the lerps
    slack = (8 + 8 * max(H, W)) * R.F32_EPS * float(np.abs(R.f64(x)).max())
    return stored_f16(dev, R.upsample_ac(x, OH, OW), slack, what)


@pytest.mark.parametrize("name,B", [("vits", 1), ("vits", 4), ("tiny", 2), ("vitb", 1)])
def test_neck_and_head(name, B):
    rig, _, _, Fd, out = stage(name, B)
    P, cfg, ph, pw = rig.P, rig.cfg, rig.ph, rig.pw
    Fz = cfg["fusion"]
    for b, T in Fd["tail"].items():
        tag = f"{name} B={B} image {b}"
        dims, feats = [], []
        for i, C in enumerate(cfg["neck"]):
            CP = (C + 63) // 64 * 64
            tap = T[f"tap{i}"]
            p = T[f"r{i}.p"]
            lin_check(p, tap, P[f"r{i}.proj.w"], P[f"r{i}.proj.b"], f"r{i}.p (1x1, {C} -> {CP} channels) {tag}")
            assert not p[:, C:].any()
            if i < 2:
                kk = 4 if i == 0 else 2
                fh, fw = ph * kk, pw * kk
                s = T[f"r{i}.s"]
                w, bias = P[f"r{i}.up.w"], P[f"r{i}.up.b"]
                ref = R.conv_transpose_scatter(R.linear(p, w, bias), ph, pw, kk, CP)
                slack = R.conv_transpose_scatter(ACC(CP) * R.linear_abs(p, w, bias), ph, pw, kk, CP)
                stored_f16(s, ref, slack, f"r{i}.s (EPI_CONVT k = {kk}) {tag}")
            elif i == 2:
                fh, fw, s = ph, pw, p.reshape(ph, pw, CP)
            else:
                fh, fw = (ph - 1) // 2 + 1, (pw - 1) // 2 + 1
                col = T["r3.col"]
                assert np.array_equal(col, R.im2col_s2(p.reshape(ph, pw, CP)).astype(np.float16)), "k_im2col_s2"
                s = T["r3.s"].reshape(fh * fw, CP)
                lin_check(s, col, P["r3.down.w"], P["r3.down.b"], f"r3.s (stride-2 conv) {tag}")
                s = s.reshape(fh, fw, CP)
            f = T[f"f{i}"]
            conv_check(f, s, P[f"n{i}.conv.w"], None, f"f{i} (3x3, {CP} -> {Fz}) {tag}")
            dims.append((fh, fw))
            feats.append(f)
        # last fusion stage (the fu.* buffers hold it): residual_layer1 on f0 is recomputed through its two f16
        # intermediates, which the stage overwrites; residual_layer2 is checked buffer by buffer
        fh, fw = dims[0]
        g = T.__getitem__
        relu0, hraw, hrelu, mid, y = g("fu.relu"), g("fu.h"), g("fu.hrelu"), g("fu.mid"), g("fu.y")
        assert np.array_equal(relu0, np.maximum(feats[0], 0)), "k_relu_f16"
        assert np.array_equal(hrelu, np.maximum(hraw, 0)), "k_add_relu_f16: relu copy"
        fused2 = T["fused2"]
        w1, b1, w2, b2 = (P[f"f3.rl1.{n}"] for n in ("c1.w", "c1.b", "c2.w", "c2.b"))
        mid1 = np.maximum(R.conv3x3(relu0, w1, b1), 0)
        e_mid = 0.5 * R.f16_ulp(mid1) + ACC(9 * Fz) * R.conv3x3_abs(relu0, w1, b1)
        y1 = R.conv3x3(mid1, w2, b2) + R.f64(feats[0])
        e_y1 = R.conv3x3(e_mid, np.abs(R.f64(w2))) + ACC(9 * Fz) * (R.conv3x3_abs(mid1, w2, b2) + np.abs(R.f64(feats[0])))
        e_y1 = e_y1 + 0.5 * R.f16_ulp(np.abs(y1) + e_y1)
        stored_f16(hraw, R.f64(fused2) + y1, e_y1 + 4 * R.F32_EPS * (np.abs(y1) + np.abs(R.f64(fused2))),
                   f"fu.h (residual_layer1 + k_add_relu_f16) {tag}")
        conv_check(mid, hrelu, P["f3.rl2.c1.w"], P["f3.rl2.c1.b"], f"fu.mid (3x3 + ReLU) {tag}", relu=True)
        conv_check(y, mid, P["f3.rl2.c2.w"], P["f3.rl2.c2.b"], f"fu.y (3x3 + f16 residual) {tag}", res=hraw)
        up = T["fu.up3"]
        up_check(up, y, 2 * fh, 2 * fw, f"fu.up3 (k_upsample_ac) {tag}")
        fused3 = T["fused3"]
        lin_check(fused3, up, P["f3.proj.w"], P["f3.proj.b"], f"fused3 (1x1) {tag}")
        F2 = (Fz // 2 + 63) // 64 * 64
        h1 = T["h1"]
        conv_check(h1, fused3, P["h.c1.w"], P["h.c1.b"], f"h1 (3x3) {tag}")
        h1u = T["h1u"]
        up_check(h1u, h1, rig.h, rig.w, f"h1u (k_upsample_ac to the image) {tag}")
        depth = T["depth"]
        assert np.array_equal(depth, out[b][0])         # frames at the processed size: nothing is resized back
        w3 = np.abs(R.f64(P["h.c3.w"]))
        t = np.maximum(R.conv3x3(h1u, P["h.c2.w"], P["h.c2.b"]), 0)
        ref = R.head(h1u, P["h.c2.w"], P["h.c2.b"], P["h.c3.w"], P["h.c3.b"])
        tol = (ACC(9 * F2) * R.conv3x3_abs(h1u, P["h.c2.w"], P["h.c2.b"])) @ w3 + 40 * R.F32_EPS * (t @ w3 + abs(float(P["h.c3.b"][0])))
        report(f"EPI_HEAD {tag}", np.abs(R.f64(depth) - ref), tol + 1e-30)
        assert 0.05 < (ref == 0).mean() < 0.95, "the fixture no longer exercises the final ReLU on both sides"


def test_create_rejects_unsupported_shapes():
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200.depth_engine import DepthEngine
    for cfg, h, w in ((R.small_config(192, TINY[1], 64), 70, 98), (R.small_config(128, TINY[1], 64), 71, 98),
                      (R.small_config(128, TINY[1], 64), 14 * 56, 14 * 56)):
        with pytest.raises(_lib.Vd3dError):
            DepthEngine(cfg, h, w)
