"""GPU: every kernel of the Real-ESRGAN networks on its own, against the float64 restatements of
tests/sr_kernel_refs.py (pinned to torch, oracle/sr.py and tests/rrdb_oracle.py in tests/test_sr_kernel_refs_cpu.py).

Each check reads the activation buffers of the last forward (vd3d_depth_get_buffer) and recomputes ONE kernel in
float64 from the f16 inputs the device itself stored for it and the f16 weights it was given, so the error budget is
one kernel's.  The weights are stress weights (sr_kernel_refs.stress_*): PReLU slopes distinct per channel over
[-0.5, 1.5] with one 0, biases distinct per output channel over [-0.5, 0.5], every conv at He scale, so that a slope,
bias or channel read from the wrong index moves outputs by O(1) and not by a fraction of an ulp.

Error model (asserted, printed beside the observed worst case as "observed / bound", 1.0 = at the bound), that of
tests/test_depth_kernels_gpu.py:
  * fp32 accumulation of f16 products on the tensor core: ACC(K) of sum |x| |w| (+ |bias|);
  * the EPI_SR residual chain res2 + rs2 (res + rs a): the accumulation error scaled by rs rs2, plus a few fp32
    roundings of the terms; PReLU / LeakyReLU scale the error by max(1, |slope|);
  * one f16 store: half an ulp of the stored value.  f32 outputs have no store rounding.
The byte kernels (k_sr_in, k_sr_out, k_rrdb_out) are compared bit for bit with their numpy float32 restatements.

Sizes (sr_kernel_refs.SIZES) cover every tile shape of pick_tile, each exact and partial, a map narrower than its
tile and one of more tiles than SMs.  Above LIMIT rows (columns) only a sample is recomputed: both borders, tile
boundaries and evenly spread pixels."""
import ctypes as C

import numpy as np
import pytest

from tests import sr_kernel_refs as K
from visiondepth3d_b200 import merged_pipeline as MP
from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu

LIMIT = 64


def report(what, err, bound):
    """worst observed error as a fraction of its bound; fails above 1."""
    r = np.asarray(err, np.float64) / np.asarray(bound, np.float64)
    i = int(np.argmax(r))
    print(f"[sr-kernels] {what}: observed / bound = {r.flat[i]:.3f} (worst abs err {np.ravel(err)[i]:.3e})")
    assert np.isfinite(r.flat[i]) and r.flat[i] <= 1.0, (what, float(r.flat[i]))


def stored_f16(dev, ref, slack, what):
    """dev: the f16 values the device stored; ref: float64; slack: bound on the error before the store."""
    report(what, np.abs(K.f64(dev) - ref), 0.5 * K.f16_ulp(np.abs(ref) + slack) + slack)


def stored_f32(dev, ref, slack, what):
    report(what, np.abs(K.f64(dev) - ref), slack + 2.0 ** -126)


def exact(dev, ref, what):
    d = np.abs(dev.astype(np.int64) - ref.astype(np.int64))
    print(f"[sr-kernels] {what}: bytes differing {int((d > 0).sum())} of {d.size}")
    assert dev.shape == ref.shape and not d.any(), (what, int(d.max()))


def lrelu_stores(ref, bound, n):
    """ref and bound after n identity convs with LeakyReLU, each an f16 store: a positive value passes exactly, a
    negative one is scaled by 0.2 (its error too) and rounded again; near 0 either may happen."""
    for _ in range(n):
        neg = ref < -bound
        store = np.where(ref > bound, 0.0, 0.5 * K.f16_ulp(np.abs(ref) + bound))
        ref = K.lrelu(ref)
        bound = np.where(neg, 0.2, 1.0) * bound + store + K.F32_EPS * np.abs(ref)
    return ref, bound


class Net:
    """One SR engine loaded with stress weights through the engine's own loader."""

    def __init__(self, sd):
        self.sd = sd
        self.e = MP.SrEngine(sd)
        self.e.lib.vd3d_depth_get_buffer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t]
        self.e.lib.vd3d_depth_get_buffer.restype = C.c_int

    def buf(self, name, shape, dtype=np.float16):
        out = np.empty(shape, dtype)
        self.e.check(self.e.lib.vd3d_depth_get_buffer(self.e.h, name.encode(), out.ctypes.data, out.nbytes))
        return out

    def w(self, name):
        return K.pack3x3(self.sd[name + ".weight"]), self.sd[name + ".bias"]

    def close(self):
        self.e.close()


_nets = {}


def net(kind, *args):
    if (kind,) + args not in _nets:
        if kind == "srvgg":
            _nets[(kind,) + args] = Net(K.stress_srvgg_state_dict(*args, seed=args[0]))
        else:
            nb, scale = args
            sd = K.stress_rrdb_state_dict(nb, scale, seed=10 * nb + scale)
            if nb > 1:
                # the last block's first RDB adds nothing (zero conv5): its output in rr.d1 is then that block's input
                # exactly, the residual the third RDB adds in place over the buffer holding it
                sd[f"body.{nb - 1}.rdb1.conv5.weight"] = np.zeros_like(sd[f"body.{nb - 1}.rdb1.conv5.weight"])
                sd[f"body.{nb - 1}.rdb1.conv5.bias"] = np.zeros_like(sd[f"body.{nb - 1}.rdb1.conv5.bias"])
            _nets[(kind,) + args] = Net(sd)
    return _nets[(kind,) + args]


@pytest.fixture(scope="module", autouse=True)
def _close_nets():
    yield
    for n in _nets.values():
        n.close()
    _nets.clear()


def tiles(w, h):
    tw, th, ex, n = K.tile_case(w, h)
    return f"{w}x{h} on {tw}x{th} tiles ({'exact' if ex else 'partial'}, {n} tiles)"


def grid(w, h):
    tw, th = K.pick_tile(w, h)
    return K.sample(h, th, LIMIT), K.sample(w, tw, LIMIT)


def conv_check(x, wb, rows, cols, cin_k):
    """float64 conv of the stored input at rows x cols and its accumulation slack (K = 9 * cin_k on the device)."""
    y = K.conv3x3_at(x, wb[0], wb[1], rows, cols)
    return y, K.ACC(9 * cin_k) * K.conv3x3_at_abs(x, wb[0], wb[1], rows, cols)


def sub(a, rows, cols):
    return a[rows][:, cols]


# ---------------------------------------------------------------------------------------------------------------------
# SRVGGNetCompact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", K.SIZES)
@pytest.mark.parametrize("num_conv", [1, 2])
def test_srvgg_kernels(num_conv, w, h):
    """The last PReLU conv (stress slopes), the f32 last conv on all 48 columns (its second BN = 32 tile holds 16),
    and k_sr_out bit for bit.  Conv i writes sr.x1 when i is even and sr.x0 when it is odd (num_conv 1 and 2: both)."""
    n = net("srvgg", num_conv)
    fr = synth_frame(30 + num_conv, w, h, "natural")[0]
    out = n.e.upscale(fr)
    print(f"\nSRVGG num_conv={num_conv}: {tiles(w, h)}")
    rows, cols = grid(w, h)
    i = num_conv
    src, dst = ("sr.x0", "sr.x1") if i % 2 == 0 else ("sr.x1", "sr.x0")
    x = n.buf(src, (h, w, 64))
    y, s = conv_check(x, n.w(f"body.{2 * i}"), rows, cols, 64)
    a = n.sd[f"body.{2 * i + 1}.weight"]
    stored_f16(sub(n.buf(dst, (h, w, 64)), rows, cols), K.prelu(y, a), np.maximum(1.0, np.abs(a)) * s,
               f"SRVGG nc={num_conv} {w}x{h} conv{i} + PReLU ({src} -> {dst})")
    last = n.buf(dst, (h, w, 64))
    cv = n.buf("sr.cv", (h, w, 48), np.float32)
    y, s = conv_check(last, n.w(f"body.{2 * (i + 1)}"), rows, cols, 64)
    got = sub(cv, rows, cols)
    stored_f32(got[..., :32], y[..., :32], s[..., :32], f"SRVGG nc={num_conv} {w}x{h} last conv columns 0-31")
    stored_f32(got[..., 32:], y[..., 32:], s[..., 32:], f"SRVGG nc={num_conv} {w}x{h} last conv columns 32-47")
    assert np.array_equal(n.buf("sr.in", (h, w, 3), np.uint8), fr)
    ref = K.sr_out(cv, fr)
    exact(n.buf("sr.outu8", (4 * h, 4 * w, 3), np.uint8), ref, f"SRVGG nc={num_conv} {w}x{h} k_sr_out")
    assert np.array_equal(out, ref)
    assert 0.1 < ((ref > 0) & (ref < 255)).mean()


# ---------------------------------------------------------------------------------------------------------------------
# RRDBNet
# ---------------------------------------------------------------------------------------------------------------------
def _hr_names(scale):
    """(buffer holding conv_hr's output, buffer holding conv_last's f32 output)"""
    return ("rr.u0", "rr.u1") if scale == 2 else ("rr.u1", "rr.u0")


@pytest.mark.parametrize("w,h", K.SIZES)
@pytest.mark.parametrize("scale,nb", [(4, 1), (2, 1), (4, 2), (2, 2)])
def test_rrdb_kernels(scale, nb, w, h):
    """One forward: k_sr_in, conv_first, every conv of the last RRDB's second and third dense blocks, the in-place
    RRDB residual, the zero padding channels of the growth slices, conv_body (rs = 1), conv_last (f32, columns 3-31
    exactly zero) and k_rrdb_out.  The first dense block's convs are not checked: their input (channels 0..63 of
    rr.d0) is overwritten in place by the RRDB output."""
    n = net("rrdb", nb, scale)
    fr = synth_frame(40 + nb, w, h, "natural")[0]
    out = n.e.upscale(fr)
    H, W = scale * h, scale * w
    print(f"\nRRDB x{scale} nb={nb}: {tiles(w, h)}; conv_hr / conv_last: {tiles(W, H)}")
    rows, cols = grid(w, h)
    tag = f"RRDB x{scale} nb={nb} {w}x{h}"
    x0 = n.buf("rr.x0", (h, w, 64))
    exact(x0.view(np.uint16), K.sr_in(fr).view(np.uint16), f"{tag} k_sr_in")
    feat = n.buf("rr.feat", (h, w, 64))
    y, s = conv_check(x0[..., :3], n.w("conv_first"), rows, cols, 64)
    stored_f16(sub(feat, rows, cols), y, s, f"{tag} conv_first")
    d = [n.buf(f"rr.d{i}", (h, w, 320)) for i in range(3)]
    for i in range(3):
        for k in range(1, 5):
            assert not d[i][..., 64 * k + 32:64 * (k + 1)].any(), ("padding channels written", i, k)
    b = nb - 1
    rin = feat if nb == 1 else d[1][..., :64]
    for j in (1, 2):
        X = d[j]
        for k in range(1, 6):
            y, s = conv_check(X[..., K.dense_cols(k)], n.w(f"body.{b}.rdb{j + 1}.conv{k}"), rows, cols, 64 * k)
            what = f"{tag} rdb{j + 1}.conv{k}"
            if k < 5:
                stored_f16(sub(X, rows, cols)[..., 64 * k:64 * k + 32], K.lrelu(y), s, what + " + LeakyReLU")
                continue
            xs = sub(X[..., :64], rows, cols)
            if j == 1:
                ref = K.sr_residual(y, xs, 0.2)
                slack = 0.2 * s + 4 * K.F32_EPS * (np.abs(K.f64(xs)) + 0.2 * s)
                stored_f16(sub(d[2][..., :64], rows, cols), ref, slack, what + ": x + 0.2 x5")
            else:
                rs = sub(rin, rows, cols)
                ref = K.sr_residual(y, xs, 0.2, rs, 0.2)
                slack = 0.04 * s + 4 * K.F32_EPS * (np.abs(K.f64(rs)) + 0.2 * np.abs(K.f64(xs)) + 0.04 * s)
                stored_f16(sub(d[0][..., :64], rows, cols), ref, slack, what + ": RRDB in + 0.2 (x + 0.2 x5), in place")
    body = n.buf("rr.body", (h, w, 64))
    y, s = conv_check(d[0][..., :64], n.w("conv_body"), rows, cols, 64)
    fs = sub(feat, rows, cols)
    stored_f16(sub(body, rows, cols), K.sr_residual(y, fs, 1.0), s + 4 * K.F32_EPS * (np.abs(K.f64(fs)) + s),
               f"{tag} conv_body + trunk")
    hr_name, last_name = _hr_names(scale)
    hr = n.buf(hr_name, (H, W, 64))
    last = n.buf(last_name, (H, W, 32), np.float32)
    R, Cc = grid(W, H)
    y, s = conv_check(hr, n.w("conv_last"), R, Cc, 64)
    stored_f32(sub(last, R, Cc)[..., :3], y, s, f"{tag} conv_last (f32, at {W}x{H})")
    assert not last[..., 3:].any(), "conv_last columns 3..31 must be exactly zero"
    ref = K.rrdb_out(last)
    exact(n.buf("sr.outu8", (H, W, 3), np.uint8), ref, f"{tag} k_rrdb_out")
    assert np.array_equal(out, ref) and 0.5 < ((ref > 0) & (ref < 255)).mean()


def _with_identity(n, convs):
    """the engine tensors of the named convs replaced by identity convs, packed by the engine's own packer;
    returns the original tensors for _restore."""
    sd = dict(n.sd)
    for c in convs:
        sd[c + ".weight"], sd[c + ".bias"] = K.identity_conv()
    names = {"conv_up1": "rr.up1", "conv_up2": "rr.up2", "conv_hr": "rr.hr"}
    _, _, new = MP.pack_rrdb(sd)
    _, _, old = MP.pack_rrdb(n.sd)
    keep = {}
    for c in convs:
        for s in (".w", ".b"):
            keep[names[c] + s] = old[names[c] + s]
            n.e._set(names[c] + s, new[names[c] + s])
    return keep


def _restore(n, keep):
    for name, arr in keep.items():
        n.e._set(name, arr)


def _phase(n, u):
    _, _, t = MP.pack_rrdb(n.sd)
    return t[f"rr.up{u}.w"], t[f"rr.up{u}.b"]


def _up_rows(rows):
    """output rows (columns) of a nearest x2 + conv computed at low-resolution rows: 2 r and 2 r + 1"""
    return np.stack([2 * rows, 2 * rows + 1], 1).ravel()


@pytest.mark.parametrize("w,h", K.SIZES)
@pytest.mark.parametrize("scale", [4, 2])
def test_rrdb_upsampling_convs(scale, w, h):
    """The up-convs (nearest x2 + conv as four phase convs on the engine's packed [256, 576] weights, pixel-shuffle
    scatter) and conv_hr, whose inputs and outputs later convs overwrite: the convs around the one checked are made
    identities (1.0 centre tap, zero bias), so that the retained conv_hr output is the checked conv's output passed
    through LeakyReLU f16 stores, or the checked conv's input is a LeakyReLU chain of rr.body numpy reproduces."""
    n = net("rrdb", 1, scale)
    fr = synth_frame(50, w, h, "natural")[0]
    H, W = scale * h, scale * w
    hr_name = _hr_names(scale)[0]
    tag = f"RRDB x{scale} {w}x{h}"
    print(f"\n{tag}: up1 at {tiles(w, h)}" + (f"; up2 at {tiles(2 * w, 2 * h)}" if scale == 4 else "")
          + f"; conv_hr at {tiles(W, H)}")
    ups = ["conv_up1", "conv_up2"][:scale // 2]
    # conv_hr: every up-conv the identity
    keep = _with_identity(n, ups)
    try:
        n.e.upscale(fr)
        x = n.buf("rr.body", (h, w, 64))
        for _ in ups:
            x = K.lrelu_f16(K.nearest2(x))
        R, Cc = grid(W, H)
        y, s = conv_check(x, n.w("conv_hr"), R, Cc, 64)
        stored_f16(sub(n.buf(hr_name, (H, W, 64)), R, Cc), K.lrelu(y), s, f"{tag} conv_hr + LeakyReLU")
    finally:
        _restore(n, keep)
    # each up-conv: the other one and conv_hr the identity
    for u in range(1, len(ups) + 1):
        keep = _with_identity(n, [c for c in ups if c != f"conv_up{u}"] + ["conv_hr"])
        try:
            n.e.upscale(fr)
            x = n.buf("rr.body", (h, w, 64))
            lh, lw = h, w
            if u == 2:
                x, lh, lw = K.lrelu_f16(K.nearest2(x)), 2 * h, 2 * w
            rows, cols = grid(lw, lh)
            wp, bp = _phase(n, u)
            y = K.phase_conv(x, wp, bp, rows, cols)
            s = K.ACC(576) * K.phase_conv(np.abs(K.f64(x)), np.abs(K.f64(wp)), np.abs(bp), rows, cols)
            ref = K.lrelu(y)
            bound = 0.5 * K.f16_ulp(np.abs(ref) + s) + s
            ur, uc = _up_rows(rows), _up_rows(cols)
            after = len(ups) - u + 1   # identity LeakyReLU stores between this conv and conv_hr's output
            ref, bound = lrelu_stores(ref, bound, after)
            if u == 1 and scale == 4:   # the identity up2 repeats each pixel 2 x 2
                ur, uc = 2 * ur, 2 * uc
            dev = sub(n.buf(hr_name, (H, W, 64)), ur, uc)
            report(f"{tag} conv_up{u} + LeakyReLU, scattered (then {after} identity LeakyReLU stores)",
                   np.abs(K.f64(dev) - ref), bound)
        finally:
            _restore(n, keep)
