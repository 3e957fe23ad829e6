"""CPU: the restatements of tests/sr_kernel_refs.py against torch ops, oracle/sr.py::srvgg_forward and
tests/rrdb_oracle.py::rrdb_forward, the byte kernels' restatements against preprocess_esr / postprocess_esr, and the
list of GPU check sizes against every conv tile case."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sr as S
from tests import depth_kernel_refs as DR
from tests import rrdb_oracle as RO
from tests import sr_kernel_refs as K
from visiondepth3d_b200 import merged_pipeline as MP
from visiondepth3d_b200.synth import synth_frame


def nchw(x):
    return torch.from_numpy(np.ascontiguousarray(K.f64(x).transpose(2, 0, 1)))[None]


def nhwc(t):
    return t[0].permute(1, 2, 0).numpy()


def test_conv_at_selected_pixels_matches_torch():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((13, 17, 8))
    w = rng.standard_normal((5, 8, 3, 3))
    b = rng.standard_normal(5)
    ref = nhwc(F.conv2d(nchw(x), torch.from_numpy(w), torch.from_numpy(b), padding=1))
    assert np.allclose(K.conv3x3_at(x, K.pack3x3(w), b), ref, rtol=0, atol=1e-12)
    assert np.allclose(K.conv3x3_at(x, K.pack3x3(w), b), DR.conv3x3(x, K.pack3x3(w), b), rtol=0, atol=1e-12)
    rows, cols = np.array([0, 1, 6, 11, 12]), np.array([0, 7, 15, 16])
    assert np.allclose(K.conv3x3_at(x, K.pack3x3(w), b, rows, cols), ref[rows][:, cols], rtol=0, atol=1e-12)
    assert np.allclose(K.conv3x3_at_abs(x, K.pack3x3(w), b, rows, cols),
                       DR.conv3x3_abs(x, K.pack3x3(w), b)[rows][:, cols], rtol=0, atol=1e-12)
    s = K.sample(180, 2, 24)
    assert s[0] == 0 and s[-1] == 179 and {1, 178, 1, 2, 3, 4}.issubset(set(s)) and len(s) <= 48
    assert np.array_equal(K.sample(20, 8, 24), np.arange(20))


def test_activations_and_residual_match_torch():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((6, 7, 64)) * 2
    a = K.stress_slopes(rng)
    assert np.array_equal(K.prelu(x, a), nhwc(F.prelu(nchw(x), torch.from_numpy(K.f64(a)))))
    assert np.array_equal(K.lrelu(x), nhwc(F.leaky_relu(nchw(x), 0.2)))
    r1, r2 = rng.standard_normal(x.shape), rng.standard_normal(x.shape)
    assert np.allclose(K.sr_residual(x, r1, 0.2, r2, 0.2), r2 + 0.2 * (r1 + 0.2 * x), rtol=0, atol=1e-14)
    assert np.allclose(K.sr_residual(x, r1, 1.0), r1 + x, rtol=0, atol=1e-14)
    assert np.array_equal(K.sr_residual(x), x)
    # the f16 identity-conv LeakyReLU: fp32 0.2f * x, one rounding to f16
    h = (rng.standard_normal(4096) * 3).astype(np.float16)
    exp = np.where(h > 0, h, (np.float32(0.2) * h.astype(np.float32))).astype(np.float16)
    assert np.array_equal(K.lrelu_f16(h), exp)
    assert np.array_equal(K.nearest2(x), nhwc(F.interpolate(nchw(x), scale_factor=2, mode="nearest")))


def test_phase_conv_equals_nearest_x2_and_conv():
    """phase_conv with unrounded combined weights is nearest x2 + conv; phase_weights is the engine's packing; with the
    combined weights rounded to f16 (what the engine stores) the error stays within 2^-11 of sum |x| |w_combined|, and
    weights whose combined sums are exact in f16 give the same result exactly."""
    rng = np.random.default_rng(2)
    x = rng.standard_normal((7, 9, 64))
    w = K._f16(rng.standard_normal((64, 64, 3, 3)) / 24)
    b = rng.standard_normal(64)
    ref = nhwc(F.conv2d(F.interpolate(nchw(x), scale_factor=2, mode="nearest"), torch.from_numpy(K.f64(w)),
                        torch.from_numpy(b), padding=1))
    wc = K.phase_weights(w)
    assert np.allclose(K.phase_conv(x, wc, np.tile(b, 4)), ref, rtol=0, atol=1e-11)
    packed = MP._pack3x3(MP._phase_weights(w), list(range(64)), 64)
    assert np.array_equal(packed, wc.astype(np.float16))
    got = K.phase_conv(x, packed, np.tile(b, 4))
    slack = K.F16_EPS * K.phase_conv(np.abs(x), np.abs(wc))
    err = np.abs(got - ref)
    assert (err <= slack).all() and err.max() > 0, float((err / slack).max())
    # rows / cols select low-resolution pixels, scattered to their four phases
    rows, cols = np.array([0, 3, 6]), np.array([0, 8])
    sub = K.phase_conv(x, packed, np.tile(b, 4), rows, cols)
    full_rows = np.stack([2 * rows, 2 * rows + 1], 1).ravel()
    full_cols = np.stack([2 * cols, 2 * cols + 1], 1).ravel()
    assert np.allclose(sub, got[full_rows][:, full_cols], rtol=0, atol=1e-12)
    wq = np.round(rng.standard_normal((64, 64, 3, 3)) * 8) / 64
    refq = nhwc(F.conv2d(F.interpolate(nchw(x), scale_factor=2, mode="nearest"), torch.from_numpy(wq), padding=1))
    pq = MP._pack3x3(MP._phase_weights(wq.astype(np.float32)), list(range(64)), 64)
    assert np.allclose(K.phase_conv(x, pq), refq, rtol=0, atol=1e-11)


def test_byte_kernels_match_the_pre_and_post_processing():
    fr = synth_frame(3, 37, 21, "natural")[0]
    x = S.preprocess_esr(fr)
    xi = K.sr_in(fr)
    assert xi.dtype == np.float16 and xi.shape == (21, 37, 64) and not xi[..., 3:].any()
    assert np.array_equal(xi[..., :3], x[0].transpose(1, 2, 0).astype(np.float16))
    rng = np.random.default_rng(3)
    cv = (rng.standard_normal((21, 37, 48)) * 0.4).astype(np.float32)
    t = F.pixel_shuffle(torch.from_numpy(cv.transpose(2, 0, 1).copy())[None], 4)
    t = t + F.interpolate(torch.from_numpy(x), scale_factor=4, mode="nearest")
    ref = S.postprocess_esr(t.numpy())
    got = K.sr_out(cv, fr)
    assert np.array_equal(got, ref)
    assert 0.2 < ((got > 0) & (got < 255)).mean() and 0.05 < (got == 0).mean() + (got == 255).mean()
    rgb = (rng.standard_normal((84, 148, 32)) * 0.6 + 0.5).astype(np.float32)
    assert np.array_equal(K.rrdb_out(rgb), S.postprocess_esr(rgb[..., :3].transpose(2, 0, 1)[None]))


@pytest.mark.parametrize("num_conv", [1, 2])
def test_srvgg_composed_matches_the_oracle(num_conv):
    sd = K.stress_srvgg_state_dict(num_conv, seed=4)
    fr = synth_frame(4, 23, 17, "natural")[0]
    x = S.preprocess_esr(fr)
    with torch.no_grad():
        ref = S.srvgg_forward({k: torch.from_numpy(v) for k, v in sd.items()}, torch.from_numpy(x))[0]
    t = x[0].transpose(1, 2, 0)
    n = num_conv + 2
    for i in range(n):
        t = K.conv3x3_at(t, K.pack3x3(sd[f"body.{2 * i}.weight"]), sd[f"body.{2 * i}.bias"])
        if i < n - 1:
            t = K.prelu(t, sd[f"body.{2 * i + 1}.weight"])
    ps = F.pixel_shuffle(torch.from_numpy(t.transpose(2, 0, 1).copy())[None], 4)[0].numpy()
    got = ps + np.repeat(np.repeat(x[0], 4, 1), 4, 2)
    scale = float(np.abs(ref.numpy()).max())
    assert np.abs(got - ref.numpy()).max() <= 1e-5 * scale
    assert np.abs(t).max() > 1.0 and (t < 0).mean() > 0.2   # the last conv is not scaled down


@pytest.mark.parametrize("scale,nb", [(4, 1), (2, 2)])
def test_rrdb_composed_matches_the_oracle(scale, nb):
    """conv_first, the dense blocks on the engine's [.., 320] buffer layout, the RRDB residual in one epilogue,
    conv_body with its trunk residual, the up-convs as phase convs, conv_hr and conv_last against rrdb_forward."""
    sd = K.stress_rrdb_state_dict(nb, scale, seed=5)
    fr = synth_frame(5, 19, 13, "natural")[0]
    x = S.preprocess_esr(fr)
    with torch.no_grad():
        ref = RO.rrdb_forward(sd, torch.from_numpy(x))[0].permute(1, 2, 0).numpy()
    cv = lambda t, n, **kw: K.conv3x3_at(t, K.pack3x3(sd[n + ".weight"]), sd[n + ".bias"], **kw)
    h, w = fr.shape[:2]
    feat = cv(x[0].transpose(1, 2, 0), "conv_first")
    t = feat
    for i in range(nb):
        rin = t
        for j in range(1, 4):
            d = np.zeros((h, w, 320))
            d[..., :64] = t
            for k in range(1, 5):
                d[..., 64 * k:64 * k + 32] = K.lrelu(cv(d[..., K.dense_cols(k)], f"body.{i}.rdb{j}.conv{k}"))
            x5 = cv(d[..., K.dense_cols(5)], f"body.{i}.rdb{j}.conv5")
            t = K.sr_residual(x5, t, 0.2, rin, 0.2) if j == 3 else K.sr_residual(x5, t, 0.2)
    t = K.sr_residual(cv(t, "conv_body"), feat, 1.0)
    for u in range(1, 2 if scale == 2 else 3):
        t = K.lrelu(K.phase_conv(t, K.phase_weights(sd[f"conv_up{u}.weight"]), np.tile(sd[f"conv_up{u}.bias"], 4)))
    got = cv(K.lrelu(cv(t, "conv_hr")), "conv_last")
    assert got.shape == ref.shape == (scale * h, scale * w, 3)
    assert np.abs(got - ref).max() <= 1e-4 * float(np.abs(ref).max())
    assert ref.std() > 0.1 and ((ref > 0) & (ref < 1)).mean() > 0.5


def test_stress_weights_and_their_packing():
    rng = np.random.default_rng(6)
    a = K.stress_slopes(rng)
    assert len(np.unique(a)) == 64 and (a == 0).sum() == 1 and a.min() <= -0.45 and a.max() >= 1.45
    sd = K.stress_srvgg_state_dict(2, seed=0)
    for i in range(4):
        b = sd[f"body.{2 * i}.bias"]
        assert len(np.unique(b)) == len(b) and np.abs(b).max() >= 0.45
        assert np.array_equal(sd[f"body.{2 * i}.weight"].astype(np.float16).astype(np.float32), sd[f"body.{2 * i}.weight"])
    # the last conv at the scale of the others (not scaled by 0.1)
    assert sd["body.6.weight"].std() > 0.5 * sd["body.4.weight"].std()
    rr = K.stress_rrdb_state_dict(2, 4, seed=0)
    nb, scale, t = MP.pack_rrdb(rr)
    assert (nb, scale) == (2, 4)
    assert np.array_equal(t["rr.1.2.3.w"].astype(np.float64)[:, :9 * 192].reshape(32, 9, 192)[:, :, K.dense_cols(3)],
                          K.pack3x3(rr["body.1.rdb3.conv3.weight"]).reshape(32, 9, 128))
    assert np.array_equal(t["rr.up2.w"], K.phase_weights(rr["conv_up2.weight"]).astype(np.float16))
    assert not t["rr.last.w"][3:].any() and not t["rr.last.b"][3:].any()
    wi, bi = K.identity_conv()
    x = rng.standard_normal((5, 6, 64))
    assert np.array_equal(K.conv3x3_at(x, K.pack3x3(wi), bi), x)
    assert np.array_equal(K.phase_conv(x, MP._pack3x3(MP._phase_weights(wi), list(range(64)), 64)), K.nearest2(x))


def test_pick_tile_and_the_sizes_cover_every_case():
    """The restated pick_tile on its defining cases, and SIZES: every tile shape exact and partial, a map narrower
    than its tile (8 x 8 on 16 x 8), and a map of more tiles than SMs (persistent CTAs wrap)."""
    assert K.pick_tile(128, 8) == (128, 1) and K.pick_tile(64, 48) == (64, 2)
    assert K.pick_tile(32, 12) == (32, 4) and K.pick_tile(48, 16) == (16, 8)
    assert K.pick_tile(8, 8) == (16, 8) and K.pick_tile(320, 180) == (64, 2)
    cases = {K.tile_case(w, h)[:3] for w, h in K.SIZES}
    for tile in K.TILES:
        assert tile + (True,) in cases and tile + (False,) in cases, tile
    assert any(K.tile_case(w, h)[0] > w for w, h in K.SIZES)
    assert any(K.tile_case(w, h)[3] > K.NUM_SMS for w, h in K.SIZES)
    assert min(min(w, h) for w, h in K.SIZES) == 8
