"""CPU: loading and packing of the RRDBNet upscalers (RealESRGAN_x4plus, BSRGAN x4 / x2) in both key namings, the
random init the GPU tests run on, the f16 budget of the CPU restatement (tests/rrdb_oracle.py) that the GPU gates rest
on, and run_esrgan's model-name quirk for every (network scale, name) pair."""
import numpy as np
import pytest
import torch

from oracle.sr import preprocess_esr
from tests import rrdb_oracle as RO
from visiondepth3d_b200 import merged_pipeline as MP
from visiondepth3d_b200.synth import synth_frame


def _save(sd, path, wrap):
    t = {k: torch.from_numpy(v) for k, v in sd.items()}
    torch.save({wrap: t} if wrap else t, path)


@pytest.mark.parametrize("scale", [4, 2])
def test_namings_and_wrappers_load_to_the_same_packed_tensors(tmp_path, scale):
    ref = MP.pack_rrdb(MP.random_rrdb_state_dict(2, scale, seed=3))
    assert ref[:2] == (2, scale)
    for naming in ("basicsr", "esrgan"):
        sd = MP.random_rrdb_state_dict(2, scale, seed=3, naming=naming)
        assert ("RRDB_trunk.1.RDB3.conv5.weight" in sd) == (naming == "esrgan")
        for wrap in (None, "params_ema", "params"):
            p = str(tmp_path / f"{naming}_{wrap}.pth")
            _save(sd, p, wrap)
            nb, s, t = MP.pack_rrdb(MP._read_state_dict(p))
            assert (nb, s) == (2, scale) and sorted(t) == sorted(ref[2])
            assert all(t[k].dtype == ref[2][k].dtype and np.array_equal(t[k], ref[2][k]) for k in t), (naming, wrap)
    assert ("rr.up2.w" in ref[2]) == (scale == 4)


def test_packed_layouts():
    sd = MP.random_rrdb_state_dict(1, 4, seed=5)
    _, _, t = MP.pack_rrdb(sd)
    w = sd["body.0.rdb2.conv3.weight"]                      # [32, 128, 3, 3]: x (64) + x1 (32) + x2 (32)
    p = t["rr.0.1.3.w"].astype(np.float32).reshape(32, 9, 192)
    assert t["rr.0.1.3.w"].shape == (32, 9 * 192)
    taps = w.transpose(0, 2, 3, 1).reshape(32, 9, 128).astype(np.float16).astype(np.float32)
    assert np.array_equal(p[:, :, :64], taps[:, :, :64])
    assert np.array_equal(p[:, :, 64:96], taps[:, :, 64:96]) and np.array_equal(p[:, :, 128:160], taps[:, :, 96:128])
    assert not p[:, :, 96:128].any() and not p[:, :, 160:].any()  # the padding columns of each growth slice
    assert t["rr.last.w"].shape == (32, 576) and not t["rr.last.w"][3:].any() and not t["rr.last.b"][3:].any()
    assert t["rr.up1.w"].shape == (256, 576) and np.array_equal(t["rr.up1.b"], np.tile(sd["conv_up1.bias"], 4))
    assert t["rr.first.w"].shape == (64, 576) and not t["rr.first.w"].reshape(64, 9, 64)[:, :, 3:].any()


def test_phase_weights_equal_nearest_upsample_then_conv():
    import torch.nn.functional as F
    rng = np.random.default_rng(0)
    w = rng.standard_normal((8, 5, 3, 3)).astype(np.float32)
    x = torch.from_numpy(rng.standard_normal((1, 5, 7, 6)).astype(np.float32)).double()
    ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), torch.from_numpy(w).double(), padding=1)
    ph = F.conv2d(x, torch.from_numpy(MP._phase_weights(w)).double(), padding=1)   # [1, 4 * 8, 7, 6]
    got = ph.reshape(1, 2, 2, 8, 7, 6).permute(0, 3, 4, 1, 5, 2).reshape(1, 8, 14, 12)
    assert torch.allclose(got, ref, rtol=0, atol=1e-5)  # the phase weights are float32 sums


def test_nb_and_scale_detected():
    for nb, scale in ((1, 2), (3, 4), (23, 2)):
        for naming in ("basicsr", "esrgan"):
            _, n, s = MP.rrdb_layout(MP.random_rrdb_state_dict(nb, scale, seed=0, naming=naming))
            assert (n, s) == (nb, scale)
            assert RO.net_scale(MP.random_rrdb_state_dict(1, scale, naming=naming)) == scale


def test_bad_dicts_raise(tmp_path):
    good = MP.random_rrdb_state_dict(2, 4, seed=1)
    bad = []
    d = dict(good)
    d["conv_first.weight"] = np.zeros((64, 12, 3, 3), np.float32)  # basicsr x2: pixel-unshuffle in front
    bad.append((d, "input channels"))
    d = dict(good)
    d["conv_first.weight"] = np.zeros((64, 48, 3, 3), np.float32)  # basicsr x1
    bad.append((d, "input channels"))
    d = dict(good)
    del d["body.1.rdb2.conv4.bias"]
    bad.append((d, "RRDBNet"))
    d = dict(good)
    d["body.0.rdb1.conv2.weight"] = np.zeros((32, 64, 3, 3), np.float32)  # not a dense block
    bad.append((d, "RRDBNet"))
    d = dict(good)
    d["conv_last.weight"] = np.zeros((4, 64, 3, 3), np.float32)
    bad.append((d, "RRDBNet"))
    d = {k: v for k, v in good.items() if not k.startswith("body.")}
    bad.append((d, "RRDBNet"))
    d = dict(good)
    d["extra.weight"] = np.zeros(3, np.float32)
    bad.append((d, "RRDBNet"))
    d = dict(good)
    nf = 32  # num_feat 32
    d["conv_first.weight"] = np.zeros((nf, 3, 3, 3), np.float32)
    bad.append((d, "RRDBNet"))
    bad.append(({"conv_first.bias": np.zeros(64, np.float32)}, "conv_first"))
    for i, (sd, msg) in enumerate(bad):
        with pytest.raises(ValueError, match=msg):
            MP.rrdb_layout(sd)
        p = str(tmp_path / f"bad{i}.pth")
        _save(sd, p, "params_ema")
        with pytest.raises(ValueError, match=msg):
            MP._read_state_dict(p)
    with pytest.raises(ValueError):
        MP.random_rrdb_state_dict(1, 4, naming="onnx")


def test_forward_is_the_same_on_both_namings():
    x = torch.from_numpy(preprocess_esr(synth_frame(2, 24, 20, "natural")[0]))
    for scale in (4, 2):
        a = RO.rrdb_forward(MP.random_rrdb_state_dict(2, scale, seed=4), x)
        b = RO.rrdb_forward(MP.random_rrdb_state_dict(2, scale, seed=4, naming="esrgan"), x)
        assert a.shape == (1, 3, 20 * scale, 24 * scale) and torch.equal(a, b)


def _u8(t):
    return RO.postprocess_esr(t.numpy())


# (scale, nb, w, h): the sizes of tests/test_rrdb_gpu.py::test_forward_matches_f16_oracle
SIZES = [(4, 23, 64, 48), (2, 23, 67, 45), (4, 2, 160, 90)]


@pytest.mark.parametrize("scale,nb,w,h", SIZES)
def test_f16_budget(scale, nb, w, h):
    """What f16 storage through the network costs at the GPU tests' sizes, and how much of the u8 output a different
    fp32 accumulation order alone moves.  The second number is the margin the GPU gate needs against
    rrdb_forward_f16: the tensor cores accumulate in another order than torch on the CPU, and every f16 rounding that
    this flips travels through the remaining convs.  Here float64 accumulation stands in for that other order: at these
    sizes it moves 1-2.5 % of the bytes by one LSB (never more), so the GPU gate is max 1 LSB on at most 5 % of the
    bytes, and 2e-3 on the float output."""
    sd = MP.random_rrdb_state_dict(nb, scale, seed=0)
    x = torch.from_numpy(preprocess_esr(synth_frame(3, w, h, "natural")[0]))
    f32 = RO.rrdb_forward(sd, x)
    f16 = RO.rrdb_forward_f16(sd, x)
    d = np.abs(_u8(f32).astype(int) - _u8(f16))
    assert d.max() <= 6 and d.mean() <= 0.5, (d.max(), d.mean())
    sd64 = {k: v.double() for k, v in RO._t(sd).items()}
    q = lambda t: t.to(torch.float16).to(torch.float64)
    f64 = RO._graph(sd64, x.double(), q, q).float()
    d2 = np.abs(_u8(f64).astype(int) - _u8(f16))
    assert d2.max() <= 1 and (d2 > 0).mean() <= 0.03, (d2.max(), (d2 > 0).mean())
    assert float((f64 - f16).abs().max()) <= 1e-3


@pytest.mark.parametrize("scale", [4, 2])
def test_random_init_is_not_degenerate(scale):
    """The output of a natural frame spreads over the u8 range with little clipping: a kernel that writes zeros, a
    constant or a saturated image cannot pass the GPU gates against it."""
    sd = MP.random_rrdb_state_dict(23, scale, seed=0)
    for seed, (w, h) in ((3, (64, 48)), (4, (67, 45))):
        out = RO.upscale(sd, synth_frame(seed, w, h, "natural")[0])
        assert out.shape == (scale * h, scale * w, 3)
        std = out.reshape(-1, 3).std(0)
        clipped = ((out == 0) | (out == 255)).mean()
        assert std.min() > 15 and clipped < 0.05, (std, clipped)


@pytest.mark.parametrize("name", ["RealESR_Gx4_fp16", "RealESRGAN_x4_fp16", "BSRGANx4_fp16", "BSRGANx2_fp16",
                                  "bsrganX2"])
@pytest.mark.parametrize("net", [4, 2])
def test_upscale_params_quirk_for_every_scale_and_name(name, net):
    """run_esrgan's second resize goes to scale x the network input with scale from the NAME, whatever the network
    produced: the parameters carry the name's scale, and the oracle chain's output size is the original size."""
    p = MP.upscale_params("OFF", 100, name)
    assert p.scale == (2 if "x2" in name.lower() else 4)
    seen = []

    def fake_net(f):
        seen.append(f.shape)
        return np.zeros((net * f.shape[0], net * f.shape[1], 3), np.uint8)

    fr = synth_frame(1, 20, 12, "natural")[0]
    out = RO.run_esrgan(None, fr, "OFF", 100, name, network=fake_net)
    assert out.shape == fr.shape and seen == [fr.shape]
