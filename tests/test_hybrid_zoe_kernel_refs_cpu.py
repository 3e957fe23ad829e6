"""CPU: the float64 restatements of tests/hybrid_zoe_kernel_refs.py, composed on the engine's packed tensors, equal the
torch oracles: the BiT backbone stage by stage (tests/dpt_hybrid_oracle.backbone) and ZoeDepth's metric head on both
routes and with one configuration (tests/zoedepth_oracle.metric_head).  So the GPU tests that compare kernels with
these functions do not restate a packing mistake of the engine (tap order, SAME pad side, the block-diagonal seed
conv2, the configurations' columns)."""
import numpy as np
import pytest
import torch

from tests import dpt_hybrid_oracle as OH
from tests import hybrid_zoe_kernel_refs as HZ
from tests import zoedepth_oracle as ZO


def _f16(t):
    """the rounding of depth_weights' f16 tensors and of the engine's f16 stores: through f32"""
    return t.to(torch.float32).to(torch.float16).to(t.dtype)


def test_same_im2col_pads_after_on_even_sides_and_both_on_odd():
    x = np.arange(5 * 4 * 1, dtype=np.float64).reshape(5, 4, 1) + 1
    cols = HZ.same_im2col_s2(x)          # 5 rows: pad 1 before, 1 after; 4 columns: 0 before, 1 after
    assert cols.shape == (3 * 2, 9)
    assert cols[0].tolist() == [0, 0, 0, 1, 2, 3, 5, 6, 7]
    assert cols[-1].tolist() == [15, 16, 0, 19, 20, 0, 0, 0, 0]
    torch_ref = torch.nn.functional.conv2d(torch.nn.functional.pad(torch.from_numpy(x).permute(2, 0, 1)[None],
                                                                   (0, 1, 1, 1)),
                                           torch.ones(1, 1, 3, 3, dtype=torch.float64), stride=2)
    assert np.array_equal(cols.sum(1), torch_ref.reshape(-1).numpy())


@pytest.fixture(scope="module")
def hybrid():
    from visiondepth3d_b200.depth_weights import prepare_dpt_hybrid
    sd, cfg = OH.random_model(small=True)
    S = cfg["image_size"]
    return sd, cfg, prepare_dpt_hybrid(sd, cfg, S, S)


def test_bit_stages_equal_the_oracle_backbone(hybrid):
    """From the oracle's max-pool output, bit_stages on prepare_dpt_hybrid's tensors (f16 weights, f16 activations
    where the engine stores them) equals the oracle's backbone run with the same roundings, stage by stage."""
    sd, cfg, P = hybrid
    S = cfg["image_size"]
    sd64 = {k: v.double() for k, v in sd.items()}
    px = torch.randn(3, S, S, generator=torch.Generator().manual_seed(1), dtype=torch.float64)[None]
    with torch.no_grad():
        stages, parts = OH.backbone(sd64, px, q=_f16, return_parts=True)
    pool = parts["pool"][0].permute(1, 2, 0).numpy()
    got = HZ.bit_stages(P, pool, rnd=lambda a: a.astype(np.float32).astype(np.float16).astype(np.float64))
    for i, (g, r) in enumerate(zip(got, stages)):
        r = r[0].permute(1, 2, 0).numpy()
        assert g.shape == r.shape, i
        err = float(np.abs(g - r).max() / np.abs(r).max())
        share = float((g != r).mean())
        print(f"stage {i + 1}: max |restated - oracle| / max {err:.2e}, share of elements that differ {share:.2e}")
        # summation order flips an f16 rounding now and then; a packing or padding slip moves whole rows by O(1)
        assert err <= 2e-3 and share <= 1e-3, (i, err, share)


def test_bit_conv_kinds_equal_torch_same_convs():
    """Each kind on the weight packing of prepare_dpt_hybrid against dpt_hybrid_oracle.conv_same (SAME pads)."""
    from visiondepth3d_b200.depth_weights import _conv3
    rng = np.random.default_rng(0)
    for H, W in ((8, 6), (7, 5)):
        x = rng.standard_normal((H, W, 64))
        xt = torch.from_numpy(x).permute(2, 0, 1)[None]
        for kind, k, s in ((HZ.BIT_1X1, 1, 1), (HZ.BIT_3X3, 3, 1), (HZ.BIT_3X3_S2, 3, 2), (HZ.BIT_1X1_S2, 1, 2)):
            w = torch.from_numpy(rng.standard_normal((64, 64, k, k)))
            packed = (_conv3(w, 64) if k == 3 else w.reshape(64, 64).numpy()).astype(np.float64)
            wq = torch.from_numpy(packed.reshape(64, k, k, 64)).permute(0, 3, 1, 2) if k == 3 else \
                torch.from_numpy(packed).reshape(64, 64, 1, 1)
            ref = OH.conv_same(xt, wq, s, ws=False)[0].permute(1, 2, 0).reshape(-1, 64).numpy()
            got = HZ.bit_conv(x, packed, kind)
            assert got.shape == ref.shape and np.allclose(got, ref, rtol=1e-12, atol=1e-10), (H, W, kind)


@pytest.fixture(scope="module")
def zoe_models():
    return {True: ZO.random_model(multi=True, seed=3), False: ZO.random_model(multi=False, seed=4)}


@pytest.mark.parametrize("multi,route", [(True, 0), (True, 1), (False, 0)])
def test_metric_head_equals_the_oracle(zoe_models, multi, route):
    """metric_head composed on prepare_zoedepth's z.* tensors (f16 weights rounded as the engine holds them, given to
    the oracle too) against zoedepth_oracle.metric_head with the route forced, in float64."""
    from visiondepth3d_b200.depth_weights import prepare_zoedepth, zoedepth_attractors
    sd, cfg = zoe_models[multi]
    sd = {k: (_f16(v) if k.startswith(ZO.M) and v.is_floating_point() else v) for k, v in sd.items()}
    H, W = 64, 96
    P = prepare_zoedepth(sd, cfg, H, W)
    sd64 = {k: v.double() for k, v in sd.items() if v.is_floating_point()}
    F_ = cfg["fusion"]
    g = torch.Generator().manual_seed(5 + route)
    # the fusion outputs at the engine's sizes (coarse to fine: H / 16 .. H / 2), a bottleneck at H / 32
    sizes = [(H // 16, W // 16), (H // 8, W // 8), (H // 4, W // 4), (H // 2, W // 2)]
    blocks = [torch.randn(1, F_, h, w, generator=g, dtype=torch.float64) for h, w in sizes]
    bh, bw = H // 32, W // 32
    bott = torch.randn(1, F_, bh, bw, generator=g, dtype=torch.float64)
    act = torch.relu(torch.randn(1, 32, H, W, generator=g, dtype=torch.float64))
    rel = None
    if not multi:
        rel = torch.relu(torch.nn.functional.conv2d(act, sd64["relative_head.conv3.weight"],
                                                    sd64["relative_head.conv3.bias"]))
    with torch.no_grad():
        ref, _, rt = ZO.metric_head(sd64, cfg, act, bott, blocks, rel, route=route if multi else None)
    assert rt == route
    nhwc = lambda t: t[0].permute(1, 2, 0).reshape(-1, t.shape[1]).numpy()  # noqa: E731
    nc = 2 if multi else 1
    assert zoedepth_attractors(sd, cfg) == [int(P[f"z.a{j}.2.b"].shape[1]) for j in range(4)]
    got, _ = HZ.metric_head(P, nc, route, nhwc(bott), bh, bw, [(nhwc(b), h, w) for b, (h, w) in zip(blocks, sizes)],
                            nhwc(act), H, W, cfg["min_temp"], cfg["max_temp"], cat=not multi)
    ref = ref.numpy().reshape(-1)
    err = float(np.abs(got - ref).max() / (ref.max() - ref.min()))
    print(f"metric head multi={multi} route={route}: max |restated - oracle| / range {err:.2e}")
    # the oracle builds log C(63, k) from f32 constants, as transformers does (about 1e-7 relative of ~260, over the
    # temperature 0.0212): a few 1e-6 of the range.  A packing slip moves the depth by O(range).
    assert err <= 1e-4
    if multi:  # the other configuration's columns give another depth: the route is not a no-op
        other, _ = HZ.metric_head(P, nc, 1 - route, nhwc(bott), bh, bw,
                                  [(nhwc(b), h, w) for b, (h, w) in zip(blocks, sizes)], nhwc(act), H, W,
                                  cfg["min_temp"], cfg["max_temp"])
        assert np.abs(other - ref).max() > 0.05 * (ref.max() - ref.min())


def test_router64_equals_the_oracle_router(zoe_models):
    sd, cfg = zoe_models[True]
    sd64 = {k: v.double() for k, v in sd.items() if v.is_floating_point()}
    x = torch.randn(1, cfg["fusion"], 3, 5, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    with torch.no_grad():
        assert torch.allclose(HZ.router64(sd64, x), ZO.router(sd64, x), rtol=1e-6, atol=1e-6)
