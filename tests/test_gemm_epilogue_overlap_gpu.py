"""GPU: k_umma_gemm hands every finished tile from the MMA warpgroups to the epilogue warpgroup through one shared
staging tile.  At the token shapes of a 4-frame DA-V2 batch (M = 10123 rows, 80 m-tiles) each persistent CTA walks
about 4-20 tiles, so the hand-off wraps many times per launch; a missed wait on the staging tile shows up as wrong
or run-to-run different results."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M_BATCH4 = 10123  # stacked token rows of a 4-frame 518 x 924 batch: 3 x 2560 (padded) + 2443 (37 x 66 patches + cls)


@pytest.fixture(scope="module")
def eng():
    from visiondepth3d_b200.depth_engine import DepthEngine
    e = DepthEngine("vits", 70, 98)
    yield e
    e.close()


@pytest.mark.parametrize("nk", [(2304, 768), (768, 768), (3072, 768), (768, 3072)])
def test_token_gemm_matches_numpy(eng, nk):
    N, K = nk
    rng = np.random.default_rng(N * 31 + K)
    A = (rng.standard_normal((M_BATCH4, K)) * 0.5).astype(np.float16)
    B = (rng.standard_normal((N, K)) * 0.5).astype(np.float16)
    ref = A.astype(np.float32) @ B.astype(np.float32).T
    bns = (0, 64, 32) if N == 768 else (0,)
    for bn in bns:
        out = eng.gemm(A, B, bn)
        assert np.abs(out - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), (nk, bn)


def test_batched_vitb_forward_is_deterministic():
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import hf_config
    from visiondepth3d_b200.synth import synth_frame
    torch.manual_seed(0)
    sd = DepthAnythingForDepthEstimation(hf_config("vitb")).eval().state_dict()
    e = DepthEngine("vitb", 518, 924)
    e.load_state_dict(sd)
    frames = [synth_frame(i, 1920, 1080, "natural")[0] for i in range(4)]
    first = e.infer_batch(frames)
    second = e.infer_batch(frames)
    for k in range(4):
        assert np.array_equal(first[k][0].view(np.uint32), second[k][0].view(np.uint32)), k
        assert np.array_equal(first[k][1], second[k][1]), k
    e.close()
