"""GPU: a forward whose per-image tail fails leaves the depth engine usable.  With two or more images each tail runs on
a side stream; a tail that stops early (here at a missing neck weight) must hand the engine's helpers back to the
engine stream, so that later unit-test hooks and forwards are ordered with their copies and synchronisations."""
import ctypes as C

import numpy as np
import pytest

from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu

VD3D_ERR_STATE = -5
H, W = 180, 320


def _engine(sd, skip=()):
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import prepare
    e = DepthEngine("vits", 70, 126)
    for name, arr in prepare(sd, e.cfg, e.image_h, e.image_w).items():
        if name not in skip:
            arr = np.ascontiguousarray(arr)
            e.check(e.lib.vd3d_depth_set_tensor(e.h, name.encode(), arr.ctypes.data, arr.nbytes))
    return e


def test_engine_after_a_failed_tail():
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200.depth_weights import hf_config, prepare
    torch.manual_seed(0)
    sd = DepthAnythingForDepthEstimation(hf_config("vits")).eval().state_dict()
    frames = [synth_frame(i, W, H, "natural")[0] for i in (1, 2)]
    e = _engine(sd, skip=("n0.conv.w",))
    fresh = _engine(sd)
    try:
        n = len(frames)
        d32 = [np.empty((H, W), np.float32) for _ in frames]
        d8 = [np.empty((H, W), np.uint8) for _ in frames]
        vp = C.c_void_p
        rc = e.lib.vd3d_depth_infer_batch(e.h, n, (vp * n)(*[f.ctypes.data for f in frames]), H, W,
                                          (vp * n)(*[a.ctypes.data for a in d32]),
                                          (vp * n)(*[a.ctypes.data for a in d8]), 0)
        assert rc == VD3D_ERR_STATE
        assert b"n0.conv.w" in e.lib.vd3d_depth_last_error(e.h)

        rng = np.random.default_rng(0)
        a = rng.standard_normal((384, 256)).astype(np.float16)
        b = rng.standard_normal((192, 256)).astype(np.float16)
        ref = a.astype(np.float64) @ b.astype(np.float64).T
        assert np.abs(e.gemm(a, b) - ref).max() <= 1e-3

        w = np.ascontiguousarray(prepare(sd, e.cfg, e.image_h, e.image_w)["n0.conv.w"])
        e.check(e.lib.vd3d_depth_set_tensor(e.h, b"n0.conv.w", w.ctypes.data, w.nbytes))
        for (g32, g8), (f32, f8) in zip(e.infer_batch(frames, check_size=False),
                                        fresh.infer_batch(frames, check_size=False)):
            assert np.array_equal(g32, f32) and np.array_equal(g8, f8)
    finally:
        e.close()
        fresh.close()
