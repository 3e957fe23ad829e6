"""GPU: the Real-ESRGAN stage (SURVEY 8(f) rank 3) -- SRVGGNetCompact on the wgmma implicit-GEMM convs against the
fp32 torch restatement (oracle/sr.py; the reference's ONNX model runs in fp16), and run_esrgan's resize / blend chain
against the cv2-pinned oracle."""
import numpy as np
import pytest

from oracle import sr as S
from tests.util import u8_diff
from visiondepth3d_b200.synth import synth_frame

pytestmark = pytest.mark.gpu


def _np_sd(sd):
    return {k: v.numpy() for k, v in sd.items()}


@pytest.mark.parametrize("num_conv,w,h", [(4, 96, 54), (16, 160, 90), (32, 320, 180), (32, 157, 93)])
def test_sr_forward_matches_oracle(num_conv, w, h):
    """u8 output <= 1 LSB against the fp32 oracle; f16 activations through up to 34 layers put a few per cent of the
    bytes on the other side of the x255 truncation (the reference's own ONNX model runs in fp16 end to end)."""
    import torch
    from visiondepth3d_b200 import merged_pipeline as MP
    sd = S.srvgg_state_dict(num_conv=num_conv, seed=3)
    eng = MP.SrEngine(_np_sd(sd))
    fr, _ = synth_frame(2, w, h, "natural")
    out = eng.upscale(fr)
    with torch.no_grad():
        ref = S.postprocess_esr(S.srvgg_forward(sd, torch.from_numpy(S.preprocess_esr(fr))).numpy())
    assert out.shape == ref.shape == (4 * h, 4 * w, 3)
    mx, f0, f1 = u8_diff(out, ref)
    assert mx <= 1 and f0 <= 0.04, (num_conv, w, h, mx, f0)
    # the network really contributes: the output is not the nearest-upsampled input
    base = fr.repeat(4, axis=0).repeat(4, axis=1)
    assert np.abs(out.astype(int) - base.astype(int)).mean() > 1.0
    eng.close()


def test_run_esrgan_chain_matches_oracle():
    """run_esrgan (core/merged_pipeline.py:240-267): input_res_pct resize, network, INTER_CUBIC back to the original size,
    target_size, blend -- every stage on the GPU, against the oracle chain (whose cv2 pieces are pinned on CPU)."""
    from visiondepth3d_b200 import merged_pipeline as MP
    sd = S.srvgg_state_dict(num_conv=8, seed=5)
    MP.load_esrgan(_np_sd(sd))
    fr, _ = synth_frame(4, 256, 144, "natural")
    assert MP.run_esrgan(fr) is not fr
    for kw in (dict(), dict(blend_mode="LOW"), dict(input_res_pct=50, blend_mode="MEDIUM"),
               dict(target_size=(384, 216)), dict(input_res_pct=50, target_size=(256, 144), blend_mode="HIGH")):   # blending needs equal sizes (cv2.addWeighted raises otherwise)
        out = MP.run_esrgan(fr, **kw)
        ref = S.run_esrgan(sd, fr, kw.get("blend_mode", "OFF"), kw.get("input_res_pct", 100), kw.get("target_size"))
        assert out.shape == ref.shape
        mx, f0, f1 = u8_diff(out, ref)
        assert mx <= 2 and f1 <= 1e-3 and f0 <= 0.06, (kw, mx, f0, f1)   # one network LSB through two cubic resamplings
    # stage ops against the oracle on identical inputs: exact
    rng = np.random.default_rng(2)
    a = rng.integers(0, 256, (90, 160, 3), dtype=np.uint8)
    b = rng.integers(0, 256, (90, 160, 3), dtype=np.uint8)
    for mode in ("LOW", "MEDIUM", "HIGH"):
        assert np.array_equal(MP.blend_images(a, b, mode), S.blend_images(a, b, mode)), mode
    for (ow, oh) in ((640, 360), (100, 57), (160, 90)):
        assert np.array_equal(MP._resize_cubic(a, ow, oh), S.resize_cubic_bgr(a, ow, oh)), (ow, oh)
    # tiled mode keeps the reference's (cropping) behaviour and no model -> input returned
    t = MP.run_esrgan(fr, tile=64, tile_pad=8)
    assert t.shape == fr.shape
    MP.esrgan_session.close()
    MP.esrgan_session = None
    assert MP.run_esrgan(fr) is fr
