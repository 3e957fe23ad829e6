"""Device time of the fused ViT attention launch (k_umma_attention) alone, at the depth-video shape: 518x924 input,
2443 tokens, DA-V2-Base (12 heads) and -Large (16 heads) widths, batch 4 and 8.

    python tools/attn_bench.py [--reps 10]

Each attention launch of an eager forward is bracketed by CUDA events (vd3d_depth_profile(e, 2), the `attn` launch
class of tools/depth_spans.py); prints us per launch and the attention's algorithmic TFLOP/s
(4 * N^2 * 64 * heads * B per launch), beside the GPU name and power limit read in the same run.  Random-init
weights: the timing does not depend on them."""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import CONFIGS, hf_config
    from visiondepth3d_b200.synth import synth_frame
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(f"gpu: {q[0] if q else torch.cuda.get_device_name(0)}")
    frames = [synth_frame(i, 1920, 1080, "natural")[0] for i in range(8)]
    for arch in ("vitb", "vitl"):
        e = DepthEngine(arch, 518, 924)
        torch.manual_seed(0)
        e.load_state_dict(DepthAnythingForDepthEstimation(hf_config(arch)).eval().state_dict())
        ntok = (518 // 14) * (924 // 14) + 1
        heads = CONFIGS[arch]["heads"]
        for B in (4, 8):
            for _ in range(3):
                e.infer_batch(frames[:B])
            e.check(e.lib.vd3d_depth_profile(e.h, 2))
            for _ in range(a.reps):
                e.infer_batch(frames[:B])
            buf = C.create_string_buffer(1 << 16)
            e.check(e.lib.vd3d_depth_profile_spans(e.h, buf, len(buf)))
            e.check(e.lib.vd3d_depth_profile(e.h, 0))
            spans = {ln.rsplit(" ", 2)[0]: ln.rsplit(" ", 2)[1:] for ln in buf.value.decode().splitlines()}
            ms, n = float(spans["attn"][0]), int(spans["attn"][1])
            us = ms * 1e3 / n
            tflops = 4.0 * ntok * ntok * 64 * heads * B / (us * 1e-6) / 1e12
            print(f"{arch}: {ntok} tokens, {heads} heads, batch {B}: {us:8.1f} us per launch, {tflops:6.1f} TFLOP/s "
                  f"({n} launches)", flush=True)
        del e


if __name__ == "__main__":
    main()
