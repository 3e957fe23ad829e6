"""Depth Anything V1-Large and V2-Metric-Large next to V2-Large on the same frames: frames/s of the depth-video pass
at 1920x1080 (render_depth.iter_depth_frames on in-memory frames, no inference size, no tracker) at batch 4 and 8.
The three have the same shapes; V1 only taps other layers and the metric model ends its head in max_depth * sigmoid,
so they should run at the same rate.  The models are timed in turns, `--reps` rounds, and each line gives the
median and the spread over the rounds.

    python tools/da_family_bench.py [--frames 48] [--reps 5]

Prints the GPU name and power limit (read in the same run).  Random-init weights: the timing does not depend on them."""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


class _Cap:
    def __init__(self, frames):
        self.frames, self.pos = frames, 0

    def read(self):
        if self.pos >= len(self.frames):
            return False, None
        self.pos += 1
        return True, self.frames[self.pos - 1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200 import render_depth as RD
    from visiondepth3d_b200.depth_weights import V1_TAPS, da_spec, hf_config
    from visiondepth3d_b200.synth import synth_frame
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(f"gpu: {q[0] if q else torch.cuda.get_device_name(0)}")
    frames = [synth_frame(k % 8, 1920, 1080, "natural")[0] for k in range(a.frames)]
    torch.manual_seed(0)
    sd = DepthAnythingForDepthEstimation(hf_config("vitl")).eval().state_dict()  # one set of weights for all three
    models = {"V2-Large": da_spec("vitl"), "V1-Large": da_spec("vitl", taps=V1_TAPS["vitl"]),
              "V2-Metric-Large (max_depth 20)": da_spec("vitl", head="metric", max_depth=20.0)}
    rates = {(m, b): [] for m in models for b in (4, 8)}
    for rnd in range(a.reps + 1):  # round 0 is a warm-up
        for name, spec in models.items():
            RD.load_depth_model(spec, sd, 1920, 1080)
            for batch in (4, 8):  # the new engine's first batches: buffers and staging, untimed
                sum(1 for _ in RD.iter_depth_frames(_Cap(frames[:2 * batch]), 1920, 1080, batch_size=batch))
            for batch in (4, 8):
                t0 = time.perf_counter()
                n = sum(1 for _ in RD.iter_depth_frames(_Cap(frames), 1920, 1080, batch_size=batch))
                dt = time.perf_counter() - t0
                if rnd:
                    rates[(name, batch)].append(n / dt)
    for (name, batch), r in rates.items():
        r = sorted(r)
        print(f"{name}: depth video 1920x1080 batch {batch}: {r[len(r) // 2]:.1f} frames/s "
              f"(min {r[0]:.1f}, max {r[-1]:.1f} over {len(r)} rounds)")


if __name__ == "__main__":
    main()
