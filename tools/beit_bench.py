"""dpt-beit-large-512 (MiDaS v3.1 BEiT-L 512) next to DPT-Large and DA-V2 Large:

  video:  frames/s of the depth-video pass at 1920x1080 (render_depth.iter_depth_frames on in-memory frames, no
          inference size, no tracker) at batch 4 and 8, BEiT and DPT-Large in turns over several rounds
  attn:   device time of the attention per layer (the "attn" span of vd3d_depth_profile_spans, eager batch-4 forwards)
          and its algorithmic FLOP/s, 4 NT^2 64 heads B: BEiT's k_umma_attention<true> at 512x896 (NT 1793, the
          1080p processed size) beside DA-V2 Large's bias-free kernel at 518x672 (NT 1777) and 518x924 (NT 2443)

    python tools/beit_bench.py [--frames 48] [--reps 3] [--rounds 3]

Prints the GPU name and power limit (read in the same run), then one line per model and workload.  Random-init
weights with the bias tables filled (transformers initialises them to zeros): the timing does not depend on the
values, but a zero table would not be a model anyone runs."""
import argparse
import ctypes as C
import os
import statistics
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


def attn_per_launch(eng, frames, reps):
    """us per attention launch (one layer, the whole batch) over `reps` eager forwards of `frames` (one batch)."""
    for _ in range(2):
        eng.infer_batch(frames, check_size=False)
    eng.check(eng.lib.vd3d_depth_profile(eng.h, 2))
    for _ in range(reps):
        eng.infer_batch(frames, check_size=False)
    buf = C.create_string_buffer(1 << 16)
    eng.check(eng.lib.vd3d_depth_profile_spans(eng.h, buf, len(buf)))
    eng.check(eng.lib.vd3d_depth_profile(eng.h, 0))
    for line in buf.value.decode().splitlines():
        tag, ms, n = line.rsplit(" ", 2)
        if tag == "attn":
            return float(ms) * 1e3 / int(n)
    raise RuntimeError("no attn span recorded")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from transformers import DepthAnythingForDepthEstimation, DPTForDepthEstimation
    from visiondepth3d_b200 import render_depth as RD
    from visiondepth3d_b200.depth_engine import DepthEngine
    from visiondepth3d_b200.depth_weights import DPT_BEIT_PROCESSOR, hf_config, hf_dpt_beit_config
    from visiondepth3d_b200.synth import synth_frame
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(f"gpu: {q[0] if q else torch.cuda.get_device_name(0)}")
    frames = [synth_frame(k % 8, 1920, 1080, "natural")[0] for k in range(a.frames)]

    torch.manual_seed(0)
    sd = DPTForDepthEstimation(hf_dpt_beit_config()).eval().state_dict()
    g = torch.Generator().manual_seed(1)
    for k in sd:
        if k.endswith("relative_position_bias_table"):
            sd[k] = torch.randn(sd[k].shape, generator=g) * 2 ** 0.5
    models = {}
    for arch, state, proc in (("dpt-beit-large-512", sd, DPT_BEIT_PROCESSOR), ("dpt-large", None, None)):
        RD._engines = {}  # keep the other model's engines: the rounds below switch between the two
        RD.load_depth_model(arch, state, 1920, 1080, seed=0, processor=proc)
        models[arch] = (RD._state_dict, RD._arch, RD._spec, RD._processor, RD._engines)
    rates = {(m, b): [] for m in models for b in (4, 8)}
    for _ in range(a.rounds):
        for arch, st in models.items():
            RD._state_dict, RD._arch, RD._spec, RD._processor, RD._engines = st
            for batch in (4, 8):
                run = lambda: sum(1 for _ in RD.iter_depth_frames(_Cap(frames), 1920, 1080, batch_size=batch))  # noqa: E731
                run()  # warm-up: engine, buffers, pinned staging
                t0 = time.perf_counter()
                n = sum(run() for _ in range(a.reps))
                rates[(arch, batch)].append(n / (time.perf_counter() - t0))
    for (arch, batch), r in rates.items():
        print(f"{arch}: depth video 1920x1080 batch {batch}: {statistics.median(r):.1f} frames/s "
              f"(median of {len(r)} rounds, min {min(r):.1f}, max {max(r):.1f})")

    def report(name, eng, heads, B=4):
        P = 14 if eng.family == "da-v2" else 16
        nt = (eng.image_h // P) * (eng.image_w // P) + 1
        us = attn_per_launch(eng, frames[:B], a.reps)
        flop = 4.0 * nt * nt * 64 * heads * B
        print(f"{name}: attn {us:8.1f} us per layer (NT {nt}, {heads} heads, B {B}): {flop / us / 1e6:.1f} TFLOP/s")
        return flop / us

    r_beit = report("dpt-beit-large-512 512x896 (bias)", models["dpt-beit-large-512"][4][(512, 896)], 16)
    torch.manual_seed(0)
    da_sd = DepthAnythingForDepthEstimation(hf_config("vitl")).eval().state_dict()
    for h, w in ((518, 672), (518, 924)):
        da = DepthEngine("vitl", h, w)
        da.load_state_dict(da_sd)
        r_da = report(f"DA-V2 Large {h}x{w} (no bias)", da, 16)
        print(f"  BEiT attention per FLOP vs this: {100 * (r_da / r_beit - 1):+.1f} % time")
        da.close()


if __name__ == "__main__":
    main()
