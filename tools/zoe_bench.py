"""ZoeDepth (Intel/zoedepth-nyu-kitti's configuration) next to dpt-beit-large-512:

  video:  frames/s of the depth-video pass at 1920x1080 (render_depth.iter_depth_frames on in-memory frames, no
          inference size, no tracker) at batch 4 and 8, the two models in turns over several rounds
  spans:  device time per launch class of eager batch-4 forwards (vd3d_depth_profile_spans) and the share of the
          forward spent in the metric head's zoe.* spans

    python tools/zoe_bench.py [--frames 48] [--reps 3] [--rounds 3]

Prints the GPU name and power limit (read in the same run), then one line per model and workload.  Random-init
weights with filled bias tables: the timing does not depend on the values."""
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


def spans(eng, frames, reps):
    """{tag: ms per forward} over `reps` eager forwards of one batch."""
    for _ in range(2):
        eng.infer_batch(frames, check_size=False)
    eng.check(eng.lib.vd3d_depth_profile(eng.h, 2))
    for _ in range(reps):
        eng.infer_batch(frames, check_size=False)
    buf = C.create_string_buffer(1 << 16)
    eng.check(eng.lib.vd3d_depth_profile_spans(eng.h, buf, len(buf)))
    eng.check(eng.lib.vd3d_depth_profile(eng.h, 0))
    out = {}
    for line in buf.value.decode().splitlines():
        tag, ms, _ = line.rsplit(" ", 2)
        out[tag] = float(ms) / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from transformers import DPTForDepthEstimation, ZoeDepthForDepthEstimation
    from visiondepth3d_b200 import render_depth as RD
    from visiondepth3d_b200.depth_weights import (DPT_BEIT_PROCESSOR, ZOEDEPTH_PROCESSOR, hf_dpt_beit_config,
                                                  hf_zoedepth_config)
    from visiondepth3d_b200.synth import synth_frame
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(f"gpu: {q[0] if q else torch.cuda.get_device_name(0)}")
    frames = [synth_frame(k % 8, 1920, 1080, "natural")[0] for k in range(a.frames)]

    def filled(sd):
        g = torch.Generator().manual_seed(1)
        for k in sd:
            if k.endswith("relative_position_bias_table"):
                sd[k] = torch.randn(sd[k].shape, generator=g) * 2 ** 0.5
        return sd
    torch.manual_seed(0)
    zoe = filled(ZoeDepthForDepthEstimation(hf_zoedepth_config()).eval().state_dict())
    beit = filled(DPTForDepthEstimation(hf_dpt_beit_config()).eval().state_dict())
    models = {}
    for arch, state, proc in (("zoedepth-nyu-kitti", zoe, ZOEDEPTH_PROCESSOR),
                              ("dpt-beit-large-512", beit, DPT_BEIT_PROCESSOR)):
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
    eng = models["zoedepth-nyu-kitti"][4][(384, 672)]
    sp = spans(eng, frames[:4], a.reps)
    total = sp.pop("tail(all images, forked)", 0.0) + sum(v for k, v in sp.items() if k in (
        "embed", "ln", "qkv", "attn", "proj", "fc1", "fc2"))
    for tag, ms in sorted(sp.items()):
        print(f"  span {tag}: {ms:.3f} ms per batch-4 forward")
    # the zoe.* spans run on the four tails' side streams: their sum is device time, not wall time
    zoe_ms = sum(v for k, v in sp.items() if k.startswith("zoe."))
    print(f"zoedepth batch 4: zoe.* spans {zoe_ms:.3f} ms of device time (summed over the images' tails), the "
          f"forward's transformer spans + forked tail {total:.3f} ms")


if __name__ == "__main__":
    main()
