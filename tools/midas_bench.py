"""MiDaS 3.0 (DPT-Hybrid) next to DPT-Large on the same frames:

  video:  frames/s of the depth-video pass at 1920x1080 (render_depth.iter_depth_frames on in-memory frames, no
          inference size, no tracker) at batch 4 and 8
  images: images/s of render_depth.depth_images on a folder of mixed-size synthetic photos (12 MP landscape and
          portrait, 1600x1200, 1080p)
  spans:  MiDaS 3.0's device time per launch class of an eager batch-4 forward (vd3d_depth_profile_spans), and the
          BiT backbone's share of it (the bit.* spans)

    python tools/midas_bench.py [--frames 48] [--reps 3]

Prints the GPU name and power limit (read in the same run), then one line per model and workload.  Random-init
weights: the timing does not depend on them."""
import argparse
import ctypes as C
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


def spans(eng, frames, reps):
    """{tag: us per frame} of `reps` eager forwards of `frames` (one batch)."""
    for _ in range(2):
        eng.infer_batch(frames)
    eng.check(eng.lib.vd3d_depth_profile(eng.h, 2))
    for _ in range(reps):
        eng.infer_batch(frames)
    buf = C.create_string_buffer(1 << 16)
    eng.check(eng.lib.vd3d_depth_profile_spans(eng.h, buf, len(buf)))
    eng.check(eng.lib.vd3d_depth_profile(eng.h, 0))
    out = {}
    for line in buf.value.decode().splitlines():
        tag, ms, _n = line.rsplit(" ", 2)
        out[tag] = float(ms) * 1e3 / (reps * len(frames))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    from PIL import Image
    from visiondepth3d_b200 import render_depth as RD
    from visiondepth3d_b200.synth import synth_frame
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(f"gpu: {q[0] if q else torch.cuda.get_device_name(0)}")
    frames = [synth_frame(k % 8, 1920, 1080, "natural")[0] for k in range(a.frames)]
    sizes = [(4032, 3024)] * 4 + [(3024, 4032)] * 4 + [(1600, 1200)] * 4 + [(1920, 1080)] * 4
    photos = [Image.fromarray(synth_frame(k, w, h, "natural")[0][..., ::-1].copy()) for k, (w, h) in enumerate(sizes)]
    for arch in ("dpt-large", "dpt-hybrid-midas"):
        RD.load_depth_model(arch, None, 1920, 1080, seed=0)
        for batch in (4, 8):
            run = lambda: sum(1 for _ in RD.iter_depth_frames(_Cap(frames), 1920, 1080, batch_size=batch))  # noqa: E731
            run()  # warm-up: engine, buffers, pinned staging
            t0 = time.perf_counter()
            n = sum(run() for _ in range(a.reps))
            dt = time.perf_counter() - t0
            print(f"{arch}: depth video 1920x1080 batch {batch}: {n / dt:.1f} frames/s")
        RD.depth_images(photos)  # warm-up
        t0 = time.perf_counter()
        for _ in range(a.reps):
            RD.depth_images(photos)
        dt = (time.perf_counter() - t0) / a.reps
        print(f"{arch}: still images ({len(photos)} mixed sizes): {len(photos) / dt:.2f} img/s")
        if arch == "dpt-hybrid-midas":
            sp = spans(RD._engine_for(1920, 1080), frames[:4], a.reps)
            tot = sum(sp.values())
            bit = sum(v for k, v in sp.items() if k.startswith("bit."))
            for k, v in sorted(sp.items(), key=lambda kv: -kv[1]):
                print(f"  span {k:28s} {v:9.1f} us/frame")
            print(f"{arch}: device time per frame (eager, batch 4) {tot:.1f} us, BiT backbone {bit:.1f} us "
                  f"({100 * bit / tot:.1f} %)")


if __name__ == "__main__":
    main()
