"""Images per second of the still-image depth path on a folder of mixed-size synthetic photos (12 MP landscape and
portrait, 1600x1200, 1080p), with and without an inference size:

  gpu:  render_depth.depth_images -- Pillow resize, DPT processor, one forward per processed size (sources of one
        aspect merged), post-resize, min-max u8 and the resize back on the device (vd3d_depth_infer_images)
  host: the composition it replaces -- hf_batch_safe_pipe (Pillow resize on the host, then one forward per source
        shape), convert_depth_to_grayscale and cv2 INTER_CUBIC back on the host

    python tools/image_depth_bench.py [--reps 3] [--arch vits]

Prints the GPU name and power limit, then one line per configuration.  Random-init weights: the timing does not
depend on them."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def photos():
    from visiondepth3d_b200.synth import synth_frame
    sizes = [(4032, 3024)] * 4 + [(3024, 4032)] * 4 + [(1600, 1200)] * 4 + [(1920, 1080)] * 4
    from PIL import Image
    return [Image.fromarray(synth_frame(k, w, h, "natural")[0][..., ::-1].copy()) for k, (w, h) in enumerate(sizes)]


def host_path(RD, images, inference_size):
    import cv2
    out = []
    for img, res in zip(images, RD.hf_batch_safe_pipe(images, inference_size)):
        d8 = RD.convert_depth_to_grayscale(res["predicted_depth"])
        if d8.shape[::-1] != img.size:
            d8 = cv2.resize(d8, img.size, interpolation=cv2.INTER_CUBIC)
        out.append(d8)
    return out


def timed(fn, reps):
    fn()  # warm-up: engines, tables, buffers
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--arch", default="vits")
    a = ap.parse_args()
    import torch
    from visiondepth3d_b200 import render_depth as RD
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print(f"gpu: {q[0] if q else torch.cuda.get_device_name(0)}")
    RD.load_depth_model(a.arch, None, 640, 480, seed=0)
    images = photos()
    n = len(images)
    for inf in (None, (910, 518)):
        gpu = lambda: RD.depth_images(images, inf)  # noqa: E731
        host = lambda: host_path(RD, images, inf)  # noqa: E731
        same = max(int(np.abs(x.astype(int) - y.astype(int)).max()) for x, y in zip(gpu(), host()))
        tg, th = timed(gpu, a.reps), timed(host, a.reps)
        print(f"inference_size={inf}: {n} images  gpu {n / tg:.2f} img/s  host {n / th:.2f} img/s  "
              f"speed-up {th / tg:.2f}x  (max |gpu - host| = {same} LSB)")


if __name__ == "__main__":
    main()
