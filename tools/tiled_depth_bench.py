"""Tiled depth-video throughput (render_depth.USE_TILED_DEPTH): vd3d_depth_tiled on batches of 8 frames, on device
frames and on host frames, against the untiled pass on the same frames and against the reference-structured loop
(infer_depth_tile's one synchronous pipe call per tile, restated here).  Random-init weights: the forward's cost does
not depend on them.  Prints the card, its power limit and SM clock from the same run.

    python tools/tiled_depth_bench.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"nvidia-smi unavailable: {e}"
    return q


def timed(fn, reps):
    import torch
    fn()  # warm-up: engines, plan, buffers
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def reference_loop(R, frames, W, H):
    """infer_depth_tile as the reference runs it: one pipe call per tile, then the blend and _normalize_to_u8."""
    import cv2
    from PIL import Image
    for f in frames:
        rgb = f[..., ::-1]
        acc = np.zeros((H, W), np.float32)
        wacc = np.zeros((H, W), np.float32)
        for y0, y1, x0, x1, yp0, yp1, xp0, xp1, rh, rw in R.tile_plan(W, H):
            c = rgb[yp0:yp1, xp0:xp1]
            if c.shape[:2] != (rh, rw):
                c = cv2.resize(c, (rw, rh), interpolation=cv2.INTER_CUBIC)
            pred = R.pipe([Image.fromarray(np.ascontiguousarray(c))], inference_size=(rw, rh))[0]["predicted_depth"]
            p = pred.numpy()[y0 - yp0:y0 - yp0 + y1 - y0, x0 - xp0:x0 - xp0 + x1 - x0]
            wm = R.tile_weights(y1 - y0, x1 - x0)
            acc[y0:y1, x0:x1] += p * wm
            wacc[y0:y1, x0:x1] += wm
        R._normalize_to_u8(acc / np.maximum(wacc, 1e-8), (W, H))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    from visiondepth3d_b200 import render_depth as R
    print(json.dumps({"card": card()}))
    for arch, (W, H) in (("vitb", (1920, 1080)), ("vitl", (3840, 2160))):
        R.load_depth_model(arch, None, W, H, seed=0)
        rng = np.random.default_rng(0)
        frames = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(8)]
        dev = torch.from_numpy(np.stack(frames)).cuda()
        eng = R._engine_for(W, H)
        res = {"arch": arch, "size": f"{W}x{H}", "batch": 8, "tiles": len(R.tile_plan(W, H))}
        res["tiled_device_fps"] = 8 / timed(lambda: R.depth_tiled(dev, W, H, (W, H)), a.reps)
        res["tiled_host_fps"] = 8 / timed(lambda: R.depth_tiled(frames, W, H, (W, H)), a.reps)
        res["untiled_host_fps"] = 8 / timed(lambda: eng.infer_batch(frames), a.reps)
        res["reference_loop_fps"] = 2 / timed(lambda: reference_loop(R, frames[:2], W, H), 1)
        print(json.dumps(res))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
