"""BASELINE config 4: 1080p depth + stereo (DA-V2-Base, Full-SBS, preserve_original_aspect -> 3840x1080) followed by the
Real-ESRGAN x4 stage (realesr-general-x4v3 shape: 32 body convs, random init) to a 7680x2160 target, all on the device:
vd3d_render_clip_depth with device outputs, then vd3d_sr_upscale on those frames.  Prints one JSON line: the joined
rate, the SR stage alone, the untiled run_esrgan chain as composed before vd3d_sr_upscale (per frame, host buffers) at
1920x1080 and 3840x1080, the network's TFLOP/s, and the card, its power limit and the median SM clock of the run.
    python tools/config4_bench.py [--frames 8] [--reps 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def _smi(q):
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        return None


class _Clock:
    def __init__(self):
        self.mhz, self.stop = [], threading.Event()

    def run(self):
        while not self.stop.is_set():
            v = _smi("clocks.sm")
            try:
                self.mhz.append(float(v))
            except (TypeError, ValueError):
                pass
            self.stop.wait(0.2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    from transformers import DepthAnythingForDepthEstimation
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import merged_pipeline as MP
    from visiondepth3d_b200 import render_3d as R
    from visiondepth3d_b200.depth_engine import DepthEngine, processed_size
    from visiondepth3d_b200.depth_weights import hf_config
    from visiondepth3d_b200.synth import synth_frame
    w, h, n, nc = 1920, 1080, a.frames, 32
    ctx = _lib.default_context(0)
    torch.manual_seed(0)
    sd = DepthAnythingForDepthEstimation(hf_config("vitb")).eval().state_dict()
    ih, iw = processed_size(w, h)
    deng = DepthEngine("vitb", ih, iw, ctx=ctx)
    deng.load_state_dict(sd)
    del sd
    rp = R.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, "Full-SBS", 16 / 9, 0.0, 10.0, 9, True, True,
                              preserve_original_aspect=True, zero_parallax_strength=0.01)
    oshape = R.output_shape(rp, R.plan_sizes(w, h, rp))           # (1080, 3840, 3)
    target = (7680, 2160)
    sr = MP.load_esrgan(MP.random_srvgg_state_dict(nc, 0))
    params = MP.upscale_params(target_size=target)
    dev = torch.device("cuda", 0)
    fd = [torch.from_numpy(synth_frame(i, w, h, "noise")[0]).to(dev) for i in range(n)]
    sbs = [torch.empty(oshape, dtype=torch.uint8, device=dev) for _ in range(n)]
    up = [torch.empty((target[1], target[0], 3), dtype=torch.uint8, device=dev) for _ in range(n)]
    fp = (C.c_void_p * n)(*[t.data_ptr() for t in fd])
    sp = (C.c_void_p * n)(*[t.data_ptr() for t in sbs])
    torch.cuda.synchronize()

    def joined():
        ctx.check(ctx.lib.vd3d_render_clip_depth(ctx.h, deng.h, n, fp, h, w, C.byref(rp), sp, _lib.MEM_DEVICE))
        sr_only()

    def sr_only():
        sr.upscale_ptrs([t.data_ptr() for t in sbs], oshape[0], oshape[1], params, [t.data_ptr() for t in up],
                        _lib.MEM_DEVICE)

    def rate(fn, frames):
        fn()  # warm-up: buffers, tables, graphs
        best = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            fn()
            best.append(frames / (time.perf_counter() - t0))
        return float(np.median(best))

    def old_chain(frame):
        u = sr.upscale(frame)
        u = MP._resize_cubic(u, 4 * frame.shape[1], 4 * frame.shape[0])
        u = MP._resize_cubic(u, frame.shape[1], frame.shape[0])
        return MP._resize_cubic(u, target[0], target[1])

    def new_host(frame):
        return sr.upscale_chain([frame], params, target)

    clk = _Clock()
    th = threading.Thread(target=clk.run, daemon=True)
    th.start()
    res = {"joined_fps": rate(joined, n), "sr_stage_fps": rate(sr_only, n)}
    for fw in (1920, 3840):
        fr = np.ascontiguousarray(np.concatenate([synth_frame(i, 1920, 1080, "noise")[0] for i in range(fw // 1920)], 1))
        k = 3
        res[f"old_run_esrgan_{fw}x1080_fps"] = rate(lambda: [old_chain(fr) for _ in range(k)], k)
        res[f"new_run_esrgan_{fw}x1080_fps"] = rate(lambda: [new_host(fr) for _ in range(k)], k)
    clk.stop.set()
    th.join()
    tflop = 2.0 * oshape[1] * oshape[0] * 9 * 64 * (64 * (nc + 1) + 48) / 1e12
    res.update({
        "sr_tflop_per_frame": round(tflop, 2),
        "sr_tflops": round(tflop * res["sr_stage_fps"], 1),
        "frames": n, "sbs_shape": list(oshape), "target": list(target), "body_convs": nc,
        "gpu": _smi("name"), "power_limit_w": _smi("power.limit"),
        "sm_clock_mhz_median": float(np.median(clk.mhz)) if clk.mhz else None,
    })
    print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in res.items()}))
    ctx.check(ctx.lib.vd3d_release_depth(ctx.h, deng.h))


if __name__ == "__main__":
    main()
