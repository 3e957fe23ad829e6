"""The RRDBNet upscalers (nb = 23, random init) on the device: forward frames/s and algorithmic TFLOP/s at 960x540,
1920x1080 and 3840x1080 inputs for x4 and x2 (vd3d_sr_forward, device memory), and BASELINE config 4 with
RealESRGAN_x4: 1080p depth + Full-SBS (DA-V2-Base, preserve_original_aspect -> 3840x1080), then run_esrgan's chain to a
7680x2160 target (vd3d_render_clip_depth, then vd3d_sr_upscale, device memory).  FLOPs are counted on the unpadded
network (35.9 MFLOP per input pixel at x4, 33.8 at x2), not on what the padded dense convs execute.  Prints one JSON
line with the card, its power limit and the median SM clock of the run.
    python tools/rrdb_bench.py [--reps 3] [--frames 2] [--skip-config4]"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.config4_bench import _Clock, _smi  # noqa: E402


def flop_per_pixel(nb, scale):
    """2 x 9 x sum(Cin x Cout) over the convs, per input pixel (the up-convs and the tail run on scale^2 pixels)."""
    rdb = sum(32 * (64 + 32 * k) for k in range(4)) + 64 * 192
    trunk = 3 * 64 + nb * 3 * rdb + 64 * 64
    tail = sum(64 * 64 * 4 ** u for u in range(1, 2 if scale == 2 else 3)) + (64 * 64 + 64 * 3) * scale * scale
    return 2.0 * 9 * (trunk + tail)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--skip-config4", action="store_true")
    a = ap.parse_args()
    import torch
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import merged_pipeline as MP
    from visiondepth3d_b200.synth import synth_frame
    if not torch.cuda.is_available():
        raise SystemExit("rrdb_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    clk = _Clock()
    th = threading.Thread(target=clk.run, daemon=True)
    th.start()
    res = {}

    def rate(fn, frames):
        fn()  # warm-up: buffers, tensor maps, kernel attributes
        torch.cuda.synchronize()
        runs = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            runs.append(frames / (time.perf_counter() - t0))
        return float(np.median(runs))

    for scale in (4, 2):
        eng = MP.SrEngine(MP.random_rrdb_state_dict(23, scale, seed=0))
        for w, h in ((960, 540), (1920, 1080), (3840, 1080)):
            fr = np.ascontiguousarray(np.concatenate([synth_frame(i, min(w, 1920), h, "natural")[0]
                                                      for i in range(max(1, w // 1920))], 1))
            x = torch.from_numpy(fr).to(dev)
            out = torch.empty((scale * h, scale * w, 3), dtype=torch.uint8, device=dev)
            torch.cuda.synchronize()

            def fwd():
                eng.check(eng.lib.vd3d_sr_forward(eng.h, x.data_ptr(), h, w, 0, out.data_ptr(), _lib.MEM_DEVICE))

            fps = rate(fwd, 1)
            res[f"x{scale}_{w}x{h}_fps"] = fps
            res[f"x{scale}_{w}x{h}_tflops"] = flop_per_pixel(23, scale) * w * h * fps / 1e12
            del x, out
        eng.close()
        torch.cuda.empty_cache()

    if not a.skip_config4:
        from transformers import DepthAnythingForDepthEstimation
        from visiondepth3d_b200 import render_3d as R
        from visiondepth3d_b200.depth_engine import DepthEngine, processed_size
        from visiondepth3d_b200.depth_weights import hf_config
        w, h, n = 1920, 1080, a.frames
        ctx = _lib.default_context(0)
        torch.manual_seed(0)
        sd = DepthAnythingForDepthEstimation(hf_config("vitb")).eval().state_dict()
        ih, iw = processed_size(w, h)
        deng = DepthEngine("vitb", ih, iw, ctx=ctx)
        deng.load_state_dict(sd)
        del sd
        rp = R.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, "Full-SBS", 16 / 9, 0.0, 10.0, 9, True, True,
                                  preserve_original_aspect=True, zero_parallax_strength=0.01)
        oshape = R.output_shape(rp, R.plan_sizes(w, h, rp))  # (1080, 3840, 3)
        target = (7680, 2160)
        sr = MP.load_esrgan(MP.random_rrdb_state_dict(23, 4, seed=0))
        params = MP.upscale_params(target_size=target)
        fd = [torch.from_numpy(synth_frame(i, w, h, "natural")[0]).to(dev) for i in range(n)]
        sbs = [torch.empty(oshape, dtype=torch.uint8, device=dev) for _ in range(n)]
        up = [torch.empty((target[1], target[0], 3), dtype=torch.uint8, device=dev) for _ in range(n)]
        fp = (C.c_void_p * n)(*[t.data_ptr() for t in fd])
        sp = (C.c_void_p * n)(*[t.data_ptr() for t in sbs])
        torch.cuda.synchronize()

        def sr_only():
            sr.upscale_ptrs([t.data_ptr() for t in sbs], oshape[0], oshape[1], params, [t.data_ptr() for t in up],
                            _lib.MEM_DEVICE)

        def joined():
            ctx.check(ctx.lib.vd3d_render_clip_depth(ctx.h, deng.h, n, fp, h, w, C.byref(rp), sp, _lib.MEM_DEVICE))
            sr_only()

        res["config4_rrdb_x4_joined_fps"] = rate(joined, n)
        res["config4_rrdb_x4_sr_stage_fps"] = rate(sr_only, n)
        res["config4_frames"] = n
        ctx.check(ctx.lib.vd3d_release_depth(ctx.h, deng.h))
    clk.stop.set()
    th.join()
    res.update({"nb": 23, "mflop_per_input_pixel": {"x4": flop_per_pixel(23, 4) / 1e6, "x2": flop_per_pixel(23, 2) / 1e6},
                "gpu": _smi("name"), "power_limit_w": _smi("power.limit"),
                "sm_clock_mhz_median": float(np.median(clk.mhz)) if clk.mhz else None})
    print(json.dumps({k: (round(v, 3) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
