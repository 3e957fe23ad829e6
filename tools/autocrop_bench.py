"""auto_crop_black_bars cost: DIBR-only vd3d_render_clip frames/s on device-resident letterboxed clips (2.39:1 content
with dark bars inside a 16:9 frame), CUDA graphs on, auto-crop off vs on.

    python tools/autocrop_bench.py [--frames 96] [--runs 5] [--only 1080p|4k]

1080p: 1920x1080 source -> Half-SBS 1920x1080 (the bench.py 1080p arm's DIBR configuration).
4k: 3840x2160 source -> Full-SBS 7680x2160 with preserve_original_aspect (the 4K arm's); with auto-crop off this takes
the identity path that samples the u8 frame directly, with it on the frame goes through the RGBx plane.
Each setting has a context of its own (its own captured graphs); the settings alternate, `runs` timed calls each after
one warm-up call.  Prints the GPU name and power limit with the numbers, and one JSON line at the end."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

CONFIGS = {
    "1080p": dict(w=1920, h=1080, fmt="Half-SBS", preserve=False),
    "4k": dict(w=3840, h=2160, fmt="Full-SBS", preserve=True),
}


def letterboxed(i, w, h):
    """Natural synthetic content with 2.39:1 picture rows and dark (gray <= 6) bars above and below."""
    from visiondepth3d_b200.synth import synth_frame
    f, d = synth_frame(i, w, h, "natural")
    bar = (h - int(w / 2.39)) // 2
    rng = np.random.default_rng(100 + i)
    f[:bar] = rng.integers(0, 7, (bar, w, 3), dtype=np.uint8)
    f[h - bar:] = rng.integers(0, 7, (bar, w, 3), dtype=np.uint8)
    return f, d, bar


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=96)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--only", choices=sorted(CONFIGS), default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("autocrop_bench.py needs a CUDA device")
    from visiondepth3d_b200 import _lib
    from visiondepth3d_b200 import render_3d as R
    name, limit = gpu_info()
    print(f"GPU: {name}, power limit {limit}", flush=True)
    dev = torch.device("cuda", 0)
    result = {"gpu": name, "power_limit": limit, "frames_per_call": args.frames, "runs": args.runs}
    for key, cfg in CONFIGS.items():
        if args.only and key != args.only:
            continue
        w, h, n = cfg["w"], cfg["h"], args.frames
        pool = [letterboxed(i, w, h) for i in range(3)]
        f = [torch.from_numpy(a).to(dev) for a, _, _ in pool]
        d = [torch.from_numpy(b).to(dev) for _, b, _ in pool]
        ctxs, params, outs = {}, {}, {}
        for on in (0, 1):
            rp = R.make_render_params(w, h, 4.5, -1.5, -6.0, 0.2, cfg["fmt"], 16 / 9, 0.0, 10.0, 9, True, True,
                                      preserve_original_aspect=cfg["preserve"], zero_parallax_strength=0.01,
                                      auto_crop_black_bars=on)
            shape = R.output_shape(rp, R.plan_sizes(w, h, rp))
            ctxs[on], params[on] = _lib.Context(0), rp
            outs[on] = [torch.empty(shape, dtype=torch.uint8, device=dev) for _ in range(3)]
        idx = [i % 3 for i in range(n)]
        pa = (C.c_void_p * n)(*[f[i].data_ptr() for i in idx])
        pd = (C.c_void_p * n)(*[d[i].data_ptr() for i in idx])
        po = {on: (C.c_void_p * n)(*[outs[on][i].data_ptr() for i in idx]) for on in (0, 1)}
        torch.cuda.synchronize()

        def run(on):
            c = ctxs[on]
            t0 = time.perf_counter()
            c.check(c.lib.vd3d_render_clip(c.h, n, pa, pd, 3, h, w, C.byref(params[on]), po[on], _lib.MEM_DEVICE, None))
            torch.cuda.synchronize()  # vd3d_render_clip synchronises its streams; this covers torch's as well
            return n / (time.perf_counter() - t0)

        for on in (0, 1):
            run(on)  # warm-up: allocations, eager frames, graph capture
        fps = {0: [], 1: []}
        for _ in range(args.runs):
            for on in (0, 1):
                fps[on].append(run(on))
        tb = (C.c_int32 * (2 * n))()
        ctxs[1].check(ctxs[1].lib.vd3d_last_crops(ctxs[1].h, tb, n))
        assert all(tb[2 * k] == pool[idx[k]][2] and tb[2 * k + 1] == pool[idx[k]][2] for k in range(n)), "crop rows"
        for on in (0, 1):
            ctxs[on].close()
        off_m, on_m = float(np.median(fps[0])), float(np.median(fps[1]))
        print(f"{key} ({w}x{h} -> {cfg['fmt']}, {pool[0][2]}-row bars): auto-crop off "
              f"{' '.join(f'{v:.1f}' for v in fps[0])} frames/s (median {off_m:.1f}); on "
              f"{' '.join(f'{v:.1f}' for v in fps[1])} (median {on_m:.1f}); on/off {on_m / off_m:.3f}", flush=True)
        result[key] = {"off_frames_per_s": fps[0], "on_frames_per_s": fps[1], "off_median": off_m, "on_median": on_m,
                       "ratio": on_m / off_m, "bar_rows": pool[0][2]}
        del f, d, outs
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
