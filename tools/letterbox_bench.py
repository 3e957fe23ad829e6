"""Cost of the letterbox tracker of the depth-video pass.  Prints one JSON line:
- stats_us / repad_us: host wall time per frame of the synchronous vd3d_letterbox_stats (row/frame statistics + Canny,
  including the record download) and vd3d_letterbox_repad calls on device-resident data, batches of 8 frames (stats),
  at 1080p and 4K;
- video_ms: in-memory depth-video time per frame (render_depth.iter_depth_frames, random-init weights) with the
  tracker off and on: vitb at 1080p, vitl at 4K;
- oracle_ms: the numpy / cv2 statement of the same per-frame work on the host cores (all row / frame statistics,
  Canny, the scene-cut test and the single-frame detection), for reference.
Usage: python tools/letterbox_bench.py [--frames 24]"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class _Cap:
    def __init__(self, frames):
        self.frames, self.pos = frames, 0

    def read(self):
        if self.pos >= len(self.frames):
            return False, None
        self.pos += 1
        return True, self.frames[self.pos - 1]


def _wall_us(fn, reps):
    fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()  # each call synchronises the library's stream before it returns
    return (time.perf_counter() - t0) * 1e6 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=24)
    args = ap.parse_args()
    import torch
    from tests import letterbox_oracle as L
    from visiondepth3d_b200 import _lib, render_depth as RD
    from visiondepth3d_b200.synth import synth_frame
    ctx = _lib.default_context(0)
    res = {"stats_us": {}, "repad_us": {}, "video_ms": {}, "oracle_ms": {}}
    for name, (w, h, arch) in {"1080p": (1920, 1080, "vitb"), "4k": (3840, 2160, "vitl")}.items():
        f = synth_frame(1, w, h, "letterbox")[0]
        n = 8
        fr = torch.from_numpy(np.ascontiguousarray(np.stack([f] * n))).cuda()
        rec = [np.empty(s, t) for s, t in (((n, h), np.float32),) * 3 + (((n, h), np.int32), ((n,), np.float32),
                                                                          ((n, 64), np.uint32), ((n,), np.uint64))]
        torch.cuda.synchronize()
        stats = lambda: ctx.check(ctx.lib.vd3d_letterbox_stats(ctx.h, n, fr.data_ptr(), h, w, None, _lib.MEM_DEVICE,
                                                                *(r.ctypes.data for r in rec), None))
        res["stats_us"][name] = round(_wall_us(stats, 5) / n, 1)
        d = torch.from_numpy(f[..., 1].copy()).cuda()
        o = torch.empty_like(d)
        torch.cuda.synchronize()
        repad = lambda: ctx.check(ctx.lib.vd3d_letterbox_repad(ctx.h, d.data_ptr(), h, w, h // 8, h // 8,
                                                                o.data_ptr(), _lib.MEM_DEVICE))
        res["repad_us"][name] = round(_wall_us(repad, 20), 1)
        prev = L.gray_of(synth_frame(2, w, h, "letterbox")[0])
        t0 = time.perf_counter()
        for _ in range(3):
            st = L.frame_stats(f, prev)
            L.scene_cut(prev, st.gray)
            L.bars_of_frame(f)
        res["oracle_ms"][name] = round((time.perf_counter() - t0) / 3 * 1000, 1)
        RD.load_depth_model(arch, width=w, height=h, seed=0)
        frames = [synth_frame(i, w, h, "letterbox")[0] for i in range(args.frames)]
        out = {}
        for mode in ("off", "on", "off2", "on2"):
            tr = None
            if mode.startswith("on"):
                tr = RD.LetterboxTracker(h, 24)
            list(RD.iter_depth_frames(_Cap(frames[:8]), w, h, batch_size=8, tracker=tr))  # warm
            t0 = time.perf_counter()
            k = sum(1 for _ in RD.iter_depth_frames(_Cap(frames), w, h, batch_size=8, tracker=tr))
            out[mode] = (time.perf_counter() - t0) / k * 1000
        off, on = min(out["off"], out["off2"]), min(out["on"], out["on2"])
        res["video_ms"][f"{name}_{arch}"] = {"off": round(off, 2), "on": round(on, 2),
                                             "overhead_pct": round(100 * (on / off - 1), 1)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
