"""DIBR stage only (no depth engine) on device-resident synthetic frames: a profiler target for the DIBR
kernels.   python tools/dibr_only.py [1080p|4k] [frames] [--eager] [--exact]"""
import ctypes as C
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

import bench  # noqa: E402
from visiondepth3d_b200 import _lib  # noqa: E402
from visiondepth3d_b200 import render_3d as R  # noqa: E402


def main():
    key = sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("-") else "1080p"
    n = int(sys.argv[2]) if len(sys.argv) > 2 and sys.argv[2].isdigit() else 12
    wl = bench.WORKLOADS[key]
    ctx = _lib.Context(0)
    if "--exact" in sys.argv:
        ctx.set_exact(True)
    if "--eager" in sys.argv:
        ctx.check(ctx.lib.vd3d_set_graphs(ctx.h, 0))
    rp = bench.render_params(R, wl)
    pl = R.plan_sizes(wl["w"], wl["h"], rp)
    oshape = R.output_shape(rp, pl)
    dev = torch.device("cuda", 0)
    pool = bench.make_pool(wl, 3)
    f = [torch.from_numpy(a).to(dev) for a, _ in pool]
    d = [torch.from_numpy(b).to(dev) for _, b in pool]
    o = [torch.empty(oshape, dtype=torch.uint8, device=dev) for _ in range(3)]
    idx = [i % 3 for i in range(n)]
    pa = (C.c_void_p * n)(*[f[i].data_ptr() for i in idx])
    pd = (C.c_void_p * n)(*[d[i].data_ptr() for i in idx])
    po = (C.c_void_p * n)(*[o[i].data_ptr() for i in idx])
    torch.cuda.synchronize()
    for rep in range(3):
        t0 = time.perf_counter()
        ctx.check(ctx.lib.vd3d_render_clip(ctx.h, n, pa, pd, 3, wl["h"], wl["w"], C.byref(rp), po, _lib.MEM_DEVICE, None))
        torch.cuda.synchronize()
        print(f"{key} rep {rep}: {n / (time.perf_counter() - t0):.1f} frames/s ({(time.perf_counter() - t0) / n * 1e3:.3f} ms/frame)")


if __name__ == "__main__":
    main()
