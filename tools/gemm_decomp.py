"""Time decomposition of the token GEMMs of the batched DA-V2 forward (k_umma_gemm<128,4>, vd3d_gemm_bench):
   python tools/gemm_decomp.py [M] [iters]      (M defaults to 10123 = the token rows of a 4-frame 518 x 924 batch)

Each shape runs in three modes of the kernel's tuning hook:
  full      the launch as the forward runs it;
  no-epi    the epilogue warpgroup only releases the staging tile (mainloop + hand-off);
  no-tma    no operand loads (tensor-core issue rate with the epilogue).
fc1 runs the bias + GELU epilogue, proj / fc2 the fp32 LayerScale + residual read-modify-write, and QKV the plain
f16 epilogue as a proxy (the hook has no head split)."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from visiondepth3d_b200.depth_engine import DepthEngine  # noqa: E402

RESID = 0x100
GELU = 1
# (model, name, N, K, act) of the per-layer token GEMMs
SHAPES = [
    ("vitb", "qkv", 2304, 768, 0), ("vitb", "proj", 768, 768, RESID),
    ("vitb", "fc1", 3072, 768, GELU), ("vitb", "fc2", 768, 3072, RESID),
    ("vitl", "qkv", 3072, 1024, 0), ("vitl", "proj", 1024, 1024, RESID),
    ("vitl", "fc1", 4096, 1024, GELU), ("vitl", "fc2", 1024, 4096, RESID),
]
MODES = [("full", 0), ("no-epi", 4), ("no-tma", 2)]


def main():
    M = int(sys.argv[1]) if len(sys.argv) > 1 else 10123
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 50
    e = DepthEngine("vits", 70, 98)
    print(f"k_umma_gemm<128,4>, M = {M}, {iters} launches per mode: us per launch (TFLOP/s)")
    print(f"{'shape':22s}" + "".join(f"{m:>22s}" for m, _ in MODES) + f"{'full - no-epi':>16s}")
    for model, name, N, K, act in SHAPES:
        flop = 2.0 * M * N * K
        us = {}
        for mode, dbg in MODES:
            us[mode] = e.gemm_bench(M, N, K, variant=0, dbg=dbg, act=act, iters=iters) * 1e3
        cells = "".join(f"{us[m]:12.1f} ({flop / us[m] / 1e6:6.1f})" for m, _ in MODES)
        print(f"{model} {name:4s} {N:5d}x{K:<5d}    {cells}{us['full'] - us['no-epi']:14.1f}")
    e.close()


if __name__ == "__main__":
    main()
