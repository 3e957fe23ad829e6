"""Depth stage only: batched DA-V2 forward on synthetic frames (a profiler target for the wgmma kernels).
   python tools/depth_only.py [vitb|vitl|vits] [batch] [reps]"""
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402
from transformers import DepthAnythingForDepthEstimation  # noqa: E402

from visiondepth3d_b200.depth_engine import DepthEngine  # noqa: E402
from visiondepth3d_b200.depth_weights import hf_config  # noqa: E402
from visiondepth3d_b200.synth import synth_frame  # noqa: E402

arch = sys.argv[1] if len(sys.argv) > 1 else "vitb"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 3
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
torch.manual_seed(0)
sd = DepthAnythingForDepthEstimation(hf_config(arch)).eval().state_dict()
e = DepthEngine(arch, 518, 924)
e.load_state_dict(sd)
frames = [synth_frame(i, 1920, 1080, "natural")[0] for i in range(B)]
for r in range(reps):
    t0 = time.perf_counter()
    e.infer_batch(frames)
    print(f"{arch} batch {B} rep {r}: {(time.perf_counter() - t0) * 1e3 / B:.3f} ms/frame (host-buffer API, synchronous)")
