"""Per-kernel split of the bench step on ONE stream (torch.profiler, a run of its own).

    python scripts/gpu_step_split.py [--root DIR] [--steps K]

Runs the bench workload (8 pairs of 64 x 2048, 4 rotating input sets, pipeline on one stream) and prints the mean
device time per step of every kernel, plus the one-stream step time from CUDA events in a separate, unprofiled pass.
--root imports the package from another checkout (to set two builds side by side in one run).
"""
import argparse
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--steps", type=int, default=50)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from delora_b200 import synthetic  # noqa: E402
from delora_b200.pipeline import ScanPairPipeline  # noqa: E402

B, H, W, ROT = 8, 64, 2048, 4
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.strip()
print("gpu:", q, "| root:", os.path.abspath(args.root))
cfg = synthetic.fov_config(h=H, w=W)
hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
raw = [synthetic.make_pair(i, w_raw=2048) for i in range(B * ROT)]
nmax = max(max(p[0].shape[1], p[1].shape[1]) for p in raw)
pipes = []
for s in range(ROT):
    p = ScanPairPipeline(B, nmax, H, W, hf, vf, concurrency=1)
    sub = raw[s * B:(s + 1) * B]
    p.load([x[0] for x in sub], [x[1] for x in sub], torch.stack([x[3] for x in sub]))
    pipes.append(p)
for i in range(10):
    pipes[i % ROT].step()
torch.cuda.synchronize()

K = args.steps
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for i in range(K):
    pipes[i % ROT].step()
e1.record()
torch.cuda.synchronize()
print(f"one-stream step {e0.elapsed_time(e1) / K * 1e3:.1f} us")

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for i in range(K):
        pipes[i % ROT].step()
    torch.cuda.synchronize()
rows = []
for e in prof.key_averages():
    us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    if us > 0:
        rows.append((e.key.split("(")[0].split("<")[0].replace("void ", "").replace("delora::", ""), us / K, e.count / K))
for name, us, n in sorted(rows, key=lambda r: -r[1]):
    print(f"  {name:40s} {us:8.1f} us/step  ({n:.0f} launches/step)")
print(f"  {'sum':40s} {sum(r[1] for r in rows):8.1f} us/step")
print("losses[0]", pipes[(K - 1) % ROT].losses[0].tolist())
