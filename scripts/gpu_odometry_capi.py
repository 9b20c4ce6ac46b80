"""Per-frame latency of odometry through the C ABI at 64 x 2048 (BASELINE config #5's shape), next to OdometryStream.

Host to host per frame: pinned H2D of the scan and its count, delora_odometry_push (eager, then one captured call
replayed as a CUDA graph), D2H of T, synchronise.  OdometryStream.push (its own CUDA graph, torch heads) runs in the
same process on the same frames.  Then torch.profiler splits one push into kernels and the fully connected tail
(odometry_linear_kernel + odometry_out_kernel) is set against its weight-byte floor at the data-sheet HBM rate.
The card's name, power limit and SM clock are read in the same run.

    python scripts/gpu_odometry_capi.py [--frames 300] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from delora_b200 import synthetic  # noqa: E402
from delora_b200.deploy import export  # noqa: E402
from delora_b200.deploy.capi import InferenceWorkspace  # noqa: E402
from delora_b200.deploy.stream import OdometryStream  # noqa: E402
from delora_b200.models.model import OdometryModel  # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable"


def pct(ts, p):
    return float(np.percentile(np.array(ts) * 1e6, p))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = "cuda:0"
    h, w = 64, 2048
    cfg = synthetic.fov_config(h=h, w=w, device=dev)
    cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                "use_dropout": False})
    torch.manual_seed(0)
    model = OdometryModel(cfg).to(dev).eval()
    scans = []
    for i in range(3):
        s1, s2, _, _ = synthetic.make_pair(i, w_raw=2048, rings=64)
        scans += [s1, s2]
    n_stride = max(s.shape[1] for s in scans)
    info_before = gpu_info()

    res = {"gpu_before": info_before, "H": h, "W": w, "n_stride": n_stride}
    for mb in (1, 16):
        dd = export.desc_from_config(cfg, "kitti", n_stride, mb)
        res[f"workspace_bytes_max_batch_{mb}"] = InferenceWorkspace.workspace_bytes(dd)
    st = torch.cuda.current_stream()
    blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), cfg)).to(dev)
    ws = InferenceWorkspace(export.desc_from_config(cfg, "kitti", n_stride, 1), blob)

    host_pts = torch.zeros((len(scans), 3, n_stride), dtype=torch.float32).pin_memory()
    host_cnt = torch.zeros((len(scans),), dtype=torch.int32).pin_memory()
    for i, s in enumerate(scans):
        host_pts[i, :, :s.shape[1]] = s
        host_cnt[i] = s.shape[1]
    pts = torch.zeros((1, 3, n_stride), dtype=torch.float32, device=dev)
    cnt = torch.zeros((1,), dtype=torch.int32, device=dev)
    t_dev = torch.zeros((16,), dtype=torch.float32, device=dev)
    t_host = torch.zeros((16,), dtype=torch.float32).pin_memory()

    def upload(k):
        pts.copy_(host_pts[k % len(scans)][None], non_blocking=True)
        cnt.copy_(host_cnt[k % len(scans)][None], non_blocking=True)

    def push(k, first=False):
        upload(k)
        ws.push(pts, cnt, None if first else t_dev)

    def timed(step, n):
        ts = []
        for k in range(n):
            t0 = time.perf_counter()
            step(k)
            t_host.copy_(t_dev, non_blocking=True)
            st.synchronize()
            ts.append(time.perf_counter() - t0)
        return ts

    push(0, first=True)
    for k in range(1, 20):
        push(k)
    st.synchronize()
    eager = timed(lambda k: push(k + 1), args.frames)

    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ws.push(pts, cnt, t_dev)

    def replay(k):
        upload(k)
        graph.replay()
    for k in range(20):
        replay(k)
    st.synchronize()
    graphed = timed(replay, args.frames)

    stream = OdometryStream(model, cfg, "kitti", n_stride)
    stream.push(scans[0])
    for k in range(1, 20):
        stream.push(scans[k % len(scans)])
    ts_stream = []
    for k in range(args.frames):
        t0 = time.perf_counter()
        stream.push(scans[(k + 1) % len(scans)])
        ts_stream.append(time.perf_counter() - t0)

    # one-frame parity against the stream (same model, same pair of frames)
    stream2 = OdometryStream(model, cfg, "kitti", n_stride)
    stream2.push(scans[0])
    t_ref = torch.from_numpy(stream2.push(scans[1])[0]).reshape(16)
    push(0, first=True)
    push(1)
    st.synchronize()
    res["max_abs_T_diff_vs_stream"] = float((t_dev.cpu() - t_ref).abs().max())

    for name, ts in (("capi_push_eager", eager), ("capi_push_graph", graphed), ("odometry_stream_push", ts_stream)):
        res[name] = {"p50_us": pct(ts, 50), "p99_us": pct(ts, 99), "frames": len(ts)}

    # per-kernel split of the graph-replayed push
    from torch.profiler import ProfilerActivity, profile
    n_prof = 50
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(n_prof):
            push(k + 1)
        st.synchronize()
    kernels = {}
    for e in prof.events():
        if "cuda" in str(e.device_type).lower():          # kernels and copies on the device timeline
            kernels[e.name] = kernels.get(e.name, 0.0) + e.time_range.elapsed_us() / n_prof
    tail_us = sum(v for k, v in kernels.items() if "odometry_linear_kernel" in k or "odometry_out_kernel" in k)
    res["per_push_kernels_us"] = dict(sorted(kernels.items(), key=lambda kv: -kv[1])[:20])
    tail_floats = 512 * 1000 + 1000 + 2 * (1000 * 100 + 100) + 4 * 100 + 4 + 3 * 100 + 3
    floor_us = tail_floats * 4 / HBM_BYTES_PER_S * 1e6
    res["tail"] = {"kernel_us": tail_us, "weight_bytes": tail_floats * 4, "hbm_floor_us": floor_us,
                   "share_of_floor": floor_us / tail_us if tail_us > 0 else None}
    res["gpu_after"] = gpu_info()
    line = json.dumps(res, indent=1)
    print(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line)


if __name__ == "__main__":
    main()
