"""Per-frame latency of odometry through the C ABI at 64 x 2048 (BASELINE config #5's shape), next to OdometryStream.

Host to host per frame: pinned H2D of the scan and its count, delora_odometry_push (eager, then one captured call
replayed as a CUDA graph), D2H of T, synchronise.  OdometryStream.push (its own CUDA graph, torch heads) runs in the
same process on the same frames.  Then torch.profiler splits one push into kernels and the fully connected tail
(odometry_linear_kernel + odometry_out_kernel) is set against its weight-byte floor at the data-sheet HBM rate.
The card's name, power limit and SM clock are read in the same run.

    python scripts/gpu_odometry_capi.py [--frames 300] [--json out.json]
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from delora_b200.deploy import export  # noqa: E402
from delora_b200.deploy.capi import InferenceWorkspace  # noqa: E402
from delora_b200.deploy.stream import OdometryStream  # noqa: E402
from delora_b200.models.model import OdometryModel  # noqa: E402
from measure import DEV, capture, emit, gpu_info, model_config, n_stride, pairs, staged  # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def pct(ts, p):
    return float(np.percentile(np.array(ts) * 1e6, p))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    h, w = 64, 2048
    cfg = model_config(h, w)
    torch.manual_seed(0)
    model = OdometryModel(cfg).to(DEV).eval()
    ps = pairs(64, 3)
    scans = [s for p in ps for s in p]
    stride = n_stride(ps)

    res = {"gpu_before": gpu_info(), "H": h, "W": w, "n_stride": stride}
    for mb in (1, 16):
        dd = export.desc_from_config(cfg, "kitti", stride, mb)
        res[f"workspace_bytes_max_batch_{mb}"] = InferenceWorkspace.workspace_bytes(dd)
    st = torch.cuda.current_stream()
    blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), cfg)).to(DEV)
    ws = InferenceWorkspace(export.desc_from_config(cfg, "kitti", stride, 1), blob)

    # every frame is uploaded from pinned host memory, as a caller's would be
    host_pts, host_cnt = (t.cpu().pin_memory() for t in staged(scans, stride))
    pts = torch.zeros((1, 3, stride), dtype=torch.float32, device=DEV)
    cnt = torch.zeros((1,), dtype=torch.int32, device=DEV)
    t_dev = torch.zeros((16,), dtype=torch.float32, device=DEV)
    t_host = torch.zeros((16,), dtype=torch.float32).pin_memory()

    def upload(k):
        pts.copy_(host_pts[k % len(scans)][None], non_blocking=True)
        cnt.copy_(host_cnt[k % len(scans)][None], non_blocking=True)

    def push(k, first=False):
        upload(k)
        ws.push(pts, cnt, None if first else t_dev)

    def latencies(step, n):
        """Seconds from each frame's upload to its T on the host."""
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
    eager = latencies(lambda k: push(k + 1), args.frames)

    graph = capture(lambda: ws.push(pts, cnt, t_dev), warmup=0)

    def replay(k):
        upload(k)
        graph.replay()
    for k in range(20):
        replay(k)
    st.synchronize()
    graphed = latencies(replay, args.frames)

    stream = OdometryStream(model, cfg, "kitti", stride)
    stream.push(scans[0])
    for k in range(1, 20):
        stream.push(scans[k % len(scans)])
    ts_stream = []
    for k in range(args.frames):
        t0 = time.perf_counter()
        stream.push(scans[(k + 1) % len(scans)])
        ts_stream.append(time.perf_counter() - t0)

    # one-frame parity against the stream (same model, same pair of frames)
    stream2 = OdometryStream(model, cfg, "kitti", stride)
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
    emit(res, args.json)


if __name__ == "__main__":
    main()
