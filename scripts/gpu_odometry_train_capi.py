"""Time the C training step (delora_odometry_train_step) against SyntheticTrainStep on the same scans, on one GPU.

BASELINE config #3's shape: B = 16 pairs of 64 x 2048 range images, tanh, two heads, layers [2, 2, 2, 2].  Both paths
start from the same weights and step on the same pairs.  End-to-end: CUDA events around each step, after warm-up,
the two paths alternating for `--rounds` rounds.  Then, in a separate torch.profiler pass, the per-kernel time of the
kernels this path adds (the tail backward, Adam, the ICP scratch re-arm) against their byte floor at 3.35 TB/s
(H100 SXM data sheet HBM3 bandwidth).  Prints the card name, power limit and SM clock of the run.

    python scripts/gpu_odometry_train_capi.py [--batch 16] [--rounds 10] [--out DIR]

Prints the result as JSON; with --out it is also written to DIR/odometry_train_capi.json.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12
NEW_KERNELS = ("odometry_out_bwd_kernel", "odometry_linear_bwd_kernel", "odometry_adam_kernel",
               "odometry_icp_rearm_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--h", type=int, default=64)
    ap.add_argument("--w", type=int, default=2048)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for odometry_train_capi.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    from delora_b200 import _lib, synthetic
    from delora_b200.deploy import export
    from delora_b200.train_step import SyntheticTrainStep
    dev = torch.device("cuda:0")
    b = a.batch
    scans = []
    for i in range(b):
        s1, s2, _, _ = synthetic.make_pair(i, w_raw=a.w, rings=a.h)
        scans.append((s1, s2))
    n_max = max(max(x.shape[1], y.shape[1]) for x, y in scans)
    allsc = [s[0] for s in scans] + [s[1] for s in scans]
    pts = torch.zeros((2 * b, 3, n_max), dtype=torch.float32)
    for i, s in enumerate(allsc):
        pts[i, :, :s.shape[1]] = s
    counts = torch.tensor([s.shape[1] for s in allsc], dtype=torch.int32)
    pts, counts = pts.to(dev), counts.to(dev)

    cfg = synthetic.fov_config(h=a.h, w=a.w, device="cuda:0")
    torch.manual_seed(0)
    py = SyntheticTrainStep(cfg, b, n_max)
    py.load(pts, counts)
    cfg = py.cfg
    L = _lib.lib()
    d = export.desc_from_config(cfg, "kitti", n_max, b)
    dp = ctypes.byref(d)
    nb = cfg["kitti"]["neighborhood_side_length"]
    hp = _lib.OdometryTrainParams(lr=py.optimizer.param_groups[0]["lr"], beta1=0.9, beta2=0.999, eps=1e-8,
                                  lambda_po2pl=cfg["lambda_po2pl"], loss_flags=2 | 4, nb_h=nb[0], nb_w=nb[1],
                                  epsilon_range=cfg["epsilon_range"],
                                  min_neighbors=cfg["min_num_points_in_neighborhood_to_determine_point_class"])
    blob = torch.from_numpy(export.pack_state_dict(py.model.state_dict(), cfg)).to(dev)
    ws_bytes = int(L.delora_odometry_train_workspace_bytes(dp))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(L.delora_odometry_train_init(dp, blob.data_ptr(), ws.data_ptr(), st()), "train_init")

    def c_step(bsz=b):
        _lib.check(L.delora_odometry_train_step(dp, ctypes.byref(hp), pts.data_ptr(), counts.data_ptr(), bsz,
                                                ws.data_ptr(), None, None, None, None, st()), "train_step")

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    for _ in range(a.warmup):
        c_step()
        py.step()
    torch.cuda.synchronize()
    t_c, t_py = [], []
    for _ in range(a.rounds):
        t_c.append(timed(c_step))
        t_py.append(timed(py.step))
    res = {"card": card(), "batch": b, "H": a.h, "W": a.w, "workspace_bytes": ws_bytes,
           "c_step_ms": {"median": statistics.median(t_c), "min": min(t_c), "max": max(t_c)},
           "synthetic_train_step_ms": {"median": statistics.median(t_py), "min": min(t_py), "max": max(t_py)}}

    # per-kernel times in a separate, profiled pass; the re-arm kernel once with an unchanged B (every CTA exits) and
    # once after a step with another B (it zeroes the ICP scratch)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            c_step()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if ev.key in NEW_KERNELS or any(ev.key.startswith(k) or k in ev.key for k in NEW_KERNELS):
            name = next(k for k in NEW_KERNELS if k in ev.key)
            kernels[name] = {"us_per_call": ev.device_time_total / max(ev.count, 1), "calls_per_step": ev.count / 5}
    with profile(activities=[ProfilerActivity.CUDA]) as prof2:
        for _ in range(3):
            c_step(b)
            c_step(b - 1)
        torch.cuda.synchronize()
    for ev in prof2.key_averages():
        if "odometry_icp_rearm_kernel" in ev.key:
            kernels["odometry_icp_rearm_kernel (B alternating)"] = {"us_per_call": ev.device_time_total / max(ev.count, 1)}
    c_step(b)
    torch.cuda.synchronize()
    n = int(L.delora_odometry_weight_floats(dp))
    floors = {"odometry_adam_kernel": n * 28, "odometry_icp_rearm_kernel (B alternating)":
              int(L.delora_icp_scratch_floats(b, a.h * a.w)) * 4}
    for k, v in kernels.items():
        if k in floors:
            v["bytes"] = floors[k]
            v["floor_us"] = floors[k] / HBM_BYTES_PER_S * 1e6
    res["kernels"] = kernels
    res["new_kernels_us_per_step"] = sum(v["us_per_call"] * v.get("calls_per_step", 0) for v in kernels.values())
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "odometry_train_capi.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
