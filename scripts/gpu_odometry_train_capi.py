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
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import DEV, alternate, emit, events_ms, gpu_info, n_stride, staged, summary  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
NEW_KERNELS = ("odometry_out_bwd_kernel", "odometry_linear_bwd_kernel", "odometry_adam_kernel",
               "odometry_icp_rearm_kernel")


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
    from delora_b200.deploy import capi, export
    from delora_b200.train_step import SyntheticTrainStep
    b = a.batch
    scans = [synthetic.make_pair(i, w_raw=a.w, rings=a.h)[:2] for i in range(b)]
    n_max = n_stride(scans)
    pts, counts = staged([s[0] for s in scans] + [s[1] for s in scans], n_max)

    cfg = synthetic.fov_config(h=a.h, w=a.w, device=DEV)
    torch.manual_seed(0)
    py = SyntheticTrainStep(cfg, b, n_max)
    py.load(pts, counts)
    cfg = py.cfg
    blob = torch.from_numpy(export.pack_state_dict(py.model.state_dict(), cfg)).to(DEV)
    tr = capi.TrainingWorkspace(export.desc_from_config(cfg, "kitti", n_max, b), blob,
                                capi.train_params(cfg, py.optimizer.param_groups[0]["lr"]))
    ws_bytes = tr.workspace.numel()

    def c_step(bsz=b):
        # B = rows // 2: at bsz < b the step reads the buffer's first 2 * bsz rows (they serve the timing only)
        tr.step(pts[:2 * bsz], counts[:2 * bsz], outputs=False)

    for _ in range(a.warmup):
        c_step()
        py.step()
    torch.cuda.synchronize()
    t = alternate({"c": c_step, "py": py.step}, a.rounds, lambda fn: events_ms(fn, calls=1)[0])
    res = {"card": gpu_info(), "batch": b, "H": a.h, "W": a.w, "workspace_bytes": ws_bytes,
           "c_step_ms": summary(t["c"]), "synthetic_train_step_ms": summary(t["py"])}

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
    floors = {"odometry_adam_kernel": tr.n * 28, "odometry_icp_rearm_kernel (B alternating)":
              int(_lib.lib().delora_icp_scratch_floats(b, a.h * a.w)) * 4}
    for k, v in kernels.items():
        if k in floors:
            v["bytes"] = floors[k]
            v["floor_us"] = floors[k] / HBM_BYTES_PER_S * 1e6
    res["kernels"] = kernels
    res["new_kernels_us_per_step"] = sum(v["us_per_call"] * v.get("calls_per_step", 0) for v in kernels.values())
    emit(res, a.out and os.path.join(a.out, "odometry_train_capi.json"))


if __name__ == "__main__":
    main()
