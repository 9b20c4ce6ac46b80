"""What the dropouts of a use_dropout model cost in a training step: delora_odometry_train_step with DELORA_TRAIN_DROPOUT
against the same step without it, on one GPU.

Settings: B in {1, 4, 16} pairs at 64 x 720 with w_pre = 2250 (the reference's recipe), and B = 16 at 64 x 2048 with
w_pre = 2250; tanh, two heads, layers [2, 2, 2, 2], synthetic 64-ring scans of 2048 columns, both workspaces from the
same weights.  The heads' last layers are near the identity transform (weights * 0.01, the identity quaternion as
bias), as after the reference's identity pre-training: the dense ICP's search cost depends on T, and dropout changes T,
so with freshly initialised heads the two settings would time different ICP work.  The largest |T_on - T_off| of the
first step is reported.  Each setting's step is captured into a CUDA graph; a sample = CUDA events around `--replays`
back-to-back replays; the flag-on and flag-off graphs alternate for `--rounds` samples each, and the cost of dropout is
the difference of each pair of adjacent samples (median, min, max).  The card's name, power limit and SM clocks are read
in the same run.  Prints the result as JSON; with --out DIR also writes DIR/train_dropout_h100_<power>w.json.

    python scripts/gpu_train_dropout.py [--rounds 15] [--replays 20] [--out profiles]
"""
import argparse
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from measure import (alternate, capture, emit, events_ms, gpu_info, model_config, n_stride,  # noqa: E402
                     near_identity_blob, paired, pairs, staged, summary)

H, W_PRE, W_RAW = 64, 2250, 2048
SETTINGS = [(720, 1), (720, 4), (720, 16), (2048, 16)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for train_dropout_h100_<power>w.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    from delora_b200 import ops
    from delora_b200.deploy import capi, export
    ps = pairs(H, max(b for _, b in SETTINGS))
    n_max = n_stride(ps)
    res = {"card": gpu_info(), "H": H, "w_pre": W_PRE, "scan_columns": W_RAW, "rounds": a.rounds,
           "replays_per_sample": a.replays, "steps": []}

    for w, b in SETTINGS:
        cfg = model_config(H, w)
        blob = near_identity_blob(cfg)
        pts, counts = staged([p[0] for p in ps[:b]] + [p[1] for p in ps[:b]], n_max)
        d = export.desc_from_config(cfg, "kitti", n_max, b)
        d.w_pre = W_PRE
        runs = {}
        for on in (False, True):
            flags = ops.LOSS_PO2PL | ops.LOSS_PL2PL | (ops.TRAIN_DROPOUT if on else 0)
            runs[on] = capi.TrainingWorkspace(d, blob, capi.train_params(cfg, 1e-6, loss_flags=flags))
        t_diff = (runs[True].step(pts, counts)[1] - runs[False].step(pts, counts)[1]).abs().max().item()
        graphs = {}
        for on in (False, True):
            graphs[on] = capture(lambda on=on: runs[on].step(pts, counts, outputs=False), warmup=a.warmup)
            graphs[on].replay()
        torch.cuda.synchronize()
        t = alternate({on: g.replay for on, g in graphs.items()}, a.rounds,
                      lambda fn: events_ms(fn, calls=a.replays)[0])
        deltas, added = paired(t[False], t[True])
        res["steps"].append({"W": w, "B": b, "max_abs_T_on_minus_off": t_diff, "step_ms_off": summary(t[False]),
                             "step_ms_on": summary(t[True]), "added_ms_paired": summary(deltas),
                             "added_percent_median": 100.0 * added / statistics.median(t[False])})
        del runs, graphs
        torch.cuda.empty_cache()

    parts = [p.strip() for p in res["card"].split(",")]
    power = parts[1].split()[0].split(".")[0] if len(parts) > 1 else "unknown"
    emit(res, a.out and os.path.join(a.out, f"train_dropout_h100_{power}w.json"))


if __name__ == "__main__":
    main()
