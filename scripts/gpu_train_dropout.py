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
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, W_PRE, W_RAW = 64, 2250, 2048
SETTINGS = [(720, 1), (720, 4), (720, 16), (2048, 16)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def summary(ts):
    return {"median": statistics.median(ts), "min": min(ts), "max": max(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for train_dropout_h100_<power>w.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    from delora_b200 import ops, synthetic
    from delora_b200.deploy import capi, export
    from delora_b200.models.model import OdometryModel
    dev = torch.device("cuda:0")
    b_max = max(b for _, b in SETTINGS)
    pairs = [synthetic.make_pair(i, w_raw=W_RAW, rings=H)[:2] for i in range(b_max)]
    n_max = max(max(x.shape[1], y.shape[1]) for x, y in pairs)
    res = {"card": card(), "H": H, "w_pre": W_PRE, "scan_columns": W_RAW, "rounds": a.rounds,
           "replays_per_sample": a.replays, "steps": []}

    for w, b in SETTINGS:
        cfg = synthetic.fov_config(h=H, w=w, device="cuda:0")
        cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                    "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                    "use_dropout": False, "lambda_po2pl": 1.0})
        torch.manual_seed(0)
        model = OdometryModel(cfg)
        with torch.no_grad():
            for head, bias in ((model.fully_connected_rotation, [0.0, 0.0, 0.0, 1.0]),
                               (model.fully_connected_translation, [0.0, 0.0, 0.0])):
                head[3].weight.mul_(0.01)
                head[3].bias.copy_(torch.tensor(bias))
        blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), cfg)).to(dev)
        scans = [p[0] for p in pairs[:b]] + [p[1] for p in pairs[:b]]
        pts = torch.zeros((2 * b, 3, n_max), dtype=torch.float32)
        for i, s in enumerate(scans):
            pts[i, :, :s.shape[1]] = s
        counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
        pts, counts = pts.to(dev), counts.to(dev)
        d = export.desc_from_config(cfg, "kitti", n_max, b)
        d.w_pre = W_PRE
        runs = {}
        for on in (False, True):
            flags = ops.LOSS_PO2PL | ops.LOSS_PL2PL | (ops.TRAIN_DROPOUT if on else 0)
            runs[on] = capi.TrainingWorkspace(d, blob, capi.train_params(cfg, 1e-6, loss_flags=flags))
        t_diff = (runs[True].step(pts, counts)[1] - runs[False].step(pts, counts)[1]).abs().max().item()
        for _ in range(a.warmup):
            for on in (False, True):
                runs[on].step(pts, counts, outputs=False)
        torch.cuda.synchronize()
        graphs = {}
        for on in (False, True):
            graphs[on] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[on]):
                runs[on].step(pts, counts, outputs=False)
            graphs[on].replay()
        torch.cuda.synchronize()
        t = {False: [], True: []}
        for _ in range(a.rounds):
            for on in (False, True):
                t[on].append(timed(graphs[on].replay, a.replays))
        deltas = [y - x for x, y in zip(t[False], t[True])]
        off = statistics.median(t[False])
        res["steps"].append({"W": w, "B": b, "max_abs_T_on_minus_off": t_diff, "step_ms_off": summary(t[False]),
                             "step_ms_on": summary(t[True]), "added_ms_paired": summary(deltas),
                             "added_percent_median": 100.0 * statistics.median(deltas) / off})
        del runs, graphs
        torch.cuda.empty_cache()

    if a.out:
        parts = [p.strip() for p in res["card"].split(",")]
        power = parts[1].split()[0].split(".")[0] if len(parts) > 1 else "unknown"
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f"train_dropout_h100_{power}w.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
