"""What training on several sensor geometries from one workspace costs (delora_odometry_train_geometries_* and
delora_odometry_train_use_geometry).

Two sets of two geometries: 64 x 2048 (KITTI vfov, w_pre 0) with 64 x 720 (KITTI vfov, w_pre 2250), and 64 x 720
(w_pre 2250) with 64 x 512 (vfov +-22.5 degrees, w_pre 512, DARPA's).  For each (max_batch, B) of --configs: the
workspaces sized for max_batch, steps of B pairs of synthetic scans per geometry (the same near-identity model and lr 0
as gpu_odometry_eval.py).  The re-arm zeroes the geometry section, which max_batch sizes, so max_batch 16 at B = 1 is
the case of a checkpoint exported for 16 pairs and trained at the reference's batch size of 1.  Graph-replayed:
  - use_ms: one delora_odometry_train_use_geometry, from a graph of 10 calls alternating between the two geometries;
  - per geometry g, a step right after a switch (a graph of _use_geometry(g) + _train_step) against a steady step (a
    graph of _train_step alone), sampled alternately; the paired differences and their median.
The memory of the shared workspace against the sum of the single-geometry workspaces comes from the host-only size
queries.  The card's name, power limit and SM clocks are read in the same run.  Writes train_geometries.json to --out.

    python scripts/gpu_train_geometries.py [--configs 1:1,4:4,16:16,16:1,16:4] [--seconds 0.2] [--samples 7]
                                           [--out DIR]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from delora_b200 import _lib, synthetic  # noqa: E402
from delora_b200.deploy import capi, export  # noqa: E402
from gpu_odometry_eval import near_identity_blob  # noqa: E402
from gpu_odometry_streams import DEV, gpu_info, staged  # noqa: E402

KITTI = (-24.5, 2.0)
GEOMETRIES = {"64x2048": (64, 2048, KITTI, 0), "64x720_w2250": (64, 720, KITTI, 2250),
              "64x512_w512": (64, 512, (-22.5, 22.5), 512)}
SETS = (("64x2048", "64x720_w2250"), ("64x720_w2250", "64x512_w512"))


def model_config(h, w, vfov):
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov, device=DEV)
    cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                "use_dropout": False})
    return cfg


def geometry(name, B, max_batch):
    """-> (descriptor for max_batch pairs, points, counts) of B synthetic pairs at the geometry."""
    h, w, vfov, w_pre = GEOMETRIES[name]
    pairs = [synthetic.make_pair(i, w_raw=2048, rings=h, vfov_deg=vfov)[:2] for i in range(B)]
    n_stride = max(max(a.shape[1], b.shape[1]) for a, b in pairs)
    d = export.desc_from_config(model_config(h, w, vfov), "kitti", n_stride, max_batch)
    d.w_pre = w_pre
    pts, counts = staged([p[0] for p in pairs] + [p[1] for p in pairs], n_stride)
    return d, pts, counts


def capture(fn):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    return g


def time_graph(g, seconds):
    """ms per replay, device events around at least `seconds` of replays (calibrated on a first short run)."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def run(n):
        start.record()
        for _ in range(n):
            g.replay()
        end.record()
        end.synchronize()
        return start.elapsed_time(end) / n

    n = max(3, int(seconds * 1e3 / max(run(3), 1e-3)))
    return run(n)


def measure(names, max_batch, B, blob, seconds, samples):
    L = _lib.lib()
    geo = [geometry(n, B, max_batch) for n in names]
    descs = [g[0] for g in geo]
    ws = capi.GeometriesTrainingWorkspace(descs, blob, capi.train_params(model_config(64, 720, KITTI), 0.0))
    singles = [int(L.delora_odometry_train_workspace_bytes(ctypes.byref(d))) for d in descs]
    out = {"max_batch": max_batch, "batch": B, "n_stride": [d.n_stride for d in descs],
           "shared_bytes": ws.workspace.numel(), "single_bytes": singles, "sum_single_bytes": sum(singles),
           "shared_MiB": ws.workspace.numel() / 2 ** 20, "sum_single_MiB": sum(singles) / 2 ** 20}
    for g in (1, 0):                                            # warm-up: every geometry's step once, eagerly
        ws.use(g)
        ws.step(geo[g][1], geo[g][2], outputs=False)
    torch.cuda.synchronize()

    def alternate_uses():
        for k in range(10):
            ws.use(k % 2)

    g_use = capture(alternate_uses)
    out["use_samples_ms"] = [time_graph(g_use, seconds) / 10 for _ in range(samples)]
    out["use_ms"] = statistics.median(out["use_samples_ms"])
    for g, name in enumerate(names):
        def switched(g=g):
            ws.use(g)
            ws.step(geo[g][1], geo[g][2], outputs=False)

        def steady(g=g):
            ws.step(geo[g][1], geo[g][2], outputs=False)

        ws.use(g)
        g_switch, g_steady = capture(switched), capture(steady)
        xs, ys = [], []
        for _ in range(samples):
            xs.append(time_graph(g_steady, seconds))
            ys.append(time_graph(g_switch, seconds))
        diffs = [y - x for x, y in zip(xs, ys)]
        out[name] = {"steady_step_ms": statistics.median(xs), "step_after_switch_ms": statistics.median(ys),
                     "paired_difference_ms": statistics.median(diffs), "steady_samples_ms": xs,
                     "after_switch_samples_ms": ys, "paired_differences_ms": diffs}
        del g_switch, g_steady
    del g_use, ws
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="1:1,4:4,16:16,16:1,16:4", help="max_batch:B, comma-separated")
    ap.add_argument("--seconds", type=float, default=0.2)
    ap.add_argument("--samples", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    torch.cuda.set_device(0)
    blob = near_identity_blob(model_config(64, 720, KITTI))
    res = {"gpu_before": gpu_info(), "gpu_query": "name, power.limit, clocks.sm, clocks.max.sm",
           "seconds_per_sample": args.seconds, "geometries": {k: {"H": v[0], "W": v[1], "vfov_deg": v[2],
                                                                  "w_pre": v[3]} for k, v in GEOMETRIES.items()},
           "sets": {}}
    for names in SETS:
        key = " + ".join(names)
        res["sets"][key] = [measure(names, int(mb), int(b), blob, args.seconds, args.samples)
                            for mb, b in (c.split(":") for c in args.configs.split(","))]
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "train_geometries.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
