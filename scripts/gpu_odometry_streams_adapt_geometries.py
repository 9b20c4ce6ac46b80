"""What adapting one model from the streams of two sensor geometries in one workspace
(delora_odometry_streams_push_adapt_geometries) costs, against the two single-geometry _push_adapt workspaces a host
would otherwise tick one after the other.

Geometries: 64 x 720 with w_pre 2250 (KITTI's recipe) and 64 x 512 with w_pre 512, S_g streams each for S_g = 1 and 4,
every stream active and alternating between the two scans of a synthetic pair, a near-identity model and lr 0 (Adam
runs, the weights stay put).  For each S_g and each value of update, one captured graph holds two fleet ticks and
another holds two ticks of each single-geometry workspace (geometry 0's, then geometry 1's); the graphs alternate and
the paired differences are reported with their median.  The two-workspace composition is not one model: each
workspace steps its own copy, which is why the memory of both is reported beside the fleet workspace's.

The card's name, power limit and SM clocks are read in the same run.  Writes odometry_streams_adapt_geometries.json to
--out.

    python scripts/gpu_odometry_streams_adapt_geometries.py [--seconds 0.5] [--samples 5] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from delora_b200 import ops, synthetic  # noqa: E402
from delora_b200.deploy import capi, export  # noqa: E402
from gpu_odometry_eval import near_identity_blob  # noqa: E402
from gpu_odometry_streams import DEV, gpu_info, staged  # noqa: E402

GEOMS = ((64, 720, 2250), (64, 512, 512))
STREAMS = (1, 4)


def _desc(cfg, h, w, w_pre, n_stride, S):
    c = dict(cfg, kitti=dict(cfg["kitti"], vertical_cells=h, horizontal_cells=w))
    d = export.desc_from_config(c, "kitti", n_stride, S)
    d.w_pre = w_pre
    return d


class Ticks:
    """One captured graph of two ticks with `update`: the fleet workspace, or both single-geometry workspaces."""

    def __init__(self, cfg, blob, pairs, n_stride, S, update, fleet):
        self.descs = [_desc(cfg, h, w, wp, n_stride, S) for h, w, wp in GEOMS]
        hp = capi.train_params(cfg, 0.0)
        n = len(GEOMS)
        # geometry g's streams serve pairs g * S .. g * S + S - 1
        self.frames = [[staged([p[i] for p in pairs[g * S:(g + 1) * S]], n_stride) for g in range(n)] for i in (0, 1)]
        self.frames = [[tuple(t.to(DEV) for t in f) for f in fr] for fr in self.frames]
        if fleet:
            self.ws = [capi.GeometriesAdaptingStreamsWorkspace(self.descs, blob, hp)]
            self.bytes = capi.GeometriesAdaptingStreamsWorkspace.shared_bytes(self.descs)
        else:
            self.ws = [capi.AdaptiveStreamsWorkspace(d, blob, hp) for d in self.descs]
            self.bytes = sum(capi.AdaptiveStreamsWorkspace.workspace_bytes(d) for d in self.descs)
        self.fleet, self.update, self.n, self.S = fleet, update, n, S
        self.out = (torch.zeros((n * S, 16), dtype=torch.float32, device=DEV),
                    torch.zeros((n * S,), dtype=torch.int32, device=DEV),
                    torch.zeros((n * S, ops.LOSS_ROW), dtype=torch.float32, device=DEV))
        self.active = torch.ones((n * S,), dtype=torch.int32, device=DEV)
        self.ticks()                                          # warm-up: the first frames, and every launcher
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.ticks()
        torch.cuda.synchronize()

    def ticks(self):
        T, valid, losses = self.out
        S = self.S
        for fr in self.frames:
            if self.fleet:
                self.ws[0].push([f[0] for f in fr], [f[1] for f in fr], self.active, T, valid, losses,
                                update=self.update)
                continue
            for g, ws in enumerate(self.ws):
                r = slice(g * S, (g + 1) * S)
                ws.push(fr[g][0], fr[g][1], self.active[r], T[r], valid[r], losses[r], update=self.update)

    def time(self, seconds):
        """ms per tick (host clock around synchronised replays of two ticks), over >= `seconds`."""
        for _ in range(4):
            self.graph.replay()
        torch.cuda.synchronize()
        n, t0 = 0, time.perf_counter()
        while True:
            self.graph.replay()
            n += 1
            if n % 4 == 0:
                torch.cuda.synchronize()
                el = time.perf_counter() - t0
                if el >= seconds:
                    return el * 1e3 / n / 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": "name, power.limit, clocks.sm, clocks.max.sm",
           "geometries": [f"{h}x{w}_wpre{wp}" for h, w, wp in GEOMS], "lr": 0.0,
           "seconds_per_sample": args.seconds, "streams_per_geometry": {}}
    cfg = synthetic.fov_config(h=GEOMS[0][0], w=GEOMS[0][1], device=DEV)
    cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                "use_dropout": False})
    blob = near_identity_blob(cfg)
    pairs_all = [synthetic.make_pair(i, w_raw=2048, rings=64)[:2] for i in range(len(GEOMS) * max(STREAMS))]
    n_stride = max(max(a.shape[1], b.shape[1]) for a, b in pairs_all)
    for S in STREAMS:
        row = {}
        for update in (0, 1):
            fleet = Ticks(cfg, blob, pairs_all, n_stride, S, bool(update), True)
            pair = Ticks(cfg, blob, pairs_all, n_stride, S, bool(update), False)
            xs, ys = [], []
            for _ in range(args.samples):
                xs.append(pair.time(args.seconds))
                ys.append(fleet.time(args.seconds))
            diffs = [y - x for x, y in zip(xs, ys)]
            row[f"update{update}"] = {
                "fleet_ms_per_tick": statistics.median(ys), "two_push_adapt_ms_per_tick": statistics.median(xs),
                "paired_difference_ms": statistics.median(diffs), "fleet_samples_ms": ys, "two_samples_ms": xs,
                "paired_differences_ms": diffs, "all_valid": bool(fleet.out[1].all()),
                "fleet_step_count": int(fleet.ws[0].get_state()[3][0])}
            row["fleet_workspace_mib"] = fleet.bytes / 2 ** 20
            row["two_workspaces_mib"] = pair.bytes / 2 ** 20
            del fleet, pair
            torch.cuda.empty_cache()
        res["streams_per_geometry"][S] = row
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "odometry_streams_adapt_geometries.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
