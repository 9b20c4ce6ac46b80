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
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from delora_b200 import ops  # noqa: E402
from delora_b200.deploy import capi  # noqa: E402
from measure import (DEV, GEOMS, GEOMS_STREAMS, GPU_QUERY, alternate, capture, emit, geom_desc, gpu_info,  # noqa: E402
                     host_ms, model_config, n_stride, near_identity_blob, paired, pairs, staged)

class Ticks:
    """One captured graph of two ticks with `update`: the fleet workspace, or both single-geometry workspaces."""

    def __init__(self, cfg, blob, pairs, n_stride, S, update, fleet):
        self.descs = [geom_desc(cfg, h, w, wp, n_stride, S) for h, w, wp in GEOMS]
        hp = capi.train_params(cfg, 0.0)
        n = len(GEOMS)
        # geometry g's streams serve pairs g * S .. g * S + S - 1
        self.frames = [[staged([p[i] for p in pairs[g * S:(g + 1) * S]], n_stride) for g in range(n)] for i in (0, 1)]
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
        self.graph = capture(self.ticks, warmup=1)            # the warm-up caches the first frames

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



def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": GPU_QUERY,
           "geometries": [f"{h}x{w}_wpre{wp}" for h, w, wp in GEOMS], "lr": 0.0,
           "seconds_per_sample": args.seconds, "streams_per_geometry": {}}
    cfg = model_config(GEOMS[0][0], GEOMS[0][1])
    blob = near_identity_blob(cfg)
    pairs_all = pairs(64, len(GEOMS) * max(GEOMS_STREAMS))
    stride = n_stride(pairs_all)
    for S in GEOMS_STREAMS:
        row = {}
        for update in (0, 1):
            fleet = Ticks(cfg, blob, pairs_all, stride, S, bool(update), True)
            pair = Ticks(cfg, blob, pairs_all, stride, S, bool(update), False)
            t = alternate({"pair": pair.graph.replay, "fleet": fleet.graph.replay}, args.samples,
                          lambda fn: host_ms(fn, args.seconds, (DEV,), every=4, warmup=4) / 2)    # two ticks per replay
            xs, ys = t["pair"], t["fleet"]
            diffs, diff = paired(xs, ys)
            row[f"update{update}"] = {
                "fleet_ms_per_tick": statistics.median(ys), "two_push_adapt_ms_per_tick": statistics.median(xs),
                "paired_difference_ms": diff, "fleet_samples_ms": ys, "two_samples_ms": xs,
                "paired_differences_ms": diffs, "all_valid": bool(fleet.out[1].all()),
                "fleet_step_count": int(fleet.ws[0].get_state()[3][0])}
            row["fleet_workspace_mib"] = fleet.bytes / 2 ** 20
            row["two_workspaces_mib"] = pair.bytes / 2 ** 20
            del fleet, pair
            torch.cuda.empty_cache()
        res["streams_per_geometry"][S] = row
    res["gpu_after"] = gpu_info()
    emit(res, args.out and os.path.join(args.out, "odometry_streams_adapt_geometries.json"))


if __name__ == "__main__":
    main()
