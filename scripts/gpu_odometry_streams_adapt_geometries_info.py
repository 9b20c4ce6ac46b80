"""What serving each frame's ICP information costs the adapting streams of several sensor geometries: one
delora_odometry_streams_push_adapt_geometries tick against one delora_odometry_streams_push_adapt_geometries_info tick on
the same frames.

Workload of gpu_odometry_streams_adapt_geometries.py: 64 x 720 with w_pre 2250 (KITTI's recipe) and 64 x 512 with
w_pre 512, S_g streams each for S_g = 1 and 4, every stream active and alternating between the two scans of a synthetic
pair, a near-identity model and lr 0 (Adam runs, the weights stay put).  For each S_g and each value of update, one
captured graph holds two ticks of each workspace; the graphs alternate and the paired differences are reported with
their median.  Both workspaces hold the same weights and frames, so the only difference is the information operator in
place of the ICP and the copy of the rows.

The card's name, power limit and SM clocks are read in the same run.  Writes odometry_streams_adapt_geometries_info.json
to --out.

    python scripts/gpu_odometry_streams_adapt_geometries_info.py [--seconds 0.5] [--samples 7] [--out DIR]
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
    """One captured graph of two fleet ticks with `update`, with or without the information."""

    def __init__(self, cfg, blob, pairs, n_stride, S, update, info):
        self.descs = [geom_desc(cfg, h, w, wp, n_stride, S) for h, w, wp in GEOMS]
        hp = capi.train_params(cfg, 0.0)
        n = len(GEOMS)
        # geometry g's streams serve pairs g * S .. g * S + S - 1
        self.frames = [[staged([p[i] for p in pairs[g * S:(g + 1) * S]], n_stride) for g in range(n)] for i in (0, 1)]
        kind = capi.GeometriesAdaptingInformationStreamsWorkspace if info else capi.GeometriesAdaptingStreamsWorkspace
        self.ws = kind(self.descs, blob, hp)
        self.bytes = kind.shared_bytes(self.descs)
        self.update = update
        self.out = (torch.zeros((n * S, 16), dtype=torch.float32, device=DEV),
                    torch.zeros((n * S,), dtype=torch.int32, device=DEV),
                    torch.zeros((n * S, ops.LOSS_ROW), dtype=torch.float32, device=DEV))
        if info:
            self.out += (torch.zeros((n * S, ops.INFO_ROW), dtype=torch.float32, device=DEV),)
        self.active = torch.ones((n * S,), dtype=torch.int32, device=DEV)
        self.graph = capture(self.ticks, warmup=1)            # the warm-up caches the first frames

    def ticks(self):
        for fr in self.frames:
            self.ws.push([f[0] for f in fr], [f[1] for f in fr], self.active, *self.out, update=self.update)



def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=7)
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
            plain = Ticks(cfg, blob, pairs_all, stride, S, bool(update), False)
            info = Ticks(cfg, blob, pairs_all, stride, S, bool(update), True)
            t = alternate({"plain": plain.graph.replay, "info": info.graph.replay}, args.samples,
                          lambda fn: host_ms(fn, args.seconds, (DEV,), every=4, warmup=4) / 2)    # two ticks per replay
            xs, ys = t["plain"], t["info"]
            diffs, diff = paired(xs, ys)
            same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(plain.out[1:3], info.out[1:3]))
            row[f"update{update}"] = {
                "push_adapt_geometries_ms_per_tick": statistics.median(xs),
                "push_adapt_geometries_info_ms_per_tick": statistics.median(ys),
                "paired_difference_ms": diff, "plain_samples_ms": xs, "info_samples_ms": ys,
                "paired_differences_ms": diffs, "all_valid": bool(info.out[1].all()),
                "valid_and_losses_bit_identical": bool(same),
                "info_rows_with_pairs": int((info.out[3][:, 78] > 0).sum())}
            row["push_adapt_geometries_workspace_mib"] = plain.bytes / 2 ** 20
            row["push_adapt_geometries_info_workspace_mib"] = info.bytes / 2 ** 20
            del plain, info
            torch.cuda.empty_cache()
        res["streams_per_geometry"][S] = row
    res["gpu_after"] = gpu_info()
    emit(res, args.out and os.path.join(args.out, "odometry_streams_adapt_geometries_info.json"))


if __name__ == "__main__":
    main()
