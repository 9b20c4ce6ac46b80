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
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from delora_b200 import ops, synthetic  # noqa: E402
from delora_b200.deploy import capi  # noqa: E402
from gpu_odometry_eval import near_identity_blob  # noqa: E402
from gpu_odometry_streams import DEV, gpu_info, staged  # noqa: E402
from gpu_odometry_streams_adapt_geometries import GEOMS, STREAMS, _desc  # noqa: E402


class Ticks:
    """One captured graph of two fleet ticks with `update`, with or without the information."""

    def __init__(self, cfg, blob, pairs, n_stride, S, update, info):
        self.descs = [_desc(cfg, h, w, wp, n_stride, S) for h, w, wp in GEOMS]
        hp = capi.train_params(cfg, 0.0)
        n = len(GEOMS)
        # geometry g's streams serve pairs g * S .. g * S + S - 1
        self.frames = [[staged([p[i] for p in pairs[g * S:(g + 1) * S]], n_stride) for g in range(n)] for i in (0, 1)]
        self.frames = [[tuple(t.to(DEV) for t in f) for f in fr] for fr in self.frames]
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
        self.ticks()                                          # warm-up: the first frames, and every launcher
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.ticks()
        torch.cuda.synchronize()

    def ticks(self):
        for fr in self.frames:
            self.ws.push([f[0] for f in fr], [f[1] for f in fr], self.active, *self.out, update=self.update)

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
    ap.add_argument("--samples", type=int, default=7)
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
            plain = Ticks(cfg, blob, pairs_all, n_stride, S, bool(update), False)
            info = Ticks(cfg, blob, pairs_all, n_stride, S, bool(update), True)
            xs, ys = [], []
            for _ in range(args.samples):
                xs.append(plain.time(args.seconds))
                ys.append(info.time(args.seconds))
            diffs = [y - x for x, y in zip(xs, ys)]
            same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(plain.out[1:3], info.out[1:3]))
            row[f"update{update}"] = {
                "push_adapt_geometries_ms_per_tick": statistics.median(xs),
                "push_adapt_geometries_info_ms_per_tick": statistics.median(ys),
                "paired_difference_ms": statistics.median(diffs), "plain_samples_ms": xs, "info_samples_ms": ys,
                "paired_differences_ms": diffs, "all_valid": bool(info.out[1].all()),
                "valid_and_losses_bit_identical": bool(same),
                "info_rows_with_pairs": int((info.out[3][:, 78] > 0).sum())}
            row["push_adapt_geometries_workspace_mib"] = plain.bytes / 2 ** 20
            row["push_adapt_geometries_info_workspace_mib"] = info.bytes / 2 ** 20
            del plain, info
            torch.cuda.empty_cache()
        res["streams_per_geometry"][S] = row
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "odometry_streams_adapt_geometries_info.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
