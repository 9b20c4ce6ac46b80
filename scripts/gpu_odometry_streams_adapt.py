"""What serving several sensors while the model adapts to them costs on the GPU, against the two workspaces a host
needs without delora_odometry_streams_push_adapt.

Per tick, ms at S in {1, 4, 16} for 64 x 720 (w_pre 0 and 2250) and 64 x 2048 (w_pre 0), all streams active, on the
same near-identity weights (gpu_odometry_eval.near_identity_blob), lr 0 (Adam runs, the weights stay put, so every
sample times the same work):
  adapt0     delora_odometry_streams_push_adapt, update = 0 (serve and score);
  adapt1     delora_odometry_streams_push_adapt, update = 1 (serve, score and one Adam step on the S pairs);
  train      delora_odometry_train_step at B = S on the stacked pairs alone (the expected cost of adapt1);
  compose    what a host composes today: a streams tick (delora_odometry_streams_push_residual at w_pre 0,
             _streams_push_pre at w_pre > 0), _train_step at B = S on the stacked (previous, this) pairs and
             _train_weights, graph-replayed, then delora_odometry_streams_load_weights, which is not capturable (it
             copies its prep table from host memory) and runs eagerly.  The host-side copy of every previous scan is
             not counted.
Each stream alternates between the two scans of a synthetic pair, so every tick sees a consecutive frame; one captured
graph holds two ticks.  The sides alternate (adapt0, adapt1, train, compose, adapt0, ...) over at least --seconds of
work per sample; the medians and every sample are reported.  The card's name, power limit and SM clocks are read in
the same run.  Writes odometry_streams_adapt.json to --out.

    python scripts/gpu_odometry_streams_adapt.py [--seconds 0.3] [--samples 5] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from delora_b200 import ops, synthetic  # noqa: E402
from delora_b200.deploy import capi, export  # noqa: E402
from gpu_odometry_eval import near_identity_blob  # noqa: E402
from gpu_odometry_streams import DEV, gpu_info, staged, time_replays  # noqa: E402

SIZES = ((64, 720, 0), (64, 720, 2250), (64, 2048, 0))
STREAMS = (1, 4, 16)
SIDES = ("adapt0", "adapt1", "train", "compose")


def _graph(fn):
    fn()                                 # warms the launchers' host-side state
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


class Sides:
    """Every side's workspaces and graphs for S streams, each stream alternating between its pair's two scans."""

    def __init__(self, cfg, blob, pairs, n_stride, w_pre):
        S = len(pairs)
        d = export.desc_from_config(cfg, "kitti", n_stride, S, preprocessing_normals=w_pre > 0)
        hp = capi.train_params(cfg, 0.0)
        rp = capi.residual_params(cfg)
        self.frames = [staged([p[i] for p in pairs], n_stride) for i in (0, 1)]
        # the train step's rows: (scan_1 x S, scan_2 x S) and the reverse, the pairs of the two ticks
        self.stacked = [staged([p[i] for p in pairs] + [p[1 - i] for p in pairs], n_stride) for i in (1, 0)]
        self.active = torch.ones((S,), dtype=torch.int32, device=DEV)
        self.T = torch.zeros((S, 16), dtype=torch.float32, device=DEV)
        self.valid = torch.zeros((S,), dtype=torch.int32, device=DEV)
        self.losses = torch.zeros((S, ops.LOSS_ROW), dtype=torch.float32, device=DEV)
        self.adapt = capi.AdaptiveStreamsWorkspace(d, blob, hp)
        self.train = capi.TrainingWorkspace(d, blob, hp)
        self.streams = (capi.PreStreamsWorkspace(d, blob, rp) if w_pre > 0 else
                        capi.ResidualStreamsWorkspace(d, blob, rp))
        self.weights = blob.clone()
        self.graphs = {"adapt0": _graph(lambda: self.adapt_ticks(False)),
                       "adapt1": _graph(lambda: self.adapt_ticks(True)),
                       "train": _graph(self.train_steps)}
        self.compose_graphs = [_graph(lambda i=i: self.compose_tick(i)) for i in (0, 1)]
        self.fn = {k: g.replay for k, g in self.graphs.items()}
        self.fn["compose"] = self.compose

    def adapt_ticks(self, update):
        for pts, counts in self.frames:
            self.adapt.push(pts, counts, self.active, self.T, self.valid, self.losses, update=update)

    def train_steps(self):
        for pts, counts in self.stacked:
            self.train.step(pts, counts, outputs=False)

    def compose_tick(self, i):
        self.streams.push(*self.frames[i], self.active, self.T, self.valid, self.losses)
        self.train.step(*self.stacked[i], outputs=False)
        self.train._call("delora_odometry_train_weights", self.train.workspace.data_ptr(), self.weights.data_ptr())

    def compose(self):
        for g in self.compose_graphs:
            g.replay()
            self.streams.load_weights(self.weights)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.3)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": "name, power.limit, clocks.sm, clocks.max.sm",
           "seconds_per_sample": args.seconds, "lr": 0.0, "sizes": {}}
    for h, w, w_pre in SIZES:
        cfg = synthetic.fov_config(h=h, w=w, device=DEV)
        cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                    "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                    "use_dropout": False})
        if w_pre:
            cfg["kitti"]["horizontal_cells_preprocessing"] = w_pre
        blob = near_identity_blob(cfg)
        pairs_all = [synthetic.make_pair(i, w_raw=2048, rings=h)[:2] for i in range(max(STREAMS))]
        n_stride = max(max(a.shape[1], b.shape[1]) for a, b in pairs_all)
        per_s = {}
        for S in STREAMS:
            sides = Sides(cfg, blob, pairs_all[:S], n_stride, w_pre)
            samples = {k: [] for k in SIDES}
            for _ in range(args.samples):
                for k in SIDES:
                    samples[k].append(time_replays(sides.fn[k], args.seconds)[0] / 2)      # two ticks per call
            torch.cuda.synchronize()
            med = {k: statistics.median(v) for k, v in samples.items()}
            per_s[S] = {**{f"{k}_ms_per_tick": m for k, m in med.items()},
                        **{f"{k}_samples_ms": v for k, v in samples.items()},
                        "adapt1_over_train_ms": med["adapt1"] - med["train"],
                        "compose_minus_adapt1_ms": med["compose"] - med["adapt1"],
                        "adapt_all_valid": bool(sides.valid.all()),
                        "adapt_step_count": int(sides.adapt.get_state()[3][0]),
                        "workspace_MiB": {"adapt": sides.adapt.workspace.numel() / 2**20,
                                          "train": sides.train.workspace.numel() / 2**20,
                                          "streams": sides.streams.workspace.numel() / 2**20}}
            del sides
            torch.cuda.empty_cache()
        res["sizes"][f"{h}x{w}_wpre{w_pre}"] = {"n_stride": n_stride, "streams_S": per_s}
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "odometry_streams_adapt.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
