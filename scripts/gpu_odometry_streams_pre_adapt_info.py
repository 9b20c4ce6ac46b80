"""What the Gauss-Newton information costs beside the recipe streams and the adapting streams on the GPU.

delora_odometry_streams_push_pre -> _push_pre_info (w_pre 2250) and delora_odometry_streams_push_adapt ->
_push_adapt_info (w_pre 0, update = 1, lr 0, so every tick does the same work), ms per tick at S in {1, 4, 16} for
64 x 2048 and 64 x 720, all streams active, with the near-identity model and consecutive synthetic frames of
gpu_odometry_eval.py (one captured graph of two ticks per workspace).  The two sides alternate (a, b, a, b, ...) and
the medians are reported with every sample.  The card's name, power limit and SM clocks are read in the same run.
Writes odometry_streams_pre_adapt_info.json to --out.

    python scripts/gpu_odometry_streams_pre_adapt_info.py [--seconds 0.3] [--samples 3] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from delora_b200 import ops, synthetic  # noqa: E402
from delora_b200.deploy import capi, export  # noqa: E402
from gpu_odometry_eval import near_identity_blob  # noqa: E402
from gpu_odometry_streams import DEV, gpu_info, staged, time_replays  # noqa: E402

SIZES = ((64, 2048), (64, 720))
BATCHES = (1, 4, 16)
W_PRE = 2250


class Ticks:
    """One workspace of `mode` ('pre' or 'adapt', with or without the information) and a graph of two ticks: every
    stream's scan_1, then scan_2."""

    def __init__(self, cfg, blob, pairs, n_stride, mode, info):
        S = len(pairs)
        self.info = info
        self.mode = mode
        if mode == "pre":
            d = export.desc_from_config(cfg, "kitti", n_stride, S, preprocessing_normals=True)
            kind = capi.PreInformationStreamsWorkspace if info else capi.PreStreamsWorkspace
            self.ws = kind(d, blob, capi.residual_params(cfg))
        else:
            d = export.desc_from_config(cfg, "kitti", n_stride, S)
            kind = capi.AdaptiveInformationStreamsWorkspace if info else capi.AdaptiveStreamsWorkspace
            self.ws = kind(d, blob, capi.train_params(cfg, 0.0))
        self.frames = [staged([p[i] for p in pairs], n_stride) for i in (0, 1)]
        self.active = torch.ones((S,), dtype=torch.int32, device=DEV)
        self.T = torch.zeros((S, 16), dtype=torch.float32, device=DEV)
        self.valid = torch.zeros((S,), dtype=torch.int32, device=DEV)
        self.losses = torch.zeros((S, ops.LOSS_ROW), dtype=torch.float32, device=DEV)
        self.rows = torch.zeros((S, ops.INFO_ROW), dtype=torch.float32, device=DEV)
        self.two_ticks()
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.two_ticks()

    def two_ticks(self):
        out = (self.T, self.valid, self.losses) + ((self.rows,) if self.info else ())
        for pts, counts in self.frames:
            if self.mode == "pre":
                self.ws.push(pts, counts, self.active, *out)
            else:
                self.ws.push(pts, counts, self.active, *out, update=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.3)
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": "name, power.limit, clocks.sm, clocks.max.sm",
           "seconds_per_sample": args.seconds, "w_pre_of_pre": W_PRE, "sizes": {}}
    for h, w in SIZES:
        cfg = synthetic.fov_config(h=h, w=w, device=DEV)
        cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                    "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                    "use_dropout": False})
        cfg["kitti"]["horizontal_cells_preprocessing"] = W_PRE
        blob = near_identity_blob(cfg)
        pairs_all = [synthetic.make_pair(i, w_raw=2048, rings=h)[:2] for i in range(max(BATCHES))]
        n_stride = max(max(a.shape[1], b.shape[1]) for a, b in pairs_all)
        per = {}
        for mode in ("pre", "adapt"):
            for n in BATCHES:
                pairs = pairs_all[:n]
                a = Ticks(cfg, blob, pairs, n_stride, mode, False)
                b = Ticks(cfg, blob, pairs, n_stride, mode, True)
                xs, ys = [], []
                for _ in range(args.samples):
                    xs.append(time_replays(a.graph.replay, args.seconds)[0] / 2)      # two ticks per replay
                    ys.append(time_replays(b.graph.replay, args.seconds)[0] / 2)
                torch.cuda.synchronize()
                ms_a, ms_b = statistics.median(xs), statistics.median(ys)
                per[f"{mode}_S{n}"] = {
                    f"push_{mode}_ms_per_tick": ms_a, f"push_{mode}_info_ms_per_tick": ms_b,
                    "added_ms_per_tick": ms_b - ms_a, "samples_ms": [xs, ys],
                    "T_losses_bit_identical": bool(torch.equal(a.T, b.T)) and bool(torch.equal(a.losses, b.losses))
                    and bool(b.valid.all()),
                    "smallest_over_largest_eigenvalue_last_tick": (b.rows[:, 36] / b.rows[:, 41]).cpu().tolist(),
                    "workspace_MiB": [a.ws.workspace.numel() / 2**20, b.ws.workspace.numel() / 2**20]}
                print(f"{h}x{w} {mode} S={n}: {ms_a:.3f} -> {ms_b:.3f} ms per tick", flush=True)
                del a, b
                torch.cuda.empty_cache()
        res["sizes"][f"{h}x{w}"] = {"n_stride": n_stride, "ticks": per}
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "odometry_streams_pre_adapt_info.json"), "w") as f:
            f.write(text)
    else:
        print(text)


if __name__ == "__main__":
    main()
