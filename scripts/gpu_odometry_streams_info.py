"""What the Gauss-Newton information costs on the GPU.

(a) delora_odometry_streams_push_info against delora_odometry_streams_push_residual, ms per tick at S in {1, 4, 16}
    for 64 x 2048 and 64 x 720, all streams active, with the near-identity model and consecutive synthetic frames of
    gpu_odometry_eval.py (one captured graph of two ticks per side).  The two sides alternate (a, b, a, b, ...) and the
    medians are reported with every sample.
(b) The information pass's own kernels (icp_info_rows_kernel + icp_info_finalize_kernel) from torch.profiler in a
    separate run over graph replays of _push_info, microseconds per tick.

The card's name, power limit and SM clocks are read in the same run.  Writes odometry_streams_info.json to --out.

    python scripts/gpu_odometry_streams_info.py [--seconds 0.5] [--samples 3] [--out DIR]
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
INFO_KERNELS = ("icp_info_rows_kernel", "icp_info_finalize_kernel")


class Ticks:
    """One residual or information streams workspace and a graph of two ticks: every stream's scan_1, then scan_2."""

    def __init__(self, cfg, blob, pairs, n_stride, info):
        S = len(pairs)
        d = export.desc_from_config(cfg, "kitti", n_stride, S)
        kind = capi.InformationStreamsWorkspace if info else capi.ResidualStreamsWorkspace
        self.ws = kind(d, blob, capi.residual_params(cfg))
        self.frames = [staged([p[i] for p in pairs], n_stride) for i in (0, 1)]
        self.active = torch.ones((S,), dtype=torch.int32, device=DEV)
        self.T = torch.zeros((S, 16), dtype=torch.float32, device=DEV)
        self.valid = torch.zeros((S,), dtype=torch.int32, device=DEV)
        self.losses = torch.zeros((S, ops.LOSS_ROW), dtype=torch.float32, device=DEV)
        self.out = (self.T, self.valid, self.losses)
        if info:
            self.info = torch.zeros((S, ops.INFO_ROW), dtype=torch.float32, device=DEV)
            self.out += (self.info,)
        self.two_ticks()
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.two_ticks()

    def two_ticks(self):
        for pts, counts in self.frames:
            self.ws.push(pts, counts, self.active, *self.out)


def info_kernel_us(ticks, replays=50):
    """Microseconds per tick of the information kernels, from a profiled run of graph replays."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(replays):
            ticks.graph.replay()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        for k in INFO_KERNELS:
            if k in ev.name:
                per[k] = per.get(k, 0.0) + ev.device_time
    return {k: v / (2 * replays) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": "name, power.limit, clocks.sm, clocks.max.sm",
           "seconds_per_sample": args.seconds, "sizes": {}}
    for h, w in SIZES:
        cfg = synthetic.fov_config(h=h, w=w, device=DEV)
        cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                    "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                    "use_dropout": False})
        blob = near_identity_blob(cfg)
        pairs_all = [synthetic.make_pair(i, w_raw=2048, rings=h)[:2] for i in range(max(BATCHES))]
        n_stride = max(max(a.shape[1], b.shape[1]) for a, b in pairs_all)
        streams = {}
        for n in BATCHES:
            pairs = pairs_all[:n]
            resid, info = Ticks(cfg, blob, pairs, n_stride, False), Ticks(cfg, blob, pairs, n_stride, True)
            xs, ys = [], []
            for _ in range(args.samples):
                xs.append(time_replays(resid.graph.replay, args.seconds)[0] / 2)      # two ticks per replay
                ys.append(time_replays(info.graph.replay, args.seconds)[0] / 2)
            torch.cuda.synchronize()
            ms_r, ms_i = statistics.median(xs), statistics.median(ys)
            ev = info.info[:, 36:42].cpu()
            streams[n] = {"push_residual_ms_per_tick": ms_r, "push_info_ms_per_tick": ms_i,
                          "added_ms_per_tick": ms_i - ms_r, "push_residual_samples_ms": xs, "push_info_samples_ms": ys,
                          "info_kernels_us_per_tick": info_kernel_us(info),
                          "T_losses_bit_identical": bool(torch.equal(resid.T, info.T))
                          and bool(torch.equal(resid.losses, info.losses)) and bool(info.valid.all()),
                          "eigenvalues_last_tick": ev.tolist(),
                          "workspace_MiB": [resid.ws.workspace.numel() / 2**20, info.ws.workspace.numel() / 2**20]}
            del resid, info
            torch.cuda.empty_cache()
        res["sizes"][f"{h}x{w}"] = {"n_stride": n_stride, "streams_S": streams}
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "odometry_streams_info.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
