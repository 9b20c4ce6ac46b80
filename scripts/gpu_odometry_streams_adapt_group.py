"""What adapting one model from the streams of several GPUs (delora_odometry_streams_push_adapt_group) costs.

--gpus 1: the world = 1 group tick against delora_odometry_streams_push_adapt, update = 1, ms per tick at S = 1, 4, 16
    for 64 x 720 (w_pre 0), all streams active, each alternating between the two scans of a synthetic pair, the same
    near-identity model and lr 0 as gpu_odometry_streams_adapt.py (Adam runs, the weights stay put).  One captured
    graph holds two ticks; the two graphs alternate (plain, group, plain, ...) and the paired differences are reported
    with their median.  With world = 1 the group tick launches what _push_adapt launches, so the expected difference
    is zero.
--gpus N (N > 1): one rank per GPU 0 .. N-1 of this process (peer access both ways, unicast path), S streams per GPU,
    each rank's two ticks captured on its own device; a sample replays every rank's graph, alternating with N plain
    _push_adapt workspaces.  The difference is the cost of the collectives per tick.  A torch.profiler pass then reads
    the device time of the valid-count exchange (count_allreduce_kernel) on every rank, and its share of the tick.
    Ranks that share one GPU give no such number, so this needs a multi-GPU node.

The card's name, power limit and SM clocks are read in the same run.  Writes odometry_streams_adapt_group.json to
--out.

    python scripts/gpu_odometry_streams_adapt_group.py [--gpus N] [--seconds 0.5] [--samples 5] [--out DIR]
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
from gpu_train_group import enable_peer_access  # noqa: E402

H, W = 64, 720
STREAMS = (1, 4, 16)


class Ranks:
    """N adapting workspaces (one per device, or N = 1) of S streams each, and one captured graph of two update = 1
    ticks per rank: the group tick (group=True) or _push_adapt."""

    def __init__(self, cfg, blob, pairs, n_stride, n, group):
        S = len(pairs)
        self.devs = [torch.device("cuda", i) for i in range(n)]
        self.ws, self.frames, self.bufs, self.streams = [], [], [], []
        kind = capi.AdaptiveStreamsGroupWorkspace if group else capi.AdaptiveStreamsWorkspace
        for dev in self.devs:
            with torch.cuda.device(dev):
                d = export.desc_from_config(cfg, "kitti", n_stride, S)
                d.w_pre = 0
                self.ws.append(kind(d, blob.to(dev), capi.train_params(cfg, 0.0)))
                self.frames.append([tuple(t.to(dev) for t in staged([p[i] for p in pairs], n_stride)) for i in (0, 1)])
                self.bufs.append((torch.ones((S,), dtype=torch.int32, device=dev),
                                  torch.zeros((S, 16), dtype=torch.float32, device=dev),
                                  torch.zeros((S,), dtype=torch.int32, device=dev),
                                  torch.zeros((S, ops.LOSS_ROW), dtype=torch.float32, device=dev)))
                self.streams.append(torch.cuda.Stream(dev))
        self.group = capi.AdaptingStreamsGroup(self.ws) if group else None
        self.tick_all()                                       # warm-up: the first frames, and every launcher
        self.sync()
        self.graphs = []
        for r, dev in enumerate(self.devs):
            with torch.cuda.device(dev):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self.streams[r]):
                    self.ticks(r)
                self.graphs.append(g)
        self.sync()

    def ticks(self, r):
        active, T, valid, losses = self.bufs[r]
        for pts, counts in self.frames[r]:
            if self.group:
                self.group.push(r, pts, counts, active, update=True, out=(T, valid, losses))
            else:
                self.ws[r].push(pts, counts, active, T, valid, losses, update=True)

    def tick_all(self):
        for r, dev in enumerate(self.devs):
            with torch.cuda.device(dev), torch.cuda.stream(self.streams[r]):
                self.ticks(r)

    def replay(self):
        for r, dev in enumerate(self.devs):
            with torch.cuda.device(dev), torch.cuda.stream(self.streams[r]):
                self.graphs[r].replay()

    def sync(self):
        for dev in self.devs:
            torch.cuda.synchronize(dev)

    def time(self, seconds):
        """ms per tick of every rank (host clock around synchronised replays of two ticks), over >= `seconds`."""
        for _ in range(4):
            self.replay()
        self.sync()
        n, t0 = 0, time.perf_counter()
        while True:
            self.replay()
            n += 1
            if n % 4 == 0:
                self.sync()
                el = time.perf_counter() - t0
                if el >= seconds:
                    return el * 1e3 / n / 2

    def exchange_us(self, replays=20):
        """Median device time of count_allreduce_kernel per rank over `replays` replays (torch.profiler)."""
        from torch.profiler import ProfilerActivity, profile
        self.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(replays):
                self.replay()
            self.sync()
        per_dev = {}
        for ev in prof.events():
            if ev.name == "count_allreduce_kernel" and ev.device_type == torch.autograd.DeviceType.CUDA:
                per_dev.setdefault(ev.device_index, []).append(ev.device_time_total)
        return {str(k): statistics.median(v) for k, v in sorted(per_dev.items())}

    def status(self):
        return [int(s.item()) for s in self.group.status] if self.group else []

    def steps(self):
        return [int(w.get_state()[3][0]) for w in self.ws]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    assert torch.cuda.device_count() >= args.gpus, f"--gpus {args.gpus}: {torch.cuda.device_count()} GPU(s) here"
    if args.gpus > 1:
        enable_peer_access(args.gpus)
    res = {"gpu_before": gpu_info(), "gpu_query": "name, power.limit, clocks.sm, clocks.max.sm", "gpus": args.gpus,
           "size": f"{H}x{W}_wpre0", "lr": 0.0, "seconds_per_sample": args.seconds, "streams_S": {}}
    cfg = synthetic.fov_config(h=H, w=W, device=DEV)
    cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                "use_dropout": False})
    blob = near_identity_blob(cfg)
    pairs_all = [synthetic.make_pair(i, w_raw=2048, rings=H)[:2] for i in range(max(STREAMS))]
    n_stride = max(max(a.shape[1], b.shape[1]) for a, b in pairs_all)
    for S in STREAMS:
        plain = Ranks(cfg, blob, pairs_all[:S], n_stride, args.gpus, False)
        group = Ranks(cfg, blob, pairs_all[:S], n_stride, args.gpus, True)
        xs, ys = [], []
        for _ in range(args.samples):
            xs.append(plain.time(args.seconds))
            ys.append(group.time(args.seconds))
        diffs = [y - x for x, y in zip(xs, ys)]
        row = {"push_adapt_ms_per_tick": statistics.median(xs), "group_ms_per_tick": statistics.median(ys),
               "paired_difference_ms": statistics.median(diffs), "push_adapt_samples_ms": xs,
               "group_samples_ms": ys, "paired_differences_ms": diffs, "status": group.status(),
               "group_step_counts": group.steps(), "plain_step_counts": plain.steps(),
               "all_valid": bool(all(bool(b[2].all()) for b in group.bufs))}
        if args.gpus > 1:
            ex = group.exchange_us()
            row["exchange_us_per_rank"] = ex
            row["exchange_share_of_tick"] = {k: v * 1e-3 / row["group_ms_per_tick"] for k, v in ex.items()}
        res["streams_S"][S] = row
        del plain, group
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "odometry_streams_adapt_group.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
