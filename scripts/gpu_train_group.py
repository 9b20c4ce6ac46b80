"""What the data-parallel training step of the C ABI (delora_odometry_train_step_group) costs on the GPU.

--gpus 1: the world = 1 group step against delora_odometry_train_step, ms per graph replay at B = 16 (--batch) for
    64 x 720 and 64 x 2048, the same near-identity model and lr 0 as gpu_odometry_eval.py.  The two graphs alternate
    (plain, group, plain, group, ...) and the paired differences are reported with their median.  With world = 1 the
    group step launches what the plain step launches, so the expected difference is zero.
--gpus N (N > 1): one rank per GPU 0 .. N-1 of this process (peer access enabled both ways, unicast path), each rank's
    group step captured on its own device; a sample replays every rank's graph once per step, and the same for N plain
    steps with no collective, alternating.  The difference is the all-reduce time the backward does not hide (per step,
    B pairs per GPU).  Not measured yet: this needs a multi-GPU NVLink node.

The card's name, power limit and SM clocks are read in the same run.  Writes train_group.json to --out.

    python scripts/gpu_train_group.py [--gpus N] [--batch 16] [--seconds 0.5] [--samples 5] [--out DIR]
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from delora_b200.deploy import capi, export  # noqa: E402
from measure import (GPU_QUERY, alternate, capture, emit, enable_peer_access, gpu_info, host_ms,  # noqa: E402
                     model_config, n_stride, near_identity_blob, paired, pairs, staged)

SIZES = ((64, 720), (64, 2048))


class Ranks:
    """N training workspaces (one per device, or N = 1), each with B pairs, and one captured step per rank: the
    group step (group=True) or the plain step."""

    def __init__(self, cfg, blob, pairs, n_stride, n, group):
        B = len(pairs)
        self.devs = [torch.device("cuda", i) for i in range(n)]
        self.ws, self.inputs, self.streams = [], [], []
        for dev in self.devs:
            with torch.cuda.device(dev):
                d = export.desc_from_config(cfg, "kitti", n_stride, B)
                d.w_pre = 0
                self.ws.append(capi.TrainingWorkspace(d, blob.to(dev), capi.train_params(cfg, 0.0)))
                pts, counts = staged([p[0] for p in pairs] + [p[1] for p in pairs], n_stride)
                self.inputs.append((pts.to(dev), counts.to(dev)))
                self.streams.append(torch.cuda.Stream(dev))
        self.group = capi.TrainingGroup(self.ws) if group else None
        self.step_all()                                       # warm-up, and the ICP scratch's batch size
        self.sync()
        self.graphs = []
        for r, dev in enumerate(self.devs):
            with torch.cuda.device(dev):
                self.graphs.append(capture(lambda r=r: self.step(r), warmup=0, stream=self.streams[r]))

    def step(self, r):
        if self.group:
            self.group.step(r, *self.inputs[r], outputs=False)
        else:
            self.ws[r].step(*self.inputs[r], outputs=False)

    def step_all(self):
        for r, dev in enumerate(self.devs):
            with torch.cuda.device(dev), torch.cuda.stream(self.streams[r]):
                self.step(r)

    def replay(self):
        for r, dev in enumerate(self.devs):
            with torch.cuda.device(dev), torch.cuda.stream(self.streams[r]):
                self.graphs[r].replay()

    def sync(self):
        for dev in self.devs:
            torch.cuda.synchronize(dev)

    def status(self):
        return [int(s.item()) for s in self.group.status] if self.group else []


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    assert torch.cuda.device_count() >= args.gpus, f"--gpus {args.gpus}: {torch.cuda.device_count()} GPU(s) here"
    if args.gpus > 1:
        enable_peer_access(args.gpus)
    res = {"gpu_before": gpu_info(), "gpu_query": GPU_QUERY, "gpus": args.gpus,
           "batch_per_gpu": args.batch, "seconds_per_sample": args.seconds, "sizes": {}}
    for h, w in SIZES:
        cfg = model_config(h, w)
        blob = near_identity_blob(cfg)
        ps = pairs(h, args.batch)
        stride = n_stride(ps)
        plain = Ranks(cfg, blob, ps, stride, args.gpus, False)
        group = Ranks(cfg, blob, ps, stride, args.gpus, True)
        t = alternate({"plain": plain, "group": group}, args.samples,
                      lambda ranks: host_ms(ranks.replay, args.seconds, ranks.devs, every=8, warmup=0))
        xs, ys = t["plain"], t["group"]
        diffs, diff = paired(xs, ys)
        res["sizes"][f"{h}x{w}"] = {
            "n_stride": stride, "train_step_ms": statistics.median(xs), "train_step_group_ms": statistics.median(ys),
            "paired_difference_ms": diff, "train_step_samples_ms": xs,
            "train_step_group_samples_ms": ys, "paired_differences_ms": diffs, "status": group.status()}
        del plain, group
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    emit(res, args.out and os.path.join(args.out, "train_group.json"))


if __name__ == "__main__":
    main()
