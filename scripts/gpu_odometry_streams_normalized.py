"""What serving several sensors of a normalised model from one workspace costs on the GPU.

Per tick, ms at S in {1, 4, 16} for 64 x 2048 and 64 x 720, all streams active, graph-replayed:
  push             delora_odometry_streams_push on the same weights as an unnormalised model (the image cache);
  push_normalized  delora_odometry_streams_push_normalized;
  pairs_b1         S captured delora_odometry_pairs_normalized calls at B = 1 per tick (a host's route without the
                   normalised streams workspace: one call per sensor).
Each stream alternates between the two scans of a synthetic pair, so every tick sees a consecutive frame; one captured
graph holds two ticks.  The heads are near the identity (measure.near_identity_blob).  The three sides
alternate (a, b, c, a, b, c, ...) over at least --seconds of work per sample, and the medians are reported with every
sample.  The last tick's T rows and factors of push_normalized are compared byte for byte with pairs_b1's.  The card's
name, power limit and SM clocks are read in the same run.  Writes odometry_streams_normalized.json to --out.

    python scripts/gpu_odometry_streams_normalized.py [--seconds 0.5] [--samples 3] [--out DIR]
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from delora_b200.deploy import capi, export  # noqa: E402
from measure import (DEV, GPU_QUERY, alternate, capture, emit, events_ms, gpu_info, model_config,  # noqa: E402
                     n_stride, near_identity_blob, pairs, staged)

SIZES = ((64, 2048), (64, 720))
STREAMS = (1, 4, 16)


class StreamTicks:
    """A streams workspace (plain or normalised) and a graph of two ticks: every stream's scan_1, then its scan_2."""

    def __init__(self, cfg, blob, pairs, n_stride, normalized):
        S = len(pairs)
        d = export.desc_from_config(cfg, "kitti", n_stride, S)
        self.ws = capi.NormalizedStreamsWorkspace(d, blob) if normalized else capi.StreamsWorkspace(d, blob)
        self.frames = [staged([p[i] for p in pairs], n_stride) for i in (0, 1)]
        self.active = torch.ones((S,), dtype=torch.int32, device=DEV)
        self.out = (torch.zeros((S, 16), dtype=torch.float32, device=DEV),
                    torch.zeros((S,), dtype=torch.int32, device=DEV))
        if normalized:
            self.out += (torch.zeros((S,), dtype=torch.float32, device=DEV),)
        self.graph = capture(self.two_ticks, warmup=1)      # the warm-up caches the first frames

    def two_ticks(self):
        for pts, counts in self.frames:
            self.ws.push(pts, counts, self.active, *self.out)


class PairsTicks:
    """One inference workspace and a graph of the same two ticks as S pairs_normalized calls at B = 1 each."""

    def __init__(self, cfg, blob, pairs, n_stride):
        self.ws = capi.InferenceWorkspace(export.desc_from_config(cfg, "kitti", n_stride, 1), blob)
        # tick 0: (scan_2, scan_1) -- the previous tick of a replay ended on scan_2; tick 1: (scan_1, scan_2)
        self.calls = [[staged([p[1], p[0]], n_stride) for p in pairs], [staged([p[0], p[1]], n_stride) for p in pairs]]
        self.graph = capture(self.two_ticks, warmup=1)

    def two_ticks(self):
        for tick in self.calls:
            self.last = [self.ws.pairs_normalized(pts, counts) for pts, counts in tick]    # (T, pooled, factor) each


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": GPU_QUERY,
           "seconds_per_sample": args.seconds, "sizes": {}}
    for h, w in SIZES:
        cfg = model_config(h, w)
        blob = near_identity_blob(cfg)
        pairs_all = pairs(h, max(STREAMS))
        stride = n_stride(pairs_all)
        per_s = {}
        for S in STREAMS:
            ps = pairs_all[:S]
            sides = {"push": StreamTicks(cfg, blob, ps, stride, False),
                     "push_normalized": StreamTicks(cfg, blob, ps, stride, True),
                     "pairs_b1": PairsTicks(cfg, blob, ps, stride)}
            samples = alternate({k: side.graph.replay for k, side in sides.items()}, args.samples,
                                lambda fn: events_ms(fn, seconds=args.seconds)[0] / 2)     # two ticks per replay
            torch.cuda.synchronize()
            norm, pb1 = sides["push_normalized"], sides["pairs_b1"]
            T_pairs = torch.stack([t.reshape(16) for t, _, _ in pb1.last])
            f_pairs = torch.cat([f for _, _, f in pb1.last])
            med = {k: statistics.median(v) for k, v in samples.items()}
            per_s[S] = {**{f"{k}_ms_per_tick": m for k, m in med.items()},
                        **{f"{k}_samples_ms": v for k, v in samples.items()},
                        "push_normalized_ms_per_stream": med["push_normalized"] / S,
                        "pairs_b1_ms_per_stream": med["pairs_b1"] / S,
                        "bit_identical_to_pairs_b1": bool(norm.out[1].all())
                        and bool(torch.equal(norm.out[0].view(torch.int32), T_pairs.view(torch.int32)))
                        and bool(torch.equal(norm.out[2].view(torch.int32), f_pairs.view(torch.int32))),
                        "workspace_MiB": {"push": sides["push"].ws.workspace.numel() / 2**20,
                                          "push_normalized": norm.ws.workspace.numel() / 2**20}}
            del sides, norm, pb1
            torch.cuda.empty_cache()
        res["sizes"][f"{h}x{w}"] = {"n_stride": stride, "streams_S": per_s}
    res["gpu_after"] = gpu_info()
    emit(res, args.out and os.path.join(args.out, "odometry_streams_normalized.json"))


if __name__ == "__main__":
    main()
