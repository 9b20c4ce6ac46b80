"""Batched streaming odometry (delora_odometry_streams_push) against S independent delora_odometry_push workspaces.

For S in {1, 2, 4, 8, 16} at 64 x 2048 and 64 x 720: ms per tick and frames/s of
  - streams: one streams workspace, one captured _streams_push (all S streams active) replayed per tick;
  - pushes:  S push workspaces, one captured _push each, the S graphs replayed one after another on one stream;
both on the same seeded frames (stream s gets the same frame in both), timed with CUDA events over warmed-up replays
and at least --seconds of work.  The card's name, power limit and SM clock are read in the same run.  With --profile
torch.profiler splits one eager tick (streams, and the S pushes) into kernels at the sizes of --profile_sizes.

    python scripts/gpu_odometry_streams.py [--seconds 1.0] [--profile] [--out DIR]
"""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from delora_b200.deploy import export  # noqa: E402
from delora_b200.deploy.capi import InferenceWorkspace, StreamsWorkspace  # noqa: E402
from measure import DEV, capture, emit, events_ms, gpu_info, model_config, pairs, staged, untrained_blob  # noqa: E402

STREAMS = (1, 2, 4, 8, 16)
SIZES = ((64, 2048), (64, 720))


def frames(h, n):
    pool = [s for p in pairs(h, 3) for s in p]
    out = []
    for s in range(n):
        yaw = math.radians(7.0 * s)
        c, si = math.cos(yaw), math.sin(yaw)
        rot = torch.tensor([[c, -si, 0.0], [si, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
        out.append((rot @ pool[s % len(pool)]).contiguous())
    return out


class StreamsRun:
    def __init__(self, cfg, blob, scans, n_stride):
        S = len(scans)
        self.ws = StreamsWorkspace(export.desc_from_config(cfg, "kitti", n_stride, S), blob)
        self.pts, self.counts = staged(scans, n_stride)
        self.active = torch.ones((S,), dtype=torch.int32, device=DEV)
        self.T = torch.zeros((S, 16), dtype=torch.float32, device=DEV)
        self.valid = torch.zeros((S,), dtype=torch.int32, device=DEV)
        self.graph = capture(self.push, warmup=1)      # the warm-up caches the first frames

    def push(self):
        self.ws.push(self.pts, self.counts, self.active, self.T, self.valid)


class PushRun:
    def __init__(self, cfg, blob, scans, n_stride):
        self.ws, self.pts, self.counts, self.T = [], [], [], []
        for s in scans:
            ws = InferenceWorkspace(export.desc_from_config(cfg, "kitti", n_stride, 1), blob)
            p, c = staged([s], n_stride)
            self.ws.append(ws), self.pts.append(p), self.counts.append(c)
            self.T.append(torch.zeros((16,), dtype=torch.float32, device=DEV))
        for i in range(len(scans)):
            self.push(i, first=True)
            self.push(i)
        self.graphs = [capture(lambda i=i: self.push(i), warmup=0) for i in range(len(scans))]

    def push(self, i, first=False):
        self.ws[i].push(self.pts[i], self.counts[i], None if first else self.T[i])

    def replay(self):
        for g in self.graphs:
            g.replay()


def kernel_split(fn, n=20):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    k = {}
    for e in prof.events():
        if "cuda" in str(e.device_type).lower():
            k[e.name] = k.get(e.name, 0.0) + e.time_range.elapsed_us() / n
    return {"total_us": sum(k.values()), "kernels_us": dict(sorted(k.items(), key=lambda kv: -kv[1])[:16])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--profile_sizes", default="64x2048")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "seconds_per_point": args.seconds, "sizes": {}}
    for h, w in SIZES:
        cfg = model_config(h, w)
        blob = untrained_blob(cfg)
        scans_all = frames(h, max(STREAMS))
        n_stride = max(s.shape[1] for s in scans_all)
        key = f"{h}x{w}"
        rows = {}
        for S in STREAMS:
            scans = scans_all[:S]
            st = StreamsRun(cfg, blob, scans, n_stride)
            pu = PushRun(cfg, blob, scans, n_stride)
            # alternate the two so drift of the card's clock hits both alike
            ms_s1, n_s = events_ms(st.graph.replay, seconds=args.seconds / 2)
            ms_p1, n_p = events_ms(pu.replay, seconds=args.seconds / 2)
            ms_s2, _ = events_ms(st.graph.replay, seconds=args.seconds / 2)
            ms_p2, _ = events_ms(pu.replay, seconds=args.seconds / 2)
            ms_s, ms_p = (ms_s1 + ms_s2) / 2, (ms_p1 + ms_p2) / 2
            torch.cuda.synchronize()
            same = all(torch.equal(st.T[i], pu.T[i]) for i in range(S)) and bool(st.valid.all())
            rows[S] = {"streams_ms_per_tick": ms_s, "streams_frames_per_s": S * 1e3 / ms_s,
                       "pushes_ms_per_tick": ms_p, "pushes_frames_per_s": S * 1e3 / ms_p,
                       "speedup": ms_p / ms_s, "streams_ms_runs": [ms_s1, ms_s2], "pushes_ms_runs": [ms_p1, ms_p2],
                       "replays": [n_s, n_p], "T_bit_identical": same,
                       "streams_workspace_MiB": st.ws.workspace.numel() / 2**20,
                       "pushes_workspace_MiB": sum(x.workspace.numel() for x in pu.ws) / 2**20}
            if args.profile and key in args.profile_sizes.split(",") and S in (1, 16):
                rows[S]["profile_streams"] = kernel_split(st.push)
                rows[S]["profile_pushes"] = kernel_split(lambda: [pu.push(i) for i in range(S)])
            del st, pu
            torch.cuda.empty_cache()
        res["sizes"][key] = {"n_stride": n_stride, "S": rows}
    res["gpu_after"] = gpu_info()
    emit(res, args.out and os.path.join(args.out, "odometry_streams.json"))


if __name__ == "__main__":
    main()
