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
import ctypes
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from delora_b200 import _lib, synthetic  # noqa: E402
from delora_b200.deploy import export  # noqa: E402
from delora_b200.models.model import OdometryModel  # noqa: E402

DEV = "cuda:0"
STREAMS = (1, 2, 4, 8, 16)
SIZES = ((64, 2048), (64, 720))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable"


def sp():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def frames(h, n):
    pool = []
    for i in range(3):
        s1, s2, _, _ = synthetic.make_pair(i, w_raw=2048, rings=h)
        pool += [s1, s2]
    out = []
    for s in range(n):
        yaw = math.radians(7.0 * s)
        c, si = math.cos(yaw), math.sin(yaw)
        rot = torch.tensor([[c, -si, 0.0], [si, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
        out.append((rot @ pool[s % len(pool)]).contiguous())
    return out


def time_replays(fn, seconds):
    """ms per call of fn (graph replays), from CUDA events, over >= `seconds` of work after a warm-up."""
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        fn()
    e1.record()
    e1.synchronize()
    est = e0.elapsed_time(e1) / 10
    n = max(50, int(math.ceil(seconds * 1e3 / max(est, 1e-3))))
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n, n


def staged(scans, n_stride):
    pts = torch.zeros((len(scans), 3, n_stride), dtype=torch.float32)
    for i, s in enumerate(scans):
        pts[i, :, :s.shape[1]] = s
    counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
    return pts.to(DEV), counts.to(DEV)


class StreamsRun:
    def __init__(self, L, cfg, blob, scans, n_stride):
        S = len(scans)
        self.L = L
        self.d = export.desc_from_config(cfg, "kitti", n_stride, S)
        self.dp = ctypes.byref(self.d)
        self.ws = torch.empty((int(L.delora_odometry_streams_workspace_bytes(self.dp)),), dtype=torch.uint8, device=DEV)
        _lib.check(L.delora_odometry_streams_init(self.dp, self.ws.data_ptr(), sp()), "streams_init")
        _lib.check(L.delora_odometry_streams_load_weights(self.dp, blob.data_ptr(), self.ws.data_ptr(), sp()), "load")
        self.pts, self.counts = staged(scans, n_stride)
        self.active = torch.ones((S,), dtype=torch.int32, device=DEV)
        self.T = torch.zeros((S, 16), dtype=torch.float32, device=DEV)
        self.valid = torch.zeros((S,), dtype=torch.int32, device=DEV)
        self.push()                 # first frames: cached; also warms the launchers' host-side state
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.push()

    def push(self):
        _lib.check(self.L.delora_odometry_streams_push(self.dp, self.pts.data_ptr(), self.counts.data_ptr(),
                                                       self.active.data_ptr(), self.ws.data_ptr(), self.T.data_ptr(),
                                                       self.valid.data_ptr(), sp()), "streams_push")


class PushRun:
    def __init__(self, L, cfg, blob, scans, n_stride):
        self.L = L
        self.d = export.desc_from_config(cfg, "kitti", n_stride, 1)
        self.dp = ctypes.byref(self.d)
        nbytes = int(L.delora_odometry_workspace_bytes(self.dp))
        self.ws, self.pts, self.counts, self.T, self.graphs = [], [], [], [], []
        for s in scans:
            ws = torch.empty((nbytes,), dtype=torch.uint8, device=DEV)
            _lib.check(L.delora_odometry_init(self.dp, ws.data_ptr(), sp()), "init")
            _lib.check(L.delora_odometry_load_weights(self.dp, blob.data_ptr(), ws.data_ptr(), sp()), "load")
            p, c = staged([s], n_stride)
            self.ws.append(ws), self.pts.append(p), self.counts.append(c)
            self.T.append(torch.zeros((16,), dtype=torch.float32, device=DEV))
        for i in range(len(scans)):
            self.push(i, first=True)
            self.push(i)
        torch.cuda.synchronize()
        for i in range(len(scans)):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self.push(i)
            self.graphs.append(g)

    def push(self, i, first=False):
        _lib.check(self.L.delora_odometry_push(self.dp, self.pts[i].data_ptr(), self.counts[i].data_ptr(),
                                               self.ws[i].data_ptr(), None if first else self.T[i].data_ptr(), sp()),
                   "push")

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
    L = _lib.lib()
    res = {"gpu_before": gpu_info(), "seconds_per_point": args.seconds, "sizes": {}}
    for h, w in SIZES:
        cfg = synthetic.fov_config(h=h, w=w, device=DEV)
        cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                    "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                    "use_dropout": False})
        torch.manual_seed(0)
        model = OdometryModel(cfg).to(DEV).eval()
        blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), cfg)).to(DEV)
        scans_all = frames(h, max(STREAMS))
        n_stride = max(s.shape[1] for s in scans_all)
        key = f"{h}x{w}"
        rows = {}
        for S in STREAMS:
            scans = scans_all[:S]
            st = StreamsRun(L, cfg, blob, scans, n_stride)
            pu = PushRun(L, cfg, blob, scans, n_stride)
            # alternate the two so drift of the card's clock hits both alike
            ms_s1, n_s = time_replays(st.graph.replay, args.seconds / 2)
            ms_p1, n_p = time_replays(pu.replay, args.seconds / 2)
            ms_s2, _ = time_replays(st.graph.replay, args.seconds / 2)
            ms_p2, _ = time_replays(pu.replay, args.seconds / 2)
            ms_s, ms_p = (ms_s1 + ms_s2) / 2, (ms_p1 + ms_p2) / 2
            torch.cuda.synchronize()
            same = all(torch.equal(st.T[i], pu.T[i]) for i in range(S)) and bool(st.valid.all())
            rows[S] = {"streams_ms_per_tick": ms_s, "streams_frames_per_s": S * 1e3 / ms_s,
                       "pushes_ms_per_tick": ms_p, "pushes_frames_per_s": S * 1e3 / ms_p,
                       "speedup": ms_p / ms_s, "streams_ms_runs": [ms_s1, ms_s2], "pushes_ms_runs": [ms_p1, ms_p2],
                       "replays": [n_s, n_p], "T_bit_identical": same,
                       "streams_workspace_MiB": st.ws.numel() / 2**20,
                       "pushes_workspace_MiB": sum(x.numel() for x in pu.ws) / 2**20}
            if args.profile and key in args.profile_sizes.split(",") and S in (1, 16):
                rows[S]["profile_streams"] = kernel_split(st.push)
                rows[S]["profile_pushes"] = kernel_split(lambda: [pu.push(i) for i in range(S)])
            del st, pu
            torch.cuda.empty_cache()
        res["sizes"][key] = {"n_stride": n_stride, "S": rows}
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "odometry_streams.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
