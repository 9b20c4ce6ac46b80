"""Cost of running a model trained with normalization_scaling through the C ABI, on the GPU.

At 64 x 2048 and 64 x 720, graph-replayed calls, CUDA events around 20 replays per sample, the two routes of each
comparison alternated sample by sample (paired differences):
  - streaming, batch 1: delora_odometry_push (one projection per frame, the previous image cached) against the
    normalised route, delora_odometry_pairs_normalized at B = 1 on (previous scan, this scan) plus the device copy
    that makes this scan the previous one;
  - batches: delora_odometry_pairs_normalized against delora_odometry_pairs at B = 8 and 16;
  - the factor alone (delora_normalization_factors) at B = 1, 8, 16.
The card's name, power limit and SM clocks are read in the same run.

    python scripts/gpu_odometry_normalized.py [--samples 30] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from delora_b200 import ops, synthetic  # noqa: E402
from delora_b200.deploy import export  # noqa: E402
from delora_b200.deploy.capi import InferenceWorkspace  # noqa: E402
from delora_b200.models.model import OdometryModel  # noqa: E402

REPLAYS = 20


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unavailable"


def capture(fn):
    st = torch.cuda.current_stream()
    for _ in range(3):                      # warm-up: launcher caches, allocator
        fn()
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def per_call_us(g):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(REPLAYS):
        g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / REPLAYS


def paired(g_a, g_b, samples):
    """Alternating samples -> medians of each and of the paired difference b - a (us per call)."""
    for _ in range(5):
        per_call_us(g_a), per_call_us(g_b)
    ta, tb = [], []
    for k in range(samples):
        if k % 2:
            tb.append(per_call_us(g_b)); ta.append(per_call_us(g_a))
        else:
            ta.append(per_call_us(g_a)); tb.append(per_call_us(g_b))
    d = np.array(tb) - np.array(ta)
    return {"a_us": float(np.median(ta)), "b_us": float(np.median(tb)), "b_minus_a_us": float(np.median(d)),
            "b_minus_a_p10_p90_us": [float(np.percentile(d, 10)), float(np.percentile(d, 90))]}


def run_shape(h, w, samples, dev):
    cfg = synthetic.fov_config(h=h, w=w, device=dev)
    cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                "use_dropout": False})
    torch.manual_seed(0)
    model = OdometryModel(cfg).to(dev).eval()
    scans = []
    for i in range(16):
        s1, s2, _, _ = synthetic.make_pair(i, w_raw=2048, rings=64)
        scans += [s1, s2]
    n_stride = max(s.shape[1] for s in scans)
    pts_all = torch.zeros((len(scans), 3, n_stride), dtype=torch.float32)
    for i, s in enumerate(scans):
        pts_all[i, :, :s.shape[1]] = s
    pts_all = pts_all.to(dev)
    cnt_all = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32, device=dev)
    blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), cfg)).to(dev)
    out = {"n_stride": n_stride}

    # streaming, batch 1
    ws1 = InferenceWorkspace(export.desc_from_config(cfg, "kitti", n_stride, 1), blob)
    t = torch.zeros((16,), dtype=torch.float32, device=dev)
    ws1.push(pts_all[:1], cnt_all[:1], None)
    g_push = capture(lambda: ws1.push(pts_all[1:2], cnt_all[1:2], t))
    pair, pair_cnt = pts_all[:2].clone(), cnt_all[:2].clone()
    t1, f1 = torch.zeros((1, 4, 4), device=dev), torch.zeros((1,), device=dev)

    def norm_frame():
        ws1._call("delora_odometry_pairs_normalized", pair.data_ptr(), pair_cnt.data_ptr(), 1,
                  ws1.workspace.data_ptr(), t1.data_ptr(), None, f1.data_ptr())
        pair[0].copy_(pair[1])
        pair_cnt[0].copy_(pair_cnt[1])
    out["stream_push_vs_normalized"] = paired(g_push, capture(norm_frame), samples)

    # batches
    ws16 = InferenceWorkspace(export.desc_from_config(cfg, "kitti", n_stride, 16), blob)
    for b in (8, 16):
        pts, cnt = pts_all[:2 * b].contiguous(), cnt_all[:2 * b].contiguous()
        tb, pb, fb = (torch.zeros((b, 4, 4), device=dev), torch.zeros((b, 512), device=dev),
                      torch.zeros((b,), device=dev))
        args = (pts.data_ptr(), cnt.data_ptr(), b, ws16.workspace.data_ptr(), tb.data_ptr(), pb.data_ptr())
        g_p = capture(lambda: ws16._call("delora_odometry_pairs", *args))
        g_n = capture(lambda: ws16._call("delora_odometry_pairs_normalized", *args, fb.data_ptr()))
        out[f"pairs_vs_normalized_B{b}"] = paired(g_p, g_n, samples)

    for b in (1, 8, 16):
        pts, cnt = pts_all[:2 * b].contiguous(), cnt_all[:2 * b].contiguous()
        fb = torch.zeros((b,), device=dev)
        L = ws16._L
        g = capture(lambda: L.delora_normalization_factors(pts.data_ptr(), cnt.data_ptr(), b, n_stride, fb.data_ptr(),
                                                           ops._stream()))
        out[f"factor_B{b}_us"] = float(np.median([per_call_us(g) for _ in range(samples)]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=30)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "replays_per_sample": REPLAYS, "samples": args.samples}
    for h, w in ((64, 2048), (64, 720)):
        res[f"{h}x{w}"] = run_shape(h, w, args.samples, "cuda:0")
    res["gpu_after"] = gpu_info()
    line = json.dumps(res, indent=1)
    print(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line)


if __name__ == "__main__":
    main()
