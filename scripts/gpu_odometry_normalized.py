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
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from delora_b200 import ops  # noqa: E402
from delora_b200.deploy import export  # noqa: E402
from delora_b200.deploy.capi import InferenceWorkspace  # noqa: E402
from measure import (DEV, capture, emit, events_ms, gpu_info, model_config, n_stride, paired, pairs,  # noqa: E402
                     staged, untrained_blob)

REPLAYS = 20


def us(g):
    return events_ms(g.replay, calls=REPLAYS)[0] * 1e3


def compare(g_a, g_b, samples):
    """Samples in the order a, b, then b, a, ... -> medians of each and of the paired difference b - a (us per call)."""
    for _ in range(5):
        us(g_a), us(g_b)
    ta, tb = [], []
    for k in range(samples):
        if k % 2:
            tb.append(us(g_b)); ta.append(us(g_a))
        else:
            ta.append(us(g_a)); tb.append(us(g_b))
    d, med = paired(ta, tb)
    return {"a_us": float(np.median(ta)), "b_us": float(np.median(tb)), "b_minus_a_us": med,
            "b_minus_a_p10_p90_us": [float(np.percentile(d, 10)), float(np.percentile(d, 90))]}


def run_shape(h, w, samples):
    cfg = model_config(h, w)
    ps = pairs(64, 16)
    stride = n_stride(ps)
    pts_all, cnt_all = staged([s for p in ps for s in p], stride)
    blob = untrained_blob(cfg)
    out = {"n_stride": stride}

    # streaming, batch 1
    ws1 = InferenceWorkspace(export.desc_from_config(cfg, "kitti", stride, 1), blob)
    t = torch.zeros((16,), dtype=torch.float32, device=DEV)
    ws1.push(pts_all[:1], cnt_all[:1], None)
    g_push = capture(lambda: ws1.push(pts_all[1:2], cnt_all[1:2], t), warmup=3)
    pair, pair_cnt = pts_all[:2].clone(), cnt_all[:2].clone()
    t1, f1 = torch.zeros((1, 4, 4), device=DEV), torch.zeros((1,), device=DEV)

    def norm_frame():
        ws1._call("delora_odometry_pairs_normalized", pair.data_ptr(), pair_cnt.data_ptr(), 1,
                  ws1.workspace.data_ptr(), t1.data_ptr(), None, f1.data_ptr())
        pair[0].copy_(pair[1])
        pair_cnt[0].copy_(pair_cnt[1])
    out["stream_push_vs_normalized"] = compare(g_push, capture(norm_frame, warmup=3), samples)

    # batches
    ws16 = InferenceWorkspace(export.desc_from_config(cfg, "kitti", stride, 16), blob)
    for b in (8, 16):
        pts, cnt = pts_all[:2 * b].contiguous(), cnt_all[:2 * b].contiguous()
        tb, pb, fb = (torch.zeros((b, 4, 4), device=DEV), torch.zeros((b, 512), device=DEV),
                      torch.zeros((b,), device=DEV))
        args = (pts.data_ptr(), cnt.data_ptr(), b, ws16.workspace.data_ptr(), tb.data_ptr(), pb.data_ptr())
        g_p = capture(lambda: ws16._call("delora_odometry_pairs", *args), warmup=3)
        g_n = capture(lambda: ws16._call("delora_odometry_pairs_normalized", *args, fb.data_ptr()), warmup=3)
        out[f"pairs_vs_normalized_B{b}"] = compare(g_p, g_n, samples)

    for b in (1, 8, 16):
        pts, cnt = pts_all[:2 * b].contiguous(), cnt_all[:2 * b].contiguous()
        fb = torch.zeros((b,), device=DEV)
        L = ws16._L
        g = capture(lambda: L.delora_normalization_factors(pts.data_ptr(), cnt.data_ptr(), b, stride, fb.data_ptr(),
                                                           ops._stream()), warmup=3)
        out[f"factor_B{b}_us"] = float(np.median([us(g) for _ in range(samples)]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=30)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "replays_per_sample": REPLAYS, "samples": args.samples}
    for h, w in ((64, 2048), (64, 720)):
        res[f"{h}x{w}"] = run_shape(h, w, args.samples)
    res["gpu_after"] = gpu_info()
    emit(res, args.json)


if __name__ == "__main__":
    main()
