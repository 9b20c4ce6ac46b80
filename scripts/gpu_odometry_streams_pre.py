"""What serving several sensors on the reference's two-resolution recipe costs on the GPU, and how often its image
differs from the raw-scan one.

Per tick, ms at S in {1, 4, 16} for 64 x 720 and 64 x 2048, both with w_pre 2250, all streams active,
graph-replayed, on the same near-identity weights (measure.near_identity_blob):
  push           delora_odometry_streams_push (raw scans projected at H x W, the image cache);
  push_residual  delora_odometry_streams_push_residual (the same, plus normals at H x W and the ICP);
  push_pre       delora_odometry_streams_push_pre (projection + normals at H x w_pre, both frames of every pair
                 projected again at H x W, the ICP, the cache write).
Each stream alternates between the two scans of a synthetic pair, so every tick sees a consecutive frame; one captured
graph holds two ticks.  The three sides alternate (a, b, c, a, b, c, ...) over at least --seconds of work per sample;
the medians and every sample are reported.  Also, per size, the fraction of H x W pixels whose image (x, y, z, range)
differs between the raw-scan projection (delora_project_fwd) and the recipe's (projection + normals at H x w_pre, then
delora_project_grids_fwd), over the scans used here.  The card's name, power limit and SM clocks are read in the same
run.  Writes odometry_streams_pre.json to --out.

    python scripts/gpu_odometry_streams_pre.py [--seconds 0.5] [--samples 5] [--out DIR]
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from delora_b200 import ops  # noqa: E402
from delora_b200.deploy import capi, export  # noqa: E402
from measure import (DEV, GPU_QUERY, alternate, capture, emit, events_ms, gpu_info, model_config,  # noqa: E402
                     n_stride, near_identity_blob, pairs, staged)

SIZES = ((64, 720), (64, 2048))
W_PRE = 2250
STREAMS = (1, 4, 16)


class StreamTicks:
    """A streams workspace of one kind and a graph of two ticks: every stream's scan_1, then its scan_2."""

    def __init__(self, cfg, blob, pairs, n_stride, kind):
        S = len(pairs)
        d = export.desc_from_config(cfg, "kitti", n_stride, S, preprocessing_normals=True)
        rp = capi.residual_params(cfg)
        self.ws = {"push": lambda: capi.StreamsWorkspace(d, blob),
                   "push_residual": lambda: capi.ResidualStreamsWorkspace(d, blob, rp),
                   "push_pre": lambda: capi.PreStreamsWorkspace(d, blob, rp)}[kind]()
        self.frames = [staged([p[i] for p in pairs], n_stride) for i in (0, 1)]
        self.active = torch.ones((S,), dtype=torch.int32, device=DEV)
        self.out = (torch.zeros((S, 16), dtype=torch.float32, device=DEV),
                    torch.zeros((S,), dtype=torch.int32, device=DEV))
        if kind != "push":
            self.out += (torch.zeros((S, ops.LOSS_ROW), dtype=torch.float32, device=DEV),)
        self.graph = capture(self.two_ticks, warmup=1)      # the warm-up caches the first frames

    def two_ticks(self):
        for pts, counts in self.frames:
            self.ws.push(pts, counts, self.active, *self.out)


def differing_pixels(cfg, scans, n_stride):
    """-> (pixels whose image differs between the raw-scan and the recipe projection, pixels in all)."""
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = cfg["horizontal_field_of_view"], ds["vertical_field_of_view"]
    pts, counts = staged(scans, n_stride)
    raw, _ = ops.project(pts, counts, h, w, hf, vf)
    _, _, pg, ng = ops.project_normals(pts, counts, h, W_PRE, hf, vf, ds["neighborhood_side_length"],
                                       cfg["epsilon_range"], cfg["min_num_points_in_neighborhood_to_determine_point_class"])
    recipe, _, _, _ = ops.project_grids(pg, ng, h, W_PRE, w, hf, vf, index_map=False)
    diff = (raw.view(torch.int32) != recipe.view(torch.int32)).any(dim=1)
    return int(diff.sum()), diff.numel()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": GPU_QUERY,
           "seconds_per_sample": args.seconds, "w_pre": W_PRE, "sizes": {}}
    for h, w in SIZES:
        cfg = model_config(h, w)
        cfg["kitti"]["horizontal_cells_preprocessing"] = W_PRE
        blob = near_identity_blob(cfg)
        pairs_all = pairs(h, max(STREAMS))
        stride = n_stride(pairs_all)
        n_diff, n_pix = differing_pixels(cfg, [s for p in pairs_all for s in p], stride)
        per_s = {}
        for S in STREAMS:
            sides = {k: StreamTicks(cfg, blob, pairs_all[:S], stride, k) for k in ("push", "push_residual", "push_pre")}
            samples = alternate({k: side.graph.replay for k, side in sides.items()}, args.samples,
                                lambda fn: events_ms(fn, seconds=args.seconds)[0] / 2)     # two ticks per replay
            torch.cuda.synchronize()
            med = {k: statistics.median(v) for k, v in samples.items()}
            per_s[S] = {**{f"{k}_ms_per_tick": m for k, m in med.items()},
                        **{f"{k}_samples_ms": v for k, v in samples.items()},
                        "push_pre_over_push_ms": med["push_pre"] - med["push"],
                        "push_pre_over_push_residual_ms": med["push_pre"] - med["push_residual"],
                        "push_pre_all_valid": bool(sides["push_pre"].out[1].all()),
                        "workspace_MiB": {k: s.ws.workspace.numel() / 2**20 for k, s in sides.items()}}
            del sides
            torch.cuda.empty_cache()
        res["sizes"][f"{h}x{w}"] = {"n_stride": stride, "streams_S": per_s,
                                    "recipe_vs_raw_image": {"differing_pixels": n_diff, "pixels": n_pix,
                                                            "fraction": n_diff / n_pix,
                                                            "scans": 2 * max(STREAMS)}}
    res["gpu_after"] = gpu_info()
    emit(res, args.out and os.path.join(args.out, "odometry_streams_pre.json"))


if __name__ == "__main__":
    main()
