"""What the po2po_alone objective (DELORA_LOSS_PO2PO_ALONE) costs on the GPU against the shipped objective.

Per call, ms at B = S in {1, 16} for 64 x 720 with w_pre 2250 and 64 x 2048 with w_pre 0, on the same near-identity
weights (measure.near_identity_blob), lr 0 (Adam runs, the weights stay put, so every sample times the same work):
  step_shipped   delora_odometry_train_step, DELORA_LOSS_PO2PL | _PL2PL (normals estimated, 7 x 11);
  step_alone     delora_odometry_train_step, DELORA_LOSS_PO2PO | _PO2PO_ALONE (the points-only front end);
  adapt_shipped  delora_odometry_streams_push_adapt, update = 1, the shipped objective;
  adapt_alone    delora_odometry_streams_push_adapt, update = 1, po2po_alone;
  front_normals  delora_project_normals_fwd of the 2B scans of a step at H x (w_pre or W);
  front_points   delora_project_points_fwd of the same scans.
The two objectives pair different points, so the ICP's work differs too; the front-end rows isolate the projection and
normals.  Every side is one captured graph of two calls (the adapting streams alternate between the two scans of each
pair), replayed back to back over at least --seconds per sample; the sides alternate and the medians and every sample
are reported.  The card's name, power limit and SM clocks are read in the same run.  Writes train_objective.json to
--out.

    python scripts/gpu_train_objective.py [--seconds 0.3] [--samples 5] [--out DIR]
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

SIZES = ((64, 720, 2250), (64, 2048, 0))
BATCHES = (1, 16)
OBJECTIVES = {"shipped": ops.LOSS_PO2PL | ops.LOSS_PL2PL, "alone": ops.LOSS_PO2PO | ops.LOSS_PO2PO_ALONE}


class Sides:
    """Every side's workspaces and graphs for B pairs / S = B streams."""

    def __init__(self, cfg, blob, pairs, n_stride, w_pre):
        B = len(pairs)
        h, w = cfg["kitti"]["vertical_cells"], cfg["kitti"]["horizontal_cells"]
        d = export.desc_from_config(cfg, "kitti", n_stride, B, preprocessing_normals=w_pre > 0)
        self.stacked = [staged([p[i] for p in pairs] + [p[1 - i] for p in pairs], n_stride) for i in (0, 1)]
        self.frames = [staged([p[i] for p in pairs], n_stride) for i in (0, 1)]
        self.active = torch.ones((B,), dtype=torch.int32, device=DEV)
        self.T = torch.zeros((B, 16), dtype=torch.float32, device=DEV)
        self.valid = torch.zeros((B,), dtype=torch.int32, device=DEV)
        self.losses = torch.zeros((B, ops.LOSS_ROW), dtype=torch.float32, device=DEV)
        self.train, self.adapt, self.fn = {}, {}, {}
        for name, flags in OBJECTIVES.items():
            hp = capi.train_params(cfg, 0.0, loss_flags=flags)
            self.train[name] = capi.TrainingWorkspace(d, blob, hp)
            self.adapt[name] = capi.AdaptiveStreamsWorkspace(d, blob, hp)
            self.fn[f"step_{name}"] = capture(lambda n=name: self.steps(n), warmup=1).replay
            self.fn[f"adapt_{name}"] = capture(lambda n=name: self.ticks(n), warmup=1).replay
        wf = w_pre or w
        hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
        for name, op in (("normals", ops.project_normals), ("points", ops.project_points)):
            self.fn[f"front_{name}"] = capture(lambda op=op: [op(p, c, h, wf, hf, vf) for p, c in self.stacked],
                                               warmup=1).replay
        torch.cuda.synchronize()
        a = ops.project_normals(*self.stacked[0], h, wf, hf, vf)
        b = ops.project_points(*self.stacked[0], h, wf, hf, vf)
        torch.cuda.synchronize()
        self.front_same = all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a[:3], b[:3]))
        self.front_zero_normals = not bool(b[3].view(torch.int32).any())

    def steps(self, name):
        for pts, counts in self.stacked:
            self.train[name].step(pts, counts, outputs=False)

    def ticks(self, name):
        for pts, counts in self.frames:
            self.adapt[name].push(pts, counts, self.active, self.T, self.valid, self.losses, update=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.3)
    ap.add_argument("--samples", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": GPU_QUERY, "seconds_per_sample": args.seconds, "lr": 0.0,
           "sizes": {}}
    for h, w, w_pre in SIZES:
        cfg = model_config(h, w)
        if w_pre:
            cfg["kitti"]["horizontal_cells_preprocessing"] = w_pre
        blob = near_identity_blob(cfg)
        pairs_all = pairs(h, max(BATCHES))
        stride = n_stride(pairs_all)
        per_b = {}
        for B in BATCHES:
            sides = Sides(cfg, blob, pairs_all[:B], stride, w_pre)
            samples = alternate(sides.fn, args.samples,
                                lambda fn: events_ms(fn, seconds=args.seconds)[0] / 2)      # two calls per replay
            torch.cuda.synchronize()
            med = {k: statistics.median(v) for k, v in samples.items()}
            per_b[B] = {**{f"{k}_ms_per_call": m for k, m in med.items()},
                        **{f"{k}_samples_ms": v for k, v in samples.items()},
                        "step_alone_minus_shipped_ms": med["step_alone"] - med["step_shipped"],
                        "adapt_alone_minus_shipped_ms": med["adapt_alone"] - med["adapt_shipped"],
                        "front_points_minus_normals_ms": med["front_points"] - med["front_normals"],
                        "front_same_bits": sides.front_same, "front_zero_normals": sides.front_zero_normals}
            del sides
            torch.cuda.empty_cache()
        res["sizes"][f"{h}x{w}_wpre{w_pre}"] = {"n_stride": stride, "batch_B": per_b}
    res["gpu_after"] = gpu_info()
    emit(res, args.out and os.path.join(args.out, "train_objective.json"))


if __name__ == "__main__":
    main()
