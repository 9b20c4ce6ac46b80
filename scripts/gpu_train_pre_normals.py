"""What training on the reference's two-resolution recipe costs: delora_odometry_train_step with w_pre = 2250 (normals
at 64 x 2250, the points then projected at the model's 64 x 720) against w_pre = 0 (normals at 64 x 720), on one GPU.

1. Step time, B in {1, 4, 16} pairs, tanh, two heads, layers [2, 2, 2, 2], synthetic 64-ring scans of 2048 columns,
   on workspaces that start from the same weights: each setting's step captured into a CUDA graph, a sample = CUDA
   events around `--replays` back-to-back replays, the two settings alternating for `--rounds` samples each.  The cost
   of the option is the difference of each pair of adjacent samples (median, min, max).
2. The re-projection alone, on the 64 x 2250 grids of 2B = 32 scans: delora_project_grids_fwd (two launches) against
   the list path it replaces (delora_lists_from_images, the channels-first copies, delora_project_fwd,
   delora_grids_from_projection), each timed with CUDA events over `--reps` calls, alternating, and against the
   bytes the new kernels must move at 3.35 TB/s (H100 SXM data sheet HBM3 bandwidth).
Prints the card name, power limit and SM clocks of the run, and the result as JSON (with --out also to
DIR/train_pre_normals.json).

    python scripts/gpu_train_pre_normals.py [--rounds 15] [--replays 20] [--reps 50] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12
H, W, W_PRE, W_RAW = 64, 720, 2250, 2048


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def summary(ts):
    return {"median": statistics.median(ts), "min": min(ts), "max": max(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4,16")
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for train_pre_normals.json (default: print only)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    from delora_b200 import _lib, ops, synthetic
    from delora_b200.deploy import export
    from delora_b200.models.model import OdometryModel
    dev = torch.device("cuda:0")
    L = _lib.lib()
    st = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    batches = [int(v) for v in a.batches.split(",")]
    b_max = max(batches)
    pairs = [synthetic.make_pair(i, w_raw=W_RAW, rings=H)[:2] for i in range(b_max)]
    n_max = max(max(x.shape[1], y.shape[1]) for x, y in pairs)

    cfg = synthetic.fov_config(h=H, w=W, device="cuda:0")
    cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                "use_dropout": False, "lambda_po2pl": 1.0})
    torch.manual_seed(0)
    blob = torch.from_numpy(export.pack_state_dict(OdometryModel(cfg).state_dict(), cfg)).to(dev)
    nb = cfg["kitti"]["neighborhood_side_length"]
    hp = _lib.OdometryTrainParams(lr=1e-6, beta1=0.9, beta2=0.999, eps=1e-8, lambda_po2pl=1.0, loss_flags=2 | 4,
                                  nb_h=nb[0], nb_w=nb[1], epsilon_range=cfg["epsilon_range"],
                                  min_neighbors=cfg["min_num_points_in_neighborhood_to_determine_point_class"])
    res = {"card": card(), "H": H, "W": W, "w_pre": W_PRE, "scan_columns": W_RAW, "steps": {}}

    for b in batches:
        scans = [p[0] for p in pairs[:b]] + [p[1] for p in pairs[:b]]
        pts = torch.zeros((2 * b, 3, n_max), dtype=torch.float32)
        for i, s in enumerate(scans):
            pts[i, :, :s.shape[1]] = s
        counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
        pts, counts = pts.to(dev), counts.to(dev)
        runs = {}
        for w_pre in (0, W_PRE):
            d = export.desc_from_config(cfg, "kitti", n_max, b)
            d.w_pre = w_pre
            ws = torch.empty((int(L.delora_odometry_train_workspace_bytes(ctypes.byref(d))),), dtype=torch.uint8,
                             device=dev)
            _lib.check(L.delora_odometry_train_init(ctypes.byref(d), blob.data_ptr(), ws.data_ptr(), st()), "init")
            runs[w_pre] = (d, ws)

        def step(w_pre):
            d, ws = runs[w_pre]
            _lib.check(L.delora_odometry_train_step(ctypes.byref(d), ctypes.byref(hp), pts.data_ptr(), counts.data_ptr(),
                                                    b, ws.data_ptr(), None, None, None, None, st()), "train_step")

        for _ in range(a.warmup):
            step(0)
            step(W_PRE)
        torch.cuda.synchronize()
        # one captured step per setting: a sample is the mean of `replays` back-to-back replays (no host gaps), the
        # settings alternate sample by sample, and the cost of the option is the paired difference of adjacent samples
        graphs = {}
        for w_pre in (0, W_PRE):
            graphs[w_pre] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[w_pre]):
                step(w_pre)
            graphs[w_pre].replay()
        torch.cuda.synchronize()
        t = {0: [], W_PRE: []}
        for _ in range(a.rounds):
            for w_pre in (0, W_PRE):
                t[w_pre].append(timed(graphs[w_pre].replay, a.replays))
        deltas = [y - x for x, y in zip(t[0], t[W_PRE])]
        res["steps"][b] = {"workspace_bytes": {str(k): int(v[1].numel()) for k, v in runs.items()},
                           "samples": a.rounds, "replays_per_sample": a.replays,
                           "step_ms_w_pre_0": summary(t[0]), f"step_ms_w_pre_{W_PRE}": summary(t[W_PRE]),
                           "added_ms_paired": summary(deltas)}
        del runs, graphs
        torch.cuda.empty_cache()

    # the re-projection alone, 2 * b_max scans
    scans = [p[0] for p in pairs] + [p[1] for p in pairs]
    s = len(scans)
    pts = torch.full((s, 3, n_max), float("nan"))
    for i, c in enumerate(scans):
        pts[i, :, :c.shape[1]] = c
    counts = torch.tensor([c.shape[1] for c in scans], dtype=torch.int32)
    pts, counts = pts.to(dev), counts.to(dev)
    hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
    image_pre, _, pg, ng = ops.project_normals(pts, counts, H, W_PRE, hf, vf)
    normals = ops.normals(image_pre)
    torch.cuda.synchronize()

    def new():
        return ops.project_grids(pg, ng, H, W_PRE, W, hf, vf, index_map=False)

    def old():
        pts4, nrm4, _, n = ops.lists_from_images(image_pre, normals)
        p = pts4[:, :, :3].transpose(1, 2).contiguous()
        q = nrm4[:, :, :3].transpose(1, 2).contiguous()
        img, imap = ops.project(p, n, H, W, hf, vf)
        return img, ops.grids_from_projection(p, q, imap)

    a_img, _, a_pg, a_ng = new()
    b_img, (b_pg, b_ng) = old()
    torch.cuda.synchronize()
    same = all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in ((a_img, b_img), (a_pg, b_pg),
                                                                                     (a_ng, b_ng)))
    for _ in range(5):
        new()
        old()
    tn, to = [], []
    for _ in range(5):
        tn.append(timed(new, a.reps))
        to.append(timed(old, a.reps))
    # bytes the two kernels must move: the pre-resolution points grid once (scatter), per model pixel its key
    # read + re-arm, the image, and the two grids; per kept point its two pre-grid entries (gathers)
    kept = int((a_pg[:, :, 3].view(torch.int32) >= 0).sum())
    bytes_ = s * H * W_PRE * 16 + s * H * W * (16 + 16 + 32) + kept * 32
    # the public wrapper allocates its four outputs with torch each call; time the bare C call too
    img = torch.empty((s, 4, H, W), device=dev)
    opg, ong = torch.empty((s, H * W, 4), device=dev), torch.empty((s, H * W, 4), device=dev)
    keys = ops._keys(dev, s, H * W)

    def bare():
        _lib.check(L.delora_project_grids_fwd(pg.data_ptr(), ng.data_ptr(), s, H, W_PRE, W, hf[0], hf[1], vf[0], vf[1], 0,
                                              keys.data_ptr(), img.data_ptr(), None, opg.data_ptr(), ong.data_ptr(),
                                              st()), "project_grids")

    bare()
    tb = [timed(bare, a.reps) for _ in range(5)]
    res["reprojection"] = {
        "scans": s, "bit_identical": same, "kept_points": kept,
        "project_grids_ms": summary(tb), "ops_project_grids_ms": summary(tn), "list_path_ms": summary(to),
        "bytes": bytes_, "floor_ms": bytes_ / HBM_BYTES_PER_S * 1e3,
        "bandwidth_TB_s": bytes_ / (statistics.median(tb) * 1e-3) / 1e12}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "train_pre_normals.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
