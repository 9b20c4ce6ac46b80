"""Exploration on the GPU box: per-operator timings of the batched pipeline (not the bench)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from delora_b200 import synthetic, _lib, ops
from delora_b200.pipeline import ScanPairPipeline

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
W = int(sys.argv[2]) if len(sys.argv) > 2 else 2048
cfg = synthetic.fov_config(h=64, w=W)
hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
pairs = [synthetic.make_pair(i, w_raw=2048) for i in range(B)]
nmax = max(max(p[0].shape[1], p[1].shape[1]) for p in pairs)
pipe = ScanPairPipeline(B, nmax, 64, W, hf, vf)
pipe.load([p[0] for p in pairs], [p[1] for p in pairs], torch.stack([p[3] for p in pairs]))
L = _lib.lib()
st = torch.cuda.current_stream().cuda_stream
b2, H, hw = 2 * B, 64, 64 * W

def t_proj():
    _lib.check(L.delora_project_fwd(pipe.points.data_ptr(), pipe.n_points.data_ptr(), b2, 3, pipe.N, H, W, hf[0], hf[1], vf[0], vf[1], 0, pipe.keys.data_ptr(), pipe.image.data_ptr(), pipe.index_map.data_ptr(), st), "p")
def t_norm():
    _lib.check(L.delora_normals_fwd(pipe.image.data_ptr(), b2, 4, H, W, 7, 11, 0.5, 10, None, pipe.pts_grid.data_ptr(), pipe.nrm_grid.data_ptr(), st), "n")
def t_icp():
    _lib.check(L.delora_icp_dense_fwd_bwd(pipe.pts_grid.data_ptr() + B * hw * 16, pipe.nrm_grid.data_ptr() + B * hw * 16, pipe.transform.data_ptr(), pipe.pts_grid.data_ptr(), pipe.nrm_grid.data_ptr(), B, H, W, hf[0], hf[1], vf[0], vf[1], 1.0, 6, pipe.losses.data_ptr(), pipe.grad_T.data_ptr(), pipe.icp_scratch.data_ptr(), st), "i")

flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
def timeit(fn, name, iters=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    print(f"{name:12s} median {ts[len(ts)//2]*1e3:9.1f} us   min {ts[0]*1e3:9.1f} us")
    return ts[len(ts)//2]

print(f"B={B} pairs, 64x{W}, N~{nmax}")
tot = 0
for fn, name in ((t_proj, "projection"), (t_norm, "normals"), (t_icp, "icp_dense")):
    tot += timeit(fn, name)
step = timeit(lambda: pipe.step(), "full step")
print(f"sum of parts {tot*1e3:.1f} us; step {step*1e3:.1f} us -> {B/(step*1e-3):.0f} pairs/s")
print("losses", pipe.losses[0].tolist())
import json
from torch.profiler import profile, ProfilerActivity

def t_icp_stats():
    _lib.check(L.delora_icp_dense_fwd_bwd(pipe.pts_grid.data_ptr() + B * hw * 16, pipe.nrm_grid.data_ptr() + B * hw * 16, pipe.transform.data_ptr(), pipe.pts_grid.data_ptr(), pipe.nrm_grid.data_ptr(), B, H, W, hf[0], hf[1], vf[0], vf[1], 1.0, 6 | ops.ICP_STATS, pipe.losses.data_ptr(), pipe.grad_T.data_ptr(), pipe.icp_scratch.data_ptr(), st), "i")
def stats(tag):
    ops.icp_stats(reset=True); t_icp_stats(); torch.cuda.synchronize()
    print(tag, json.dumps(ops.icp_stats(reset=True)))

def split(tag, reps=10):
    """Per-kernel split of one ICP call (torch.profiler, a run of its own; L2 flushed before every call)."""
    t_icp(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            flush.zero_(); t_icp()
        torch.cuda.synchronize()
    parts = []
    for e in prof.key_averages():
        if "icp" in e.key or "extents" in e.key:
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            parts.append((e.key.split("(")[0].split("<")[0].replace("void ", "").replace("delora::", ""), us / reps))
    print(f"split({tag})", "  ".join(f"{n} {t:.1f} us" for n, t in sorted(parts, key=lambda x: -x[1])),
          f"  sum {sum(t for _, t in parts):.1f} us")

def case(tag, iters=20):
    timeit(t_icp, "icp_" + tag, iters=iters)
    split(tag)
    stats(f"stats({tag})")
    print(f"losses({tag})", pipe.losses[0].tolist())

case("predictedT")
# misaligned cases (what an untrained network produces): identity transform instead of the (nearly correct)
# predicted one -> NN distances ~0.5 m; and a bad transform (2 m, 10 deg)
import math
saved_T = pipe.transform.clone()
pipe.transform.copy_(torch.eye(4, device="cuda")[:3, :].reshape(1, 12).repeat(B, 1))
case("identityT")
tb = torch.from_numpy(synthetic.transform_matrix(2.0, 1.0, 0.3, math.radians(10.0), math.radians(2.0), 0.0)).float().cuda()
pipe.transform.copy_(tb[:3, :].reshape(1, 12).repeat(B, 1))
case("badT", iters=5)
pipe.transform.copy_(saved_T)
