"""-m gpu: training through the C ABI on the reference's two-resolution recipe (descriptor w_pre > 0): normals at
H x w_pre, the points that won a preprocessing pixel then projected at the model's H x W.

The Python step built from the mirror is the reference's data path: Preprocesser.preprocess_scans in memory (the
offline stage's row-major point and normal lists), ops.project at W and ops.grids_from_projection (Deployer.step), then
the tensor-core model, the fused ICP losses, mean over the pairs, backward.  The bounds are those of
test_gpu_odometry_train_capi.py (same model, same kernels from the images on)."""
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H

pytestmark = pytest.mark.gpu
DEV = H.DEV


SIZES = [(64, 720, 2048, 2250), (16, 259, 512, 512)]                   # H, W, w_raw, w_pre
VARIANTS = [("tanh", False), ("relu", False), ("tanh", True), ("relu", True)]
STEP_CASES = [pytest.param(act, single, *size, b, id="-".join(map(str, (act, single) + size + (b,))))
              for size in SIZES for b in (1, 2, 4) for act, single in VARIANTS]


@pytest.mark.parametrize("act,single,h,w,w_raw,w_pre,b", STEP_CASES)
def test_step_matches_the_reference_recipe(cuda_lib, act, single, h, w, w_raw, w_pre, b):
    cfg = H.config(h, w, act, single)
    model = H.model(cfg, near_identity=True)
    pairs = H.pairs(h, w_raw, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    tr = H.trainer(cfg, n_stride, b, H.blob(model, cfg), w_pre=w_pre)
    losses, T, pooled, grads = tr.step(pts, counts)
    py = H.python_step(model, cfg, pts, counts, w_pre=w_pre)
    torch.cuda.synchronize()
    assert torch.equal(pooled, py.pooled), "pooled features differ from the reference recipe's"
    t_err = (T - py.T).abs().max().item()
    assert t_err <= 1e-5, f"max |T - T_py| = {t_err:.3e}"
    l_err = H.rel(losses[:, :3], py.losses[:, :3])
    assert l_err <= 1e-5, f"losses differ by {l_err:.3e} (relative)"
    tail, trunk = H.grad_spread(H.grad_dict(grads, cfg), py.grads)
    print(f"\n[{h}x{w} w_pre={w_pre} B={b} {act} single={single}] T {t_err:.2e}  losses {l_err:.2e}  grads: tail "
          f"{tail:.2e}, trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= H.TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"


def test_adam_is_torch_adam(cuda_lib):
    """The update after a w_pre step is torch's Adam on that step's gradient."""
    lr = 1e-3
    cfg = H.config(16, 259, "tanh", False)
    model = H.model(cfg, 1, near_identity=True)
    pairs = H.pairs(16, 512, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob0 = H.blob(model, cfg)
    tr = H.trainer(cfg, n_stride, 2, blob0, lr, w_pre=512)
    g = tr.step(pts, counts)[3]
    from delora_b200.deploy import export
    from delora_b200.models.model import OdometryModel
    m = OdometryModel(cfg).to(DEV)
    m.load_state_dict(export.unpack_blob(blob0.cpu().numpy(), cfg))
    opt = torch.optim.Adam(m.parameters(), lr=lr, fused=True)
    gd = H.grad_dict(g, cfg)
    for k, p in m.named_parameters():
        p.grad = gd[k].to(DEV)
    opt.step()
    got = H.grad_dict(tr.weights(), cfg)
    worst = max(H.rel(got[k].to(DEV), p.detach()) for k, p in m.named_parameters())
    assert worst <= 1e-6, f"the master weights differ from torch's Adam by {worst:.3e}"


def _zero_free(pairs):
    return tuple(tuple(s[:, (s != 0).all(dim=0)] for s in p) for p in pairs)


def test_same_width_is_the_plain_step(cuda_lib):
    """w_pre == W re-projects every kept point into its own pixel: the step is bit-identical to w_pre = 0 (on clouds
    without exact zero coordinates, which are image pixels but not valid cells)."""
    cfg = H.config(64, 720, "tanh", False)
    model = H.model(cfg, 2, near_identity=True)
    pairs = _zero_free(H.pairs(64, 1024, 2))
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    a, b = H.trainer(cfg, n_stride, 2, blob, 1e-4, w_pre=0), H.trainer(cfg, n_stride, 2, blob, 1e-4, w_pre=720)
    for _ in range(2):
        x, y = a.step(pts, counts), b.step(pts, counts)
        torch.cuda.synchronize()
        for u, v, name in zip(x, y, ("losses", "T", "pooled", "grads")):
            assert torch.equal(u, v), f"w_pre = W: {name} differ from w_pre = 0"


def test_the_option_changes_the_objective(cuda_lib):
    """On the same 64 x 720 scans, normals at 64 x 2250 give other losses than normals at 64 x 720."""
    cfg = H.config(64, 720, "tanh", False)
    model = H.model(cfg, 3, near_identity=True)
    pairs = H.pairs(64, 2048, 4)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    plain = H.trainer(cfg, n_stride, 4, blob, w_pre=0).step(pts, counts)
    pre = H.trainer(cfg, n_stride, 4, blob, w_pre=2250).step(pts, counts)
    torch.cuda.synchronize()
    lam = float(cfg["lambda_po2pl"])
    obj = [(l[:, 0] + lam * l[:, 1] + l[:, 2]).mean().item() for l in (plain[0], pre[0])]
    rel = [((pre[0][:, i] - plain[0][:, i]).abs() / plain[0][:, i].abs()).max().item() for i in (1, 2)]
    pairs_n = [plain[0][:, 3].sum().item(), pre[0][:, 3].sum().item()]
    gdiff = H.rel(pre[3], plain[3])
    print(f"\n[64x720, B=4] objective w_pre=0 {obj[0]:.6e}  w_pre=2250 {obj[1]:.6e}  (relative {abs(obj[1] - obj[0]) / obj[0]:.3e}); "
          f"po2pl max rel {rel[0]:.3e}, pl2pl max rel {rel[1]:.3e}; pairs {pairs_n[0]:.0f} vs {pairs_n[1]:.0f}; "
          f"gradient blob max-abs difference / max-abs {gdiff:.3e}")
    assert not torch.equal(plain[0][:, :3], pre[0][:, :3])
    assert abs(obj[1] - obj[0]) > 1e-4 * obj[0]


def test_deterministic_and_graph_replay(cuda_lib):
    cfg = H.config(64, 720, "relu", False)
    model = H.model(cfg, 4, near_identity=True)
    pairs = H.pairs(64, 2048, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    a, b = H.trainer(cfg, n_stride, 2, blob, 1e-4, w_pre=2250), H.trainer(cfg, n_stride, 2, blob, 1e-4, w_pre=2250)
    for _ in range(3):
        a.step(pts, counts, outputs=False)
        b.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert torch.equal(a.weights(), b.weights()), "two workspaces with the same steps differ"

    eager, graphed = H.trainer(cfg, n_stride, 2, blob, 1e-4, w_pre=2250), H.trainer(cfg, n_stride, 2, blob, 1e-4, w_pre=2250)
    for _ in range(3):
        eager.step(pts, counts, outputs=False)
    graphed.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.step(pts, counts, outputs=False)
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(graphed.weights(), eager.weights()), "graph replay differs from eager stepping"


def test_batch_size_may_change_between_steps(cuda_lib):
    cfg = H.config(64, 720, "tanh", True)
    model = H.model(cfg, 5, near_identity=True)
    pairs = H.pairs(64, 2048, 4)
    n_stride = H.n_stride(pairs)
    tr = H.trainer(cfg, n_stride, 4, H.blob(model, cfg), 1e-4, w_pre=2250)
    for bsz in (4, 1, 3):
        pts, counts = H.stack_pairs(pairs[:bsz], n_stride)
        before = tr.weights()
        got = tr.step(pts, counts)
        fresh = H.trainer(cfg, n_stride, 4, before, 1e-4, w_pre=2250).step(pts, counts)
        torch.cuda.synchronize()
        for x, y, name in zip(got, fresh, ("losses", "T", "pooled", "grads")):
            assert torch.equal(x, y), f"B={bsz}: {name} differ from a fresh workspace"


def test_finetune_example_program_with_preprocessing_normals(cuda_lib, tmp_path):
    """examples/odometry_finetune.c on a .dlw exported with preprocessing normals: it trains with w_pre from the file."""
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    cfg["kitti"]["horizontal_cells_preprocessing"] = 1024
    model = H.model(cfg, 6, near_identity=True)
    dlw, out = os.path.join(tmp_path, "in.dlw"), os.path.join(tmp_path, "out.dlw")
    desc = export.desc_from_config(cfg, "kitti", 4096, 2, preprocessing_normals=True)
    assert desc.w_pre == 1024
    export.write_dlw(dlw, desc, export.pack_state_dict(model.state_dict(), cfg))
    bins = []
    for i in range(4):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    exe = H.build_example("odometry_finetune", tmp_path, link=True)
    r = subprocess.run([exe, dlw, out, "3", "1e-4"] + bins, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert len(r.stdout.strip().splitlines()) == 3
    assert "preprocessing resolution 16x1024" in r.stderr, r.stderr
    h, d, blob = export.read_dlw(out)
    assert (d.H, d.W, d.max_batch, d.w_pre) == (16, 720, 2, 1024)
    scans = [torch.from_numpy(np.fromfile(p, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()) for p in bins]
    tr = H.trainer(cfg, 4096, 2, H.blob(model, cfg), 1e-4, w_pre=1024)
    plain = H.trainer(cfg, 4096, 2, H.blob(model, cfg), 1e-4, w_pre=0)
    for ks in ((0, 1), (2, 0), (1, 2)):
        pts, counts = H.stack_pairs([(scans[k], scans[k + 1]) for k in ks], 4096)
        tr.step(pts, counts, outputs=False)
        plain.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert np.array_equal(tr.weights().cpu().numpy(), blob)
    assert not np.array_equal(plain.weights().cpu().numpy(), blob)
