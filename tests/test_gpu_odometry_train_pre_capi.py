"""-m gpu: training through the C ABI on the reference's two-resolution recipe (descriptor w_pre > 0): normals at
H x w_pre, the points that won a preprocessing pixel then projected at the model's H x W.

The Python step built from the mirror is the reference's data path: Preprocesser.preprocess_scans in memory (the
offline stage's row-major point and normal lists), ops.project at W and ops.grids_from_projection (Deployer.step), then
the tensor-core model, the fused ICP losses, mean over the pairs, backward.  The bounds are those of
test_gpu_odometry_train_capi.py (same model, same kernels from the images on)."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from test_gpu_odometry_train_capi import (DEV, FLAGS, TAIL_TOL, TRUNK_TOL, _blob, _config, _grad_dict, _grad_spread,
                                          _model, _n_stride, _pairs, _rel, _stack, _stream)

pytestmark = pytest.mark.gpu


class _Trainer:
    """One descriptor (with w_pre) + training workspace."""

    def __init__(self, cfg, n_stride, max_batch, blob, w_pre, lr=1e-5):
        from delora_b200 import _lib
        from delora_b200.deploy import export
        self.L = _lib.lib()
        self.d = export.desc_from_config(cfg, "kitti", n_stride, max_batch)
        self.d.w_pre = w_pre
        self.dp = ctypes.byref(self.d)
        self.n = int(self.L.delora_odometry_weight_floats(self.dp))
        nb = cfg["kitti"]["neighborhood_side_length"]
        self.hp = _lib.OdometryTrainParams(
            lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, lambda_po2pl=cfg["lambda_po2pl"], loss_flags=FLAGS, nb_h=nb[0],
            nb_w=nb[1], epsilon_range=cfg["epsilon_range"],
            min_neighbors=cfg["min_num_points_in_neighborhood_to_determine_point_class"])
        size = int(self.L.delora_odometry_train_workspace_bytes(self.dp))
        assert size > 0, self.L.delora_last_error()
        self.ws = torch.empty((size,), dtype=torch.uint8, device=DEV)
        _lib.check(self.L.delora_odometry_train_init(self.dp, blob.data_ptr(), self.ws.data_ptr(), _stream()),
                   "delora_odometry_train_init")

    def step(self, pts, counts, outputs=True):
        from delora_b200 import _lib
        b = pts.shape[0] // 2
        out = None
        if outputs:
            out = (torch.empty((b, 8), device=DEV), torch.empty((b, 4, 4), device=DEV), torch.empty((b, 512), device=DEV),
                   torch.empty((self.n,), device=DEV))
        ptr = (lambda i: out[i].data_ptr()) if outputs else (lambda i: None)
        _lib.check(self.L.delora_odometry_train_step(self.dp, ctypes.byref(self.hp), pts.data_ptr(), counts.data_ptr(), b,
                                                     self.ws.data_ptr(), ptr(0), ptr(1), ptr(2), ptr(3), _stream()),
                   "delora_odometry_train_step")
        return out

    def weights(self):
        from delora_b200 import _lib
        w = torch.empty((self.n,), device=DEV)
        _lib.check(self.L.delora_odometry_train_weights(self.dp, self.ws.data_ptr(), w.data_ptr(), _stream()),
                   "delora_odometry_train_weights")
        return w


def _preprocessed_lists(cfg, pts, counts, w_pre):
    """The offline stage (Preprocesser.preprocess_scans at horizontal_cells_preprocessing = w_pre) of every scan ->
    padded channels-first point and normal lists [2B, 3, P] and their lengths [2B]."""
    from delora_b200.preprocessing.normal_computation import NormalsComputer
    from delora_b200.preprocessing.preprocesser import Preprocesser
    pcfg = copy.deepcopy(cfg)
    pcfg["dataset"] = "kitti"
    pcfg["kitti"]["horizontal_cells"] = w_pre
    pre = Preprocesser(config=pcfg)
    pre.normals_computer = NormalsComputer(config=pcfg, dataset_name="kitti")
    n_host = counts.cpu().tolist()
    out = pre.preprocess_scans([pts[i, :, :n].cpu() for i, n in enumerate(n_host)])
    p_max = max(max(p.shape[0] for _, p in out), 1)
    plist = torch.zeros((len(out), 3, p_max), dtype=torch.float32)
    nlist = torch.zeros_like(plist)
    for i, (nrm, p) in enumerate(out):
        plist[i, :, :p.shape[0]] = torch.from_numpy(p).t()
        nlist[i, :, :nrm.shape[0]] = torch.from_numpy(nrm).t()
    lens = torch.tensor([p.shape[0] for _, p in out], dtype=torch.int32)
    return plist.to(DEV), nlist.to(DEV), lens.to(DEV)


def _python_step(model, cfg, pts, counts, w_pre):
    """The reference's recipe through the mirror: -> (losses [B,8], T [B,4,4], pooled [B,512], {name: grad})."""
    from delora_b200 import ops
    from delora_b200.deploy.deployer import _FusedIcp
    from delora_b200.models.model_parts import GeometryHandler
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    b = pts.shape[0] // 2
    plist, nlist, lens = _preprocessed_lists(cfg, pts, counts, w_pre)
    image, imap = ops.project(plist, lens, h, w, hf, vf)
    pg, ng = ops.grids_from_projection(plist, nlist, imap)
    img1, img2 = image[:b].contiguous(), image[b:].contiguous()
    with torch.no_grad():
        pooled = model._tensor_core_path().pooled_features(img1, img2)
    model.zero_grad(set_to_none=True)
    trans, quat = model(image_1=img1, image_2=img2)
    T = GeometryHandler.get_transformation_matrix_quaternion(trans.float(), quat.float(), DEV)
    total, parts = _FusedIcp.apply(T, pg[b:].contiguous(), ng[b:].contiguous(), pg[:b].contiguous(),
                                   ng[:b].contiguous(), (h, w, hf, vf), float(cfg["lambda_po2pl"]), FLAGS,
                                   ops.icp_scratch(b, h * w, pts.device))
    total.mean().backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    return parts.detach(), T.detach(), pooled, grads


SIZES = [(64, 720, 2048, 2250), (16, 259, 512, 512)]                   # H, W, w_raw, w_pre
VARIANTS = [("tanh", False), ("relu", False), ("tanh", True), ("relu", True)]
STEP_CASES = [pytest.param(act, single, *size, b, id="-".join(map(str, (act, single) + size + (b,))))
              for size in SIZES for b in (1, 2, 4) for act, single in VARIANTS]


@pytest.mark.parametrize("act,single,h,w,w_raw,w_pre,b", STEP_CASES)
def test_step_matches_the_reference_recipe(cuda_lib, act, single, h, w, w_raw, w_pre, b):
    cfg = _config(h, w, act, single)
    model = _model(cfg)
    pairs = _pairs(h, w_raw, b)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    tr = _Trainer(cfg, n_stride, b, _blob(model, cfg), w_pre)
    losses, T, pooled, grads = tr.step(pts, counts)
    py_losses, py_T, py_pooled, py_grads = _python_step(model, cfg, pts, counts, w_pre)
    torch.cuda.synchronize()
    assert torch.equal(pooled, py_pooled), "pooled features differ from the reference recipe's"
    t_err = (T - py_T).abs().max().item()
    assert t_err <= 1e-5, f"max |T - T_py| = {t_err:.3e}"
    l_err = _rel(losses[:, :3], py_losses[:, :3])
    assert l_err <= 1e-5, f"losses differ by {l_err:.3e} (relative)"
    tail, trunk = _grad_spread(_grad_dict(grads, cfg), py_grads)
    print(f"\n[{h}x{w} w_pre={w_pre} B={b} {act} single={single}] T {t_err:.2e}  losses {l_err:.2e}  grads: tail "
          f"{tail:.2e}, trunk {trunk:.2e}")
    assert tail <= TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"


def test_adam_is_torch_adam(cuda_lib):
    """The update after a w_pre step is torch's Adam on that step's gradient."""
    lr = 1e-3
    cfg = _config(16, 259, "tanh", False)
    model = _model(cfg, 1)
    pairs = _pairs(16, 512, 2)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    blob0 = _blob(model, cfg)
    tr = _Trainer(cfg, n_stride, 2, blob0, 512, lr=lr)
    g = tr.step(pts, counts)[3]
    from delora_b200.deploy import export
    from delora_b200.models.model import OdometryModel
    m = OdometryModel(cfg).to(DEV)
    m.load_state_dict(export.unpack_blob(blob0.cpu().numpy(), cfg))
    opt = torch.optim.Adam(m.parameters(), lr=lr, fused=True)
    gd = _grad_dict(g, cfg)
    for k, p in m.named_parameters():
        p.grad = gd[k].to(DEV)
    opt.step()
    got = _grad_dict(tr.weights(), cfg)
    worst = max(_rel(got[k].to(DEV), p.detach()) for k, p in m.named_parameters())
    assert worst <= 1e-6, f"the master weights differ from torch's Adam by {worst:.3e}"


def _zero_free(pairs):
    return tuple(tuple(s[:, (s != 0).all(dim=0)] for s in p) for p in pairs)


def test_same_width_is_the_plain_step(cuda_lib):
    """w_pre == W re-projects every kept point into its own pixel: the step is bit-identical to w_pre = 0 (on clouds
    without exact zero coordinates, which are image pixels but not valid cells)."""
    cfg = _config(64, 720, "tanh", False)
    model = _model(cfg, 2)
    pairs = _zero_free(_pairs(64, 1024, 2))
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    blob = _blob(model, cfg)
    a, b = _Trainer(cfg, n_stride, 2, blob, 0, 1e-4), _Trainer(cfg, n_stride, 2, blob, 720, 1e-4)
    for _ in range(2):
        x, y = a.step(pts, counts), b.step(pts, counts)
        torch.cuda.synchronize()
        for u, v, name in zip(x, y, ("losses", "T", "pooled", "grads")):
            assert torch.equal(u, v), f"w_pre = W: {name} differ from w_pre = 0"


def test_the_option_changes_the_objective(cuda_lib):
    """On the same 64 x 720 scans, normals at 64 x 2250 give other losses than normals at 64 x 720."""
    cfg = _config(64, 720, "tanh", False)
    model = _model(cfg, 3)
    pairs = _pairs(64, 2048, 4)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    blob = _blob(model, cfg)
    plain = _Trainer(cfg, n_stride, 4, blob, 0).step(pts, counts)
    pre = _Trainer(cfg, n_stride, 4, blob, 2250).step(pts, counts)
    torch.cuda.synchronize()
    lam = float(cfg["lambda_po2pl"])
    obj = [(l[:, 0] + lam * l[:, 1] + l[:, 2]).mean().item() for l in (plain[0], pre[0])]
    rel = [((pre[0][:, i] - plain[0][:, i]).abs() / plain[0][:, i].abs()).max().item() for i in (1, 2)]
    pairs_n = [plain[0][:, 3].sum().item(), pre[0][:, 3].sum().item()]
    gdiff = _rel(pre[3], plain[3])
    print(f"\n[64x720, B=4] objective w_pre=0 {obj[0]:.6e}  w_pre=2250 {obj[1]:.6e}  (relative {abs(obj[1] - obj[0]) / obj[0]:.3e}); "
          f"po2pl max rel {rel[0]:.3e}, pl2pl max rel {rel[1]:.3e}; pairs {pairs_n[0]:.0f} vs {pairs_n[1]:.0f}; "
          f"gradient blob max-abs difference / max-abs {gdiff:.3e}")
    assert not torch.equal(plain[0][:, :3], pre[0][:, :3])
    assert abs(obj[1] - obj[0]) > 1e-4 * obj[0]


def test_deterministic_and_graph_replay(cuda_lib):
    cfg = _config(64, 720, "relu", False)
    model = _model(cfg, 4)
    pairs = _pairs(64, 2048, 2)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    blob = _blob(model, cfg)
    a, b = _Trainer(cfg, n_stride, 2, blob, 2250, 1e-4), _Trainer(cfg, n_stride, 2, blob, 2250, 1e-4)
    for _ in range(3):
        a.step(pts, counts, outputs=False)
        b.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert torch.equal(a.weights(), b.weights()), "two workspaces with the same steps differ"

    eager, graphed = _Trainer(cfg, n_stride, 2, blob, 2250, 1e-4), _Trainer(cfg, n_stride, 2, blob, 2250, 1e-4)
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
    cfg = _config(64, 720, "tanh", True)
    model = _model(cfg, 5)
    pairs = _pairs(64, 2048, 4)
    n_stride = _n_stride(pairs)
    tr = _Trainer(cfg, n_stride, 4, _blob(model, cfg), 2250, 1e-4)
    for bsz in (4, 1, 3):
        pts, counts = _stack(pairs[:bsz], n_stride)
        before = tr.weights()
        got = tr.step(pts, counts)
        fresh = _Trainer(cfg, n_stride, 4, before, 2250, 1e-4).step(pts, counts)
        torch.cuda.synchronize()
        for x, y, name in zip(got, fresh, ("losses", "T", "pooled", "grads")):
            assert torch.equal(x, y), f"B={bsz}: {name} differ from a fresh workspace"


def test_finetune_example_program_with_preprocessing_normals(cuda_lib, tmp_path):
    """examples/odometry_finetune.c on a .dlw exported with preprocessing normals: it trains with w_pre from the file."""
    import os
    import subprocess
    from delora_b200 import build, synthetic
    from delora_b200.deploy import export
    from helpers import ROOT
    vfov = (-15.0, 15.0)
    cfg = _config(16, 720, "tanh", False)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    cfg["kitti"]["horizontal_cells_preprocessing"] = 1024
    model = _model(cfg, 6)
    dlw, out = os.path.join(tmp_path, "in.dlw"), os.path.join(tmp_path, "out.dlw")
    desc = export.desc_from_config(cfg, "kitti", 4096, 2, preprocessing_normals=True)
    assert desc.w_pre == 1024
    export.write_dlw(dlw, desc, export.pack_state_dict(model.state_dict(), cfg))
    bins = []
    for i in range(4):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    nvcc = build._nvcc()
    cuda_home = os.path.dirname(os.path.dirname(os.path.realpath(nvcc)))
    libdir = os.path.dirname(build.LIB)
    exe = os.path.join(tmp_path, "odometry_finetune")
    r = subprocess.run([nvcc, os.path.join(ROOT, "examples", "odometry_finetune.c"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(cuda_home, "include"), "-L", libdir, "-ldelora_b200", "-lcudart",
                        "-Xlinker", "-rpath=" + libdir, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([exe, dlw, out, "3", "1e-4"] + bins, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert len(r.stdout.strip().splitlines()) == 3
    assert "preprocessing resolution 16x1024" in r.stderr, r.stderr
    h, d, blob = export.read_dlw(out)
    assert (d.H, d.W, d.max_batch, d.w_pre) == (16, 720, 2, 1024)
    scans = [torch.from_numpy(np.fromfile(p, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()) for p in bins]
    tr = _Trainer(cfg, 4096, 2, _blob(model, cfg), 1024, lr=1e-4)
    plain = _Trainer(cfg, 4096, 2, _blob(model, cfg), 0, lr=1e-4)
    for ks in ((0, 1), (2, 0), (1, 2)):
        pts, counts = _stack([(scans[k], scans[k + 1]) for k in ks], 4096)
        tr.step(pts, counts, outputs=False)
        plain.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert np.array_equal(tr.weights().cpu().numpy(), blob)
    assert not np.array_equal(plain.weights().cpu().numpy(), blob)
