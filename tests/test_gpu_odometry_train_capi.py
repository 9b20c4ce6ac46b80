"""Odometry training through the C ABI (delora_odometry_train_*) against the Python training path, on the H100.

The Python step is SyntheticTrainStep's: ops.project + ops.normals, OdometryModel's training forward (TensorCoreEncoder
with autograd, torch heads), GeometryHandler's quaternion -> T, the fused ICP losses, mean over the pairs, backward.
  - pooled: bit-identical to TensorCoreEncoder.pooled_features (the same kernels in the same order).
  - T: within 1e-5 (torch's cuBLAS heads and the C tail sum in different orders).
  - losses: within 1e-5 relative (they see T, which differs in the last bits).
  - gradients, relative to each tensor's max-abs: the fc / head tensors are fp32 on both sides and differ only in
    summation order (TAIL_TOL); the trunk's run the same bf16 kernels, but their input, d(pooled), carries the tail's
    last-bit differences, and one flipped bf16 rounding of a data gradient moves that element by 2^-8 relative, which
    the chain of dgrad layers spreads (TRUNK_TOL).
Measured on an H100 over the 16 size x variant cases: tail <= 4.8e-7, trunk <= 6.0e-3 (16 x 259, tanh, single MLP;
relu cases are often bit-identical: relu' does not depend on the bits of the activation).  The bounds leave a 10x
(tail) and 1.7x (trunk) margin.
"""
import ctypes
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VFOV = (-24.5, 2.0)
FLAGS = 2 | 4                      # DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL, SyntheticTrainStep's losses
TAIL_TOL = 5e-6
TRUNK_TOL = 1e-2


def _config(h, w, act="tanh", single=False, layers=(2, 2, 2, 2), nout=1000):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=VFOV, device=DEV)
    cfg.update({"activation_fct": act, "use_single_mlp_at_output": single, "layers": list(layers), "resnet_outputs": nout,
                "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1, "use_dropout": False})
    return cfg


def _model(cfg, seed=0):
    """Random weights with small last layers and the identity quaternion as bias: T near I (as after the reference's
    identity pre-training), and every layer gets a gradient."""
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(seed)
    m = OdometryModel(cfg).to(DEV)
    with torch.no_grad():
        if cfg["use_single_mlp_at_output"]:
            last = m.fully_connected_rot_trans[-1]
            last.weight.mul_(0.01)
            last.bias.copy_(torch.tensor([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]))
        else:
            for head, bias in ((m.fully_connected_rotation, [0.0, 0.0, 0.0, 1.0]),
                               (m.fully_connected_translation, [0.0, 0.0, 0.0])):
                head[3].weight.mul_(0.01)
                head[3].bias.copy_(torch.tensor(bias))
    return m


@functools.lru_cache(maxsize=None)
def _pairs(rings, w_raw, count):
    from delora_b200 import synthetic
    return tuple(synthetic.make_pair(i, w_raw=w_raw, rings=rings, vfov_deg=VFOV)[:2] for i in range(count))


def _stack(pairs, n_stride):
    scans = [p[0] for p in pairs] + [p[1] for p in pairs]              # scan_1 x B, then scan_2 x B
    pts = torch.zeros((len(scans), 3, n_stride), dtype=torch.float32)
    for i, s in enumerate(scans):
        pts[i, :, :s.shape[1]] = s
    counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
    return pts.to(DEV), counts.to(DEV)


def _n_stride(pairs):
    return max(max(a.shape[1], b.shape[1]) for a, b in pairs)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _blob(model, cfg):
    from delora_b200.deploy import export
    return torch.from_numpy(export.pack_state_dict(model.state_dict(), cfg)).to(DEV)


class _Trainer:
    """Test-side holder of one descriptor + training workspace (device memory from torch)."""

    def __init__(self, cfg, n_stride, max_batch, blob, lr=1e-5):
        from delora_b200 import _lib
        from delora_b200.deploy import export
        self.L, self.cfg = _lib.lib(), cfg
        self.d = export.desc_from_config(cfg, "kitti", n_stride, max_batch)
        self.dp = ctypes.byref(self.d)
        self.n = int(self.L.delora_odometry_weight_floats(self.dp))
        nb = cfg["kitti"]["neighborhood_side_length"]
        self.hp = _lib.OdometryTrainParams(
            lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, lambda_po2pl=cfg["lambda_po2pl"], loss_flags=FLAGS, nb_h=nb[0],
            nb_w=nb[1], epsilon_range=cfg["epsilon_range"],
            min_neighbors=cfg["min_num_points_in_neighborhood_to_determine_point_class"])
        self.ws = torch.empty((int(self.L.delora_odometry_train_workspace_bytes(self.dp)),), dtype=torch.uint8,
                              device=DEV)
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


def _python_step(model, cfg, pts, counts):
    """SyntheticTrainStep.step without the optimizer: -> (losses [B,8], T [B,4,4], pooled [B,512], {name: grad})."""
    from delora_b200 import ops
    from delora_b200.deploy.deployer import _FusedIcp
    from delora_b200.models.model_parts import GeometryHandler
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    b = pts.shape[0] // 2
    image, _ = ops.project(pts, counts, h, w, hf, vf)
    _, pg, ng = ops.normals(image, ds["neighborhood_side_length"], cfg["epsilon_range"],
                            cfg["min_num_points_in_neighborhood_to_determine_point_class"], grids=True)
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


def _grad_dict(flat, cfg):
    from delora_b200.deploy import export
    return export.unpack_blob(flat.cpu().numpy(), cfg)


def _is_tail(name):
    return name.startswith("resnet.fc") or name.startswith("fully_connected")


def _grad_spread(c_grads, py_grads):
    """-> (worst relative error of the tail tensors, of the trunk tensors), relative to each tensor's max-abs."""
    worst = {True: 0.0, False: 0.0}
    for k, ref in py_grads.items():
        ref = ref.cpu()
        scale = ref.abs().max().item()
        assert scale > 0, f"{k}: zero gradient in the Python step"
        err = (c_grads[k] - ref).abs().max().item() / scale
        worst[_is_tail(k)] = max(worst[_is_tail(k)], err)
    return worst[True], worst[False]


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


SIZES = [(64, 2048, 2048, 4), (64, 720, 1024, 2), (16, 720, 1024, 2), (16, 259, 512, 2)]     # H, W, w_raw, B
VARIANTS = [("tanh", False), ("relu", False), ("tanh", True), ("relu", True)]
# resnet_outputs = 1002: every head layer starts at a float offset = 2 (mod 4) in the master blob the tail reads, so
# the tail must not read it with float4 loads
STEP_CASES = ([pytest.param(act, single, *size, 1000, id="-".join(map(str, (act, single) + size)))
               for act, single in VARIANTS for size in SIZES] +
              [pytest.param("tanh", single, 16, 259, 512, 2, 1002, id=f"tanh-{single}-16-259-512-2-nout1002")
               for single in (False, True)])


@pytest.mark.parametrize("act,single,h,w,w_raw,b,nout", STEP_CASES)
def test_step_matches_the_python_training_step(cuda_lib, h, w, w_raw, b, act, single, nout):
    cfg = _config(h, w, act, single, nout=nout)
    model = _model(cfg)
    pairs = _pairs(h, w_raw, b)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    tr = _Trainer(cfg, n_stride, b, _blob(model, cfg))
    losses, T, pooled, grads = tr.step(pts, counts)
    py_losses, py_T, py_pooled, py_grads = _python_step(model, cfg, pts, counts)
    torch.cuda.synchronize()
    assert torch.equal(pooled, py_pooled), "pooled features differ from TensorCoreEncoder.pooled_features"
    t_err = (T - py_T).abs().max().item()
    assert t_err <= 1e-5, f"max |T - T_py| = {t_err:.3e}"
    l_err = _rel(losses[:, :3], py_losses[:, :3])
    assert l_err <= 1e-5, f"losses differ by {l_err:.3e} (relative)"
    tail, trunk = _grad_spread(_grad_dict(grads, cfg), py_grads)
    print(f"\n[{h}x{w} B={b} {act} single={single} nout={nout}] T {t_err:.2e}  losses {l_err:.2e}  grads: tail {tail:.2e}, "
          f"trunk {trunk:.2e}")
    assert tail <= TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"


def _adam_reference(blob, grads_seq, cfg, lr):
    from delora_b200.deploy import export
    from delora_b200.models.model import OdometryModel
    m = OdometryModel(cfg).to(DEV)
    m.load_state_dict(export.unpack_blob(blob.cpu().numpy(), cfg))
    opt = torch.optim.Adam(m.parameters(), lr=lr, fused=True)
    params = dict(m.named_parameters())
    for g in grads_seq:
        gd = _grad_dict(g, cfg)
        for k, p in params.items():
            p.grad = gd[k].to(DEV)
        opt.step()
    return {k: p.detach() for k, p in params.items()}


@pytest.mark.parametrize("act,single", [("tanh", False), ("relu", True)])
def test_adam_matches_torch(cuda_lib, act, single):
    lr = 1e-3
    cfg = _config(16, 720, act, single)
    model = _model(cfg, 1)
    pairs = _pairs(16, 1024, 2)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    blob0 = _blob(model, cfg)
    tr = _Trainer(cfg, n_stride, 2, blob0, lr=lr)
    seq = []
    for k in range(3):
        seq.append(tr.step(pts, counts)[3])
        if k in (0, 2):
            want = _adam_reference(blob0, seq, cfg, lr)
            got = _grad_dict(tr.weights(), cfg)
            worst = max(_rel(got[n].to(DEV), want[n]) for n in want)
            print(f"\n[Adam, {k + 1} step(s)] worst relative difference {worst:.2e}")
            assert worst <= 1e-6, f"after {k + 1} step(s) the master weights differ from torch's Adam by {worst:.3e}"


def test_round_trip_to_inference_and_torch(cuda_lib):
    from delora_b200 import _lib
    from delora_b200.deploy import export
    from delora_b200.models import model_parts
    from delora_b200.models.model import OdometryModel
    cfg = _config(64, 720, "tanh", False)
    model = _model(cfg, 2)
    pairs = _pairs(64, 1024, 2)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    tr = _Trainer(cfg, n_stride, 2, _blob(model, cfg), lr=1e-4)
    for _ in range(2):
        tr.step(pts, counts, outputs=False)
    tuned = tr.weights()
    L = tr.L
    ws = torch.empty((int(L.delora_odometry_workspace_bytes(tr.dp)),), dtype=torch.uint8, device=DEV)
    _lib.check(L.delora_odometry_init(tr.dp, ws.data_ptr(), _stream()), "init")
    _lib.check(L.delora_odometry_load_weights(tr.dp, tuned.data_ptr(), ws.data_ptr(), _stream()), "load")
    T = torch.empty((2, 4, 4), device=DEV)
    _lib.check(L.delora_odometry_pairs(tr.dp, pts.data_ptr(), counts.data_ptr(), 2, ws.data_ptr(), T.data_ptr(), None,
                                       _stream()), "pairs")
    m2 = OdometryModel(cfg).to(DEV).eval()
    m2.load_state_dict(export.unpack_blob(tuned.cpu().numpy(), cfg))
    assert not torch.equal(tuned, _blob(model, cfg)), "the steps did not change the weights"
    from delora_b200 import ops
    img, _ = ops.project(pts, counts, 64, 720, cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"])
    with torch.no_grad():
        trans, quat = m2(image_1=img[:2].contiguous(), image_2=img[2:].contiguous())
        T_ref = model_parts.GeometryHandler.get_transformation_matrix_quaternion(trans, quat, DEV)
    torch.cuda.synchronize()
    assert (T - T_ref).abs().max().item() <= 1e-5


def test_deterministic_and_graph_replay(cuda_lib):
    cfg = _config(64, 720, "relu", False)
    model = _model(cfg, 3)
    pairs = _pairs(64, 1024, 2)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    blob = _blob(model, cfg)
    a, b = _Trainer(cfg, n_stride, 2, blob, 1e-4), _Trainer(cfg, n_stride, 2, blob, 1e-4)
    for _ in range(5):
        a.step(pts, counts, outputs=False)
        b.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert torch.equal(a.weights(), b.weights()), "two workspaces with the same steps differ"

    eager, graphed = _Trainer(cfg, n_stride, 2, blob, 1e-4), _Trainer(cfg, n_stride, 2, blob, 1e-4)
    for _ in range(3):
        eager.step(pts, counts, outputs=False)
    graphed.step(pts, counts, outputs=False)        # eager first: sets up the launchers' host-side state
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
    model = _model(cfg, 4)
    pairs = _pairs(64, 1024, 4)
    n_stride = _n_stride(pairs)
    tr = _Trainer(cfg, n_stride, 4, _blob(model, cfg), 1e-4)
    for bsz in (4, 2, 4):
        pts, counts = _stack(pairs[:bsz], n_stride)
        before = tr.weights()
        got = tr.step(pts, counts)
        fresh = _Trainer(cfg, n_stride, 4, before, 1e-4).step(pts, counts)
        torch.cuda.synchronize()
        for x, y, name in zip(got, fresh, ("losses", "T", "pooled", "grads")):
            assert torch.equal(x, y), f"B={bsz}: {name} differ from a fresh workspace"


def test_finetune_example_program(cuda_lib, tmp_path):
    """examples/odometry_finetune.c on a .dlw and four KITTI .bin scans: its weights are the C step's on those pairs."""
    import os
    import subprocess
    from delora_b200 import build, synthetic
    from delora_b200.deploy import export
    from helpers import ROOT
    vfov = (-15.0, 15.0)
    cfg = _config(16, 720, "tanh", False)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    model = _model(cfg, 5)
    dlw, out = os.path.join(tmp_path, "in.dlw"), os.path.join(tmp_path, "out.dlw")
    desc = export.desc_from_config(cfg, "kitti", 4096, 2)
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
    _, d, blob = export.read_dlw(out)
    assert (d.H, d.W, d.max_batch) == (16, 720, 2)
    # the program's three steps (two pairs each, cycling): (0,1) (1,2); (2,3) (0,1); (1,2) (2,3)
    scans = [torch.from_numpy(np.fromfile(p, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()) for p in bins]
    tr = _Trainer(cfg, 4096, 2, _blob(model, cfg), lr=1e-4)
    for ks in ((0, 1), (2, 0)):
        pts, counts = _stack([(scans[k], scans[k + 1]) for k in ks], 4096)
        tr.step(pts, counts, outputs=False)
    pts, counts = _stack([(scans[1], scans[2]), (scans[2], scans[3])], 4096)
    tr.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert np.array_equal(tr.weights().cpu().numpy(), blob)


def test_training_lowers_the_objective_next_to_synthetic_train_step(cuda_lib):
    from delora_b200.deploy import export
    from delora_b200.train_step import SyntheticTrainStep
    lr, steps, b = 1e-4, 20, 4
    pairs = _pairs(64, 2048, b)
    n_stride = _n_stride(pairs)
    pts, counts = _stack(pairs, n_stride)
    torch.manual_seed(0)
    ref = SyntheticTrainStep(_config(64, 2048), b, n_stride, lr=lr)
    ref.load(pts, counts)
    cfg = ref.cfg
    blob = torch.from_numpy(export.pack_state_dict(ref.model.state_dict(), cfg)).to(DEV)
    tr = _Trainer(cfg, n_stride, b, blob, lr)
    lam = float(cfg["lambda_po2pl"])
    c_curve, py_curve = [], []
    for _ in range(steps):
        losses = tr.step(pts, counts)[0]
        c_curve.append((losses[:, 0] + lam * losses[:, 1] + losses[:, 2]).mean().item())
        py_curve.append(ref.step()[0].item())
    print("\nC step          :", " ".join(f"{v:.6f}" for v in c_curve))
    print("SyntheticTrainStep:", " ".join(f"{v:.6f}" for v in py_curve))
    assert c_curve[-1] < c_curve[0] and py_curve[-1] < py_curve[0]
    assert abs(c_curve[0] - py_curve[0]) <= 1e-5 * py_curve[0]
    worst = max(abs(c - p) / p for c, p in zip(c_curve, py_curve))
    assert worst <= 1e-2, f"the C curve leaves SyntheticTrainStep's by {worst:.3e} (relative)"
