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
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200.deploy.capi import InferenceWorkspace

pytestmark = pytest.mark.gpu
DEV = H.DEV


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
    cfg = H.config(h, w, act, single, nout=nout)
    model = H.model(cfg, near_identity=True)
    pairs = H.pairs(h, w_raw, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    tr = H.trainer(cfg, n_stride, b, H.blob(model, cfg))
    losses, T, pooled, grads = tr.step(pts, counts)
    py = H.python_step(model, cfg, pts, counts)
    torch.cuda.synchronize()
    assert torch.equal(pooled, py.pooled), "pooled features differ from TensorCoreEncoder.pooled_features"
    t_err = (T - py.T).abs().max().item()
    assert t_err <= 1e-5, f"max |T - T_py| = {t_err:.3e}"
    l_err = H.rel(losses[:, :3], py.losses[:, :3])
    assert l_err <= 1e-5, f"losses differ by {l_err:.3e} (relative)"
    tail, trunk = H.grad_spread(H.grad_dict(grads, cfg), py.grads)
    print(f"\n[{h}x{w} B={b} {act} single={single} nout={nout}] T {t_err:.2e}  losses {l_err:.2e}  grads: tail {tail:.2e}, "
          f"trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= H.TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"


def _adam_reference(blob, grads_seq, cfg, lr):
    from delora_b200.deploy import export
    from delora_b200.models.model import OdometryModel
    m = OdometryModel(cfg).to(DEV)
    m.load_state_dict(export.unpack_blob(blob.cpu().numpy(), cfg))
    opt = torch.optim.Adam(m.parameters(), lr=lr, fused=True)
    params = dict(m.named_parameters())
    for g in grads_seq:
        gd = H.grad_dict(g, cfg)
        for k, p in params.items():
            p.grad = gd[k].to(DEV)
        opt.step()
    return {k: p.detach() for k, p in params.items()}


@pytest.mark.parametrize("act,single", [("tanh", False), ("relu", True)])
def test_adam_matches_torch(cuda_lib, act, single):
    lr = 1e-3
    cfg = H.config(16, 720, act, single)
    model = H.model(cfg, 1, near_identity=True)
    pairs = H.pairs(16, 1024, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob0 = H.blob(model, cfg)
    tr = H.trainer(cfg, n_stride, 2, blob0, lr=lr)
    seq = []
    for k in range(3):
        seq.append(tr.step(pts, counts)[3])
        if k in (0, 2):
            want = _adam_reference(blob0, seq, cfg, lr)
            got = H.grad_dict(tr.weights(), cfg)
            worst = max(H.rel(got[n].to(DEV), want[n]) for n in want)
            print(f"\n[Adam, {k + 1} step(s)] worst relative difference {worst:.2e}")
            assert worst <= 1e-6, f"after {k + 1} step(s) the master weights differ from torch's Adam by {worst:.3e}"


def test_round_trip_to_inference_and_torch(cuda_lib):
    from delora_b200.deploy import export
    from delora_b200.models import model_parts
    from delora_b200.models.model import OdometryModel
    cfg = H.config(64, 720, "tanh", False)
    model = H.model(cfg, 2, near_identity=True)
    pairs = H.pairs(64, 1024, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    tr = H.trainer(cfg, n_stride, 2, H.blob(model, cfg), lr=1e-4)
    for _ in range(2):
        tr.step(pts, counts, outputs=False)
    tuned = tr.weights()
    T, _ = InferenceWorkspace(tr.desc, tuned).pairs(pts, counts)
    m2 = OdometryModel(cfg).to(DEV).eval()
    m2.load_state_dict(export.unpack_blob(tuned.cpu().numpy(), cfg))
    assert not torch.equal(tuned, H.blob(model, cfg)), "the steps did not change the weights"
    from delora_b200 import ops
    img, _ = ops.project(pts, counts, 64, 720, cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"])
    with torch.no_grad():
        trans, quat = m2(image_1=img[:2].contiguous(), image_2=img[2:].contiguous())
        T_ref = model_parts.GeometryHandler.get_transformation_matrix_quaternion(trans, quat, DEV)
    torch.cuda.synchronize()
    assert (T - T_ref).abs().max().item() <= 1e-5


def test_deterministic_and_graph_replay(cuda_lib):
    cfg = H.config(64, 720, "relu", False)
    model = H.model(cfg, 3, near_identity=True)
    pairs = H.pairs(64, 1024, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    a, b = H.trainer(cfg, n_stride, 2, blob, 1e-4), H.trainer(cfg, n_stride, 2, blob, 1e-4)
    for _ in range(5):
        a.step(pts, counts, outputs=False)
        b.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert torch.equal(a.weights(), b.weights()), "two workspaces with the same steps differ"

    eager, graphed = H.trainer(cfg, n_stride, 2, blob, 1e-4), H.trainer(cfg, n_stride, 2, blob, 1e-4)
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
    cfg = H.config(64, 720, "tanh", True)
    model = H.model(cfg, 4, near_identity=True)
    pairs = H.pairs(64, 1024, 4)
    n_stride = H.n_stride(pairs)
    tr = H.trainer(cfg, n_stride, 4, H.blob(model, cfg), 1e-4)
    for bsz in (4, 2, 4):
        pts, counts = H.stack_pairs(pairs[:bsz], n_stride)
        before = tr.weights()
        got = tr.step(pts, counts)
        fresh = H.trainer(cfg, n_stride, 4, before, 1e-4).step(pts, counts)
        torch.cuda.synchronize()
        for x, y, name in zip(got, fresh, ("losses", "T", "pooled", "grads")):
            assert torch.equal(x, y), f"B={bsz}: {name} differ from a fresh workspace"


def test_finetune_example_program(cuda_lib, tmp_path):
    """examples/odometry_finetune.c on a .dlw and four KITTI .bin scans: its weights are the C step's on those pairs."""
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    model = H.model(cfg, 5, near_identity=True)
    dlw, out = os.path.join(tmp_path, "in.dlw"), os.path.join(tmp_path, "out.dlw")
    desc = export.desc_from_config(cfg, "kitti", 4096, 2)
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
    _, d, blob = export.read_dlw(out)
    assert (d.H, d.W, d.max_batch) == (16, 720, 2)
    # the program's three steps (two pairs each, cycling): (0,1) (1,2); (2,3) (0,1); (1,2) (2,3)
    scans = [torch.from_numpy(np.fromfile(p, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()) for p in bins]
    tr = H.trainer(cfg, 4096, 2, H.blob(model, cfg), lr=1e-4)
    for ks in ((0, 1), (2, 0)):
        pts, counts = H.stack_pairs([(scans[k], scans[k + 1]) for k in ks], 4096)
        tr.step(pts, counts, outputs=False)
    pts, counts = H.stack_pairs([(scans[1], scans[2]), (scans[2], scans[3])], 4096)
    tr.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert np.array_equal(tr.weights().cpu().numpy(), blob)


def test_training_lowers_the_objective_next_to_synthetic_train_step(cuda_lib):
    from delora_b200.train_step import SyntheticTrainStep
    lr, steps, b = 1e-4, 20, 4
    pairs = H.pairs(64, 2048, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    torch.manual_seed(0)
    ref = SyntheticTrainStep(H.config(64, 2048), b, n_stride, lr=lr)
    ref.load(pts, counts)
    cfg = ref.cfg
    tr = H.trainer(cfg, n_stride, b, H.blob(ref.model, cfg), lr)
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
