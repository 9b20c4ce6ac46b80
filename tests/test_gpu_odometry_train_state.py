"""-m gpu: resumable training through the C ABI -- delora_odometry_train_get_state / _set_state, the .dlt training
checkpoint, identity pre-training (DELORA_LOSS_IDENTITY_FIT) and examples/odometry_train.c -- on the H100.

  - resume: a workspace that stops after K steps, goes through a .dlt file and continues in a fresh workspace gives
    the same bits as one that never stopped (weights, m, v, step, and every output of the later steps);
  - set_state continues torch's fused Adam (few steps, and a state at step 10 000) within the existing 1e-6 bound,
    and re-preps the bf16 filters (the first step equals a workspace initialised with the same weights);
  - the identity fit against the Python step with unsupervised_at_start: False (odometry_harness.python_step), with
    test_gpu_odometry_train_capi.py's gradient metric (each tensor's error relative to its max-abs) and bounds.  At B > 1 the identity fit's head gradient is ill-conditioned in fp32: rows 0..B-2 get theirs
    only through the block norm, and in row B-1 most of d(quaternion) cancels against the norm's backward.  Both fp32
    steps then leave the exact gradient by a few 1e-6, so the fc / head tensors are held to TAIL_TOL against a float64
    evaluation of the tail from the (bit-identical) pooled features, and the C-Python distance to the Python step's own
    distance from it plus TAIL_TOL.  Measured on an H100 at 64 x 720, B = 4, tanh, two heads: C 3.5e-6, Python 6.5e-6
    and C-Python 7.8e-6 from / apart; trunk 2.5e-3.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200.ops import LOSS_IDENTITY_FIT

pytestmark = pytest.mark.gpu
DEV = H.DEV


def _batch(pairs, s, b, n_stride):
    """Step s's pairs: b consecutive ones starting at s (cycling), so consecutive steps see different data."""
    return H.stack_pairs([pairs[(s + j) % len(pairs)] for j in range(b)], n_stride)


# ------------------------------------------------------------------------------------------------------------ resume
@pytest.mark.parametrize("b1,b2,w_pre", [(2, 2, 0), (2, 1, 0), (1, 3, 0), (2, 2, 1440)],
                         ids=["B2", "B2-then-1", "B1-then-3", "B2-w_pre"])
def test_resume_through_a_dlt_file_is_exact(cuda_lib, tmp_path, b1, b2, w_pre):
    from delora_b200.deploy import export
    K = 3
    cfg = H.config(16, 720, "tanh", False)
    model = H.model(cfg, 10, near_identity=True)
    pairs = H.pairs(16, 1024, 4)
    n_stride = H.n_stride(pairs)
    blob = H.blob(model, cfg)
    bs = [b1] * K + [b2] * K
    a = H.trainer(cfg, n_stride, 3, blob, 1e-4, w_pre)
    outs_a = [a.step(*_batch(pairs, s, bs[s], n_stride)) for s in range(2 * K)]
    b = H.trainer(cfg, n_stride, 3, blob, 1e-4, w_pre)
    for s in range(K):
        b.step(*_batch(pairs, s, bs[s], n_stride), outputs=False)
    w, m, v, step = [t.cpu() for t in b.get_state()]
    path = os.path.join(tmp_path, "k.dlt")
    export.write_dlt(path, b.desc, export.TrainingState(w.numpy(), m.numpy(), v.numpy(), int(step[0]), 1, 1, 1e-4))
    _, d, st = export.read_dlt(path)
    assert st.step == K and d.w_pre == w_pre
    c = H.trainer(cfg, n_stride, 3, torch.from_numpy(st.weights).to(DEV), 1e-4, w_pre)
    c.set_state(st.weights, st.exp_avg, st.exp_avg_sq, st.step)
    outs_c = [c.step(*_batch(pairs, s, bs[s], n_stride)) for s in range(K, 2 * K)]
    torch.cuda.synchronize()
    for s, (x, y) in enumerate(zip(outs_a[K:], outs_c)):
        for xx, yy, name in zip(x, y, ("losses", "T", "pooled", "grads")):
            assert torch.equal(xx, yy), f"step {K + s + 1}: {name} differ after the resume"
    for xa, xc, name in zip(a.get_state(), c.get_state(), ("weights", "exp_avg", "exp_avg_sq", "step")):
        assert torch.equal(xa, xc), f"{name} differ after the resume"
    assert int(c.get_state()[3][0]) == 2 * K


# ------------------------------------------------------------------------------------------------- torch's Adam state
@pytest.mark.parametrize("start_step", [None, 10000], ids=["fresh-steps", "step10000"])
def test_set_state_continues_torch_adam(cuda_lib, start_step):
    from delora_b200.deploy import export
    lr = 1e-3
    cfg = H.config(16, 720, "relu", True)
    model = H.model(cfg, 11, near_identity=True)
    opt = torch.optim.Adam(model.parameters(), lr=lr, fused=True)
    gen = torch.Generator(device=DEV).manual_seed(3)
    for _ in range(3):
        for p in model.parameters():
            p.grad = torch.randn(p.shape, device=DEV, generator=gen) * 1e-2
        opt.step()
    if start_step is not None:
        for s in opt.state.values():
            s["step"].fill_(start_step)
    st = export.training_state_from_checkpoint({"model_state_dict": model.state_dict(),
                                                "optimizer_state_dict": opt.state_dict()}, cfg)
    assert st.step == (start_step or 3)
    pairs = H.pairs(16, 1024, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    tr = H.trainer(cfg, n_stride, 2, H.blob(model, cfg), lr)
    tr.set_state(st.weights, st.exp_avg, st.exp_avg_sq, st.step)
    params = dict(model.named_parameters())
    for k in range(2):
        grads = H.grad_dict(tr.step(pts, counts)[3], cfg)
        for name, p in params.items():
            p.grad = grads[name].to(DEV)
        opt.step()
        got = H.grad_dict(tr.get_state()[0], cfg)
        worst = max(H.rel(got[n].to(DEV), p.detach()) for n, p in params.items())
        print(f"\n[Adam from step {st.step}, {k + 1} step(s)] worst relative difference {worst:.2e}")
        assert worst <= 1e-6, f"the master weights leave torch's Adam by {worst:.3e}"
    assert int(tr.get_state()[3][0]) == st.step + 2


def test_set_state_reprepares_the_filters(cuda_lib):
    cfg = H.config(64, 720, "tanh", False)
    pairs = H.pairs(64, 1024, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob0, blob1 = H.blob(H.model(cfg, 12, near_identity=True), cfg), H.blob(H.model(cfg, 13, near_identity=True), cfg)
    x = H.trainer(cfg, n_stride, 2, blob0, 1e-4)
    x.step(pts, counts, outputs=False)                 # m, v, step and the ICP scratch are in use
    zeros = torch.zeros_like(blob1)
    x.set_state(blob1, zeros, zeros, 0)
    y = H.trainer(cfg, n_stride, 2, blob1, 1e-4)
    ox, oy = x.step(pts, counts), y.step(pts, counts)
    torch.cuda.synchronize()
    for a, b, name in zip(ox, oy, ("losses", "T", "pooled", "grads")):
        assert torch.equal(a, b), f"{name}: set_state differs from _train_init with the same weights"
    for a, b, name in zip(x.get_state(), y.get_state(), ("weights", "exp_avg", "exp_avg_sq", "step")):
        assert torch.equal(a, b), name


# ------------------------------------------------------------------------------------------------- identity fit
def _tail_grads_fp64(model, cfg, pooled):
    """The fc / head gradients of the identity fit in float64 on the CPU, from the (bit-identical) pooled features: the
    tail of OdometryModel.forward, the oracle's quaternion -> T, MSELoss(T_{B-1}, I) / B."""
    import copy
    from oracle import delora_oracle as orc
    b = pooled.shape[0]
    names = ["resnet.fc"] + (["fully_connected_rot_trans"] if cfg["use_single_mlp_at_output"]
                             else ["fully_connected_rotation", "fully_connected_translation"])
    mods = {n: copy.deepcopy(model.get_submodule(n)).double().cpu() for n in names}
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        x = mods["resnet.fc"](pooled.detach().double().cpu())
        if cfg["use_single_mlp_at_output"]:
            y = mods["fully_connected_rot_trans"](x)
            rot, trans = y[:, :4], y[:, 4:]
        else:
            rot, trans = mods["fully_connected_rotation"](x), mods["fully_connected_translation"](x)
        T = orc.transformation_matrix_quaternion(trans, rot / torch.norm(rot))
        (torch.nn.MSELoss()(T[-1:], torch.eye(4).view(1, 4, 4)) / b).backward()
    finally:
        torch.set_default_dtype(default)
    return {f"{n}.{k}": p.grad for n, mod in mods.items() for k, p in mod.named_parameters()}


@pytest.mark.parametrize("act,single,b", [("tanh", False, 1), ("tanh", False, 4), ("relu", True, 4)])
def test_identity_fit_matches_the_python_step(cuda_lib, act, single, b):
    cfg = H.config(64, 720, act, single)
    model = H.model(cfg, 14)
    pairs = H.pairs(64, 1024, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    losses, T, pooled, grads = H.trainer(cfg, n_stride, b, blob, flags=H.FLAGS | LOSS_IDENTITY_FIT).step(pts, counts)
    icp_losses = H.trainer(cfg, n_stride, b, blob).step(pts, counts)[0]
    py = H.python_step(model, cfg, pts, counts, identity=True)
    py_grads, py_obj = py.grads, py.objective
    torch.cuda.synchronize()
    assert torch.equal(pooled, py.pooled)
    t_err = (T - py.T).abs().max().item()
    assert t_err <= 1e-5, f"max |T - T_py| = {t_err:.3e}"
    assert torch.equal(losses[:, :5], icp_losses[:, :5]), "the identity bit changed the ICP losses"
    assert torch.equal(losses[:, 6:], icp_losses[:, 6:]) and not icp_losses[:, 5].any()
    assert not losses[:b - 1, 5].any(), "column 5 is not 0 outside row B-1"
    obj = losses[b - 1, 5].item()
    e = (T[b - 1] - torch.eye(4, device=DEV)).double()
    own = ((e * e).sum() / 16 / b).item()                           # the objective of the step's own T
    assert abs(obj - own) <= 1e-6 * own, f"objective {obj} vs MSELoss of the step's T {own}"
    # against the Python objective: T agrees within t_err, so the objective within 2 * sum|T - I| * t_err / (16 B)
    bound = 2.0 * e.abs().sum().item() * max(t_err, 1e-7) / (16 * b) + 1e-6 * own
    assert abs(obj - py_obj) <= bound, f"objective {obj} vs the Python step's {py_obj}"
    c_grads = H.grad_dict(grads, cfg)
    tail, trunk = H.grad_spread(c_grads, py_grads)
    exact = _tail_grads_fp64(model, cfg, pooled)
    c_tail = max(H.rel(c_grads[k], g.float()) for k, g in exact.items())
    py_tail = max(H.rel(py_grads[k].cpu(), g.float()) for k, g in exact.items())
    print(f"\n[identity fit 64x720 B={b} {act} single={single}] T {t_err:.2e}  objective {obj:.6e} "
          f"(python {py_obj:.6e})  grads: tail {tail:.2e} (C vs fp64 {c_tail:.2e}, Python vs fp64 {py_tail:.2e}), "
          f"trunk {trunk:.2e}")
    assert c_tail <= H.TAIL_TOL, f"fc / head gradients differ from the fp64 tail by {c_tail:.3e} of their max-abs"
    assert tail <= py_tail + H.TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= H.TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"


def test_identity_fit_deterministic_and_graph_replay(cuda_lib):
    cfg = H.config(64, 720, "tanh", False)
    blob = H.blob(H.model(cfg, 15), cfg)
    pairs = H.pairs(64, 1024, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    mk = lambda: H.trainer(cfg, n_stride, 2, blob, 1e-4, flags=H.FLAGS | LOSS_IDENTITY_FIT)    # noqa: E731
    a, b = mk(), mk()
    for _ in range(3):
        oa, ob = a.step(pts, counts), b.step(pts, counts)
        for x, y, name in zip(oa, ob, ("losses", "T", "pooled", "grads")):
            assert torch.equal(x, y), f"two runs differ in {name}"
    for x, y in zip(a.get_state(), b.get_state()):
        assert torch.equal(x, y)
    eager, graphed = mk(), mk()
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
    for x, y, name in zip(graphed.get_state(), eager.get_state(), ("weights", "exp_avg", "exp_avg_sq", "step")):
        assert torch.equal(x, y), f"graph replay differs from eager stepping in {name}"


# ------------------------------------------------------------------------------------------------- the example
def test_train_example_program(cuda_lib, tmp_path):
    """examples/odometry_train.c from an --init-seed .dlt: two epochs in one run equal one epoch, a stop and a resumed
    epoch, byte for byte; the switch to the ICP objective after the first epoch; the .pth tool's checkpoint loads into
    the mirror Trainer."""
    import sys
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    from helpers import ROOT
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False, layers=(1, 1, 1, 1), nout=64)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    init = os.path.join(tmp_path, "init.dlt")
    export.write_dlt(init, export.desc_from_config(cfg, "kitti", 4096, 2),
                     export.initial_training_state(dict(cfg, learning_rate=1e-4), 7))
    bins = []
    for i in range(4):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    exe = H.build_example("odometry_train", tmp_path, link=True)

    def run(src, dst, epochs):
        r = subprocess.run([exe, "--switch-below", "1e30", src, dst, str(epochs), "2"] + bins, capture_output=True,
                           text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        return r.stdout.strip().splitlines()

    full, mid, resumed = (os.path.join(tmp_path, n) for n in ("full.dlt", "mid.dlt", "resumed.dlt"))
    lines = run(init, full, 2)
    assert [ln.split()[-1] for ln in lines] == ["0", "1"], lines          # epoch 0 identity fit, epoch 1 ICP
    assert run(init, mid, 1) == lines[:1]
    assert run(mid, resumed, 1) == lines[1:]
    assert open(full, "rb").read() == open(resumed, "rb").read(), "stop + resume differs from one run"
    _, d, st = export.read_dlt(full)
    assert (st.step, st.epoch, st.unsupervised) == (4, 2, 1)              # 3 pairs at B = 2: two steps per epoch
    assert st.loss == pytest.approx(float(lines[1].split()[3]), rel=1e-6)
    _, _, st_mid = export.read_dlt(mid)
    assert (st_mid.step, st_mid.epoch, st_mid.unsupervised) == (2, 1, 1) and st_mid.exp_avg.any()

    pth = os.path.join(tmp_path, "full.pth")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "training_state_to_checkpoint.py"), "--dlt", full,
                        "--out", pth, "--config_dir", os.path.join(tmp_path, "no_config")], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    from delora_b200.deploy.trainer import Trainer
    (tmp_path / "pre" / "00" / "scans").mkdir(parents=True)
    (tmp_path / "pre" / "00" / "normals").mkdir(parents=True)
    tcfg = dict(cfg)
    tcfg.update({"batch_size": 1, "learning_rate": 1e-4, "store_dataset_in_RAM": False, "num_dataloader_workers": 0,
                 "normalization_scaling": False, "inference_only": False, "unsupervised_at_start": False,
                 "mode": "training", "experiment": "test", "training_run_name": "pytest_run", "run_name": "pytest_run",
                 "checkpoint": pth, "checkpoint_dir": str(tmp_path)})
    tcfg["kitti"] = dict(cfg["kitti"], preprocessed_path=str(tmp_path / "pre"), data_identifiers=[0])
    trainer = Trainer(config=tcfg)
    assert trainer.config["unsupervised_at_start"] is True
    got = export.pack_state_dict(trainer.model.state_dict(), cfg)
    assert np.array_equal(got, st.weights)
    opt_state = trainer.optimizer.state_dict()["state"]
    assert np.array_equal(np.concatenate([opt_state[i]["exp_avg"].cpu().reshape(-1).numpy()
                                          for i in range(len(opt_state))]), st.exp_avg)
    assert all(float(s["step"]) == 4.0 for s in opt_state.values())
