"""-m gpu: training a model that uses normalization_scaling through the C ABI (DELORA_TRAIN_NORMALIZATION_SCALING, on
the reference's two-resolution recipe, w_pre > 0).

The Python step is test_gpu_odometry_train_pre_capi.py's mirror with the C factor injected: Preprocesser.preprocess_scans
in memory (the stored row-major point and normal lists), the points divided by the pair's factor, ops.project at W and
ops.grids_from_projection (Deployer.step after normalize_input), the tensor-core model, the fused ICP losses (in
normalised units), backward.  The bounds are that file's."""
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200 import ops

pytestmark = pytest.mark.gpu
DEV = H.DEV
FLAGS = H.FLAGS | ops.TRAIN_NORMALIZATION_SCALING


def _python_step(m, cfg, pts, counts, w_pre, factor, identity=False):
    """-> (Step with the unscaled T, the stored lists and their lengths)."""
    from delora_b200.deploy.deployer import _FusedIcp
    from delora_b200.models.model_parts import GeometryHandler
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    b = pts.shape[0] // 2
    plist, nlist, lens = H._preprocessed_lists(cfg, pts, counts, w_pre)
    scaled = plist / torch.cat((factor, factor)).view(2 * b, 1, 1)
    image, imap = ops.project(scaled, lens, h, w, hf, vf)
    pg, ng = ops.grids_from_projection(scaled, nlist, imap)
    img1, img2 = image[:b].contiguous(), image[b:].contiguous()
    with torch.no_grad():
        pooled = m._tensor_core_path().pooled_features(img1, img2)
    m.zero_grad(set_to_none=True)
    trans, quat = m(image_1=img1, image_2=img2)
    T = GeometryHandler.get_transformation_matrix_quaternion(trans.float(), quat.float(), DEV)
    total, parts = _FusedIcp.apply(T, pg[b:].contiguous(), ng[b:].contiguous(), pg[:b].contiguous(),
                                   ng[:b].contiguous(), (h, w, hf, vf), float(cfg["lambda_po2pl"]), H.FLAGS,
                                   ops.icp_scratch(b, h * w, pts.device))
    if identity:
        loss = torch.nn.MSELoss()(T[-1:], torch.eye(4, device=DEV).view(1, 4, 4)) / b
    else:
        loss = total.mean()
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    return H.Step(parts.detach(), T.detach(), pooled, grads, loss.item()), plist, lens


def _factor_f64(plist, lens):
    p, n = plist.cpu().numpy(), lens.cpu().numpy()
    b = p.shape[0] // 2
    means = []
    for i in range(2 * b):
        x, y, z = (p[i, c, :n[i]] for c in range(3))
        means.append(np.float32(np.sqrt((x * x + y * y) + z * z).astype(np.float64).sum() / n[i]))
    return np.array([(means[i] + means[b + i]) / np.float32(2.0) for i in range(b)], dtype=np.float32)


def _trainer(cfg, stride, max_batch, blob, w_pre, lr=1e-5, flags=FLAGS):
    return H.trainer(cfg, stride, max_batch, blob, lr, w_pre=w_pre, flags=flags)


CASES = [pytest.param("tanh", False, 64, 720, 2048, 2250, 1, id="tanh-64x720-2250-B1"),
         pytest.param("relu", True, 64, 720, 2048, 2250, 4, id="relu-single-64x720-2250-B4"),
         pytest.param("tanh", False, 16, 259, 512, 512, 2, id="tanh-16x259-512-B2"),
         pytest.param("relu", False, 16, 259, 512, 512, 4, id="relu-16x259-512-B4")]


@pytest.mark.parametrize("act,single,h,w,w_raw,w_pre,b", CASES)
def test_step_matches_the_mirror(cuda_lib, act, single, h, w, w_raw, w_pre, b):
    cfg = H.config(h, w, act, single)
    model = H.model(cfg, near_identity=True)
    pairs = H.pairs(h, w_raw, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    losses, T, pooled, grads = _trainer(cfg, n_stride, b, H.blob(model, cfg), w_pre).step(pts, counts)
    torch.cuda.synchronize()
    factor = losses[:, 6].clone()
    py, plist, lens = _python_step(model, cfg, pts, counts, w_pre, factor)
    torch.cuda.synchronize()
    ref_f = _factor_f64(plist, lens)
    got_f = factor.cpu().numpy()
    assert np.all(np.abs(got_f - ref_f) <= np.spacing(ref_f)), (got_f, ref_f)
    assert bool((factor > 1.0).all()), "the factor of metre-scale scans should exceed 1"
    assert torch.equal(pooled, py.pooled), "pooled features differ from the normalised mirror"
    t_ref = py.T.clone()
    t_ref[:, :3, 3] *= factor.view(b, 1)
    assert torch.equal(T[:, 3], t_ref[:, 3])
    t_err = (T - t_ref).abs().max().item() / max(1.0, t_ref.abs().max().item())
    assert t_err <= 1e-5, f"max |T - T_py| = {t_err:.3e} (relative to the transform's scale)"
    l_err = H.rel(losses[:, :3], py.losses[:, :3])
    assert l_err <= 1e-5, f"losses differ by {l_err:.3e} (relative)"
    tail, trunk = H.grad_spread(H.grad_dict(grads, cfg), py.grads)
    print(f"\n[{h}x{w} w_pre={w_pre} B={b} {act} single={single}] factor {got_f}  T {t_err:.2e}  losses {l_err:.2e}  "
          f"grads: tail {tail:.2e}, trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= H.TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"


def test_identity_fit_with_normalisation(cuda_lib):
    """The identity objective is taken on the unscaled T, with test_gpu_odometry_train_state.py's bounds."""
    from test_gpu_odometry_train_state import _tail_grads_fp64
    cfg = H.config(64, 720, "tanh", False)
    model = H.model(cfg, 14)
    pairs = H.pairs(64, 2048, 1)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    losses, T, pooled, grads = _trainer(cfg, n_stride, 1, blob, 2250, flags=FLAGS | ops.LOSS_IDENTITY_FIT).step(pts,
                                                                                                              counts)
    icp_losses = _trainer(cfg, n_stride, 1, blob, 2250).step(pts, counts)[0]
    torch.cuda.synchronize()
    factor = losses[:, 6].clone()
    py, _, _ = _python_step(model, cfg, pts, counts, 2250, factor, identity=True)
    torch.cuda.synchronize()
    assert torch.equal(pooled, py.pooled)
    assert torch.equal(losses[:, :5], icp_losses[:, :5]) and torch.equal(losses[:, 6:], icp_losses[:, 6:])
    t_unscaled = T.clone()
    t_unscaled[:, :3, 3] /= factor.view(1, 1)
    t_err = (t_unscaled - py.T).abs().max().item()
    assert t_err <= 1e-5, f"max |T / f - T_py| = {t_err:.3e}"
    obj = losses[0, 5].item()
    e = (py.T[0] - torch.eye(4, device=DEV)).double()
    own = (e * e).sum().item() / 16
    bound = 2.0 * e.abs().sum().item() * max(t_err, 1e-7) / 16 + 1e-6 * own
    assert abs(obj - py.objective) <= bound, f"objective {obj} vs the Python step's {py.objective} (bound {bound:.3e})"
    c_grads = H.grad_dict(grads, cfg)
    tail, trunk = H.grad_spread(c_grads, py.grads)
    exact = _tail_grads_fp64(model, cfg, pooled)
    c_tail = max(H.rel(c_grads[k], g.float()) for k, g in exact.items())
    py_tail = max(H.rel(py.grads[k].cpu(), g.float()) for k, g in exact.items())
    print(f"\n[identity fit, normalised, 64x720 B=1] factor {factor.item():.6g}  T {t_err:.2e}  objective {obj:.6e} "
          f"(python {py.objective:.6e})  grads: tail {tail:.2e} (C vs fp64 {c_tail:.2e}), trunk {trunk:.2e}")
    assert c_tail <= H.TAIL_TOL, f"fc / head gradients differ from the fp64 tail by {c_tail:.3e} of their max-abs"
    assert tail <= py_tail + H.TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= H.TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"


def test_deterministic_graph_replay_and_changing_batch(cuda_lib):
    cfg = H.config(64, 720, "relu", False)
    model = H.model(cfg, 4, near_identity=True)
    pairs = H.pairs(64, 2048, 4)
    n_stride = H.n_stride(pairs)
    blob = H.blob(model, cfg)
    pts, counts = H.stack_pairs(pairs[:2], n_stride)
    a, b = _trainer(cfg, n_stride, 4, blob, 2250, 1e-4), _trainer(cfg, n_stride, 4, blob, 2250, 1e-4)
    for _ in range(2):
        x, y = a.step(pts, counts), b.step(pts, counts)
        torch.cuda.synchronize()
        for u, v, name in zip(x, y, ("losses", "T", "pooled", "grads")):
            assert torch.equal(u, v), f"{name} differ between two workspaces"

    eager, graphed = _trainer(cfg, n_stride, 4, blob, 2250, 1e-4), _trainer(cfg, n_stride, 4, blob, 2250, 1e-4)
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

    tr = _trainer(cfg, n_stride, 4, blob, 2250, 1e-4)
    for bsz in (4, 1, 3):
        p, c = H.stack_pairs(pairs[:bsz], n_stride)
        before = tr.weights()
        got = tr.step(p, c)
        fresh = _trainer(cfg, n_stride, 4, before, 2250, 1e-4).step(p, c)
        torch.cuda.synchronize()
        for x, y, name in zip(got, fresh, ("losses", "T", "pooled", "grads")):
            assert torch.equal(x, y), f"B={bsz}: {name} differ from a fresh workspace"
        # a pair's factor does not depend on the batch
        assert torch.equal(got[0][:, 6], fresh[0][:, 6])


def test_the_bit_changes_the_step_and_train_params_sets_it(cuda_lib):
    from delora_b200.deploy import capi
    cfg = H.config(16, 259, "tanh", False)
    model = H.model(cfg, 8, near_identity=True)
    pairs = H.pairs(16, 512, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    plain = _trainer(cfg, n_stride, 2, blob, 512, flags=H.FLAGS).step(pts, counts)
    norm = _trainer(cfg, n_stride, 2, blob, 512).step(pts, counts)
    ncfg = dict(cfg, normalization_scaling=True)
    assert capi.train_params(ncfg, 1e-5, loss_flags=H.FLAGS).loss_flags == FLAGS
    via_config = capi.TrainingWorkspace(H.desc(ncfg, n_stride, 2, 512), blob,
                                        capi.train_params(ncfg, 1e-5, loss_flags=H.FLAGS)).step(pts, counts)
    torch.cuda.synchronize()
    assert bool((plain[0][:, 6] == 0).all())
    assert not torch.equal(plain[2], norm[2]), "the images the model sees do not change with the bit"
    for x, y in zip(norm, via_config):
        assert torch.equal(x, y)


def test_finetune_example_on_a_flagged_file(cuda_lib, tmp_path):
    """examples/odometry_finetune.c sets the bit for a flagged .dlw with w_pre > 0 and refuses one with w_pre = 0."""
    from delora_b200 import _lib, synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    cfg["kitti"]["horizontal_cells_preprocessing"] = 1024
    model = H.model(cfg, 6, near_identity=True)
    bins = []
    for i in range(4):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    exe = H.build_example("odometry_finetune", tmp_path, link=True)
    flag = _lib.MODEL_NORMALIZATION_SCALING

    bad = os.path.join(tmp_path, "plain.dlw")
    export.write_dlw(bad, export.desc_from_config(cfg, "kitti", 4096, 2), export.pack_state_dict(model.state_dict(), cfg),
                     flag)
    r = subprocess.run([exe, bad, os.path.join(tmp_path, "x.dlw"), "1", "1e-4"] + bins, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode != 0 and "w_pre" in r.stderr, r.stderr

    dlw, out = os.path.join(tmp_path, "in.dlw"), os.path.join(tmp_path, "out.dlw")
    desc = export.desc_from_config(cfg, "kitti", 4096, 2, preprocessing_normals=True)
    export.write_dlw(dlw, desc, export.pack_state_dict(model.state_dict(), cfg), flag)
    r = subprocess.run([exe, dlw, out, "3", "1e-4"] + bins, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    h, _, blob = export.read_dlw(out)
    assert h["model_flags"] == flag
    scans = [torch.from_numpy(np.fromfile(p, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()) for p in bins]
    tr = _trainer(cfg, 4096, 2, H.blob(model, cfg), 1024, 1e-4)
    for ks in ((0, 1), (2, 0), (1, 2)):
        p, c = H.stack_pairs([(scans[k], scans[k + 1]) for k in ks], 4096)
        tr.step(p, c, outputs=False)
    torch.cuda.synchronize()
    assert np.array_equal(tr.weights().cpu().numpy(), blob)
