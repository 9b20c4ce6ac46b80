"""-m gpu: the po2po_alone objective (DELORA_LOSS_PO2PO_ALONE) and the objective a .dlw records, on the H100.

- the points-only front end (delora_project_points_fwd) writes the image, index map and point grid of
  delora_project_normals_fwd bit for bit and an all-zero normal grid, on synthetic scans at the model width and at a
  preprocessing width and on the adversarial projection clouds;
- the dense operator on all-zero normal grids with DELORA_LOSS_PO2PO keeps every source's exact nearest neighbour
  (tests/nn_reference.py) on the dense search's tie and near-tie grids;
- _train_step under the bit matches the Python mirror's step with po2po_alone (Deployer.step: zero normal grids,
  LOSS_PO2PO) within the bounds of the other training tests, at w_pre 0 and 2250, B 1 and 3, and with the identity fit;
  with DROPOUT and NORMALIZATION_SCALING its loss rows have the objective's shape ([po2po, 0, 0, 0, M', ...]) and
  two workspaces give the same bits;
- _train_eval is the step's outputs bit for bit and leaves the model section alone;
- the adapting streams at S = 1 serve the rows and state of _train_step at B = 1; the residual and recipe streams
  serve the shipped objective's T, point-to-point rows only, the residual's the dense operator's on points-only grids;
- the objective read from a .dlw gives the bits of the same flags passed by hand."""
import os

import numpy as np
import pytest
import torch

import odometry_harness as H
import projection_reference as PR
from delora_b200 import ops
from delora_b200.deploy import capi, export
from nn_scenes import GRID_IDS, GRIDS, Scene, near_tie_scene, tie_scene

pytestmark = pytest.mark.gpu
DEV = H.DEV
ALONE = ops.LOSS_PO2PO | ops.LOSS_PO2PO_ALONE
LR = 1e-4


def _cfg(h, w, w_pre=0, **over):
    cfg = H.config(h, w)
    cfg.update({"po2po_alone": True, "point_to_point_loss": True, "point_to_plane_loss": False,
                "plane_to_plane_loss": False})
    if w_pre:
        cfg["kitti"]["horizontal_cells_preprocessing"] = w_pre
    cfg.update(over)
    return cfg


def _front_ends(pts, counts, h, w, hf, vf):
    torch.cuda.synchronize()
    a = ops.project_normals(pts, counts, h, w, hf, vf)
    b = ops.project_points(pts, counts, h, w, hf, vf)
    torch.cuda.synchronize()
    for name, x, y in zip(("image", "index_map", "pts_grid"), a[:3], b[:3]):
        if x.dtype == torch.float32:
            assert PR.same(x.cpu().numpy(), y.cpu().numpy()).all(), f"{name} differs from the fused kernel's"
        else:
            assert torch.equal(x, y), f"{name} differs from the fused kernel's"
    assert int((b[2][..., 3].view(torch.int32) >= 0).sum()) == int((a[2][..., 3].view(torch.int32) >= 0).sum())
    assert not bool(b[3].view(torch.int32).any()), "the points-only front end wrote a non-zero normal grid"
    assert bool(a[3][..., 3].any()), "the scene has no normal: it does not tell the two front ends apart"


@pytest.mark.parametrize("w", [720, 2250, 2048], ids=["64x720", "64x2250-w_pre", "64x2048"])
def test_points_only_front_end_on_scans(cuda_lib, w):
    cfg = H.config(64, w)
    frames = H.frames(64, 2048, 4)
    pts, counts = H.stack(frames, max(f.shape[1] for f in frames))
    _front_ends(pts, counts, 64, w, cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"])


@pytest.mark.parametrize("family", sorted(PR.FAMILIES))
def test_points_only_front_end_on_adversarial_clouds(cuda_lib, family):
    for h, w, fov in ((64, 720, "full"), (16, 180, "narrow")):
        cloud = PR.family(family, 5, h, w, fov)
        pts = torch.from_numpy(np.ascontiguousarray(cloud, np.float32))[None].to(DEV)
        counts = torch.tensor([cloud.shape[1]], dtype=torch.int32, device=DEV)
        hf, vf = PR.FOVS[fov]
        torch.cuda.synchronize()
        a = ops.project_normals(pts, counts, h, w, hf, vf)
        b = ops.project_points(pts, counts, h, w, hf, vf)
        torch.cuda.synchronize()
        assert PR.same(a[0].cpu().numpy(), b[0].cpu().numpy()).all(), f"{family}: image differs"
        assert torch.equal(a[1], b[1]), f"{family}: index map differs"
        assert PR.same(a[2].cpu().numpy(), b[2].cpu().numpy()).all(), f"{family}: point grid differs"
        assert not bool(b[3].view(torch.int32).any()), f"{family}: non-zero normal grid"


@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_nn_ids_on_zero_normal_grids_are_exact(cuda_lib, grid):
    h, w, hf, vf = grid
    scenes = [Scene(f"ties {m}", h, w, hf, vf, *tie_scene(h, w, hf, vf, 7 + h, m)[:2]) for m in (False, True)]
    scenes.append(Scene("near ties", h, w, hf, vf, *near_tie_scene(h, w, hf, vf, 1e-6, 3)[:2]))
    for sc in scenes:
        zeros = torch.zeros((sc.B, h * w, 4), dtype=torch.float32, device=DEV)
        out = ops.icp_dense_information(sc.sg, zeros, sc.eye, sc.tg, zeros, h, w, hf, vf, 1.0, ops.LOSS_PO2PO)
        torch.cuda.synchronize()
        got = out[3].cpu().numpy().astype(np.int64)
        want = np.full((sc.B, h * w), -1, np.int64)
        if len(sc.pix):
            want[sc.pair, sc.slot] = sc.ref.nn
        bad = np.argwhere(got != want)
        assert len(bad) == 0, f"{sc.name}: {len(bad)} NN ids differ from the exact NN, first {bad[0].tolist()}"
        lo = out[0].cpu().numpy()
        assert (lo[:, 1:4] == 0).all() and (lo[:, 4] > 0).all(), "pairs other than point to point"


def _mirror_step(m, cfg, pts, counts, w_pre=0, identity=False):
    """H.python_step as Deployer.step runs po2po_alone: the normal grids zeroed, LOSS_PO2PO."""
    from delora_b200.deploy.deployer import _FusedIcp
    from delora_b200.models.model_parts import GeometryHandler
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    b = pts.shape[0] // 2
    if w_pre > 0:
        plist, nlist, lens = H._preprocessed_lists(cfg, pts, counts, w_pre)
        image, imap = ops.project(plist, lens, h, w, hf, vf)
        pg, ng = ops.grids_from_projection(plist, nlist, imap)
    else:
        image, _ = ops.project(pts, counts, h, w, hf, vf)
        _, pg, ng = ops.normals(image, ds["neighborhood_side_length"], cfg["epsilon_range"],
                                cfg["min_num_points_in_neighborhood_to_determine_point_class"], grids=True)
    ng = torch.zeros_like(ng)
    img1, img2 = image[:b].contiguous(), image[b:].contiguous()
    with torch.no_grad():
        pooled = m._tensor_core_path().pooled_features(img1, img2)
    m.zero_grad(set_to_none=True)
    trans, quat = m(image_1=img1, image_2=img2)
    T = GeometryHandler.get_transformation_matrix_quaternion(trans.float(), quat.float(), DEV)
    total, parts = _FusedIcp.apply(T, pg[b:].contiguous(), ng[b:].contiguous(), pg[:b].contiguous(),
                                   ng[:b].contiguous(), (h, w, hf, vf), float(cfg["lambda_po2pl"]), ops.LOSS_PO2PO,
                                   ops.icp_scratch(b, h * w, pts.device))
    loss = torch.nn.MSELoss()(T[-1:], torch.eye(4, device=DEV).view(1, 4, 4)) / b if identity else total.mean()
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    return H.Step(parts.detach(), T.detach(), pooled, grads, loss.item())


STEP_CASES = [(0, 1, False), (0, 3, False), (2250, 1, False), (2250, 3, False), (0, 3, True), (2250, 3, True)]


@pytest.mark.parametrize("w_pre,b,identity", STEP_CASES,
                         ids=[f"w_pre{w}-B{b}{'-identity' if i else ''}" for w, b, i in STEP_CASES])
def test_step_matches_the_mirror(cuda_lib, w_pre, b, identity):
    cfg = _cfg(64, 720, w_pre)
    model = H.model(cfg, near_identity=True)
    pairs = H.pairs(64, 2048, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    flags = ALONE | (ops.LOSS_IDENTITY_FIT if identity else 0)
    tr = H.trainer(cfg, n_stride, b, H.blob(model, cfg), w_pre=w_pre, flags=flags)
    losses, T, pooled, grads = tr.step(pts, counts)
    py = _mirror_step(model, cfg, pts, counts, w_pre=w_pre, identity=identity)
    torch.cuda.synchronize()
    assert torch.equal(pooled, py.pooled), "pooled features differ from the mirror's"
    t_err = (T - py.T).abs().max().item()
    assert t_err <= 1e-5, f"max |T - T_py| = {t_err:.3e}"
    assert float(losses[:, 1:4].abs().max()) == 0.0, "pairs other than point to point"
    assert float(losses[:, 4].min()) > 100, "too few pairs for a meaningful comparison"
    l_err = H.rel(losses[:, :3], py.losses[:, :3])
    assert l_err <= 1e-5, f"losses differ by {l_err:.3e} (relative)"
    tail, trunk = H.grad_spread(H.grad_dict(grads, cfg), py.grads)
    print(f"\n[w_pre={w_pre} B={b} identity={identity}] T {t_err:.2e} losses {l_err:.2e} grads: tail {tail:.2e}, "
          f"trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= H.TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"


@pytest.mark.parametrize("extra", ["dropout", "normalization_scaling"])
def test_step_with_dropout_or_scaling(cuda_lib, extra):
    cfg = _cfg(64, 720, 2250, **{("use_dropout" if extra == "dropout" else extra): True})
    model = H.model(cfg, near_identity=True)
    pairs = H.pairs(64, 2048, 3)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    hp = capi.train_params(cfg, LR)
    bit = ops.TRAIN_DROPOUT if extra == "dropout" else ops.TRAIN_NORMALIZATION_SCALING
    assert hp.loss_flags == ALONE | bit
    runs = [capi.TrainingWorkspace(H.desc(cfg, n_stride, 3, 2250), H.blob(model, cfg), hp) for _ in range(2)]
    outs = [ws.step(pts, counts) for ws in runs]
    torch.cuda.synchronize()
    for x, y in zip(*outs):
        assert H.same(x, y), "two workspaces with the same step differ"
    assert H.same_state(H.state(runs[0]), H.state(runs[1]))
    losses = outs[0][0]
    assert float(losses[:, 1:4].abs().max()) == 0.0, "pairs other than point to point"
    assert float(losses[:, 0].min()) > 0 and float(losses[:, 4].min()) > 100
    # the step without the bit estimates normals, and pairs differently
    plain = capi.TrainingWorkspace(H.desc(cfg, n_stride, 3, 2250), H.blob(model, cfg),
                                   capi.train_params(cfg, LR, loss_flags=ops.LOSS_PO2PO)).step(pts, counts)[0]
    torch.cuda.synchronize()
    assert not torch.equal(plain[:, 4], losses[:, 4])


@pytest.mark.parametrize("w_pre", [0, 2250])
def test_eval_is_the_step_and_leaves_the_model(cuda_lib, w_pre):
    cfg = _cfg(64, 720, w_pre)
    model = H.model(cfg, 3, near_identity=True)
    pairs = H.pairs(64, 2048, 3)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    ev = H.trainer(cfg, n_stride, 3, blob, LR, w_pre, ALONE)
    before = H.state(ev)
    got = ev.eval(pts, counts)
    step = H.trainer(cfg, n_stride, 3, blob, LR, w_pre, ALONE).step(pts, counts)
    torch.cuda.synchronize()
    for name, x, y in zip(("losses", "T", "pooled"), got, step[:3]):
        assert H.same(x, y), f"{name}: _train_eval differs from _train_step"
    assert H.same_state(H.state(ev), before), "_train_eval changed the model section"


def _ticks(frames, n_stride):
    return H.stage_ticks(np.ones((len(frames), 1), dtype=bool), n_stride, lambda k, s: frames[k])


@pytest.mark.parametrize("w_pre", [0, 360])
def test_one_adapting_stream_is_the_training_step(cuda_lib, w_pre):
    K = 4
    cfg = _cfg(16, 180, w_pre)
    frames = H.frames(16, 512, K)
    n_stride = max(f.shape[1] for f in frames)
    blob = H.blob(H.model(cfg, 11, near_identity=True), cfg)
    d = H.desc(cfg, n_stride, 1, w_pre)
    hp = capi.train_params(cfg, LR)
    assert hp.loss_flags == ALONE
    ws = capi.AdaptiveStreamsWorkspace(d, blob, hp)
    tr = capi.TrainingWorkspace(d, blob, hp)
    out = H.run_streams(ws, _ticks(frames, n_stride), ("losses",), updates=[True] * K, hook=H.state)
    for k, (T, valid, losses, state) in enumerate(out):
        assert int(valid[0]) == (1 if k else 0)
        if k:
            pts, counts = H.stack([frames[k - 1], frames[k]], n_stride)
            l_ref, t_ref = tr.step(pts, counts)[:2]
            torch.cuda.synchronize()
            assert H.same(T[0], t_ref.reshape(16).cpu()), f"tick {k}: T differs from _train_step at B = 1"
            assert H.same(losses[0], l_ref[0].cpu()), f"tick {k}: {losses[0].tolist()} != {l_ref[0].tolist()}"
            assert float(losses[0, 1:4].abs().max()) == 0.0 and float(losses[0, 4]) > 0
        assert H.same_state(state, H.state(tr)), f"tick {k}: the training state differs from _train_step's"


@pytest.mark.parametrize("kind,w_pre", [("residual", 0), ("pre", 360)])
def test_residual_and_recipe_streams(cuda_lib, kind, w_pre):
    """T and valid are the bits the shipped objective's workspace serves (the points are the same, only the normals are
    not estimated); every valid row is point to point only, and the residual's row is the dense operator's at B = 1 on
    the points-only grids of the two frames with DELORA_LOSS_PO2PO."""
    K = 4
    cfg = _cfg(16, 180, w_pre)
    frames = H.frames(16, 512, K)
    n_stride = max(f.shape[1] for f in frames)
    blob = H.blob(H.model(cfg, 11, near_identity=True), cfg)
    d = H.desc(cfg, n_stride, 1, w_pre)
    kind_cls = capi.ResidualStreamsWorkspace if kind == "residual" else capi.PreStreamsWorkspace
    rp = capi.residual_params(cfg)
    assert rp.loss_flags == ALONE
    got = H.run_streams(kind_cls(d, blob, rp), _ticks(frames, n_stride), ("losses",))
    shipped = H.run_streams(kind_cls(d, blob, capi.residual_params(cfg, ops.LOSS_PO2PL | ops.LOSS_PL2PL)),
                            _ticks(frames, n_stride), ("losses",))
    hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
    for k, ((T, valid, losses), (T2, valid2, _)) in enumerate(zip(got, shipped)):
        assert H.same(T, T2) and torch.equal(valid, valid2), f"tick {k}: T or valid differ from the shipped objective's"
        assert int(valid[0]) == (1 if k else 0)
        if not k:
            continue
        assert float(losses[0, 1:4].abs().max()) == 0.0 and float(losses[0, 4]) > 0
        if kind == "residual":
            pts, counts = H.stack([frames[k - 1], frames[k]], n_stride)
            _, _, pg, ng = ops.project_points(pts, counts, 16, 180, hf, vf)
            row = ops.icp_dense_fwd_bwd(pg[1:], ng[1:], T[:, :12].contiguous().to(DEV), pg[:1], ng[:1], 16, 180, hf, vf,
                                        1.0, ops.LOSS_PO2PO)[0]
            torch.cuda.synchronize()
            assert H.same(losses[0], row[0].cpu()), f"tick {k}: {losses[0].tolist()} != {row[0].tolist()}"


OBJECTIVES = {"linear": {"normal_loss": "linear"}, "lambda_10": {"lambda_po2pl": 10.0},
              "point_to_point": {"point_to_point_loss": True},
              "po2po_alone": {"po2po_alone": True, "point_to_point_loss": True, "point_to_plane_loss": False,
                              "plane_to_plane_loss": False}}
BY_HAND = {"linear": (ops.LOSS_PO2PL | ops.LOSS_PL2PL | ops.NORMAL_LINEAR, 1.0),
           "lambda_10": (ops.LOSS_PO2PL | ops.LOSS_PL2PL, 10.0),
           "point_to_point": (ops.LOSS_PO2PO | ops.LOSS_PO2PL | ops.LOSS_PL2PL, 1.0), "po2po_alone": (ALONE, 1.0)}


@pytest.mark.parametrize("name", sorted(OBJECTIVES))
def test_the_objective_read_from_a_file_is_the_flags_by_hand(cuda_lib, tmp_path, name):
    """Export -> read_dlw -> config_from_desc -> the binding's default parameters give the bits of a step whose flags
    and lambda_po2pl are passed by hand; the shipped objective differs."""
    base = H.config(16, 180)
    cfg = dict(base, **OBJECTIVES[name])
    model = H.model(cfg, 4, near_identity=True)
    pairs = H.pairs(16, 512, 2)
    n_stride = H.n_stride(pairs)
    d = H.desc(cfg, n_stride, 2)
    dlw = os.path.join(tmp_path, "m.dlw")
    export.write_dlw(dlw, d, export.pack_state_dict(model.state_dict(), cfg), 0, export.objective_from_config(cfg))
    h, d2, blob = export.read_dlw(dlw)
    from_file = export.config_from_desc(d2, base, "kitti", h["model_flags"], (h["objective_flags"], h["lambda_po2pl"]))
    pts, counts = H.stack_pairs(pairs, n_stride)
    weights = torch.from_numpy(blob).to(DEV)
    hp_file = capi.train_params(from_file, LR)
    flags, lam = BY_HAND[name]
    hp_hand = capi.train_params(dict(base, lambda_po2pl=lam), LR, loss_flags=flags)
    assert (hp_file.loss_flags, hp_file.lambda_po2pl) == (hp_hand.loss_flags, hp_hand.lambda_po2pl)
    a = capi.TrainingWorkspace(d2, weights, hp_file).step(pts, counts)
    b = capi.TrainingWorkspace(d2, weights, hp_hand).step(pts, counts)
    shipped = capi.TrainingWorkspace(d2, weights, capi.train_params(base, LR)).step(pts, counts)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert H.same(x, y)
    assert not H.same(a[0], shipped[0]) or not H.same(a[3], shipped[3])


@pytest.mark.parametrize("objective", ["po2po_alone", "zeros"])
def test_examples_train_and_adapt_on_the_files_objective(cuda_lib, tmp_path, objective):
    """odometry_train on a .dlt and odometry_streams --adapt on a .dlw print the objective the header records (the
    shipped one for a file with zeros there) and run on it: the po2po_alone file trains to other weights."""
    import subprocess
    from delora_b200 import synthetic
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 180, "tanh", False, layers=(1, 1, 1, 1), nout=64)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    alone = dict(cfg, **OBJECTIVES["po2po_alone"])
    rec = export.objective_from_config(alone) if objective == "po2po_alone" else None
    want = "objective po2po_alone, lambda_po2pl 1" if rec else "objective po2pl pl2pl (squared normal loss), lambda_po2pl 1"
    d = export.desc_from_config(cfg, "kitti", 4096, 1)
    model = H.model(cfg, 6, near_identity=True)
    blob = export.pack_state_dict(model.state_dict(), cfg)
    dlw, dlt = os.path.join(tmp_path, "m.dlw"), os.path.join(tmp_path, "m.dlt")
    export.write_dlw(dlw, d, blob, 0, rec)
    export.write_dlt(dlt, d, export.TrainingState(blob, np.zeros_like(blob), np.zeros_like(blob), unsupervised=1,
                                                   lr=1e-4), 0, rec)
    stream = os.path.join(tmp_path, "s0")
    os.makedirs(stream)
    for i in range(3):
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(os.path.join(stream, f"{i:06d}.bin"))
    bins = [os.path.join(stream, f"{i:06d}.bin") for i in range(3)]
    train = H.build_example("odometry_train", tmp_path, link=True)
    r = subprocess.run([train, dlt, os.path.join(tmp_path, "out.dlt"), "1", "1"] + bins, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert f"odometry_train: {want}" in r.stderr, r.stderr
    trained = export.read_dlt(os.path.join(tmp_path, "out.dlt"))
    assert (trained[0]["objective_flags"], trained[0]["lambda_po2pl"]) == (rec or (0, 0.0))
    streams = H.build_example("odometry_streams", tmp_path, link=True)
    out = os.path.join(tmp_path, "a.dlw")
    r = subprocess.run([streams, "--adapt", "1e-4", "--adapt-out", out, dlw, stream], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    assert f"odometry_streams: {want}" in r.stderr, r.stderr
    assert len(r.stdout.strip().splitlines()) == 2, r.stdout
    # the same file with its objective cleared adapts on the shipped objective, to other weights
    if rec:
        plain = os.path.join(tmp_path, "plain.dlw")
        export.write_dlw(plain, d, blob)
        out2 = os.path.join(tmp_path, "b.dlw")
        r2 = subprocess.run([streams, "--adapt", "1e-4", "--adapt-out", out2, plain, stream], capture_output=True,
                            text=True, timeout=300)
        assert r2.returncode == 0, r2.stderr
        assert not np.array_equal(export.read_dlw(out)[2], export.read_dlw(out2)[2])
