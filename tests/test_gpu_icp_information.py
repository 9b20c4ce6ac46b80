"""-m gpu: the Gauss-Newton information of the ICP objective (delora_icp_dense_information) and the information streams
(delora_odometry_streams_push_info) on the H100.

  - Operator, on ray-cast single-plane, corridor, two-plane and box-room scenes and a synthetic street scan, over every
    loss-flag combination: the NN ids are the exact NN (nn_reference) under the losses' masks; H matches the float64
    restatement (info_reference) within 64 u A + u |H|, A the magnitude sum the fp32 rounding is relative to; the
    eigen-pairs match numpy.linalg.eigh; losses and grad_T are delora_icp_dense_fwd_bwd's bits; rows are repeatable
    bit for bit and the same at B = 1 as inside a batch.
  - Degeneracy is seen (po2pl only): in a corridor along x the smallest eigenvalue is below 2e-3 of the largest with
    its eigenvector within 5 degrees of x-translation; a single plane has three eigenvalues below 1e-3 of the largest;
    a box room has all six above 1e-2 of the largest.
  - Streams: T, valid and losses are _push_residual's bytes over a history with resets and inactive streams; each valid
    info row is the operator's row alone at B = 1; invalid rows are zeros; a graph-replayed tick equals an eager one.
"""
import functools
import math

import numpy as np
import pytest
import torch

import icp_reference as R
import info_reference as IR
import nn_reference as NR
import odometry_harness as OH
from delora_b200 import ops, synthetic
from delora_b200.deploy import capi

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
HH, WW = 32, 360
VFOV = (-25.0, 15.0)

# axis-aligned rectangles: (axis of the normal, coordinate, bounds of the other two axes in order)
SCENES = {
    "plane": [(2, -1.7, (-60, 60), (-60, 60))],
    "corridor": [(1, -2.0, (-40, 40), (-1.5, 1.5)), (1, 2.0, (-40, 40), (-1.5, 1.5)),
                 (2, -1.5, (-40, 40), (-2, 2)), (2, 1.5, (-40, 40), (-2, 2))],
    "two-plane": [(2, -1.7, (-60, 60), (-60, 60)), (0, 6.0, (-60, 60), (-1.7, 4))],
    "box-room": [(0, -5.0, (-4, 3), (-1.7, 2.5)), (0, 7.0, (-4, 3), (-1.7, 2.5)), (1, -4.0, (-5, 7), (-1.7, 2.5)),
                 (1, 3.0, (-5, 7), (-1.7, 2.5)), (2, -1.7, (-5, 7), (-4, 3)), (2, 2.5, (-5, 7), (-4, 3))],
}
POSE = IR.exp_se3(np.array([0.25, 0.08, 0.02, 0.004, -0.003, 0.02]))     # source sensor in the target's frame


def _fov():
    cfg = synthetic.fov_config(h=HH, w=WW, vfov_deg=VFOV)
    return tuple(cfg["horizontal_field_of_view"]), tuple(cfg["kitti"]["vertical_field_of_view"])


def _raycast(rects, pose, seed, n=4 * HH * WW):
    """[3, N] fp32 points in the sensor frame of `pose` (4 x 4, world <- sensor): the nearest rectangle hit by each of
    n seeded rays spread over the field of view."""
    g = np.random.default_rng(seed)
    az = g.uniform(-math.pi, math.pi, n)
    el = np.radians(g.uniform(VFOV[0], VFOV[1], n))
    d = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1)
    dw, o = d @ pose[:3, :3].T, pose[:3, 3]
    best = np.full(n, np.inf)
    for ax, c, b0, b1 in rects:
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (c - o[ax]) / dw[:, ax]
        x = o + t[:, None] * dw
        others = [k for k in range(3) if k != ax]
        ok = (t > 0.3) & (t < 80) & (x[:, others[0]] >= b0[0]) & (x[:, others[0]] <= b0[1]) \
            & (x[:, others[1]] >= b1[0]) & (x[:, others[1]] <= b1[1])
        best = np.where(ok & (t < best), t, best)
    hit = np.isfinite(best)
    return (d[hit] * best[hit, None]).T.astype(np.float32)


@functools.lru_cache(maxsize=None)
def scene(name):
    """-> (target grids pg, ng [1, HW, 4], source grids, T [1, 12]) of one scene on the GPU."""
    hf, vf = _fov()
    if name == "random":
        made = synthetic.make_pair(41, w_raw=4 * WW, rings=HH, vfov_deg=VFOV)
        clouds, T = [made[0], made[1]], made[3].numpy().astype(np.float32)[:3]
    else:
        clouds = [_raycast(SCENES[name], np.eye(4), 1), _raycast(SCENES[name], POSE, 2)]
        clouds = [torch.from_numpy(c) for c in clouds]
        T = POSE[:3].astype(np.float32)
    out = []
    for c in clouds:
        c = c[0] if c.dim() == 3 else c
        pts = c.reshape(1, 3, -1).contiguous().to(DEV)
        cnt = torch.tensor([pts.shape[2]], dtype=torch.int32, device=DEV)
        _, _, pg, ng = ops.project_normals(pts, cnt, HH, WW, hf, vf)
        out.append((pg, ng))
    return out[0], out[1], torch.from_numpy(np.ascontiguousarray(T.reshape(1, 12))).to(DEV)


def run(names, flags, lam=1.0):
    hf, vf = _fov()
    tg = torch.cat([scene(n)[0][0] for n in names]), torch.cat([scene(n)[0][1] for n in names])
    sg = torch.cat([scene(n)[1][0] for n in names]), torch.cat([scene(n)[1][1] for n in names])
    T = torch.cat([scene(n)[2] for n in names])
    return ops.icp_dense_information(sg[0], sg[1], T, tg[0], tg[1], HH, WW, hf, vf, lam, flags)


def reference(name, flags, lam=1.0):
    """-> (expected kept NN ids [HW] int64, ids without a safe exact answer, H, A, M, M') in float64."""
    (tp, tn), (sp, sn), T = scene(name)
    tp, tn, sp, sn = (x[0].cpu().numpy() for x in (tp, tn, sp, sn))
    T = T[0].cpu().numpy()
    t_ok = tp[:, 3].view(np.int32) >= 0
    s_ok = sp[:, 3].view(np.int32) >= 0
    t_ids = np.nonzero(t_ok)[0]
    s, _ = R.apply_rigid(T, sp[s_ok, :3], sn[s_ok, :3])
    res = NR.nearest(tp[t_ok, :3], t_ids, s)
    nn = np.full(HH * WW, -1, np.int64)
    nn[np.nonzero(s_ok)[0]] = res.nn
    unsafe = np.nonzero(s_ok)[0][res.unsafe]
    kind = IR.pair_masks(T, sp[:, :3], sn[:, :3], tn[:, :3], tn[:, 3] != 0, nn, flags)
    expected = np.where(kind > 0, nn, -1)
    Hm, A, M, Mp = IR.information(T, sp[:, :3], sn[:, :3], tn[:, :3], tn[:, 3] != 0, expected, flags, lam)
    return expected, unsafe, Hm, A, M, Mp


def check_eigen(info, Hm, label):
    ev, V = info[36:42].astype(np.float64), info[42:78].reshape(6, 6).astype(np.float64)
    ref_ev, ref_V = IR.eig_row(Hm)
    lmax = max(abs(ref_ev).max(), 1e-30)
    dH = np.linalg.norm(info[:36].reshape(6, 6).astype(np.float64) - Hm) + 1e-6 * lmax
    assert np.all(np.diff(ev) >= 0), f"{label}: eigenvalues not ascending"
    assert np.abs(ev - ref_ev).max() <= dH, (label, ev, ref_ev)
    for k in range(6):
        v = V[k]
        assert abs(np.linalg.norm(v) - 1.0) < 1e-5, label
        big = int(np.argmax(np.abs(v)))
        assert v[big] > 0, f"{label}: eigenvector {k} breaks the sign convention"
        gap = min([abs(ref_ev[k] - ref_ev[j]) for j in range(6) if j != k])
        if gap > 1e-3 * lmax:
            assert abs(v @ ref_V[k]) >= 1.0 - 2.0 * (dH / gap) ** 2 - 1e-5, (label, k, v, ref_V[k])


FLAGS = R.flag_matrix()


@pytest.mark.parametrize("name", ["plane", "corridor", "two-plane", "box-room", "random"])
@pytest.mark.parametrize("flags", FLAGS, ids=R.flag_name)
def test_operator_against_float64(name, flags, cuda_lib):
    lam = 0.6
    losses, grad, info, nn = run([name], flags, lam)
    expected, unsafe, Hm, A, M, Mp = reference(name, flags, lam)
    got = nn[0].cpu().numpy().astype(np.int64)
    keep = np.ones(HH * WW, bool)
    keep[unsafe] = False
    bad = np.nonzero((got != expected) & keep)[0]
    assert bad.size == 0, f"{name}: {bad.size} NN ids differ from the exact NN, first {bad[:5]}"
    if unsafe.size:                       # an ambiguous source may take either answer: restate H with the kernel's
        (_, tn), (sp, sn), T = scene(name)
        tn = tn[0].cpu().numpy()
        Hm, A, M, Mp = IR.information(T[0].cpu().numpy(), sp[0].cpu().numpy()[:, :3], sn[0].cpu().numpy()[:, :3],
                                      tn[:, :3], tn[:, 3] != 0, got, flags, lam)
    row = info[0].cpu().numpy()
    Hg = row[:36].reshape(6, 6).astype(np.float64)
    tol = 64 * U * A + U * np.abs(Hm)
    assert np.all(np.abs(Hg - Hm) <= tol), f"{name}: max |dH| / tol = {(np.abs(Hg - Hm) / tol).max():.3g}"
    assert row[78] == M and row[79] == Mp and row[78] == float(losses[0, 3]) and row[79] == float(losses[0, 4])
    check_eigen(row, Hm, name)
    hf, vf = _fov()
    (tp, tn), (sp, sn), T = scene(name)
    l2, g2 = ops.icp_dense_fwd_bwd(sp, sn, T, tp, tn, HH, WW, hf, vf, lam, flags)
    assert torch.equal(losses.view(torch.int32), l2.view(torch.int32)), f"{name}: losses differ from fwd_bwd"
    assert torch.equal(grad.view(torch.int32), g2.view(torch.int32)), f"{name}: grad_T differs from fwd_bwd"


@pytest.mark.parametrize("flags", [ops.LOSS_PO2PL | ops.LOSS_PL2PL, R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL | 8])
def test_repeatable_and_independent_of_the_batch(flags, cuda_lib):
    names = ["plane", "corridor", "box-room", "random", "two-plane"]
    first = run(names, flags)
    again = run(names, flags)
    for a, b in zip(first, again):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "a second run differs"
    for k, n in enumerate(names):
        alone = run([n], flags)
        for a, b in zip(first, alone):
            assert torch.equal(a[k].view(torch.int32), b[0].view(torch.int32)), f"{n}: B = 1 differs from the batch"


def _eig(name):
    info = run([name], ops.LOSS_PO2PL)[2][0].cpu().numpy().astype(np.float64)
    return info[36:42], info[42:78].reshape(6, 6)


def test_corridor_leaves_translation_along_it_free(cuda_lib):
    ev, V = _eig("corridor")
    ratio = ev[0] / ev[5]
    angle = math.degrees(math.acos(min(1.0, abs(V[0, 0]))))
    print(f"corridor: lambda_min / lambda_max = {ratio:.3g}, angle to x-translation {angle:.3g} deg")
    assert ratio < 2e-3 and angle < 5.0, (ev, V[0])
    assert ev[1] > 1e-2 * ev[5]


def test_single_plane_has_three_free_directions(cuda_lib):
    ev, V = _eig("plane")
    print(f"plane: eigenvalues / largest = {ev / ev[5]}")
    assert np.all(ev[:3] < 1e-3 * ev[5]) and np.all(ev[3:] > 1e-2 * ev[5]), ev
    free = V[:3]                          # x, y translation and rotation about z span the free subspace
    for axis in (0, 1, 5):
        assert np.linalg.norm(free[:, axis]) > 0.99, (axis, free)


def test_box_room_constrains_every_direction(cuda_lib):
    ev, _ = _eig("box-room")
    print(f"box room: eigenvalues / largest = {ev / ev[5]}")
    assert np.all(ev > 1e-2 * ev[5]), ev


# ============================================================================================ _push_info
from test_gpu_odometry_eval import _streams_setup  # noqa: E402


def _info_rows(cfg, ticks, act, resets, out, flags):
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    S = act.shape[1]
    prev, rows = [None] * S, {}
    for k, (p, c, _) in enumerate(ticks):
        for s in resets.get(k, []):
            prev[s] = None
        T = out[k][0]
        for s in range(S):
            if not act[k, s]:
                continue
            _, _, pg, ng = ops.project_normals(p[s:s + 1].to(DEV), c[s:s + 1].to(DEV), h, w, hf, vf,
                                               ds["neighborhood_side_length"], cfg["epsilon_range"],
                                               cfg["min_num_points_in_neighborhood_to_determine_point_class"])
            if prev[s] is not None:
                rows[(k, s)] = ops.icp_dense_information(pg, ng, T[s:s + 1, :12].contiguous().to(DEV), prev[s][0],
                                                         prev[s][1], h, w, hf, vf, float(cfg["lambda_po2pl"]),
                                                         flags)[2][0].cpu()
            prev[s] = (pg, ng)
    return rows


@pytest.mark.parametrize("S,flags", [(1, ops.LOSS_PO2PL | ops.LOSS_PL2PL), (4, ops.LOSS_PO2PL | ops.LOSS_PL2PL),
                                     (4, R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL | 8)],
                         ids=["S1", "S4", "S4-all-losses-linear"])
def test_streams_info_rows_beside_the_residuals_bytes(S, flags, cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _streams_setup(S)
    d = OH.desc(cfg, n_stride, S)
    res = OH.run_streams(capi.ResidualStreamsWorkspace(d, blob, capi.residual_params(cfg, flags)), ticks, ("losses",),
                         resets=resets)
    out = OH.run_streams(capi.InformationStreamsWorkspace(d, blob, capi.residual_params(cfg, flags)), ticks,
                         ("losses", "info"), resets=resets)
    for k, (r, o) in enumerate(zip(res, out)):
        assert torch.equal(r[1], o[1]), f"tick {k}: valid differs from _push_residual"
        for a, b, what in ((r[0], o[0], "T"), (r[2], o[2], "losses")):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"tick {k}: {what} differs"
    rows = _info_rows(cfg, ticks, act, resets, out, flags)
    matched = 0
    for k, (_, valid, _, info) in enumerate(out):
        for s in range(S):
            if int(valid[s]):
                assert torch.equal(info[s].view(torch.int32), rows[(k, s)].view(torch.int32)), \
                    f"tick {k} stream {s}: the info row differs from the operator alone at B = 1"
                matched += int(info[s][78] > 0)
            else:
                assert float(info[s].abs().max()) == 0.0, f"tick {k} stream {s}: an invalid row is not zero"
    assert matched > 0


def test_streams_info_graph_replay_matches_eager(cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _streams_setup(4)
    d = OH.desc(cfg, n_stride, 4)
    rp = capi.residual_params(cfg)
    eager = OH.run_streams(capi.InformationStreamsWorkspace(d, blob, rp), ticks, ("losses", "info"), resets=resets)
    graphed = OH.run_streams(capi.InformationStreamsWorkspace(d, blob, rp), ticks, ("losses", "info"), resets=resets,
                             graph=True)
    for k, (e, g) in enumerate(zip(eager, graphed)):
        for a, b in zip(e, g):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"tick {k}: the replay differs"


def test_python_class_returns_info_beside_the_residual(cuda_lib):
    from delora_b200.deploy.stream import InformationOdometryStreams, OdometryStreams
    cfg = OH.config(16, 180)
    model = OH.model(cfg, 32, near_identity=True).eval()
    pool = OH.frames(16, 256, 4)
    n_max = max(s.shape[1] for s in pool) + 8
    a = OdometryStreams(model, cfg, "kitti", 2, n_max, residual=True)
    b = InformationOdometryStreams(model, cfg, "kitti", 2, n_max)
    for k in range(3):
        scans = [pool[k].cpu(), pool[(k + 1) % 4].cpu()]
        ra, rb = a.push(scans), b.push(scans)
        for x, y in zip(ra, rb):
            if x is None:
                assert y is None
                continue
            assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
            assert y[2].shape == (ops.INFO_ROW,) and np.all(np.diff(y[2][36:42]) >= 0)
