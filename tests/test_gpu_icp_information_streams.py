"""-m gpu: the information in metres for normalised pairs (delora_icp_dense_information_scaled), the recipe streams with
the information (delora_odometry_streams_push_pre_info) and the adapting streams with the information
(delora_odometry_streams_push_adapt_info / _push_adapt_group_info) on the H100.

  - Scaled operator: with unit factors every output is delora_icp_dense_information's, bit for bit; with factors 0.05,
    0.3 and 7, H is D H D of the unscaled row (float64) within 2 u |H| per entry, the eigen-pairs match numpy's eigh of
    the served H, and losses, grad_T and the NN ids are the unscaled call's bits.
  - Recipe streams, plain and normalised, over a history with resets, inactive streams and an empty frame: T, valid,
    losses and factor are _push_pre's bytes; each valid row is the B = 1 operator's bits on the pair's grids (scaled
    with the pair's factor for the normalised model); invalid rows are zeros; a graph-replayed tick equals an eager one.
    A ray-cast corridor served to a normalised model leaves translation along it free.
  - Adapting streams: ticks with update 0 / 1 give T, valid, losses and the training state (_train_get_state) of
    _push_adapt, byte for byte, at w_pre = 0, w_pre > 0 and for a normalised model; each valid row is the B = 1 operator
    on the tick's grids at the served T.  The group push at world 1 is _push_adapt_info; at worlds 2 and 4 (ranks on one
    device) every rank gets _push_adapt_group's bytes.
  - The Python classes and the example program return the same bits as without the information.
"""
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import info_reference as IR
import odometry_harness as H
from delora_b200 import ops
from delora_b200.deploy import capi

pytestmark = pytest.mark.gpu
DEV = H.DEV
U = 2.0 ** -24
SENTINEL = 1234.5
ICP = ops.LOSS_PO2PL | ops.LOSS_PL2PL
LR = 1e-4


def _norm(normalized):
    return ops.TRAIN_NORMALIZATION_SCALING if normalized else 0


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ============================================================================================ scenes
# ray-cast scenes of test_gpu_icp_information.py: axis-aligned rectangles (axis of the normal, coordinate, bounds of
# the other two axes in order), seen from the identity and from POSE
HH, WW = 32, 360
VFOV = (-25.0, 15.0)
SCENES = {
    "corridor": [(1, -2.0, (-40, 40), (-1.5, 1.5)), (1, 2.0, (-40, 40), (-1.5, 1.5)),
                 (2, -1.5, (-40, 40), (-2, 2)), (2, 1.5, (-40, 40), (-2, 2))],
    "box-room": [(0, -5.0, (-4, 3), (-1.7, 2.5)), (0, 7.0, (-4, 3), (-1.7, 2.5)), (1, -4.0, (-5, 7), (-1.7, 2.5)),
                 (1, 3.0, (-5, 7), (-1.7, 2.5)), (2, -1.7, (-5, 7), (-4, 3)), (2, 2.5, (-5, 7), (-4, 3))],
}
POSE = IR.exp_se3(np.array([0.25, 0.08, 0.02, 0.004, -0.003, 0.02]))


def _fov():
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=HH, w=WW, vfov_deg=VFOV)
    return tuple(cfg["horizontal_field_of_view"]), tuple(cfg["kitti"]["vertical_field_of_view"])


def _raycast(rects, pose, seed, n=4 * HH * WW):
    """[3, N] fp32 points in the sensor frame of `pose`: the nearest rectangle hit by each of n seeded rays."""
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
    return torch.from_numpy((d[hit] * best[hit, None]).T.astype(np.float32))


def _scene_grids(name):
    hf, vf = _fov()
    out = []
    for pose, seed in ((np.eye(4), 1), (POSE, 2)):
        pts = _raycast(SCENES[name], pose, seed).reshape(1, 3, -1).contiguous().to(DEV)
        cnt = torch.tensor([pts.shape[2]], dtype=torch.int32, device=DEV)
        _, _, pg, ng = ops.project_normals(pts, cnt, HH, WW, hf, vf)
        out.append((pg, ng))
    return out, torch.from_numpy(np.ascontiguousarray(POSE[:3].astype(np.float32).reshape(1, 12))).to(DEV)


# ============================================================================================ the scaled operator
def test_scaled_operator_with_unit_factors_is_the_operator(cuda_lib):
    hf, vf = _fov()
    tg, sg, Ts = [], [], []
    for name in SCENES:
        ((tp, tn), (sp, sn)), T = _scene_grids(name)
        tg.append((tp, tn))
        sg.append((sp, sn))
        Ts.append(T)
    cat = lambda xs, i: torch.cat([x[i] for x in xs])
    args = (cat(sg, 0), cat(sg, 1), torch.cat(Ts), cat(tg, 0), cat(tg, 1), HH, WW, hf, vf)
    for flags in (ICP, ops.LOSS_PO2PO | ICP | ops.NORMAL_LINEAR, ops.LOSS_PO2PL):
        ones = torch.ones((len(Ts),), dtype=torch.float32, device=DEV)
        a = ops.icp_dense_information(*args, 0.6, flags)
        b = ops.icp_dense_information_scaled(*args, ones, 0.6, flags)
        for x, y, what in zip(a, b, ("losses", "grad_T", "info", "nn")):
            assert _bits_equal(x, y), f"flags {flags}: {what} differs with unit factors"


@pytest.mark.parametrize("name", list(SCENES))
def test_scaled_operator_is_D_H_D_in_metres(cuda_lib, name):
    hf, vf = _fov()
    ((tp, tn), (sp, sn)), T = _scene_grids(name)
    factors = [0.05, 0.3, 7.0]
    B = len(factors)
    rep = lambda x: x.expand(B, *x.shape[1:]).contiguous()
    args = (rep(sp), rep(sn), rep(T), rep(tp), rep(tn), HH, WW, hf, vf)
    f = torch.tensor(factors, dtype=torch.float32, device=DEV)
    base = ops.icp_dense_information(*args, 1.0, ICP)
    got = ops.icp_dense_information_scaled(*args, f, 1.0, ICP)
    for i, what in ((0, "losses"), (1, "grad_T"), (3, "NN ids")):
        assert _bits_equal(base[i], got[i]), f"{name}: {what} differ from the unscaled call"
    for b, fb in enumerate(factors):
        row, ref_row = got[2][b].cpu().numpy(), base[2][b].cpu().numpy()
        D = np.diag([1.0 / float(np.float32(fb))] * 3 + [1.0] * 3)
        want = D @ ref_row[:36].reshape(6, 6).astype(np.float64) @ D
        Hg = row[:36].reshape(6, 6).astype(np.float64)
        tol = 2 * U * np.abs(want) * (1 + 1e-6)
        assert np.all(np.abs(Hg - want) <= tol), f"{name} f={fb}: max |dH| / tol = {(np.abs(Hg - want) / tol).max()}"
        assert row[78] == ref_row[78] and row[79] == ref_row[79]
        ev, V = row[36:42].astype(np.float64), row[42:78].reshape(6, 6).astype(np.float64)
        ref_ev, ref_V = np.linalg.eigh(Hg)
        lmax = np.abs(ref_ev).max()
        assert np.all(np.diff(ev) >= 0)
        assert np.abs(ev - ref_ev).max() <= 1e-5 * lmax, (name, fb, ev, ref_ev)
        for k in range(6):
            v = V[k]
            assert abs(np.linalg.norm(v) - 1.0) < 1e-5 and v[int(np.argmax(np.abs(v)))] > 0
            gap = min(abs(ref_ev[k] - ref_ev[j]) for j in range(6) if j != k)
            if gap > 1e-3 * lmax:
                assert abs(v @ ref_V[:, k]) >= 1.0 - 1e-4, (name, fb, k, v, ref_V[:, k])
        if fb != 1.0:
            assert not np.allclose(Hg[:3, :3], ref_row[:36].reshape(6, 6)[:3, :3])


# ============================================================================================ recipe streams
from test_gpu_odometry_streams_pre import _history, _setup as _pre_setup  # noqa: E402

W_PRE_CASE = (16, 180, 512, 360)             # H, W, w_raw, w_pre


def _run_pre(st, ticks, resets, normalized, info, graph=False):
    """Every tick through one recipe workspace (with info: the information one) -> [(T, valid, losses, factor, info)]."""
    S = st.desc.max_batch
    n_stride = ticks[0][0].shape[2]
    pts = torch.zeros((S, 3, n_stride), dtype=torch.float32, device=DEV)
    counts = torch.zeros((S,), dtype=torch.int32, device=DEV)
    active = torch.zeros((S,), dtype=torch.int32, device=DEV)
    T = torch.full((S, 16), SENTINEL, dtype=torch.float32, device=DEV)
    valid = torch.full((S,), 7, dtype=torch.int32, device=DEV)
    losses = torch.full((S, ops.LOSS_ROW), SENTINEL, dtype=torch.float32, device=DEV)
    factor = torch.full((S,), SENTINEL, dtype=torch.float32, device=DEV) if normalized else None
    guarded = torch.full((S + 2, ops.INFO_ROW), SENTINEL, dtype=torch.float32, device=DEV)
    rows = guarded[1:S + 1]
    mask = torch.zeros((S,), dtype=torch.int32, device=DEV)

    def push():
        if info:
            st.push(pts, counts, active, T, valid, losses, rows, factor)
        else:
            st.push(pts, counts, active, T, valid, losses, factor)
    g = None
    if graph:
        push()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            push()
    out = []
    for k, (p, c, a) in enumerate(ticks):
        if k in resets:
            mask.zero_()
            mask[resets[k]] = 1
            st.reset(mask)
        pts.copy_(p)
        counts.copy_(c)
        active.copy_(a)
        if g is not None:
            g.replay()
        else:
            push()
        torch.cuda.synchronize()
        out.append((T.cpu().clone(), valid.cpu().clone(), losses.cpu().clone(),
                    None if factor is None else factor.cpu().clone(), rows.cpu().clone() if info else None))
        assert bool((guarded[0] == SENTINEL).all()) and bool((guarded[S + 1] == SENTINEL).all())
    return out


def _pre_grids(cfg, frame, count, ft=None):
    """The recipe's H x W grids of one frame: projection + normals at H x w_pre, divided by ft when given, then the
    H x W projection (what the workspace's ICP reads)."""
    ds = cfg["kitti"]
    h, w, w_pre = ds["vertical_cells"], ds["horizontal_cells"], ds["horizontal_cells_preprocessing"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    _, _, pg, ng = ops.project_normals(frame[None].to(DEV), count.view(1).to(DEV), h, w_pre, hf, vf,
                                       ds["neighborhood_side_length"], cfg["epsilon_range"],
                                       cfg["min_num_points_in_neighborhood_to_determine_point_class"])
    if ft is not None:
        pg = torch.cat((pg[..., :3] / ft, pg[..., 3:]), dim=-1)
    _, _, g_pts, g_nrm = ops.project_grids(pg.contiguous(), ng, h, w_pre, w, hf, vf, index_map=False)
    return g_pts, g_nrm


def _operator_row(cfg, src, tgt, T12, ft, flags=ICP):
    """The B = 1 information operator on the pair's grids, scaled with ft (a [1] device tensor) when given."""
    ds = cfg["kitti"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    args = (src[0], src[1], T12, tgt[0], tgt[1], ds["vertical_cells"], ds["horizontal_cells"], hf, vf)
    if ft is None:
        return ops.icp_dense_information(*args, float(cfg["lambda_po2pl"]), flags)
    return ops.icp_dense_information_scaled(*args, ft, float(cfg["lambda_po2pl"]), flags)


def _model_T12(T_served, f, want_losses, op):
    """T's 3x4 in the model's units.  Plain (f None): the served rows.  Normalised: the served translation is
    fl(t * f); the t with that product whose operator call reproduces the served loss row -> (T12, operator output)."""
    t16 = T_served.reshape(16).numpy().astype(np.float32)
    if f is None:
        T12 = torch.from_numpy(t16[:12].copy()).view(1, 12).to(DEV)
        return T12, op(T12)
    f32 = np.float32(f)
    cands = []
    for e in (3, 7, 11):
        c0 = np.float32(t16[e] / f32)
        near = [c0]
        for _ in range(2):
            near = [np.nextafter(near[0], np.float32(-np.inf)), *near, np.nextafter(near[-1], np.float32(np.inf))]
        cands.append([c for c in near if np.float32(c * f32) == t16[e]])
    for tx in cands[0]:
        for ty in cands[1]:
            for tz in cands[2]:
                t = t16[:12].copy()
                t[3], t[7], t[11] = tx, ty, tz
                T12 = torch.from_numpy(t).view(1, 12).to(DEV)
                res = op(T12)
                if _bits_equal(res[0][0, :6].cpu(), want_losses[:6]):
                    return T12, res
    raise AssertionError("no model-unit translation reproduces the served T and loss row")


@pytest.mark.parametrize("normalized", [False, True], ids=["plain", "normalized"])
def test_pre_info_streams_are_push_pre_bytes_and_the_operators_rows(cuda_lib, normalized):
    h, w, w_raw, w_pre = W_PRE_CASE
    S = 3
    cfg, blob, n_stride, ticks, act, resets = _pre_setup(h, w, w_raw, w_pre, normalized, S)
    d = H.desc(cfg, n_stride, S, w_pre)
    rp = capi.residual_params(cfg, ICP | _norm(normalized))
    ref = _run_pre(capi.PreStreamsWorkspace(d, blob, rp), ticks, resets, normalized, False)
    out = _run_pre(capi.PreInformationStreamsWorkspace(d, blob, rp), ticks, resets, normalized, True)
    for k, (r, o) in enumerate(zip(ref, out)):
        for i, what in enumerate(("T", "valid", "losses", "factor")):
            assert r[i] is None or _bits_equal(r[i], o[i]), f"tick {k}: {what} differs from _push_pre"
    pairs = _history(ticks, act, resets)
    checked = 0
    for k, (T, valid, losses, factor, rows) in enumerate(out):
        for s in range(S):
            if not int(valid[s]):
                assert float(rows[s].abs().max()) == 0.0, f"tick {k} stream {s}: an invalid row is not zero"
                continue
            (p1, c1), (p2, c2) = pairs[(k, s)]
            f = float(factor[s]) if normalized else None
            if normalized and not math.isfinite(f):       # an empty frame: no pixel, no pair (M = 0)
                assert float(rows[s][78]) == 0.0
                continue
            ft = torch.tensor([f], dtype=torch.float32, device=DEV) if normalized else None
            tgt, src = _pre_grids(cfg, p1, c1, ft), _pre_grids(cfg, p2, c2, ft)
            T12, res = _model_T12(T[s], f, losses[s], lambda T12: _operator_row(cfg, src, tgt, T12, ft))
            assert _bits_equal(losses[s], res[0][0].cpu()), f"tick {k} stream {s}: losses differ from the operator"
            assert _bits_equal(rows[s], res[2][0].cpu()), f"tick {k} stream {s}: the row differs from the operator"
            checked += int(rows[s][78] > 0)
    assert checked >= 6


def test_pre_info_graph_replay_matches_eager(cuda_lib):
    h, w, w_raw, w_pre = W_PRE_CASE
    cfg, blob, n_stride, ticks, act, resets = _pre_setup(h, w, w_raw, w_pre, True, 3, seed=5)
    d = H.desc(cfg, n_stride, 3, w_pre)
    rp = capi.residual_params(cfg, ICP | ops.TRAIN_NORMALIZATION_SCALING)
    eager = _run_pre(capi.PreInformationStreamsWorkspace(d, blob, rp), ticks, resets, True, True)
    graphed = _run_pre(capi.PreInformationStreamsWorkspace(d, blob, rp), ticks, resets, True, True, graph=True)
    for k, (e, g) in enumerate(zip(eager, graphed)):
        for a, b in zip(e, g):
            assert _bits_equal(a, b), f"tick {k}: the replay differs from the eager call"


def test_corridor_served_to_a_normalised_model_leaves_translation_along_it_free(cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=HH, w=WW, vfov_deg=VFOV)
    base = H.config(HH, WW)
    base["kitti"] = cfg["kitti"]
    base["horizontal_field_of_view"] = cfg["horizontal_field_of_view"]
    base["kitti"]["horizontal_cells_preprocessing"] = 2 * WW
    base["normalization_scaling"] = True
    frames = [_raycast(SCENES["corridor"], np.eye(4), 1), _raycast(SCENES["corridor"], POSE, 2)]
    n_stride = max(f.shape[1] for f in frames)
    blob = H.blob(H.model(base, 3, near_identity=True), base)
    st = capi.PreInformationStreamsWorkspace(H.desc(base, n_stride, 1, 2 * WW), blob,
                                             capi.residual_params(base, ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING))
    ticks = []
    for f in frames:
        p = torch.zeros((1, 3, n_stride), dtype=torch.float32)
        p[0, :, :f.shape[1]] = f
        ticks.append((p, torch.tensor([f.shape[1]], dtype=torch.int32), torch.ones((1,), dtype=torch.int32)))
    out = _run_pre(st, ticks, {}, True, True)
    T, valid, losses, factor, rows = out[1]
    assert int(valid[0]) == 1 and float(factor[0]) > 0
    row = rows[0].numpy().astype(np.float64)
    ev, V = row[36:42], row[42:78].reshape(6, 6)
    ratio = ev[0] / ev[5]
    angle = math.degrees(math.acos(min(1.0, abs(V[0, 0]))))
    print(f"\ncorridor, normalised model (factor {float(factor[0]):.3g}): lambda_min / lambda_max = {ratio:.3g}, "
          f"angle to x-translation {angle:.3g} deg")
    assert ratio < 2e-3 and angle < 5.0, (ev, V[0])


# ============================================================================================ adapting streams
from test_gpu_odometry_streams_adapt import _Io, _pattern, _ticks  # noqa: E402


def _adapt_cfg(h, w, w_pre, normalized):
    cfg = H.config(h, w)
    cfg["kitti"]["horizontal_cells_preprocessing"] = w_pre
    cfg["normalization_scaling"] = normalized
    return cfg


def _train_params(cfg, normalized):
    return capi.train_params(cfg, LR, loss_flags=ICP | _norm(normalized))


def _run_adapt(ws, ticks, updates, resets, info):
    S = ws.desc.max_batch
    io = _Io(S, ticks[0][0].shape[2])
    rows = torch.full((S, ops.INFO_ROW), SENTINEL, dtype=torch.float32, device=DEV)
    out = []
    for k, (p, c, a) in enumerate(ticks):
        if k in resets:
            io.mask.zero_()
            io.mask[resets[k]] = 1
            ws.reset(io.mask)
        io.load(p, c, a)
        if info:
            ws.push(*io.args(), rows, update=updates[k])
        else:
            ws.push(*io.args(), update=updates[k])
        T, valid, losses = io.out()
        out.append((T, valid, losses, rows.cpu().clone() if info else None, H.state(ws)))
    return out


@pytest.mark.parametrize("w_pre,normalized", [(0, False), (360, False), (360, True)],
                         ids=["w_pre0", "pre360", "pre360-normalized"])
def test_adapt_info_is_push_adapt_bytes_and_the_operators_rows(cuda_lib, w_pre, normalized):
    h, w, w_raw, S = 16, 180, 512, 3
    cfg = _adapt_cfg(h, w, w_pre, normalized)
    pool = H.frames(h, w_raw, 8)
    n_stride = max(f.shape[1] for f in pool)
    act, empty, resets = _pattern(S)
    ticks = _ticks(pool, S, n_stride, act, empty)
    blob = H.blob(H.model(cfg, 5, near_identity=True), cfg)
    d = H.desc(cfg, n_stride, S, w_pre)
    updates = [True, True, False, True, True, False, True]
    ref = _run_adapt(capi.AdaptiveStreamsWorkspace(d, blob, _train_params(cfg, normalized)), ticks, updates, resets,
                     False)
    out = _run_adapt(capi.AdaptiveInformationStreamsWorkspace(d, blob, _train_params(cfg, normalized)), ticks, updates,
                     resets, True)
    for k, (r, o) in enumerate(zip(ref, out)):
        assert _bits_equal(r[1], o[1]), f"tick {k}: valid differs from _push_adapt"
        assert _bits_equal(r[2], o[2]), f"tick {k}: losses differ from _push_adapt"
        for s in range(S):
            if int(r[1][s]):
                assert _bits_equal(r[0][s], o[0][s]), f"tick {k} stream {s}: T differs from _push_adapt"
        assert H.same_state(r[4], o[4]), f"tick {k}: the training state differs from _push_adapt's"
    assert int(out[-1][4][3][0]) >= 3
    # each valid row: the B = 1 operator on the tick's grids at the served T (the weights before the tick's update)
    ds = cfg["kitti"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    pairs = _history(ticks, act, resets)
    checked = 0
    for k, (T, valid, losses, rows, _) in enumerate(out):
        for s in range(S):
            if not int(valid[s]):
                assert float(rows[s].abs().max()) == 0.0, f"tick {k} stream {s}: an invalid row is not zero"
                continue
            (p1, c1), (p2, c2) = pairs[(k, s)]
            f = float(losses[s][6]) if normalized else None
            if normalized and not math.isfinite(f):       # an empty frame: no pixel, no pair (M = 0)
                assert float(rows[s][78]) == 0.0
                continue
            ft = torch.tensor([f], dtype=torch.float32, device=DEV) if normalized else None
            if w_pre:
                tgt, src = _pre_grids(cfg, p1, c1, ft), _pre_grids(cfg, p2, c2, ft)
            else:
                grid = lambda p, c: ops.project_normals(p[None].to(DEV), c.view(1).to(DEV), h, w, hf, vf,
                                                        ds["neighborhood_side_length"], cfg["epsilon_range"],
                                                        cfg["min_num_points_in_neighborhood_to_determine_point_class"])[2:]
                tgt, src = grid(p1, c1), grid(p2, c2)
            T12, res = _model_T12(T[s], f, losses[s], lambda T12: _operator_row(cfg, src, tgt, T12, ft))
            assert _bits_equal(losses[s][:6], res[0][0, :6].cpu()), f"tick {k} stream {s}: losses vs the operator"
            assert _bits_equal(rows[s], res[2][0].cpu()), f"tick {k} stream {s}: the row differs from the operator"
            checked += int(rows[s][78] > 0)
    assert checked >= 6


from test_gpu_odometry_streams_adapt_group import (_group_tick, _setup as _group_setup, _single,  # noqa: E402
                                                   _single_tick, _status_ok, _tick_inputs)


def _info_group(cfg, blob, n_stride, world, S=2):
    ws = [capi.AdaptiveInformationStreamsWorkspace(H.desc(cfg, n_stride, S), blob, capi.train_params(cfg, LR))
          for _ in range(world)]
    return capi.AdaptingStreamsGroup(ws), [torch.cuda.Stream() for _ in range(world)]


def _plain_group(cfg, blob, n_stride, world, S=2):
    ws = [capi.AdaptiveStreamsGroupWorkspace(H.desc(cfg, n_stride, S), blob, capi.train_params(cfg, LR))
          for _ in range(world)]
    return capi.AdaptingStreamsGroup(ws), [torch.cuda.Stream() for _ in range(world)]


def _warm(cfg, blob, pool, n_stride, S):
    """One update tick of _push_adapt and of _push_adapt_info at the ranks' shape loads every kernel of a group tick
    but the collectives (which _adapt_info_init loads): the ranks here share one device and one host thread, and under
    lazy module loading a kernel's first launch waits for the device's running kernels, a rank spinning in the count
    exchange among them."""
    inp = _tick_inputs(pool, S, n_stride, 0, [1] * S)
    _single_tick(_single(cfg, blob, n_stride, S), *inp, True)
    ws = capi.AdaptiveInformationStreamsWorkspace(H.desc(cfg, n_stride, S), blob, capi.train_params(cfg, LR))
    io = _Io(S, n_stride)
    io.load(*inp)
    ws.push(*io.args(), torch.empty((S, ops.INFO_ROW), dtype=torch.float32, device=DEV), update=True)
    torch.cuda.synchronize()


def test_adapt_group_info_at_world_1_is_push_adapt_info(cuda_lib):
    cfg, blob, pool, n_stride = _group_setup()
    S = 3
    _warm(cfg, blob, pool, n_stride, S)
    g, streams = _info_group(cfg, blob, n_stride, 1, S)
    one = capi.AdaptiveInformationStreamsWorkspace(H.desc(cfg, n_stride, S), blob, capi.train_params(cfg, LR))
    io = _Io(S, n_stride)
    rows = torch.empty((S, ops.INFO_ROW), dtype=torch.float32, device=DEV)
    updates = [True, False, True, True, False, True]
    acts = [[1, 1, 0], [1, 1, 1], [1, 0, 1], [0, 0, 0], [1, 1, 1], [1, 1, 1]]
    for k, (u, a) in enumerate(zip(updates, acts)):
        inp = _tick_inputs(pool, S, n_stride, k, a)
        (got,) = _group_tick(g, streams, [inp], [u])
        io.load(*inp)
        one.push(*io.args(), rows, update=u)
        want = io.out() + (rows.cpu(),)
        assert _bits_equal(got[1], want[1]), f"tick {k}: valid"
        for s in range(S):
            if int(want[1][s]):
                assert _bits_equal(got[0][s], want[0][s]), f"tick {k}, stream {s}: T"
        assert _bits_equal(got[2], want[2]) and _bits_equal(got[3], want[3]), f"tick {k}: losses or info"
        assert H.same_state(H.state(g.workspaces[0]), H.state(one)), f"tick {k}: the training state"
    assert _status_ok(g)


@pytest.mark.parametrize("world", [2, 4])
def test_adapt_group_info_ranks_are_push_adapt_group_bytes(cuda_lib, world):
    cfg, blob, pool, n_stride = _group_setup()
    S = 2
    _warm(cfg, blob, pool, n_stride, S)
    gi, si = _info_group(cfg, blob, n_stride, world, S)
    gp, sp = _plain_group(cfg, blob, n_stride, world, S)
    rng = np.random.default_rng(world)
    for k in range(5):
        acts = [[int(x) for x in rng.integers(0, 2, S)] if k else [1] * S for _ in range(world)]
        inputs = [_tick_inputs(pool, S, n_stride, k, acts[r], offset=r * S) for r in range(world)]
        got = _group_tick(gi, si, inputs, [True] * world)
        want = _group_tick(gp, sp, inputs, [True] * world)
        for r in range(world):
            assert _bits_equal(got[r][1], want[r][1]), f"tick {k} rank {r}: valid"
            for s in range(S):
                if int(want[r][1][s]):
                    assert _bits_equal(got[r][0][s], want[r][0][s]), f"tick {k} rank {r} stream {s}: T"
                else:
                    assert float(got[r][3][s].abs().max()) == 0.0
            assert _bits_equal(got[r][2], want[r][2]), f"tick {k} rank {r}: losses"
            assert H.same_state(H.state(gi.workspaces[r]), H.state(gp.workspaces[r])), f"tick {k} rank {r}: state"
    assert _status_ok(gi) and _status_ok(gp)


# ============================================================================================ Python and the example
def test_python_classes_return_the_same_bits_with_the_information(cuda_lib):
    from delora_b200.deploy.stream import AdaptiveOdometryStreams, PreprocessedOdometryStreams
    h, w, w_raw, w_pre = W_PRE_CASE
    cfg = _adapt_cfg(h, w, w_pre, True)
    model = H.model(cfg, 9, near_identity=True).eval()
    pool = H.frames(h, w_raw, 4)
    n_max = max(s.shape[1] for s in pool) + 8
    a = PreprocessedOdometryStreams(model, cfg, "kitti", 2, n_max)
    b = PreprocessedOdometryStreams(model, cfg, "kitti", 2, n_max, information=True)
    c = AdaptiveOdometryStreams(model, cfg, "kitti", 2, n_max, LR, preprocessing_normals=True)
    e = AdaptiveOdometryStreams(model, cfg, "kitti", 2, n_max, LR, preprocessing_normals=True, information=True)
    seen = 0
    for k in range(3):
        scans = [pool[k].cpu(), pool[(k + 1) % 4].cpu()]
        for x, y in zip(a.push(scans), b.push(scans)):
            assert (x is None) == (y is None)
            if x is not None:
                assert len(y) == 4 and np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
                assert np.float32(x[2]).view(np.int32) == np.float32(y[3]).view(np.int32)
                assert y[2].shape == (ops.INFO_ROW,) and np.all(np.diff(y[2][36:42]) >= 0)
                seen += 1
        for x, y in zip(c.push(scans), e.push(scans)):
            assert (x is None) == (y is None)
            if x is not None:
                assert len(y) == 3 and np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
                assert y[2].shape == (ops.INFO_ROW,) and np.all(np.diff(y[2][36:42]) >= 0)
                seen += 1
    assert seen >= 8
    for k, v in c.state_dict().items():
        assert np.array_equal(np.asarray(v), np.asarray(e.state_dict()[k])), k


def test_example_information_columns_beside_the_recipe_and_adapt_modes(cuda_lib, tmp_path):
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = _adapt_cfg(16, 720, 1024, True)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    model = H.model(cfg, 6, near_identity=True).eval()
    dlw = os.path.join(tmp_path, "m.dlw")
    desc = export.desc_from_config(cfg, "kitti", 4096, 1, preprocessing_normals=True)
    export.write_dlw(dlw, desc, export.pack_state_dict(model.state_dict(), cfg), export.model_flags_from_config(cfg))
    dirs = []
    for s, n in enumerate((4, 3)):
        dd = os.path.join(tmp_path, f"stream{s}")
        os.makedirs(dd)
        dirs.append(dd)
        for i in range(n):
            synthetic.kitti_bin_scan(10 * s + i, vfov_deg=vfov).tofile(os.path.join(dd, f"{i:06d}.bin"))
    exe = H.build_example("odometry_streams", tmp_path, link=True)

    def run(args):
        r = subprocess.run([exe] + args + [dlw] + dirs, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        return [ln.split() for ln in r.stdout.strip().splitlines()]

    adapt = lambda name: ["--adapt", "1e-4", "--adapt-out", os.path.join(tmp_path, name)]
    for base, extra in ((["--preprocessing"], ["--information"]), (adapt("a.dlw"), ["--information"]),
                        (adapt("c.dlw") + ["--gpus", "1"], ["--information"])):
        plain = run(base)
        with_info = run([x.replace(".dlw", "-info.dlw") for x in base] + extra)
        assert len(plain) == len(with_info) == 5
        for p, q in zip(plain, with_info):
            assert q[:len(p)] == p and len(q) == len(p) + 8, (p, q)
            assert abs(sum(float(x) ** 2 for x in q[len(p) + 1:len(p) + 7]) - 1) < 1e-4
    for name in ("a", "c"):
        assert open(os.path.join(tmp_path, f"{name}.dlw"), "rb").read() == \
            open(os.path.join(tmp_path, f"{name}-info.dlw"), "rb").read()
