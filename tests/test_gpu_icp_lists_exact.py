"""The list ICP operator behind ICPLosses (pack_lists -> delora_grid_build -> delora_icp_fwd_bwd -> delora_icp_point_grads)
on arbitrary point lists, against exact references, on the H100.

Unlike the lists delora_lists_from_images makes (one point per cell, each in the cell the projection gives it), these
lists put tens of points in a cell, targets outside the vertical and the horizontal field of view, exact ties and
duplicates in shuffled order, ragged and empty lists in one batch.

  - The cell sort (delora_grid_build), exactly: every target's cell is computed on the host from the projection's
    float32 coordinates (tests/projection_reference.py) and cell_of's rule (rint, rows clamped, an out-of-field azimuth
    in the border column nearer around the circle: tests/lists_reference.py), on points kept 1e-3 px away from every
    rounding boundary and from the gap's midpoint (the list path's CUDA arithmetic and the projection's may round those
    differently).  cell_start is the exclusive prefix of that histogram; the rows of each cell are the expected
    (x, y, z, bits(list index)) and (normal, has-normal), as a multiset (atomics order a cell); the slots from n on are
    untouched; the cursor starts with garbage and the lists carry garbage beyond n.
  - Every nearest neighbour (nn_index of delora_icp_fwd_bwd, pointwise) equals the exact reference
    (tests/nn_reference.py: lowest list index on exact ties), once with T = None on sources transformed on the host
    (icp_reference.apply_rigid, the kernel's rounding) and once with T in the kernel.  Families: dense clouds on coarse
    grids, targets above and below the vertical field of view, exact ties across cells and across the seam, duplicate
    points, a ragged B = 3 batch with an empty target list, transforms that move sources out of the field of view, and
    the decoy scenes of tests/lists_reference.py on partial horizontal fields of view at W = 180, 720 and 2048.
  - Losses and per-point gradients of the ICPLosses module (plain, with the linear normal loss, and po2po_alone)
    against tests/icp_reference.py in float64, with the bars of test_gpu_icp_losses.py.
  - Repeatability: a second run, and a run on a permuted target list, give the same neighbours and the same loss bits.

Before the nearer-border binning, the partial-field family failed on an H100 (700 W) on every case with a one-sided gap
wider than half a pitch and only there: 9 of the 18 sources (all those at the sharp seam edge) took the decoy at each of
W = 180, 720 and 2048, with T = None and with T alike; the controls (0.3 pitches, [-pi/4, pi/4], +-179.9 deg) passed.
The losses of the decoy scene missed their bars in all three modes, and the cell sort differed from the rule on the
three fields with a one-sided gap.
"""
import itertools
import math

import numpy as np
import pytest
import torch

import icp_reference as R
import lists_reference as LR
import nn_reference as NR
import projection_reference as PR

pytestmark = pytest.mark.gpu

DEV = "cuda"
VF15 = (math.radians(-15.0), math.radians(15.0))
KITTI_VF = (math.radians(-24.5), math.radians(2.0))
HF_SYN = (math.radians(-179.9), math.radians(179.9))
HF_FULL = (-math.pi, math.pi)
LOSS_TOL = 1e-6         # relative to the float64 loss (test_gpu_icp_losses.py)
POINT_TOL = 1e-6        # per-point gradients, relative to the tensor's max-abs
UPSTREAM = (0.7, 1.3, 2.1)
SENTINEL = np.int32(0x7FA11A11)    # a NaN payload no kernel writes


def one_sided(k, w, side):
    g = LR.gap_for(k, w)
    return (-math.pi, math.pi - g) if side == "left" else (-math.pi + g, math.pi)


def _xyz(r, az, el):
    return np.stack((r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)), axis=-1)


def _garbage(gen, shape):
    pool = np.array([np.nan, np.inf, -np.inf, 1e30, -3.0, 0.0, 7.5], np.float32)
    return pool[gen.integers(0, len(pool), shape)]


def _normals(gen, n, zero_frac=0.25):
    m = gen.standard_normal((n, 3))
    m /= np.linalg.norm(m, axis=1, keepdims=True)
    m = m.astype(np.float32)
    zero = gen.random(n) < zero_frac
    m[zero] = 0.0
    m[zero & (gen.random(n) < 0.3), 0] = -0.0          # (-0, 0, 0) has no normal either
    return m


def random_points(gen, n, hfov, vfov, pad=0.05, r_lo=0.5, r_hi=90.0):
    az = gen.uniform(hfov[0] - pad, hfov[1] + pad, n)
    el = gen.uniform(vfov[0] - pad, vfov[1] + pad, n)
    r = np.exp(gen.uniform(math.log(r_lo), math.log(r_hi), n))
    return _xyz(r, az, el).astype(np.float32)


# ---- running the operator ------------------------------------------------------------------------------------------
def run_nn(h, w, hfov, vfov, tgts, srcs, T=None, seed=0):
    """B pairs of lists ([N, 3] fp32 each; garbage beyond every n) -> list of nn_index arrays (int64)."""
    from delora_b200 import ops
    gen = np.random.default_rng(seed)
    b = len(tgts)
    nt, ns = [len(t) for t in tgts], [len(s) for s in srcs]
    ts, ss = max(nt + [1]) + 3, max(ns + [1]) + 5
    tp, sp = _garbage(gen, (b, 3, ts)), _garbage(gen, (b, 3, ss))
    for k in range(b):
        tp[k, :, :nt[k]] = np.asarray(tgts[k], np.float32).T
        sp[k, :, :ns[k]] = np.asarray(srcs[k], np.float32).T
    n_t = torch.tensor(nt, dtype=torch.int32, device=DEV)
    n_s = torch.tensor(ns, dtype=torch.int32, device=DEV)
    s4, sn4 = ops.pack_lists(torch.from_numpy(sp).to(DEV), None, n_s)
    t4, tn4, cs = ops.grid_build(torch.from_numpy(tp).to(DEV), None, n_t, h, w, hfov, vfov)
    tt = None if T is None else torch.from_numpy(np.asarray(T, np.float32).reshape(b, 12)).to(DEV)
    _, _, nn, _, _ = ops.icp_fwd_bwd(s4, sn4, n_s, tt, t4, tn4, cs, h, w, hfov, vfov, pointwise=True)
    nn = nn.cpu().numpy().astype(np.int64)
    return [nn[k, :ns[k]] for k in range(b)]


def check_nn(label, h, w, hfov, vfov, tgts, srcs, T=None):
    """Both runs (T = None on host-transformed sources, and T in the kernel; T = identity when not given) against the
    exact reference.  -> (wrong with T = None, wrong with T) summed over the pairs; asserts nothing."""
    b = len(tgts)
    T = np.tile(np.eye(4)[:3].reshape(1, 12), (b, 1)) if T is None else np.asarray(T, np.float64).reshape(b, 12)
    moved, want = [], []
    for k in range(b):
        s = np.asarray(srcs[k], np.float32).reshape(-1, 3)
        s_t, _ = R.apply_rigid(T[k].astype(np.float32), s, np.zeros_like(s)) if len(s) else (s, None)
        moved.append(s_t)
        ref = NR.nearest(np.asarray(tgts[k], np.float32).reshape(-1, 3), np.arange(len(tgts[k])), s_t)
        assert len(ref.unsafe) == 0, f"{label} pair {k}: separations below 2^-45 at sources {ref.unsafe[:8]}"
        want.append(ref.nn)
    wrong = []
    for tt, ss in ((None, moved), (T, srcs)):
        got = run_nn(h, w, hfov, vfov, tgts, ss, tt)
        bad = 0
        for k in range(b):
            miss = np.nonzero(got[k] != want[k])[0]
            bad += len(miss)
            if len(miss) and not wrong:
                i = miss[0]
                print(f"  {label} ({'T' if tt is not None else 'T = None'}) pair {k} source {i} "
                      f"{np.asarray(ss[k])[i].tolist()}: {got[k][i]} vs {want[k][i]}", flush=True)
        wrong.append(bad)
    return tuple(wrong)


def assert_nn(label, *args, **kw):
    wrong = check_nn(label, *args, **kw)
    assert wrong == (0, 0), f"{label}: nn_index differs from the exact NN at {wrong} sources (T = None, T)"


# ---- the cell sort -------------------------------------------------------------------------------------------------
SORT_CASES = [(4, 16, HF_FULL, VF15), (16, 180, one_sided(1.0, 180, "left"), VF15),
              (16, 180, one_sided(0.6, 180, "right"), VF15), (64, 720, (-math.pi / 4, math.pi / 4), KITTI_VF),
              (64, 2048, (-math.pi, 0.0), KITTI_VF), (64, 2048, HF_SYN, KITTI_VF)]
SORT_IDS = ["4x16-full", "16x180-gap1du", "16x180-gap0.6du-right", "64x720-quarter", "64x2048-half", "64x2048-syn"]


def sort_cloud(gen, h, w, hfov, vfov, n):
    """Directions over the whole sphere, in-field points, azimuths across the horizontal gap, a 300-point cluster in one
    cell and exact duplicates, kept
    1e-3 px away from every rounding boundary and from the gap's midpoint; then a few NaN points."""
    prg, g = PR.Grid(h, w, hfov, vfov), LR.Grid(h, w, hfov, vfov)
    sph = _xyz(np.exp(gen.uniform(math.log(0.3), math.log(120.0), n // 2)), gen.uniform(-math.pi, math.pi, n // 2),
               np.arcsin(gen.uniform(-1, 1, n // 2)))
    inside = random_points(gen, n // 2, hfov, vfov)
    gap = hfov[1] + gen.uniform(0.02, 0.98, 300) * (2 * math.pi - (hfov[1] - hfov[0]))
    gap = _xyz(np.exp(gen.uniform(0.0, 4.0, 300)), gap, gen.uniform(*vfov, 300))
    c_az, c_el = gen.uniform(*hfov), gen.uniform(*vfov)
    clus = _xyz(np.exp(gen.uniform(0.0, 4.0, 300)), np.full(300, c_az), np.full(300, c_el))
    pts = np.concatenate((sph, inside, gap, clus)).astype(np.float32)
    pts = np.concatenate((pts, pts[gen.integers(0, len(pts), n // 10)]))
    u64, v64, du, dv = PR.float64_coords(prg, pts[:, 0], pts[:, 1], pts[:, 2])
    past = np.mod(u64 - (w - 1), 2 * math.pi / g.du)
    keep = (du > 1e-3) & (dv > 1e-3) & (np.abs(past - g.gap_px / 2) > 1e-3)
    pts = pts[keep]
    nan = random_points(gen, 5, hfov, vfov)
    nan[:, 0] = np.nan                                    # cell 0 in any arithmetic
    pts = np.concatenate((pts, nan))
    return pts[gen.permutation(len(pts))]


def host_cells(h, w, hfov, vfov, pts):
    prg, g = PR.Grid(h, w, hfov, vfov), LR.Grid(h, w, hfov, vfov)
    u, v, _ = PR.coords(prg, pts[:, 0], pts[:, 1], pts[:, 2])
    return LR.rows(g, v) * w + LR.columns(g, u, "nearer")


@pytest.mark.parametrize("case", SORT_CASES, ids=SORT_IDS)
def test_cell_sort_exact(case, cuda_lib):
    from delora_b200 import _lib, ops
    h, w, hfov, vfov = case
    hw = h * w
    gen = np.random.default_rng(h * 7 + w)
    clouds = [sort_cloud(gen, h, w, hfov, vfov, 6000) for _ in range(2)]
    n_stride = len(clouds[0])
    lists = [clouds[0], clouds[0][:0], clouds[1][:min(len(clouds[1]), 1234)], clouds[1][:1]]   # n_stride, 0, ragged, 1
    b = len(lists)
    n = np.array([len(x) for x in lists], np.int32)
    pts = _garbage(gen, (b, 3, n_stride))
    nrm = _garbage(gen, (b, 3, n_stride))
    nrms = [_normals(gen, len(x)) for x in lists]
    for k, x in enumerate(lists):
        pts[k, :, :len(x)] = x.T
        nrm[k, :, :len(x)] = nrms[k].T
    L = _lib.lib()
    for trial in range(2):
        pts4 = torch.full((b, n_stride, 4), 0, dtype=torch.int32, device=DEV).fill_(int(SENTINEL)).view(torch.float32)
        nrm4 = pts4.clone()
        cs = torch.full((b, hw + 1), -12345, dtype=torch.int32, device=DEV)
        cursor = torch.randint(-2 ** 31, 2 ** 31 - 1, (b, hw), dtype=torch.int32,
                               generator=torch.Generator().manual_seed(trial)).to(DEV)
        scratch = torch.randint(-2 ** 31, 2 ** 31 - 1, (b * L.delora_scan_blocks(hw),), dtype=torch.int32,
                                generator=torch.Generator().manual_seed(10 + trial)).to(DEV)
        pt, nt_, nn_ = (torch.from_numpy(a).to(DEV) for a in (pts, nrm, n))
        _lib.check(L.delora_grid_build(pt.data_ptr(), nt_.data_ptr(), nn_.data_ptr(), b, n_stride, h, w,
                                       float(hfov[0]), float(hfov[1]), float(vfov[0]), float(vfov[1]), pts4.data_ptr(),
                                       nrm4.data_ptr(), cs.data_ptr(), cursor.data_ptr(), scratch.data_ptr(),
                                       ops._stream()), "delora_grid_build")
        torch.cuda.synchronize()
        p4 = pts4.view(torch.int32).cpu().numpy()
        q4 = nrm4.view(torch.int32).cpu().numpy()
        cs_h = cs.cpu().numpy()
        for k in range(b):
            nk = int(n[k])
            label = f"{SORT_IDS[SORT_CASES.index(case)]} trial {trial} pair {k} (n = {nk})"
            cell = host_cells(h, w, hfov, vfov, lists[k])
            hist = np.bincount(cell, minlength=hw)
            assert np.array_equal(cs_h[k], np.concatenate(([0], np.cumsum(hist)))), f"{label}: cell_start"
            idx = p4[k, :nk, 3].astype(np.int64)
            assert np.array_equal(np.sort(idx), np.arange(nk)), f"{label}: the list indices are not a permutation"
            at = np.repeat(np.arange(hw), hist)
            bad = np.nonzero(cell[idx] != at)[0]
            assert len(bad) == 0, (f"{label}: {len(bad)} rows in the wrong cell, first list index {idx[bad[0]]} "
                                   f"in cell {at[bad[0]]}, want {cell[idx[bad[0]]]}")
            want_p = pts[k, :, idx].view(np.int32)
            assert np.array_equal(p4[k, :nk, :3], want_p), f"{label}: point bits"
            q = nrm[k, :, idx]
            assert np.array_equal(q4[k, :nk, :3], q.view(np.int32)), f"{label}: normal bits"
            has = (q != 0).any(axis=1).astype(np.float32)
            assert np.array_equal(q4[k, :nk, 3], has.view(np.int32)), f"{label}: has-normal"
            assert (p4[k, nk:] == SENTINEL).all() and (q4[k, nk:] == SENTINEL).all(), f"{label}: slots beyond n"
            if k == 0:
                assert hist.max() >= 20, f"{label}: the densest cell holds only {hist.max()} points"
    g = LR.Grid(h, w, hfov, vfov)
    # the border columns and rows received out-of-field points
    u, v, _ = PR.coords(PR.Grid(h, w, hfov, vfov), clouds[0][:, 0], clouds[0][:, 1], clouds[0][:, 2])
    with np.errstate(invalid="ignore"):
        assert (v < -0.5).any() and (v > h - 0.5).any()
        if g.gap_px > 0.55:
            assert (u < -0.5).any() or (u > w - 0.5).any()


# ---- nearest neighbours ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,n_t", [(4, 16, 3000), (16, 180, 80000)], ids=["4x16", "16x180"])
def test_nn_dense_clouds_on_coarse_grids(h, w, n_t, cuda_lib):
    gen = np.random.default_rng(h + w)
    for hfov in (HF_SYN, one_sided(1.0, w, "left")):
        tgt = random_points(gen, n_t, hfov, VF15)
        clus = _xyz(np.exp(gen.uniform(0.0, 4.0, 400)), np.full(400, 0.3), np.full(400, 0.05)).astype(np.float32)
        tgt = np.concatenate((tgt, clus))
        near = tgt[gen.integers(0, len(tgt), 2000)] + gen.normal(0, 0.05, (2000, 3)).astype(np.float32)
        src = np.concatenate((near, random_points(gen, 1000, hfov, VF15))).astype(np.float32)
        assert_nn(f"{h}x{w} dense hfov {hfov}", h, w, hfov, VF15, [tgt], [src])


@pytest.mark.parametrize("h,w,vfov", [(16, 180, VF15), (64, 720, KITTI_VF)], ids=["16x180", "64x720"])
def test_nn_targets_above_and_below_the_vertical_field(h, w, vfov, cuda_lib):
    gen = np.random.default_rng(h * w)
    n = 20000
    el = np.concatenate((gen.uniform(-math.pi / 2, vfov[0], n // 2), gen.uniform(vfov[1], math.pi / 2, n // 2)))
    tgt = _xyz(np.exp(gen.uniform(0.0, 4.0, n)), gen.uniform(-math.pi, math.pi, n), el)
    poles = np.array([[1e-4, 0.0, 5.0], [0.0, -1e-4, -5.0], [-2e-3, 1e-3, 9.0], [3e-3, 3e-3, -2.0]])
    tgt = np.concatenate((tgt, poles, random_points(gen, 3000, HF_SYN, vfov))).astype(np.float32)
    src = np.concatenate((random_points(gen, 2000, HF_SYN, vfov),
                          _xyz(np.exp(gen.uniform(0.0, 4.0, 1000)), gen.uniform(-math.pi, math.pi, 1000),
                               gen.uniform(-math.pi / 2, math.pi / 2, 1000)))).astype(np.float32)
    assert_nn(f"{h}x{w} out of the vertical field", h, w, HF_SYN, vfov, [tgt], [src])


def tie_lists(g, gen, n_rand=50):
    """Dyadic sources s and 2 to 8 targets s + d, d signed permutations of one dyadic offset (exactly equidistant),
    0.3 to 4 pixels of angle apart; groups in the horizontal gap with one partner in column 0 and one in column W-1; a
    background at 40 m; the list shuffled.  -> targets, sources."""
    unit = 2.0 ** -12
    du, dv = g.du, g.dv
    tg, src = [random_points(gen, 3000, g.hfov, g.vfov, r_lo=39.0, r_hi=41.0)], []
    anchors = list(zip(gen.uniform(3, g.W - 4, n_rand), gen.uniform(1, g.H - 2, n_rand)))
    for u, v in anchors:
        r = gen.uniform(6.0, 12.0)
        s = np.round(_xyz(r, g.hfov[0] + u * du, g.vfov[0] + v * dv) / unit)
        mag = np.maximum(np.round(gen.uniform(0.3, 4.0, 3) * r * min(du, dv) / unit), 1.0)
        variants = sorted({tuple(np.array(sg) * np.array(q)) for q in itertools.permutations(mag)
                           for sg in itertools.product((-1, 1), repeat=3)})
        k = int(gen.integers(2, 9))
        pick = [np.array(variants[i]) for i in gen.choice(len(variants), min(k, len(variants)), replace=False)]
        tg.append(np.stack([(s + d) * unit for d in pick]))
        src.append(s * unit)
    # seam groups: s at the middle of the gap, d tangential, partners s + d and s + (-d_x, -d_y, d_z) (the same exact
    # norm) half a pitch past the border columns on either side
    az_m = g.hfov[1] + (2 * math.pi - (g.hfov[1] - g.hfov[0])) / 2
    for v in np.linspace(1, g.H - 2, 4):
        r = gen.uniform(6.0, 12.0)
        el = g.vfov[0] + v * dv
        s = np.round(_xyz(r, az_m, el) / unit)
        t = (g.gap_px / 2 + 0.45) * du * r * math.cos(el) / unit
        d = np.array([round(-math.sin(az_m) * t), round(math.cos(az_m) * t), round(gen.uniform(-0.3, 0.3) * t)])
        tg.append(np.stack([(s + d) * unit, (s + d * np.array([-1, -1, 1])) * unit]))
        src.append(s * unit)
    tgt = np.concatenate(tg).astype(np.float32)
    return tgt[gen.permutation(len(tgt))], np.array(src, np.float32)


@pytest.mark.parametrize("hfov_name", ["syn", "gap1du-left", "gap0.6du-right"])
def test_nn_exact_ties_across_cells_and_the_seam(hfov_name, cuda_lib):
    h, w = 16, 180
    hfov = {"syn": HF_SYN, "gap1du-left": one_sided(1.0, w, "left"),
            "gap0.6du-right": one_sided(0.6, w, "right")}[hfov_name]
    g = LR.Grid(h, w, hfov, VF15)
    gen = np.random.default_rng(len(hfov_name))
    tgt, src = tie_lists(g, gen)
    ref = NR.nearest(tgt, np.arange(len(tgt)), src)
    assert (ref.ties > 1).sum() >= len(src) // 2, f"only {(ref.ties > 1).sum()} of {len(src)} sources tie"
    # the tied partners of a source sit in different cells, and across the seam
    cell = host_cells(h, w, hfov, VF15, tgt)
    t64 = tgt.astype(np.float64)
    split = seam = 0
    for i, s in enumerate(src):
        if ref.ties[i] < 2:
            continue
        near = np.argsort(((t64 - s) ** 2).sum(1))[:12]
        d = [NR.exact_d2(s, tgt[j]) for j in near]
        members = near[np.array([x == min(d) for x in d])]
        cols = set((cell[members] % w).tolist())
        split += int(len(set(cell[members].tolist())) > 1)
        seam += int(0 in cols and w - 1 in cols)
    assert split > 10 and seam > 0, (split, seam)
    assert_nn(f"ties {hfov_name}", h, w, hfov, VF15, [tgt], [src])


def test_nn_duplicate_points(cuda_lib):
    h, w = 16, 180
    gen = np.random.default_rng(3)
    base = random_points(gen, 3000, HF_SYN, VF15)
    dup = np.repeat(base[gen.integers(0, 3000, 500)], gen.integers(1, 5, 500), axis=0)
    tgt = np.concatenate((base, dup))
    tgt = tgt[gen.permutation(len(tgt))]
    src = np.concatenate((tgt[gen.integers(0, len(tgt), 600)], dup[:300] + np.float32(1e-3),
                          random_points(gen, 600, HF_SYN, VF15)))
    src = np.concatenate((src, src[:100])).astype(np.float32)              # duplicate sources too
    ref = NR.nearest(tgt, np.arange(len(tgt)), src)
    assert (ref.ties > 1).sum() > 100
    assert_nn("duplicates", h, w, HF_SYN, VF15, [tgt], [src])


def test_nn_ragged_batch_with_an_empty_list(cuda_lib):
    """B = 3: (targets, sources) = (dense, 1500), (none, 40), (37, 700); every list carries garbage beyond its n."""
    h, w = 16, 180
    gen = np.random.default_rng(8)
    hfov = one_sided(1.0, w, "left")
    tgts = [random_points(gen, 20000, hfov, VF15), np.zeros((0, 3), np.float32), random_points(gen, 37, hfov, VF15)]
    srcs = [random_points(gen, n, hfov, VF15) for n in (1500, 40, 700)]
    T = np.stack([np.eye(4)[:3].reshape(12)] * 3)
    got = run_nn(h, w, hfov, VF15, tgts, srcs, T)
    assert (got[1] == -1).all(), "a source of an empty target list found a neighbour"
    assert_nn("ragged B = 3", h, w, hfov, VF15, tgts, srcs)


def _transform(tx, ty, tz, yaw, pitch, roll):
    from delora_b200 import synthetic
    return synthetic.transform_matrix(tx, ty, tz, yaw, pitch, roll)[:3].reshape(12)


def test_nn_transforms_that_move_sources_out_of_the_field(cuda_lib):
    from delora_b200 import synthetic
    h, w = 16, 180
    s1, s2, _, _ = synthetic.make_pair(31, w_raw=192, rings=h, vfov_deg=(-15.0, 15.0))
    tgt, p = s1.numpy().T.astype(np.float32), s2.numpy().T.astype(np.float32)
    p = p[np.random.default_rng(2).choice(len(p), 2500, replace=False)]
    ts = [_transform(0, 0, 0, math.radians(179.0), 0, 0), _transform(0, 0, 0, math.radians(181.0), 0, 0),
          _transform(0.5, 0, 0, 0, math.radians(40.0), 0), _transform(0, 0, 0, 0, 0, math.radians(90.0)),
          _transform(3.0, -2.0, 15.0, 0.3, 0.1, 0), _transform(0, 0, -20.0, math.radians(-170.0), math.radians(-35.0),
                                                                0.2)]
    for hfov in (HF_SYN, one_sided(2.0, w, "right"), (-math.pi / 4, math.pi / 4)):
        for k, T in enumerate(ts):
            assert_nn(f"transform {k} hfov {hfov}", h, w, hfov, VF15, [tgt], [p], T[None])


@pytest.mark.parametrize("name", LR.HFOV_NAMES)
def test_nn_partial_horizontal_fields_of_view(name, cuda_lib):
    """The decoy scenes at both seam edges, at W = 180, 720 and 2048 (tests/lists_reference.py)."""
    rows = []
    for h, w, vf in LR.DECOY_GRIDS:
        _, hf, sharp_edge = next(c for c in LR.hfov_cases(w) if c[0] == name)
        g = LR.Grid(h, w, hf, vf)
        sc = LR.decoy_scene(g)
        wrong = check_nn(f"{h}x{w} {name}", h, w, hf, vf, [sc["tgt"]], [sc["src"]])
        rows.append((w, len(sc["src"]), wrong))
    table = "; ".join(f"W = {w}: {a} (T = None), {b} (T) of {n}" for w, n, (a, b) in rows)
    print(f"  {name}: wrong sources {table}", flush=True)
    assert all(r[2] == (0, 0) for r in rows), f"{name}: wrong sources {table}"


# ---- losses and per-point gradients ---------------------------------------------------------------------------------
def loss_scenes():
    """(name, h, w, hfov, vfov, targets, sources): lists the NN families above are made of."""
    gen = np.random.default_rng(77)
    out = []
    hf = one_sided(1.0, 180, "left")
    tgt = random_points(gen, 30000, hf, VF15)
    src = np.concatenate((tgt[gen.integers(0, len(tgt), 3000)] + gen.normal(0, 0.05, (3000, 3)).astype(np.float32),
                          random_points(gen, 500, hf, VF15))).astype(np.float32)
    out.append(("dense 16x180 gap 1du", 16, 180, hf, VF15, tgt, src))
    g = LR.Grid(16, 180, hf, VF15)
    sc = LR.decoy_scene(g)
    bg = random_points(gen, 4000, hf, VF15, r_lo=40.0, r_hi=60.0)
    out.append(("decoys 16x180 gap 1du", 16, 180, hf, VF15, np.concatenate((sc["tgt"], bg)),
                np.concatenate((sc["src"], random_points(gen, 300, hf, VF15, r_lo=40.0, r_hi=60.0)))))
    el = gen.uniform(-math.pi / 2, math.pi / 2, 8000)
    tgt = _xyz(np.exp(gen.uniform(0.0, 4.0, 8000)), gen.uniform(-math.pi, math.pi, 8000), el).astype(np.float32)
    src = (tgt[gen.integers(0, 8000, 2000)] + gen.normal(0, 0.1, (2000, 3))).astype(np.float32)
    out.append(("vertical 64x720", 64, 720, HF_SYN, KITTI_VF, tgt, src))
    return out


LOSS_SCENE_IDS = ["dense", "decoys", "vertical"]
MODES = ["squared", "linear", "po2po_alone"]


def loss_config(h, w, hfov, vfov, mode):
    return {"datasets": ["kitti"], "kitti": {"vertical_cells": h, "horizontal_cells": w,
                                              "vertical_field_of_view": list(vfov)},
            "horizontal_field_of_view": list(hfov), "point_to_point_loss": True, "point_to_plane_loss": True,
            "plane_to_plane_loss": True, "normal_loss": "linear" if mode == "linear" else "squared",
            "po2po_alone": mode == "po2po_alone"}


def icp_module_run(cfg, src, src_n, tgt, tgt_n):
    """ICPLosses forward and backward of 0.7 po2po + 1.3 po2pl + 2.1 pl2pl -> (losses [3] float64, grad points,
    grad normals [N, 3] float64 (None when it gets none), the loss bits)."""
    from delora_b200.losses.icp_losses import ICPLosses
    s = torch.from_numpy(src.T[None].copy()).to(DEV).requires_grad_(True)
    sn = torch.from_numpy(src_n.T[None].copy()).to(DEV).requires_grad_(True)
    t = torch.from_numpy(tgt.T[None].copy()).to(DEV)
    tn = torch.from_numpy(tgt_n.T[None].copy()).to(DEV)
    lo, _ = ICPLosses(cfg)(s, sn, t, tn, False)
    vals = [lo["loss_po2po"], lo["loss_po2pl"], lo["loss_pl2pl"]]
    total = sum(float(u) * x.sum() for u, x in zip(UPSTREAM, vals))
    total.backward()
    torch.cuda.synchronize()
    bits = torch.cat([x.detach().reshape(1) for x in vals]).cpu().view(torch.int32).numpy()
    gp = s.grad[0].double().cpu().numpy().T
    gn = None if sn.grad is None else sn.grad[0].double().cpu().numpy().T
    return np.array([x.detach().item() for x in vals]), gp, gn, bits


@pytest.mark.parametrize("scene", range(3), ids=LOSS_SCENE_IDS)
@pytest.mark.parametrize("mode", MODES)
def test_icp_losses_module_against_float64(scene, mode, cuda_lib):
    from delora_b200 import ops
    name, h, w, hf, vf, tgt, src = loss_scenes()[scene]
    gen = np.random.default_rng(scene * 10 + MODES.index(mode))
    src_n, tgt_n = _normals(gen, len(src)), _normals(gen, len(tgt))
    cfg = loss_config(h, w, hf, vf, mode)
    ref = NR.nearest(tgt, np.arange(len(tgt)), src)
    assert len(ref.unsafe) == 0
    if mode == "po2po_alone":
        flags, sn_ref, tn_ref = R.LOSS_PO2PO, np.zeros_like(src_n), np.zeros_like(tgt_n)
    else:
        flags = R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL | (R.NORMAL_LINEAR if mode == "linear" else 0)
        sn_ref, tn_ref = src_n, tgt_n
    pr = R.prepare(src, sn_ref, None, tgt, tn_ref, (tn_ref != 0).any(axis=1), nn=ref.nn)
    res = R.evaluate(pr, flags, 1.0, upstream=UPSTREAM)
    label = f"{name} {mode}"
    assert res.M + res.Mp > 100, label
    # pair counts through the operator itself
    ns = torch.tensor([len(src)], dtype=torch.int32, device=DEV)
    nt = torch.tensor([len(tgt)], dtype=torch.int32, device=DEV)
    s4, sn4 = ops.pack_lists(torch.from_numpy(src.T[None].copy()).to(DEV),
                             torch.from_numpy(sn_ref.T[None].copy()).to(DEV), ns)
    t4, tn4, cs = ops.grid_build(torch.from_numpy(tgt.T[None].copy()).to(DEV),
                                 torch.from_numpy(tn_ref.T[None].copy()).to(DEV), nt, h, w, hf, vf)
    row, _, nn, _, _ = ops.icp_fwd_bwd(s4, sn4, ns, None, t4, tn4, cs, h, w, hf, vf, flags=flags, pointwise=True)
    row = row[0].cpu().numpy()
    assert np.array_equal(nn[0].cpu().numpy(), ref.nn), f"{label}: nn_index"
    assert int(row[3]) == res.M and int(row[4]) == res.Mp, f"{label}: (M, M') = {row[3:5]}, want {(res.M, res.Mp)}"
    losses, gp, gn, _ = icp_module_run(cfg, src, src_n, tgt, tgt_n)
    for j in range(3):
        want = res.losses[j]
        if want == 0.0:
            assert losses[j] == 0.0, f"{label}: loss {j} = {losses[j]}, want exactly 0"
        else:
            err = abs(losses[j] - want) / want
            assert err <= LOSS_TOL, f"{label}: loss {j} {losses[j]} vs float64 {want}: {err:.3e} relative"
    for what, got, want in (("points", gp, res.grad_pts), ("normals", gn, res.grad_nrm)):
        if mode == "po2po_alone" and what == "normals":
            assert got is None or not got.any(), f"{label}: po2po_alone sends a gradient to the normals"
            continue
        scale = np.abs(want).max()
        err = np.abs(got - want).max() / scale if scale > 0 else np.abs(got).max()
        assert err <= POINT_TOL, f"{label}: {what} gradients differ from float64 by {err:.3e} of their max-abs"


@pytest.mark.parametrize("scene", range(3), ids=LOSS_SCENE_IDS)
def test_repeatable_and_independent_of_target_order(scene, cuda_lib):
    name, h, w, hf, vf, tgt, src = loss_scenes()[scene]
    gen = np.random.default_rng(500 + scene)
    src_n, tgt_n = _normals(gen, len(src)), _normals(gen, len(tgt))
    ref = NR.nearest(tgt, np.arange(len(tgt)), src)
    assert (ref.ties == 1).all(), "the permuted run needs scenes without exact ties"
    cfg = loss_config(h, w, hf, vf, "squared")
    perm = gen.permutation(len(tgt))
    first = run_nn(h, w, hf, vf, [tgt], [src])[0]
    again = run_nn(h, w, hf, vf, [tgt], [src])[0]
    permuted = run_nn(h, w, hf, vf, [tgt[perm]], [src])[0]
    assert np.array_equal(first, again), f"{name}: a second run changes the neighbours"
    assert np.array_equal(perm[permuted], first), f"{name}: permuting the target list changes the neighbours"
    a = icp_module_run(cfg, src, src_n, tgt, tgt_n)
    b = icp_module_run(cfg, src, src_n, tgt, tgt_n)
    c = icp_module_run(cfg, src, src_n, tgt[perm], tgt_n[perm])
    for other, what in ((b, "a second run"), (c, "the permuted target list")):
        assert np.array_equal(a[3], other[3]), f"{name}: {what} changes the loss bits"
        assert np.array_equal(a[1].view(np.int64), other[1].view(np.int64)), f"{name}: {what} changes the gradients"
