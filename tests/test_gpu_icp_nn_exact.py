"""Every nearest neighbour the ICP operators choose, point by point, against the exact reference (tests/nn_reference.py)
on adversarial grids, on the H100.

The dense operator (delora_icp_dense_fwd_bwd) returns no neighbours, only a losses row and grad_T, so it is observed
through the normal-code fingerprint (nn_reference.py): flags = LOSS_PL2PL, T = identity, target normals replaced by
small integer codes with has-normal 1, source normals in {-1, 0, 1}^3.  Its grad_T is then (2 rn(1/M)) S for the
exact integer sums S = sum (m_i - q_nn(i)) m_i^T, and is compared BIT FOR BIT (M must be the number of sources).  A
single wrong neighbour changes S unless its code equals the right one in all three components; every scene runs
with two independent code draws.  Transformed scenes move the source points on the host (the kernel re-derives each
point's cell from the point itself; the source grid's cell only decides warp membership); one case per size keeps
T != I, with a float64 expectation and a tolerance far below one code step.

Every scene runs through the four dense instantiations (PL2PL and PO2PO|PL2PL, with and without ICP_STATS) at the
window-search hand-over limits given by the family (DELORA_ICP_MAX_STRIPS); the fingerprint must be the same bits in
every run.  The CSR operator (delora_icp_fwd_bwd) runs on lists of the same target grid and its nn_index is compared
with the reference directly.

Targets obey the operators' contract: each sits in the cell the projection gives it (tests/projection_reference.py,
the projection's float32 arithmetic, one point per cell, the nearest in range).  Sources are free.

Families:
  A  synthetic scans at 16x180, 15x180, 64x720, 64x2048 and 64x2250 under identity, T_pred, 2 m / 10 deg, yaw 178 and
     181 deg and three arbitrary transforms;
  B  exact ties: 2 to 8 targets at one exact distance (signed permutations of one dyadic offset) around anchors on
     block corners and edges, the axis azimuths and at random, plus groups on the seam with one partner in column 0
     and one in column W-1; every group again with its offsets negated, which reverses the row and column order of
     the partners.  The test counts the ties with partners in one row, adjacent rows, different 4 x 16 blocks,
     columns 0 and W-1, and inside and outside the start window, and requires each kind;
  C  near ties: exact relative separations from 2^-44 to 9e-6 (inside the fp32 band of 1e-5) and 1.2e-5, 2e-5;
  D  certification borders: the nearest target just beyond a border of the window search (e rows or columns out
     from the source's cell: the start window's border, grown windows' borders, borders at and across the seam) or
     of the block search (the border of the source's 4 x 16 block), at 1e-5 to 1e-2 relative above the exact
     distance to that border, some row targets at another range where the range-extent bound is the tighter one;
     a competitor on the source's own ray 1e-5 to 1e-3 relative farther; hand-over limits 0, 1, default, 100000;
  E  degenerate sources: the origin, the z axis, 1e-3 m and 1e4 m away, 0.4 and 50 px outside the vertical field of
     view, outside a partial horizontal field of view;
  F  degenerate targets: one target, only row 0 or row H-1, one column, adjacent blocks at 1e-3 m and 1e3 m, an empty
     grid (M = 0);
  G  grid shapes: H in {1, 2} x W in {3, 4, 5, 7}, 18x37, hfov (-90, 90) deg, a vertical field of view up to 89.5 deg;
  H  the documented limits of the search's bounds: a column pitch of 7e-4 rad (W = 8977) and a row pitch of 0.083 deg
     (360 rows over 30 deg), and grids beyond each (W = 12000, 512 rows over 30 deg).

A failing scene is localised: bisection over the sources by zeroing their normals (which leaves every search as it
was: the search never reads a normal) down to the first wrong source, then that source's chosen pixel is read with
unique codes, and the run is repeated with its warp-mates removed from the grid, which says whether the miss depends
on them.

The scenes and their builders live in tests/nn_scenes.py.
"""
import math
import time

import numpy as np
import pytest
import torch

import icp_reference as R
import nn_reference as NR
import projection_reference as PR
from nn_scenes import (DEV, GRID_IDS, GRIDS, HF, LIMITS_ALL, SEPS, SHAPES_G, SHAPES_H, SIZES_A, Scene, border_scene, deg,
                       degenerate_source_scenes, degenerate_target_scenes, near_tie_scene, random_points,
                       tie_scene, transforms_a)

pytestmark = pytest.mark.gpu

_report = []


def check(scene, family, seeds=(11, 12), T=None):
    """Run the scene through both operators; assert every neighbour; record what the family reached."""
    from delora_b200 import ops
    t0 = time.time()
    st_total = {"block_owners": 0, "f64_rerank": 0}
    for seed in seeds:
        q, m = scene.codes(seed)
        want, M = scene.expected(q, m)
        for limit in scene.limits:
            for flags in (R.LOSS_PL2PL, R.LOSS_PO2PO | R.LOSS_PL2PL):
                for stats in (False, True):
                    f = flags | (ops.ICP_STATS if stats else 0)
                    if stats:
                        ops.icp_stats(reset=True)
                    lo, g = scene.dense(q, m, f, limit)
                    if stats:
                        st = ops.icp_stats(reset=True)
                        if seed == seeds[0] and limit is None and flags == R.LOSS_PL2PL:
                            st_total = st
                    label = f"{scene.name} seed {seed} limit {limit} flags {f}"
                    assert np.array_equal(lo[:, 3], M.astype(np.float32)), f"{label}: M {lo[:, 3]} != {M}"
                    assert not lo[:, 4].any(), label
                    for b in range(scene.B):
                        if not np.array_equal(g[b], want[b]):
                            pytest.fail(f"{label}: dense fingerprint differs: {g[b]} vs {want[b]}\n  "
                                        + scene.localise(q, m, f & ~ops.ICP_STATS, limit, b))
    nn = scene.csr()
    bad = np.nonzero(nn != scene.ref.nn)[0]
    assert len(bad) == 0, (f"{scene.name}: CSR nn_index differs at {len(bad)} sources, first {bad[0]}: "
                           f"{nn[bad[0]]} vs {scene.ref.nn[bad[0]]}, point {scene.src[bad[0]].tolist()}")
    ref = scene.ref
    row = (family, scene.name, len(scene.src), int((ref.ties > 1).sum()), int(((ref.sep > 0) & (ref.sep < 2e-5)).sum()),
           st_total["block_owners"], st_total["f64_rerank"], time.time() - t0)
    _report.append(row)
    print(f"  [{family}] {scene.name}: {row[2]} sources, {row[3]} exact ties, {row[4]} near ties, "
          f"{row[5]} block-search lanes, {row[6]} float64 re-rankings ({row[7]:.1f} s)", flush=True)
    return row


def summary(family):
    rows = [r for r in _report if r[0] == family]
    return tuple(sum(r[k] for r in rows) for k in (2, 3, 4, 5, 6))


@pytest.mark.parametrize("size", SIZES_A, ids=[f"{h}x{w}" for h, w, _, _ in SIZES_A])
def test_a_synthetic_scans(size, cuda_lib):
    from delora_b200 import ops, synthetic
    h, w, w_raw, vfov = size
    vf = deg(*vfov)
    s1, s2, _, t_pred = synthetic.make_pair(40, w_raw=w_raw, rings=h, vfov_deg=vfov)
    src_pr = PR.project(s2.numpy(), h, w, HF, vf)
    imap = src_pr["index_map"].reshape(-1)
    slots = np.nonzero(imap >= 0)[0]
    p = s2.numpy().T[imap[slots]]
    for name, tm in transforms_a(t_pred):
        moved = (p.astype(np.float64) @ tm[:3, :3].T + tm[:3, 3]).astype(np.float32)
        check(Scene(f"{h}x{w} {name}", h, w, HF, vf, s1.numpy().T, moved, slots), "A")
    # T != I through the kernel's transform: float64 expectation of the sums, tolerance far below one code step
    if h * w <= 64 * 720:
        T = t_pred[:3, :].reshape(1, 12).contiguous().to(DEV)
        sc = Scene(f"{h}x{w} T_pred in the kernel", h, w, HF, vf, s1.numpy().T, p, slots)
        s_t, _ = R.apply_rigid(T.cpu().numpy(), p, np.zeros_like(p))
        ref = NR.nearest(sc.tgt, sc.pix, s_t)
        assert len(ref.unsafe) == 0, f"T != I: separations below 2^-45 at sources {ref.unsafe[:8]}"
        for seed in (21, 22):
            q, m = sc.codes(seed)
            _, ns = R.apply_rigid(T.cpu().numpy(), p, m)
            S = np.einsum("ia,ib->ab", ns.astype(np.float64) - q[ref.nn].astype(np.float64), m.astype(np.float64))
            tn = np.zeros((h * w, 4), np.float32)
            tn[:, :3], tn[:, 3] = q, 1.0
            sn = np.zeros((1, h * w, 4), np.float32)
            sn[0, slots, :3] = m
            lo, g = ops.icp_dense_fwd_bwd(sc.sg, torch.from_numpy(sn).to(DEV), T, sc.tg,
                                          torch.from_numpy(tn)[None].to(DEV), h, w, HF, vf, flags=R.LOSS_PL2PL)
            got = g[0].cpu().numpy().astype(np.float64).reshape(3, 4)[:, :3] / (2.0 / len(p))
            assert int(lo[0, 3]) == len(p)
            assert np.abs(got - S).max() < 0.25, f"T != I, seed {seed}: sums {got} vs float64 {S}"
        nn = sc.csr(T=T, src=p)
        assert np.array_equal(nn, ref.nn), f"T != I: CSR nn_index differs at {np.count_nonzero(nn != ref.nn)} sources"


TIE_KINDS = ("one row", "adjacent rows", "across a block border", "across the seam", "window and block search")


def tie_kinds(sc, groups):
    """Count the sources whose exact tie (the group members in the grid at the exact minimum distance) has partners
    in one row, in adjacent rows, in different 4 x 16 blocks, in columns 0 and W-1, and both inside and outside the
    3 x 5 start window of the source's cell."""
    g = sc.g
    counts = dict.fromkeys(TIE_KINDS, 0)
    where = dict(zip(map(tuple, sc.tgt.tolist()), sc.pix.tolist()))
    u, v, _ = PR.coords(g, sc.src[:, 0], sc.src[:, 1], sc.src[:, 2])
    for i, grp in enumerate(groups):
        if sc.ref.ties[i] < 2:
            continue
        d = [NR.exact_d2(sc.src[i], t) for t in grp]
        best = min(d)
        pix = [where[tuple(t.tolist())] for t, x in zip(grp, d) if x == best and tuple(t.tolist()) in where]
        if len(pix) < 2:
            continue
        rows, cols = np.array(pix) // g.W, np.array(pix) % g.W
        counts["one row"] += int(len(rows) != len(set(rows.tolist())))
        counts["adjacent rows"] += int(any(abs(a - b) == 1 for a in rows for b in rows))
        counts["across a block border"] += int(len({(a // 4, b // 16) for a, b in zip(rows, cols)}) > 1)
        counts["across the seam"] += int(0 in cols and g.W - 1 in cols)
        cc, rc = int(np.clip(np.rint(u[i]), 0, g.W - 1)), int(np.clip(np.rint(v[i]), 0, g.H - 1))
        dcol = np.minimum(np.abs(cols - cc), g.W - np.abs(cols - cc))
        inside = (np.abs(rows - rc) <= 1) & (dcol <= 2)
        counts["window and block search"] += int(inside.any() and not inside.all())
    return counts


@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_b_exact_ties(grid, cuda_lib):
    h, w, hf, vf = grid
    total = dict.fromkeys(TIE_KINDS, 0)
    for mirror in (False, True):
        tg, src, groups = tie_scene(h, w, hf, vf, 7 + h, mirror)
        sc = Scene(f"{h}x{w} ties{' mirrored' if mirror else ''}", h, w, hf, vf, tg, src, limits=LIMITS_ALL)
        row = check(sc, "B")
        assert row[3] >= len(src) // 4, f"only {row[3]} of {len(src)} sources have an exact tie in the grid"
        kinds = tie_kinds(sc, groups)
        print(f"    tie partners: " + ", ".join(f"{k} {n}" for k, n in kinds.items()), flush=True)
        for k, n in kinds.items():
            total[k] += n
    missing = [k for k, n in total.items() if n == 0]
    assert not missing, f"no exact tie with partners {missing}: {total}"


@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_c_near_ties(grid, cuda_lib):
    h, w, hf, vf = grid
    near = 0
    for k, sep in enumerate(SEPS):
        tg, src = near_tie_scene(h, w, hf, vf, sep, 100 * h + k)
        sc = Scene(f"{h}x{w} sep {sep:.3g}", h, w, hf, vf, tg, src, limits=LIMITS_ALL)
        check(sc, "C")
        near += int(((sc.ref.sep > sep * 0.3) & (sc.ref.sep < sep * 3)).sum())
    assert near >= 60, f"only {near} sources keep their near tie"


@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_d_certification_borders(grid, cuda_lib):
    h, w, hf, vf = grid
    tg, src = border_scene(h, w, hf, vf, 300 + h)
    sc = Scene(f"{h}x{w} borders", h, w, hf, vf, tg, src, limits=LIMITS_ALL)
    check(sc, "D")
    # the nearest target is the one beyond the border, outside the 3 x 5 start window, for most sources
    beyond = outside_start_window(sc)
    assert beyond >= 0.7 * len(src), f"only {beyond} of {len(src)} nearest targets lie beyond the start window"


def outside_start_window(sc):
    """Number of sources whose exact nearest target lies outside the 3 x 5 start window of their own cell."""
    g = sc.g
    u, v, _ = PR.coords(g, sc.src[:, 0], sc.src[:, 1], sc.src[:, 2])
    cc = np.clip(np.rint(np.nan_to_num(u)), 0, g.W - 1).astype(np.int64)
    rc = np.clip(np.rint(np.nan_to_num(v)), 0, g.H - 1).astype(np.int64)
    nn = sc.ref.nn
    dr = np.abs(nn // g.W - rc)
    dc = np.abs(nn % g.W - cc)
    dc = np.minimum(dc, g.W - dc)
    return int(((nn >= 0) & ((dr > 1) | (dc > 2))).sum())


def test_e_degenerate_sources(cuda_lib):
    for sc in degenerate_source_scenes(LIMITS_ALL):
        check(sc, "E")


def test_f_degenerate_targets(cuda_lib):
    for sc in degenerate_target_scenes(LIMITS_ALL):
        check(sc, "F")


@pytest.mark.parametrize("shape", SHAPES_G, ids=[f"{s[0]}x{s[1]}-{k}" for k, s in enumerate(SHAPES_G)])
def test_g_grid_shapes(shape, cuda_lib):
    h, w, hf, vf = shape
    g = PR.Grid(h, w, hf, vf)
    gen = np.random.default_rng(h * 1000 + w)
    tgt = random_points(g, gen, max(4 * h * w, 64))
    src = random_points(g, gen, max(2 * h * w, 300))
    check(Scene(f"{h}x{w} hfov {math.degrees(hf[1]):.1f} vfov {math.degrees(vf[1]):.1f}", h, w, hf, vf, tgt, src,
                limits=LIMITS_ALL), "G")


@pytest.mark.parametrize("shape", SHAPES_H, ids=[f"{s[0]}x{s[1]}" for s in SHAPES_H])
def test_h_documented_limits(shape, cuda_lib):
    h, w, hf, vf = shape
    g = PR.Grid(h, w, hf, vf)
    gen = np.random.default_rng(h + w)
    tgt = random_points(g, gen, 2 * h * w, 2.0, 40.0)
    src = random_points(g, gen, 20000, 2.0, 40.0)
    check(Scene(f"{h}x{w}", h, w, hf, vf, tgt, src, limits=LIMITS_ALL), "H")


@pytest.fixture(scope="module", autouse=True)
def _family_report():
    """At the end of the module (or of whichever of its tests ran), per family: sources checked, exact ties, near
    ties, block-search lanes, float64 re-rankings and seconds."""
    yield
    if not _report:
        return
    print("\nper family: sources, exact ties, near ties, block-search lanes, float64 re-rankings, seconds")
    for fam in "ABCDEFGH":
        rows = [r for r in _report if r[0] == fam]
        if rows:
            print(f"  {fam}: " + ", ".join(str(x) for x in summary(fam)) + f", {sum(r[7] for r in rows):.1f}")
