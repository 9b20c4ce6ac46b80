"""-m gpu: the ICP information operator (delora_icp_dense_information[_scaled]) on the dense search's adversarial grids
and on exact designs, on the H100.

  A  NN ids, pixel by pixel, on every family of test_gpu_icp_nn_exact.py (tests/nn_scenes.py): synthetic scans under
     arbitrary transforms, exact ties, near ties, certification borders, degenerate sources and targets, H in {1, 2} x
     W in {3, 4, 5, 7} (the degenerate window branch) and the widths 8977 and 12000.  Two normal configurations keep
     every pair: a normal on every valid cell with PO2PL | PL2PL, and none anywhere with PO2PO.  Every id is
     nn_reference.nearest's under info_reference.pair_masks; at every hand-over limit (DELORA_ICP_MAX_STRIPS 0, 1,
     default, 100000: at 0 and 1 most ids are written by the block search's finisher warp) the ids, the info row,
     M and M' are the same bits, and losses and grad_T are delora_icp_dense_fwd_bwd's bits at that limit (across
     limits they are not: the handed-over lanes' terms are summed in another order).
  B  H against the float64 restatement (info_reference.information on the kernel's own ids) within 64 u A + u |H|, on
     test_gpu_icp_losses.py's six transforms (identity, T_pred, metres + 10 deg, a 178 deg yaw across the seam, no
     normals, an empty source) at 16x180, 15x180 and 64x720 for all 11 flag sets, and once on the benchmark's batch
     (B = 8 at 64x2048).  A pair whose enabled terms have no count returns the exact row (H = 0, eigenvalues 0, the
     identity's rows, M and M' as stored); every row is the same bits alone at B = 1 and inside batches that mix
     empty and full pairs.  Eigenvalues within ||dH|| (Weyl); eigenvectors checked per cluster of eigenvalues closer
     than 1e-3 of the largest, as the cluster's invariant subspace within the Davis-Kahan bound ||dH|| / gap.
  C  Exact designs (info_reference.exact_design): integer points, targets T p for a signed permutation T with an
     integer translation, grids from ops.project_normals with axis-aligned normals written on the valid cells.  Every
     fp32 sum is exact, so H is info_reference.kernel_order's rounding BIT FOR BIT, also through the scaled operator
     with factors 0.25 and 4.  Designed spectra: a tie followed by a smaller eigenvalue (the eigenvectors are the unit
     axes, the lower column first), an exact triple (orthonormal vectors whose projector is exact), three exact zeros,
     and near ties from 1e-3 down to 1e-12 of the largest eigenvalue (the cluster's subspace within Davis-Kahan).
"""
import functools
import math
import time

import numpy as np
import pytest
import torch

import icp_reference as R
import info_reference as IR
import nn_reference as NR
import projection_reference as PR
from nn_scenes import (GRIDS, HF, LIMITS_ALL, SEPS, SHAPES_G, SHAPES_H, SIZES_A, Scene, border_scene, deg,
                       degenerate_source_scenes, degenerate_target_scenes, max_strips, near_tie_scene, random_points,
                       tie_scene, transforms_a)

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
EPS = 2.0 ** -53
LAM = 0.6
EVERY = R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL
_report = {}


def bits(x):
    return x.contiguous().view(torch.int32)


# ================================================================================================ A: NN ids
def scenes_a(size):
    from delora_b200 import synthetic
    h, w, w_raw, vfov = size
    vf = deg(*vfov)
    s1, s2, _, t_pred = synthetic.make_pair(40, w_raw=w_raw, rings=h, vfov_deg=vfov)
    imap = PR.project(s2.numpy(), h, w, HF, vf)["index_map"].reshape(-1)
    slots = np.nonzero(imap >= 0)[0]
    p = s2.numpy().T[imap[slots]]
    for name, tm in transforms_a(t_pred):
        moved = (p.astype(np.float64) @ tm[:3, :3].T + tm[:3, 3]).astype(np.float32)
        yield Scene(f"{h}x{w} {name}", h, w, HF, vf, s1.numpy().T, moved, slots)


def scenes_b():
    for h, w, hf, vf in GRIDS:
        for mirror in (False, True):
            tg, src, _ = tie_scene(h, w, hf, vf, 7 + h, mirror)
            yield Scene(f"{h}x{w} ties{' mirrored' if mirror else ''}", h, w, hf, vf, tg, src)


def scenes_c():
    for h, w, hf, vf in GRIDS:
        for k, sep in enumerate(SEPS):
            tg, src = near_tie_scene(h, w, hf, vf, sep, 100 * h + k)
            yield Scene(f"{h}x{w} sep {sep:.3g}", h, w, hf, vf, tg, src)


def scenes_d():
    for h, w, hf, vf in GRIDS:
        tg, src = border_scene(h, w, hf, vf, 300 + h)
        yield Scene(f"{h}x{w} borders", h, w, hf, vf, tg, src)


def scenes_random(shapes):
    for h, w, hf, vf in shapes:
        g = PR.Grid(h, w, hf, vf)
        gen = np.random.default_rng(h * 1000 + w)
        big = h * w > 20000
        tgt = random_points(g, gen, 2 * h * w if big else max(4 * h * w, 64), *((2.0, 40.0) if big else ()))
        src = random_points(g, gen, 20000 if big else max(2 * h * w, 300), *((2.0, 40.0) if big else ()))
        yield Scene(f"{h}x{w}", h, w, hf, vf, tgt, src)


FAMILIES = {**{f"A-{s[0]}x{s[1]}": functools.partial(scenes_a, s) for s in SIZES_A[:3]},
            "B-ties": scenes_b, "C-near-ties": scenes_c, "D-borders": scenes_d,
            "E-degenerate-sources": degenerate_source_scenes, "F-degenerate-targets": degenerate_target_scenes,
            "G-shapes": functools.partial(scenes_random, SHAPES_G[:8]),
            "H-limits": functools.partial(scenes_random, SHAPES_H[:2])}


def normal_grids(sc, with_normals, seed):
    """(source normal grid, target normal grid) on the GPU: seeded unit normals with has-normal 1 on every valid cell
    of both grids, or zeros everywhere; and the host copies [B, HW, 3], [HW, 3], [HW] the reference reads."""
    hw = sc.h * sc.w
    gen = np.random.default_rng(seed)
    tn = np.zeros((hw, 4), np.float32)
    sn = np.zeros((sc.B, hw, 4), np.float32)
    if with_normals:
        v = gen.normal(size=(hw, 3))
        tn[sc.pix, :3] = (v / np.linalg.norm(v, axis=1, keepdims=True))[sc.pix]
        tn[sc.pix, 3] = 1.0
        v = gen.normal(size=(len(sc.src), 3))
        sn[sc.pair, sc.slot, :3] = v / np.linalg.norm(v, axis=1, keepdims=True)
    tn_dev = torch.from_numpy(np.broadcast_to(tn, (sc.B, hw, 4)).copy()).to(DEV)
    return torch.from_numpy(sn).to(DEV), tn_dev, sn[:, :, :3], tn[:, :3], tn[:, 3] != 0


def expected_ids(sc, sn, tn, t_has, flags):
    """[B, HW] the exact NN of every source under the losses' masks, -1 elsewhere."""
    out = np.full((sc.B, sc.h * sc.w), -1, np.int64)
    eye = sc.eye[0].cpu().numpy()
    for b in range(sc.B):
        k = sc.pair == b
        kind = IR.pair_masks(eye, sc.src[k], sn[b, sc.slot[k]], tn, t_has, sc.ref.nn[k], flags)
        out[b, sc.slot[k]] = np.where(kind > 0, sc.ref.nn[k], -1)
    return out


def check_ids(sc, family):
    from delora_b200 import ops
    t0 = time.time()
    for with_normals, flags in ((True, R.LOSS_PO2PL | R.LOSS_PL2PL), (False, R.LOSS_PO2PO)):
        sn, tn, sn_h, tn_h, t_has = normal_grids(sc, with_normals, 3)
        want = expected_ids(sc, sn_h, tn_h, t_has, flags)
        first = None
        for limit in LIMITS_ALL:
            label = f"{family} {sc.name} {R.flag_name(flags)} limit {limit}"
            with max_strips(limit):
                out = ops.icp_dense_information(sc.sg, sn, sc.eye, sc.tg, tn, sc.h, sc.w, sc.hfov, sc.vfov, LAM, flags)
                lo, g = ops.icp_dense_fwd_bwd(sc.sg, sn, sc.eye, sc.tg, tn, sc.h, sc.w, sc.hfov, sc.vfov, LAM, flags)
                torch.cuda.synchronize()
            got = out[3].cpu().numpy().astype(np.int64)
            bad = np.argwhere(got != want)
            assert len(bad) == 0, (f"{label}: {len(bad)} NN ids differ from the exact NN, first (pair, pixel) "
                                   f"{bad[0].tolist()}: {got[tuple(bad[0])]} vs {want[tuple(bad[0])]}")
            assert torch.equal(bits(out[0]), bits(lo)) and torch.equal(bits(out[1]), bits(g)), \
                f"{label}: losses or grad_T differ from icp_dense_fwd_bwd"
            if first is None:
                first = out
            # the info pass reads only the ids; losses and grad_T add the handed-over lanes' terms to their warp's
            # partial row after the window search's, so only their counts are the same bits at every limit
            for a, b, what in ((first[2], out[2], "info"), (first[3], out[3], "ids"), (first[0][:, 3:5], out[0][:, 3:5],
                                                                                      "M, M'")):
                assert torch.equal(bits(a), bits(b)), f"{label}: {what} differs from limit {LIMITS_ALL[0]}'s"
    n = _report.setdefault(family, [0, 0, 0.0])
    n[0] += 2 * len(sc.src)                         # Scene refuses scenes with unsafe sources: none is excluded
    n[1] += 2 * len(sc.ref.unsafe)
    n[2] += time.time() - t0


@pytest.mark.parametrize("family", list(FAMILIES))
def test_nn_ids_on_the_adversarial_families(family, cuda_lib):
    for sc in FAMILIES[family]():
        check_ids(sc, family)
    print(f"  [{family}] {_report[family][0]} ids compared, {_report[family][1]} excluded as unsafe "
          f"({_report[family][2]:.1f} s)", flush=True)


# ================================================================================================ B: H against float64
SIZES = [(16, 180, 192, (-15.0, 15.0)), (15, 180, 192, (-15.0, 15.0)), (64, 720, 1024, (-24.5, 2.0))]
NB = 6


def transforms(t_pred):
    from delora_b200 import synthetic
    ts = [np.eye(4), t_pred.numpy().astype(np.float64),
          synthetic.transform_matrix(1.5, -0.4, 0.1, math.radians(10.0), math.radians(1.0), 0.0),
          synthetic.transform_matrix(0.5, 0.2, 0.0, math.radians(178.0)),
          t_pred.numpy().astype(np.float64), t_pred.numpy().astype(np.float64)]
    return torch.tensor(np.stack([t[:3, :] for t in ts]).reshape(NB, 12), dtype=torch.float32)


class Pairs:
    """Targets in rows 0..B-1, sources in rows B..2B-1 of grids from ops.project_normals; a quarter of the normals
    dropped; pair 4 has no normal anywhere, pair 5 an empty source."""

    def __init__(self, h, w, w_raw, vfov, n=NB, seed=40, drop=True):
        from delora_b200 import ops, synthetic
        self.h, self.w, self.n = h, w, n
        cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov)
        self.hf, self.vf = tuple(cfg["horizontal_field_of_view"]), tuple(cfg["kitti"]["vertical_field_of_view"])
        made = [synthetic.make_pair(seed + k, w_raw=w_raw, rings=h, vfov_deg=vfov) for k in range(n)]
        scans = [m[0] for m in made] + [m[1] for m in made]
        stride = max(s.shape[1] for s in scans)
        pts = torch.zeros((2 * n, 3, stride))
        counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
        for i, s in enumerate(scans):
            pts[i, :, :s.shape[1]] = s
        if drop:
            counts[n + 5] = 0
        _, _, pg, ng = ops.project_normals(pts.to(DEV), counts.to(DEV), h, w, self.hf, self.vf)
        if drop:
            valid = pg[:, :, 3].view(torch.int32) >= 0
            gen = torch.Generator(device=DEV).manual_seed(h * 100000 + w)
            gone = valid & (torch.rand(valid.shape, generator=gen, device=DEV) < 0.25)
            gone[4], gone[n + 4] = valid[4], valid[n + 4]
            ng[gone] = 0.0
            self.T = transforms(made[0][3]).to(DEV)
        else:
            self.T = torch.stack([m[3][:3, :].reshape(12) for m in made]).float().to(DEV)
        self.pg, self.ng = pg, ng

    def run(self, flags, pairs=None, lam=LAM):
        from delora_b200 import ops
        k = torch.arange(self.n, device=DEV) if pairs is None else torch.tensor(pairs, device=DEV)
        return ops.icp_dense_information(self.pg[self.n + k].contiguous(), self.ng[self.n + k].contiguous(),
                                         self.T[k].contiguous(), self.pg[k].contiguous(), self.ng[k].contiguous(),
                                         self.h, self.w, self.hf, self.vf, lam, flags)

    def host(self, k):
        tp, tn, sp, sn = (x.cpu().numpy() for x in (self.pg[k], self.ng[k], self.pg[self.n + k], self.ng[self.n + k]))
        return tp, tn, sp, sn, self.T[k].cpu().numpy()


@functools.lru_cache(maxsize=None)
def pairs(size_index):
    return Pairs(*SIZES[size_index])


def exact_nn(tp, sp, T):
    """-> (exact NN pixel per source pixel, -1 where invalid; source pixels without a safe exact answer)."""
    t_ok, s_ok = tp[:, 3].view(np.int32) >= 0, sp[:, 3].view(np.int32) >= 0
    nn = np.full(len(sp), -1, np.int64)
    if not s_ok.any():
        return nn, np.zeros(0, np.int64)
    s, _ = R.apply_rigid(T, sp[s_ok, :3], np.zeros_like(sp[s_ok, :3]))
    res = NR.nearest(tp[t_ok, :3], np.nonzero(t_ok)[0], s)
    nn[s_ok] = res.nn
    return nn, np.nonzero(s_ok)[0][res.unsafe]


def check_eigen(row, Hm, label):
    """Eigenvalues ascending within ||dH|| of numpy's (Weyl); unit eigenvectors with the sign convention; for every
    cluster of reference eigenvalues closer than 1e-3 of the largest, the projector on the row's vectors within
    2 ||dH|| / gap + 1e-5 of the reference projector (Davis-Kahan; gap: to the rest of the spectrum)."""
    ev, V = row[36:42].astype(np.float64), row[42:78].reshape(6, 6).astype(np.float64)
    ref_ev, ref_V = np.linalg.eigh(Hm)
    lmax = max(abs(ref_ev).max(), 1e-30)
    dH = np.linalg.norm(row[:36].reshape(6, 6).astype(np.float64) - Hm, 2) + 1e-6 * lmax
    assert np.all(np.diff(ev) >= 0), f"{label}: eigenvalues not ascending"
    assert np.abs(ev - ref_ev).max() <= dH, (label, ev, ref_ev)
    for k in range(6):
        assert abs(np.linalg.norm(V[k]) - 1.0) < 1e-5, label
        big = int(np.argmax(np.abs(V[k])))
        assert V[k, big] > 0, f"{label}: eigenvector {k} breaks the sign convention"
    start = 0
    for k in range(1, 7):
        if k < 6 and ref_ev[k] - ref_ev[k - 1] <= 1e-3 * lmax:
            continue
        c = list(range(start, k))
        rest = [j for j in range(6) if j not in c]
        if rest:
            gap = min(abs(ref_ev[i] - ref_ev[j]) for i in c for j in rest)
            P, Pr = V[c].T @ V[c], ref_V[:, c] @ ref_V[:, c].T
            err = np.linalg.norm(P - Pr, 2)
            assert err <= 2.0 * dH / gap + 1e-5, (label, c, err, dH, gap)
        start = k


def exact_empty_row(row, lrow, label):
    want = np.zeros(IR.INFO_ROW, np.float32)
    want[42:78] = np.eye(6, dtype=np.float32).reshape(-1)
    want[78:80] = lrow[3:5]
    assert np.array_equal(row.view(np.int32), want.view(np.int32)), f"{label}: not the exact row of a pair without H"


def check_h(pr, k, out, flags, lam, label, counts):
    losses, _, info, nn = (x[k].cpu().numpy() for x in out)
    tp, tn, sp, sn, T = pr.host(k)
    ids = nn.astype(np.int64)
    exact, unsafe = exact_nn(tp, sp, T)
    kind = IR.pair_masks(T, sp[:, :3], sn[:, :3], tn[:, :3], tn[:, 3] != 0, exact, flags)
    want = np.where(kind > 0, exact, -1)
    keep = np.ones(len(ids), bool)
    keep[unsafe] = False
    bad = np.nonzero((ids != want) & keep)[0]
    assert bad.size == 0, f"{label}: {bad.size} NN ids differ from the exact NN, first {bad[:5]}"
    counts[0] += int((sp[:, 3].view(np.int32) >= 0).sum()) - len(unsafe)
    counts[1] += len(unsafe)
    Hm, A, M, Mp = IR.information(T, sp[:, :3], sn[:, :3], tn[:, :3], tn[:, 3] != 0, ids, flags, lam)
    assert info[78] == M == losses[3] and info[79] == Mp == losses[4], (label, info[78:], M, Mp, losses[3:5])
    if not (flags & (R.LOSS_PO2PL | R.LOSS_PL2PL) and M) and not (flags & R.LOSS_PO2PO and Mp):
        exact_empty_row(info, losses, label)
        return False
    Hg = info[:36].reshape(6, 6).astype(np.float64)
    tol = 64 * U * A + U * np.abs(Hm)
    assert np.all(np.abs(Hg - Hm) <= tol), f"{label}: max |dH| / tol = {(np.abs(Hg - Hm) / tol).max():.3g}"
    check_eigen(info, Hm, label)
    return True


@pytest.mark.parametrize("size_index", range(len(SIZES)), ids=[f"{h}x{w}" for h, w, _, _ in SIZES])
def test_h_against_float64_on_every_flag_set(size_index, cuda_lib):
    pr = pairs(size_index)
    counts, empty = [0, 0], 0
    for flags in R.flag_matrix():
        out = pr.run(flags)
        for k in range(NB):
            label = f"{pr.h}x{pr.w} pair {k} {R.flag_name(flags)}"
            empty += not check_h(pr, k, out, flags, LAM, label, counts)
            alone = pr.run(flags, [k])
            for a, b in zip(out, alone):
                assert torch.equal(bits(a[k]), bits(b[0])), f"{label}: B = 1 differs from the batch"
    assert empty >= sum(1 + (not f & R.LOSS_PO2PO) for f in R.flag_matrix())   # pair 5; pair 4 without PO2PO
    print(f"  [B {pr.h}x{pr.w}] {counts[0]} ids compared, {counts[1]} excluded as unsafe, {empty} exact empty rows")


def test_batches_mixing_empty_and_full_pairs(cuda_lib):
    pr = pairs(0)
    for flags in (R.LOSS_PO2PL | R.LOSS_PL2PL, EVERY | R.NORMAL_LINEAR, R.LOSS_PO2PO):
        alone = {k: pr.run(flags, [k]) for k in (0, 3, 4, 5)}
        for order in ([5, 0, 5, 3], [4, 5, 4], [3, 5, 0, 4, 5]):
            out = pr.run(flags, order)
            for i, k in enumerate(order):
                for a, b in zip(out, alone[k]):
                    assert torch.equal(bits(a[i]), bits(b[0])), f"{R.flag_name(flags)} {order}: pair {k} at {i} differs"
            torch.cuda.synchronize()
        exact_empty_row(alone[5][2][0].cpu().numpy(), alone[5][0][0].cpu().numpy(), f"{R.flag_name(flags)} empty")


def test_benchmark_batch(cuda_lib):
    """B = 8 synthetic 64x2048 pairs at their T_pred, the benchmark's loss flags."""
    pr = Pairs(64, 2048, 2048, (-24.5, 2.0), n=8, seed=0, drop=False)
    flags = R.LOSS_PO2PL | R.LOSS_PL2PL
    out = pr.run(flags, lam=1.0)
    counts = [0, 0]
    for k in range(8):
        assert check_h(pr, k, out, flags, 1.0, f"64x2048 pair {k}", counts)
    print(f"  [B 64x2048 x 8] {counts[0]} ids compared, {counts[1]} excluded as unsafe")


# ================================================================================================ C: exact designs
@functools.lru_cache(maxsize=None)
def design_grids(name):
    """-> (design, [2, HW, 4] point and normal grids (source, target) on the GPU, the source and the target pixel of
    every design point)."""
    from delora_b200 import ops
    d = IR.exact_design(name)
    h, w, hf, vf = IR.DESIGN_GRID
    n = len(d.p)
    pts = torch.from_numpy(np.stack([d.p.T, d.tgt_p.T])).contiguous().to(DEV)
    _, imap, pg, ng = ops.project_normals(pts, torch.tensor([n, n], dtype=torch.int32, device=DEV), h, w, hf, vf)
    imap = imap.reshape(2, -1).cpu().numpy().astype(np.int64)
    where = np.full((2, n), -1, np.int64)
    for b in range(2):
        cells = np.nonzero(imap[b] >= 0)[0]
        where[b, imap[b, cells]] = cells
        assert len(cells) == n and (where[b] >= 0).all(), f"{name}: a design point does not own its pixel"
    host = ng.cpu().numpy()
    for b, (nrm, has) in enumerate(((d.m, np.any(d.m != 0, axis=1)), (d.tgt_n, d.tgt_has))):
        host[b] = 0.0
        host[b, where[b], :3] = nrm
        host[b, where[b], 3] = has.astype(np.float32)
    return d, pg, torch.from_numpy(host).to(DEV), where[0], where[1]


def run_design(name, flags, lam, factor=None):
    """One design through the operator: every id the twin's pixel, M and M' the design's, H kernel_order's bits.
    -> (info row, the float64 H the kernel solves, label)."""
    from delora_b200 import ops
    d, pg, ng, src_pix, tgt_pix = design_grids(name)
    h, w, hf, vf = IR.DESIGN_GRID
    T = torch.from_numpy(d.T.reshape(1, 12)).to(DEV)
    args = (pg[:1], ng[:1], T, pg[1:], ng[1:], h, w, hf, vf)
    if factor is None:
        out = ops.icp_dense_information(*args, lam, flags)
    else:
        out = ops.icp_dense_information_scaled(*args, torch.tensor([factor], dtype=torch.float32, device=DEV),
                                               lam, flags)
    _, _, info, nn = (x[0].cpu().numpy() for x in out)
    S, M, Mp = IR.design_sums(d, flags)
    Hd, H32 = IR.kernel_order(S, M, Mp, flags, lam, factor)
    label = f"{name} {R.flag_name(flags)} lam {lam:.3g} factor {factor}"
    kind = IR.pair_masks(d.T, d.p, d.m, d.tgt_n, d.tgt_has, np.arange(len(d.p)), flags)
    want = np.full(len(nn), -1, np.int64)
    want[src_pix] = np.where(kind > 0, tgt_pix, -1)
    assert np.array_equal(nn.astype(np.int64), want), f"{label}: an NN id is not the twin's pixel"
    assert info[78] == M and info[79] == Mp, (label, info[78:], M, Mp)
    got = info[:36].reshape(6, 6)
    assert np.array_equal(got.view(np.int32), H32.view(np.int32)), \
        f"{label}: H is not the kernel-order value bit for bit, max |dH| {np.abs(got - H32).max():.3g}"
    return info, Hd, label


FACTORS = (None, 0.25, 4.0)


@pytest.mark.parametrize("factor", FACTORS, ids=["unscaled", "f0.25", "f4"])
def test_mixed_design_is_bit_exact_on_every_flag_set(factor, cuda_lib):
    for flags in R.flag_matrix():
        info, Hd, label = run_design("mixed", flags, LAM, factor)
        check_eigen(info, Hd, label)


def check_axes_in_tie_order(info, Hd, label, cols=tuple(range(6))):
    """H diagonal on the columns `cols`, whose values are the smallest: the first eigenvalues are their fp32 roundings
    in (value, column) order, the eigenvectors the unit axes of those columns."""
    diag = np.diag(Hd)
    order = sorted(cols, key=lambda c: (diag[c], c))
    ev, V = info[36:42], info[42:78].reshape(6, 6)
    assert np.array_equal(ev[:len(cols)], diag[order].astype(np.float32)), (label, ev, diag[order])
    for x, c in enumerate(order):
        assert np.array_equal(V[x], np.eye(6, dtype=np.float32)[c]), \
            f"{label}: eigenvector {x} is {V[x].tolist()}, the unit axis {c} was expected (order {order})"


@pytest.mark.parametrize("factor", FACTORS, ids=["unscaled", "f0.25", "f4"])
def test_tied_eigenvalues_keep_the_lower_column_first(factor, cuda_lib):
    """tie: translation diagonal (b, b, a), a < b (the old selection swapped columns 0 and 2, so the tie came out as
    column 1, then 0); zeros: three exact zeros (PL2PL only, linear too), the axes 0, 1, 2 in order."""
    info, Hd, label = run_design("tie", IR.LOSS_PO2PL, 1.0, factor)
    assert Hd[0, 0] == Hd[1, 1] > Hd[2, 2]
    check_axes_in_tie_order(info, Hd, label)
    for flags in (IR.LOSS_PL2PL, IR.LOSS_PL2PL | IR.NORMAL_LINEAR):
        info, Hd, label = run_design("zeros", flags, 1.0, factor)
        assert not Hd[:3].any() and np.array_equal(info[36:39], np.zeros(3, np.float32)), label
        check_axes_in_tie_order(info, Hd, label)


@pytest.mark.parametrize("factor", FACTORS, ids=["unscaled", "f0.25", "f4"])
def test_exact_triple_eigenvalue(factor, cuda_lib):
    """Two exact triples: each triple's vectors orthonormal, their projector the exact one within 8 u (each stored
    component is the float64 one rounded to fp32, relative error u; the three outer products add 3 (2 u + u^2))."""
    info, Hd, label = run_design("triple", R.LOSS_PO2PO, 1.0, factor)
    ev, V = info[36:42].astype(np.float64), info[42:78].reshape(6, 6).astype(np.float64)
    assert np.array_equal(info[36:42], np.sort(np.diag(Hd)).astype(np.float32)), (label, ev)
    for c, block in ((slice(0, 3), np.diag([1.0, 1, 1, 0, 0, 0])), (slice(3, 6), np.diag([0.0, 0, 0, 1, 1, 1]))):
        Q = V[c]
        assert np.abs(Q @ Q.T - np.eye(3)).max() <= 8 * U, (label, Q @ Q.T)
        assert np.abs(Q.T @ Q - block).max() <= 8 * U, (label, Q.T @ Q)


@pytest.mark.parametrize("ratio", (1e-3, 1e-6, 1e-9, 1e-12))
@pytest.mark.parametrize("factor", (None, 4.0), ids=["unscaled", "f4"])
def test_near_ties_keep_their_invariant_subspace(ratio, factor, cuda_lib):
    """The near design: two rotation eigenvalues ratio of the largest apart.  Their individual vectors are not
    determined to better than ||dH|| / (ratio lmax); the pair's subspace is, within Davis-Kahan's ||dH|| / gap to the
    rest of the spectrum (dH: the float64 solve's backward error, 64 eps ||H||, and the fp32 rounding of the stored
    vectors).  The exact ties in the translation block keep the unit axes in column order."""
    d = IR.exact_design("near")
    lam = IR.near_tie_lambda(d, ratio)
    info, Hd, label = run_design("near", d.flags, lam, factor)
    ref_ev, ref_V = np.linalg.eigh(Hd)
    ev, V = info[36:42].astype(np.float64), info[42:78].reshape(6, 6).astype(np.float64)
    lmax = ref_ev[5]
    dH = 64 * EPS * np.linalg.norm(Hd, 2)
    assert np.abs(ev - ref_ev).max() <= dH + U * lmax, (label, ev, ref_ev)
    assert ratio / 3 <= (ref_ev[5] - ref_ev[4]) / lmax <= 3 * ratio, label
    gap = ref_ev[4] - ref_ev[3]
    P, Pr = V[4:].T @ V[4:], ref_V[:, 4:] @ ref_V[:, 4:].T
    err = np.linalg.norm(P - Pr, 2)
    print(f"  [near {ratio:.0e} {factor}] subspace error {err:.3g}, bound {2 * dH / gap + 8 * U:.3g}")
    assert err <= 2 * dH / gap + 8 * U, (label, err, dH, gap)
    assert np.abs(V[4:] @ V[4:].T - np.eye(2)).max() <= 8 * U, label
    assert not Hd[:3, 3:].any() and Hd[0, 0] == Hd[1, 1]
    check_axes_in_tie_order(info, Hd, label, cols=(0, 1, 2))


@pytest.fixture(scope="module", autouse=True)
def _id_report():
    yield
    if _report:
        print("\nNN ids per family: compared, excluded as unsafe, seconds")
        for fam, (n, u, t) in _report.items():
            print(f"  {fam}: {n}, {u}, {t:.1f}")
