"""Float64 reference of the Gauss-Newton information of delora_icp_dense_information (test infrastructure, CPU only).

For one scan pair with fixed correspondences (the exact NN of nn_reference, with the masks of the losses), H is
restated in float64 from explicit Jacobian matrices of the right perturbation T(xi) = T Exp(xi), xi = (rho, phi):
  po2pl   r = n_t^T (s - q)      J = n_t^T [R, -R [p]x]             (1 x 6)
  pl2pl   e = R m - n_t          J = [0, -R [m]x]                   (3 x 6)   squared
          o = 1 - n_t^T R m      J = [0, n_t^T R [m]x]              (1 x 6)   linear
  po2po   d = s - q              J = [R, -R [p]x]                   (3 x 6)
  H = 2 (lambda / M sum_po2pl J^T J + 1 / M sum_pl2pl J^T J + 1 / (3 M') sum_po2po J^T J)
with the losses' means (po2po over the 3 M' coordinates).  `objective` is that loss in float64 at T Exp(xi), for
checking H against finite differences where every residual is zero (there the Hessian is exactly Gauss-Newton).
"""
import collections
import itertools
import math
from fractions import Fraction

import numpy as np

import icp_reference as R
import projection_reference as PR

INFO_ROW = 80
LOSS_PO2PO, LOSS_PO2PL, LOSS_PL2PL, NORMAL_LINEAR = R.LOSS_PO2PO, R.LOSS_PO2PL, R.LOSS_PL2PL, R.NORMAL_LINEAR


def skew(v):
    x, y, z = v
    return np.array([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]])


def exp_se3(xi):
    """4 x 4 float64 Exp of xi = (rho, phi)."""
    rho, phi = np.asarray(xi[:3], np.float64), np.asarray(xi[3:], np.float64)
    th = np.linalg.norm(phi)
    K = skew(phi)
    if th < 1e-12:
        Rm, V = np.eye(3) + K, np.eye(3) + 0.5 * K
    else:
        Rm = np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K
        V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * K + (th - np.sin(th)) / th ** 3 * K @ K
    out = np.eye(4)
    out[:3, :3], out[:3, 3] = Rm, V @ rho
    return out


def pair_masks(T, p, m, tgt_n, tgt_has, nn, flags):
    """Per source: kind 0 none, 1 (normal, normal), 2 po2po, as the losses keep them (rotated source normal non-zero,
    target has-normal flag; po2po pairs only with LOSS_PO2PO)."""
    _, ns = R.apply_rigid(T, p, m)
    src_has = np.any(ns != 0, axis=1)
    paired = nn >= 0
    t_has = np.zeros(len(p), bool)
    t_has[paired] = tgt_has[nn[paired]]
    kind = np.zeros(len(p), np.int64)
    kind[paired & src_has & t_has] = 1
    if flags & LOSS_PO2PO:
        kind[paired & ~src_has & ~t_has] = 2
    return kind


def jacobians(T, p, m, n_t, kind, flags):
    """Per kept pair: list of (term, J [k, 6] float64), term in {'po2pl', 'pl2pl', 'po2po'}."""
    T = np.asarray(T, np.float32).reshape(3, 4).astype(np.float64)
    Rm = T[:, :3]
    out = []
    p, m, n_t = (np.asarray(a, np.float32).astype(np.float64) for a in (p, m, n_t))
    if kind == 1:
        if flags & LOSS_PO2PL:
            out.append(("po2pl", (n_t @ np.hstack([Rm, -Rm @ skew(p)]))[None, :]))
        if flags & LOSS_PL2PL:
            if flags & NORMAL_LINEAR:
                out.append(("pl2pl", np.hstack([np.zeros(3), n_t @ Rm @ skew(m)])[None, :]))
            else:
                out.append(("pl2pl", np.hstack([np.zeros((3, 3)), -Rm @ skew(m)])))
    elif kind == 2:
        out.append(("po2po", np.hstack([Rm, -Rm @ skew(p)])))
    return out


def term_jacobians(T, p, m, n_t, kind, flags):
    """The Jacobians of every kept pair at once: {term: J [n, k, 6] float64} over the pairs with kind 1 ('po2pl',
    'pl2pl') or kind 2 ('po2po'), in source order; the same matrices as `jacobians`."""
    T = np.asarray(T, np.float32).reshape(3, 4).astype(np.float64)
    Rm = T[:, :3]
    p, m, n_t = (np.asarray(a, np.float32).reshape(-1, 3).astype(np.float64) for a in (p, m, n_t))
    kind = np.asarray(kind).reshape(-1)

    def skews(v):
        out = np.zeros((len(v), 3, 3))
        out[:, 0, 1], out[:, 0, 2], out[:, 1, 2] = -v[:, 2], v[:, 1], -v[:, 0]
        return out - out.transpose(0, 2, 1)

    out = {}
    b, c = kind == 1, kind == 2
    if b.any():
        if flags & LOSS_PO2PL:
            full = np.concatenate([np.broadcast_to(Rm, (int(b.sum()), 3, 3)), -Rm @ skews(p[b])], axis=2)
            out["po2pl"] = np.einsum("na,nab->nb", n_t[b], full)[:, None, :]
        if flags & LOSS_PL2PL:
            rot = Rm @ skews(m[b])
            if flags & NORMAL_LINEAR:
                out["pl2pl"] = np.concatenate([np.zeros((int(b.sum()), 3)), np.einsum("na,nab->nb", n_t[b], rot)],
                                              axis=1)[:, None, :]
            else:
                out["pl2pl"] = np.concatenate([np.zeros((int(b.sum()), 3, 3)), -rot], axis=2)
    if c.any():
        out["po2po"] = np.concatenate([np.broadcast_to(Rm, (int(c.sum()), 3, 3)), -Rm @ skews(p[c])], axis=2)
    return out


def _kept(T, p, m, tgt_n, tgt_has, nn, flags):
    p = np.asarray(p, np.float32).reshape(-1, 3)
    m = np.asarray(m, np.float32).reshape(-1, 3)
    tgt_n = np.asarray(tgt_n, np.float32).reshape(-1, 3)
    tgt_has = np.asarray(tgt_has, bool).reshape(-1)
    nn = np.asarray(nn, np.int64).reshape(-1)
    kind = pair_masks(T, p, m, tgt_n, tgt_has, nn, flags)
    n_t = np.zeros_like(p)
    n_t[kind > 0] = tgt_n[nn[kind > 0]]
    return p, m, n_t, kind


def term_sums(T, p, m, tgt_n, tgt_has, nn, flags):
    """-> ({term: sum of J^T J [6, 6] float64}, M, M'): the unweighted sums of the three terms (zero for a term the
    flags leave out), the sums the kernels accumulate."""
    p, m, n_t, kind = _kept(T, p, m, tgt_n, tgt_has, nn, flags)
    S = dict.fromkeys(("po2pl", "pl2pl", "po2po"))
    J = term_jacobians(T, p, m, n_t, kind, flags)
    for term in S:
        S[term] = np.einsum("nka,nkb->ab", J[term], J[term]) if term in J else np.zeros((6, 6))
    return S, int((kind == 1).sum()), int((kind == 2).sum())


def weights(M, Mp, flags, lam):
    """The three terms' float64 weights as icp_info_finalize_kernel forms them: 2 lam / M, 2 / M, 2 / (3 M')."""
    lam = float(np.float32(lam))
    w_pl = 2.0 * lam / float(M) if M > 0 and flags & LOSS_PO2PL else 0.0
    w_nn = 2.0 / float(M) if M > 0 and flags & LOSS_PL2PL else 0.0
    w_pp = 2.0 / (3.0 * float(Mp)) if Mp > 0 and flags & LOSS_PO2PO else 0.0
    return w_pl, w_nn, w_pp


def information(T, p, m, tgt_n, tgt_has, nn, flags, lam=1.0):
    """-> (H [6, 6] float64, A [6, 6] float64, M, M').  A is the same weighted sum with every |J_i J_j| replaced by
    s_i s_j, s = (1, 1, 1, |p|, |p|, |p|) per Jacobian row: the magnitude the kernels' fp32 rounding is relative to."""
    p, m, n_t, kind = _kept(T, p, m, tgt_n, tgt_has, nn, flags)
    M, Mp = int((kind == 1).sum()), int((kind == 2).sum())
    w = dict(zip(("po2pl", "pl2pl", "po2po"), weights(M, Mp, flags, lam)))
    H, A = np.zeros((6, 6)), np.zeros((6, 6))
    r = np.maximum(1.0, np.linalg.norm(p.astype(np.float64), axis=1))
    for term, J in term_jacobians(T, p, m, n_t, kind, flags).items():
        H += w[term] * np.einsum("nka,nkb->ab", J, J)
        rows = r[kind == 1] if term != "po2po" else r[kind == 2]
        sc = np.stack([np.ones_like(rows)] * 3 + [rows] * 3, axis=1)
        A += w[term] * J.shape[1] * np.einsum("na,nb->ab", sc, sc)
    return H, A, M, Mp


def _fma(a, b, c):
    """float64 a * b + c rounded once (Fraction is exact; its float() rounds to nearest, ties to even)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def kernel_order(S, M, Mp, flags, lam=1.0, factor=None):
    """H as icp_info_finalize_kernel evaluates it from exact sums S (term_sums): per entry
    h = fma(w_pp, S_po2po, fma(w_nn, S_pl2pl, w_pl * S_po2pl)) in float64 (the contraction nvcc makes of
    w_pl * S1 + w_nn * S2 + w_pp * S3), with the scaled operator's h *= 1 / f once per translation index.
    -> (the float64 H the kernel solves, its fp32 rounding: the row's H)."""
    w_pl, w_nn, w_pp = weights(M, Mp, flags, lam)
    inv_f = 1.0 / float(np.float32(factor)) if factor is not None else 1.0
    H = np.zeros((6, 6))
    for i in range(6):
        for j in range(i, 6):
            h = _fma(w_pp, S["po2po"][i, j], _fma(w_nn, S["pl2pl"][i, j], w_pl * S["po2pl"][i, j]))
            if factor is not None:
                if i < 3:
                    h *= inv_f
                if j < 3:
                    h *= inv_f
            H[i, j] = H[j, i] = h
    return H, H.astype(np.float32)


def objective(T, xi, p, m, tgt_p, tgt_n, kind, nn, flags, lam=1.0):
    """po2po + lam po2pl + pl2pl in float64 at T Exp(xi) with the correspondences held fixed."""
    T4 = np.eye(4)
    T4[:3, :] = np.asarray(T, np.float64).reshape(3, 4)
    Tx = T4 @ exp_se3(xi)
    Rm, t = Tx[:3, :3], Tx[:3, 3]
    p, m, tgt_p, tgt_n = (np.asarray(a, np.float64) for a in (p, m, tgt_p, tgt_n))
    s = p @ Rm.T + t
    ns = m @ Rm.T
    f = 0.0
    b = kind == 1
    if b.any():
        q, n = tgt_p[nn[b]], tgt_n[nn[b]]
        M = b.sum()
        if flags & LOSS_PO2PL:
            f += lam * np.mean(np.sum((s[b] - q) * n, axis=1) ** 2)
        if flags & LOSS_PL2PL:
            if flags & NORMAL_LINEAR:
                f += np.sum((1.0 - np.sum(ns[b] * n, axis=1)) ** 2) / M
            else:
                f += np.sum((ns[b] - n) ** 2) / M
    c = kind == 2
    if c.any():
        f += np.mean((s[c] - tgt_p[nn[c]]) ** 2)
    return f


def residuals(T, xi, p, m, tgt_p, tgt_n, kind, nn, flags, lam=1.0):
    """The objective's residuals at T Exp(xi), each scaled by the square root of its weight, so that
    objective = sum(residuals ** 2) and its Gauss-Newton Hessian is 2 J^T J of this vector."""
    T4 = np.eye(4)
    T4[:3, :] = np.asarray(T, np.float64).reshape(3, 4)
    Tx = T4 @ exp_se3(xi)
    Rm, t = Tx[:3, :3], Tx[:3, 3]
    p, m, tgt_p, tgt_n = (np.asarray(a, np.float64) for a in (p, m, tgt_p, tgt_n))
    s, ns = p @ Rm.T + t, m @ Rm.T
    out = []
    b, c = kind == 1, kind == 2
    M, Mp = b.sum(), c.sum()
    if M:
        q, n = tgt_p[nn[b]], tgt_n[nn[b]]
        if flags & LOSS_PO2PL:
            out.append(np.sqrt(lam / M) * np.sum((s[b] - q) * n, axis=1))
        if flags & LOSS_PL2PL:
            if flags & NORMAL_LINEAR:
                out.append(np.sqrt(1.0 / M) * (1.0 - np.sum(ns[b] * n, axis=1)))
            else:
                out.append(np.sqrt(1.0 / M) * (ns[b] - n).reshape(-1))
    if Mp:
        out.append(np.sqrt(1.0 / (3 * Mp)) * (s[c] - tgt_p[nn[c]]).reshape(-1))
    return np.concatenate(out) if out else np.zeros(0)


def fd_jacobian(fun, h=1e-6):
    """Central first differences of fun: R^6 -> R^k at 0, as [k, 6]."""
    E = np.eye(6) * h
    return np.stack([(fun(E[i]) - fun(-E[i])) / (2 * h) for i in range(6)], axis=1)


def fd_hessian(fun, h=1e-4):
    """Central second differences of fun: R^6 -> R at 0."""
    H = np.zeros((6, 6))
    E = np.eye(6) * h
    for i in range(6):
        for j in range(i, 6):
            H[i, j] = H[j, i] = (fun(E[i] + E[j]) - fun(E[i] - E[j]) - fun(-E[i] + E[j]) + fun(-E[i] - E[j])) / (4 * h * h)
    return H


def eig_row(H):
    """Eigenvalues ascending and unit eigenvectors (rows) of H with the kernels' sign convention: each eigenvector's
    largest-magnitude component (the first of equals) positive."""
    ev, V = np.linalg.eigh(H)
    V = V.T.copy()
    for k in range(6):
        big = int(np.argmax(np.abs(V[k])))
        if V[k, big] < 0:
            V[k] = -V[k]
    return ev, V


# ------------------------------------------------------------------------------------------------ exact designs
# Integer source points p, each alone in its pixel; targets T p with T a signed permutation rotation and an integer
# translation, so every source's NN is its twin at distance 0; axis-aligned unit normals.  Every Jacobian entry is then
# a small integer and every fp32 sum the kernels form is exact, so the row's H is kernel_order(term_sums(...)) bit for
# bit.  Point sets closed under a symmetry group zero the off-diagonal sums: p -> -p zeroes the translation-rotation
# block, the 8 sign flips every off-diagonal entry, the 48 signed permutations make the po2po H two exact triples.
DESIGN_GRID = (32, 360, (math.radians(-179.9), math.radians(179.9)), (math.radians(-60.0), math.radians(60.0)))
DESIGN_T = np.array([[0, -1, 0, 3], [1, 0, 0, -2], [0, 0, 1, 1]], np.float32)      # yaw 90 deg, (3, -2, 1) m
AXES = np.eye(3, dtype=np.float32)
Design = collections.namedtuple("Design", "name flags lam T p m tgt_p tgt_n tgt_has")


def _group(kind):
    if kind == "one":
        return [np.eye(3)]
    if kind == "centro":
        return [np.eye(3), -np.eye(3)]
    flips = [np.diag(s) for s in itertools.product((1, -1), repeat=3)]
    if kind == "flips":
        return flips
    perms = [np.eye(3)[list(q)] for q in itertools.permutations(range(3))]
    return [f @ q for f in flips for q in perms]                                    # "cubic": 48 signed permutations


def _orbits(gen, group, n_orbits, lo=2, hi=12, z_hi=6, distinct=False):
    """Up to n_orbits orbits of integer points (no zero coordinate, nor in T p) whose sources and targets all own
    their pixels of DESIGN_GRID."""
    h, w, hf, vf = DESIGN_GRID
    g = PR.Grid(h, w, hf, vf)
    Rm, t = DESIGN_T[:, :3].astype(np.float64), DESIGN_T[:, 3].astype(np.float64)
    used_s, used_t, out = set(), set(), []
    for _ in range(4000):
        if len(out) == n_orbits:
            break
        base = gen.integers(lo, hi + 1, 3) * gen.choice([-1, 1], 3)
        base[2] = gen.integers(1, z_hi + 1) * gen.choice([-1, 1])
        if distinct and len(set(np.abs(base).tolist())) < 3:
            continue
        pts = np.unique(np.stack([q @ base for q in group]), axis=0)
        tgt = pts @ Rm.T + t
        if (pts == 0).any() or (tgt == 0).any():
            continue
        ps = PR.pixels(g, *PR.coords(g, *pts.T.astype(np.float32))[:2])
        pt = PR.pixels(g, *PR.coords(g, *tgt.T.astype(np.float32))[:2])
        if (ps < 0).any() or (pt < 0).any() or len(set(ps.tolist())) < len(ps) or len(set(pt.tolist())) < len(pt):
            continue
        if used_s & set(ps.tolist()) or used_t & set(pt.tolist()):
            continue
        used_s |= set(ps.tolist())
        used_t |= set(pt.tolist())
        out.append(pts)
    assert len(out) == n_orbits, f"only {len(out)} of {n_orbits} orbits fit the grid"
    return out


def exact_design(name, seed=0, lam=1.0):
    """The designs of tests/test_gpu_icp_information_exact.py:
      tie     po2pl, 8-flip orbits, 4 with x normals, 4 with y, 2 with z: H diagonal, its translation diagonal
              (b, b, a) with a < b below the rotation diagonal (two equal eigenvalues, then a smaller one);
      triple  po2po, 48-fold cubic orbits: H = diag(c, c, c, d, d, d), two exact triples;
      zeros   pl2pl (J does not read p): the translation block exactly 0 (three exact zeros), the rotation block
              diagonal;
      near    po2pl + pl2pl, centrosymmetric orbits, n_x = n_y source normals: the pl2pl rotation diagonal has a tie
              in (rot x, rot y) that lam times the po2pl rotation block (not diagonal) splits;
      mixed   every term: points with a normal on both sides, on neither, and on one side only, no symmetry.
    Target normals are R m (the source normals' twins) except in `mixed`, where they are drawn independently."""
    gen = np.random.default_rng(seed)
    counts = {"tie": [4, 4, 2], "zeros": [3, 5, 2], "near": [3, 3, 6]}
    if name == "triple":
        orbits = _orbits(gen, _group("cubic"), 3, 4, 10, 10, distinct=True)
        normal = [np.zeros(3, np.float32)] * 3
    elif name == "mixed":
        orbits = _orbits(gen, _group("one"), 120)
        cat = np.arange(120) % 4                                   # 0 both, 1 neither, 2 source only, 3 target only
        normal = [AXES[gen.integers(3)] * gen.choice([-1, 1]) if c in (0, 2) else np.zeros(3, np.float32) for c in cat]
    else:
        n_axis = counts[name]
        group = _group("centro" if name == "near" else "flips")
        orbits = _orbits(gen, group, sum(n_axis), z_hi=6 if name != "tie" else 4)
        axis = np.repeat(np.arange(3), n_axis)
        normal = [AXES[a] for a in axis]
    p = np.concatenate(orbits).astype(np.float32)
    m = np.concatenate([np.broadcast_to(n, (len(o), 3)) for n, o in zip(normal, orbits)]).astype(np.float32)
    Rm = DESIGN_T[:, :3].astype(np.float64)
    tgt_p = (p.astype(np.float64) @ Rm.T + DESIGN_T[:, 3].astype(np.float64)).astype(np.float32)
    tgt_n = (m.astype(np.float64) @ Rm.T).astype(np.float32)
    if name == "mixed":
        tgt_n = np.zeros_like(m)
        first = np.cumsum([0] + [len(o) for o in orbits])[:-1]
        for k, c in enumerate(cat):
            if c in (0, 3):
                tgt_n[first[k]] = AXES[gen.integers(3)] * gen.choice([-1, 1])
    flags = {"tie": LOSS_PO2PL, "triple": R.LOSS_PO2PO, "zeros": LOSS_PL2PL, "near": LOSS_PO2PL | LOSS_PL2PL,
             "mixed": R.LOSS_PO2PO | LOSS_PO2PL | LOSS_PL2PL}[name]
    tgt_has = np.any(tgt_n != 0, axis=1)
    return Design(name, flags, float(np.float32(lam)), DESIGN_T.copy(), p, m, tgt_p, tgt_n, tgt_has)


def design_sums(d, flags=None):
    """term_sums of a design with every source paired with its twin."""
    return term_sums(d.T, d.p, d.m, d.tgt_n, d.tgt_has, np.arange(len(d.p)), d.flags if flags is None else flags)


def near_tie_lambda(d, ratio):
    """lam (fp32) that splits the `near` design's tied pl2pl rotation eigenvalues by about ratio of the largest: the
    split is lam times that of the po2pl rotation block's (rot x, rot y) part."""
    S, M, Mp = design_sums(d)
    A = S["po2pl"][3:5, 3:5] * (2.0 / M)
    split = math.hypot(A[0, 0] - A[1, 1], 2.0 * A[0, 1])
    top = S["pl2pl"][3, 3] * (2.0 / M)
    return float(np.float32(ratio * top / split))
