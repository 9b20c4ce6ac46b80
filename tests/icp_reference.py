"""Float64 reference of the ICP operators (delora_icp_fwd_bwd, delora_icp_dense_fwd_bwd, delora_icp_point_grads) for
every loss configuration (test infrastructure, imported like helpers).

What it restates, per scan pair (include/delora_b200.h, delora_b200/csrc/icp_common.cuh):
  - the transform s = R p + t and n_s = R m exactly as the kernels round it (apply_rigid: an fmaf chain, then + t, in
    fp32).  Python has no fmaf; fmaf(a, b, c) is emulated as float32(float64(a) * float64(b) + float64(c)): the product
    of two fp32 numbers is exact in float64, so the only departure from a single rounding is a double rounding when the
    float64 sum lands exactly on a float32 midpoint (about one operation in 2^28, and then by one ulp).
  - the nearest neighbour of every transformed source point: oracle.delora_oracle.nearest_neighbors (cKDTree, the
    exact float64 Euclidean NN the kernels promise).
  - the masks: the source has a normal iff its ROTATED normal is non-zero, the target iff its has-normal flag is set;
    a (normal, normal) pair counts in M, a pair without a normal on either side is a po2po pair and counts in M' only
    when LOSS_PO2PO is set.
  - the `losses` row: the three unweighted means in float64 on the fp32 transformed points (po2po is the mean over the
    3 M' coordinates); a loss whose bit is not set is 0.
  - grad_T = d(po2po + lambda po2pl + pl2pl) / d(R | t) and the per-point gradients of g0 po2po + g1 po2pl + g2 pl2pl,
    by torch autograd in float64 with the NN and the masks held fixed.

One deliberate divergence from torch: a mean over an empty set (M = 0, or M' = 0) is 0 here, and so are its gradient
terms, because that is what the operators document (torch's MSELoss would return NaN).
"""
import collections

import numpy as np
import torch

from oracle import delora_oracle as orc

LOSS_PO2PO, LOSS_PO2PL, LOSS_PL2PL, NORMAL_LINEAR = 1, 2, 4, 8


def flag_matrix():
    """The 7 non-empty subsets of {PO2PO, PO2PL, PL2PL}, and the 4 with PL2PL once more with NORMAL_LINEAR: 11 sets."""
    out = []
    for bits in range(1, 8):
        f = (LOSS_PO2PO if bits & 1 else 0) | (LOSS_PO2PL if bits & 2 else 0) | (LOSS_PL2PL if bits & 4 else 0)
        out.append(f)
        if f & LOSS_PL2PL:
            out.append(f | NORMAL_LINEAR)
    return out


def flag_name(flags):
    names = [n for bit, n in ((LOSS_PO2PO, "po2po"), (LOSS_PO2PL, "po2pl"), (LOSS_PL2PL, "pl2pl"),
                              (NORMAL_LINEAR, "linear")) if flags & bit]
    return "+".join(names)


def fmaf(a, b, c):
    """fp32 fused multiply-add, emulated in float64 (see the module docstring)."""
    return (np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
            + np.asarray(c, np.float32).astype(np.float64)).astype(np.float32)


def apply_rigid(T, p, m):
    """The kernels' transform (icp_common.cuh apply_rigid).  T [3,4] (or [12]) fp32, p, m [N,3] fp32 ->
    s = R p + t, n_s = R m as [N,3] fp32 arrays: fmaf(r2, z, fmaf(r1, y, r0 * x)), then + t."""
    T = np.asarray(T, np.float32).reshape(3, 4)
    p = np.asarray(p, np.float32)
    m = np.asarray(m, np.float32)

    def rot(v, k):
        return fmaf(T[k, 2], v[:, 2], fmaf(T[k, 1], v[:, 1], T[k, 0] * v[:, 0]))

    s = np.stack([rot(p, k) + T[k, 3] for k in range(3)], axis=1)
    ns = np.stack([rot(m, k) for k in range(3)], axis=1)
    return s.astype(np.float32), ns.astype(np.float32)


Pair = collections.namedtuple("Pair", "p m s ns tgt_p tgt_n tgt_has nn src_has")


def prepare(src_p, src_n, T, tgt_p, tgt_n, tgt_has, nn=None):
    """One scan pair, ready for evaluate(): the flag-independent part (transform, NN, masks).

    src_p, src_n [N,3] fp32: source points / normals BEFORE the transform;  T [3,4] fp32, or None when the source is
    already transformed (the drop-in path);  tgt_p, tgt_n [Nt,3] fp32, tgt_has [Nt] bool.  nn: precomputed NN indices
    into the target list, or None to run cKDTree."""
    src_p = np.asarray(src_p, np.float32).reshape(-1, 3)
    src_n = np.asarray(src_n, np.float32).reshape(-1, 3)
    tgt_p = np.asarray(tgt_p, np.float32).reshape(-1, 3)
    tgt_n = np.asarray(tgt_n, np.float32).reshape(-1, 3)
    tgt_has = np.asarray(tgt_has, bool).reshape(-1)
    if T is None:
        s, ns = src_p, src_n
    else:
        s, ns = apply_rigid(T, src_p, src_n)
    if nn is None:
        nn = orc.nearest_neighbors(tgt_p, s) if len(tgt_p) else np.full(len(s), -1, np.int64)
    nn = np.asarray(nn, np.int64)
    src_has = (ns != 0).any(axis=1)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))   # noqa: E731
    return Pair(d(src_p), d(src_n), d(s), d(ns), d(tgt_p), d(tgt_n), torch.from_numpy(tgt_has), torch.from_numpy(nn),
                torch.from_numpy(src_has))


def _masks(pr, flags):
    if len(pr.tgt_p) == 0 or len(pr.s) == 0:
        none = torch.zeros(len(pr.s), dtype=torch.bool)
        return none, none
    th = pr.tgt_has[pr.nn]
    both = pr.src_has & th
    po2po = (~pr.src_has & ~th) if flags & LOSS_PO2PO else torch.zeros_like(both)
    return both, po2po


def _losses(pr, flags, s, ns):
    """(po2po, po2pl, pl2pl) as float64 tensors, differentiable in s and ns; M, M' as ints."""
    both, pp = _masks(pr, flags)
    M, Mp = int(both.sum()), int(pp.sum())
    zero = s.sum() * 0.0 + ns.sum() * 0.0          # an empty set's 0, still a function of s and ns (gradient 0)
    po2po = po2pl = pl2pl = zero
    if M == 0 and Mp == 0:
        return (po2po, po2pl, pl2pl), M, Mp
    nn = pr.nn.clamp_min(0)
    t, q = pr.tgt_p[nn], pr.tgt_n[nn]
    d = s - t
    if Mp:
        po2po = (d[pp] ** 2).sum() / (3.0 * Mp)
    if M:
        if flags & LOSS_PO2PL:
            r = (d[both] * q[both]).sum(dim=1)
            po2pl = (r ** 2).sum() / M
        if flags & LOSS_PL2PL:
            if flags & NORMAL_LINEAR:
                pl2pl = ((1.0 - (ns[both] * q[both]).sum(dim=1)) ** 2).sum() / M
            else:
                pl2pl = ((ns[both] - q[both]) ** 2).sum() / M
    return (po2po, po2pl, pl2pl), M, Mp


def objective(pr, flags, lam, dT):
    """po2po + lam po2pl + pl2pl at T0 + dT ([3,4] float64), as the kernel's fp32 transformed points plus the exact
    first-order change (s and n_s are affine in T, so this has the true derivative w.r.t. R | t at every dT)."""
    s = pr.s + pr.p @ dT[:, :3].T + dT[:, 3]
    ns = pr.ns + pr.m @ dT[:, :3].T
    (po2po, po2pl, pl2pl), _, _ = _losses(pr, flags, s, ns)
    return po2po + lam * po2pl + pl2pl


Result = collections.namedtuple("Result", "losses M Mp grad_T grad_pts grad_nrm")


def evaluate(pr, flags, lam=1.0, upstream=None):
    """-> Result: losses [3] float64 numpy (po2po, po2pl, pl2pl), M, M', grad_T [3,4] float64 numpy, and with
    upstream = (g_po2po, g_po2pl, g_pl2pl) the per-point gradients of g . losses w.r.t. the transformed source points
    and normals, [N,3] float64 numpy each (else None)."""
    (po2po, po2pl, pl2pl), M, Mp = _losses(pr, flags, pr.s, pr.ns)
    losses = np.array([float(po2po), float(po2pl), float(pl2pl)])
    dT = torch.zeros((3, 4), dtype=torch.float64, requires_grad=True)
    grad_T = torch.autograd.grad(objective(pr, flags, float(lam), dT), dT)[0].numpy()
    gp = gn = None
    if upstream is not None:
        s, ns = pr.s.clone().requires_grad_(True), pr.ns.clone().requires_grad_(True)
        lo, _, _ = _losses(pr, flags, s, ns)
        total = sum(float(g) * x for g, x in zip(upstream, lo))
        gp, gn = (x.numpy() for x in torch.autograd.grad(total, (s, ns)))
    return Result(losses, M, Mp, grad_T, gp, gn)
