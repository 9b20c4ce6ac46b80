"""Exact nearest-neighbour reference for the ICP operators (test infrastructure, CPU only).

The operators promise the exact Euclidean nearest neighbour of every fp32 source point among fp32 targets, the lowest
pixel id on exact ties (include/delora_b200.h).  `nearest` computes that answer with no rounding at all:
  - cKDTree (float64) proposes the k nearest targets of every source;
  - every candidate whose float64 squared distance lies within REL_BAND of the smallest one is re-measured exactly:
    fp32 values are dyadic rationals, so (s - t)^2 summed over Fractions is the true squared distance;
  - the smallest exact distance wins, the lowest id among equals.
If all k candidates of a source fall inside the band, that source asks for four times as many until one falls
outside, so that no target inside the band is missed.

Besides the answer it reports, per source, how many targets share the exact minimum (an exact tie) and the relative
separation of the exact second-best distance.  A separation in (0, 2^-45) is UNSAFE: a correct float64 ranking (the
kernels' nn_d2_exact, which nvcc may contract to DFMA) can round either way there, so a scene meant to have one right
answer must keep such cases out.  `Result.unsafe` lists them.
"""
import collections
from fractions import Fraction

import numpy as np
import scipy.spatial

REL_BAND = 1e-9            # float64 candidates this close to the best are re-measured exactly
UNSAFE_SEP = 2.0 ** -45    # exact separations below this are left to float64 rounding

Result = collections.namedtuple("Result", "nn ties sep unsafe")
Result.__doc__ = """nn [Ns] int64: id of the exact nearest target (-1 without targets);  ties [Ns] int64: number of
targets at exactly that distance (1 = no tie);  sep [Ns] float64: relative separation of the second-best distance,
(d2_second - d2_best) / d2_best (exact when it is below REL_BAND, float64 otherwise; inf with one target);
unsafe: indices of the sources with 0 < sep < 2^-45."""


def exact_d2(s, t):
    """Exact squared distance of two fp32 3-vectors, as a Fraction."""
    return sum((Fraction(float(a)) - Fraction(float(b))) ** 2 for a, b in zip(s, t))


def _resolve(s, cand, tgt, ids):
    """Exact ranking of candidate rows `cand` for source s -> (best id, tie count, exact relative separation)."""
    d = sorted((exact_d2(s, tgt[j]), int(ids[j])) for j in cand)
    best, bid = d[0]
    ties = sum(1 for x, _ in d if x == best)
    rest = [x for x, _ in d if x != best]
    if not rest:
        sep = np.inf
    elif best == 0:
        sep = np.inf
    else:
        sep = float((rest[0] - best) / best)
    return bid, ties, sep


def nearest(targets, ids, sources, k=8):
    """targets [Nt,3] fp32, ids [Nt] int (pixel ids, distinct), sources [Ns,3] fp32 -> Result."""
    tgt = np.ascontiguousarray(targets, np.float32).reshape(-1, 3)
    src = np.ascontiguousarray(sources, np.float32).reshape(-1, 3)
    ids = np.asarray(ids, np.int64).reshape(-1)
    ns, nt = len(src), len(tgt)
    assert len(ids) == nt and len(np.unique(ids)) == nt, "target ids must be distinct"
    if nt == 0 or ns == 0:
        return Result(np.full(ns, -1, np.int64), np.zeros(ns, np.int64), np.full(ns, np.inf), np.zeros(0, np.int64))
    t64, s64 = tgt.astype(np.float64), src.astype(np.float64)
    k = min(k, nt)
    tree = scipy.spatial.cKDTree(t64)
    _, idx = tree.query(s64, k=k)
    idx = idx.reshape(ns, k)
    d2 = ((s64[:, None, :] - t64[idx]) ** 2).sum(-1)          # float64 on the candidates, in a fixed order
    order = np.argsort(d2, axis=1, kind="stable")
    idx = np.take_along_axis(idx, order, 1)
    d2 = np.take_along_axis(d2, order, 1)
    nn = ids[idx[:, 0]].copy()
    ties = np.ones(ns, np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        sep = (d2[:, 1] - d2[:, 0]) / d2[:, 0] if k > 1 else np.full(ns, np.inf)
    sep = np.where(np.isnan(sep), np.inf, sep)
    in_band = d2 <= d2[:, :1] * (1.0 + REL_BAND)
    for i in np.nonzero(in_band[:, 1:].any(axis=1) if k > 1 else np.zeros(ns, bool))[0]:
        ci, cd, kk = idx[i], d2[i], k
        while (cd <= cd[0] * (1.0 + REL_BAND)).all() and kk < nt:  # the band may hold more than kk targets
            kk = min(nt, 4 * kk)
            ci = np.atleast_1d(tree.query(s64[i], k=kk)[1])
            cd = ((s64[i] - t64[ci]) ** 2).sum(-1)
            o = np.argsort(cd, kind="stable")
            ci, cd = ci[o], cd[o]
        n_in = int((cd <= cd[0] * (1.0 + REL_BAND)).sum())
        cand = list(ci[:n_in + 1])                             # the band, and the first target beyond it
        nn[i], ties[i], sep[i] = _resolve(src[i], cand, tgt, ids)
    unsafe = np.nonzero((sep > 0) & (sep < UNSAFE_SEP))[0]
    return Result(nn, ties, sep, unsafe)


# ---- the normal-code fingerprint ---------------------------------------------------------------------------------
# With flags = LOSS_PL2PL (squared normal loss), T = identity, every target carrying has-normal = 1 and a small
# integer code normal q_j, and every source an integer normal m_i in {-1, 0, 1}^3 \ {0}, the pair term of the
# gradient columns kColGnM is the integer matrix (m_i - q_nn(i)) m_i^T.  The kernels' fp32 warp sums and fp64 column
# sums of integers below 2^24 are exact, so the nine sums equal S = sum_i (m_i - q_nn(i)) m_i^T exactly, and the
# finalize turns them into grad_T[:, :3] = (2 rn(1 / M)) S in fp32, grad_T[:, 3] = 0 (csrc/icp.cu, icp_finalize_kernel).
# While every |S| < 2^22 a change of one in any sum changes its fp32 gradient entry: a wrong neighbour shows unless
# its code equals the right one in all three components.

def code_normals(n, seed, c=7):
    """[n, 3] fp32 integer codes in [-c, c]^3 from a seed."""
    return np.random.default_rng(seed).integers(-c, c + 1, (n, 3)).astype(np.float32)


def source_normals(n, seed):
    """[n, 3] fp32 integer normals in {-1, 0, 1}^3 without the zero vector, from a seed."""
    m = np.random.default_rng(seed).integers(-1, 2, (n, 3))
    zero = ~m.any(axis=1)
    m[zero, np.arange(n)[zero] % 3] = 1
    return m.astype(np.float32)


def code_sums(m, q_nn):
    """Exact S = sum_i (m_i - q_nn(i)) m_i^T as int64 [3, 3] (rows: the normal's component, columns: m's)."""
    m = np.asarray(m, np.float64).astype(np.int64)
    d = m - np.asarray(q_nn, np.float64).astype(np.int64)
    return np.einsum("ia,ib->ab", d, m)


def fingerprint(S, M):
    """grad_T [12] fp32 the finalize computes from exact column sums S [3, 3] and M pairs: (2 rn(1/M)) S."""
    S = np.asarray(S, np.int64)
    assert np.abs(S).max(initial=0) < 2 ** 22, "code sums must stay below 2^22 to be seen one by one"
    k = np.float32(2.0) * (np.float32(1.0) / np.float32(M)) if M > 0 else np.float32(0.0)
    g = np.zeros((3, 4), np.float32)
    g[:, :3] = k * S.astype(np.float32)
    return g.reshape(12)


def finalize_model(m, ns, q, paired, warp=32):
    """A Python model of what the dense and CSR kernels do with (source normal m, rotated normal ns, matched target
    code q) under LOSS_PL2PL: per-pair columns (ns - q) m^T in fp32, fp32 sums over groups of `warp` consecutive
    sources (unpaired lanes add zeros), fp64 sums of those, rounded to fp32, then the finalize's
    k_pl * 0 + k_nn * S + k_pp * 0 with k_nn = 2 rn(1/M).  -> grad_T [12] fp32, M."""
    m, ns, q = (np.asarray(a, np.float32) for a in (m, ns, q))
    paired = np.asarray(paired, bool)
    h = np.where(paired[:, None], ns - q, np.float32(0)).astype(np.float32)
    terms = (h[:, :, None] * np.where(paired[:, None], m, np.float32(0))[:, None, :]).astype(np.float32)
    sums = np.zeros((3, 3), np.float64)
    for w0 in range(0, len(m), warp):
        part = np.zeros((3, 3), np.float32)
        for t in terms[w0:w0 + warp]:
            part = (part + t).astype(np.float32)
        sums += part.astype(np.float64)
    S = sums.astype(np.float32)
    M = np.float32(paired.sum())
    inv_m = np.float32(1.0) / M if M > 0 else np.float32(0.0)
    k_nn = np.float32(2.0) * inv_m
    g = np.zeros((3, 4), np.float32)
    g[:, :3] = (np.float32(0.0) + k_nn * S).astype(np.float32)
    return g.reshape(12), int(M)
