"""The exact nearest-neighbour reference (tests/nn_reference.py) and the normal-code fingerprint, on the CPU.

  - on random clouds the reference equals float64 brute force (oracle.delora_oracle.nearest_neighbors "brute");
  - on hand-made exact ties (2 to 8 targets at one exact distance, ids in arbitrary order) it returns the lowest id and
    counts the tie;  on ties that exist only in exact arithmetic (coordinate permutations whose naive float64 sums
    round differently) it still sees the tie;  near ties below 2^-45 are reported as unsafe;
  - the restated fingerprint (2 rn(1/M)) S equals a Python model of the kernels' accumulation and finalize.
"""
import itertools

import numpy as np
import pytest

import nn_reference as NR
from oracle import delora_oracle as orc


def naive_d2(s, t):
    e = np.asarray(s, np.float64) - np.asarray(t, np.float64)
    return (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]


@pytest.mark.parametrize("seed", range(4))
def test_reference_equals_brute_force(seed):
    gen = np.random.default_rng(seed)
    nt, ns = [(1, 50), (7, 300), (500, 400), (3000, 2000)][seed]
    tgt = (gen.standard_normal((nt, 3)) * gen.uniform(0.1, 30.0)).astype(np.float32)
    src = (gen.standard_normal((ns, 3)) * 10.0).astype(np.float32)
    ids = np.arange(nt) * 3 + 5                             # increasing: brute force's lowest index is the lowest id
    res = NR.nearest(tgt, ids, src)
    want = ids[orc.nearest_neighbors(tgt, src, "brute")]
    assert np.array_equal(res.nn, want)
    assert len(res.unsafe) == 0 and (res.ties == 1).all()


@pytest.mark.parametrize("k", range(2, 9))
def test_exact_ties_take_the_lowest_id(k):
    """k targets at the same exact distance: sign and axis permutations of one dyadic offset around a dyadic source,
    among farther decoys; the ids are shuffled, so the lowest id sits anywhere."""
    gen = np.random.default_rng(100 + k)
    for trial in range(20):
        s = (gen.integers(-2 ** 12, 2 ** 12, 3) * 2.0 ** -8).astype(np.float32)
        a = gen.integers(1, 2 ** 10, 3) * 2.0 ** -10
        offs = {tuple(sg * np.array(p)) for p in itertools.permutations(a) for sg in itertools.product((-1, 1), repeat=3)}
        offs = sorted(offs)
        pick = [offs[i] for i in gen.choice(len(offs), min(k, len(offs)), replace=False)]
        tgt = [s + np.array(o, np.float32) for o in pick]
        r = float(np.linalg.norm(a))
        dec = s + (gen.standard_normal((30, 3)) * r * 3).astype(np.float32)
        dec = dec[np.linalg.norm(dec - s, axis=1) > r * 1.01]
        tgt = np.concatenate([np.array(tgt, np.float32), dec.astype(np.float32)])
        ids = gen.permutation(10 * len(tgt))[:len(tgt)]
        res = NR.nearest(tgt, ids, s[None])
        n_tie = len(pick)
        assert res.nn[0] == ids[:n_tie].min(), trial
        assert res.ties[0] == n_tie and len(res.unsafe) == 0, trial
        # the brute force on the tie's members in id order agrees (argmin keeps the first of equals)
        o = np.argsort(ids)
        assert ids[o][orc.nearest_neighbors(tgt[o], s[None], "brute")][0] == res.nn[0]


def test_ties_that_naive_float64_misses():
    """(a, b, c) and (c, b, a) around the origin are exactly equidistant, but the naive float64 sum
    (x^2 + y^2) + z^2 rounds them differently when the magnitudes differ widely: the reference still sees a tie, and
    takes the lower id whichever of the two naive float64 calls the nearer."""
    gen = np.random.default_rng(7)
    found = 0
    while found < 40:
        v = (gen.integers(1, 2 ** 12, 3) * 2.0 ** gen.integers(-30, 1, 3)).astype(np.float32)
        a, b = v.copy(), v[[2, 1, 0]].copy()
        zero = np.zeros(3, np.float32)
        if naive_d2(zero, a) == naive_d2(zero, b):
            continue
        found += 1
        for ids in ((4, 9), (9, 4)):
            res = NR.nearest(np.stack([a, b]), ids, zero[None])
            assert res.nn[0] == 4 and res.ties[0] == 2 and np.isinf(res.sep[0]), (a, b, ids)


def test_near_ties_are_separated_exactly_and_unsafe_ones_reported():
    """Integer offsets with |D_B|^2 = |D_A|^2 + delta: the reference picks A for every delta >= 1 whatever the ids,
    reports the exact separation delta / |D_A|^2, and lists the ones below 2^-45 as unsafe."""
    unit = 2.0 ** -20
    s = np.array([2 ** 23, 0, 0], np.float64)
    for n2, delta in ((2 ** 40, 1), (2 ** 44, 1), (2 ** 46, 1), (2 ** 30, 9000)):
        # D_A = (x, y, 0), D_B = (x', y', 0): search the circle of radius^2 n2 + delta for a lattice point
        x = int(np.sqrt(n2))
        da = np.array([x, 0, 0])
        nb = x * x + delta
        for xb in range(x, 0, -1):
            rest = nb - xb * xb
            yb = int(np.sqrt(rest))
            while yb * yb > rest:
                yb -= 1
            if yb * yb == rest:
                break
        db = np.array([0, xb, yb])
        tgt = np.stack([(s + da) * unit, (s + db) * unit]).astype(np.float32)
        assert np.array_equal(tgt.astype(np.float64) / unit - s, np.stack([da, db]))     # exact in fp32
        src = (s * unit).astype(np.float32)[None]
        for ids in ((3, 8), (8, 3)):
            res = NR.nearest(tgt, ids, src)
            assert res.nn[0] == ids[0] and res.ties[0] == 1
            sep = delta / float(x * x)
            assert res.sep[0] == pytest.approx(sep, rel=1e-12)
            assert (len(res.unsafe) == 1) == (sep < 2.0 ** -45)


def test_fingerprint_equals_the_model_of_accumulation_and_finalize():
    gen = np.random.default_rng(3)
    for n in (1, 31, 32, 33, 1000, 20000):
        m = NR.source_normals(n, n)
        q = NR.code_normals(n, n + 1)
        paired = gen.random(n) < 0.9 if n > 1 else np.ones(1, bool)
        S = NR.code_sums(m[paired], q[paired])
        want = NR.fingerprint(S, int(paired.sum()))
        got, M = NR.finalize_model(m, m, q, paired)
        assert M == int(paired.sum())
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), n
        # one changed code of one paired source changes the fingerprint
        i = int(np.nonzero(paired)[0][0])
        q2 = q.copy()
        q2[i, 0] += 1
        assert not np.array_equal(NR.fingerprint(NR.code_sums(m[paired], q2[paired]), int(paired.sum())), want)
    assert not NR.fingerprint(np.zeros((3, 3), np.int64), 0).any()
