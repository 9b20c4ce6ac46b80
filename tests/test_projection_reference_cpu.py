"""-m "not gpu": tests/projection_reference.py, the float32 restatement the exact projection tests compare the kernels
with, checked against the oracle's torch-CPU projection (oracle.project_to_img) bit for bit on every adversarial
family, against float64 away from rounding boundaries, and for being adversarial at all."""

import numpy as np
import pytest
import torch

import projection_reference as pr
from helpers import unsort_uv
from oracle import delora_oracle as orc

# (fov, H, W, channels): the full circle at KITTI's 64 x 2250, the narrow view at 16 x 180 with a reflectance channel,
# the whole sphere at an odd 17 x 33, the synthetic scans' view at 64 x 720
GRIDS = [("full", 64, 2250, 3), ("narrow", 16, 180, 4), ("sphere", 17, 33, 3), ("synthetic", 64, 720, 3)]


def padded(cloud, c, seed):
    """cloud [3, n] -> [c, n'] with n' a multiple of 32: torch evaluates no element of a multiple of 32 with its scalar
    libm tail (one thread, as conftest.py sets).  The padding points are NaN (they have no pixel); further channels
    are random values with NaNs and infinities among them."""
    pad = (-cloud.shape[1]) % 32
    cloud = np.concatenate((cloud, np.full((3, pad), np.nan, np.float32)), axis=1)
    if c > 3:
        gen = np.random.default_rng(seed)
        extra = gen.standard_normal((c - 3, cloud.shape[1])).astype(np.float32)
        extra[:, ::17] = np.nan
        extra[:, 5::23] = -np.inf
        cloud = np.concatenate((cloud, extra), axis=0)
    return cloud


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{g[0]}_{g[1]}x{g[2]}" for g in GRIDS])
@pytest.mark.parametrize("name", list(pr.FAMILIES))
def test_restatement_equals_oracle(name, grid):
    fov, h, w, c = grid
    hfov, vfov = pr.FOVS[fov]
    cloud = padded(pr.family(name, 11, h, w, fov), c, 3)
    ref = pr.project(cloud, h, w, hfov, vfov)
    t = torch.from_numpy(cloud)
    image, u, v, idx, i2p = orc.project_to_img(t[None], h, w, hfov, vfov)
    uo, vo, ro = unsort_uv(t, u[0], v[0])
    imap = np.full((h, w), -1, np.int64)
    imap[i2p[0, :, 0].numpy(), i2p[0, :, 1].numpy()] = idx.numpy()
    assert np.array_equal(image[0].numpy().view(np.int32), ref["image"].view(np.int32))
    assert np.array_equal(imap, ref["index_map"])
    for label, got, want in (("u", uo, ref["u"]), ("v", vo, ref["v"]), ("range", ro, ref["r"])):
        bad = ~pr.same(got.numpy(), want)
        assert not bad.any(), f"{label}: {int(bad.sum())} of {len(want)} differ"
    assert (ref["pixel"] >= 0).sum() > 0


def _ulp_hits(val, targets):
    """(exact, one ulp below, one ulp above): how many distinct targets k + 0.5 are hit each way."""
    t = np.asarray(targets, np.float32)
    lo, hi = np.nextafter(t, np.float32(-np.inf)), np.nextafter(t, np.float32(np.inf))
    return tuple(len(np.intersect1d(val[np.isin(val, s)], s)) for s in (t, lo, hi))


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{g[0]}_{g[1]}x{g[2]}" for g in GRIDS])
def test_boundary_family_is_on_the_boundaries(grid):
    """F1 holds points whose float32 u is exactly k + 0.5, one ulp below it and one ulp above it, and the same for v;
    by float64, nearly every point is closer to a boundary than the float32 arithmetic can resolve."""
    fov, h, w, _ = grid
    g = pr.Grid(h, w, *pr.FOVS[fov])
    cloud = pr.family("boundaries", 11, h, w, fov)
    ref = pr.project(cloud, h, w, *pr.FOVS[fov])
    hits_u = _ulp_hits(ref["u"], np.arange(-1, w) + 0.5)
    hits_v = _ulp_hits(ref["v"], np.arange(-1, h) + 0.5)
    print(f"{fov} {h}x{w}: n={cloud.shape[1]} u hits (on, below, above) {hits_u}, v hits {hits_v}")
    assert min(hits_u) >= 20 and min(hits_v) >= min(h, 10), (hits_u, hits_v)
    mu, mv = pr.sanity_margin(g)
    near = (ref["du"] < mu) | (ref["dv"] < mv)
    assert near.mean() > 0.95, near.mean()


def test_seam_and_magnitude_families_reach_their_branches():
    """F2 puts points on both sides of the +-pi seam; F3 reaches the atan2's rescaling branch (|x| < 2^-128), has
    subnormals and zeros of both signs, the origin at range +0 with a pixel, and overflowing squares (range +inf)
    with a pixel."""
    h, w = 17, 33
    hfov, vfov = pr.FOVS["sphere"]
    seam = pr.project(pr.family("seam", 11, h, w, "sphere"), h, w, hfov, vfov)
    cols = seam["pixel"][seam["pixel"] >= 0] % w
    assert (cols == 0).any() and (cols == w - 1).any()
    cloud = pr.family("magnitudes", 11, h, w, "sphere")
    ref = pr.project(cloud, h, w, hfov, vfov)
    x, y = cloud[0], cloud[1]
    rescaled = (np.abs(x) < np.float32(2.0 ** -128)) & (x != 0)
    assert rescaled.sum() >= 100 and (rescaled & (y != 0)).sum() >= 50
    sub = (np.abs(cloud) < np.finfo(np.float32).tiny) & (cloud != 0)
    assert sub.sum() >= 300
    for c in range(3):
        col = cloud[c]
        assert ((col == 0) & np.signbit(col)).any() and ((col == 0) & ~np.signbit(col)).any()
    origin = (cloud == 0).all(axis=0)
    assert (origin & (ref["pixel"] >= 0)).any() and (ref["r"][origin].view(np.int32) == 0).all()
    inf_in = np.isinf(ref["r"]) & (ref["pixel"] >= 0) & np.isfinite(cloud).all(axis=0)
    assert inf_in.sum() >= 50
    # a winner at range +inf, a winner at range +0 and a winner whose range underflowed to +0
    img_r = ref["image"][3]
    assert np.isinf(img_r).any() and ((img_r == 0) & (ref["index_map"] >= 0)).any()


def test_tie_family_has_ties():
    """F5: pixels where several points share the winning range, one of them with 64."""
    h, w = 64, 2250
    hfov, vfov = pr.FOVS["full"]
    cloud = pr.family("ties", 11, h, w, "full")
    ref = pr.project(cloud, h, w, hfov, vfov)
    pix, r = ref["pixel"], ref["r"]
    inside = pix >= 0
    win_r = ref["image"][3].ravel()
    tied = np.bincount(pix[inside], weights=(r[inside] == win_r[pix[inside]]), minlength=h * w)
    assert (tied >= 2).sum() >= 40 and tied.max() >= 64, ((tied >= 2).sum(), tied.max())


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{g[0]}_{g[1]}x{g[2]}" for g in GRIDS])
@pytest.mark.parametrize("name", ["random", "boundaries", "seam", "ties", "magnitudes", "nonfinite"])
def test_restatement_against_float64(name, grid):
    """Where the squares neither overflow nor underflow, the float32 (u, v) lie within the sanity margin of float64's,
    and every point farther than that margin from a rounding boundary has float64's pixel."""
    fov, h, w, _ = grid
    hfov, vfov = pr.FOVS[fov]
    g = pr.Grid(h, w, hfov, vfov)
    if name == "random":
        cloud = pr.random_cloud(np.random.default_rng(5), 20000, g)
    else:
        cloud = pr.family(name, 11, h, w, fov)
    ref = pr.project(cloud, h, w, hfov, vfov)
    mu, mv = pr.sanity_margin(g)
    ok = np.isfinite(cloud).all(axis=0) & (ref["r"] > 1e-18) & (ref["r"] < 1e18)
    assert abs(ref["u"][ok] - ref["u64"][ok]).max() <= mu
    assert abs(ref["v"][ok] - ref["v64"][ok]).max() <= mv
    far = ok & (ref["du"] > mu) & (ref["dv"] > mv)
    ru, rv = np.rint(ref["u64"][far]), np.rint(ref["v64"][far])
    inside = (ru >= 0) & (ru <= w - 1) & (rv >= 0) & (rv <= h - 1)
    pix64 = np.where(inside, rv * w + ru, -1).astype(np.int64)
    assert np.array_equal(ref["pixel"][far], pix64)
    print(f"{name} {fov}: {int(ok.sum())} points in the float64 domain, {int(far.sum())} away from a boundary")
