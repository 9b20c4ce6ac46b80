"""Float32 restatement of the reference's projection (src/utility/projection.py:21-106), CPU and numpy, and seeded
families of adversarial clouds for it (test infrastructure).

`project` follows the reference's arithmetic operation by operation, in float32:
  * range  r = sqrt((x*x + y*y) + z*z)                                   (torch.norm over x, y, z: :59-60)
  * u = ((atan2(y, x) - hf0) / hspan) * (W - 1)                          (:21-31, compute_2D_coordinates)
    v = ((atan2(z, sqrt(x*x + y*y)) - vf0) / vspan) * (H - 1)
    with atan2 = SLEEF's atan2f_u10 (torch.atan2 on CPU float32 tensors), taken from its scalar C twin
    oracle/sleef_atan2f.c (oracle/_ref/libsleef_atan2f.so, which build() makes), and the constants rounded the
    way torch rounds a Python scalar operand: float32(hf0), float32(hf1 - hf0) formed in double, float32(W - 1);
  * (u, v) rounded half to even (torch.round), then the field-of-view test of :74-77;
  * in each pixel the in-view point of minimum (range, id) wins: the reference's range sort (:63) made stable.

Next to the float32 result it returns the float64 (u, v) of every point (double arctan2 and hypot on the same
float32 inputs, exact constants) and their distance in pixels to the nearest rounding boundary k + 0.5.  The
families use that distance to show that their points sit where the float32 arithmetic decides the pixel.
"""
import ctypes
import math
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWIN = os.path.join(ROOT, "oracle", "_ref", "libsleef_atan2f.so")

KITTI_VFOV = (math.radians(-24.5), math.radians(2.0))
# (hfov, vfov) in radians: the reference's full circle, the synthetic scans' +-179.9 deg, a narrow asymmetric view
# with a symmetric +-15 deg vertical field, and the whole sphere (every direction has a pixel: the families of tiny,
# huge and non-finite coordinates reach the image through it).
FOVS = {
    "full": ((-math.pi, math.pi), KITTI_VFOV),
    "synthetic": ((math.radians(-179.9), math.radians(179.9)), KITTI_VFOV),
    "narrow": ((-math.pi / 4, math.pi / 3), (math.radians(-15.0), math.radians(15.0))),
    "sphere": ((-math.pi, math.pi), (-math.pi / 2, math.pi / 2)),
}

_lib = [None]


def _twin():
    if _lib[0] is None:
        if not os.path.exists(TWIN):
            subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "oracle")], check=True)
        lib = ctypes.CDLL(TWIN)
        lib.delora_sleef_atan2f_array.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_long]
        lib.delora_sleef_atan2f_array.restype = None
        _lib[0] = lib
    return _lib[0]


def atan2f(y, x):
    """SLEEF's atan2f_u10 (torch.atan2 on CPU float32) element by element, through the C twin."""
    y, x = np.broadcast_arrays(np.asarray(y, np.float32), np.asarray(x, np.float32))
    y, x = np.ascontiguousarray(y), np.ascontiguousarray(x)
    out = np.empty(y.shape, np.float32)
    _twin().delora_sleef_atan2f_array(y.ctypes.data, x.ctypes.data, out.ctypes.data, y.size)
    return out


class Grid:
    """The float32 constants of an H x W grid, rounded as make_grid (csrc/common.cuh) and torch round them."""

    def __init__(self, h, w, hfov, vfov):
        self.H, self.W = int(h), int(w)
        self.hfov, self.vfov = (float(hfov[0]), float(hfov[1])), (float(vfov[0]), float(vfov[1]))
        self.hf0, self.hspan, self.wm1 = np.float32(hfov[0]), np.float32(hfov[1] - hfov[0]), np.float32(w - 1)
        self.vf0, self.vspan, self.hm1 = np.float32(vfov[0]), np.float32(vfov[1] - vfov[0]), np.float32(h - 1)


def coords(g, x, y, z):
    """float32 (u, v, range) of points x, y, z (float32 arrays) in the reference's operation order."""
    x, y, z = (np.asarray(a, np.float32) for a in (x, y, z))
    with np.errstate(all="ignore"):
        xy = x * x + y * y
        u = ((atan2f(y, x) - g.hf0) / g.hspan) * g.wm1
        v = ((atan2f(z, np.sqrt(xy)) - g.vf0) / g.vspan) * g.hm1
        r = np.sqrt(xy + z * z)
    return u, v, r


def pixels(g, u, v):
    """Pixel id v * W + u of rounded (u, v) inside the image, -1 outside (NaN included)."""
    with np.errstate(invalid="ignore"):
        ru, rv = np.rint(u), np.rint(v)
        inside = (ru <= g.wm1) & (ru >= 0) & (rv <= g.hm1) & (rv >= 0)
    pix = np.full(u.shape, -1, np.int64)
    pix[inside] = rv[inside].astype(np.int64) * g.W + ru[inside].astype(np.int64)
    return pix


def float64_coords(g, x, y, z):
    """(u, v) in float64 with the exact constants, and each one's distance in pixels to the nearest k + 0.5."""
    with np.errstate(all="ignore"):                       # a signalling NaN raises "invalid" when widened
        x, y, z = (np.asarray(a, np.float64) for a in (x, y, z))
        u = (np.arctan2(y, x) - g.hfov[0]) / (g.hfov[1] - g.hfov[0]) * (g.W - 1)
        v = (np.arctan2(z, np.hypot(x, y)) - g.vfov[0]) / (g.vfov[1] - g.vfov[0]) * (g.H - 1)
        du = np.abs((u - 0.5) - np.rint(u - 0.5))
        dv = np.abs((v - 0.5) - np.rint(v - 0.5))
    return u, v, du, dv


def project(points, h, w, hfov, vfov, ids=None):
    """points [C, n] float32 (x, y, z, further channels) -> dict of
       u, v, r [n] float32, pixel [n] int64 (-1 outside), image [C+1, H, W] float32 (channels, then range; 0 where
       empty), index_map [H, W] int64 (the winner's id, -1 where empty), u64, v64, du, dv [n] float64.
    ids [n] (default 0..n-1) are the tie-break ids and what index_map holds."""
    g = Grid(h, w, hfov, vfov)
    points = np.asarray(points, np.float32)
    c, n = points.shape
    ids = np.arange(n, dtype=np.int64) if ids is None else np.asarray(ids, np.int64)
    u, v, r = coords(g, points[0], points[1], points[2])
    pix = pixels(g, u, v)
    image = np.zeros((c + 1, h * w), np.float32)
    index_map = np.full(h * w, -1, np.int64)
    sel = np.nonzero(pix >= 0)[0]
    assert not np.isnan(r[sel]).any()                     # a NaN coordinate never has a pixel
    order = sel[np.lexsort((ids[sel], r[sel]))]           # ascending (range, id); a range is never -0
    _, first = np.unique(pix[order], return_index=True)
    win = order[first]
    image[:c, pix[win]] = points[:, win]
    image[c, pix[win]] = r[win]
    index_map[pix[win]] = ids[win]
    u64, v64, du, dv = float64_coords(g, points[0], points[1], points[2])
    return dict(u=u, v=v, r=r, pixel=pix, image=image.reshape(c + 1, h, w), index_map=index_map.reshape(h, w),
                u64=u64, v64=v64, du=du, dv=dv, grid=g)


def sanity_margin(g):
    """Pixels by which the float32 (u, v) may miss the float64 ones: 1e-4 px, plus a few ulp of the angle and of the
    three roundings (sub, div, mul) and of the rounded constants, scaled by pixels per radian.  Only the float64 guard
    on the restatement uses it; every comparison of the kernels with the restatement is exact."""
    eu = 2.0 ** -21 * (math.pi / float(g.hspan) + 1.0) * max(g.W - 1, 1)
    ev = 2.0 ** -21 * (math.pi / float(g.vspan) + 1.0) * max(g.H - 1, 1)
    return 1e-4 + eu, 1e-4 + ev


# ------------------------------------------------------------------------------------------------ families
# Each family is a seeded generator of a float32 cloud [3, n] for a grid.

def _sphere_dirs(gen, n, g, pad_rad=0.05):
    """Directions with azimuth and elevation uniform over the field of view widened by pad_rad on each side."""
    az = gen.uniform(g.hfov[0] - pad_rad, g.hfov[1] + pad_rad, n)
    el = gen.uniform(g.vfov[0] - pad_rad, g.vfov[1] + pad_rad, n)
    return az, el


def _xyz(r, az, el):
    return np.stack((r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el))).astype(np.float32)


def random_cloud(gen, n, g, r_lo=0.5, r_hi=90.0):
    """An ordinary scan-like cloud: directions over the field of view and a little beyond, log-uniform ranges."""
    az, el = _sphere_dirs(gen, n, g)
    r = np.exp(gen.uniform(math.log(r_lo), math.log(r_hi), n))
    return _xyz(r, az, el)


def _nudge(a, k):
    """a moved by k float32 steps away from zero (toward it for k < 0; a must stay clear of zero by |k| steps)."""
    bits = np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
    return (bits + k).astype(np.int32).view(np.float32)


def _pick_boundary(val, targets):
    """For each row of val [T, K] and its target t (k + 0.5 in float32): the columns where val == t, val is one ulp
    below t and val is one ulp above it (or, when that value is not reached, the closest value on that side).
    -> list of (row, column) pairs."""
    lo = np.nextafter(targets, np.float32(-np.inf))[:, None]
    hi = np.nextafter(targets, np.float32(np.inf))[:, None]
    t = targets[:, None]
    out = []
    finite = np.isfinite(val)
    below = np.where(finite & (val < t), val, -np.inf)
    above = np.where(finite & (val > t), val, np.inf)
    for row in range(val.shape[0]):
        eq = np.nonzero(val[row] == t[row])[0]
        if eq.size:
            out.append((row, eq[0]))
        b = np.nonzero(val[row] == lo[row])[0]
        b = b[0] if b.size else int(np.argmax(below[row]))
        a = np.nonzero(val[row] == hi[row])[0]
        a = a[0] if a.size else int(np.argmin(above[row]))
        if np.isfinite(below[row, b]):
            out.append((row, b))
        if np.isfinite(above[row, a]):
            out.append((row, a))
    return out


def boundary_cloud(gen, g, n_u=96, n_v=None, ranges=(0.7, 7.3, 55.0, 140.0), window=12):
    """F1: points whose float32 u (or v) is exactly k + 0.5, one ulp below it or one ulp above it.

    For each target boundary a point is aimed at it in float64; then a (2 window + 1)^2 lattice of float32 neighbours
    (y and x moved by up to `window` steps for u, z and x for v) is evaluated with the restatement's own arithmetic
    and the neighbours on, just below and just above the boundary are kept.  The targets include the field-of-view
    edges -0.5 and W - 0.5 (H - 0.5).  Returns the cloud [3, n] float32."""
    offs = np.arange(-window, window + 1)
    oa, ob = [o.ravel() for o in np.meshgrid(offs, offs)]
    pts = []
    # u boundaries
    ks = np.concatenate(([-1, g.W - 1], gen.integers(0, max(g.W - 1, 1), n_u)))
    for r in ranges:
        t = (ks + 0.5).astype(np.float32)
        az = g.hfov[0] + (ks + 0.5) / max(g.W - 1, 1) * (g.hfov[1] - g.hfov[0])
        el = gen.uniform(g.vfov[0], g.vfov[1], len(ks))
        x, y, z = _xyz(r, az, el)
        # move the coordinate atan2(y, x) is more sensitive to by `oa`, the other by `ob`
        ymain = np.abs(x) >= np.abs(y)
        main = np.where(ymain, y, x)[:, None]
        other = np.where(ymain, x, y)[:, None]
        mm = _nudge(np.broadcast_to(main, (len(ks), oa.size)), oa[None, :])
        oo = _nudge(np.broadcast_to(other, (len(ks), ob.size)), ob[None, :])
        xx = np.where(ymain[:, None], oo, mm)
        yy = np.where(ymain[:, None], mm, oo)
        zz = np.broadcast_to(z[:, None], xx.shape)
        u, _, _ = coords(g, xx, yy, zz)
        for row, col in _pick_boundary(u, t):
            pts.append((xx[row, col], yy[row, col], zz[row, col]))
    # v boundaries
    kv = np.arange(-1, g.H) if n_v is None else np.concatenate(([-1, g.H - 1], gen.integers(0, max(g.H - 1, 1), n_v)))
    for r in ranges:
        t = (kv + 0.5).astype(np.float32)
        el = g.vfov[0] + (kv + 0.5) / max(g.H - 1, 1) * (g.vfov[1] - g.vfov[0])
        az = gen.uniform(g.hfov[0], g.hfov[1], len(kv))
        x, y, z = _xyz(r, az, el)
        big_x = np.abs(x) >= np.abs(y)
        side = np.where(big_x, x, y)[:, None]
        zz = _nudge(np.broadcast_to(z[:, None], (len(kv), oa.size)), oa[None, :])
        ss = _nudge(np.broadcast_to(side, (len(kv), ob.size)), ob[None, :])
        xx = np.where(big_x[:, None], ss, np.broadcast_to(x[:, None], ss.shape))
        yy = np.where(big_x[:, None], np.broadcast_to(y[:, None], ss.shape), ss)
        _, v, _ = coords(g, xx, yy, zz)
        for row, col in _pick_boundary(v, t):
            pts.append((xx[row, col], yy[row, col], zz[row, col]))
    return np.array(pts, np.float32).T.copy()


def seam_cloud(gen, g, n=64):
    """F2: the +-pi seam (x < 0 with y = +0, -0 and +- the smallest subnormal: u at 0 and at W - 1), and points aimed
    at the four field-of-view edges u = -0.5, W - 0.5, v = -0.5, H - 0.5 (the boundary search of boundary_cloud
    restricted to those edges)."""
    tiny = np.float32(1e-45)
    x = -np.exp(gen.uniform(math.log(0.5), math.log(80.0), n)).astype(np.float32)
    el = gen.uniform(g.vfov[0], g.vfov[1], n)
    z = (np.abs(x) * np.tan(el)).astype(np.float32)
    ys = [np.float32(0.0), np.float32(-0.0), tiny, -tiny]
    seam = np.concatenate([np.stack((x, np.full(n, yv, np.float32), z)) for yv in ys], axis=1)
    edges = boundary_cloud(gen, g, n_u=0, n_v=0, ranges=(3.1, 31.0))
    return np.concatenate((seam, edges), axis=1)


def magnitude_cloud(gen, g):
    """F3: |x|, |y| below 2^-128 (the atan2's rescaling branch), subnormals, +-0 in each coordinate, the origin,
    points on and near the z axis, and coordinates from 1e19 to 3e38 whose squares overflow (range +inf, finite
    pixel)."""
    tiny = np.array([1e-45, 3e-45, 1e-42, 2.5e-40, 2.9e-39, 2.94e-39, 2.95e-39, 5e-39, 1.1e-38, 1.2e-38], np.float32)
    big = np.array([1e19, 1.9e19, 3e19, 1e25, 1e30, 1e36, 3e38, np.finfo(np.float32).max], np.float32)
    ordinary = np.array([0.5, 3.0, 17.0], np.float32)
    zeros = np.array([0.0, -0.0], np.float32)
    pool = np.concatenate((tiny, -tiny, big, -big, ordinary, -ordinary, zeros))
    # every combination of magnitudes on a coarse sample, plus random picks from the pool
    a = np.concatenate((tiny[::3], -tiny[1::3], big[::3], -big[1::3], ordinary[:1], -ordinary[1:2], zeros))
    xx, yy, zz = [m.ravel() for m in np.meshgrid(a, a, a, indexing="ij")]
    rnd = pool[gen.integers(0, len(pool), (3, 1024))]
    axis = np.array([[0.0, 0.0, 5.0], [-0.0, 0.0, -5.0], [0.0, -0.0, 1e-3], [1e-7, 0.0, 5.0], [0.0, -1e-7, -5.0],
                     [1e-20, 1e-20, 2.0], [-3e-39, 1e-45, 1.0], [0.0, 0.0, 0.0], [-0.0, -0.0, -0.0]], np.float32).T
    return np.concatenate((np.stack((xx, yy, zz)).astype(np.float32), rnd.astype(np.float32), axis), axis=1)


def nonfinite_cloud(gen, g, n=256):
    """F4: NaN (several payloads, both signs) in one coordinate; +-inf in one or two coordinates; the rest ordinary."""
    base = random_cloud(gen, n, g)
    nans = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x7FA5A5A5], np.uint32).view(np.float32)
    infs = np.array([np.inf, -np.inf], np.float32)
    out = [base]
    for c in range(3):
        p = base.copy()
        p[c] = nans[gen.integers(0, len(nans), n)]
        out.append(p)
        q = base.copy()
        q[c] = infs[gen.integers(0, 2, n)]
        out.append(q)
        q2 = base.copy()
        c2 = (c + 1) % 3
        q2[c] = infs[gen.integers(0, 2, n)]
        q2[c2] = infs[gen.integers(0, 2, n)]
        out.append(q2)
    return np.concatenate(out, axis=1)


def tie_cloud(gen, g, n_groups=48):
    """F5: equal ranges in one pixel.  Exact duplicates; sign- and axis-permuted points of equal range ((a, b, c),
    (b, a, c), (a, b, -c), (b, a, -c) with a ~ b and c ~ 0 land in one pixel with the same range bits, because
    float addition commutes); one pixel holding 64 copies of a point.  The points are shuffled, so the lowest index of
    each tie sits anywhere in the cloud."""
    pts = []
    for _ in range(n_groups):
        r = gen.uniform(2.0, 60.0)
        a = np.float32(r * math.cos(math.pi / 4))
        b = np.float32(a * (1.0 + gen.uniform(-1e-6, 1e-6)))
        c = np.float32(r * gen.uniform(-1e-4, 1e-4))
        s = gen.choice([-1.0, 1.0], 2).astype(np.float32)
        grp = [(s[0] * a, s[1] * b, c), (s[0] * b, s[1] * a, c), (s[0] * a, s[1] * b, -c), (s[0] * b, s[1] * a, -c)]
        pts += grp * int(gen.integers(1, 4))
    base = random_cloud(gen, 256, g)
    dup = base[:, gen.integers(0, 256, 128)]
    many = np.repeat(base[:, :1], 64, axis=1)
    cloud = np.concatenate((np.array(pts, np.float32).T, base, dup, many), axis=1)
    return cloud[:, gen.permutation(cloud.shape[1])].copy()


FAMILIES = {
    "boundaries": boundary_cloud,
    "seam": seam_cloud,
    "magnitudes": magnitude_cloud,
    "nonfinite": nonfinite_cloud,
    "ties": tie_cloud,
}


def family(name, seed, h, w, fov):
    """The cloud [3, n] float32 of family `name` for an H x W grid over FOVS[fov], from a seed."""
    hfov, vfov = FOVS[fov]
    gen = np.random.default_rng(seed)
    return FAMILIES[name](gen, Grid(h, w, hfov, vfov))


def same(a, b):
    """Bit-identical float arrays, except that any NaN equals any NaN: the hardware picks a NaN's sign and payload
    (x86 propagates an operand's, the GPU returns its canonical NaN), and no pixel decision reads them."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    eq = a.view(np.int32) == b.view(np.int32)
    return eq | (np.isnan(a) & np.isnan(b))
