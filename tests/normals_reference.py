"""Float64 reference of the normals operators (delora_normals_fwd, delora_project_normals_fwd) and a checker with a
priori error bounds (test infrastructure, imported like helpers).

What it restates, per pixel of one [3, H, W] fp32 image (include/delora_b200.h, delora_b200/csrc/normals.cu):
  - the (2a+1) x (2b+1) tap multiset, a = int(nb_h / 2), b = int(nb_w / 2), with the reference's edge clamp;
  - the range gate in fp32 exactly as the kernels compute it: range3 = sqrt((x*x + y*y) + z*z) with a rounding after
    every operation (numpy float32, no FMA), |q.w - c.w| > eps in fp32; a neighbour counts when the gate passes and
    one of its coordinates is non-zero; a centre is valid when all three are.  The has-normal mask (valid and
    n >= max(min_neighbors, 2)) and the count n are therefore exact, not approximate;
  - the covariance of the gated set in float64 from the fp32 coordinates (two passes, relative to the centre), its
    float64 eigh (lambda0 <= lambda1 <= lambda2, eigenvector v0) and the reference's orientation rule (v0 . c <= 0).

Error bound.  u = 2^-24.  For one pixel let d_i = q_i - c over the n gated taps (exact in float64), A_k = sum |d_ik|,
B_kl = sum |d_ik| |d_il| (so B_kl <= D = sum ||d_i||^2) and M = (n - 1) C.  The 7x11 kernels form
C = (sum d d^T - s s^T / n) / (n - 1), s = sum d, in one fp32 pass; the bound on each entry of (n - 1)(C_kernel - C) is
the sum of
  1. one rounding per component of d (d^ = d (1 + e), |e| <= u):             (2u + u^2) (B_kl + A_k A_l / n)
  2. the n + 1 roundings of the one-pass sums (each partial sum of |terms| is at most B_kl, resp. A_k; the error of s
     enters s s^T / n twice):                                                   (n + 1) u B_kl + 2u A_k A_l
  3. the fmaf mean correction (m = s * fl(1/n): two roundings, then one for the fma) and the product with
     fl(1/(n - 1)) (two roundings):                                             2u A_k A_l / n + 3u |M_kl|
times (1 + 4 (n + 3) u) for the products of these first-order terms.  eps_cov is the Frobenius norm of that matrix
divided by n - 1.  The generic normals_kernel forms C in two passes on the absolute coordinates; its model is
  mean: m^ = fl(fl(fl(s^ / K) K) / n) with s^ the n-term fp32 sum of the coordinates, so
        |m^_k - m_k| <= mu_k = (n + 3) u sum |q_ik| / n, which adds n mu_k mu_l (the cross terms sum to zero);
  second pass: d^ = fl(q - m^), n fma roundings, |d^_k| <= (|q_k - m_k| + mu_k)(1 + u) =: t_k:
        (2u + u^2 + n u) sum t_k t_l;  the product with fl(1/(n - 1)): 2u |M_kl|.
On top of either, the eigen-solve (cyclic Jacobi, normals.cu smallest_eigenvector):
  4. the stop rule ignores an off-diagonal with sum |a_ij| <= 3e-8 sum |a_ii|, of Frobenius norm at most
     sqrt(2) 3e-8 (tr|C| + 3 eps_cov);
  5. at most 8 sweeps of 3 rotations (R = 24).  A rotation's c, s, tau come from the MUFU rsqrt / rcp (relative
     error below 2^-22 = 4u) and two or three roundings, so each rotation is an orthogonal one up to a relative
     8u in its entries: R (2 * 4u + 6u) (||C||_F + eps_cov) of backward error in the matrix, and a direct error of
     eps_vec = R (4u + 4u) + 4u in the returned vector (the last 4u: the final fp32 normalisation).
eps = eps_cov + eps_stop + eps_jacobi.  The kernel's vector n is then an exact eigenvector of some C' with
||C' - C|| <= eps, up to an angle eps_vec.  With x = n / ||n||:
  - Rayleigh residual x^T C x - lambda0 <= 2 eps + (lambda2 + eps) eps_vec^2 (independent of the eigen-gap);
  - when lambda1 - lambda0 > 4 eps: sin^2 theta(n, v0) <= Rayleigh bound / (lambda1 - lambda0), and the sharper
    Davis-Kahan form sin theta <= eps / (lambda1 - lambda0 - eps) + eps_vec;
  - orientation: the kernel flips n when its fp32 dot with c is > 0, so n . c <= 4u sum |n_k c_k|; and n agrees in sign
    with the oriented v0 wherever |v0 . c^| exceeds the angle bound;
  - a zero covariance (every gated neighbour equals the centre): the 7x11 kernels' C is exactly 0, the Jacobi stops at
    off = 0 with the identity, so n = -sign(c_x) e_x exactly (eigh's identity result on the zero matrix, oriented).
Nothing here is fitted to observed errors.
"""
import collections

import numpy as np

from icp_reference import fmaf

U = 2.0 ** -24
MUFU_REL = 2.0 ** -22           # rsqrt.approx / rcp.approx relative error (PTX ISA: below 2^-22.9 / 2^-23)
ROTATIONS = 24                  # 8 sweeps x 3 rotations
STOP = 3e-8                     # the Jacobi stop rule, off <= 3e-8 * diag
EPS_VEC = ROTATIONS * (MUFU_REL + 4 * U) + 4 * U


def range3(p):
    """|p| as the kernels round it: sqrt((x*x + y*y) + z*z), every operation in fp32."""
    p = np.asarray(p, np.float32)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    with np.errstate(over="ignore", invalid="ignore"):
        return np.sqrt((x * x + y * y) + z * z)


def patch_offsets(nb):
    a, b = int(nb[0] / 2), int(nb[1] / 2)
    dv = np.repeat(np.arange(-a, a + 1), 2 * b + 1)
    du = np.tile(np.arange(-b, b + 1), 2 * a + 1)
    return a, b, dv, du


def gather(img, nb):
    """img [3, H, W] fp32 -> taps [H*W, K, 3] (edge-clamped, rows of the patch outer, the reference's order) and the
    centres [H*W, 3]."""
    _, h, w = img.shape
    _, _, dv, du = patch_offsets(nb)
    v = np.repeat(np.arange(h), w)
    u = np.tile(np.arange(w), h)
    vv = np.clip(v[:, None] + dv[None], 0, h - 1)
    uu = np.clip(u[:, None] + du[None], 0, w - 1)
    pts = np.ascontiguousarray(img.reshape(3, -1).T)
    return pts[vv * w + uu], pts


def gate(q, c, eps_range):
    """-> present [P, K] (the gate passes and the neighbour is not (0, 0, 0)), valid [P] (all centre coordinates != 0)."""
    dw = np.abs(range3(q) - range3(c)[:, None])
    present = ~(dw > np.float32(eps_range)) & (q != 0).any(axis=-1)
    return present, (c != 0).all(axis=-1)


Ref = collections.namedtuple("Ref", "shape valid count has pix C lam V eps eps_cov two_pass pts")


def reference(img, nb=(7, 11), eps_range=0.5, min_nb=10, two_pass=False):
    """One image [3, H, W] -> Ref.  valid, count, has: [H*W]; pix: the pixels with a normal; C [len(pix), 3, 3],
    lam [.., 3] ascending, V [.., 3, 3] (columns), eps and eps_cov [..] for those pixels.  two_pass selects the
    generic normals_kernel's error model instead of the 7x11 kernels' one-pass one."""
    img = np.ascontiguousarray(img[:3], dtype=np.float32)
    q, c = gather(img, nb)
    present, valid = gate(q, c, eps_range)
    count = present.sum(axis=1)
    has = valid & (count >= max(int(min_nb), 2))
    pix = np.nonzero(has)[0]
    m = present[pix][..., None]
    n = count[pix].astype(np.float64)
    q64, c64 = q[pix].astype(np.float64), c[pix].astype(np.float64)
    d = (q64 - c64[:, None]) * m
    mean = d.sum(axis=1) / n[:, None]
    e = (d - mean[:, None]) * m
    M = np.einsum("pki,pkj->pij", e, e)
    C = M / (n - 1)[:, None, None]
    lam, V = np.linalg.eigh(C) if len(pix) else (np.zeros((0, 3)), np.zeros((0, 3, 3)))
    nn = n[:, None, None]
    if not two_pass:
        ad = np.abs(d)
        A = ad.sum(axis=1)
        AA = A[:, :, None] * A[:, None, :]
        B = np.einsum("pki,pkj->pij", ad, ad)
        E = ((2 * U + U * U) * (B + AA / nn)                 # 1. rounding of d
             + (nn + 1) * U * B + 2 * U * AA                 # 2. the one-pass sums
             + 2 * U * AA / nn + 3 * U * np.abs(M))          # 3. mean correction, 1 / (n - 1)
        E *= 1 + 4 * (nn + 3) * U
    else:
        mu = (n + 3)[:, None] * U * (np.abs(q64) * m).sum(axis=1) / n[:, None]
        t = (np.abs(q64 - (c64 + mean)[:, None]) + mu[:, None]) * (1 + U) * m
        T = np.einsum("pki,pkj->pij", t, t)
        E = nn * mu[:, :, None] * mu[:, None, :] + (2 * U + U * U + nn * U) * T + 2 * U * np.abs(M)
        E *= 1 + 4 * (nn + 3) * U
    eps_cov = np.sqrt((E ** 2).sum(axis=(1, 2))) / (n - 1)
    tr = np.abs(np.diagonal(C, axis1=1, axis2=2)).sum(axis=1)
    fro = np.sqrt((C ** 2).sum(axis=(1, 2)))
    eps_stop = np.sqrt(2.0) * STOP * (tr + 3 * eps_cov) * (1 + 1e-6)
    eps_jac = ROTATIONS * (2 * MUFU_REL + 6 * U) * (fro + eps_cov)
    return Ref(img.shape[1:], valid, count, has, pix, C, lam, V, eps_cov + eps_stop + eps_jac, eps_cov, two_pass,
               c)


def restate_7x11_cov(img, eps_range):
    """The 7x11 kernels' covariance formation restated in numpy fp32 (normals_7x11_body): taps column by column, rows
    inside, d = q - c, predicated sums and fmaf second moments, then fmaf(-s_k, s_l * fl(1/max(n,1)), a_kl) times
    fl(1/(n - 1)).  -> C [H*W, 3, 3] fp32 (meaningful where n >= 2) and n [H*W]."""
    img = np.ascontiguousarray(img[:3], dtype=np.float32)
    q, c = gather(img, (7, 11))
    present, _ = gate(q, c, eps_range)
    _, _, dv, du = patch_offsets((7, 11))
    order = np.lexsort((dv, du))                        # du outer, dv inner
    P = c.shape[0]
    s = np.zeros((P, 3), np.float32)
    a = np.zeros((P, 3, 3), np.float32)
    cnt = np.zeros(P, np.float32)
    for k in order:
        g = present[:, k]
        dk = (q[:, k] - c).astype(np.float32)
        s = np.where(g[:, None], s + dk, s)
        cnt = np.where(g, cnt + np.float32(1), cnt)
        prod = fmaf(dk[:, :, None], dk[:, None, :], a)
        a = np.where(g[:, None, None], prod, a)
    n = cnt.astype(np.int64)
    with np.errstate(divide="ignore"):
        inv_n = (np.float32(1) / np.maximum(n, 1).astype(np.float32)).astype(np.float32)
        f = (np.float32(1) / (n - 1).astype(np.float32)).astype(np.float32)
    mn = (s * inv_n[:, None]).astype(np.float32)
    cov = fmaf(-s[:, :, None], mn[:, None, :], a)
    iu = np.triu_indices(3, 1)                          # the kernel forms the upper triangle only
    cov[:, iu[1], iu[0]] = cov[:, iu[0], iu[1]]
    with np.errstate(invalid="ignore", over="ignore"):
        cov = (cov * f[:, None, None]).astype(np.float32)
    return cov, n


Stats = collections.namedtuple("Stats", "sin sin_gapped rayleigh_ratio angle_ratio n_has")


def _fail(label, what, pix, shape):
    v, u = np.divmod(np.asarray(pix)[:5], shape[1])
    raise AssertionError(f"{label}: {what} at (v, u) = {list(zip(v.tolist(), u.tolist()))}")


def check(ref, normals=None, pts_grid=None, nrm_grid=None, label=""):
    """Holds one image's outputs to the reference.  normals [3, H, W] fp32 or None; pts_grid, nrm_grid [H*W, 4] fp32
    or None (both or neither).  Raises AssertionError naming the first pixels that fail; returns Stats:
    sin [has pixels] sin theta(n, v0), sin_gapped (those with lambda1 - lambda0 > 4 eps), the largest Rayleigh
    residual / its bound and the largest sin theta / its Davis-Kahan bound."""
    h, w = ref.shape
    P = h * w
    if pts_grid is not None:
        pg = np.asarray(pts_grid, np.float32).reshape(P, 4)
        want = np.full((P, 4), np.inf, np.float32)
        want[:, 3] = np.arange(P, dtype=np.int32).view(np.float32)
        want[~ref.valid, 3] = np.array(-1, np.int32).view(np.float32)
        want[ref.valid, :3] = ref.pts[ref.valid]
        bad = np.nonzero((pg.view(np.int32) != want.view(np.int32)).any(axis=1))[0]
        if len(bad):
            _fail(label, "pts_grid differs", bad, ref.shape)
    vec = None
    if nrm_grid is not None:
        ng = np.asarray(nrm_grid, np.float32).reshape(P, 4)
        bad = np.nonzero(ng[:, 3] != ref.has.astype(np.float32))[0]
        if len(bad):
            _fail(label, "has-normal flag (nrm_grid.w) differs", bad, ref.shape)
        vec = ng[:, :3]
    if normals is not None:
        nv = np.ascontiguousarray(np.asarray(normals, np.float32).reshape(3, P).T)
        if vec is not None:
            bad = np.nonzero((nv.view(np.int32) != vec.view(np.int32)).any(axis=1))[0]
            if len(bad):
                _fail(label, "normals output and nrm_grid differ", bad, ref.shape)
        vec = nv
    assert vec is not None, "nothing to check"
    off = np.nonzero(~ref.has & (vec != 0).any(axis=1))[0]
    if len(off):
        _fail(label, "a normal where the reference has none", off, ref.shape)
    n = vec[ref.pix].astype(np.float64)
    norm = np.sqrt((n ** 2).sum(axis=1))
    bad = ~(np.abs(norm - 1) <= 1e-6)
    if bad.any():
        _fail(label, f"|n| - 1 = {np.abs(norm - 1)[bad][:3]}", ref.pix[bad], ref.shape)
    x = n / norm[:, None]
    c = ref.pts[ref.pix].astype(np.float64)
    lam0, lam1, lam2 = ref.lam[:, 0], ref.lam[:, 1], ref.lam[:, 2]
    eps = ref.eps
    # Rayleigh residual
    ray = np.einsum("pi,pij,pj->p", x, ref.C, x) - lam0
    ray_bound = 2 * eps + (np.abs(lam2) + eps) * EPS_VEC ** 2 + 1e-300
    bad = ~(ray <= ray_bound)
    if bad.any():
        _fail(label, f"Rayleigh residual {ray[bad][:3]} above its bound {ray_bound[bad][:3]}", ref.pix[bad], ref.shape)
    # orientation: the kernel's flip rule
    dot = (n * c).sum(axis=1)
    bad = ~(dot <= 4 * U * np.abs(n * c).sum(axis=1))
    if bad.any():
        _fail(label, f"normal points away from the sensor (n . c = {dot[bad][:3]})", ref.pix[bad], ref.shape)
    v0 = ref.V[:, :, 0]
    sin = np.sqrt((np.cross(x, v0) ** 2).sum(axis=1))
    gap = lam1 - lam0
    gapped = gap > 4 * eps
    sin2_bound = ray_bound / np.where(gapped, gap, 1.0)
    bad = gapped & ~(sin ** 2 <= sin2_bound)
    if bad.any():
        _fail(label, f"sin^2 theta {sin[bad][:3] ** 2} above {sin2_bound[bad][:3]}", ref.pix[bad], ref.shape)
    dk = eps / np.where(gapped, gap - eps, 1.0) + EPS_VEC
    bad = gapped & ~(sin <= dk)
    if bad.any():
        _fail(label, f"sin theta {sin[bad][:3]} above the Davis-Kahan bound {dk[bad][:3]}", ref.pix[bad], ref.shape)
    # sign: where v0 is clearly not perpendicular to the line of sight, n lies on the oriented v0's side
    chat = c / np.sqrt((c ** 2).sum(axis=1))[:, None]
    v0c = (v0 * chat).sum(axis=1)
    v0o = v0 * np.where(v0c > 0, -1.0, 1.0)[:, None]
    decided = gapped & (np.abs(v0c) > dk + 8 * U)
    bad = decided & ~((x * v0o).sum(axis=1) > 0)
    if bad.any():
        _fail(label, "orientation differs from the reference's", ref.pix[bad], ref.shape)
    if not ref.two_pass:
        zero = (ref.C == 0).all(axis=(1, 2))
        want = np.zeros((len(ref.pix), 3))
        want[:, 0] = -np.sign(c[:, 0])
        bad = zero & ~(n == want).all(axis=1)
        if bad.any():
            _fail(label, "zero covariance without the normal -sign(c_x) e_x", ref.pix[bad], ref.shape)
    ray_ratio = float((np.maximum(ray, 0) / ray_bound).max()) if len(ray) else 0.0
    ang_ratio = float((sin[gapped] / dk[gapped]).max()) if gapped.any() else 0.0
    return Stats(sin, sin[gapped], ray_ratio, ang_ratio, len(ref.pix))


def oriented_eigvec(ref, j=0):
    """Float64 eigenvector j of every pixel with a normal, flipped toward the sensor, rounded to fp32 -> [len(pix), 3]."""
    v = ref.V[:, :, j].copy()
    c = ref.pts[ref.pix].astype(np.float64)
    v[(v * c).sum(axis=1) > 0] *= -1
    return v.astype(np.float32)


def outputs(ref, vec):
    """Kernel-shaped outputs from per-pixel normals vec [len(pix), 3] -> normals [3, H, W], pts_grid, nrm_grid [H*W, 4]."""
    h, w = ref.shape
    P = h * w
    nv = np.zeros((P, 3), np.float32)
    nv[ref.pix] = vec
    ng = np.zeros((P, 4), np.float32)
    ng[:, :3] = nv
    ng[ref.pix, 3] = 1.0
    pg = np.full((P, 4), np.inf, np.float32)
    pg[:, 3] = np.arange(P, dtype=np.int32).view(np.float32)
    pg[~ref.valid, 3] = np.array(-1, np.int32).view(np.float32)
    pg[ref.valid, :3] = ref.pts[ref.valid]
    return np.ascontiguousarray(nv.T.reshape(3, h, w)), pg, ng


# ------------------------------------------------------------------------------------------------------ image families
# Every family is a list of B = 3 different fp32 images [3, H, W] plus the gate (eps) and min_neighbors of the call.
Family = collections.namedtuple("Family", "name images eps min_nb scalable")


def _sphere_dirs(h, w, az0=-6.0, daz=0.2, el0=-4.0, dele=0.4):
    az = np.radians(az0 + daz * np.arange(w))[None, :]
    el = np.radians(el0 + dele * np.arange(h))[:, None]
    return np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el) * np.ones_like(az)])


def _plane(h, w, normal, dist, noise, rng):
    """Ray-cast the plane {x : normal . x = dist} onto the spherical grid; range noise along the ray; misses are 0."""
    r = _sphere_dirs(h, w)
    nrm = np.asarray(normal, np.float64)
    nrm = nrm / np.linalg.norm(nrm)
    den = np.einsum("i,ihw->hw", nrm, r)
    hit = den > 1e-9
    t = np.where(hit, dist / np.where(hit, den, 1.0), 0.0)
    hit &= t < 50 * dist
    t = t + noise * rng.standard_normal(t.shape)
    return np.where(hit[None], r * t[None], 0.0).astype(np.float32)


def _incidence_normal(deg):
    """A plane normal at `deg` from the centre ray (+x) of the grid, tilted about z."""
    a = np.radians(deg)
    return np.array([np.cos(a), -np.sin(a), 0.0])


def family_planes(h=24, w=64):
    out = []
    for dist in (2.0, 20.0, 80.0, 200.0):
        rng = np.random.default_rng(int(dist))
        imgs = [_plane(h, w, _incidence_normal(tilt), dist, noise, rng)
                for tilt, noise in ((10.0, 0.0), (35.0, 1e-3), (60.0, 2e-2))]
        out.append(Family(f"F1-plane-{int(dist)}m", imgs, 0.5, 10, True))
    rng = np.random.default_rng(5)
    imgs = [_plane(h, w, _incidence_normal(deg), 10.0, 1e-3 * (k > 0), rng) for k, deg in enumerate((85.0, 87.0, 89.0))]
    out.append(Family("F1-grazing", imgs, 0.5, 10, True))
    return out


def family_one_sided(h=24, w=64):
    """Depth steps of 3 m (beyond the gate) through the patch: pixels on the step's edge see gated sets on one side."""
    rng = np.random.default_rng(7)
    base = _plane(h, w, _incidence_normal(20.0), 10.0, 1e-3, rng)
    far = _plane(h, w, _incidence_normal(-15.0), 13.0, 1e-3, rng)
    vv, uu = np.mgrid[0:h, 0:w]
    masks = [uu >= w // 2, vv >= h // 2, (uu >= w // 3) & (vv >= h // 3)]
    imgs = [np.where(mk[None], far, base).astype(np.float32) for mk in masks]
    # the third image: a near strip two pixels wide in front of the far plane (sets on one side of the centre)
    imgs[2] = np.where(((uu % 9) < 2)[None], base, far).astype(np.float32)
    return [Family("F2-one-sided", imgs, 0.5, 10, True)]


def family_thin(h=24, w=64):
    """Poles (three columns of points along z, lateral spread s) and rings (a single row): lambda1/lambda2 from 1e-2
    down to 1e-7; the last image is an exactly collinear row."""
    imgs = []
    for spread in (1e-1, 3e-3, 3e-4):
        img = np.zeros((3, h, w), np.float32)
        for k, u in enumerate(range(w // 2 - 1, w // 2 + 2)):
            ang = 0.7 * (k - 1)
            img[0, :, u] = 10.0 + spread * np.cos(ang)
            img[1, :, u] = 2.0 + spread * np.sin(ang)
            img[2, :, u] = 0.1 * (np.arange(h) - h / 2) + 0.05
        imgs.append(img)
    out = [Family("F3-poles", imgs, 0.5, 3, True)]
    rings = []
    for radius in (10.0, 40.0):
        img = np.zeros((3, h, w), np.float32)
        phi = np.radians(0.2 * np.arange(w) - 6.0)
        img[0, h // 2] = radius * np.cos(phi)
        img[1, h // 2] = radius * np.sin(phi)
        img[2, h // 2] = -1.5
        rings.append(img)
    line = np.zeros((3, h, w), np.float32)
    line[0, h // 3] = 8.0
    line[1, h // 3] = 0.25 * (np.arange(w) - w // 2) + 0.125
    line[2, h // 3] = -1.0
    rings.append(line)
    out.append(Family("F3-rings-collinear", rings, 0.5, 3, True))
    return out


def family_isotropic(h=24, w=64):
    rng = np.random.default_rng(11)
    imgs = []
    for radius in (0.1, 0.01, 0.3):
        p = rng.standard_normal((3, h, w))
        p *= radius * rng.random((1, h, w)) ** (1 / 3) / np.linalg.norm(p, axis=0, keepdims=True)
        imgs.append((p + np.array([10.0, -3.0, 1.0])[:, None, None]).astype(np.float32))
    return [Family("F4-isotropic", imgs, 0.5, 10, True)]


def _variants(s):
    """Points of exact fp32 range: range 6s (the centre's), 7s and 5s (|dr| = s), 9s (|dr| = 3s)."""
    def perms(t):
        import itertools
        out = set()
        for p in itertools.permutations(t):
            for sg in itertools.product((1, -1), repeat=3):
                out.add(tuple(a * b for a, b in zip(p, sg)))
        return sorted(out)
    f = np.float32
    return {6: np.array(perms((2, 4, 4)), f) * f(s), 7: np.array(perms((2, 3, 6)), f) * f(s),
            5: np.array([(0, 3, 4), (3, 0, 4), (4, 3, 0), (0, 4, 3), (0, 0, 5), (5, 0, 0), (0, 5, 0)], f) * f(s),
            9: np.array(perms((1, 4, 8)), f) * f(s)}


def _ulp_point(p, up):
    """p scaled by 1 + k 2^-24 (smallest |k|) so that range3 is one ulp above (up) or below range3(p)."""
    p = np.asarray(p, np.float32)
    r = range3(p)
    target = np.nextafter(r, np.float32(np.inf if up else 0))
    for k in range(1, 200):
        cand = (p.astype(np.float64) * (1 + (k if up else -k) * 2.0 ** -24)).astype(np.float32)
        if range3(cand) == target:
            return cand
    raise AssertionError("no fp32 point one ulp away")


def _gate_image(eps, min_nb, slot):
    """2 x 3 cells of 7 x 11 pixels, each cell's patch exactly the cell around its centre (3, 5): centre (2, 4, 4) s
    (range 6s).  s = eps, or 0.5 for eps = 0 where the range-6s points are the gate's edge.  Cells: min_nb - 1 and
    min_nb present taps; neighbours exactly at |dr| = eps; neighbours one ulp inside / outside; neighbours with one or
    two zero coordinates; all-zero pixels around."""
    s = eps if eps > 0 else 0.5
    var = _variants(s)
    rng = np.random.default_rng(100 * slot + min_nb + int(8 * eps))
    img = np.zeros((3, 14, 33), np.float32)
    centre = np.array((2, 4, 4), np.float32) * np.float32(s)
    rot = slot % 3

    def cell(ci, cj, fill):
        taps = [(r, q) for r in range(7) for q in range(11) if (r, q) != (3, 5)]
        rng.shuffle(taps)
        img[:, 7 * ci + 3, 11 * cj + 5] = np.roll(centre, rot)
        for (r, q), p in zip(taps, fill):
            img[:, 7 * ci + r, 11 * cj + q] = p

    inside = var[6]                                      # |dr| = 0: present for every eps >= 0
    edge = np.concatenate([var[7], var[5]]) if eps > 0 else var[6]
    out = var[9]
    cnt_lo = [inside[i % len(inside)] for i in range(max(min_nb - 2, 0))] + [out[i] for i in range(4)]
    cnt_hi = [inside[i % len(inside)] for i in range(min_nb - 1)] + [out[i] for i in range(4)]
    cell(0, 0, cnt_lo[:76])
    cell(0, 1, cnt_hi[:76])
    cell(0, 2, [edge[i % len(edge)] for i in range(12)] + [out[i] for i in range(6)])
    ulp = [_ulp_point(edge[i], i % 2 == 0) for i in range(8)]
    cell(1, 0, ulp + [inside[i] for i in range(6)])
    cell(1, 1, list(var[5]) + [inside[i] for i in range(4)] + [out[i] for i in range(3)])
    cell(1, 2, [inside[i] for i in range(3)])
    return img


def family_gate(eps_values=(0.0, 0.25, 0.5, 3.0), min_nbs=(2, 3, 10, 77)):
    out = []
    for eps in eps_values:
        for mn in min_nbs:
            out.append(Family(f"F5-gate-eps{eps:g}-min{mn}", [_gate_image(eps, mn, k) for k in range(3)], eps, mn,
                              True))
    return out


def family_degenerate():
    """Constant patches (zero covariance), isolated returns (n = 1), H = W = 1, one row, smaller than the patch."""
    const = np.broadcast_to(np.array([5.0, 3.0, 1.0], np.float32)[:, None, None], (3, 16, 40)).copy()
    const_neg = const.copy()
    const_neg[0] *= -1
    iso = np.zeros((3, 16, 40), np.float32)
    iso[:, 2::8, 4::12] =np.array([7.0, -2.0, 0.5], np.float32)[:, None, None]
    iso[:, 5, 30] = np.array([-4.0, 1.0, -0.25], np.float32)
    iso[:, 15, 39] = np.array([3.0, 3.0, 3.0], np.float32)            # a corner
    rng = np.random.default_rng(3)
    row = _plane(1, 40, _incidence_normal(25.0), 6.0, 1e-3, rng)
    small = _plane(5, 9, _incidence_normal(30.0), 4.0, 1e-3, rng)
    one = np.array([2.0, -1.0, 0.5], np.float32).reshape(3, 1, 1)
    return [Family("F6-constant-isolated", [const, const_neg, iso], 0.5, 2, True),
            Family("F6-1x1", [one, -one, one * 3], 0.5, 2, False),
            Family("F6-1x40", [row, row[:, :, ::-1].copy(), -row], 0.5, 2, False),
            Family("F6-5x9", [small, small[:, ::-1].copy(), small * 2], 0.5, 2, False)]


def families():
    return (family_planes() + family_one_sided() + family_thin() + family_isotropic() + family_gate()
            + family_degenerate())
