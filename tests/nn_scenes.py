"""Adversarial ICP scenes for the nearest-neighbour searches (test infrastructure, CPU only; the scenes' device grids
are built on the GPU).

A Scene is a target grid built from points by the projection's rule (tests/projection_reference.py: one point per
cell, the nearest in range, every target in the cell its projection gives) and a list of free source points, with the
exact NN of every source (tests/nn_reference.py).  The builders make the families of tests/test_gpu_icp_nn_exact.py:
synthetic scans under arbitrary transforms (SIZES_A, transforms_a), exact ties (tie_scene), near ties
(near_tie_scene), certification borders of the window and block searches (border_scene), ordinary scans and clouds
(scan_points, random_points), the small grid shapes (SHAPES_G) and the documented limits of the search (SHAPES_H).
"""
import contextlib
import itertools
import os
import math

import numpy as np
import torch

import nn_reference as NR
import projection_reference as PR

DEV = "cuda"
HF = (math.radians(-179.9), math.radians(179.9))
LIMITS_DEFAULT = (None,)
LIMITS_ALL = ("0", "1", None, "100000")       # DELORA_ICP_MAX_STRIPS: every hand-over limit a family runs


@contextlib.contextmanager
def max_strips(limit):
    """The dense window search's hand-over limit (DELORA_ICP_MAX_STRIPS) for the calls inside; None: the default."""
    old = os.environ.get("DELORA_ICP_MAX_STRIPS")
    try:
        if limit is None:
            os.environ.pop("DELORA_ICP_MAX_STRIPS", None)
        else:
            os.environ["DELORA_ICP_MAX_STRIPS"] = limit
        yield
    finally:
        if old is None:
            os.environ.pop("DELORA_ICP_MAX_STRIPS", None)
        else:
            os.environ["DELORA_ICP_MAX_STRIPS"] = old


def deg(a, b):
    return (math.radians(a), math.radians(b))


def direction(g, u, v):
    """float64 unit vector of pixel coordinates (u, v) of grid g (projection_reference.Grid)."""
    az = g.hfov[0] + np.asarray(u, np.float64) / max(g.W - 1, 1) * (g.hfov[1] - g.hfov[0])
    el = g.vfov[0] + np.asarray(v, np.float64) / max(g.H - 1, 1) * (g.vfov[1] - g.vfov[0])
    return np.stack((np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)), axis=-1)


class Scene:
    """A target grid (built from points by the projection's rule) and a list of free source points."""

    def __init__(self, name, h, w, hfov, vfov, tgt_points, src_points, slots=None, limits=LIMITS_DEFAULT):
        self.name, self.h, self.w, self.hfov, self.vfov = name, h, w, hfov, vfov
        self.g = PR.Grid(h, w, hfov, vfov)
        tp = np.asarray(tgt_points, np.float32).reshape(-1, 3)
        tp = tp[np.isfinite(tp).all(axis=1) & (tp != 0).all(axis=1)]      # the lists keep only nonzero x, y, z
        hw = h * w
        if len(tp):
            pr = PR.project(tp.T, h, w, hfov, vfov)
            imap = pr["index_map"].reshape(-1)
        else:
            imap = np.full(hw, -1, np.int64)
        self.pix = np.nonzero(imap >= 0)[0]
        self.tgt = tp[imap[self.pix]] if len(self.pix) else np.zeros((0, 3), np.float32)
        self.src = np.asarray(src_points, np.float32).reshape(-1, 3)
        ns = len(self.src)
        self.slots = np.arange(ns) if slots is None else np.asarray(slots, np.int64)
        self.pair = self.slots // hw
        self.slot = self.slots % hw
        self.B = int(self.pair.max()) + 1 if ns else 1
        self.limits = limits
        self.ref = NR.nearest(self.tgt, self.pix, self.src)
        assert len(self.ref.unsafe) == 0, f"{name}: scene has separations below 2^-45 at sources {self.ref.unsafe[:8]}"
        # device grids
        tg = np.full((hw, 4), np.inf, np.float32)
        tg[:, 3] = np.array(-1, np.int32).view(np.float32)
        tg[self.pix, :3] = self.tgt
        tg[self.pix, 3] = self.pix.astype(np.int32).view(np.float32)
        self.tg = torch.from_numpy(np.broadcast_to(tg, (self.B, hw, 4)).copy()).to(DEV)
        sg = np.full((self.B, hw, 4), np.inf, np.float32)
        sg[:, :, 3] = np.array(-1, np.int32).view(np.float32)
        sg[self.pair, self.slot, :3] = self.src
        sg[self.pair, self.slot, 3] = self.slot.astype(np.int32).view(np.float32)
        self.sg_host = sg
        self.sg = torch.from_numpy(sg).to(DEV)
        self.eye = torch.tensor([[1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]], dtype=torch.float32).repeat(self.B, 1).to(DEV)

    # -- the dense operator through the fingerprint ------------------------------------------------------------
    def codes(self, seed):
        """Code normals per pixel [HW, 3] (bounded so that every |S| < 2^22) and the source normals [Ns, 3]."""
        c = int(min(7, max(1, 2 ** 22 // max(1, 2 * len(self.src)) - 1)))
        return NR.code_normals(self.h * self.w, seed, c), NR.source_normals(len(self.src), seed + 1)

    def expected(self, q, m, sel=None):
        """fp32 grad_T [B, 12] and M [B] of the fingerprint, sources `sel` (bool [Ns]) carrying normals."""
        sel = np.ones(len(self.src), bool) if sel is None else sel
        has = len(self.pix) > 0
        out = np.zeros((self.B, 12), np.float32)
        M = np.zeros(self.B, np.int64)
        for b in range(self.B):
            k = (self.pair == b) & sel & has
            M[b] = int(k.sum())
            out[b] = NR.fingerprint(NR.code_sums(m[k], q[self.ref.nn[k]]), M[b])
        return out, M

    def dense(self, q, m, flags, limit=None, sel=None, src_mask=None):
        from delora_b200 import ops
        tn = np.zeros((self.h * self.w, 4), np.float32)
        tn[:, :3] = q
        tn[:, 3] = 1.0
        tn = torch.from_numpy(np.broadcast_to(tn, (self.B, self.h * self.w, 4)).copy()).to(DEV)
        sn = np.zeros((self.B, self.h * self.w, 4), np.float32)
        mm = m if sel is None else np.where(sel[:, None], m, np.float32(0))
        sn[self.pair, self.slot, :3] = mm
        sg = self.sg
        if src_mask is not None:
            host = self.sg_host.copy()
            host[src_mask] = np.inf
            host[src_mask + (3,)] = np.array(-1, np.int32).view(np.float32)
            sg = torch.from_numpy(host).to(DEV)
        with max_strips(limit):
            lo, g = ops.icp_dense_fwd_bwd(sg, torch.from_numpy(sn).to(DEV), self.eye, self.tg, tn, self.h, self.w,
                                          self.hfov, self.vfov, flags=flags)
            torch.cuda.synchronize()
        return lo.cpu().numpy(), g.cpu().numpy()

    def csr(self, T=None, src=None):
        """nn_index of the CSR operator for every source (one list, pair 0's target grid)."""
        from delora_b200 import ops
        hw = self.h * self.w
        img = np.zeros((1, 4, hw), np.float32)
        img3 = img[0]
        img3[:3, self.pix] = self.tgt.T
        img[0, 3, self.pix] = np.sqrt((self.tgt.astype(np.float64) ** 2).sum(1)).astype(np.float32)
        img = torch.from_numpy(img.reshape(1, 4, self.h, self.w)).to(DEV)
        nrm = torch.zeros((1, 3, self.h, self.w), device=DEV)
        pts4, nrm4, cs, counts = ops.lists_from_images(img, nrm)
        assert int(counts[0]) == len(self.pix)
        src = self.src if src is None else src
        ns = max(len(src), 1)
        s4 = torch.zeros((1, ns, 4), device=DEV)
        s4[0, :len(src), :3] = torch.from_numpy(src).to(DEV)
        n = torch.tensor([len(src)], dtype=torch.int32, device=DEV)
        _, _, nn, _, _ = ops.icp_fwd_bwd(s4, torch.zeros_like(s4), n, T, pts4, nrm4, cs, self.h, self.w, self.hfov,
                                         self.vfov, pointwise=True)
        return nn[0, :len(src)].cpu().numpy().astype(np.int64)

    # -- localisation --------------------------------------------------------------------------------------------
    def localise(self, q, m, flags, limit, b):
        """-> a message naming the first wrong source of pair b, its chosen and correct pixels and distances."""
        idx = np.nonzero(self.pair == b)[0]

        def bad(lo, hi):
            sel = np.zeros(len(self.src), bool)
            sel[idx[lo:hi]] = True
            want, _ = self.expected(q, m, sel)
            _, g = self.dense(q, m, flags, limit, sel)
            return not np.array_equal(g[b], want[b])

        lo, hi = 0, len(idx)
        if not bad(lo, hi):
            return f"pair {b}: the miss does not reproduce"
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if bad(lo, mid):
                hi = mid
            else:
                lo = mid
        i = int(idx[lo])
        hw = self.h * self.w
        j = np.arange(hw)
        uq = np.stack((j & 4095, j >> 12, np.zeros_like(j)), axis=1).astype(np.float32)
        e0 = np.zeros_like(m)
        e0[:, 0] = 1.0
        sel = np.zeros(len(self.src), bool)
        sel[i] = True

        def chosen(mask=None):
            # one paired source with m = e_0: M = 1, grad_T[:, 0] = 2 (e_0 - q), q = (j & 4095, j >> 12, 0)
            _, g = self.dense(uq, e0, flags, limit, sel, src_mask=mask)
            qv = np.array([1.0, 0.0, 0.0]) - g[b].reshape(3, 4)[:, 0].astype(np.float64) / 2.0
            return int(round(qv[0])) + (int(round(qv[1])) << 12)

        got = chosen()
        slot = int(self.slot[i])
        mates = np.zeros(self.sg_host.shape[:2], bool)
        mates[b, (slot // 32) * 32:(slot // 32) * 32 + 32] = True
        mates[b, slot] = False
        alone = chosen(np.nonzero(mates))
        want = int(self.ref.nn[i])
        tj = lambda p: self.tgt[np.searchsorted(self.pix, p)]       # noqa: E731
        d_got = NR.exact_d2(self.src[i], tj(got)) if got in set(self.pix.tolist()) else None
        d_want = NR.exact_d2(self.src[i], tj(want))
        return (f"pair {b} source {i} (slot {slot}, point {self.src[i].tolist()}): chose pixel {got} "
                f"(d^2 {float(d_got) if d_got is not None else 'n/a'!r}), the nearest is pixel {want} "
                f"(d^2 {float(d_want)!r}); with its warp-mates removed it chooses {alone} "
                f"({'still wrong' if alone != want else 'right: the miss depends on the warp-mates'})")


# ---- A: synthetic scans at full density ---------------------------------------------------------------------------
SIZES_A = [(16, 180, 192, (-15.0, 15.0)), (15, 180, 192, (-15.0, 15.0)), (64, 720, 1024, (-24.5, 2.0)),
           (64, 2048, 2048, (-24.5, 2.0)), (64, 2250, 2250, (-24.5, 2.0))]


def transforms_a(t_pred):
    from delora_b200 import synthetic
    ts = [("identity", np.eye(4)), ("T_pred", t_pred.numpy().astype(np.float64)),
          ("2m-10deg", synthetic.transform_matrix(2.0, 0.0, 0.0, math.radians(10.0))),
          ("yaw178", synthetic.transform_matrix(0.0, 0.0, 0.0, math.radians(178.0))),
          ("yaw181", synthetic.transform_matrix(0.0, 0.0, 0.0, math.radians(181.0)))]
    gen = np.random.default_rng(5)
    for k in range(3):
        ang = gen.uniform(-math.pi, math.pi, 3) * np.array([1.0, 0.1, 0.1])
        ts.append((f"arbitrary{k}", synthetic.transform_matrix(*gen.uniform(-3, 3, 3), *ang)))
    return ts

# ---- synthetic grids for the adversarial families --------------------------------------------------------------
GRIDS = [(16, 180, HF, deg(-15.0, 15.0)), (64, 720, HF, deg(-24.5, 2.0))]
GRID_IDS = ["16x180", "64x720"]


def background(g, gen, r=40.0, fill=0.6):
    """A sphere of targets at range r on a random `fill` of the cells (directions jittered inside their cell)."""
    n = int(g.H * g.W * fill)
    cells = gen.choice(g.H * g.W, n, replace=False)
    u = cells % g.W + gen.uniform(-0.4, 0.4, n)
    v = cells // g.W + gen.uniform(-0.4, 0.4, n)
    return (direction(g, u, v) * r).astype(np.float32)


def pitch(g):
    return (g.hfov[1] - g.hfov[0]) / max(g.W - 1, 1), (g.vfov[1] - g.vfov[0]) / max(g.H - 1, 1)


def anchors(g, gen, n_rand=40):
    """Pixel positions the tie groups are built around: block corners and edges, the seam, the azimuths on the axes,
    and random ones, all inside the image."""
    out = []
    for bc in range(16, g.W - 1, 16 * max(1, g.W // 160)):
        for br in range(4, g.H - 1, 4 * max(1, g.H // 16)):
            out += [(bc - 0.5, br - 0.5), (bc - 0.5, br + 1.3), (bc + 2.2, br - 0.5)]
    for v in np.linspace(1, g.H - 2, 4):
        out += [(g.W - 1 + 0.45, v), (-0.45, v)]                     # the seam
        for az in (0.0, math.pi / 2, -math.pi / 2):
            out.append(((az - g.hfov[0]) / (g.hfov[1] - g.hfov[0]) * (g.W - 1), v))
    out += list(zip(gen.uniform(1, g.W - 2, n_rand), gen.uniform(1, g.H - 2, n_rand)))
    return out


def spaced(points, min_px, g):
    """Greedy subset of anchor positions at least min_px apart (in pixels, the seam wrapping)."""
    keep = []
    for u, v in points:
        if all(min(abs(u - a), g.W - abs(u - a)) >= min_px or abs(v - b) >= min_px for a, b in keep):
            keep.append((u, v))
    return keep


def tie_scene(h, w, hf, vf, seed, mirror):
    """Tie groups around the anchors: a dyadic source s and 2 to 8 targets s + d, d signed permutations of one dyadic
    offset (exactly equidistant).  `mirror` negates every offset, a point reflection through s that keeps the
    distances and reverses both the row and the column order of the partners, so the lower id changes sides.
    -> targets [Nt, 3], sources [Ns, 3], and per source the [k, 3] targets of its group."""
    g = PR.Grid(h, w, hf, vf)
    gen = np.random.default_rng(seed)
    du, dv = pitch(g)
    tg, src, groups = [background(g, gen)], [], []
    unit = 2.0 ** -12
    for (u, v) in spaced(anchors(g, gen), 24, g):
        r = gen.uniform(6.0, 12.0)
        s = np.round(direction(g, u, v) * r / unit)
        # offsets of 0.3 to 8 px in angle, on the 2^-12 m lattice; signed permutations keep the exact norm
        mag = np.round(gen.uniform(0.3, 8.0, 3) * r * min(du, dv) / unit * gen.choice([1.0, 0.1], 3))
        mag = np.maximum(mag, 1.0)
        variants = sorted({tuple(sg * np.array(p)) for p in itertools.permutations(mag)
                           for sg in itertools.product((-1, 1), repeat=3)})
        k = int(gen.integers(2, 9))
        pick = [np.array(variants[i]) for i in gen.choice(len(variants), min(k, len(variants)), replace=False)]
        if mirror:
            pick = [-d for d in pick]
        groups.append(np.stack([(s + d) * unit for d in pick]).astype(np.float32))
        src.append((s * unit).astype(np.float32))
    # groups on the seam: s at azimuth 180 deg (y = 0), partners d and d with y negated, one in column 0 and one in
    # column W-1 (|y| about half a pixel)
    for v in np.linspace(1, g.H - 2, 3 if g.H > 3 else 1):
        r = gen.uniform(6.0, 12.0)
        el = g.vfov[0] + v / max(g.H - 1, 1) * (g.vfov[1] - g.vfov[0])
        s = np.round(np.array([-r * math.cos(el), 0.0, r * math.sin(el)]) / unit)
        ay = max(1.0, round(0.5 * r * du / unit))
        d = np.array([round(gen.uniform(-0.3, 0.3) * ay), ay, round(gen.uniform(-0.3, 0.3) * ay)])
        pick = [d, d * np.array([1, -1, 1])]
        if mirror:
            pick = [-x for x in pick]
        groups.append(np.stack([(s + x) * unit for x in pick]).astype(np.float32))
        src.append((s * unit).astype(np.float32))
    tg = np.concatenate(tg + groups)
    return tg, np.stack(src), groups


SEPS = (2.0 ** -44, 2.0 ** -40, 2.0 ** -30, 1e-7, 1e-6, 5e-6, 9e-6, 1.2e-5, 2e-5)


def near_tie_scene(h, w, hf, vf, sep, seed):
    """Sources s and pairs of targets s + D_A, s + D_B with D_A = (x, y, z), D_B = (y, x, z + 1) in units of 2^-20 m
    under a random signed axis permutation: |D_B|^2 - |D_A|^2 = 2 z + 1 exactly, so the relative separation is
    (2 z + 1) / |D_A|^2 ~ sep."""
    g = PR.Grid(h, w, hf, vf)
    gen = np.random.default_rng(seed)
    unit = 2.0 ** -20
    L = min(2.0 ** 22, 0.5 / sep)                                   # |D| in units; the offsets stay below 4 m
    z = max(0, int(round((sep * L * L - 1) / 2)))
    r_m = 8.0
    ang = L * unit / r_m                                            # angle the group spans (radians)
    du, dv = pitch(g)
    tg, src = [background(g, gen, r=40.0)], []
    for (u, v) in spaced(anchors(g, gen, 60), max(3.0, 3 * ang / min(du, dv)), g):
        s = np.round(direction(g, u, v) * r_m / unit)
        rest = L * L - z * z
        phi = gen.uniform(0, 2 * math.pi)
        x, y = int(round(math.sqrt(rest) * math.cos(phi))), int(round(math.sqrt(rest) * math.sin(phi)))
        da, db = np.array([x, y, z]), np.array([y, x, z + 1])
        perm, sign = gen.permutation(3), gen.choice([-1, 1], 3)
        da, db = sign * da[perm], sign * db[perm]
        tg.append(np.stack([(s + da) * unit, (s + db) * unit]).astype(np.float32))
        src.append((s * unit).astype(np.float32))
    return np.concatenate(tg), np.stack(src)

# ---- D: certification borders ------------------------------------------------------------------------------------
ROW_E = (1, 2, 3)          # row borders e rows out: e = 1 is the 3 x 5 start window's border
COL_E = (2, 3, 4, 6)       # column borders e columns out: e = 2 is the start window's border


def border_scene(h, w, hf, vf, seed):
    """Targets just beyond a border of the window search, not of the source's own cell.

    Each source sits at (us, vs) in cell (cc, rc), `f` px (0.001 to 0.49) inside its cell's edge on one side.  The
    border it is tested against lies e rows (cols) further out, at rc -/+ (e + 0.5) or cc -/+ (e + 0.5): the start
    window's border (e = 1 rows, 2 columns), a border the window reaches after growing, or the 4 x 16 block border
    on that side (the pending kernel's rectangle border at hand-over limit 0, e taken from the cell's place in its
    block).  Column borders include borders at and across the +-180 deg seam (cc at 0..2 or W-3..W-1).  The cells
    between the source and that border hold nothing but the far background.

    The nearest target lies beyond the border, at the foot of the perpendicular from the source on the border's
    plane (azimuth) or cone (elevation), pushed out along that perpendicular to (1 + rho) times the exact distance to
    the border, rho in {1e-5, 1e-4, 1e-3, 1e-2}: that distance is what the bound of the border computes before its
    slack and margin.  For row borders a third of the targets sit at a range 2 % above or below the foot's instead,
    where the range-extent bound (row_border_bound, range_lb2) is the tighter one.  A competitor on the source's own
    ray, inside the window, is (1 + gamma) times as far as the nearest, gamma in {1e-5, 1e-4, 1e-3}: the window
    search must not certify it.  -> targets [Nt, 3], sources [Ns, 3]."""
    g = PR.Grid(h, w, hf, vf)
    gen = np.random.default_rng(seed)
    du, dv = pitch(g)
    tg, src = [background(g, gen, r=60.0, fill=0.4)], []
    seam_cols = (0, g.W - 1, 1, g.W - 2, 2, g.W - 3)
    seam = [(seam_cols[k % 6], v) for k, v in enumerate(range(1, g.H - 1, 4))]
    cells = spaced(seam + list(zip(gen.integers(0, g.W, 6000), gen.integers(0, g.H, 6000))), 14, g)
    cells = [c for c in cells if c not in seam]
    for k, (cc, rc) in enumerate(seam + cells):
        in_seam = k < len(seam)
        if in_seam:
            side = 2 if cc <= 2 else 3
        else:
            side = int(gen.integers(0, 4))
        f = float(gen.choice([0.001, 0.01, 0.1, 0.49]))
        rho = float(gen.choice([1e-5, 1e-4, 1e-3, 1e-2]))
        gamma = float(gen.choice([1e-5, 1e-4, 1e-3]))
        r = gen.uniform(5.0, 12.0) if in_seam else gen.uniform(5.0, 30.0)
        to_block = gen.random() < 0.3
        if side in (0, 1):
            e = int(gen.choice(ROW_E))
            if to_block:                                            # the border of the source's 4-row block
                e = rc % 4 if side == 0 else 3 - rc % 4
                e = e if e >= 1 else e + 4
            vb = rc - e - 0.5 if side == 0 else rc + e + 0.5
            if not (-0.5 < vb < g.H - 0.5):
                continue
            vs = rc - 0.5 + f if side == 0 else rc + 0.5 - f
            us = cc + gen.uniform(-0.3, 0.3)
            s = direction(g, us, vs) * r
            gap = abs(vs - vb) * dv                                 # elevation from the source to the border cone
            foot = direction(g, us, vb) * r * math.cos(gap)
            kappa = float(gen.choice([0.0, 0.0, 0.02, -0.02]))
            if kappa:                                               # on the cone at another range
                foot = direction(g, us, vb) * r * (1.0 + kappa)
        else:
            e = int(gen.choice(COL_E[:2] if in_seam else COL_E))
            if to_block and not in_seam:                            # the border of the source's 16-column block
                e = cc % 16 if side == 2 else 15 - cc % 16
                e = e if e >= 2 else e + 16
            ub = cc - e - 0.5 if side == 2 else cc + e + 0.5
            us = cc - 0.5 + f if side == 2 else cc + 0.5 - f
            vs = rc + gen.uniform(-0.3, 0.3)
            s = direction(g, us, vs) * r
            ub_w = ub % g.W                                         # the same border on the circle
            az_s = math.atan2(s[1], s[0])
            dirb = direction(g, ub_w, vs)
            az_b = math.atan2(dirb[1], dirb[0])
            gap = abs((az_s - az_b + math.pi) % (2 * math.pi) - math.pi)
            if gap >= math.pi / 2:
                continue
            rxy = math.hypot(s[0], s[1])
            foot = np.array([math.cos(az_b) * rxy * math.cos(gap), math.sin(az_b) * rxy * math.cos(gap), s[2]])
        d = foot - s
        t_nn = s + d * (1.0 + rho)
        d_nn = np.linalg.norm(d) * (1.0 + rho)
        t_c = s / r * (r + d_nn * (1.0 + gamma))
        tg.append(np.stack([t_nn, t_c]).astype(np.float32))
        src.append(s.astype(np.float32))
    return np.concatenate(tg), np.stack(src)

# ---- E, F, G, H: degenerate sources, degenerate targets, grid shapes, documented limits --------------------------
def scan_points(h, w_raw, vfov, seed=40):
    from delora_b200 import synthetic
    s1, s2, _, _ = synthetic.make_pair(seed, w_raw=w_raw, rings=h, vfov_deg=vfov)
    return s1.numpy().T, s2.numpy().T

def degenerate_source_scenes(limits=LIMITS_DEFAULT):
    """Sources at the origin, on the z axis, 1e-3 m and 1e4 m away, 0.4 and 50 px outside the vertical field of view
    and outside a partial horizontal one, on 16x180 grids of the full and of a (-90, 90) deg horizontal field of view:
    each degenerate source once alone in its warp and once among ordinary warp-mates."""
    h, w = 16, 180
    vfd = (-15.0, 15.0)
    gen = np.random.default_rng(9)
    tgt, src = scan_points(h, 192, vfd)
    for hf in (HF, deg(-90.0, 90.0)):
        g = PR.Grid(h, w, hf, deg(*vfd))
        odd = [np.zeros(3), [0, 0, 5.0], [0, 0, -5.0], [0, 0, 1e-3], [1e-30, 0, 7.0]]
        dirs = direction(g, gen.uniform(0, w - 1, 12), gen.uniform(0, h - 1, 12))
        odd += list(dirs * 1e-3) + list(dirs * 1e4)
        for out_px in (0.4, 50.0):
            odd += list(direction(g, gen.uniform(0, w - 1, 6), np.full(6, -0.5 - out_px)) * 8.0)
            odd += list(direction(g, gen.uniform(0, w - 1, 6), np.full(6, h - 0.5 + out_px)) * 8.0)
        odd += list(direction(g, gen.uniform(w, 1.5 * w, 8), gen.uniform(0, h - 1, 8)) * 8.0)   # beyond the hfov
        odd = np.asarray(odd, np.float32)
        mixed = np.concatenate([src[:2000], odd, src[2000:2400]])
        slots = np.concatenate([np.arange(len(odd)) * 32, 32 * len(odd) + np.arange(len(mixed))])
        yield Scene(f"16x180 hfov {math.degrees(hf[1]):.1f}", h, w, hf, g.vfov, tgt, np.concatenate([odd, mixed]),
                    slots, limits=limits)


def degenerate_target_scenes(limits=LIMITS_DEFAULT):
    """16x180 target grids of one target, only row 0 or row H-1, one column, 4 x 16 blocks side by side at 1e-3 m and
    1e3 m, and none (M = 0), under 1500 sources of a scan."""
    h, w = 16, 180
    vf = deg(-15.0, 15.0)
    g = PR.Grid(h, w, HF, vf)
    gen = np.random.default_rng(4)
    tgt, src = scan_points(h, 192, (-15.0, 15.0))
    src = src[gen.choice(len(src), 1500, replace=False)]
    pr = PR.project(tgt.T, h, w, HF, vf)
    pix = pr["pixel"]
    row = np.where(pix >= 0, pix // w, -1)
    col = np.where(pix >= 0, pix % w, -1)
    one = tgt[pix >= 0][:1]
    near_far = []
    for bc in range(0, 10, 2):
        for k, rr in ((bc, 1e-3), (bc + 1, 1e3)):
            uu, vv = np.meshgrid(np.arange(16 * k, 16 * k + 16) + 0.1, np.arange(4, 8) + 0.1)
            near_far.append(direction(g, uu.ravel(), vv.ravel()) * rr)
    scenes = [("one target", one), ("row 0 only", tgt[row == 0]), ("row H-1 only", tgt[row == h - 1]),
              ("one column", tgt[col == 77]), ("1e-3 m / 1e3 m blocks", np.concatenate(near_far)),
              ("empty", np.zeros((0, 3)))]
    for name, t in scenes:
        yield Scene(f"16x180 {name}", h, w, HF, vf, t, src, limits=limits)


SHAPES_G = [(h, w, HF, deg(-15.0, 15.0)) for h in (1, 2) for w in (3, 4, 5, 7)] + [
    (18, 37, HF, deg(-15.0, 15.0)), (16, 180, deg(-90.0, 90.0), deg(-15.0, 15.0)),
    (32, 360, HF, deg(-30.0, 89.5)), (16, 180, HF, deg(-89.5, 89.5))]


def random_points(g, gen, n, r_lo=0.5, r_hi=60.0):
    return PR.random_cloud(gen, n, g, r_lo, r_hi).T


SHAPES_H = [(4, 8977, HF, deg(-15.0, 15.0)), (4, 12000, HF, deg(-15.0, 15.0)),
            (361, 64, HF, deg(-15.0, 15.0)), (512, 64, HF, deg(-15.0, 15.0))]
