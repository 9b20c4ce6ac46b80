"""The list path of the ICP operators restated on the CPU (test infrastructure), and the decoy scenes that tell a right
binning of out-of-field azimuths from a wrong one.

delora_grid_build (csrc/lists.cu, cell_of) sorts arbitrary target lists by spherical cell; delora_icp_fwd_bwd
(csrc/icp.cu, nn_search) searches a window of cells around each source and stops once the best distance found is below
the exactness bound of every window border.  That bound is sound only if every target sits inside the arc of azimuths
its column stands for.  Here, in numpy float32:
  - `Grid` holds make_grid's float32 constants (csrc/common.cuh), `uv` the operators' pixel coordinates (libdevice-like
    atan2f and a * (1 / span), the CUDA arithmetic the list path uses);
  - `columns` bins azimuths by either rule: "clamp", the plain clamp of rint(u) into [0, W - 1] (an out-of-field azimuth
    goes to column 0 when u < 0 and to column W - 1 when u > W - 1, which splits the gap where atan2 wraps at +-pi),
    and "nearer", the border column nearer to the azimuth around the circle (what cell_of does);
  - `search` is nn_search's window growth and stopping rule on a given binning: which cells it scans, when it stops,
    which target it returns.  Ranking is exact (float64, lowest list index on ties); only the stopping rule is float32.
  - `decoy_scene` builds, at one seam edge of a grid, sources two columns inside the field and a target T in the gap
    just beyond the border column, at the source's range and elevation, plus a decoy D on the source's own ray, farther
    than T but nearer than the exactness bound of the start window's border on T's side.  When T is binned into the
    border column on the far side of the field, the window search stops on D without scanning T's cell.

`hfov_cases(W)` lists the horizontal fields of view the decoy scenes run on: one-sided gaps [-pi, pi - g] and
[-pi + g, pi] for g in {0.3, 0.6, 1, 2} column pitches, g = 2 pi / W, [-pi, 0], [-pi/4, pi/4] and the reference's
[-179.9, 179.9] deg.  Read literally, the clamp rule breaks the bound only for a one-sided gap wider than half a pitch;
`sharp_edge` names the edge where it does (None for the controls).
"""
import math

import numpy as np

F32 = np.float32
TWO_PI = 6.283185307179586


class Grid:
    """make_grid (csrc/common.cuh) for div_mode 1, in float32."""

    def __init__(self, h, w, hfov, vfov):
        self.H, self.W = int(h), int(w)
        hf0, hf1 = float(hfov[0]), float(hfov[1])
        vf0, vf1 = float(vfov[0]), float(vfov[1])
        self.hfov, self.vfov = (hf0, hf1), (vf0, vf1)
        self.hf0, self.hspan, self.wm1 = F32(hf0), F32(hf1 - hf0), F32(w - 1)
        self.vf0, self.vspan, self.hm1 = F32(vf0), F32(vf1 - vf0), F32(h - 1)
        self.hinv, self.vinv = F32(1.0) / self.hspan, F32(1.0) / self.vspan
        self.du_rad = F32((hf1 - hf0) / (w - 1)) if w > 1 else F32(1.0)
        self.dv_rad = F32((vf1 - vf0) / (h - 1)) if h > 1 else F32(1.0)
        self.seam_px = max(F32(0.0), F32(1.0) - F32((TWO_PI - (hf1 - hf0)) / float(self.du_rad)))
        self.circ_px = F32(TWO_PI / float(self.du_rad))
        # float64 pitches and the gap in pixels, for building scenes
        self.du = (hf1 - hf0) / max(w - 1, 1)
        self.dv = (vf1 - vf0) / max(h - 1, 1)
        self.gap_px = TWO_PI / self.du - (w - 1)


def uv(g, x, y, z):
    """float32 (u, v) of points: atan2f, then (a - f0) * (1 / span) * (n - 1) rounded after every operation."""
    x, y, z = (np.asarray(a, F32) for a in (x, y, z))
    with np.errstate(all="ignore"):
        a_h = np.arctan2(y, x).astype(F32)
        rxy = np.sqrt(x * x + y * y).astype(F32)
        a_v = np.arctan2(z, rxy).astype(F32)
        u = ((a_h - g.hf0) * g.hinv) * g.wm1
        v = ((a_v - g.vf0) * g.vinv) * g.hm1
    return u.astype(F32), v.astype(F32)


def columns(g, u, rule):
    """Column of every u: rint(u) inside the field; outside it, by `rule` ("clamp" or "nearer", see the module
    docstring).  NaN goes to column 0."""
    u = np.asarray(u, F32)
    with np.errstate(invalid="ignore"):
        ru = np.rint(u)
        if rule == "nearer":
            out = (ru < 0) | (ru > g.wm1)
            past = np.where(u > g.wm1, u - g.wm1, (u + g.circ_px) - g.wm1).astype(F32)
            half = F32(0.5) * (g.circ_px - g.wm1)
            ru = np.where(out, np.where(past <= half, g.wm1, F32(0.0)), ru)
        else:
            assert rule == "clamp", rule
    return np.clip(np.nan_to_num(ru, nan=0.0), 0, g.W - 1).astype(np.int64)


def rows(g, v):
    with np.errstate(invalid="ignore"):
        return np.clip(np.nan_to_num(np.rint(np.asarray(v, F32)), nan=0.0), 0, g.H - 1).astype(np.int64)


def cells(g, pts, rule):
    """Cell id (row * W + column) of every target [N, 3] under `rule`."""
    pts = np.asarray(pts, F32).reshape(-1, 3)
    u, v = uv(g, pts[:, 0], pts[:, 1], pts[:, 2])
    return rows(g, v) * g.W + columns(g, u, rule)


class Binned:
    """A target list [N, 3] binned by `rule`: per cell the list indices it holds."""

    def __init__(self, g, tgt, rule):
        self.g, self.tgt = g, np.asarray(tgt, F32).reshape(-1, 3)
        self.t64 = self.tgt.astype(np.float64)
        self.cell = cells(g, self.tgt, rule)
        order = np.argsort(self.cell, kind="stable")
        self.order = order
        self.start = np.searchsorted(self.cell[order], np.arange(g.H * g.W + 1))

    def in_cells(self, row, c0, c1):
        """List indices in row `row`, columns c0..c1 (unwrapped, c1 - c0 + 1 <= W)."""
        W = self.g.W
        out = []
        for c in range(c0, c1 + 1):
            k = row * W + c % W
            out.append(self.order[self.start[k]:self.start[k + 1]])
        return np.concatenate(out) if out else np.zeros(0, np.int64)


def _sinf(a):
    return F32(math.sin(float(a)))


def search(b, s):
    """nn_search (csrc/icp.cu) for one float32 source s on the binned targets b.
    -> (list index of the target it returns or -1, (r_lo, r_hi, c_lo, c_hi) of the window it stopped with, the border
    bounds (down, up, left, right) it stopped on)."""
    g = b.g
    H, W = g.H, g.W
    sx, sy, sz = (F32(c) for c in s)
    if len(b.tgt) == 0:
        return -1, None, None
    us, vs = uv(g, sx, sy, sz)
    us, vs = F32(0.0) if us != us else F32(us), F32(0.0) if vs != vs else F32(vs)
    rxy = F32(math.sqrt(float(F32(sx * sx + sy * sy))))
    r = F32(math.sqrt(float(F32(sx * sx + sy * sy + sz * sz))))
    cc = int(min(max(np.rint(us), 0), W - 1))
    rc = int(min(max(np.rint(vs), 0), H - 1))
    r_lo, r_hi = max(rc - 1, 0), min(rc + 1, H - 1)
    half = min(2, (W - 1) // 2)
    c_lo, c_hi = cc - half, cc + half
    s64 = np.array([sx, sy, sz], np.float64)
    best = [np.inf, -1]

    def scan(idx):
        if len(idx) == 0:
            return
        d2 = ((b.t64[idx] - s64) ** 2).sum(1)
        k = np.lexsort((idx, d2))[0]
        if d2[k] < best[0] or (d2[k] == best[0] and idx[k] < best[1]):
            best[0], best[1] = d2[k], int(idx[k])

    for row in range(r_lo, r_hi + 1):
        scan(b.in_cells(row, c_lo, c_hi))
    half_pi, slack, inf = F32(math.pi / 2), F32(2e-3), F32(3.0e38)
    while True:
        b_dn = b_up = b_lf = b_rt = inf
        if r_lo > 0:
            d = (vs - (F32(r_lo) - F32(0.5)) - slack) * g.dv_rad
            b_dn = F32(0.0) if d <= 0 else r * _sinf(min(d, half_pi))
        if r_hi < H - 1:
            d = ((F32(r_hi) + F32(0.5)) - vs - slack) * g.dv_rad
            b_up = F32(0.0) if d <= 0 else r * _sinf(min(d, half_pi))
        width = c_hi - c_lo + 1
        if width < W:
            dl = (us - (F32(c_lo) - F32(0.5)) - slack - (g.seam_px if c_lo <= 0 else F32(0.0))) * g.du_rad
            dr = ((F32(c_hi) + F32(0.5)) - us - slack - (g.seam_px if c_hi >= W - 1 else F32(0.0))) * g.du_rad
            b_lf = F32(0.0) if dl <= 0 else rxy * _sinf(min(dl, half_pi))
            b_rt = F32(0.0) if dr <= 0 else rxy * _sinf(min(dr, half_pi))
        bmin = min(b_dn, b_up, b_lf, b_rt)
        if bmin >= inf:
            break
        if best[1] >= 0 and F32(math.sqrt(best[0])) * F32(1.00001) <= bmin * F32(0.9995):
            break
        if bmin == b_dn:
            r_lo -= 1
            scan(b.in_cells(r_lo, c_lo, c_hi))
        elif bmin == b_up:
            r_hi += 1
            scan(b.in_cells(r_hi, c_lo, c_hi))
        elif bmin == b_lf:
            step = min(2, W - width)
            for row in range(r_lo, r_hi + 1):
                scan(b.in_cells(row, c_lo - step, c_lo - 1))
            c_lo -= step
        else:
            step = min(2, W - width)
            for row in range(r_lo, r_hi + 1):
                scan(b.in_cells(row, c_hi + 1, c_hi + step))
            c_hi += step
    return best[1], (r_lo, r_hi, c_lo, c_hi), (b_dn, b_up, b_lf, b_rt)


# ---- fields of view and decoy scenes -----------------------------------------------------------------------------
def gap_for(k, w):
    """The gap g = 2 pi - hspan that is k column pitches wide: g = k (2 pi - g) / (W - 1)."""
    return TWO_PI * k / (w - 1 + k)


def hfov_cases(w):
    """[(name, (hf0, hf1), sharp_edge)]: sharp_edge is the seam edge ("left": next to column 0, "right": next to
    column W - 1) where the clamp rule puts a gap azimuth into the far border column closer to the source than the
    window search assumes; None where it never does."""
    out = []
    for k in (0.3, 0.6, 1.0, 2.0):
        g = gap_for(k, w)
        sharp = k > 0.5
        out.append((f"[-pi,pi-{k:g}du]", (-math.pi, math.pi - g), "left" if sharp else None))
        out.append((f"[-pi+{k:g}du,pi]", (-math.pi + g, math.pi), "right" if sharp else None))
    out.append(("[-pi,pi-2pi/W]", (-math.pi, math.pi - TWO_PI / w), "left"))
    out.append(("[-pi,0]", (-math.pi, 0.0), "left"))
    out.append(("[-pi/4,pi/4]", (-math.pi / 4, math.pi / 4), None))
    out.append(("[-179.9,179.9]deg", (math.radians(-179.9), math.radians(179.9)), None))
    return out


HFOV_NAMES = [c[0] for c in hfov_cases(180)]
DECOY_GRIDS = [(16, 180, (math.radians(-15.0), math.radians(15.0))),
               (64, 720, (math.radians(-24.5), math.radians(2.0))),
               (64, 2048, (math.radians(-24.5), math.radians(2.0)))]


def _xyz(r, az, el):
    return np.array([r * math.cos(el) * math.cos(az), r * math.cos(el) * math.sin(az), r * math.sin(el)])


def decoy_scene(g, edges=("left", "right"), ranges=(6.0, 12.0, 24.0), offsets=(1.6, 2.3)):
    """Decoy scenes at the seam edges of grid g (see the module docstring).

    Per edge, row band (a fifth, a half and four fifths of the way up) and range: a source S at pixel column `us`
    (1.6 or 2.3 columns inside the border column), T at the source's range and elevation a = min(0.02, 0.02 G) px past
    the border column into the gap (G: the gap in pixels), and D on the ray of S at distance
    sqrt(|S - T| * bound) from S, `bound` being the exactness bound of the start window's border on T's side, when that
    bound exceeds |S - T| by more than 2 %; else (the bound is sound: T lies beyond it) D at 1.03 |S - T|.
    -> dict: tgt [Nt, 3], src [Ns, 3] float32, t_idx, d_idx [Ns] (list indices of each source's T and D), edge [Ns],
    sharp [Ns] bool (D lies below the bound: a search that does not scan T's cell returns D)."""
    G = g.gap_px
    a = min(0.02, 0.02 * G)
    tgt, src, t_idx, d_idx, edge_of, sharp = [], [], [], [], [], []
    for edge in edges:
        for i, frac in enumerate((0.2, 0.5, 0.8)):
            v = round(frac * (g.H - 1)) + 0.1
            el = g.vfov[0] + v * g.dv
            for j, r in enumerate(ranges):
                us = offsets[(i + j) % len(offsets)]
                if edge == "left":
                    u_s, u_t = us, -a
                else:
                    u_s, u_t = (g.W - 1) - us, (g.W - 1) + a
                s = _xyz(r, g.hfov[0] + u_s * g.du, el).astype(F32)
                t = _xyz(r, g.hfov[0] + u_t * g.du, el).astype(F32)
                d_t = float(np.linalg.norm(s.astype(np.float64) - t.astype(np.float64)))
                rxy = math.hypot(float(s[0]), float(s[1]))
                seam = float(g.seam_px)
                # the start window's border on T's side: c_lo = 0 (left) or c_hi = W - 1 (right)
                ang = (us + 0.5 - 2e-3 - seam) * float(g.du_rad)
                bound = rxy * math.sin(min(max(ang, 0.0), math.pi / 2))
                is_sharp = bound > 1.02 * d_t
                d_d = math.sqrt(d_t * bound) if is_sharp else 1.03 * d_t
                rs = float(np.linalg.norm(s.astype(np.float64)))
                dd = (s.astype(np.float64) * ((rs + d_d) / rs)).astype(F32)
                t_idx.append(len(tgt))
                tgt.append(t)
                d_idx.append(len(tgt))
                tgt.append(dd)
                src.append(s)
                edge_of.append(edge)
                sharp.append(is_sharp)
    return dict(tgt=np.array(tgt, F32), src=np.array(src, F32), t_idx=np.array(t_idx), d_idx=np.array(d_idx),
                edge=np.array(edge_of), sharp=np.array(sharp))
