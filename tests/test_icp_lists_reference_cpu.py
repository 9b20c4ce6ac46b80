"""The decoy scenes of the list ICP operator are sharp, on the CPU (tests/lists_reference.py).

Restated in numpy float32, nn_search's window growth and stopping rule (csrc/icp.cu) returns the decoy D instead of the
true nearest neighbour T for every source at the sharp seam edge of a one-sided gap wider than half a column pitch when
the targets are binned by the plain clamp of rint(u); it returns T for every source of every scene when out-of-field
azimuths go to the border column nearer around the circle (csrc/lists.cu, cell_of).  The controls (a gap of 0.3
pitches, the symmetric fields of view) return T under both rules.  Each sharp scene keeps margins of 1 % between |S - T|,
|S - D| and the border's bound, far above the float32 differences between this restatement and the kernel's arithmetic
(libdevice atan2f, __sinf).

The binning rule itself: over the whole circle of azimuths, the nearer-border rule keeps every target inside the arc
of its column (half a pitch on either side; for the border columns, up to half the gap into it), which is what the
window search's border bounds assume; the clamp rule breaks that exactly for the sharp fields of view.
"""
import math

import numpy as np
import pytest

import lists_reference as LR
import nn_reference as NR


def _case(grid, name):
    h, w, vf = grid
    for case_name, hf, sharp_edge in LR.hfov_cases(w):
        if case_name == name:
            return LR.Grid(h, w, hf, vf), sharp_edge
    raise KeyError(name)


@pytest.mark.parametrize("grid", LR.DECOY_GRIDS, ids=[f"{h}x{w}" for h, w, _ in LR.DECOY_GRIDS])
@pytest.mark.parametrize("name", LR.HFOV_NAMES)
def test_decoy_scenes_stop_before_the_true_neighbour_under_the_clamp(grid, name):
    g, sharp_edge = _case(grid, name)
    sc = LR.decoy_scene(g)
    ref = NR.nearest(sc["tgt"], np.arange(len(sc["tgt"])), sc["src"])
    assert len(ref.unsafe) == 0 and (ref.ties == 1).all()
    assert np.array_equal(ref.nn, sc["t_idx"]), "T is every source's exact nearest target"
    clamp, nearer = LR.Binned(g, sc["tgt"], "clamp"), LR.Binned(g, sc["tgt"], "nearer")
    for i, s in enumerate(sc["src"]):
        got_c, win, bounds = LR.search(clamp, s)
        got_n, _, _ = LR.search(nearer, s)
        assert got_n == sc["t_idx"][i], f"{name} source {i}: the nearer-border binning misses T"
        if sc["edge"][i] == sharp_edge:
            assert sc["sharp"][i]
            assert got_c == sc["d_idx"][i], f"{name} source {i}: the clamp binning does not stop on the decoy"
            # T's cell lies outside the window the search stopped with
            r_lo, r_hi, c_lo, c_hi = win
            t_cell = clamp.cell[sc["t_idx"][i]]
            t_row, t_col = divmod(int(t_cell), g.W)
            in_cols = any((c % g.W) == t_col for c in range(c_lo, c_hi + 1))
            assert not (r_lo <= t_row <= r_hi and in_cols), f"{name} source {i}: T's cell was scanned"
            # margins far above the float32 differences of the kernel's arithmetic
            s64 = s.astype(np.float64)
            d_t = np.linalg.norm(s64 - sc["tgt"][sc["t_idx"][i]])
            d_d = np.linalg.norm(s64 - sc["tgt"][sc["d_idx"][i]])
            side = bounds[2] if sc["edge"][i] == "left" else bounds[3]
            assert d_t * 1.01 < d_d < float(side) / 1.01, (name, i, d_t, d_d, side)
        else:
            assert got_c == sc["t_idx"][i], f"{name} source {i}: a control scene misses T under the clamp binning"


def _arc_offsets(g, rule, n=200001):
    """Azimuths over the whole circle (kept 1e-3 px away from every rounding boundary and from the gap's midpoint) ->
    (column under `rule`, float64 offset of the azimuth from that column's centre in pixels, wrapped to (-C/2, C/2])."""
    az = np.linspace(-math.pi, math.pi, n)
    p = (az - g.hfov[0]) / g.du                             # float64 pixel position
    circ = 2 * math.pi / g.du
    frac = np.abs((p - 0.5) - np.rint(p - 0.5))
    past = np.mod(p - (g.W - 1), circ)
    keep = (frac > 1e-3) & (np.abs(past - g.gap_px / 2) > 1e-3)
    az = az[keep]
    x, y = np.cos(az).astype(np.float32), np.sin(az).astype(np.float32)
    u, _ = LR.uv(g, x, y, np.zeros_like(x))
    col = LR.columns(g, u, rule)
    pos = (np.arctan2(y.astype(np.float64), x.astype(np.float64)) - g.hfov[0]) / g.du
    off = np.mod(pos - col + circ / 2, circ) - circ / 2
    return col, off


@pytest.mark.parametrize("w", [180, 720, 2048])
@pytest.mark.parametrize("name", LR.HFOV_NAMES)
def test_every_column_keeps_its_arc_under_the_nearer_rule(w, name):
    h, _, vf = next(x for x in LR.DECOY_GRIDS if x[1] == w)
    g, sharp_edge = _case((h, w, vf), name)
    ext = max(0.5, g.gap_px / 2) + 1e-3

    def violations(rule):
        col, off = _arc_offsets(g, rule)
        lo = np.where(col == 0, -ext, -0.5 - 1e-3)
        hi = np.where(col == g.W - 1, ext, 0.5 + 1e-3)
        return int(((off < lo) | (off > hi)).sum())

    assert violations("nearer") == 0
    if sharp_edge is None:
        assert violations("clamp") == 0
    else:
        assert violations("clamp") > 0, "the clamp rule puts some gap azimuth outside its column's arc"
