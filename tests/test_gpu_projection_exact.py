"""-m gpu: the projection kernels against tests/projection_reference.py, the float32 restatement of the reference's
projection, on seeded adversarial clouds, with no allowance anywhere (div_mode 0, the reference's torch-CPU
arithmetic).

Every (u, v) and range the device computes must be bit-identical to the restatement's; every channel of every image
and every index map must be bit-identical too.  The clouds (projection_reference's families):
  F1 boundaries  u or v exactly on k + 0.5, one ulp below or above it;
  F2 seam        x < 0 with y = +-0 and +-the smallest subnormal, and points at the four field-of-view edges;
  F3 magnitudes  |x|, |y| < 2^-128 (the atan2's rescaling branch), subnormals, signed zeros, the origin, the z axis,
                 squares that overflow (range +inf with a pixel);
  F4 nonfinite   NaN or +-inf in one coordinate, +-inf in two;
  F5 ties        equal ranges in one pixel (duplicates, permuted coordinates, 64 copies), and closer points stored
                 beyond n_points that must not take part;
  F6 shapes      H in {1, 15, 16, 17} x W in {1, 2, 31, 33, 180, 2250}, n around the scatter's 1024-point blocks, a
                 ragged batch, C = 3, 4, 5.
The last test shows the harness is sharp: div_mode 1 (libdevice atan2f and a reciprocal multiply, an ulp-level
change of the arithmetic) must be reported, with pixel flips on F1 and float mismatches on a realistic scan.
NaNs compare equal to NaNs whatever their payload (projection_reference.same): the reference's payloads are x86's.
"""

import numpy as np
import pytest
import torch

import projection_reference as pr

pytestmark = pytest.mark.gpu

DEV = "cuda"
GARBAGE = 7          # columns past n_points in every call: closer copies of valid points, which must not take part

# (fov, H, W) of the family tests
GRIDS = [("full", 64, 2250), ("synthetic", 64, 720), ("narrow", 16, 180), ("sphere", 17, 33)]


def with_channels(cloud, c, seed):
    """cloud [3, n] -> [c, n]: further channels random, NaNs (several payloads) and infinities among them."""
    if c == 3:
        return cloud
    gen = np.random.default_rng(seed)
    extra = gen.standard_normal((c - 3, cloud.shape[1])).astype(np.float32)
    extra[:, ::13] = np.array([0x7FA5A5A5], np.uint32).view(np.float32)[0]
    extra[:, 3::17] = np.inf
    extra[:, 6::19] = -0.0
    return np.concatenate((cloud, extra), axis=0)


def with_garbage(cloud, seed):
    """[c, n] -> [c, n + GARBAGE]: past the count, half-scale copies of valid points (the same pixel, a smaller range;
    a power-of-two scale leaves the atan2 bits alone) and the origin."""
    gen = np.random.default_rng(seed)
    c, n = cloud.shape
    if n:
        g = cloud[:, gen.integers(0, n, GARBAGE)].copy()
        g[:3] *= np.float32(0.5)
    else:
        g = np.ones((c, GARBAGE), np.float32)
    g[:3, -1] = 0.0
    return np.concatenate((cloud, g), axis=1)


def batch(clouds, seed=0, full_row=None):
    """list of [c, n_b] -> points [B, c, n_stride] on the device, counts [B] int32.  Every row but `full_row` is
    followed by garbage; row `full_row` has no garbage and its count must be n_stride."""
    rows = [cl if i == full_row else with_garbage(cl, seed + i) for i, cl in enumerate(clouds)]
    stride = max(r.shape[1] for r in rows)
    assert full_row is None or clouds[full_row].shape[1] == stride
    pts = np.zeros((len(rows), rows[0].shape[0], stride), np.float32)
    for i, r in enumerate(rows):
        pts[i, :, :r.shape[1]] = r
        pts[i, :, r.shape[1]:] = r[:, -1:]
    n = torch.tensor([cl.shape[1] for cl in clouds], dtype=torch.int32, device=DEV)
    return torch.from_numpy(pts).to(DEV), n


def report(clouds, h, w, fov, div_mode=0, normals=False, seed=0, full_row=None):
    """Run project_uv, project (and project_normals) on the batch of clouds and count every difference from the
    restatement.  -> dict of counts, all zero for an exact kernel."""
    from delora_b200 import ops
    hfov, vfov = pr.FOVS[fov]
    pts, n = batch(clouds, seed, full_row)
    u, v, r = (t.cpu().numpy() for t in ops.project_uv(pts, n, h, w, hfov, vfov, div_mode))
    image, imap = (t.cpu().numpy() for t in ops.project(pts, n, h, w, hfov, vfov, div_mode))
    g = pr.Grid(h, w, hfov, vfov)
    out = dict(u=0, v=0, r=0, flips=0, image=0, index_map=0)
    for b, cl in enumerate(clouds):
        k = cl.shape[1]
        ref = pr.project(cl, h, w, hfov, vfov)
        out["u"] += int((~pr.same(u[b, :k], ref["u"])).sum())
        out["v"] += int((~pr.same(v[b, :k], ref["v"])).sum())
        out["r"] += int((~pr.same(r[b, :k], ref["r"])).sum())
        out["flips"] += int((pr.pixels(g, u[b, :k], v[b, :k]) != ref["pixel"]).sum())
        out["image"] += int((image[b].view(np.int32) != ref["image"].view(np.int32)).sum())
        out["index_map"] += int((imap[b] != ref["index_map"]).sum())
    if normals:
        img_n, imap_n, pg, ng = ops.project_normals(pts, n, h, w, hfov, vfov, div_mode=div_mode)
        pg_r, ng_r = ops.normals(img_n, grids=True)[1:]
        out["normals_image"] = int((img_n.cpu().numpy().view(np.int32) != image.view(np.int32)).sum())
        out["normals_index_map"] = int((imap_n.cpu().numpy() != imap).sum())
        out["pts_grid"] = int((pg.view(torch.int32) != pg_r.view(torch.int32)).sum())
        out["nrm_grid"] = int((ng.view(torch.int32) != ng_r.view(torch.int32)).sum())
    return out


def assert_exact(rep, label):
    print(f"{label}: {rep}")
    assert not any(rep.values()), f"{label}: differs from the float32 restatement: {rep}"


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{g[0]}_{g[1]}x{g[2]}" for g in GRIDS])
@pytest.mark.parametrize("name", list(pr.FAMILIES))
def test_families_exact(name, grid, cuda_lib):
    """F1-F5 at C = 3 and 4 through project_uv, project and project_normals, and at C = 5 (the generic resolve)."""
    fov, h, w = grid
    cloud = pr.family(name, 23, h, w, fov)
    for c in (3, 4, 5):
        assert_exact(report([with_channels(cloud, c, c)], h, w, fov, normals=c < 5),
                     f"{name} {fov} {h}x{w} C={c} n={cloud.shape[1]}")


SHAPES_H = (1, 15, 16, 17)
SHAPES_W = (1, 2, 31, 33, 180, 2250)


@pytest.mark.parametrize("h", SHAPES_H)
def test_shapes_exact(h, cuda_lib):
    """F6: every H x W of the grid above (the resolve's scalar tail where H W is not a multiple of 4, the fused kernel's
    32 x 16 tile edges) with n in {0, 1, 1023, 1024, 1025}, C cycling through 3, 4, 5."""
    for j, w in enumerate(SHAPES_W):
        fov = ("narrow", "full")[j % 2]
        g = pr.Grid(h, w, *pr.FOVS[fov])
        gen = np.random.default_rng(100 * h + w)
        pool = np.concatenate((pr.boundary_cloud(gen, g, n_u=24, ranges=(1.3, 17.0)), pr.random_cloud(gen, 1100, g)),
                              axis=1)
        pool = pool[:, gen.permutation(pool.shape[1])]
        for i, n in enumerate((0, 1, 1023, 1024, 1025)):
            c = (3, 4, 5)[(i + j) % 3]
            cl = with_channels(np.ascontiguousarray(pool[:, :n]), c, n)
            assert_exact(report([cl], h, w, fov, normals=c < 5, seed=n), f"{fov} {h}x{w} n={n} C={c}")


def test_ragged_batch_exact(cuda_lib):
    """B = 3 with counts n_stride, 0 and a ragged count; the rows past each count hold closer copies of its points."""
    h, w, fov = 64, 720, "synthetic"
    for c in (3, 4):
        a = with_channels(pr.family("boundaries", 5, h, w, fov), c, 1)
        b = with_channels(pr.family("ties", 6, h, w, fov), c, 2)[:, :777]
        empty = np.zeros((c, 0), np.float32)
        assert a.shape[1] > b.shape[1] + GARBAGE
        assert_exact(report([a, empty, b], h, w, fov, normals=True, full_row=0), f"ragged C={c}")


def test_grids_exact(cuda_lib):
    """project_grids on dense grids built directly: adversarial coordinates in valid cells (w = the cell's pixel-id
    bits) mixed with invalid cells (w < 0, holding closer points that must be ignored), re-projected at W != Wp.  The
    reference is the restatement on the valid cells in row-major order with the cell id as the tie-break."""
    from delora_b200 import ops
    for h, wp, w, fov in ((16, 180, 33, "narrow"), (64, 720, 2250, "full"), (17, 31, 180, "sphere")):
        hfov, vfov = pr.FOVS[fov]
        gen = np.random.default_rng(wp)
        n_cells = h * wp
        pool = np.concatenate([pr.family(nm, 9, h, w, fov) for nm in pr.FAMILIES], axis=1)
        s_count = 2
        pre = np.empty((s_count, n_cells, 4), np.float32)
        nrm = gen.standard_normal((s_count, n_cells, 4)).astype(np.float32)
        nrm[:, ::5, :3] = 0.0                                                 # cells without a normal
        refs = []
        for s in range(s_count):
            pick = pool[:, gen.integers(0, pool.shape[1], n_cells)].T
            valid = gen.random(n_cells) < 0.7
            with np.errstate(invalid="ignore"):                              # signalling NaNs among the picks
                pre[s, :, :3] = np.where(valid[:, None], pick, pick * np.float32(0.5))
            pre[s, :, 3] = np.where(valid, np.arange(n_cells, dtype=np.int32),
                                    -gen.integers(1, 5, n_cells).astype(np.int32)).view(np.float32)
            ids = np.nonzero(valid)[0]
            refs.append((pr.project(pre[s, ids, :3].T.copy(), h, w, hfov, vfov, ids=ids), nrm[s]))
        image, imap, pg, ng = ops.project_grids(torch.from_numpy(pre).to(DEV), torch.from_numpy(nrm).to(DEV), h, wp, w,
                                                hfov, vfov)
        image, imap, pg, ng = (t.cpu().numpy() for t in (image, imap, pg, ng))
        for s, (ref, nr) in enumerate(refs):
            cell = ref["index_map"].ravel()
            hit = cell >= 0
            pix = np.arange(h * w)
            pg_r = np.empty((h * w, 4), np.float32)
            pg_r[:, :3] = np.where(hit[:, None], ref["image"][:3].reshape(3, -1).T, np.float32(np.inf))
            pg_r[:, 3] = np.where(hit, pix, -1).astype(np.int32).view(np.float32)
            ng_r = np.zeros((h * w, 4), np.float32)
            nsel = nr[cell[hit], :3]
            ng_r[hit, :3] = nsel
            ng_r[hit, 3] = (nsel != 0).any(axis=1).astype(np.float32)
            rep = dict(image=int((image[s].view(np.int32) != ref["image"].view(np.int32)).sum()),
                       index_map=int((imap[s].ravel() != cell).sum()),
                       pts_grid=int((pg[s].view(np.int32) != pg_r.view(np.int32)).sum()),
                       nrm_grid=int((ng[s].view(np.int32) != ng_r.view(np.int32)).sum()))
            assert hit.sum() > 0
            assert_exact(rep, f"grids {h}x{wp} -> {h}x{w} scan {s}")


def test_harness_detects_div_mode_1(cuda_lib):
    """The bars catch an ulp-level change of the arithmetic: div_mode 1 (libdevice atan2f, a * (1 / span)) must show
    pixel flips on F1 and float (u, v) mismatches on a realistic scan.  The same scan is exact under div_mode 0."""
    from delora_b200 import synthetic
    h, w, fov = 64, 2250, "full"
    cloud = pr.family("boundaries", 31, h, w, fov)
    rep = report([cloud], h, w, fov, div_mode=1)
    print(f"div_mode 1 on F1: {rep}")
    assert rep["flips"] > 0 and rep["image"] > 0 and rep["index_map"] > 0, rep
    scan = synthetic.make_pair(0, w_raw=2048, rings=64)[0].numpy()
    real = report([scan], 64, 2048, "synthetic", div_mode=1)
    print(f"div_mode 1 on a synthetic KITTI scan: {real}")
    assert real["u"] > 0 and real["v"] > 0, real
    assert_exact(report([scan], 64, 2048, "synthetic", normals=True), "synthetic KITTI scan, div_mode 0")
