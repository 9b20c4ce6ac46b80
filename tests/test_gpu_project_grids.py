"""-m gpu: delora_project_grids_fwd, the dense grids of a projection at H x Wp re-projected at H x W.

It must be bit-identical to the list path the reference's training data takes (the preprocessed row-major lists of
delora_lists_from_images, projected at the model width by delora_project_fwd, gathered by
delora_grids_from_projection), leave its depth keys all-ones, and agree with the files the reference's own
preprocessing wrote (tests/golden/preprocess_16x200.npz)."""
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN

pytestmark = pytest.mark.gpu
DEV = "cuda"


def fov(cfg):
    return cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]


def batch(clouds):
    """[S, 3, N] (NaN past each scan's end) + counts [S]."""
    nmax = max([c.shape[1] for c in clouds] + [1]) + 3
    pts = torch.full((len(clouds), 3, nmax), float("nan"))
    for i, c in enumerate(clouds):
        pts[i, :, :c.shape[1]] = c
    n = torch.tensor([c.shape[1] for c in clouds], dtype=torch.int32)
    return pts.to(DEV), n.to(DEV)


def bits(t):
    return t.contiguous().view(torch.int32)


def preprocess(pts, n, h, wp, hf, vf):
    """The preprocessing stage at H x Wp: image and the dense grids."""
    from delora_b200 import ops
    image, _, pg, ng = ops.project_normals(pts, n, h, wp, hf, vf)
    return image, pg, ng


def list_path(image_pre, h, w, hf, vf):
    """lists_from_images -> channels-first -> project at H x W (C = 3) -> grids_from_projection.
    -> image, list index map, pts_grid, nrm_grid, and the pre-grid cell of every list entry."""
    from delora_b200 import ops
    normals = ops.normals(image_pre)
    pts4, nrm4, _, counts = ops.lists_from_images(image_pre, normals)
    pts = pts4[:, :, :3].transpose(1, 2).contiguous()
    nrm = nrm4[:, :, :3].transpose(1, 2).contiguous()
    image, imap = ops.project(pts, counts, h, w, hf, vf)
    pg, ng = ops.grids_from_projection(pts, nrm, imap)
    return image, imap, pg, ng, bits(pts4[:, :, 3])


def keys_rearmed(s, h, w):
    from delora_b200 import ops
    return bool((ops._keys(torch.device(DEV, torch.cuda.current_device()), s, h * w) == -1).all())


def check(clouds, h, wp, w, hf, vf):
    from delora_b200 import ops
    pts, n = batch(clouds)
    image_pre, pg_pre, ng_pre = preprocess(pts, n, h, wp, hf, vf)
    want_img, want_imap, want_pg, want_ng, cell_of_entry = list_path(image_pre, h, w, hf, vf)
    img, imap, pg, ng = ops.project_grids(pg_pre, ng_pre, h, wp, w, hf, vf)
    torch.cuda.synchronize()
    for name, a, b in (("image", img, want_img), ("pts_grid", pg, want_pg), ("nrm_grid", ng, want_ng)):
        assert torch.equal(bits(a), bits(b)), name
    # the index map names the pre-grid cell of the kept point: the cell of the list entry the list path kept
    s = len(clouds)
    li = want_imap.view(s, -1).long()
    want_cells = torch.where(li >= 0, torch.gather(cell_of_entry, 1, li.clamp_min(0)), torch.full_like(li, -1))
    assert torch.equal(imap.view(s, -1).long(), want_cells), "index_map"
    kept = imap.view(s, -1) >= 0
    assert torch.equal(kept, bits(pg[:, :, 3]) >= 0)
    cells = imap.view(s, -1).long().clamp_min(0)
    src = torch.gather(pg_pre[:, :, :3], 1, cells[:, :, None].expand(-1, -1, 3))
    assert torch.equal(bits(src[kept]), bits(pg[:, :, :3][kept]))
    assert keys_rearmed(s, h, w)
    # without an index map: the same image and grids
    img2, none, pg2, ng2 = ops.project_grids(pg_pre, ng_pre, h, wp, w, hf, vf, index_map=False)
    torch.cuda.synchronize()
    assert none is None and torch.equal(bits(img2), bits(img)) and torch.equal(bits(pg2), bits(pg))
    assert torch.equal(bits(ng2), bits(ng)) and keys_rearmed(s, h, w)
    return img, imap, pg, ng


def scans(k, rings, w_raw, vfov_deg):
    from delora_b200 import synthetic
    out = []
    for i in range(k):
        s1, s2, _, _ = synthetic.make_pair(i, w_raw=w_raw, rings=rings, vfov_deg=vfov_deg)
        out += [s1, s2]
    return out


@pytest.mark.parametrize("h,wp,w,w_raw", [(64, 2250, 720, 2048), (64, 2048, 2048, 2048), (64, 720, 1024, 1024),
                                          (16, 200, 180, 192)])
def test_matches_the_list_path(h, wp, w, w_raw, cuda_lib):
    from delora_b200 import synthetic
    vfov = synthetic.KITTI_VFOV_DEG if h == 64 else (-15.0, 15.0)
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov)
    img, _, pg, _ = check(scans(2, h, w_raw, vfov), h, wp, w, *fov(cfg))
    assert int((bits(pg[:, :, 3]) >= 0).sum()) > 0.3 * 4 * h * min(w, wp)


def test_empty_scan_and_ragged_batch(cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=16, w=180, vfov_deg=(-15.0, 15.0))
    a, b = scans(1, 16, 192, (-15.0, 15.0))
    img, imap, pg, ng = check([a, torch.zeros((3, 0)), b[:, : b.shape[1] // 3]], 16, 200, 180, *fov(cfg))
    assert float(img[1].abs().sum()) == 0.0 and bool((imap[1] == -1).all())
    assert bool((bits(pg[1, :, 3]) == -1).all()) and float(ng[1].abs().sum()) == 0.0


def test_tie_stress_cloud(cuda_lib):
    """Exact duplicate points: equal ranges in one pixel at both widths."""
    from delora_b200 import synthetic
    z = np.load(os.path.join(GOLDEN, "tie_16x512.npz"))
    cloud = torch.from_numpy(z["cloud"])
    cfg = synthetic.fov_config(h=16, w=512, vfov_deg=(-15.0, 15.0))
    for wp, w in ((512, 180), (1024, 512), (512, 512)):
        check([cloud, synthetic.tie_stress_cloud(1)], 16, wp, w, *fov(cfg))


def equal_range_pairs(h, w, wp, vfov_deg, per_row=1):
    """Pairs (a, b, c) and (b, a, c): bit-equal range ((a*a + b*b) + c*c is symmetric in a and b) and bit-equal
    elevation, azimuths mirrored about 45 degrees (and about -135: the swap maps theta to 90 - theta).  The two points
    of a pair fall in two columns of the Wp grid (both are kept there, as two valid cells) but in one column of the
    W grid, where the one with the lower cell id must win, as the lower list index does on the list path."""
    gen = torch.Generator().manual_seed(11)
    cols = []
    for v in range(h):
        el = np.radians(vfov_deg[0] + (vfov_deg[1] - vfov_deg[0]) * v / (h - 1))
        for centre, dmax in ((45.0, 0.5), (-135.0, 0.3)):
            for _ in range(per_row):
                d = np.radians(float(torch.empty(1).uniform_(0.15, dmax, generator=gen)))
                r = float(torch.empty(1).uniform_(5.0, 40.0, generator=gen))
                th = np.radians(centre) - d
                p = np.array([r * np.cos(el) * np.cos(th), r * np.cos(el) * np.sin(th), r * np.sin(el)], np.float32)
                cols += [p, p[[1, 0, 2]]]
    return torch.from_numpy(np.stack(cols, axis=1))


def test_equal_ranges_from_two_cells_in_one_model_pixel(cuda_lib):
    from delora_b200 import ops, synthetic
    h, wp, w, vfov = 16, 2048, 180, (-15.0, 15.0)
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov)
    hf, vf = fov(cfg)
    cloud = equal_range_pairs(h, w, wp, vfov)
    n_pairs = cloud.shape[1] // 2
    img, imap, pg, _ = check([cloud], h, wp, w, hf, vf)
    pts, n = batch([cloud])
    image_pre, pg_pre, _ = preprocess(pts, n, h, wp, hf, vf)
    valid = bits(pg_pre[0, :, 3]) >= 0
    assert int(valid.sum()) == 2 * n_pairs, "every point is its own valid cell at the preprocessing width"
    kept = imap[0].view(-1)[imap[0].view(-1) >= 0].long()
    assert kept.numel() == n_pairs, "each pair shares one model pixel"
    rng_pre = bits(image_pre[0, 3].reshape(-1))
    valid_cells = torch.nonzero(valid)[:, 0]
    for c in kept.tolist():
        same = valid_cells[rng_pre[valid_cells] == rng_pre[c]]
        assert same.numel() == 2 and int(same.min()) == c, f"cell {c}: equal-range cells {same.tolist()}"


def test_no_access_outside_the_buffers(cuda_lib):
    """Every buffer sits between two guard regions.  The input guards hold valid cells (a read past the grids would
    scatter them and change the result), the output and key guards a pattern no pass writes."""
    from delora_b200 import _lib, ops, synthetic
    h, wp, w = 16, 200, 180
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=(-15.0, 15.0))
    hf, vf = fov(cfg)
    pts, n = batch(scans(1, 16, 192, (-15.0, 15.0)))
    _, pg_pre, ng_pre = preprocess(pts, n, h, wp, hf, vf)
    want = ops.project_grids(pg_pre, ng_pre, h, wp, w, hf, vf)
    s, hwp, hw, g = pts.shape[0], h * wp, h * w, 4096
    donors = pg_pre[0][bits(pg_pre[0, :, 3]) >= 0]

    def guarded_input(mid, guard):
        buf = torch.cat((guard, mid.reshape(-1, 4), guard))
        return buf, buf[g:g + mid.reshape(-1, 4).shape[0]]

    guard_pts = donors[torch.arange(g, device=DEV) % donors.shape[0]]
    guard_nrm = torch.full((g, 4), 0.5, device=DEV)
    in_p, in_p_mid = guarded_input(pg_pre, guard_pts)
    in_n, in_n_mid = guarded_input(ng_pre, guard_nrm)
    pattern = 0x7FFFFFFFFFFFFFFF

    def out(n_elems, dtype, fill):
        return torch.full((g + n_elems + g,), fill, dtype=dtype, device=DEV)

    keys = out(s * hw, torch.int64, pattern)
    keys[g:g + s * hw] = -1
    image = out(s * 4 * hw, torch.float32, 7.0)
    imap = out(s * hw, torch.int32, 7)
    pg, ng = out(s * hw * 4, torch.float32, 7.0), out(s * hw * 4, torch.float32, 7.0)
    L = _lib.lib()
    _lib.check(L.delora_project_grids_fwd(in_p_mid.data_ptr(), in_n_mid.data_ptr(), s, h, wp, w, hf[0], hf[1], vf[0],
                                          vf[1], 0, keys[g:].data_ptr(), image[g:].data_ptr(), imap[g:].data_ptr(),
                                          pg[g:].data_ptr(), ng[g:].data_ptr(), torch.cuda.current_stream().cuda_stream),
               "delora_project_grids_fwd")
    torch.cuda.synchronize()
    for name, buf, ref, fill in (("image", image, want[0], 7.0), ("index_map", imap, want[1], 7),
                                 ("pts_grid", pg, want[2], 7.0), ("nrm_grid", ng, want[3], 7.0)):
        mid = buf[g:buf.numel() - g]
        assert torch.equal(bits(mid), bits(ref.reshape(-1))), name
        assert bool((buf[:g] == fill).all()) and bool((buf[-g:] == fill).all()), f"{name}: a guard was written"
    assert bool((keys[g:g + s * hw] == -1).all()), "keys not re-armed"
    assert bool((keys[:g] == pattern).all()) and bool((keys[-g:] == pattern).all()), "keys: a guard was written"
    assert torch.equal(in_p[:g], guard_pts) and torch.equal(in_p[-g:], guard_pts)


def test_equal_widths_reproduce_the_direct_projection(cuda_lib):
    """Wp == W: every kept point lands in its own pixel again, so the image and grids are those of
    delora_project_normals_fwd at W (for clouds without exact zero coordinates: such a point is an image pixel but
    not a valid cell)."""
    from delora_b200 import ops, synthetic
    for h, w, w_raw, vfov in ((16, 180, 192, (-15.0, 15.0)), (64, 720, 1024, synthetic.KITTI_VFOV_DEG)):
        cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov)
        hf, vf = fov(cfg)
        clouds = [c[:, (c != 0).all(dim=0)] for c in scans(2, h, w_raw, vfov)]
        pts, n = batch(clouds)
        image, _, pg, ng = ops.project_normals(pts, n, h, w, hf, vf)
        img2, _, pg2, ng2 = ops.project_grids(pg, ng, h, w, w, hf, vf)
        torch.cuda.synchronize()
        for name, a, b in (("image", img2, image), ("pts_grid", pg2, pg), ("nrm_grid", ng2, ng)):
            assert torch.equal(bits(a), bits(b)), f"{h}x{w}: {name}"


def test_reference_preprocessing_anchor(cuda_lib):
    """The reference's own preprocessing files (16 x 200) and the oracle's projection of them at 16 x 180."""
    from delora_b200 import ops, synthetic
    from oracle import delora_oracle as orc
    z = np.load(os.path.join(GOLDEN, "preprocess_16x200.npz"))
    cfg = synthetic.preprocessing_config("unused", "unused")
    hf, vf = fov(cfg)
    clouds = [torch.from_numpy(synthetic.kitti_bin_scan(60 + k)[:, :3]).t().contiguous() for k in range(2)]
    pts, n = batch(clouds)
    _, _, pg_pre, ng_pre = ops.project_normals(pts, n, 16, 200, hf, vf)
    img, imap, pg, ng = ops.project_grids(pg_pre, ng_pre, 16, 200, 180, hf, vf)
    torch.cuda.synchronize()
    for k in range(2):
        valid = bits(pg_pre[k, :, 3]) >= 0
        points = pg_pre[k][valid][:, :3].cpu().numpy()
        assert np.array_equal(points.view(np.int32), z[f"points_{k}"].view(np.int32)), "preprocessed point list"
        want = orc.project_to_img(torch.from_numpy(z[f"points_{k}"]).t().contiguous()[None], 16, 180, hf, vf)[0][0]
        assert torch.equal(bits(img[k].cpu()), bits(want)), "image against the oracle's projection of the list"
        # grid normals: the kept points' stored normals
        rank = torch.cumsum(valid.long(), 0) - 1                        # pre-grid cell -> list index
        kept = imap[k].view(-1) >= 0
        idx = rank[imap[k].view(-1)[kept].long()].cpu().numpy()
        ref = z[f"normals_{k}"][idx]
        got = ng[k][kept].cpu().numpy()
        has_ref = (ref != 0).any(axis=1)
        assert np.array_equal(got[:, 3] != 0, has_ref), "has-normal mask"
        err = np.linalg.norm(got[:, :3] - ref, axis=1)[has_ref]
        assert np.quantile(err, 0.99) <= 1e-6 and err.max() <= 5e-5, (np.quantile(err, 0.99), err.max())


def test_argument_errors(cuda_lib):
    L = cuda_lib
    rc = L.delora_project_grids_fwd(None, None, 1, 16, 200, 180, 0.0, 1.0, 0.0, 1.0, 0, None, None, None, None, None,
                                    None)
    assert rc != 0 and b"null pointer" in L.delora_last_error()
