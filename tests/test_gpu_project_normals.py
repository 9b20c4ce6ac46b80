"""-m gpu: delora_project_normals_fwd (projection + normals grids in one call, the normals kernel resolving the depth
keys itself) is bit-identical to delora_project_fwd followed by delora_normals_fwd, and leaves the keys all-ones."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def fov(cfg):
    return cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]


def batch(clouds, channels=3, seed=0):
    """[B, C, N] (NaN past each scan's end, a fourth channel of random reflectance for C = 4) + counts [B]."""
    nmax = max([c.shape[1] for c in clouds] + [1]) + 3
    pts = torch.full((len(clouds), channels, nmax), float("nan"))
    gen = torch.Generator().manual_seed(seed)
    for i, c in enumerate(clouds):
        pts[i, :3, :c.shape[1]] = c
        if channels > 3:
            pts[i, 3:, :c.shape[1]] = torch.rand((channels - 3, c.shape[1]), generator=gen)
    n = torch.tensor([c.shape[1] for c in clouds], dtype=torch.int32)
    return pts.to(DEV), n.to(DEV)


def two_calls(pts, n, h, w, hf, vf, nb=(7, 11), min_nb=10):
    from delora_b200 import ops
    image, imap = ops.project(pts, n, h, w, hf, vf)
    _, pg, ng = ops.normals(image, nb, 0.5, min_nb, grids=True)
    return image, imap, pg, ng


def assert_bits_equal(got, want):
    for name, a, b in zip(("image", "index_map", "pts_grid", "nrm_grid"), got, want):
        assert torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)), name


def keys_rearmed(pts, h, w):
    from delora_b200 import ops
    return bool((ops._keys(pts.device, pts.shape[0], h * w) == -1).all())


def check(clouds, h, w, hf, vf, channels=3, nb=(7, 11), min_nb=10):
    from delora_b200 import ops
    pts, n = batch(clouds, channels)
    want = two_calls(pts, n, h, w, hf, vf, nb, min_nb)
    got = ops.project_normals(pts, n, h, w, hf, vf, nb, 0.5, min_nb)
    torch.cuda.synchronize()
    assert_bits_equal(got, want)
    assert keys_rearmed(pts, h, w)
    return got


def small_scans(k, rings=16, w_raw=192, **kw):
    """k pairs -> 2k scans (vfov_deg (-15, 15) unless given)."""
    from delora_b200 import synthetic
    kw.setdefault("vfov_deg", (-15.0, 15.0))
    out = []
    for i in range(k):
        s1, s2, _, _ = synthetic.make_pair(i, w_raw=w_raw, rings=rings, **kw)
        out += [s1, s2]
    return out


def test_bench_pairs_64x2048(cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=64, w=2048)
    clouds = []
    for i in range(4):
        s1, s2, _, _ = synthetic.make_pair(i, w_raw=2048)
        clouds += [s1, s2]
    image, _, pg, _ = check(clouds, 64, 2048, *fov(cfg))
    assert int((pg[:, :, 3].view(torch.int32) >= 0).sum()) > 0.5 * 8 * 64 * 2048


@pytest.mark.parametrize("h,w,w_raw,rings,vfov", [(16, 180, 192, 16, (-15.0, 15.0)), (64, 720, 1024, 64, None),
                                                  (20, 100, 128, 24, (-15.0, 15.0))])
def test_sizes(h, w, w_raw, rings, vfov, cuda_lib):
    """16x180, 64x720 and an image whose H is not a multiple of 16 nor W of 32 (partial tiles on both edges)."""
    from delora_b200 import synthetic
    kw = {"vfov_deg": synthetic.KITTI_VFOV_DEG if vfov is None else vfov}
    cfg = synthetic.fov_config(h=h, w=w, **kw)
    check(small_scans(2, rings=rings, w_raw=w_raw, **kw), h, w, *fov(cfg))


def test_tie_and_edge_stress_clouds(cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=16, w=512, vfov_deg=(-15.0, 15.0))
    check([synthetic.tie_stress_cloud(0), synthetic.tie_stress_cloud(1)], 16, 512, *fov(cfg))
    cfg = synthetic.fov_config(h=16, w=180, vfov_deg=(-15.0, 15.0))
    edge = synthetic.edge_stress_cloud(h=16, w=180)
    assert bool(((edge == 0).all(dim=0)).any()), "the edge cloud carries zero points"
    check([edge], 16, 180, *fov(cfg))


def test_empty_scan_in_batch(cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=16, w=180, vfov_deg=(-15.0, 15.0))
    clouds = small_scans(1)
    image, imap, pg, ng = check([clouds[0], torch.zeros((3, 0)), clouds[1]], 16, 180, *fov(cfg))
    assert float(image[1].abs().sum()) == 0.0 and bool((imap[1] == -1).all())
    assert bool((pg[1, :, 3].view(torch.int32) == -1).all()) and float(ng[1].abs().sum()) == 0.0


def test_four_channels(cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=16, w=180, vfov_deg=(-15.0, 15.0))
    image, _, _, _ = check(small_scans(2), 16, 180, *fov(cfg), channels=4)
    assert image.shape[1] == 5 and float(image[:, 3].abs().sum()) > 0.0


@pytest.mark.parametrize("min_nb", [0, 1, 10])
def test_min_neighbors(min_nb, cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=64, w=720)
    check(small_scans(1, rings=64, w_raw=1024, vfov_deg=synthetic.KITTI_VFOV_DEG), 64, 720, *fov(cfg), min_nb=min_nb)


@pytest.mark.parametrize("channels,nb", [(5, (7, 11)), (3, (5, 5))])
def test_two_call_fallback(channels, nb, cuda_lib):
    """Channel counts and neighbourhoods without a fused kernel run the two calls inside the same entry point."""
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=16, w=180, vfov_deg=(-15.0, 15.0))
    check(small_scans(1), 16, 180, *fov(cfg), channels=channels, nb=nb)


def test_consecutive_calls_and_sub_batch_offsets(cuda_lib):
    """Two calls in a row on one key buffer, then per-sub-batch calls on pointer offsets into the batch buffers of a
    pair batch (pairs [b0, b0 + n): scans b0.. and B + b0..)."""
    from delora_b200 import _lib, ops, synthetic
    h, w = 16, 180
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=(-15.0, 15.0))
    hf, vf = fov(cfg)
    pts, n = batch(small_scans(3), 3)                 # B = 3 pairs -> 6 scans
    want = two_calls(pts, n, h, w, hf, vf)
    for _ in range(2):
        got = ops.project_normals(pts, n, h, w, hf, vf)
        torch.cuda.synchronize()
        assert_bits_equal(got, want)
        assert keys_rearmed(pts, h, w)

    b2, c, nmax = pts.shape
    B, hw = b2 // 2, h * w
    keys = torch.full((b2, hw), -1, dtype=torch.int64, device=DEV)
    image = torch.full((b2, c + 1, h, w), 7.0, device=DEV)
    imap = torch.full((b2, h, w), 7, dtype=torch.int32, device=DEV)
    pg = torch.full((b2, hw, 4), 7.0, device=DEV)
    ng = torch.full((b2, hw, 4), 7.0, device=DEV)
    L, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    for b0, cnt in ((0, 2), (2, 1)):
        for first in (b0, B + b0):
            _lib.check(L.delora_project_normals_fwd(pts.data_ptr() + first * c * nmax * 4, n.data_ptr() + first * 4,
                                                    cnt, c, nmax, h, w, hf[0], hf[1], vf[0], vf[1], 0,
                                                    keys.data_ptr() + first * hw * 8,
                                                    image.data_ptr() + first * (c + 1) * hw * 4,
                                                    imap.data_ptr() + first * hw * 4, 7, 11, 0.5, 10,
                                                    pg.data_ptr() + first * hw * 16, ng.data_ptr() + first * hw * 16,
                                                    None, st), "delora_project_normals_fwd")
    torch.cuda.synchronize()
    assert_bits_equal((image, imap, pg, ng), want)
    assert bool((keys == -1).all())


def test_argument_errors(cuda_lib):
    L = cuda_lib
    rc = L.delora_project_normals_fwd(None, None, 1, 3, 16, 16, 180, 0.0, 1.0, 0.0, 1.0, 0, None, None, None, 7, 11,
                                      0.5, 10, None, None, None, None)
    assert rc != 0 and b"null pointer" in L.delora_last_error()
