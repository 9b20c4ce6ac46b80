"""-m gpu: the normals kernels pixel by pixel against the float64 eigen-solve of tests/normals_reference.py, on
adversarial range images (families F1-F6 there, B = 3 different images per call so the batch offsets are exercised),
through all three kernels: normals_7x11_kernel (ops.normals), project_normals_7x11_kernel (ops.project_normals, checked
on its own output image) and the generic normals_kernel at other neighbourhoods, including the one that opts into more
than 48 KB of shared memory.  Every pixel: the has-normal mask and pts_grid exact, nrm_grid.w exact, unit length, the
Rayleigh residual and the eigenvector angle within the a priori bound, the orientation.  F7: the 7x11 normals of every
scalable family are bit-identical when the image and eps are scaled by 4^k, k = -2 .. 3.  Printed per family and path:
sin theta against float64 for the kernel and for the reference's fp32 LAPACK result (oracle.compute_normal_vectors);
asserted: the kernel's p99 on pixels with lambda1 - lambda0 > 4 eps is at most twice the reference's p99 + 1e-7."""
import numpy as np
import pytest
import torch

import normals_reference as NR
from oracle import delora_oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda"

FAMILIES = NR.families()
FAMILY_IDS = [f.name for f in FAMILIES]
GENERIC_NBS = [(3, 3), (5, 5), (5, 9), (7, 13), (9, 15)]
# Families where the one-pass covariance is NOT as accurate as the reference's two-pass LAPACK result (DESIGN.md 4.2):
# near-isotropic sets (F4: p99 9.2e-6 against 4.1e-6 on an H100) and images smaller than the patch, whose clamped sets
# repeat border pixels on one side of the centre (F6 1x40: 1.2e-4 against 5.8e-5; 5x9: 7.3e-7 against 2.6e-7).  Their
# numbers are printed, and every pixel is still held to the float64 bound.
UNCLAIMED = ("F4-", "F6-")


def _stack(images):
    return torch.from_numpy(np.stack([np.ascontiguousarray(i[:3], dtype=np.float32) for i in images])).to(DEV)


def _quantiles(x):
    if len(x) == 0:
        return "   (none)"
    return f"p50={np.quantile(x, 0.5):.1e} p99={np.quantile(x, 0.99):.1e} max={x.max():.1e}"


def _oracle_sin(img, ref, nb, eps, min_nb):
    """sin theta of the reference's fp32 LAPACK normals against float64, on the pixels with a normal."""
    n_o, enough, _, aux = orc.compute_normal_vectors(torch.from_numpy(np.ascontiguousarray(img[:3]))[None], nb, eps,
                                                     min_nb, return_aux=True)
    pix = aux["pixel_index"].numpy()
    assert np.array_equal(pix[enough.numpy()], ref.pix), "the oracle's mask differs from the float64 reference's"
    n = n_o.numpy()[enough.numpy()].astype(np.float64)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    return np.sqrt((np.cross(n, ref.V[:, :, 0]) ** 2).sum(axis=1))


def _run_and_check(name, images, nb, eps, min_nb, normals_out, pg, ng, two_pass=False, compare=True):
    """Checks every slot; prints the kernel's and the reference's error; asserts the p99 comparison."""
    sins, sins_gapped, ref_sins, ref_gapped = [], [], [], []
    ray, ang = 0.0, 0.0
    for k, img in enumerate(images):
        ref = NR.reference(img, nb, eps, min_nb, two_pass=two_pass)
        st = NR.check(ref, None if normals_out is None else normals_out[k].cpu().numpy(),
                      None if pg is None else pg[k].cpu().numpy(), None if ng is None else ng[k].cpu().numpy(),
                      label=f"{name}[{k}]")
        sins.append(st.sin)
        sins_gapped.append(st.sin_gapped)
        ray, ang = max(ray, st.rayleigh_ratio), max(ang, st.angle_ratio)
        if compare and min_nb >= 2 and len(ref.pix):
            so = _oracle_sin(img, ref, nb, eps, min_nb)
            gapped = (ref.lam[:, 1] - ref.lam[:, 0]) > 4 * ref.eps
            ref_sins.append(so)
            ref_gapped.append(so[gapped])
    sins, sg = np.concatenate(sins), np.concatenate(sins_gapped)
    print(f"[{name}] pixels with a normal {len(sins)}: kernel {_quantiles(sins)}; max Rayleigh residual / bound "
          f"{ray:.1e}, max sin / Davis-Kahan bound {ang:.1e}")
    if ref_sins:
        rs, rg = np.concatenate(ref_sins), np.concatenate(ref_gapped)
        print(f"[{name}]   reference fp32 LAPACK {_quantiles(rs)}")
        if len(sg) and len(rg) and not any(f in name for f in UNCLAIMED):
            kp, rp = np.quantile(sg, 0.99), np.quantile(rg, 0.99)
            print(f"[{name}]   gap > 4 eps ({len(sg)} pixels): kernel p99 {kp:.2e}, reference p99 {rp:.2e}")
            assert kp <= 2 * rp + 1e-7, f"{name}: kernel p99 {kp:.2e} against the reference's {rp:.2e}"
    return ray, ang


@pytest.mark.parametrize("fam", FAMILIES, ids=FAMILY_IDS)
def test_7x11_kernel_against_float64(fam, cuda_lib):
    from delora_b200 import ops
    img = _stack(fam.images)
    nrm, pg, ng = ops.normals(img, (7, 11), fam.eps, fam.min_nb, grids=True)
    torch.cuda.synchronize()
    _run_and_check(f"7x11/{fam.name}", fam.images, (7, 11), fam.eps, fam.min_nb, nrm, pg, ng)


@pytest.mark.parametrize("fam", [f for f in FAMILIES if f.scalable], ids=[f.name for f in FAMILIES if f.scalable])
def test_7x11_scaled_by_powers_of_four_is_bit_identical(fam, cuda_lib):
    from delora_b200 import ops
    img = _stack(fam.images)
    base, pg0, ng0 = ops.normals(img, (7, 11), fam.eps, fam.min_nb, grids=True)
    for k in range(-2, 4):
        f = 4.0 ** k
        nrm, pg, ng = ops.normals((img * f).contiguous(), (7, 11), fam.eps * f, fam.min_nb, grids=True)
        torch.cuda.synchronize()
        assert torch.equal(nrm.view(torch.int32), base.view(torch.int32)), f"scale 4^{k}: normals moved"
        assert torch.equal(ng.view(torch.int32), ng0.view(torch.int32)), f"scale 4^{k}: nrm_grid moved"
        assert torch.equal(pg[..., :3], pg0[..., :3] * f), f"scale 4^{k}: pts_grid"
        if k in (-2, 3):
            scaled = [np.asarray(i[:3], np.float32) * np.float32(f) for i in fam.images]
            _run_and_check(f"7x11/{fam.name}x4^{k}", scaled, (7, 11), fam.eps * f, fam.min_nb, nrm, pg, ng,
                           compare=False)


GENERIC_FAMILIES = [f for f in FAMILIES if f.name in ("F1-plane-20m", "F1-grazing", "F2-one-sided", "F3-poles",
                                                      "F4-isotropic", "F5-gate-eps0.5-min10", "F5-gate-eps3-min77",
                                                      "F6-constant-isolated", "F6-5x9", "F6-1x40")]


@pytest.mark.parametrize("nb", GENERIC_NBS, ids=[f"{a}x{b}" for a, b in GENERIC_NBS])
def test_generic_kernel_against_float64(nb, cuda_lib):
    from delora_b200 import ops
    for fam in GENERIC_FAMILIES:
        img = _stack(fam.images)
        nrm, pg, ng = ops.normals(img, nb, fam.eps, fam.min_nb, grids=True)
        torch.cuda.synchronize()
        _run_and_check(f"{nb[0]}x{nb[1]}/{fam.name}", fam.images, nb, fam.eps, fam.min_nb, nrm, pg, ng,
                       two_pass=True, compare=fam.name.startswith(("F1", "F2", "F3")))


def test_generic_kernel_with_opt_in_shared_memory(cuda_lib):
    """33 x 65 taps: a 96 x 40 float4 halo tile (60 KB) takes the launcher's opt-in above 48 KB."""
    from delora_b200 import ops
    for fam in [f for f in FAMILIES if f.name in ("F1-plane-2m", "F2-one-sided", "F6-constant-isolated")]:
        img = _stack(fam.images)
        nrm, pg, ng = ops.normals(img, (33, 65), fam.eps, fam.min_nb, grids=True)
        torch.cuda.synchronize()
        _run_and_check(f"33x65/{fam.name}", fam.images, (33, 65), fam.eps, fam.min_nb, nrm, pg, ng, two_pass=True,
                       compare=False)


def test_single_tap_gives_no_normal(cuda_lib):
    """(1, 1): every pixel's gated set is itself, n = 1 < 2, at every min_neighbors."""
    from delora_b200 import ops
    img = _stack(NR.family_planes()[0].images)
    for mn in (0, 1, 2):
        nrm, pg, ng = ops.normals(img, (1, 1), 0.5, mn, grids=True)
        torch.cuda.synchronize()
        assert float(nrm.abs().sum()) == 0.0 and float(ng.abs().sum()) == 0.0, mn
        assert int((pg[..., 3].view(torch.int32) >= 0).sum()) > 0


def test_6x10_routes_to_the_7x11_kernel(cuda_lib):
    from delora_b200 import ops
    for fam in FAMILIES[:6]:
        img = _stack(fam.images)
        a = ops.normals(img, (7, 11), fam.eps, fam.min_nb, grids=True)
        b = ops.normals(img, (6, 10), fam.eps, fam.min_nb, grids=True)
        torch.cuda.synchronize()
        for x, y in zip(a, b):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), fam.name


@pytest.mark.parametrize("h,w", [(1, 1), (1, 40), (5, 9), (20, 100), (16, 180), (64, 720)])
def test_image_sizes(h, w, cuda_lib):
    """Planes at 5, 20 and 60 m on an h x w grid (smaller than the patch, partial tiles on both edges, the bench's
    height), through the 7x11 kernel and the generic one at 5 x 9."""
    from delora_b200 import ops
    rng = np.random.default_rng(h * 1000 + w)
    images = [NR._plane(h, w, NR._incidence_normal(t), d, 1e-3, rng) for t, d in ((15.0, 5.0), (40.0, 20.0),
                                                                                  (70.0, 60.0))]
    img = _stack(images)
    nrm, pg, ng = ops.normals(img, (7, 11), 0.5, 10, grids=True)
    torch.cuda.synchronize()
    _run_and_check(f"7x11/{h}x{w}", images, (7, 11), 0.5, 10, nrm, pg, ng)
    nrm, pg, ng = ops.normals(img, (5, 9), 0.5, 10, grids=True)
    torch.cuda.synchronize()
    _run_and_check(f"5x9/{h}x{w}", images, (5, 9), 0.5, 10, nrm, pg, ng, two_pass=True)


def _adversarial_cloud():
    """Walls at 150 m, thin poles and a depth step, as a raw point cloud."""
    rng = np.random.default_rng(9)
    az = np.radians(rng.uniform(-179.0, 179.0, 20000))
    el = np.radians(rng.uniform(-14.0, 14.0, 20000))
    r = np.where(np.abs(az) < 1.0, 150.0 / np.maximum(np.cos(az), 0.2), 0.0)
    r = np.where(r == 0, np.where(az > 0, 8.0, 11.0), r)                         # a 3 m depth step at azimuth 0
    pts = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)]) * r
    poles = []
    for k, (x, y) in enumerate(((6.0, 2.0), (-4.0, -5.0), (12.0, -1.0))):
        z = np.linspace(-1.5, 1.5, 400)
        ang = rng.uniform(0, 2 * np.pi, 400)
        rad = 0.02 * (k + 1)
        poles.append(np.stack([x + rad * np.cos(ang), y + rad * np.sin(ang), z]))
    return torch.from_numpy(np.concatenate([pts] + poles, axis=1).astype(np.float32))


def test_fused_projection_and_normals_against_float64(cuda_lib):
    from delora_b200 import ops, synthetic
    cfg = synthetic.fov_config(h=16, w=180, vfov_deg=(-15.0, 15.0))
    hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
    clouds = [synthetic.make_pair(i, w_raw=192, rings=16, vfov_deg=(-15.0, 15.0))[k] for i, k in ((0, 0), (1, 1))]
    clouds.append(_adversarial_cloud())
    nmax = max(c.shape[1] for c in clouds) + 3
    pts = torch.zeros((3, 3, nmax))
    for i, c in enumerate(clouds):
        pts[i, :, :c.shape[1]] = c
    n = torch.tensor([c.shape[1] for c in clouds], dtype=torch.int32)
    for mn in (10, 3):
        image, _, pg, ng = ops.project_normals(pts.to(DEV), n.to(DEV), 16, 180, hf, vf, (7, 11), 0.5, mn)
        torch.cuda.synchronize()
        images = [image[k, :3].cpu().numpy() for k in range(3)]
        _run_and_check(f"fused/min{mn}", images, (7, 11), 0.5, mn, None, pg, ng)


@pytest.mark.parametrize("min_nb", [0, 1, 2])
def test_isolated_returns_get_no_normal(min_nb, cuda_lib):
    """A valid pixel whose only gated neighbour is itself (n = 1) has no normal, at every min_neighbors: 1/(n - 1) would
    make its covariance NaN, and a NaN normal would be flagged as present."""
    from delora_b200 import ops
    fam = NR.family_degenerate()[0]
    img = _stack(fam.images)
    for nb in ((7, 11), (5, 9)):
        nrm, pg, ng = ops.normals(img, nb, fam.eps, min_nb, grids=True)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(nrm).all()) and bool(torch.isfinite(ng).all()), f"{nb}: a NaN normal"
        _run_and_check(f"{nb[0]}x{nb[1]}/isolated-min{min_nb}", fam.images, nb, fam.eps, min_nb, nrm, pg, ng,
                       two_pass=nb != (7, 11), compare=False)


def test_epsilon_range_is_validated(cuda_lib):
    from delora_b200 import _lib, ops
    img = _stack(NR.family_planes()[0].images)
    for eps in (float("nan"), -0.5):
        with pytest.raises(RuntimeError, match="epsilon_range"):
            ops.normals(img, (7, 11), eps, 10, grids=True)
    pts = torch.zeros((1, 3, 16), device=DEV)
    n = torch.zeros((1,), dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="epsilon_range"):
        ops.project_normals(pts, n, 16, 180, (-3.1, 3.1), (-0.2, 0.2), (7, 11), float("nan"), 10)
    assert _lib.lib() is not None


def test_train_eval_with_min_neighbors_1_on_isolated_returns(cuda_lib):
    """delora_odometry_train_eval at min_neighbors = 1 on scans with isolated returns: finite losses (a NaN normal of an
    n = 1 pixel would reach the ICP losses)."""
    import odometry_harness as H
    cfg = H.config(16, 180)
    cfg["min_num_points_in_neighborhood_to_determine_point_class"] = 1
    blob = H.blob(H.model(cfg, 3, near_identity=True), cfg)
    rng = np.random.default_rng(4)
    scans = []
    for s1, s2 in H.pairs(16, 256, 2):
        for s in (s1, s2):
            az = rng.uniform(-np.pi, np.pi, 60)
            el = np.radians(rng.uniform(-20.0, 0.0, 60))
            r = rng.uniform(30.0, 60.0, 60)
            iso = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)]) * r
            scans.append(torch.cat([s, torch.from_numpy(iso.astype(np.float32))], dim=1))
    pairs = [(scans[0], scans[1]), (scans[2], scans[3])]
    n_stride = H.n_stride(pairs)
    tr = H.trainer(cfg, n_stride, 2, blob, 1e-4)
    losses, T, pooled = tr.eval(*H.stack_pairs(pairs, n_stride))
    torch.cuda.synchronize()
    assert bool(torch.isfinite(losses).all()) and bool(torch.isfinite(T).all()), losses
    assert float(losses[:, 3].min()) > 0
