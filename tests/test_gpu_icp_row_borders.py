"""Dense ICP on scenes that stress the range-certified row borders of the window search: rows beyond a border at the
same range as the source (the range bound must fall back to the angular one), target rows without any valid cell,
and image heights that are not a multiple of the 4-row range blocks.  Every case is checked against the CSR kernel
(independent search code) and against cKDTree (oracle)."""
import math

import pytest
import torch

from oracle import delora_oracle as orc

pytestmark = pytest.mark.gpu

DEV = "cuda"


def cylinder_scan(seed, rings, w_raw, vfov_deg, radius=6.0):
    """A vertical cylinder around the sensor: |t| = radius / cos(elevation), so neighbouring rows are at nearly the
    same range as the source point."""
    gen = torch.Generator().manual_seed(seed)
    n = rings * w_raw
    el0, el1 = math.radians(vfov_deg[0]), math.radians(vfov_deg[1])
    ring = torch.arange(rings, dtype=torch.float64).repeat_interleave(w_raw)
    col = torch.arange(w_raw, dtype=torch.float64).repeat(rings)
    jit = (torch.rand(2, n, generator=gen, dtype=torch.float64) - 0.5) * 0.6
    el = el0 + (ring + jit[0]) / (rings - 1) * (el1 - el0)
    az = -math.pi + (col + jit[1]) / w_raw * 2.0 * math.pi
    t = radius / torch.cos(el)
    pts = torch.stack((torch.cos(el) * torch.cos(az), torch.sin(az) * torch.cos(el), torch.sin(el))) * t
    pts = pts + 0.005 * torch.randn(3, n, generator=gen, dtype=torch.float64)
    return pts.to(torch.float32).contiguous()


def project(cloud, h, w, cfg):
    from delora_b200 import ops
    hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
    n = torch.tensor([cloud.shape[1]], dtype=torch.int32, device=DEV)
    image, _ = ops.project(cloud[None].contiguous().to(DEV), n, h, w, hf, vf)
    return image


def check_against_csr_and_kdtree(images, h, w, cfg, transforms):
    """images [2, 4, H, W]: index 0 = target, 1 = source."""
    from delora_b200 import ops
    hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
    nrm_img, pg, ng = ops.normals(images, grids=True)
    pts4, nrm4, cs, counts = ops.lists_from_images(images, nrm_img)
    p1, n1 = pts4[0, :int(counts[0]), :3].cpu(), nrm4[0, :int(counts[0]), :3].cpu()
    p2, n2 = pts4[1, :int(counts[1]), :3].cpu(), nrm4[1, :int(counts[1]), :3].cpu()
    for k, tm in enumerate(transforms):
        tm = torch.as_tensor(tm, dtype=torch.float32)
        T = tm[:3, :].reshape(1, 12).contiguous().to(DEV)
        losses, grad_t = ops.icp_dense_fwd_bwd(pg[1:2].contiguous(), ng[1:2].contiguous(), T, pg[0:1].contiguous(),
                                               ng[0:1].contiguous(), h, w, hf, vf)
        l2, g2, _, _, _ = ops.icp_fwd_bwd(pts4[1:2].contiguous(), nrm4[1:2].contiguous(), counts[1:2].contiguous(), T,
                                          pts4[0:1].contiguous(), nrm4[0:1].contiguous(), cs[0:1].contiguous(), h, w,
                                          hf, vf)
        assert float(losses[0, 3]) > 0, k
        assert float(l2[0, 3]) == float(losses[0, 3]), k
        assert torch.allclose(l2[0, :3].cpu(), losses[0, :3].cpu(), rtol=2e-6, atol=0), k
        assert torch.allclose(g2.cpu(), grad_t.cpu(), rtol=1e-4, atol=1e-7), k
        t4 = tm.view(1, 4, 4)
        lo, aux = orc.icp_losses(orc.transform_point_cloud(t4, p2.t()[None]), orc.rotate_point_cloud(t4, n2.t()[None]),
                                 p1.t()[None].contiguous(), n1.t()[None].contiguous(), return_aux=True)
        assert aux["num_pairs"] == int(losses[0, 3]), k
        assert float(losses[0, 1]) == pytest.approx(float(lo["loss_po2pl"]), rel=2e-5), k
        assert float(losses[0, 2]) == pytest.approx(float(lo["loss_pl2pl"]), rel=2e-5), k


def transforms():
    from delora_b200 import synthetic
    return [synthetic.transform_matrix(0.05, 0.0, 0.0, math.radians(0.2)),
            synthetic.transform_matrix(0.6, -0.2, 0.05, math.radians(2.0)),
            synthetic.transform_matrix(1.5, 0.4, 0.1, math.radians(8.0), math.radians(1.0), 0.0)]


SIZES = [(16, 180, 192, (-15.0, 15.0)), (64, 720, 720, (-24.5, 2.0))]


@pytest.mark.parametrize("h,w,w_raw,vfov", SIZES)
def test_dense_icp_cylinder_same_range_rows(h, w, w_raw, vfov, cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov)
    images = torch.cat((project(cylinder_scan(1, h, w_raw, vfov), h, w, cfg),
                        project(cylinder_scan(2, h, w_raw, vfov), h, w, cfg)))
    check_against_csr_and_kdtree(images, h, w, cfg, transforms())


@pytest.mark.parametrize("h,w,w_raw,vfov", SIZES)
def test_dense_icp_target_with_empty_rows(h, w, w_raw, vfov, cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov)
    s1, s2, _, _ = synthetic.make_pair(3, w_raw=w_raw, rings=h, vfov_deg=vfov)
    images = torch.cat((project(s1, h, w, cfg), project(s2, h, w, cfg)))
    # empty target rows: the first and last row, a run in the middle (inside one 4-row block and across two) and a
    # single row next to it
    empty = [0, h - 1] + list(range(h // 2 - 3, h // 2 + 2)) + [h // 2 + 3]
    images[0, :, empty, :] = 0.0
    check_against_csr_and_kdtree(images, h, w, cfg, transforms())


@pytest.mark.parametrize("h,w,w_raw,vfov", [(15, 180, 192, (-15.0, 15.0)), (18, 180, 192, (-15.0, 15.0)),
                                            (63, 720, 720, (-24.5, 2.0))])
def test_dense_icp_height_not_multiple_of_4(h, w, w_raw, vfov, cuda_lib):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov)
    s1, s2, _, _ = synthetic.make_pair(4, w_raw=w_raw, rings=h, vfov_deg=vfov)
    images = torch.cat((project(s1, h, w, cfg), project(s2, h, w, cfg)))
    check_against_csr_and_kdtree(images, h, w, cfg, transforms())
