"""Models trained with normalization_scaling through the C ABI, on the H100: delora_normalization_factors,
delora_odometry_pairs_normalized, OdometryStream's normalised route and examples/odometry_stream.c on a flagged file.

The mirror of a normalised pair is the Deployer's inference path with the C factor injected: points / f (torch's
tensor division) -> ops.project -> the tensor-core model -> GeometryHandler -> T[:, :3, 3] *= f.  Pooled features are
bit-identical to it and T is within 1e-5, the bar of delora_odometry_pairs against the Python path."""
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200 import ops

pytestmark = pytest.mark.gpu
DEV = H.DEV


def _factor_f64(pts, counts):
    """The definition evaluated on the host: fp32 ranges sqrt((x*x + y*y) + z*z), their float64 mean per scan rounded
    to fp32, then the fp32 mean of the pair's two means."""
    pts, counts = pts.cpu().numpy(), counts.cpu().numpy()
    b = pts.shape[0] // 2
    means = []
    for i in range(2 * b):
        x, y, z = (pts[i, c, :counts[i]].astype(np.float32) for c in range(3))
        r = np.sqrt((x * x + y * y) + z * z)
        means.append(np.float32(r.astype(np.float64).sum() / counts[i]))
    return np.array([(means[i] + means[b + i]) / np.float32(2.0) for i in range(b)], dtype=np.float32)


def _factor_torch(pts, counts):
    """Deployer._normalize_batch's factor (torch.norm / torch.mean on the device)."""
    n = counts.cpu().tolist()
    b = len(n) // 2
    means = [torch.mean(torch.norm(pts[i:i + 1, :, :k], dim=1), dim=1, keepdim=True) for i, k in enumerate(n)]
    return torch.stack([torch.mean(torch.cat((means[i], means[b + i]), dim=1), dim=1) for i in range(b)]).view(b)


def _ragged_scans(seed, count, n_max):
    """Random clouds and synthetic KITTI scans, each cut to a random length."""
    from delora_b200 import synthetic
    g = np.random.default_rng(seed)
    scans = []
    for i in range(count):
        if i % 2:
            s = synthetic.kitti_bin_scan(seed + i, w_raw=2048, rings=64, vfov_deg=H.VFOV)[:, :3].T
        else:
            s = g.normal(0.0, 20.0, size=(3, n_max)).astype(np.float32)
        n = int(g.integers(1, min(n_max, s.shape[1]) + 1))
        scans.append(torch.from_numpy(np.ascontiguousarray(s[:, :n], dtype=np.float32)))
    return scans


def test_factor_matches_the_definition_and_the_deployer(cuda_lib):
    scans = _ragged_scans(3, 16, 120000)
    stride = max(s.shape[1] for s in scans) + 37
    pts, counts = H.stack(scans, stride)
    f = ops.normalization_factors(pts, counts)
    f_again = ops.normalization_factors(pts, counts)
    ref = _factor_f64(pts, counts)
    torch.cuda.synchronize()
    got = f.cpu().numpy()
    assert np.all(np.abs(got - ref) <= np.spacing(ref)), (got, ref)
    assert torch.equal(f, f_again), "the factor is not deterministic"
    rel = ((f - _factor_torch(pts, counts)).abs() / f.abs()).max().item()
    assert rel <= 2e-6, f"relative difference to the Deployer's torch factor: {rel:.3e}"
    # a pair's factor does not depend on the batch it is computed in
    b = pts.shape[0] // 2
    for i in (0, 5, b - 1):
        one = ops.normalization_factors(pts[[i, b + i]].contiguous(), counts[[i, b + i]].contiguous())
        assert torch.equal(one, f[i:i + 1]), f"pair {i}: the factor changes with B"
    # counts above the stride are clamped to it
    big = ops.normalization_factors(pts, torch.full_like(counts, stride + 1000))
    full = ops.normalization_factors(pts, torch.full_like(counts, stride))
    assert torch.equal(big, full)


def _mirror(model, cfg, pts, counts, f):
    """The Deployer's normalised inference with the factor f injected -> (T [B,4,4], pooled [B,512])."""
    from delora_b200.models import model_parts
    ds = cfg["kitti"]
    b = pts.shape[0] // 2
    scaled = pts / torch.cat((f, f)).view(2 * b, 1, 1)
    img, _ = ops.project(scaled, counts, ds["vertical_cells"], ds["horizontal_cells"], cfg["horizontal_field_of_view"],
                         ds["vertical_field_of_view"])
    img1, img2 = img[:b].contiguous(), img[b:].contiguous()
    with torch.no_grad():
        x4, h4, w4 = model._tensor_core_path().features(img1, img2)[-1]
        pooled = ops.avgpool(x4, h4, w4)
        trans, quat = model(image_1=img1, image_2=img2)
        t = model_parts.GeometryHandler.get_transformation_matrix_quaternion(trans, quat, DEV)
    t[:, :3, 3] *= f.view(b, 1)
    return t, pooled


def _close(t, ref, tol=1e-5):
    err = (t - ref).abs().max().item()
    scale = max(1.0, ref.abs().max().item())
    assert err <= tol * scale, f"max |T - T_ref| = {err:.3e} at scale {scale:.3g}"


def _workspace(cfg, model, stride, max_batch):
    from delora_b200.deploy.capi import InferenceWorkspace
    return InferenceWorkspace(H.desc(cfg, stride, max_batch), H.blob(model, cfg))


@pytest.mark.parametrize("h,w,w_raw,act,single", [(64, 2048, 2048, "tanh", False), (64, 720, 1024, "relu", True),
                                                  (16, 720, 1024, "tanh", False)])
def test_pairs_normalized_matches_the_mirror(cuda_lib, h, w, w_raw, act, single):
    cfg = H.config(h, w, act, single)
    model = H.model(cfg).eval()
    frames = H.frames(h, w_raw, 8)
    stride = H.n_stride(H.pairs(h, w_raw, 4))
    ws = _workspace(cfg, model, stride, 4)
    for b in (1, 4):
        pts, counts = H.stack(list(frames[0:2 * b:2]) + list(frames[1:2 * b:2]), stride)
        t, pooled, f = ws.pairs_normalized(pts, counts)
        f_op = ops.normalization_factors(pts, counts)
        t_ref, pooled_ref = _mirror(model, cfg, pts, counts, f)
        # _pairs on a pre-divided copy: the same images, so the same pooled features and rotation
        t_div, pooled_div = ws.pairs(pts / torch.cat((f, f)).view(2 * b, 1, 1), counts)
        torch.cuda.synchronize()
        assert torch.equal(f, f_op), f"B={b}: the factor differs from delora_normalization_factors"
        assert torch.equal(pooled, pooled_ref), f"B={b}: pooled features differ from the mirror"
        assert torch.equal(pooled, pooled_div), f"B={b}: pooled features differ from _pairs on divided points"
        _close(t, t_ref)
        assert torch.equal(t[:, :3, :3], t_div[:, :3, :3]) and torch.equal(t[:, 3], t_div[:, 3])
        assert torch.equal(t[:, :3, 3], t_div[:, :3, 3] * f.view(b, 1)), f"B={b}: translation is not rescaled by f"
        assert not torch.allclose(f, torch.ones_like(f))


def test_power_of_two_scaling(cuda_lib):
    cfg = H.config(64, 720, "tanh", False)
    model = H.model(cfg, 2).eval()
    stride = H.n_stride(H.pairs(64, 1024, 3))
    ws = _workspace(cfg, model, stride, 3)
    frames = H.frames(64, 1024, 6)
    pts, counts = H.stack(list(frames[0::2]) + list(frames[1::2]), stride)
    t1, p1, f1 = ws.pairs_normalized(pts, counts)
    t2, p2, f2 = ws.pairs_normalized(pts * 2.0, counts)
    torch.cuda.synchronize()
    assert torch.equal(f2, 2.0 * f1)
    assert torch.equal(p1, p2), "pooled features change when every point is doubled"
    assert torch.equal(t1[:, :3, :3], t2[:, :3, :3]) and torch.equal(t1[:, 3], t2[:, 3])
    assert torch.equal(t2[:, :3, 3], 2.0 * t1[:, :3, 3])


def test_pairs_normalized_is_deterministic_and_capturable(cuda_lib):
    cfg = H.config(64, 720)
    model = H.model(cfg, 1).eval()
    stride = H.n_stride(H.pairs(64, 1024, 2))
    ws = _workspace(cfg, model, stride, 2)
    frames = H.frames(64, 1024, 4)
    pts, counts = H.stack(list(frames[0::2]) + list(frames[1::2]), stride)
    t1, p1, f1 = ws.pairs_normalized(pts, counts)
    t2, p2, f2 = ws.pairs_normalized(pts, counts)
    torch.cuda.synchronize()
    assert torch.equal(t1, t2) and torch.equal(p1, p2) and torch.equal(f1, f2)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ws.pairs_normalized(pts, counts)
    pts.mul_(1.5)                                       # the replay reads the new points
    t_eager, p_eager, f_eager = ws.pairs_normalized(pts, counts)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], t_eager) and torch.equal(out[1], p_eager) and torch.equal(out[2], f_eager)


def _normalized_cfg(h, w, **kw):
    cfg = H.config(h, w, **kw)
    cfg["normalization_scaling"] = True
    return cfg


def test_stream_normalized_route(cuda_lib):
    from delora_b200.deploy.stream import OdometryStream
    cfg = _normalized_cfg(64, 720)
    model = H.model(cfg, 4).eval()
    frames = H.frames(64, 1024, 6)
    stride = max(s.shape[1] for s in frames)
    ws = _workspace(cfg, model, stride, 1)
    graphed = OdometryStream(model, cfg, "kitti", stride, use_cuda_graph=True)
    eager = OdometryStream(model, cfg, "kitti", stride, use_cuda_graph=False)
    assert graphed.push(frames[0]) is None and eager.push(frames[0]) is None
    for k in range(1, len(frames)):
        t_g, t_e = graphed.push(frames[k]), eager.push(frames[k])
        pts, cnt = H.stack([frames[k - 1], frames[k]], stride)
        t_pair, pooled_pair, f_pair = ws.pairs_normalized(pts, cnt)
        with torch.no_grad():
            img = graphed.pair_image
            x4, h4, w4 = model._tensor_core_path().features(img[0:1].contiguous(), img[1:2].contiguous())[-1]
            pooled_stream = ops.avgpool(x4, h4, w4)
        torch.cuda.synchronize()
        assert np.array_equal(t_g, t_e), f"frame {k}: graph replay differs from the eager frame"
        assert torch.equal(graphed.factor, f_pair), f"frame {k}: the stream's factor differs from _pairs_normalized"
        assert torch.equal(graphed.pair_image, eager.pair_image), f"frame {k}: graph and eager images differ"
        assert torch.equal(pooled_stream, pooled_pair), f"frame {k}: pooled features differ from _pairs_normalized"
        _close(torch.from_numpy(t_g[0]), t_pair[0].cpu())


def test_example_program_on_a_flagged_file(cuda_lib, tmp_path):
    """examples/odometry_stream.c on a .dlw exported from a normalization_scaling checkpoint prints the transforms of
    delora_odometry_pairs_normalized."""
    import sys
    from delora_b200 import _lib, synthetic
    from delora_b200.deploy import export
    from helpers import ROOT
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False, (1, 1, 1, 1), 1000, vfov=vfov)
    cfg["normalization_scaling"] = True
    model = H.model(cfg, 5).eval()
    ckpt = os.path.join(tmp_path, "ckpt.pth")
    torch.save({"model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, ckpt)
    dlw = os.path.join(tmp_path, "model.dlw")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "export_odometry_weights.py"), "--checkpoint", ckpt,
                        "--out", dlw, "--n_stride", "4096"], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    h, d, blob = export.read_dlw(dlw)
    assert h["model_flags"] == _lib.MODEL_NORMALIZATION_SCALING
    bins = []
    for i in range(4):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    exe = H.build_example("odometry_stream", tmp_path, link=True)
    r = subprocess.run([exe, dlw] + bins, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    printed = np.array([[float(v) for v in line.split()] for line in r.stdout.strip().splitlines()], dtype=np.float64)
    assert printed.shape == (3, 12)

    from delora_b200.deploy.capi import InferenceWorkspace
    ws = InferenceWorkspace(H.desc(cfg, d.n_stride, d.max_batch), torch.from_numpy(blob).to(DEV))
    scans = [torch.from_numpy(np.fromfile(p, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()) for p in bins]
    want = []
    for k in range(1, len(scans)):
        pts, cnt = H.stack([scans[k - 1], scans[k]], d.n_stride)
        t, _, _ = ws.pairs_normalized(pts, cnt)
        want.append(t[0].cpu().numpy().reshape(16)[:12])
    assert np.abs(printed - np.stack(want).astype(np.float64)).max() <= 1e-6
