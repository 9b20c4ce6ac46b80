"""Odometry inference through the C ABI (delora_odometry_*) against the Python inference path, on the H100.

Trunk: `pooled` is bit-identical to TensorCoreEncoder.features + ops.avgpool on the same projected images.  Tail:
T is within 1e-5 (absolute, relative to the transform's scale when that exceeds 1) of the torch heads (cuBLAS fp32)
followed by GeometryHandler's quaternion -> T: the two differ only in the summation order of the fp32 dot products."""
import ctypes
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
VFOV = (-24.5, 2.0)


def _config(h, w, act="tanh", single=False, layers=(2, 2, 2, 2), nout=1000, vfov=VFOV):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov, device=DEV)
    cfg.update({"activation_fct": act, "use_single_mlp_at_output": single, "layers": list(layers), "resnet_outputs": nout,
                "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1, "use_dropout": False})
    return cfg


def _model(cfg, seed=0):
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(seed)
    return OdometryModel(cfg).to(DEV).eval()


@functools.lru_cache(maxsize=None)
def _frames(rings, w_raw, count, vfov=VFOV):
    """Consecutive synthetic frames: scan_1, scan_2 of pair 0, scan_1, scan_2 of pair 1, ..."""
    from delora_b200 import synthetic
    out = []
    for i in range((count + 1) // 2):
        s1, s2, _, _ = synthetic.make_pair(i, w_raw=w_raw, rings=rings, vfov_deg=vfov)
        out += [s1, s2]
    return tuple(out[:count])


def _stack(scans, n_stride):
    pts = torch.zeros((len(scans), 3, n_stride), dtype=torch.float32)
    for i, s in enumerate(scans):
        pts[i, :, :s.shape[1]] = s
    counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
    return pts.to(DEV), counts.to(DEV)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _Capi:
    """Test-side holder of one descriptor + workspace (device memory from torch)."""

    def __init__(self, cfg, n_stride, max_batch):
        from delora_b200 import _lib
        from delora_b200.deploy import export
        self.L, self.cfg = _lib.lib(), cfg
        self.d = export.desc_from_config(cfg, "kitti", n_stride, max_batch)
        self.dp = ctypes.byref(self.d)
        self.ws = torch.empty((int(self.L.delora_odometry_workspace_bytes(self.dp)),), dtype=torch.uint8, device=DEV)
        _lib.check(self.L.delora_odometry_init(self.dp, self.ws.data_ptr(), _stream()), "delora_odometry_init")
        self.blob = None

    def load(self, model):
        from delora_b200 import _lib
        from delora_b200.deploy import export
        self.blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), self.cfg)).to(DEV)
        _lib.check(self.L.delora_odometry_load_weights(self.dp, self.blob.data_ptr(), self.ws.data_ptr(), _stream()),
                   "delora_odometry_load_weights")

    def pairs(self, pts, counts):
        from delora_b200 import _lib
        b = pts.shape[0] // 2
        t = torch.empty((b, 4, 4), dtype=torch.float32, device=DEV)
        pooled = torch.empty((b, 512), dtype=torch.float32, device=DEV)
        _lib.check(self.L.delora_odometry_pairs(self.dp, pts.data_ptr(), counts.data_ptr(), b, self.ws.data_ptr(),
                                                t.data_ptr(), pooled.data_ptr(), _stream()), "delora_odometry_pairs")
        return t, pooled

    def push(self, pts, count, t):
        from delora_b200 import _lib
        _lib.check(self.L.delora_odometry_push(self.dp, pts.data_ptr(), count.data_ptr(), self.ws.data_ptr(),
                                               t.data_ptr() if t is not None else None, _stream()), "delora_odometry_push")


def _reference(model, cfg, pts, counts):
    """Python path on the same scans: projection, TensorCoreEncoder trunk + avgpool, torch heads, quaternion -> T."""
    from delora_b200 import ops
    from delora_b200.models import model_parts
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    img, _ = ops.project(pts, counts, h, w, cfg["horizontal_field_of_view"], ds["vertical_field_of_view"])
    b = pts.shape[0] // 2
    img1, img2 = img[:b].contiguous(), img[b:].contiguous()
    with torch.no_grad():
        tc = model._tensor_core_path()
        x4, h4, w4 = tc.features(img1, img2)[-1]
        pooled = ops.avgpool(x4, h4, w4)
        trans, quat = model(image_1=img1, image_2=img2)
        t = model_parts.GeometryHandler.get_transformation_matrix_quaternion(trans, quat, DEV)
    return t, pooled


def _close(t, ref, tol=1e-5):
    err = (t - ref).abs().max().item()
    scale = max(1.0, ref.abs().max().item())
    assert err <= tol * scale, f"max |T - T_ref| = {err:.3e} at scale {scale:.3g}"
    return err


SIZES = [(64, 2048, 2048), (64, 720, 1024), (64, 512, 1024), (16, 720, 1024)]   # H, W, w_raw
VARIANTS = [("tanh", False), ("relu", False), ("tanh", True), ("relu", True)]
# resnet_outputs = 1002: the heads' first layers have K = 1002, which the tail reads without float4 loads
PAIRS_CASES = ([pytest.param(act, single, *size, 1000, id="-".join(map(str, (act, single) + size)))
                for act, single in VARIANTS for size in SIZES] +
               [pytest.param("tanh", False, 16, 720, 1024, 1002, id="tanh-False-16-720-1024-nout1002")])


@pytest.mark.parametrize("act,single,h,w,w_raw,nout", PAIRS_CASES)
def test_pairs_match_the_python_path(cuda_lib, h, w, w_raw, act, single, nout):
    cfg = _config(h, w, act, single, nout=nout)
    model = _model(cfg)
    frames = _frames(h, w_raw, 8)
    n_stride = max(s.shape[1] for s in frames)
    capi = _Capi(cfg, n_stride, 4)
    capi.load(model)
    for b in (1, 4):
        scans = list(frames[0:2 * b:2]) + list(frames[1:2 * b:2])       # scan_1 x B, then scan_2 x B
        pts, counts = _stack(scans, n_stride)
        t, pooled = capi.pairs(pts, counts)
        t_ref, pooled_ref = _reference(model, cfg, pts, counts)
        torch.cuda.synchronize()
        assert torch.equal(pooled, pooled_ref), f"B={b}: pooled features differ from the Python trunk"
        _close(t, t_ref)


def _push_setup(h=64, w=720, w_raw=1024, n=6, seed=0):
    cfg = _config(h, w)
    model = _model(cfg, seed)
    frames = _frames(h, w_raw, n)
    n_stride = max(s.shape[1] for s in frames)
    return cfg, model, frames, n_stride


def _push_all(capi, frames, n_stride):
    out = []
    t = torch.empty((4, 4), dtype=torch.float32, device=DEV)
    for k, s in enumerate(frames):
        pts, cnt = _stack([s], n_stride)
        capi.push(pts, cnt, None if k == 0 else t)
        if k:
            out.append(t.clone())
    torch.cuda.synchronize()
    return out


def test_push_matches_pairs_and_the_stream(cuda_lib):
    from delora_b200.deploy.stream import OdometryStream
    cfg, model, frames, n_stride = _push_setup()
    capi = _Capi(cfg, n_stride, 1)
    capi.load(model)
    pushed = _push_all(capi, frames, n_stride)
    stream = OdometryStream(model, cfg, "kitti", n_stride)
    ref = [stream.push(s) for s in frames]
    assert ref[0] is None
    for k in range(1, len(frames)):
        pts, cnt = _stack([frames[k - 1], frames[k]], n_stride)
        t_pair, _ = capi.pairs(pts, cnt)
        torch.cuda.synchronize()
        assert torch.equal(pushed[k - 1], t_pair[0]), f"frame {k}: push differs from pairs"
        _close(pushed[k - 1].cpu(), torch.from_numpy(ref[k][0]))


def test_push_graph_replay_matches_eager(cuda_lib):
    cfg, model, frames, n_stride = _push_setup()
    capi = _Capi(cfg, n_stride, 1)
    capi.load(model)
    eager = _push_all(capi, frames, n_stride)

    capi2 = _Capi(cfg, n_stride, 1)
    capi2.load(model)
    pts = torch.zeros((1, 3, n_stride), dtype=torch.float32, device=DEV)
    cnt = torch.zeros((1,), dtype=torch.int32, device=DEV)
    t = torch.zeros((4, 4), dtype=torch.float32, device=DEV)

    def stage(s):
        p, c = _stack([s], n_stride)
        pts.copy_(p)
        cnt.copy_(c)
    stage(frames[0])
    capi2.push(pts, cnt, None)
    stage(frames[1])
    capi2.push(pts, cnt, t)                   # eager frame: also sets up the launchers' host-side state
    torch.cuda.synchronize()
    assert torch.equal(t, eager[0])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        capi2.push(pts, cnt, t)
    for k in range(2, len(frames)):
        stage(frames[k])
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(t, eager[k - 1]), f"frame {k}: graph replay differs from the eager call"


def test_deterministic_and_reload(cuda_lib):
    cfg = _config(64, 720, "relu", True)
    model_a, model_b = _model(cfg, 0), _model(cfg, 1)
    frames = _frames(64, 1024, 4)
    n_stride = max(s.shape[1] for s in frames)
    pts, counts = _stack([frames[0], frames[2], frames[1], frames[3]], n_stride)
    capi = _Capi(cfg, n_stride, 2)
    capi.load(model_a)
    t1, p1 = capi.pairs(pts, counts)
    t2, p2 = capi.pairs(pts, counts)
    torch.cuda.synchronize()
    assert torch.equal(t1, t2) and torch.equal(p1, p2)
    capi.load(model_b)
    tb, pb = capi.pairs(pts, counts)
    tb_ref, pb_ref = _reference(model_b, cfg, pts, counts)
    torch.cuda.synchronize()
    assert not torch.equal(pb, p1)
    assert torch.equal(pb, pb_ref)
    _close(tb, tb_ref)
    capi.load(model_a)
    t3, p3 = capi.pairs(pts, counts)
    torch.cuda.synchronize()
    assert torch.equal(t3, t1) and torch.equal(p3, p1)


def test_errors_launch_nothing(cuda_lib):
    from delora_b200 import _lib
    cfg = _config(16, 720)
    model = _model(cfg)
    frames = _frames(16, 1024, 4)
    n_stride = max(s.shape[1] for s in frames)
    capi = _Capi(cfg, n_stride, 1)
    capi.load(model)
    L = capi.L
    pts, counts = _stack([frames[0], frames[2], frames[1], frames[3]], n_stride)
    t = torch.full((2, 4, 4), 7.0, device=DEV)
    rc = L.delora_odometry_pairs(capi.dp, pts.data_ptr(), counts.data_ptr(), 2, capi.ws.data_ptr(), t.data_ptr(), None,
                                 _stream())
    assert rc != 0 and b"max_batch=1" in L.delora_last_error()
    rc = L.delora_odometry_pairs(capi.dp, pts.data_ptr(), counts.data_ptr(), 0, capi.ws.data_ptr(), t.data_ptr(), None,
                                 _stream())
    assert rc != 0 and b"B=0" in L.delora_last_error()
    torch.cuda.synchronize()
    assert bool((t == 7.0).all()), "a refused call wrote its output"
    # device-side counts above n_stride cannot be checked on the host without a synchronise: they are clamped
    p2, c2 = _stack([frames[0], frames[1]], n_stride)
    t_ok, pool_ok = capi.pairs(p2, c2)
    t_big, pool_big = capi.pairs(p2, torch.full_like(c2, n_stride))
    t_over, pool_over = capi.pairs(p2, torch.full_like(c2, n_stride + 100000))
    torch.cuda.synchronize()
    assert torch.equal(t_over, t_big) and torch.equal(pool_over, pool_big)
    assert bool(torch.isfinite(t_ok).all())
    with pytest.raises(RuntimeError, match="max_batch"):
        _lib.check(L.delora_odometry_pairs(capi.dp, pts.data_ptr(), counts.data_ptr(), 2, capi.ws.data_ptr(),
                                           t.data_ptr(), None, _stream()), "delora_odometry_pairs")


def test_example_program(cuda_lib, tmp_path):
    """examples/odometry_stream.c on an exported checkpoint and three KITTI .bin scans prints what _lib computes."""
    from delora_b200 import build, synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = _config(16, 720, "tanh", False, (1, 1, 1, 1), 1000, vfov=vfov)
    model = _model(cfg, 5)
    ckpt = os.path.join(tmp_path, "ckpt.pth")
    torch.save({"model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, ckpt)
    dlw = os.path.join(tmp_path, "model.dlw")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "export_odometry_weights.py"), "--checkpoint", ckpt,
                        "--out", dlw, "--n_stride", "4096"], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    bins = []
    for i in range(3):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    nvcc = build._nvcc()
    cuda_home = os.path.dirname(os.path.dirname(os.path.realpath(nvcc)))
    libdir = os.path.dirname(build.LIB)
    exe = os.path.join(tmp_path, "odometry_stream")
    r = subprocess.run([nvcc, os.path.join(ROOT, "examples", "odometry_stream.c"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(cuda_home, "include"), "-L", libdir, "-ldelora_b200", "-lcudart",
                        "-Xlinker", "-rpath=" + libdir, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([exe, dlw] + bins, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    printed = np.array([[float(v) for v in line.split()] for line in r.stdout.strip().splitlines()], dtype=np.float64)
    assert printed.shape == (2, 12)

    _, d, blob = export.read_dlw(dlw)
    capi = _Capi(cfg, d.n_stride, d.max_batch)
    blob_dev = torch.from_numpy(blob).to(DEV)
    from delora_b200 import _lib
    _lib.check(capi.L.delora_odometry_load_weights(capi.dp, blob_dev.data_ptr(), capi.ws.data_ptr(), _stream()), "load")
    scans = [torch.from_numpy(np.fromfile(p, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()) for p in bins]
    want = _push_all(capi, scans, d.n_stride)
    want = np.stack([t.cpu().numpy().reshape(16)[:12] for t in want]).astype(np.float64)
    assert np.abs(printed - want).max() <= 1e-6, (printed, want)
