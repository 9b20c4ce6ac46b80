"""-m "not gpu": the odometry entry points of the C ABI without a device -- exported symbols, descriptor validation,
weight-blob size against OdometryModel, the .dlw exporter, and that examples/odometry_stream.c compiles."""
import ctypes
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT

ODOMETRY_SYMBOLS = ("delora_odometry_weight_floats", "delora_odometry_workspace_bytes", "delora_odometry_init",
                    "delora_odometry_load_weights", "delora_odometry_pairs", "delora_odometry_push")


def _config(act="tanh", single=False, layers=(2, 2, 2, 2), nout=1000, h=64, w=720, **extra):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w)
    cfg.update({"activation_fct": act, "use_single_mlp_at_output": single, "layers": list(layers), "resnet_outputs": nout,
                "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1, "use_dropout": False})
    cfg.update(extra)
    return cfg


def _desc(cfg, n_stride=1000, max_batch=1):
    from delora_b200.deploy import export
    return export.desc_from_config(cfg, "kitti", n_stride, max_batch)


def test_symbols_exported_and_abi_version():
    from delora_b200 import _lib
    L = _lib.lib()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in ODOMETRY_SYMBOLS:
        assert hasattr(handle, name), name
        assert name in _lib.SIGNATURES, name
    assert L.delora_abi_version() == _lib.ABI_VERSION == 3


@pytest.mark.parametrize("act,single,layers,nout", list(itertools.product(
    ("tanh", "relu"), (False, True), ((2, 2, 2, 2), (1, 1, 1, 1)), (1000, 500))))
def test_weight_floats_match_the_state_dict(act, single, layers, nout):
    from delora_b200 import _lib
    from delora_b200.models.model import OdometryModel
    cfg = _config(act, single, layers, nout)
    with torch.device("meta"):
        model = OdometryModel(dict(cfg, device="cpu"))
    want = sum(t.numel() for t in model.state_dict().values())
    d = _desc(cfg)
    assert _lib.lib().delora_odometry_weight_floats(ctypes.byref(d)) == want
    assert _lib.lib().delora_odometry_workspace_bytes(ctypes.byref(d)) > 0


def test_workspace_grows_with_max_batch():
    from delora_b200 import _lib
    L = _lib.lib()
    cfg = _config(h=64, w=2048)
    one = L.delora_odometry_workspace_bytes(ctypes.byref(_desc(cfg, 131072, 1)))
    sixteen = L.delora_odometry_workspace_bytes(ctypes.byref(_desc(cfg, 131072, 16)))
    assert 0 < one < sixteen
    assert one % 256 == 0 and sixteen % 256 == 0


@pytest.mark.parametrize("field,value,message", [
    ("act", 0, b"act=0"), ("act", 3, b"act=3"), ("n_stride", 0, b"n_stride=0"), ("max_batch", 0, b"max_batch=0"),
    ("max_batch", 5000, b"max_batch=5000"), ("H", 0, b"bad image size"), ("W", 718, b"W=718"),
    ("resnet_outputs", 0, b"resnet_outputs=0"), ("single_mlp", 2, b"single_mlp=2"), ("layers", 0, b"layers[2]=0"),
    ("vfov1", -1.0, b"field of view")])
def test_invalid_descriptors_are_reported_without_a_gpu(field, value, message):
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc(_config())
    if field == "layers":
        d.layers[2] = value
    else:
        setattr(d, field, value)
    assert L.delora_odometry_weight_floats(ctypes.byref(d)) == -1
    assert message in L.delora_last_error()
    assert L.delora_odometry_workspace_bytes(ctypes.byref(d)) == -1
    assert L.delora_odometry_init(ctypes.byref(d), None, None) != 0
    assert message in L.delora_last_error()
    assert L.delora_odometry_pairs(ctypes.byref(d), None, None, 1, None, None, None, None) != 0


def test_null_arguments_are_reported_without_a_gpu():
    from delora_b200 import _lib
    L = _lib.lib()
    assert L.delora_odometry_weight_floats(None) == -1
    assert b"null descriptor" in L.delora_last_error()
    d = _desc(_config())
    assert L.delora_odometry_pairs(ctypes.byref(d), None, None, 1, None, None, None, None) != 0
    assert b"null pointer" in L.delora_last_error()
    assert L.delora_odometry_push(ctypes.byref(d), None, None, None, None, None) != 0
    assert b"null pointer" in L.delora_last_error()
    assert L.delora_odometry_load_weights(ctypes.byref(d), None, None, None) != 0
    assert b"null pointer" in L.delora_last_error()


def _checkpoint(tmp_path, cfg, seed=0):
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(seed)
    model = OdometryModel(dict(cfg, device="cpu"))
    path = os.path.join(tmp_path, "ckpt.pth")
    torch.save({"epoch": 0, "model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, path)
    return path, model


@pytest.mark.parametrize("act,single", [("tanh", False), ("relu", True)])
def test_exporter_round_trip(tmp_path, act, single):
    from delora_b200 import _lib
    from delora_b200.deploy import export
    cfg = _config(act, single, (1, 2, 1, 2), 500, h=16, w=720)
    path, model = _checkpoint(tmp_path, cfg)
    out = os.path.join(tmp_path, "model.dlw")
    export.export(path, "kitti", out, n_stride=4096, max_batch=3)
    h, d, blob = export.read_dlw(out)
    assert h["abi_version"] == _lib.ABI_VERSION and h["header_bytes"] == 128
    assert (h["H"], h["W"], h["n_stride"], h["max_batch"]) == (16, 720, 4096, 3)
    assert (h["hfov0"], h["hfov1"]) == tuple(cfg["horizontal_field_of_view"])
    assert (h["vfov0"], h["vfov1"]) == tuple(cfg["kitti"]["vertical_field_of_view"])
    assert h["act"] == (1 if act == "relu" else 2) and h["layers"] == [1, 2, 1, 2]
    assert h["resnet_outputs"] == 500 and h["single_mlp"] == int(single)
    want = np.concatenate([t.detach().float().reshape(-1).numpy() for t in model.state_dict().values()])
    assert blob.dtype == np.float32 and blob.tobytes() == want.tobytes()
    assert h["blob_floats"] == _lib.lib().delora_odometry_weight_floats(ctypes.byref(d)) == want.size
    assert os.path.getsize(out) == 128 + 4 * want.size


def test_exporter_cli(tmp_path):
    from delora_b200.deploy import export
    cfg = _config("tanh", False, (1, 1, 1, 1), 100, h=16, w=256)
    path, model = _checkpoint(tmp_path, cfg, seed=3)
    out = os.path.join(tmp_path, "cli.dlw")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "export_odometry_weights.py"), "--checkpoint", path,
                        "--dataset", "kitti", "--out", out, "--n_stride", "777", "--max_batch", "2"],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    h, _, blob = export.read_dlw(out)
    assert (h["H"], h["W"], h["n_stride"], h["max_batch"], h["layers"]) == (16, 256, 777, 2, [1, 1, 1, 1])
    assert blob.size == sum(t.numel() for t in model.state_dict().values())


@pytest.mark.parametrize("key,value", [("pre_feature_extraction", True), ("factor_fewer_resnet_channels", 2)])
def test_exporter_refuses_unsupported_models(tmp_path, key, value):
    from delora_b200.deploy import export
    cfg = _config("tanh", False, (1, 1, 1, 1), 100, h=16, w=256, **{key: value})
    path, _ = _checkpoint(tmp_path, cfg)
    with pytest.raises(ValueError, match=key):
        export.export(path, "kitti", os.path.join(tmp_path, "x.dlw"), n_stride=100)
    assert not os.path.exists(os.path.join(tmp_path, "x.dlw"))


def test_example_compiles_against_the_header(tmp_path):
    from delora_b200 import build
    nvcc = build._nvcc()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    r = subprocess.run([nvcc, "-c", os.path.join(ROOT, "examples", "odometry_stream.c"), "-I", os.path.join(ROOT, "include"),
                        "-I", cuda_inc, "-Xcompiler", "-Wall,-Werror", "-o", os.path.join(tmp_path, "odometry_stream.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
