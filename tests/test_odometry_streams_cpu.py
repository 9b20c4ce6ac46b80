"""-m "not gpu": the streams entry points of the C ABI (delora_odometry_streams_*) without a device -- exported symbols,
descriptor validation, workspace sizes, every refusal, and that examples/odometry_streams.c compiles."""
import ctypes
import os
import subprocess

import pytest

from helpers import ROOT

STREAMS_SYMBOLS = ("delora_odometry_streams_workspace_bytes", "delora_odometry_streams_init",
                   "delora_odometry_streams_load_weights", "delora_odometry_streams_push",
                   "delora_odometry_streams_reset")


def _config(h=64, w=720):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w)
    cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                "use_dropout": False})
    return cfg


def _desc(cfg, n_stride=1000, streams=1):
    from delora_b200.deploy import export
    return export.desc_from_config(cfg, "kitti", n_stride, streams)


def test_symbols_exported():
    from delora_b200 import _lib
    _lib.lib()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in STREAMS_SYMBOLS:
        assert hasattr(handle, name), name
        assert name in _lib.SIGNATURES, name


@pytest.mark.parametrize("h,w", [(64, 2048), (64, 720), (64, 2047)])
def test_workspace_grows_with_the_stream_count(h, w):
    from delora_b200 import _lib
    L = _lib.lib()
    cfg = _config(h, w)
    sizes = [L.delora_odometry_streams_workspace_bytes(ctypes.byref(_desc(cfg, 131072, s))) for s in (1, 4, 16)]
    assert 0 < sizes[0] < sizes[1] < sizes[2]
    assert all(s % 256 == 0 for s in sizes)
    # one stream keeps one cached frame where _push keeps one, but projects one scan where _pairs sizes two
    push = L.delora_odometry_workspace_bytes(ctypes.byref(_desc(cfg, 131072, 1)))
    assert sizes[0] < push


@pytest.mark.parametrize("field,value,message", [
    ("act", 0, b"act=0"), ("n_stride", 0, b"n_stride=0"), ("max_batch", 0, b"max_batch=0"),
    ("max_batch", 5000, b"max_batch=5000"), ("H", 0, b"bad image size"), ("W", 718, b"W=718"),
    ("single_mlp", 2, b"single_mlp=2"), ("layers", 0, b"layers[2]=0"), ("vfov1", -1.0, b"field of view")])
def test_invalid_descriptors_are_refused(field, value, message):
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc(_config())
    if field == "layers":
        d.layers[2] = value
    else:
        setattr(d, field, value)
    dp = ctypes.byref(d)
    assert L.delora_odometry_streams_workspace_bytes(dp) == -1
    assert message in L.delora_last_error()
    assert b"delora_odometry_streams_workspace_bytes" in L.delora_last_error()
    calls = [("delora_odometry_streams_init", lambda: L.delora_odometry_streams_init(dp, 1, None)),
             ("delora_odometry_streams_load_weights", lambda: L.delora_odometry_streams_load_weights(dp, 1, 1, None)),
             ("delora_odometry_streams_push", lambda: L.delora_odometry_streams_push(dp, 1, 1, None, 1, 1, 1, None)),
             ("delora_odometry_streams_reset", lambda: L.delora_odometry_streams_reset(dp, 1, 1, None))]
    for name, call in calls:
        assert call() != 0, name
        err = L.delora_last_error()
        assert message in err and name.encode() in err, (name, err)
    assert L.delora_odometry_streams_workspace_bytes(None) == -1
    assert b"null descriptor" in L.delora_last_error()


@pytest.mark.parametrize("missing", ["points", "n_points", "workspace", "T", "valid"])
def test_push_refuses_null_pointers_by_name(missing):
    """Non-null dummies elsewhere: the call is refused before it could launch anything."""
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc(_config(), 1000, 3)
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80}
    args[missing] = None
    rc = L.delora_odometry_streams_push(ctypes.byref(d), args["points"], args["n_points"], None, args["workspace"],
                                        args["T"], args["valid"], None)
    assert rc != 0
    assert f"delora_odometry_streams_push: null {missing}".encode() in L.delora_last_error()


def test_other_entry_points_refuse_null_pointers():
    from delora_b200 import _lib
    L = _lib.lib()
    dp = ctypes.byref(_desc(_config(), 1000, 2))
    assert L.delora_odometry_streams_init(dp, None, None) != 0
    assert b"delora_odometry_streams_init: null workspace" in L.delora_last_error()
    assert L.delora_odometry_streams_load_weights(dp, None, 16, None) != 0
    assert b"delora_odometry_streams_load_weights: null weights" in L.delora_last_error()
    assert L.delora_odometry_streams_load_weights(dp, 16, None, None) != 0
    assert b"delora_odometry_streams_load_weights: null workspace" in L.delora_last_error()
    assert L.delora_odometry_streams_reset(dp, None, 16, None) != 0
    assert b"delora_odometry_streams_reset: null mask" in L.delora_last_error()
    assert L.delora_odometry_streams_reset(dp, 16, None, None) != 0
    assert b"delora_odometry_streams_reset: null workspace" in L.delora_last_error()


def test_example_compiles_against_the_header(tmp_path):
    from delora_b200 import build
    nvcc = build._nvcc()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    r = subprocess.run([nvcc, "-c", os.path.join(ROOT, "examples", "odometry_streams.c"), "-I",
                        os.path.join(ROOT, "include"), "-I", cuda_inc, "-Xcompiler", "-Wall,-Werror", "-o",
                        os.path.join(tmp_path, "odometry_streams.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
