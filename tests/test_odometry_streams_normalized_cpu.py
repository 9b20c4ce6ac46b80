"""-m "not gpu": the normalised streams entry points of the C ABI (delora_odometry_streams_normalized_* and
delora_odometry_streams_push_normalized) without a device -- exported symbols, the header in C, the workspace size by
formula, every refusal, the Python classes' refusals and that examples/odometry_streams.c compiles."""
import ctypes
import os
import subprocess

import pytest

import odometry_harness as H
from helpers import ROOT

SYMBOLS = ("delora_odometry_streams_normalized_workspace_bytes", "delora_odometry_streams_normalized_init",
           "delora_odometry_streams_push_normalized")


def _align(n):
    return (n + 255) // 256 * 256


def _cfg(h=64, w=720, normalized=True):
    cfg = H.config(h, w, device="cpu")
    cfg["normalization_scaling"] = normalized
    return cfg


def test_symbols_exported_and_abi_unchanged():
    from delora_b200 import _lib
    L = _lib.lib()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in SYMBOLS:
        assert hasattr(handle, name), name
        assert name in _lib.SIGNATURES, name
    assert L.delora_abi_version() == 3


def test_header_compiles_as_c(tmp_path):
    from delora_b200 import build
    src = os.path.join(tmp_path, "use.c")
    with open(src, "w") as f:
        f.write('#include "delora_b200.h"\n'
                "int use(const delora_odometry_desc* d, void* ws, const float* p, const int32_t* n, float* T,\n"
                "        int32_t* valid, float* factor) {\n"
                "    if (delora_odometry_streams_normalized_workspace_bytes(d) < 0) return 1;\n"
                "    if (delora_odometry_streams_normalized_init(d, ws, 0)) return 1;\n"
                "    return delora_odometry_streams_push_normalized(d, p, n, 0, ws, T, valid, factor, 0);\n"
                "}\n"
                "_Static_assert(sizeof(delora_odometry_desc) == 80, \"desc\");\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n")
    r = subprocess.run([build._nvcc(), "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("S", [1, 4, 16])
@pytest.mark.parametrize("h,w", [(64, 2048), (64, 720), (16, 259)])
def test_workspace_is_the_streams_layout_plus_the_appended_sections(h, w, S):
    """Point rows [2S, 3, n_stride] fp32, counts [3S] int32 and factors [S] fp32, each 256-byte aligned, after the
    streams layout (W = 259 is odd: the channel-padded stem)."""
    from delora_b200 import _lib
    L = _lib.lib()
    for n_stride in (131072, 1001):
        dp = ctypes.byref(H.desc(_cfg(h, w), n_stride, S))
        streams = L.delora_odometry_streams_workspace_bytes(dp)
        got = L.delora_odometry_streams_normalized_workspace_bytes(dp)
        assert streams > 0
        assert got == streams + _align(2 * S * 3 * n_stride * 4) + _align(3 * S * 4) + _align(S * 4), (n_stride, got)


def test_invalid_descriptors_are_refused():
    from delora_b200 import _lib
    L = _lib.lib()
    d = H.desc(_cfg(), 1000, 2)
    d.act = 0
    dp = ctypes.byref(d)
    assert L.delora_odometry_streams_normalized_workspace_bytes(dp) == -1
    err = L.delora_last_error()
    assert b"act=0" in err and b"delora_odometry_streams_normalized_workspace_bytes" in err
    calls = [("delora_odometry_streams_normalized_init",
              lambda: L.delora_odometry_streams_normalized_init(dp, 1, None)),
             ("delora_odometry_streams_push_normalized",
              lambda: L.delora_odometry_streams_push_normalized(dp, 1, 1, None, 1, 1, 1, 1, None))]
    for name, call in calls:
        assert call() != 0, name
        err = L.delora_last_error()
        assert b"act=0" in err and name.encode() in err, (name, err)
    assert L.delora_odometry_streams_normalized_workspace_bytes(None) == -1
    assert b"null descriptor" in L.delora_last_error()
    d.act, d.W = 1, 718
    assert L.delora_odometry_streams_normalized_workspace_bytes(dp) == -1
    assert b"W=718" in L.delora_last_error()


@pytest.mark.parametrize("missing", ["points", "n_points", "workspace", "T", "valid", "factor"])
def test_push_refuses_null_pointers_by_name(missing):
    """Non-null dummies elsewhere: the call is refused before it could launch anything."""
    from delora_b200 import _lib
    L = _lib.lib()
    d = H.desc(_cfg(), 1000, 3)
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80, "factor": 96}
    args[missing] = None
    rc = L.delora_odometry_streams_push_normalized(ctypes.byref(d), args["points"], args["n_points"], None,
                                                   args["workspace"], args["T"], args["valid"], args["factor"], None)
    assert rc != 0
    assert f"delora_odometry_streams_push_normalized: null {missing}".encode() in L.delora_last_error()


def test_init_refuses_a_null_workspace():
    from delora_b200 import _lib
    L = _lib.lib()
    dp = ctypes.byref(H.desc(_cfg(), 1000, 2))
    assert L.delora_odometry_streams_normalized_init(dp, None, None) != 0
    assert b"delora_odometry_streams_normalized_init: null workspace" in L.delora_last_error()


def test_python_classes_refuse_the_other_kind_of_model():
    from delora_b200.deploy.stream import NormalizedOdometryStreams, OdometryStreams
    with pytest.raises(ValueError, match="normalization_scaling") as e:
        NormalizedOdometryStreams(None, _cfg(normalized=False), "kitti", 2, 1000)
    assert "OdometryStreams" in str(e.value)
    with pytest.raises(ValueError, match="normalization_scaling") as e:
        OdometryStreams(None, _cfg(), "kitti", 2, 1000)
    assert "NormalizedOdometryStreams" in str(e.value)


def test_example_compiles_against_the_header(tmp_path):
    H.build_example("odometry_streams", tmp_path, link=False)
