"""-m "not gpu": the recipe streams entry points of the C ABI (delora_odometry_streams_pre_* and
delora_odometry_streams_push_pre) without a device -- the header in C, the workspace sizes the header documents and
their formula, every refusal before any launch, the Python class's refusal and that examples/odometry_streams.c
compiles."""
import ctypes
import os
import subprocess

import pytest

import odometry_harness as H
from delora_b200 import ops
from helpers import ROOT

NAME = "delora_odometry_streams_push_pre"


def _desc(h=64, w=720, S=2, w_pre=2250, n_stride=1000):
    return H.desc(H.config(h, w, device="cpu"), n_stride, S, w_pre)


def _rp(flags=ops.LOSS_PO2PL | ops.LOSS_PL2PL):
    from delora_b200 import _lib
    return _lib.OdometryResidualParams(lambda_po2pl=1.0, loss_flags=flags, nb_h=7, nb_w=11, epsilon_range=0.5,
                                       min_neighbors=10)


def test_header_compiles_as_c(tmp_path):
    from delora_b200 import build
    src = os.path.join(tmp_path, "use.c")
    with open(src, "w") as f:
        f.write('#include "delora_b200.h"\n'
                "int use(const delora_odometry_desc* d, const delora_odometry_residual_params* rp, void* ws,\n"
                "        const float* p, const int32_t* n, float* T, int32_t* valid, float* losses, float* factor) {\n"
                "    if (delora_odometry_streams_pre_workspace_bytes(d) < 0) return 1;\n"
                "    if (delora_odometry_streams_pre_init(d, ws, 0)) return 1;\n"
                "    return delora_odometry_streams_push_pre(d, rp, p, n, 0, ws, T, valid, losses, factor, 0);\n"
                "}\n"
                "_Static_assert(sizeof(delora_odometry_desc) == 80, \"desc\");\n"
                "_Static_assert(sizeof(delora_odometry_file_header) == 128, \"header\");\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n")
    r = subprocess.run([build._nvcc(), "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


# The header's table: (H, W, S) -> MiB of the streams, residual and recipe streams workspaces at w_pre 2250
HEADER_TABLE = {(64, 720, 1): (46.2, 50.9, 63.6), (64, 720, 4): (112.8, 131.6, 182.1),
                (64, 720, 16): (379.1, 454.3, 656.4), (64, 2048, 1): (86.0, 99.3, 111.9),
                (64, 2048, 4): (271.8, 325.0, 375.5), (64, 2048, 16): (1015.1, 1227.9, 1430.0)}


@pytest.mark.parametrize("h,w,S", sorted(HEADER_TABLE))
def test_sizes_are_the_ones_the_header_documents(h, w, S):
    from delora_b200 import _lib
    L = _lib.lib()
    dp = ctypes.byref(_desc(h, w, S, 2250, 131072))
    got = (L.delora_odometry_streams_workspace_bytes(dp), L.delora_odometry_streams_residual_workspace_bytes(dp),
           L.delora_odometry_streams_pre_workspace_bytes(dp))
    assert tuple(round(b / 2 ** 20, 1) for b in got) == HEADER_TABLE[(h, w, S)]
    with open(os.path.join(ROOT, "include", "delora_b200.h")) as f:
        header = f.read()
    mib = HEADER_TABLE[(h, w, S)]
    assert f"S = {S} {mib[0]} -> {mib[1]} -> {mib[2]} MiB" in header


@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("h,w,w_pre", [(64, 720, 2250), (16, 180, 360), (16, 259, 100)])
def test_workspace_is_the_residual_layout_plus_the_appended_sections(h, w, w_pre, S):
    """Keys, image and index map at H x w_pre for S frames, the H x w_pre grids of 2S frames, T16 and the factors,
    each 256-byte aligned, after the residual layout (whose offsets, and so the streams layout's, do not move)."""
    from delora_b200 import _lib
    L = _lib.lib()
    dp = ctypes.byref(_desc(h, w, S, w_pre))
    residual = L.delora_odometry_streams_residual_workspace_bytes(dp)
    got = L.delora_odometry_streams_pre_workspace_bytes(dp)
    hwp = h * w_pre
    want = residual + sum(H.align(n) for n in (S * hwp * 8, S * 4 * hwp * 4, S * hwp * 4, 2 * S * hwp * 16,
                                               2 * S * hwp * 16, S * 16 * 4, S * 4))
    assert residual > 0 and got == want


@pytest.mark.parametrize("w_pre", [0, 1, -5, 1 << 22])
def test_w_pre_is_refused_by_name(w_pre):
    from delora_b200 import _lib
    L = _lib.lib()
    dp = ctypes.byref(_desc(64, 720, 2, w_pre))
    assert L.delora_odometry_streams_pre_workspace_bytes(dp) == -1
    err = L.delora_last_error()
    assert f"w_pre={w_pre}".encode() in err and b"delora_odometry_streams_pre_workspace_bytes" in err, err
    assert L.delora_odometry_streams_pre_init(dp, 16, None) != 0
    assert f"delora_odometry_streams_pre_init: w_pre={w_pre}".encode() in L.delora_last_error()
    rp = _rp()
    assert L.delora_odometry_streams_push_pre(dp, ctypes.byref(rp), 16, 32, None, 48, 64, 80, 96, None, None) != 0
    assert f"{NAME}: w_pre={w_pre}".encode() in L.delora_last_error()


def test_invalid_descriptors_are_refused():
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc()
    d.act = 0
    dp = ctypes.byref(d)
    assert L.delora_odometry_streams_pre_workspace_bytes(dp) == -1
    err = L.delora_last_error()
    assert b"act=0" in err and b"delora_odometry_streams_pre_workspace_bytes" in err
    assert L.delora_odometry_streams_pre_init(dp, 16, None) != 0
    assert b"delora_odometry_streams_pre_init: act=0" in L.delora_last_error()
    assert L.delora_odometry_streams_push_pre(dp, ctypes.byref(_rp()), 16, 32, None, 48, 64, 80, 96, None, None) != 0
    assert f"{NAME}: act=0".encode() in L.delora_last_error()
    assert L.delora_odometry_streams_pre_workspace_bytes(None) == -1
    assert b"null descriptor" in L.delora_last_error()


def test_init_refuses_a_null_workspace():
    from delora_b200 import _lib
    L = _lib.lib()
    assert L.delora_odometry_streams_pre_init(ctypes.byref(_desc()), None, None) != 0
    assert b"delora_odometry_streams_pre_init: null workspace" in L.delora_last_error()


def _push(rp=None, factor=None, **null):
    """delora_odometry_streams_push_pre with non-null dummies except where null names a pointer; a null stream, so a
    call that got past its checks would launch (nothing here does)."""
    from delora_b200 import _lib
    L = _lib.lib()
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80, "losses": 96}
    args.update(null)
    rc = L.delora_odometry_streams_push_pre(ctypes.byref(_desc()), None if rp is False else ctypes.byref(rp or _rp()),
                                            args["points"], args["n_points"], None, args["workspace"], args["T"],
                                            args["valid"], args["losses"], factor, None)
    return rc, L.delora_last_error()


@pytest.mark.parametrize("missing", ["points", "n_points", "workspace", "T", "valid", "losses"])
def test_push_refuses_null_pointers_by_name(missing):
    rc, err = _push(**{missing: None})
    assert rc != 0 and f"{NAME}: null {missing}".encode() in err, err


def test_push_refuses_null_params():
    rc, err = _push(rp=False)
    assert rc != 0 and f"{NAME}: null residual_params".encode() in err, err


@pytest.mark.parametrize("flags,what", [(ops.LOSS_PO2PL | 16, b"loss_flags=0x12 has a bit other"),
                                        (ops.LOSS_PO2PL | ops.LOSS_IDENTITY_FIT, b"loss_flags=0x202 has a bit other"),
                                        (ops.LOSS_PO2PL | ops.TRAIN_DROPOUT, b"loss_flags=0x802 has a bit other"),
                                        (ops.NORMAL_LINEAR, b"sets no loss bit")])
def test_push_refuses_loss_flags_by_name(flags, what):
    rc, err = _push(rp=_rp(flags))
    assert rc != 0 and NAME.encode() in err and what in err, err


@pytest.mark.parametrize("field,value", [("nb_h", 6), ("nb_w", 0), ("epsilon_range", -1.0), ("min_neighbors", -1),
                                         ("lambda_po2pl", float("nan"))])
def test_push_refuses_neighbourhood_and_weights_by_name(field, value):
    rp = _rp()
    setattr(rp, field, value)
    rc, err = _push(rp=rp)
    assert rc != 0 and f"{NAME}: {field}=".encode() in err, err


def test_factor_must_match_the_flag():
    rc, err = _push(rp=_rp(ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING), factor=None)
    assert rc != 0 and f"{NAME}: null factor with DELORA_TRAIN_NORMALIZATION_SCALING".encode() in err, err
    rc, err = _push(rp=_rp(ops.LOSS_PO2PL), factor=112)
    assert rc != 0 and f"{NAME}: factor must be NULL without".encode() in err, err


def test_python_class_needs_the_preprocessing_width():
    from delora_b200.deploy.stream import PreprocessedOdometryStreams
    cfg = H.config(64, 720, device="cpu")
    cfg["kitti"].pop("horizontal_cells_preprocessing", None)
    for normalized in (False, True):
        cfg["normalization_scaling"] = normalized
        with pytest.raises(ValueError, match="horizontal_cells_preprocessing"):
            PreprocessedOdometryStreams(None, cfg, "kitti", 2, 1000)


def test_example_compiles_against_the_header(tmp_path):
    H.build_example("odometry_streams", tmp_path, link=False)
