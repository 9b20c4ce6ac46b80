"""-m "not gpu": delora_odometry_train_eval and the per-frame ICP residual of the streams (delora_odometry_streams_residual_*,
_push_residual) without a device -- exported symbols, the unchanged ABI version, the residual workspace as the streams
layout plus appended sections, every refusal by name, and that the header and both example programs compile."""
import ctypes
import os
import subprocess

import pytest

import odometry_harness as H
from helpers import ROOT

NEW_SYMBOLS = ("delora_odometry_train_eval", "delora_odometry_streams_residual_workspace_bytes",
               "delora_odometry_streams_residual_init", "delora_odometry_streams_push_residual")


def _L():
    from delora_b200 import _lib
    return _lib.lib()


def test_symbols_exported_and_the_abi_version_stays():
    from delora_b200 import _lib
    L = _L()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert hasattr(handle, name), name
        assert name in _lib.SIGNATURES, name
    assert L.delora_abi_version() == 3


@pytest.mark.parametrize("h,w", [(64, 2048), (64, 720), (16, 180)])
@pytest.mark.parametrize("S", [1, 4, 16])
def test_residual_workspace_is_the_streams_layout_plus_the_appended_sections(h, w, S):
    """No offset query exists, so the sizes carry it: the residual workspace exceeds the streams workspace by exactly
    the appended sections (four float4 grids of S frames, S x 12 transforms, S loss rows, S x 12 dL/dT, the ICP scratch
    for B = S, each 256-byte aligned), which leaves every streams offset (weights, frames, has_prev) where it was."""
    L = _L()
    dp = ctypes.byref(H.desc(H.config(h, w, device="cpu"), 131072, S))
    streams = L.delora_odometry_streams_workspace_bytes(dp)
    residual = L.delora_odometry_streams_residual_workspace_bytes(dp)
    appended = (4 * H.align(S * h * w * 16) + H.align(S * 12 * 4) + H.align(S * 8 * 4) + H.align(S * 12 * 4) +
                H.align(L.delora_icp_scratch_floats(S, h * w) * 4))
    assert streams > 0 and residual == streams + appended


def test_invalid_descriptors_are_refused_by_field():
    L = _L()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 2)
    d.max_batch = 0
    dp = ctypes.byref(d)
    rp = ctypes.byref(_residual_params())
    assert L.delora_odometry_streams_residual_workspace_bytes(dp) == -1
    err = L.delora_last_error()
    assert b"max_batch=0" in err and b"delora_odometry_streams_residual_workspace_bytes" in err
    calls = [("delora_odometry_streams_residual_init", lambda: L.delora_odometry_streams_residual_init(dp, 16, None)),
             ("delora_odometry_streams_push_residual",
              lambda: L.delora_odometry_streams_push_residual(dp, rp, 16, 16, None, 16, 16, 16, 16, None)),
             ("delora_odometry_train_eval",
              lambda: L.delora_odometry_train_eval(dp, ctypes.byref(_train_params()), 16, 16, 1, 16, None, None, None,
                                                   None))]
    for name, call in calls:
        assert call() != 0, name
        err = L.delora_last_error()
        assert b"max_batch=0" in err and name.encode() in err, (name, err)
    assert L.delora_odometry_streams_residual_workspace_bytes(None) == -1
    assert b"null descriptor" in L.delora_last_error()


def _residual_params(**over):
    from delora_b200.deploy import capi
    rp = capi.residual_params(H.config(64, 720, device="cpu"))
    for k, v in over.items():
        setattr(rp, k, v)
    return rp


def _train_params(**over):
    from delora_b200.deploy import capi
    hp = capi.train_params(H.config(64, 720, device="cpu"), 1e-5)
    for k, v in over.items():
        setattr(hp, k, v)
    return hp


@pytest.mark.parametrize("missing", ["points", "n_points", "workspace", "T", "valid", "losses"])
def test_push_residual_refuses_null_pointers_by_name(missing):
    L = _L()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 3)
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80, "losses": 96}
    args[missing] = None
    rc = L.delora_odometry_streams_push_residual(ctypes.byref(d), ctypes.byref(_residual_params()), args["points"],
                                                 args["n_points"], None, args["workspace"], args["T"], args["valid"],
                                                 args["losses"], None)
    assert rc != 0
    assert f"delora_odometry_streams_push_residual: null {missing}".encode() in L.delora_last_error()


@pytest.mark.parametrize("over,message", [
    ({"loss_flags": 0}, b"sets no loss bit"),
    ({"loss_flags": 2 | 512}, b"loss_flags=0x202 has a bit other than"),        # DELORA_LOSS_IDENTITY_FIT
    ({"loss_flags": 6 | 1024}, b"loss_flags=0x406 has a bit other than"),       # DELORA_TRAIN_NORMALIZATION_SCALING
    ({"loss_flags": 6 | 2048}, b"loss_flags=0x806 has a bit other than"),       # DELORA_TRAIN_DROPOUT
    ({"loss_flags": 6 | 256}, b"loss_flags=0x106 has a bit other than"),        # DELORA_ICP_STATS
    ({"nb_h": 4}, b"nb_h=4"), ({"nb_w": 0}, b"nb_w=0"), ({"epsilon_range": -1.0}, b"epsilon_range=-1"),
    ({"min_neighbors": -2}, b"min_neighbors=-2"), ({"lambda_po2pl": float("inf")}, b"lambda_po2pl=inf")])
def test_push_residual_refuses_bad_parameters(over, message):
    L = _L()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 2)
    rc = L.delora_odometry_streams_push_residual(ctypes.byref(d), ctypes.byref(_residual_params(**over)), 16, 16, None,
                                                 16, 16, 16, 16, None)
    err = L.delora_last_error()
    assert rc != 0 and message in err and b"delora_odometry_streams_push_residual" in err, err
    assert L.delora_odometry_streams_push_residual(ctypes.byref(d), None, 16, 16, None, 16, 16, 16, 16, None) != 0
    assert b"null residual_params" in L.delora_last_error()


def test_residual_init_refuses_a_null_workspace():
    L = _L()
    dp = ctypes.byref(H.desc(H.config(64, 720, device="cpu"), 1000, 2))
    assert L.delora_odometry_streams_residual_init(dp, None, None) != 0
    assert b"delora_odometry_streams_residual_init: null workspace" in L.delora_last_error()


def test_train_eval_has_the_steps_refusals():
    L = _L()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 2)
    dp = ctypes.byref(d)

    def call(hp=None, points=16, n_points=16, b=1, ws=16):
        hp = _train_params() if hp is None else hp
        return L.delora_odometry_train_eval(dp, ctypes.byref(hp), points, n_points, b, ws, None, None, None, None)

    for kwargs, message in [({"points": None}, b"null pointer"), ({"n_points": None}, b"null pointer"),
                            ({"ws": None}, b"null pointer"), ({"b": 0}, b"B=0 outside [1, max_batch=2]"),
                            ({"b": 3}, b"B=3 outside [1, max_batch=2]"),
                            ({"hp": _train_params(loss_flags=512)}, b"sets no loss bit"),
                            ({"hp": _train_params(nb_h=2)}, b"nb_h=2"),
                            ({"hp": _train_params(lr=-1.0)}, b"lr=-1"),
                            ({"hp": _train_params(loss_flags=6 | 1024)}, b"needs w_pre > 0")]:
        assert call(**kwargs) != 0, kwargs
        err = L.delora_last_error()
        assert message in err and b"delora_odometry_train_eval" in err, (kwargs, err)
    assert L.delora_odometry_train_eval(dp, None, 16, 16, 1, 16, None, None, None, None) != 0
    assert b"null hyperparameters" in L.delora_last_error()
    d.w_pre = 1
    assert call() != 0 and b"w_pre=1" in L.delora_last_error()


def test_python_streams_refuse_a_normalised_model_with_the_residual_too():
    from delora_b200.deploy.stream import OdometryStreams
    cfg = H.config(64, 720, device="cpu")
    cfg["normalization_scaling"] = True
    with pytest.raises(ValueError, match="normalization_scaling"):
        OdometryStreams(None, cfg, "kitti", 2, 1000, residual=True)


def test_header_compiles_as_c(tmp_path):
    src = os.path.join(tmp_path, "use.c")
    with open(src, "w") as f:
        f.write('#include "delora_b200.h"\n'
                "int use(const delora_odometry_desc* d, const delora_odometry_train_params* hp, void* p) {\n"
                "    delora_odometry_residual_params rp = {1.0f, DELORA_LOSS_PO2PL | DELORA_LOSS_PL2PL, 7, 11, 0.5f, 10};\n"
                "    if (delora_odometry_streams_residual_workspace_bytes(d) < 0) return 1;\n"
                "    if (delora_odometry_streams_residual_init(d, p, 0)) return 1;\n"
                "    if (delora_odometry_streams_push_residual(d, &rp, p, p, p, p, p, p, p, 0)) return 1;\n"
                "    return delora_odometry_train_eval(d, hp, p, p, 1, p, p, p, p, 0);\n"
                "}\n")
    r = subprocess.run(["cc", "-std=c99", "-Wall", "-Werror", "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("name", ["odometry_train", "odometry_streams"])
def test_examples_compile_against_the_header(tmp_path, name):
    H.build_example(name, tmp_path, link=False)
