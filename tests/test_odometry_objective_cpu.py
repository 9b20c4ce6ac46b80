"""-m "not gpu": the ICP objective a model is configured with, recorded in the .dlw / .dlt header (objective_flags at
byte 108, lambda_po2pl at 112) and read back by every layer -- the header's layout, the export and its refusals, the
round trip through read_dlw / read_dlt / config_from_desc / bin/training_state_to_checkpoint.py, old files with zeros
there, delora_odometry_file_objective, the binding's defaults, and every entry point's refusal of a malformed
DELORA_LOSS_PO2PO_ALONE before any launch."""
import ctypes
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200 import ops
from helpers import ROOT

PO2PO, PO2PL, PL2PL, LINEAR, ALONE = ops.LOSS_PO2PO, ops.LOSS_PO2PL, ops.LOSS_PL2PL, ops.NORMAL_LINEAR, 4096
SHIPPED = (PO2PL | PL2PL, 1.0)

# config keys -> the (objective_flags, lambda_po2pl) the file records
CONFIGS = {
    "shipped": ({}, SHIPPED),
    "linear": ({"normal_loss": "linear"}, (PO2PL | PL2PL | LINEAR, 1.0)),
    "lambda_10": ({"lambda_po2pl": 10.0}, (PO2PL | PL2PL, 10.0)),
    "point_to_point": ({"point_to_point_loss": True}, (PO2PO | PO2PL | PL2PL, 1.0)),
    "po2po_alone": ({"po2po_alone": True, "point_to_point_loss": True, "point_to_plane_loss": False,
                     "plane_to_plane_loss": False}, (PO2PO | ALONE, 1.0)),
    "pl2pl_linear_only": ({"point_to_plane_loss": False, "normal_loss": "linear", "lambda_po2pl": 0.5},
                          (PL2PL | LINEAR, 0.5)),
}


def _L():
    from delora_b200 import _lib
    return _lib.lib()


def _cfg(**over):
    cfg = H.config(16, 720, device="cpu")
    cfg.update(over)
    return cfg


def _checkpoint(tmp_path, cfg, name="m.pth"):
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(0)
    model = OdometryModel(dict(cfg, device="cpu"))
    path = os.path.join(tmp_path, name)
    torch.save({"epoch": 0, "model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, path)
    return path


def test_constant_and_header_layout(tmp_path):
    from delora_b200 import build
    src = os.path.join(tmp_path, "layout.c")
    with open(src, "w") as f:
        f.write('#include <stddef.h>\n#include "delora_b200.h"\n'
                "_Static_assert(offsetof(delora_odometry_file_header, model_flags) == 104, \"model_flags\");\n"
                "_Static_assert(offsetof(delora_odometry_file_header, objective_flags) == 108, \"objective_flags\");\n"
                "_Static_assert(offsetof(delora_odometry_file_header, lambda_po2pl) == 112, \"lambda_po2pl\");\n"
                "_Static_assert(offsetof(delora_odometry_file_header, reserved) == 116, \"reserved\");\n"
                "_Static_assert(sizeof(delora_odometry_file_header) == 128, \"header\");\n"
                "_Static_assert(sizeof(delora_odometry_train_file_header) == 256, \"train header\");\n"
                "_Static_assert(offsetof(delora_odometry_train_file_header, step) == 128, \"step\");\n"
                "_Static_assert(sizeof(delora_odometry_desc) == 80, \"desc\");\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n"
                "_Static_assert(DELORA_LOSS_PO2PO_ALONE == 4096u, \"bit\");\n"
                "int use(const delora_odometry_file_header* h, uint32_t* f, float* l) {\n"
                "    return delora_odometry_file_objective(h, f, l);\n}\n")
    r = subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "layout.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ops.LOSS_PO2PO_ALONE == ALONE
    from delora_b200 import _lib
    assert _lib.LOSS_PO2PO_ALONE == ALONE and _lib.ABI_VERSION == 3
    assert build.LIB


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_objective_from_config(name):
    from delora_b200.deploy import export
    over, want = CONFIGS[name]
    assert export.objective_from_config(_cfg(**over)) == want
    assert export.objective_from_config(export.config_objective(want)) == want


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_the_fields_sit_at_bytes_108_and_112_and_round_trip(tmp_path, name):
    from delora_b200.deploy import export
    over, want = CONFIGS[name]
    cfg = _cfg(**over)
    dlw = os.path.join(tmp_path, "m.dlw")
    export.export(_checkpoint(tmp_path, cfg), "kitti", dlw, n_stride=512)
    raw = open(dlw, "rb").read(128)
    assert struct.unpack_from("<If", raw, 108) == (want[0], np.float32(want[1]))
    assert raw[116:128] == bytes(12)
    h, d, _ = export.read_dlw(dlw)
    assert (h["objective_flags"], h["lambda_po2pl"]) == want
    assert export.file_objective(h) == want
    back = export.config_from_desc(d, None, "kitti", h["model_flags"], (h["objective_flags"], h["lambda_po2pl"]))
    assert export.objective_from_config(back) == want
    # the C reader agrees
    from delora_b200 import _lib
    flags, lam = ctypes.c_uint32(), ctypes.c_float()
    buf = ctypes.create_string_buffer(raw, 128)
    assert _lib.lib().delora_odometry_file_objective(buf, ctypes.byref(flags), ctypes.byref(lam)) == 0
    assert (flags.value, lam.value) == want


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_checkpoint_to_dlt_and_back_keeps_the_objective(tmp_path, name):
    from delora_b200.deploy import export
    over, want = CONFIGS[name]
    dlt = os.path.join(tmp_path, "m.dlt")
    export.export(_checkpoint(tmp_path, _cfg(**over)), "kitti", dlt, n_stride=512, training_state=True)
    h = export.read_dlt(dlt)[0]
    assert (h["objective_flags"], h["lambda_po2pl"]) == want
    out = os.path.join(tmp_path, "back.pth")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "training_state_to_checkpoint.py"), "--dlt", dlt,
                        "--out", out], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    params = torch.load(out, map_location="cpu", weights_only=False)["parameters"]
    assert export.objective_from_config(params) == want
    for key, value in export.config_objective(want).items():
        assert params[key] == value, key
    # ... and exporting that checkpoint again records the same objective
    again = os.path.join(tmp_path, "again.dlw")
    export.export(out, "kitti", again, n_stride=512)
    h2 = export.read_dlw(again)[0]
    assert (h2["objective_flags"], h2["lambda_po2pl"]) == want


@pytest.mark.parametrize("kind", ["dlw", "dlt"])
def test_a_file_with_zeros_at_108_to_115_reads_as_the_shipped_objective(tmp_path, kind):
    from delora_b200.deploy import export
    d = H.desc(_cfg(), 512, 2)
    blob = np.zeros(8, dtype=np.float32)
    path = os.path.join(tmp_path, "old." + kind)
    if kind == "dlw":
        export.write_dlw(path, d, blob)
        h = export.read_dlw(path)[0]
    else:
        export.write_dlt(path, d, export.TrainingState(blob, blob, blob))
        h = export.read_dlt(path)[0]
    raw = open(path, "rb").read(128)
    assert raw[108:128] == bytes(20)
    assert (h["objective_flags"], h["lambda_po2pl"]) == (0, 0.0)
    assert export.file_objective(h) == SHIPPED
    cfg = export.config_from_desc(d, {"lambda_po2pl": 10.0, "po2po_alone": True}, "kitti", 0, (0, 0.0))
    assert export.objective_from_config(cfg) == SHIPPED
    flags, lam = ctypes.c_uint32(), ctypes.c_float()
    assert _L().delora_odometry_file_objective(ctypes.create_string_buffer(raw, 128), ctypes.byref(flags),
                                               ctypes.byref(lam)) == 0
    assert (flags.value, lam.value) == SHIPPED


@pytest.mark.parametrize("over,key", [
    ({"point_to_point_loss": False, "point_to_plane_loss": False, "plane_to_plane_loss": False}, "no loss is enabled"),
    ({"normal_loss": "cosine"}, "normal_loss"),
    ({"po2po_alone": True, "point_to_point_loss": True}, "po2po_alone"),
    ({"po2po_alone": True, "point_to_plane_loss": False}, "plane_to_plane_loss"),
    ({"po2po_alone": True, "plane_to_plane_loss": False}, "point_to_plane_loss")])
def test_export_refuses_what_the_reference_cannot_run(tmp_path, over, key):
    from delora_b200.deploy import export
    cfg = _cfg(**over)
    with pytest.raises(ValueError, match=key):
        export.objective_from_config(cfg)
    with pytest.raises(ValueError, match=key):
        export.export(_checkpoint(tmp_path, cfg), "kitti", os.path.join(tmp_path, "x.dlw"), n_stride=512)
    assert not os.path.exists(os.path.join(tmp_path, "x.dlw"))


@pytest.mark.parametrize("flags,lam,message", [
    (ALONE, 1.0, b"DELORA_LOSS_PO2PO_ALONE without DELORA_LOSS_PO2PO"),
    (PO2PO | ALONE | PO2PL, 1.0, b"with DELORA_LOSS_PO2PL"),
    (PO2PO | ALONE | PL2PL, 1.0, b"with DELORA_LOSS_PL2PL"),
    (PO2PO | ALONE | LINEAR, 1.0, b"with DELORA_NORMAL_LINEAR"),
    (LINEAR, 1.0, b"sets no loss bit"),
    (PO2PL | 1024, 1.0, b"has a bit other than"),
    (PO2PL, float("nan"), b"lambda_po2pl=nan")])
def test_file_objective_refuses_a_malformed_record(flags, lam, message):
    raw = bytearray(128)
    struct.pack_into("<If", raw, 108, flags, lam)
    f, l_ = ctypes.c_uint32(), ctypes.c_float()
    L = _L()
    assert L.delora_odometry_file_objective(ctypes.create_string_buffer(bytes(raw), 128), ctypes.byref(f),
                                            ctypes.byref(l_)) != 0
    err = L.delora_last_error()
    assert message in err and b"delora_odometry_file_objective" in err, err
    assert L.delora_odometry_file_objective(None, ctypes.byref(f), ctypes.byref(l_)) != 0
    assert b"null pointer" in L.delora_last_error()


def test_the_binding_takes_the_configured_objective_unless_given_one():
    from delora_b200.deploy import capi
    for over, (flags, lam) in CONFIGS.values():
        cfg = _cfg(**over)
        hp, rp = capi.train_params(cfg, 1e-5), capi.residual_params(cfg)
        assert (hp.loss_flags, rp.loss_flags) == (flags, flags)
        assert hp.lambda_po2pl == rp.lambda_po2pl == np.float32(lam)
    cfg = _cfg(po2po_alone=True, point_to_point_loss=True, point_to_plane_loss=False, plane_to_plane_loss=False)
    assert capi.train_params(cfg, 1e-5, loss_flags=PO2PL).loss_flags == PO2PL
    assert capi.residual_params(cfg, PO2PO).loss_flags == PO2PO
    cfg["normalization_scaling"] = True
    assert capi.train_params(cfg, 1e-5).loss_flags == PO2PO | ALONE | ops.TRAIN_NORMALIZATION_SCALING


# ---- DELORA_LOSS_PO2PO_ALONE: every entry point refuses it malformed, naming the flag, before any launch
BAD = [(ALONE, b"DELORA_LOSS_PO2PO_ALONE without DELORA_LOSS_PO2PO"),
       (PO2PO | ALONE | PO2PL, b"DELORA_LOSS_PO2PO_ALONE with DELORA_LOSS_PO2PL"),
       (PO2PO | ALONE | PL2PL, b"DELORA_LOSS_PO2PO_ALONE with DELORA_LOSS_PL2PL"),
       (PO2PO | ALONE | PO2PL | PL2PL | LINEAR, b"DELORA_LOSS_PO2PO_ALONE with DELORA_LOSS_PO2PL"),
       (PO2PO | ALONE | LINEAR, b"DELORA_LOSS_PO2PO_ALONE with DELORA_NORMAL_LINEAR")]


def _train_calls(L, flags):
    from delora_b200 import _lib
    d = H.desc(_cfg(), 1000, 2)
    d_pre = H.desc(_cfg(), 1000, 2, w_pre=360)
    descs = (_lib.OdometryDesc * 2)(d, d_pre)
    hp = H.train_params(flags)
    g = _lib.OdometryTrainGroup(rank=0, world=1, n_ctas=8, n_threads=128, status=16)
    g.peer_ws[0], g.peer_flags[0] = 4096, 4096
    ptrs = (ctypes.c_void_p * 2)(16, 16)
    by = ctypes.byref
    return {
        "delora_odometry_train_step": lambda: L.delora_odometry_train_step(by(d), by(hp), 16, 16, 1, 16, None, None,
                                                                           None, None, None),
        "delora_odometry_train_eval": lambda: L.delora_odometry_train_eval(by(d), by(hp), 16, 16, 1, 16, None, None,
                                                                           None, None),
        "delora_odometry_train_step_group": lambda: L.delora_odometry_train_step_group(
            by(d), by(hp), by(g), 16, 16, 1, 4096, None, None, None, None, None),
        "delora_odometry_streams_push_adapt": lambda: L.delora_odometry_streams_push_adapt(
            by(d), by(hp), 1, 16, 16, None, 16, 16, 16, 16, None),
        "delora_odometry_streams_push_adapt_info": lambda: L.delora_odometry_streams_push_adapt_info(
            by(d), by(hp), 1, 16, 16, None, 16, 16, 16, 16, 16, None),
        "delora_odometry_streams_push_adapt_group": lambda: L.delora_odometry_streams_push_adapt_group(
            by(d), by(hp), by(g), 1, 16, 16, None, 4096, 16, 16, 16, None),
        "delora_odometry_streams_push_adapt_group_info": lambda: L.delora_odometry_streams_push_adapt_group_info(
            by(d), by(hp), by(g), 1, 16, 16, None, 4096, 16, 16, 16, 16, None),
        "delora_odometry_streams_push_adapt_geometries": lambda: L.delora_odometry_streams_push_adapt_geometries(
            descs, 2, by(hp), 1, ptrs, ptrs, None, 16, 16, 16, 16, None),
        "delora_odometry_streams_push_adapt_geometries_info":
            lambda: L.delora_odometry_streams_push_adapt_geometries_info(descs, 2, by(hp), 1, ptrs, ptrs, None, 16, 16,
                                                                         16, 16, 16, None),
    }


def _streams_calls(L, flags):
    from delora_b200 import _lib
    d = H.desc(_cfg(), 1000, 2)
    d_pre = H.desc(_cfg(), 1000, 2, w_pre=360)
    rp = _lib.OdometryResidualParams(lambda_po2pl=1.0, loss_flags=flags, nb_h=7, nb_w=11, epsilon_range=0.5,
                                     min_neighbors=10)
    by = ctypes.byref
    return {
        "delora_odometry_streams_push_residual": lambda: L.delora_odometry_streams_push_residual(
            by(d), by(rp), 16, 16, None, 16, 16, 16, 16, None),
        "delora_odometry_streams_push_info": lambda: L.delora_odometry_streams_push_info(
            by(d), by(rp), 16, 16, None, 16, 16, 16, 16, 16, None),
        "delora_odometry_streams_push_pre": lambda: L.delora_odometry_streams_push_pre(
            by(d_pre), by(rp), 16, 16, None, 16, 16, 16, 16, None, None),
        "delora_odometry_streams_push_pre_info": lambda: L.delora_odometry_streams_push_pre_info(
            by(d_pre), by(rp), 16, 16, None, 16, 16, 16, 16, None, 16, None),
    }


@pytest.mark.parametrize("flags,message", BAD)
def test_every_entry_point_refuses_a_malformed_po2po_alone(flags, message):
    L = _L()
    calls = {**_train_calls(L, flags), **_streams_calls(L, flags)}
    assert len(calls) == 13
    for name, call in calls.items():
        assert call() != 0, name
        err = L.delora_last_error()
        assert name.encode() in err and message in err, (name, err)


@pytest.mark.parametrize("extra", [0, ops.LOSS_IDENTITY_FIT, ops.TRAIN_DROPOUT, ops.TRAIN_NORMALIZATION_SCALING])
def test_a_well_formed_po2po_alone_passes_the_objective_checks(extra):
    """PO2PO | PO2PO_ALONE with each training bit: the calls get past every flag check and stop at the argument
    refusal that follows them (a batch above max_batch, a null points), so nothing is launched."""
    from delora_b200 import _lib
    L = _L()
    d = H.desc(_cfg(), 1000, 2, w_pre=360)
    hp = H.train_params(PO2PO | ALONE | extra)
    assert L.delora_odometry_train_step(ctypes.byref(d), ctypes.byref(hp), 16, 16, 3, 16, None, None, None, None,
                                        None) != 0
    err = L.delora_last_error()
    assert b"B=3 outside [1, max_batch=2]" in err, err
    rp = _lib.OdometryResidualParams(lambda_po2pl=1.0, loss_flags=PO2PO | ALONE | (extra & ops.TRAIN_NORMALIZATION_SCALING),
                                     nb_h=7, nb_w=11, epsilon_range=0.5, min_neighbors=10)
    assert L.delora_odometry_streams_push_pre(ctypes.byref(d), ctypes.byref(rp), None, 16, None, 16, 16, 16, 16, None,
                                              None) != 0
    assert b"null points" in L.delora_last_error(), L.delora_last_error()


def test_project_points_refuses_bad_arguments():
    L = _L()
    args = [16, 16, 1, 3, 100, 16, 180, -3.14, 3.14, -0.4, 0.05, 0, 16, 16, 16, 16, 16, None]
    for i, message in [(0, b"null pointer"), (15, b"null pointer"), (16, b"null pointer")]:
        bad = list(args)
        bad[i] = None
        assert L.delora_project_points_fwd(*bad) != 0
        assert b"delora_project_points_fwd" in L.delora_last_error() and message in L.delora_last_error()
    bad = list(args)
    bad[3] = 5
    assert L.delora_project_points_fwd(*bad) != 0 and b"C must be 3 or 4" in L.delora_last_error()
