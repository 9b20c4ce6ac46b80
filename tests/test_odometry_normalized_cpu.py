"""-m "not gpu": models trained with normalization_scaling -- the header's model_flags word (byte 104 of .dlw and .dlt
files), the exporter and the conversions that carry it, the host-side refusals of delora_normalization_factors and
delora_odometry_pairs_normalized, the exported symbols, OdometryStreams' refusal and the examples' compilation."""
import ctypes
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

import odometry_harness as H
from helpers import ROOT

SYMBOLS = ("delora_normalization_factors", "delora_odometry_pairs_normalized")


def _cfg(normalized=True):
    cfg = H.config(16, 256, "tanh", False, (1, 1, 1, 1), 100, device="cpu")
    cfg["normalization_scaling"] = normalized
    return cfg


def _checkpoint(tmp_path, cfg, seed=0):
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(seed)
    model = OdometryModel(dict(cfg, device="cpu"))
    path = os.path.join(tmp_path, "ckpt.pth")
    torch.save({"epoch": 0, "model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, path)
    return path


def _word_104(path):
    with open(path, "rb") as f:
        raw = f.read(128)
    return struct.unpack_from("<I", raw, 104)[0], raw[108:128]


def test_symbols_exported():
    from delora_b200 import _lib
    _lib.lib()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in SYMBOLS:
        assert hasattr(handle, name), name
        assert name in _lib.SIGNATURES, name


def test_header_layout_in_c(tmp_path):
    """The C struct puts model_flags at byte 104 and keeps both headers' sizes."""
    from delora_b200 import build
    src = os.path.join(tmp_path, "layout.c")
    with open(src, "w") as f:
        f.write('#include <stddef.h>\n#include "delora_b200.h"\n'
                "_Static_assert(offsetof(delora_odometry_file_header, model_flags) == 104, \"model_flags\");\n"
                "_Static_assert(offsetof(delora_odometry_file_header, blob_floats) == 96, \"blob_floats\");\n"
                "_Static_assert(sizeof(delora_odometry_file_header) == 128, \"size\");\n"
                "_Static_assert(sizeof(delora_odometry_train_file_header) == 256, \"training size\");\n"
                "_Static_assert(DELORA_MODEL_NORMALIZATION_SCALING == 1u, \"flag\");\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n")
    r = subprocess.run([build._nvcc(), "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "layout.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("flags", [0, 1])
def test_flag_round_trips_through_dlw_and_dlt(tmp_path, flags):
    from delora_b200.deploy import export
    d = H.desc(_cfg(), 1000, 2)
    blob = np.arange(7, dtype=np.float32)
    dlw = os.path.join(tmp_path, "m.dlw")
    export.write_dlw(dlw, d, blob, flags)
    assert _word_104(dlw) == (flags, bytes(20))
    h, _, back = export.read_dlw(dlw)
    assert h["model_flags"] == flags and back.tobytes() == blob.tobytes()
    dlt = os.path.join(tmp_path, "m.dlt")
    export.write_dlt(dlt, d, export.TrainingState(blob, blob * 2, blob * 3, 5), flags)
    assert _word_104(dlt) == (flags, bytes(20))
    h, _, st = export.read_dlt(dlt)
    assert h["model_flags"] == flags and st.step == 5


def test_a_file_written_before_the_field_reads_as_off(tmp_path):
    """Exporters before model_flags wrote 24 zero bytes from byte 104."""
    from delora_b200 import _lib
    from delora_b200.deploy import export
    d = H.desc(_cfg(), 1000, 1)
    old = struct.Struct("<8sii" + "ii4d" + "iii4iiii" + "q" + "24x")
    path = os.path.join(tmp_path, "old.dlw")
    with open(path, "wb") as f:
        f.write(old.pack(export.MAGIC, _lib.ABI_VERSION, 128, d.H, d.W, d.hfov0, d.hfov1, d.vfov0, d.vfov1, d.n_stride,
                         d.max_batch, d.act, *list(d.layers), d.resnet_outputs, d.single_mlp, d.w_pre, 3))
        f.write(np.ones(3, dtype=np.float32).tobytes())
    h, _, _ = export.read_dlw(path)
    assert h["model_flags"] == 0
    assert export.config_from_desc(d, None, "kitti", h["model_flags"])["normalization_scaling"] is False


@pytest.mark.parametrize("normalized", [True, False])
def test_export_sets_the_flag_and_the_conversions_carry_it(tmp_path, normalized):
    from delora_b200 import _lib
    from delora_b200.deploy import export
    cfg = _cfg(normalized)
    ckpt = _checkpoint(tmp_path, cfg)
    want = _lib.MODEL_NORMALIZATION_SCALING if normalized else 0
    dlw = os.path.join(tmp_path, "m.dlw")
    export.export(ckpt, "kitti", dlw, n_stride=512)
    assert export.read_dlw(dlw)[0]["model_flags"] == want
    # checkpoint -> .dlt -> reference checkpoint: `parameters` gets normalization_scaling back
    dlt = os.path.join(tmp_path, "m.dlt")
    export.export(ckpt, "kitti", dlt, n_stride=512, training_state=True)
    h, d, _ = export.read_dlt(dlt)
    assert h["model_flags"] == want
    out = os.path.join(tmp_path, "back.pth")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "training_state_to_checkpoint.py"), "--dlt", dlt,
                        "--out", out], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    back = torch.load(out, map_location="cpu", weights_only=False)
    assert back["parameters"]["normalization_scaling"] is normalized
    # ... and exporting that checkpoint again writes the same flag
    again = os.path.join(tmp_path, "again.dlw")
    export.export(out, "kitti", again, n_stride=512)
    assert export.read_dlw(again)[0]["model_flags"] == want
    assert export.model_flags_from_config(back["parameters"]) == want


def test_factor_refusals_name_their_argument():
    from delora_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(16)                    # never dereferenced: every call below is refused first
    for args, message in [((None, p, 1, 10, p), b"null points"), ((p, None, 1, 10, p), b"null n_points"),
                          ((p, p, 1, 10, None), b"null factor"), ((p, p, 0, 10, p), b"B=0"),
                          ((p, p, 70000, 10, p), b"B=70000"), ((p, p, 1, 0, p), b"n_stride=0")]:
        assert L.delora_normalization_factors(*args, None) != 0
        assert message in L.delora_last_error(), (args, L.delora_last_error())


def test_pairs_normalized_refusals_name_their_argument():
    from delora_b200 import _lib
    L = _lib.lib()
    d = H.desc(_cfg(), 1000, 2)
    dp = ctypes.byref(d)
    p = ctypes.c_void_p(16)
    for args, message in [((None, p, 1, p, p, None, p), b"null points"), ((p, None, 1, p, p, None, p), b"null n_points"),
                          ((p, p, 1, None, p, None, p), b"null workspace"), ((p, p, 1, p, None, None, p), b"null T"),
                          ((p, p, 1, p, p, None, None), b"null factor"), ((p, p, 0, p, p, None, p), b"B=0"),
                          ((p, p, 3, p, p, None, p), b"B=3 outside [1, max_batch=2]")]:
        assert L.delora_odometry_pairs_normalized(dp, *args, None) != 0
        assert message in L.delora_last_error(), (args, L.delora_last_error())
    d.act = 0
    assert L.delora_odometry_pairs_normalized(dp, p, p, 1, p, p, None, p, None) != 0
    assert b"act=0" in L.delora_last_error()


def test_streams_refuse_a_normalised_model():
    from delora_b200.deploy.stream import OdometryStreams
    with pytest.raises(ValueError, match="normalization_scaling"):
        OdometryStreams(None, dict(_cfg(), device="cuda"), "kitti", 2, 1000)


@pytest.mark.parametrize("name", ["odometry_stream", "odometry_streams", "odometry_finetune", "odometry_train"])
def test_examples_compile(tmp_path, name):
    H.build_example(name, tmp_path, link=False)


def test_training_bit_refuses_w_pre_zero():
    """DELORA_TRAIN_NORMALIZATION_SCALING needs the reference's recipe: w_pre = 0 is refused before any launch."""
    from delora_b200 import _lib, ops
    from delora_b200.deploy import capi
    L = _lib.lib()
    cfg = _cfg()
    d = H.desc(cfg, 1000, 2)
    hp = capi.train_params(cfg, 1e-5)
    assert hp.loss_flags & ops.TRAIN_NORMALIZATION_SCALING
    assert capi.train_params(_cfg(False), 1e-5).loss_flags & ops.TRAIN_NORMALIZATION_SCALING == 0
    p = ctypes.c_void_p(16)
    rc = L.delora_odometry_train_step(ctypes.byref(d), ctypes.byref(hp), p, p, 1, p, None, None, None, None, None)
    assert rc != 0 and b"w_pre=0" in L.delora_last_error(), L.delora_last_error()
    # the training workspace does not grow with the bit: its layout is a function of the descriptor alone
    d.w_pre = 512
    assert L.delora_odometry_train_workspace_bytes(ctypes.byref(d)) > 0


def test_training_bit_matches_the_header():
    import re
    from delora_b200 import ops
    with open(os.path.join(ROOT, "include", "delora_b200.h")) as f:
        text = f.read()
    defines = {k: int(v) for k, v in re.findall(r"#define DELORA_(\w+)\s+(\d+)u?\b", text)}
    assert defines["TRAIN_NORMALIZATION_SCALING"] == ops.TRAIN_NORMALIZATION_SCALING == 1024
