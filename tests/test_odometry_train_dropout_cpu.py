"""-m "not gpu": training models configured with use_dropout through the C ABI -- the mask contract (the numpy
Philox4x32-10 of dropout_reference.py against published known-answer vectors, and against the header the kernels use,
compiled for the host),
the DELORA_MODEL_DROPOUT bit and the .dlt seed through the files and conversions, the binding, the host-side refusals
and the structs' layout."""
import ctypes
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

import odometry_harness as H
from dropout_reference import KEEP_BELOW, keep_mask, philox4x32_10
from helpers import ROOT

KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize("counter,key,want", KAT)
def test_numpy_philox_known_answers(counter, key, want):
    assert tuple(int(w) for w in philox4x32_10(counter, key)) == want


def test_the_threshold_is_0_8f():
    assert np.float32(KEEP_BELOW * 2.0 ** -24) == np.float32(0.8)
    assert np.float32((KEEP_BELOW - 1) * 2.0 ** -24) < np.float32(0.8)
    assert np.float32(1.0) / (np.float32(1.0) - np.float32(0.2)) == np.float32(1.25)


def test_the_kernels_generator_matches_numpy_on_the_host(tmp_path):
    """dropout.cuh (the device function of the step and of delora_dropout_keep_mask) compiled for the host: the known
    answers, and masks of every tensor id at large seeds and steps."""
    from delora_b200 import build
    src = os.path.join(tmp_path, "philox.cu")
    cases = [(0, 0, 0, 37), (1, 7, 1, 64), (2 ** 64 - 1, 2 ** 32 + 3, 2, 41), (0x0123456789ABCDEF, 12345, 0, 1000)]
    lines = ["#include <stdio.h>", '#include "dropout.cuh"', "using namespace delora;", "int main() {"]
    for c, k, _ in KAT:
        lines.append("  { Philox4 r = philox4x32_10(Philox4{%uu, %uu, %uu, %uu}, %uu, %uu);" % (*c, *k))
        lines.append('    printf("%08x %08x %08x %08x\\n", r.x, r.y, r.z, r.w); }')
    for seed, step, t, n in cases:
        lines.append("  for (unsigned long long i = 0; i < %du; ++i) putchar(dropout_keep(%luull, %luull, %d, i) ? '1' : '0');"
                     % (n, seed, step, t))
        lines.append('  putchar(\'\\n\');')
    lines.append("  return 0;\n}\n")
    with open(src, "w") as f:
        f.write("\n".join(lines))
    exe = os.path.join(tmp_path, "philox")
    r = subprocess.run([build._nvcc(), src, "-I", os.path.join(ROOT, "include"), "-I", build.CSRC, "-std=c++17",
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")
    for (_, _, want), line in zip(KAT, out):
        assert line == " ".join("%08x" % w for w in want)
    for (seed, step, t, n), line in zip(cases, out[len(KAT):]):
        assert line == "".join("1" if k else "0" for k in keep_mask(seed, step, t, n)), (seed, step, t)


def _cfg(dropout=True, normalized=False):
    cfg = H.config(16, 256, "tanh", False, (1, 1, 1, 1), 100, device="cpu")
    cfg["use_dropout"] = dropout
    cfg["normalization_scaling"] = normalized
    return cfg


def _checkpoint(tmp_path, cfg, name="ckpt.pth", seed=0):
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(seed)
    model = OdometryModel(dict(cfg, device="cpu"))
    path = os.path.join(tmp_path, name)
    torch.save({"epoch": 0, "model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, path)
    return path


@pytest.mark.parametrize("dropout,normalized", [(True, False), (True, True), (False, False)])
def test_export_sets_the_flag_and_the_conversions_carry_it(tmp_path, dropout, normalized):
    from delora_b200 import _lib
    from delora_b200.deploy import export
    cfg = _cfg(dropout, normalized)
    want = (_lib.MODEL_DROPOUT if dropout else 0) | (_lib.MODEL_NORMALIZATION_SCALING if normalized else 0)
    assert export.model_flags_from_config(cfg) == want
    ckpt = _checkpoint(tmp_path, cfg)
    dlw = os.path.join(tmp_path, "m.dlw")
    export.export(ckpt, "kitti", dlw, n_stride=512)
    h, d, blob = export.read_dlw(dlw)
    assert h["model_flags"] == want
    # dropout has no parameters: the blob is the one of the same model without it
    plain = os.path.join(tmp_path, "plain.dlw")
    export.export(_checkpoint(tmp_path, _cfg(False, normalized), "plain.pth"), "kitti", plain, n_stride=512)
    assert export.read_dlw(plain)[2].tobytes() == blob.tobytes()
    cfg_back = export.config_from_desc(d, None, "kitti", h["model_flags"])
    assert cfg_back["use_dropout"] is dropout and cfg_back["normalization_scaling"] is normalized
    # checkpoint -> .dlt -> reference checkpoint: `parameters` gets use_dropout back
    dlt = os.path.join(tmp_path, "m.dlt")
    export.export(ckpt, "kitti", dlt, n_stride=512, training_state=True)
    assert export.read_dlt(dlt)[0]["model_flags"] == want
    out = os.path.join(tmp_path, "back.pth")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "training_state_to_checkpoint.py"), "--dlt", dlt,
                        "--out", out], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    back = torch.load(out, map_location="cpu", weights_only=False)
    assert back["parameters"]["use_dropout"] is dropout
    assert back["parameters"]["normalization_scaling"] is normalized
    again = os.path.join(tmp_path, "again.dlw")
    export.export(out, "kitti", again, n_stride=512)
    assert export.read_dlw(again)[0]["model_flags"] == want


def test_a_file_without_the_bit_reads_as_no_dropout(tmp_path):
    """Files written before DELORA_MODEL_DROPOUT have a 0 or 1 (normalisation) in model_flags; a YAML base that says
    use_dropout: True does not win over the file."""
    from delora_b200.deploy import export
    d = H.desc(_cfg(), 1000, 1)
    for flags in (0, 1):
        path = os.path.join(tmp_path, f"old{flags}.dlw")
        export.write_dlw(path, d, np.ones(3, dtype=np.float32), flags)
        h, _, _ = export.read_dlw(path)
        assert export.config_from_desc(d, {"use_dropout": True}, "kitti", h["model_flags"])["use_dropout"] is False
    assert export.config_from_desc(d, None, "kitti", None)["use_dropout"] is False


@pytest.mark.parametrize("seed", [0, 1, 2 ** 63 + 5, 2 ** 64 - 1])
def test_the_seed_round_trips_through_dlt_bytes_164_to_171(tmp_path, seed):
    from delora_b200.deploy import export
    d = H.desc(_cfg(), 1000, 2)
    blob = np.arange(7, dtype=np.float32)
    path = os.path.join(tmp_path, "m.dlt")
    export.write_dlt(path, d, export.TrainingState(blob, blob * 2, blob * 3, 5, dropout_seed=seed), 3)
    with open(path, "rb") as f:
        raw = f.read(256)
    assert struct.unpack_from("<Q", raw, 164)[0] == seed
    assert raw[172:256] == bytes(84) and struct.unpack_from("<I", raw, 104)[0] == 3
    h, _, st = export.read_dlt(path)
    assert st.dropout_seed == seed and st.step == 5 and h["model_flags"] == 3
    # the default state writes seed 0: all zeros from byte 164, as before the field
    export.write_dlt(path, d, export.TrainingState(blob, blob, blob))
    with open(path, "rb") as f:
        assert f.read(256)[164:256] == bytes(92)


def test_train_params_sets_the_bit():
    from delora_b200 import ops
    from delora_b200.deploy import capi
    assert ops.TRAIN_DROPOUT == 2048
    assert capi.train_params(_cfg(True), 1e-5).loss_flags & ops.TRAIN_DROPOUT == 2048
    assert capi.train_params(_cfg(False), 1e-5).loss_flags & ops.TRAIN_DROPOUT == 0
    both = capi.train_params(_cfg(True, True), 1e-5).loss_flags
    assert both & ops.TRAIN_DROPOUT and both & ops.TRAIN_NORMALIZATION_SCALING


def test_symbols_and_defines():
    import re
    from delora_b200 import _lib, ops
    _lib.lib()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("delora_odometry_train_set_dropout_seed", "delora_dropout_keep_mask"):
        assert hasattr(handle, name) and name in _lib.SIGNATURES, name
    with open(os.path.join(ROOT, "include", "delora_b200.h")) as f:
        defines = {k: int(v) for k, v in re.findall(r"#define DELORA_(\w+)\s+(\d+)u?\b", f.read())}
    assert defines["TRAIN_DROPOUT"] == ops.TRAIN_DROPOUT
    assert defines["MODEL_DROPOUT"] == _lib.MODEL_DROPOUT == 2
    assert _lib.ABI_VERSION == 3


def test_set_dropout_seed_refusals_name_their_argument():
    from delora_b200 import _lib
    L = _lib.lib()
    d = H.desc(_cfg(), 1000, 2)
    assert L.delora_odometry_train_set_dropout_seed(ctypes.byref(d), 1, None, None) != 0
    assert b"null workspace" in L.delora_last_error()
    assert L.delora_odometry_train_set_dropout_seed(None, 1, ctypes.c_void_p(16), None) != 0
    assert b"null descriptor" in L.delora_last_error()
    d.act = 0
    assert L.delora_odometry_train_set_dropout_seed(ctypes.byref(d), 1, ctypes.c_void_p(16), None) != 0
    assert b"act=0" in L.delora_last_error()
    d.act, d.w_pre = 2, 1
    assert L.delora_odometry_train_set_dropout_seed(ctypes.byref(d), 1, ctypes.c_void_p(16), None) != 0
    assert b"w_pre=1" in L.delora_last_error()


def test_keep_mask_refusals_name_their_argument():
    from delora_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(16)                    # never dereferenced: every call below is refused first
    for args, message in [((0, 0, 0, 4, None), b"null keep"), ((0, 0, 0, -1, p), b"n=-1"),
                          ((0, 0, 3, 4, p), b"tensor=3"), ((0, 0, -1, 4, p), b"tensor=-1")]:
        assert L.delora_dropout_keep_mask(*args, None) != 0
        assert message in L.delora_last_error(), (args, L.delora_last_error())


def test_struct_layout_in_c(tmp_path):
    """No struct changes size; the seed sits at byte 164 of the training header."""
    from delora_b200 import build
    src = os.path.join(tmp_path, "layout.c")
    with open(src, "w") as f:
        f.write('#include <stddef.h>\n#include "delora_b200.h"\n'
                "_Static_assert(sizeof(delora_odometry_file_header) == 128, \"size\");\n"
                "_Static_assert(offsetof(delora_odometry_file_header, model_flags) == 104, \"model_flags\");\n"
                "_Static_assert(sizeof(delora_odometry_train_file_header) == 256, \"training size\");\n"
                "_Static_assert(offsetof(delora_odometry_train_file_header, loss) == 160, \"loss\");\n"
                "_Static_assert(offsetof(delora_odometry_train_file_header, dropout_seed) == 164, \"seed\");\n"
                "_Static_assert(offsetof(delora_odometry_train_file_header, reserved) == 172, \"reserved\");\n"
                "_Static_assert(sizeof(delora_odometry_train_params) == 40, \"train params\");\n"
                "_Static_assert(sizeof(delora_odometry_desc) == 80, \"desc\");\n"
                "_Static_assert(DELORA_MODEL_DROPOUT == 2u, \"model flag\");\n"
                "_Static_assert(DELORA_TRAIN_DROPOUT == 2048u, \"train flag\");\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n")
    r = subprocess.run([build._nvcc(), "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "layout.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("name", ["odometry_finetune", "odometry_train"])
def test_examples_compile(tmp_path, name):
    H.build_example(name, tmp_path, link=False)
