"""-m "not gpu": the odometry training entry points of the C ABI without a device -- exported symbols, the training
workspace size, argument validation (every refusal names its field), unpack_blob as the inverse of pack_state_dict,
and that examples/odometry_finetune.c compiles against the header."""
import ctypes
import os
import subprocess

import pytest
import torch

from helpers import ROOT

TRAIN_SYMBOLS = ("delora_odometry_train_workspace_bytes", "delora_odometry_train_init", "delora_odometry_train_step",
                 "delora_odometry_train_weights")


def _config(act="tanh", single=False, layers=(2, 2, 2, 2), nout=1000, h=64, w=720):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w)
    cfg.update({"activation_fct": act, "use_single_mlp_at_output": single, "layers": list(layers), "resnet_outputs": nout,
                "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1, "use_dropout": False})
    return cfg


def _desc(cfg, n_stride=1000, max_batch=1):
    from delora_b200.deploy import export
    return export.desc_from_config(cfg, "kitti", n_stride, max_batch)


def _params(**kw):
    from delora_b200 import _lib
    hp = _lib.OdometryTrainParams(lr=1e-5, beta1=0.9, beta2=0.999, eps=1e-8, lambda_po2pl=1.0, loss_flags=2 | 4,
                                  nb_h=7, nb_w=11, epsilon_range=0.5, min_neighbors=10)
    for k, v in kw.items():
        setattr(hp, k, v)
    return hp


def test_symbols_exported_and_abi_version_unchanged():
    from delora_b200 import _lib
    L = _lib.lib()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in TRAIN_SYMBOLS:
        assert hasattr(handle, name), name
        assert name in _lib.SIGNATURES, name
    assert L.delora_abi_version() == _lib.ABI_VERSION == 3


def test_train_workspace_bytes():
    from delora_b200 import _lib
    L = _lib.lib()
    cfg = _config(h=64, w=2048)
    sizes = [L.delora_odometry_train_workspace_bytes(ctypes.byref(_desc(cfg, 131072, mb))) for mb in (1, 4, 16)]
    assert 0 < sizes[0] < sizes[1] < sizes[2]
    assert all(s % 256 == 0 for s in sizes)
    # the training workspace holds everything inference needs and more
    assert sizes[0] > L.delora_odometry_workspace_bytes(ctypes.byref(_desc(cfg, 131072, 1)))
    for single in (False, True):
        for w in (720, 259):
            d = _desc(_config("relu", single, h=16, w=w), 4096, 2)
            n = L.delora_odometry_train_workspace_bytes(ctypes.byref(d))
            assert n > 0 and n % 256 == 0
    bad = _desc(cfg, 131072, 1)
    bad.act = 0
    assert L.delora_odometry_train_workspace_bytes(ctypes.byref(bad)) == -1
    assert b"act=0" in L.delora_last_error()
    assert L.delora_odometry_train_workspace_bytes(None) == -1
    assert b"null descriptor" in L.delora_last_error()


@pytest.mark.parametrize("field,value,message", [
    ("lr", -1e-3, b"lr="), ("lr", float("nan"), b"lr="), ("beta1", 1.0, b"beta1="), ("beta1", -0.1, b"beta1="),
    ("beta2", 1.0, b"beta2="), ("beta2", float("nan"), b"beta2="), ("eps", 0.0, b"eps="), ("eps", -1e-8, b"eps="),
    ("nb_h", 0, b"nb_h=0"), ("nb_h", 6, b"nb_h=6"), ("nb_w", 10, b"nb_w=10"), ("nb_w", -11, b"nb_w=-11"),
    ("loss_flags", 0, b"loss_flags=0x0"), ("loss_flags", 8, b"loss_flags=0x8"),
    ("lambda_po2pl", float("inf"), b"lambda_po2pl="), ("min_neighbors", -1, b"min_neighbors=-1"),
    ("epsilon_range", -0.5, b"epsilon_range=")])
def test_invalid_parameters_are_refused_without_a_gpu(field, value, message):
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc(_config(), max_batch=2)
    hp = _params(**{field: value})
    dummy = ctypes.c_void_p(16)             # never dereferenced: the call is refused before any launch
    rc = L.delora_odometry_train_step(ctypes.byref(d), ctypes.byref(hp), dummy, dummy, 1, dummy, None, None, None, None,
                                      None)
    assert rc != 0
    assert message in L.delora_last_error()


def test_invalid_arguments_are_refused_without_a_gpu():
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc(_config(), max_batch=2)
    hp = _params()
    dummy = ctypes.c_void_p(16)

    def step(desc, params, points, counts, b, ws):
        return L.delora_odometry_train_step(desc, params, points, counts, b, ws, None, None, None, None, None)

    assert step(ctypes.byref(d), ctypes.byref(hp), dummy, dummy, 3, dummy) != 0
    assert b"B=3 outside [1, max_batch=2]" in L.delora_last_error()
    assert step(ctypes.byref(d), ctypes.byref(hp), dummy, dummy, 0, dummy) != 0
    assert b"B=0" in L.delora_last_error()
    for args in ((None, dummy, dummy), (dummy, None, dummy), (dummy, dummy, None)):
        assert step(ctypes.byref(d), ctypes.byref(hp), args[0], args[1], 1, args[2]) != 0
        assert b"null pointer" in L.delora_last_error()
    assert step(ctypes.byref(d), None, dummy, dummy, 1, dummy) != 0
    assert b"null hyperparameters" in L.delora_last_error()
    assert step(None, ctypes.byref(hp), dummy, dummy, 1, dummy) != 0
    assert b"null descriptor" in L.delora_last_error()
    bad = _desc(_config(), max_batch=2)
    bad.single_mlp = 2
    assert step(ctypes.byref(bad), ctypes.byref(hp), dummy, dummy, 1, dummy) != 0
    assert b"single_mlp=2" in L.delora_last_error()
    assert L.delora_odometry_train_init(ctypes.byref(d), None, dummy, None) != 0
    assert b"null pointer" in L.delora_last_error()
    assert L.delora_odometry_train_init(ctypes.byref(bad), dummy, dummy, None) != 0
    assert b"single_mlp=2" in L.delora_last_error()
    assert L.delora_odometry_train_weights(ctypes.byref(d), None, dummy, None) != 0
    assert b"null pointer" in L.delora_last_error()
    assert L.delora_odometry_train_weights(ctypes.byref(d), dummy, None, None) != 0
    assert b"null pointer" in L.delora_last_error()


@pytest.mark.parametrize("act", ["tanh", "relu"])
@pytest.mark.parametrize("single", [False, True])
def test_unpack_blob_inverts_pack_state_dict(act, single):
    from delora_b200.deploy import export
    from delora_b200.models.model import OdometryModel
    cfg = _config(act, single, (1, 2, 1, 2), 500, h=16, w=720)
    torch.manual_seed(7)
    sd = OdometryModel(dict(cfg, device="cpu")).state_dict()
    back = export.unpack_blob(export.pack_state_dict(sd, cfg), cfg)
    assert list(back) == list(sd)
    for k in sd:
        assert back[k].dtype == torch.float32 and back[k].shape == sd[k].shape, k
        assert torch.equal(back[k], sd[k]), k
    model = OdometryModel(dict(cfg, device="cpu"))
    model.load_state_dict(back)
    with pytest.raises(ValueError, match="floats"):
        export.unpack_blob(export.pack_state_dict(sd, cfg)[:-1], cfg)


def test_finetune_example_compiles_against_the_header(tmp_path):
    from delora_b200 import build
    nvcc = build._nvcc()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    r = subprocess.run([nvcc, "-c", os.path.join(ROOT, "examples", "odometry_finetune.c"), "-I",
                        os.path.join(ROOT, "include"), "-I", cuda_inc, "-Xcompiler", "-Wall,-Werror", "-o",
                        os.path.join(tmp_path, "odometry_finetune.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
