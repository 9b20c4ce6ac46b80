"""-m "not gpu": the odometry training entry points of the C ABI without a device -- exported symbols, the training
workspace size, argument validation (every refusal names its field), unpack_blob as the inverse of pack_state_dict,
and that examples/odometry_finetune.c compiles against the header."""
import ctypes

import pytest
import torch

import odometry_harness as H

TRAIN_SYMBOLS = ("delora_odometry_train_workspace_bytes", "delora_odometry_train_init", "delora_odometry_train_step",
                 "delora_odometry_train_weights")


def _params(**kw):
    from delora_b200.deploy import capi
    hp = capi.train_params(H.config(64, 720, device="cpu"), 1e-5)
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
    cfg = H.config(64, 2048, device="cpu")
    sizes = [L.delora_odometry_train_workspace_bytes(ctypes.byref(H.desc(cfg, 131072, mb))) for mb in (1, 4, 16)]
    assert 0 < sizes[0] < sizes[1] < sizes[2]
    assert all(s % 256 == 0 for s in sizes)
    # the training workspace holds everything inference needs and more
    assert sizes[0] > L.delora_odometry_workspace_bytes(ctypes.byref(H.desc(cfg, 131072, 1)))
    for single in (False, True):
        for w in (720, 259):
            d = H.desc(H.config(16, w, "relu", single, device="cpu"), 4096, 2)
            n = L.delora_odometry_train_workspace_bytes(ctypes.byref(d))
            assert n > 0 and n % 256 == 0
    bad = H.desc(cfg, 131072, 1)
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
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 2)
    hp = _params(**{field: value})
    dummy = ctypes.c_void_p(16)             # never dereferenced: the call is refused before any launch
    rc = L.delora_odometry_train_step(ctypes.byref(d), ctypes.byref(hp), dummy, dummy, 1, dummy, None, None, None, None,
                                      None)
    assert rc != 0
    assert message in L.delora_last_error()


def test_invalid_arguments_are_refused_without_a_gpu():
    from delora_b200 import _lib
    L = _lib.lib()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 2)
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
    bad = H.desc(H.config(64, 720, device="cpu"), 1000, 2)
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
    cfg = H.config(16, 720, act, single, (1, 2, 1, 2), 500, device="cpu")
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
    H.build_example("odometry_finetune", tmp_path, link=False)
