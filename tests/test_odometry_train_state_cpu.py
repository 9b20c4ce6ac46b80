"""-m "not gpu": training checkpoints (.dlt) and the optimizer-state entry points of the C ABI without a device -- the
.dlt header byte by byte, torch Adam state -> .dlt -> checkpoint dict without a changed bit, the refusals of
checkpoints the C step cannot continue (each names its key), --init-seed, host-side refusals of
delora_odometry_train_get_state / _set_state and of an identity-only loss_flags, and that examples/odometry_train.c
compiles against the header."""
import ctypes
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT


def _config(act="tanh", single=False):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=16, w=720)
    cfg.update({"activation_fct": act, "use_single_mlp_at_output": single, "layers": [1, 1, 1, 1], "resnet_outputs": 64,
                "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1, "use_dropout": False})
    return cfg


def _desc(cfg, n_stride=1000, max_batch=2):
    from delora_b200.deploy import export
    return export.desc_from_config(cfg, "kitti", n_stride, max_batch)


def _trained(cfg, steps=3, lr=2.0 ** -10, betas=(0.875, 0.9921875), eps=2.0 ** -24, **adam):
    """A CPU model and torch Adam after `steps` updates with seeded random gradients (hyperparameters exact in fp32)."""
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(11)
    model = OdometryModel(dict(cfg, device="cpu"))
    opt = torch.optim.Adam(model.parameters(), lr=lr, betas=betas, eps=eps, **adam)
    gen = torch.Generator().manual_seed(5)
    for _ in range(steps):
        for p in model.parameters():
            p.grad = torch.randn(p.shape, generator=gen)
        opt.step()
    return model, opt


def test_dlt_header_offsets(tmp_path):
    from delora_b200 import _lib
    from delora_b200.deploy import export
    cfg = _config()
    d = _desc(cfg)
    n = 12
    st = export.TrainingState(np.arange(n, dtype=np.float32), np.full(n, 2.0, np.float32), np.full(n, 3.0, np.float32),
                              step=123456789012, epoch=7, unsupervised=1, lr=0.25, beta1=0.5, beta2=0.75, eps=0.125,
                              loss=1.5)
    path = os.path.join(tmp_path, "s.dlt")
    export.write_dlt(path, d, st)
    raw = open(path, "rb").read()
    assert len(raw) == 256 + 3 * n * 4
    assert raw[0:8] == b"DELORAT\x00"
    assert struct.unpack_from("<ii", raw, 8) == (_lib.ABI_VERSION, 256)
    assert struct.unpack_from("<ii", raw, 16) == (16, 720)
    assert struct.unpack_from("<4d", raw, 24) == (d.hfov0, d.hfov1, d.vfov0, d.vfov1)
    assert struct.unpack_from("<iii", raw, 56) == (1000, 2, 2)
    assert struct.unpack_from("<4i", raw, 68) == (1, 1, 1, 1)
    assert struct.unpack_from("<iii", raw, 84) == (64, 0, 0)
    assert struct.unpack_from("<q", raw, 96) == (n,)
    assert raw[104:128] == bytes(24)
    assert struct.unpack_from("<q", raw, 128) == (123456789012,)
    assert struct.unpack_from("<ii", raw, 136) == (7, 1)
    assert struct.unpack_from("<5f", raw, 144) == (0.25, 0.5, 0.75, 0.125, 1.5)
    assert raw[164:256] == bytes(92)
    data = np.frombuffer(raw[256:], dtype=np.float32)
    assert np.array_equal(data, np.concatenate([st.weights, st.exp_avg, st.exp_avg_sq]))
    h, d2, back = export.read_dlt(path)
    assert h["header_bytes"] == 256 and (d2.H, d2.W, d2.max_batch) == (16, 720, 2)
    assert (back.step, back.epoch, back.unsupervised, back.lr, back.loss) == (123456789012, 7, 1, 0.25, 1.5)
    with pytest.raises(ValueError, match="not an odometry weight file"):
        export.read_dlw(path)
    with pytest.raises(ValueError, match="truncated|floats after the header"):
        open(path, "ab").write(b"\0\0\0\0")
        export.read_dlt(path)


@pytest.mark.parametrize("act,single", [("tanh", False), ("relu", True)])
def test_torch_adam_state_survives_the_dlt(tmp_path, act, single):
    from delora_b200.deploy import export
    from delora_b200.models.model import OdometryModel
    cfg = _config(act, single)
    model, opt = _trained(cfg)
    ckpt = {"epoch": 4, "model_state_dict": model.state_dict(), "optimizer_state_dict": opt.state_dict(), "loss": 0.5,
            "parameters": cfg}
    path = os.path.join(tmp_path, "s.dlt")
    export.write_dlt(path, _desc(cfg), export.training_state_from_checkpoint(ckpt, cfg))
    _, _, state = export.read_dlt(path)
    assert (state.step, state.epoch, state.unsupervised) == (3, 5, 1)
    back = export.checkpoint_from_training_state(state, cfg)
    assert back["epoch"] == 4 and back["loss"] == 0.5 and back["parameters"] is cfg
    for k, t in model.state_dict().items():
        assert torch.equal(back["model_state_dict"][k], t), k
    want, got = opt.state_dict(), back["optimizer_state_dict"]
    assert list(got["state"]) == list(want["state"])
    for i, s in want["state"].items():
        for name in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(got["state"][i][name], s[name]), (i, name)
        assert float(got["state"][i]["step"]) == float(s["step"]) == 3.0
    g, w = got["param_groups"][0], want["param_groups"][0]
    assert (g["lr"], tuple(g["betas"]), g["eps"]) == (w["lr"], tuple(w["betas"]), w["eps"])
    assert g["params"] == w["params"]
    # torch accepts it, and the loaded optimizer continues exactly as the original one
    model2 = OdometryModel(dict(cfg, device="cpu"))
    model2.load_state_dict(back["model_state_dict"])
    opt2 = torch.optim.Adam(model2.parameters(), lr=1.0)
    opt2.load_state_dict(got)
    gen = torch.Generator().manual_seed(9)
    for p, p2 in zip(model.parameters(), model2.parameters()):
        p.grad = torch.randn(p.shape, generator=gen)
        p2.grad = p.grad.clone()
    opt.step()
    opt2.step()
    for (k, p), p2 in zip(model.named_parameters(), model2.parameters()):
        assert torch.equal(p, p2), k


def _refusal(cfg, ckpt, match):
    from delora_b200.deploy import export
    with pytest.raises(ValueError, match=match):
        export.training_state_from_checkpoint(ckpt, cfg)


def test_refusals_name_the_key():
    cfg = _config()
    for adam, key in (({"weight_decay": 1e-4}, "weight_decay"), ({"amsgrad": True}, "amsgrad"),
                      ({"maximize": True}, "maximize")):
        model, opt = _trained(cfg, steps=1, **adam)
        _refusal(cfg, {"model_state_dict": model.state_dict(), "optimizer_state_dict": opt.state_dict()}, key)
    model, opt = _trained(cfg, steps=2)
    sd = opt.state_dict()
    two = {"state": sd["state"], "param_groups": [dict(sd["param_groups"][0], params=[0]),
                                                  dict(sd["param_groups"][0], params=sd["param_groups"][0]["params"][1:])]}
    _refusal(cfg, {"model_state_dict": model.state_dict(), "optimizer_state_dict": two}, "param_groups")
    for bad_step, what in ((torch.tensor(1.0), "steps differ"), (torch.tensor(2.5), "step")):
        sd = opt.state_dict()
        sd["state"][3] = dict(sd["state"][3], step=bad_step)
        _refusal(cfg, {"model_state_dict": model.state_dict(), "optimizer_state_dict": sd}, what)
    sd = opt.state_dict()
    sd["state"][0] = dict(sd["state"][0], exp_avg=sd["state"][0]["exp_avg"][:1])
    _refusal(cfg, {"model_state_dict": model.state_dict(), "optimizer_state_dict": sd}, r"state\[0\]\.exp_avg")
    bad_model = dict(model.state_dict())
    first = next(iter(bad_model))
    bad_model[first] = bad_model[first][:1]
    _refusal(cfg, {"model_state_dict": bad_model, "optimizer_state_dict": opt.state_dict()}, first)


def test_checkpoint_without_optimizer_state_gives_zero_moments():
    from delora_b200.deploy import export
    cfg = dict(_config(), learning_rate=3e-4)
    model, _ = _trained(cfg, steps=0)
    for ckpt in ({"model_state_dict": model.state_dict()},
                 {"model_state_dict": model.state_dict(), "optimizer_state_dict": torch.optim.Adam(
                     model.parameters(), lr=1e-3).state_dict()}):
        st = export.training_state_from_checkpoint(ckpt, cfg)
        assert st.step == 0 and st.unsupervised == 1 and st.epoch == 0
        assert not st.exp_avg.any() and not st.exp_avg_sq.any()
        assert st.exp_avg.size == st.weights.size
    assert export.training_state_from_checkpoint({"model_state_dict": model.state_dict()}, cfg).lr == 3e-4


def _yaml_config(cdir):
    os.makedirs(cdir)
    with open(os.path.join(cdir, "config_datasets.yaml"), "w") as f:
        f.write("horizontal_field_of_view: [ -179.9, 179.9 ]\n"
                "kitti:\n  vertical_field_of_view: [ -24.5, 2.0 ]\n  vertical_cells: 16\n  horizontal_cells: 720\n")
    with open(os.path.join(cdir, "deployment_options.yaml"), "w") as f:
        f.write('datasets: ["kitti"]\nunsupervised_at_start: False\n')
    with open(os.path.join(cdir, "hyperparameters.yaml"), "w") as f:
        f.write("learning_rate: 0.00001\nuse_dropout: False\nactivation_fct: \"tanh\"\nresnet_outputs: 64\n"
                "pre_feature_extraction: False\nlayers: [ 1, 1, 1, 1 ]\nfactor_fewer_resnet_channels: 1\n"
                "use_single_mlp_at_output: False\n")


def test_init_seed_is_deterministic(tmp_path):
    from delora_b200.deploy import export
    cdir = os.path.join(tmp_path, "config")
    _yaml_config(cdir)
    outs = []
    for seed, name in ((3, "a.dlt"), (3, "b.dlt"), (4, "c.dlt")):
        out = os.path.join(tmp_path, name)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "export_odometry_weights.py"), "--init-seed",
                            str(seed), "--training-state", "--config_dir", cdir, "--n_stride", "4096", "--max_batch", "2",
                            "--out", out], capture_output=True, text=True, cwd=tmp_path)
        assert r.returncode == 0, r.stdout + r.stderr
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1] and outs[0] != outs[2]
    _, d, st = export.read_dlt(os.path.join(tmp_path, "a.dlt"))
    assert (st.step, st.epoch, st.unsupervised) == (0, 0, 0)
    assert st.lr == np.float32(1e-5) and not st.exp_avg.any() and not st.exp_avg_sq.any() and st.weights.any()
    assert (d.H, d.W, d.max_batch, d.n_stride) == (16, 720, 2, 4096)
    # the .pth tool turns it into a checkpoint torch and the model accept
    pth = os.path.join(tmp_path, "a.pth")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "training_state_to_checkpoint.py"), "--dlt",
                        os.path.join(tmp_path, "a.dlt"), "--out", pth, "--config_dir", cdir], capture_output=True,
                       text=True, cwd=tmp_path)
    assert r.returncode == 0, r.stdout + r.stderr
    ckpt = torch.load(pth, weights_only=False)
    assert ckpt["parameters"]["layers"] == [1, 1, 1, 1] and ckpt["epoch"] == -1
    from delora_b200.models.model import OdometryModel
    model = OdometryModel(dict(ckpt["parameters"], device="cpu"))
    model.load_state_dict(ckpt["model_state_dict"])
    torch.optim.Adam(model.parameters()).load_state_dict(ckpt["optimizer_state_dict"])
    # exactly one of --checkpoint / --init-seed
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "export_odometry_weights.py"), "--out", "x.dlt"],
                       capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode != 0 and "--init-seed" in r.stderr


def test_state_entry_points_refuse_without_a_gpu():
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc(_config())
    dp = ctypes.byref(d)
    dummy = ctypes.c_void_p(16)             # never dereferenced: the call is refused before any launch
    assert L.delora_odometry_train_get_state(dp, None, dummy, dummy, dummy, dummy, None) != 0
    assert b"null workspace" in L.delora_last_error()
    for i, name in enumerate((b"weights", b"exp_avg", b"exp_avg_sq", b"step", b"workspace")):
        args = [dummy] * 5
        args[i] = None
        assert L.delora_odometry_train_set_state(dp, *args, None) != 0
        assert b"null " + name in L.delora_last_error(), name
    bad = _desc(_config())
    bad.act = 0
    assert L.delora_odometry_train_set_state(ctypes.byref(bad), dummy, dummy, dummy, dummy, dummy, None) != 0
    assert b"act=0" in L.delora_last_error()
    assert L.delora_odometry_train_get_state(None, dummy, None, None, None, None, None) != 0
    assert b"null descriptor" in L.delora_last_error()


def test_identity_bit_alone_is_refused():
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc(_config())
    hp = _lib.OdometryTrainParams(lr=1e-5, beta1=0.9, beta2=0.999, eps=1e-8, lambda_po2pl=1.0,
                                  loss_flags=_lib.LOSS_IDENTITY_FIT, nb_h=7, nb_w=11, epsilon_range=0.5,
                                  min_neighbors=10)
    dummy = ctypes.c_void_p(16)
    rc = L.delora_odometry_train_step(ctypes.byref(d), ctypes.byref(hp), dummy, dummy, 1, dummy, None, None, None, None,
                                      None)
    assert rc != 0
    assert b"loss_flags=0x200 sets no loss bit" in L.delora_last_error()


def test_train_example_compiles_against_the_header(tmp_path):
    from delora_b200 import build
    nvcc = build._nvcc()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    r = subprocess.run([nvcc, "-c", os.path.join(ROOT, "examples", "odometry_train.c"), "-I",
                        os.path.join(ROOT, "include"), "-I", cuda_inc, "-Xcompiler", "-Wall,-Werror", "-o",
                        os.path.join(tmp_path, "odometry_train.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
