"""-m "not gpu": the adapting streams entry points of the C ABI (delora_odometry_streams_adapt_* and
delora_odometry_streams_push_adapt) without a device -- the exported symbols, the header in C, the workspace sizes the
header documents and their formula, every refusal before any launch, the Python class's refusals, and that
examples/odometry_streams.c builds with its documented cc line and refuses a malformed --adapt."""
import ctypes
import os
import shutil
import subprocess

import pytest

import odometry_harness as H
from delora_b200 import ops
from helpers import ROOT

NAME = "delora_odometry_streams_push_adapt"
SYMBOLS = ("delora_odometry_streams_adapt_workspace_bytes", "delora_odometry_streams_adapt_init",
           "delora_odometry_streams_push_adapt", "delora_odometry_streams_adapt_reset")


def _align(n):
    return (n + 255) // 256 * 256


def _desc(h=64, w=720, S=2, w_pre=0, n_stride=1000):
    return H.desc(H.config(h, w, device="cpu"), n_stride, S, w_pre)


def _hp(flags=ops.LOSS_PO2PL | ops.LOSS_PL2PL, lr=1e-5):
    from delora_b200 import _lib
    return _lib.OdometryTrainParams(lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, lambda_po2pl=1.0, loss_flags=flags,
                                    nb_h=7, nb_w=11, epsilon_range=0.5, min_neighbors=10)


def test_symbols_are_exported():
    from delora_b200 import build
    lib = ctypes.CDLL(build.LIB)
    for name in SYMBOLS:
        assert hasattr(lib, name), name


def test_header_compiles_as_c(tmp_path):
    from delora_b200 import build
    src = os.path.join(tmp_path, "use.c")
    with open(src, "w") as f:
        f.write('#include "delora_b200.h"\n'
                "int use(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const float* w,\n"
                "        void* ws, const float* p, const int32_t* n, const int32_t* a, float* T, int32_t* valid,\n"
                "        float* losses, const int32_t* mask) {\n"
                "    if (delora_odometry_streams_adapt_workspace_bytes(d) < 0) return 1;\n"
                "    if (delora_odometry_streams_adapt_init(d, w, ws, 0)) return 1;\n"
                "    if (delora_odometry_streams_push_adapt(d, hp, 1, p, n, a, ws, T, valid, losses, 0)) return 1;\n"
                "    return delora_odometry_streams_adapt_reset(d, mask, ws, 0);\n"
                "}\n"
                "_Static_assert(sizeof(delora_odometry_desc) == 80, \"desc\");\n"
                "_Static_assert(sizeof(delora_odometry_file_header) == 128, \"header\");\n"
                "_Static_assert(sizeof(delora_odometry_train_file_header) == 256, \"train header\");\n"
                "_Static_assert(sizeof(delora_odometry_train_params) == 40, \"params\");\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n")
    r = subprocess.run([build._nvcc(), "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


# The header's table: (H, W, w_pre, S) -> MiB of the training and the adapting streams workspaces
HEADER_TABLE = {(64, 720, 0, 1): (325.2, 327.3), (64, 720, 0, 4): (521.3, 529.8), (64, 720, 0, 16): (1305.9, 1339.7),
                (64, 720, 2250, 1): (341.0, 345.4), (64, 720, 2250, 4): (584.4, 602.0),
                (64, 720, 2250, 16): (1558.3, 1628.7), (64, 2048, 0, 1): (425.5, 431.5),
                (64, 2048, 0, 4): (922.5, 946.5), (64, 2048, 0, 16): (2910.6, 3006.6)}


@pytest.mark.parametrize("h,w,w_pre,S", sorted(HEADER_TABLE))
def test_sizes_are_the_ones_the_header_documents(h, w, w_pre, S):
    from delora_b200 import _lib
    L = _lib.lib()
    dp = ctypes.byref(_desc(h, w, S, w_pre, 131072))
    got = (L.delora_odometry_train_workspace_bytes(dp), L.delora_odometry_streams_adapt_workspace_bytes(dp))
    mib = HEADER_TABLE[(h, w, w_pre, S)]
    assert tuple(round(b / 2 ** 20, 1) for b in got) == mib
    with open(os.path.join(ROOT, "include", "delora_b200.h")) as f:
        header = f.read()
    assert f"S = {S} {mib[0]} -> {mib[1]} MiB" in header


@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("h,w,w_pre", [(64, 720, 0), (64, 720, 2250), (16, 180, 360), (16, 259, 100), (16, 180, 0)])
def test_workspace_is_the_training_layout_plus_the_stream_section(h, w, w_pre, S):
    """w_pre = 0: the cached H x W image and grids; w_pre > 0: the cached H x w_pre grids; then has_prev [S] and the
    count of valid pairs, each 256-byte aligned, after the training workspace (whose offsets do not move)."""
    from delora_b200 import _lib
    L = _lib.lib()
    dp = ctypes.byref(_desc(h, w, S, w_pre))
    train = L.delora_odometry_train_workspace_bytes(dp)
    got = L.delora_odometry_streams_adapt_workspace_bytes(dp)
    if w_pre == 0:
        cache = [S * 4 * h * w * 4, S * h * w * 16, S * h * w * 16]
    else:
        cache = [S * h * w_pre * 16, S * h * w_pre * 16]
    want = train + sum(_align(n) for n in cache + [S * 4, 4])
    assert train > 0 and got == want
    assert L.delora_odometry_train_grad_offset(dp) > 0          # the training layout is the prefix


def test_invalid_descriptors_are_refused_by_name():
    from delora_b200 import _lib
    L = _lib.lib()
    d = _desc()
    d.act = 0
    dp = ctypes.byref(d)
    assert L.delora_odometry_streams_adapt_workspace_bytes(dp) == -1
    assert b"delora_odometry_streams_adapt_workspace_bytes: act=0" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_init(dp, 16, 32, None) != 0
    assert b"delora_odometry_streams_adapt_init: act=0" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_reset(dp, 16, 32, None) != 0
    assert b"delora_odometry_streams_adapt_reset: act=0" in L.delora_last_error()
    rc, err = _push(desc=d)
    assert rc != 0 and f"{NAME}: act=0".encode() in err, err
    d = _desc(w_pre=1)
    assert L.delora_odometry_streams_adapt_workspace_bytes(ctypes.byref(d)) == -1
    assert b"w_pre=1" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_workspace_bytes(None) == -1
    assert b"null descriptor" in L.delora_last_error()


def test_reset_refuses_null_pointers_by_name():
    from delora_b200 import _lib
    L = _lib.lib()
    dp = ctypes.byref(_desc())
    assert L.delora_odometry_streams_adapt_reset(dp, None, 32, None) != 0
    assert b"delora_odometry_streams_adapt_reset: null mask" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_reset(dp, 16, None, None) != 0
    assert b"delora_odometry_streams_adapt_reset: null workspace" in L.delora_last_error()


def _push(hp=None, update=1, desc=None, **null):
    """delora_odometry_streams_push_adapt with non-null dummies except where null names a pointer; a null stream, so a
    call that got past its checks would launch (nothing here does)."""
    from delora_b200 import _lib
    L = _lib.lib()
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80, "losses": 96}
    args.update(null)
    rc = L.delora_odometry_streams_push_adapt(ctypes.byref(desc or _desc()),
                                              None if hp is False else ctypes.byref(hp or _hp()), update,
                                              args["points"], args["n_points"], None, args["workspace"], args["T"],
                                              args["valid"], args["losses"], None)
    return rc, L.delora_last_error()


@pytest.mark.parametrize("missing", ["points", "n_points", "workspace", "T", "valid", "losses"])
def test_push_refuses_null_pointers_by_name(missing):
    rc, err = _push(**{missing: None})
    assert rc != 0 and f"{NAME}: null {missing}".encode() in err, err


@pytest.mark.parametrize("update", [-1, 2, 7])
def test_push_refuses_update_by_name(update):
    rc, err = _push(update=update)
    assert rc != 0 and f"{NAME}: update={update} must be 0 or 1".encode() in err, err


@pytest.mark.parametrize("flag,what", [(ops.LOSS_IDENTITY_FIT, b"DELORA_LOSS_IDENTITY_FIT"),
                                       (ops.TRAIN_DROPOUT, b"DELORA_TRAIN_DROPOUT")])
def test_push_refuses_identity_fit_and_dropout_by_name(flag, what):
    rc, err = _push(hp=_hp(ops.LOSS_PO2PL | flag))
    assert rc != 0 and NAME.encode() in err and what in err and b"loss_flags=" in err, err


def test_push_refuses_what_the_training_step_refuses():
    rc, err = _push(hp=False)
    assert rc != 0 and f"{NAME}: null hyperparameters".encode() in err, err
    for field, value in (("lr", -1.0), ("beta1", 1.0), ("eps", 0.0), ("nb_h", 6), ("min_neighbors", -1),
                         ("lambda_po2pl", float("nan"))):
        hp = _hp()
        setattr(hp, field, value)
        rc, err = _push(hp=hp)
        assert rc != 0 and f"{NAME}: {field}=".encode() in err, (field, err)
    rc, err = _push(hp=_hp(ops.NORMAL_LINEAR))
    assert rc != 0 and b"sets no loss bit" in err, err
    # normalization_scaling needs the recipe's w_pre
    rc, err = _push(hp=_hp(ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING))
    assert rc != 0 and f"{NAME}: DELORA_TRAIN_NORMALIZATION_SCALING needs w_pre > 0".encode() in err, err


def test_python_class_refuses_dropout_and_unrecipe_normalization():
    from delora_b200.deploy.stream import AdaptiveOdometryStreams
    cfg = H.config(64, 720, device="cpu")
    cfg["use_dropout"] = True
    with pytest.raises(ValueError, match="use_dropout"):
        AdaptiveOdometryStreams(None, cfg, "kitti", 2, 1000, 1e-5)
    cfg["use_dropout"] = False
    cfg["normalization_scaling"] = True
    with pytest.raises(ValueError, match="preprocessing_normals"):
        AdaptiveOdometryStreams(None, cfg, "kitti", 2, 1000, 1e-5)


def _build_with_cc_line(tmp_path):
    """The Build line in the example's header: plain cc, cudart only."""
    from delora_b200 import build
    cc = shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler named cc")
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(build._nvcc())))
    libdir = os.path.dirname(build.LIB)
    exe = str(tmp_path / "odometry_streams")
    r = subprocess.run([cc, os.path.join(ROOT, "examples", "odometry_streams.c"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(cuda, "include"), "-L", libdir, "-ldelora_b200", "-L",
                        os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + libdir, "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return exe


def test_example_builds_with_its_cc_line_and_refuses_a_malformed_adapt(tmp_path):
    exe = _build_with_cc_line(tmp_path)
    missing = str(tmp_path / "missing.dlw")
    for lr in ("abc", "-1", "1e-5x", "", "nan", "inf"):
        r = subprocess.run([exe, "--adapt", lr, "--adapt-out", str(tmp_path / "o.dlw"), missing, "d"],
                           capture_output=True, text=True, timeout=60)
        assert r.returncode != 0 and "--adapt: LR must be a finite number >= 0" in r.stderr, (lr, r.stderr)
    r = subprocess.run([exe, "--adapt", "1e-5", missing, "d"], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "go together" in r.stderr, r.stderr
    r = subprocess.run([exe, "--adapt-out", "o.dlw", missing, "d"], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "go together" in r.stderr, r.stderr
    r = subprocess.run([exe, "--adapt", "1e-5", "--adapt-out", "o.dlw", "--residual", missing, "d"],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "drop --residual" in r.stderr, r.stderr
    # a well-formed option gets as far as the weight file
    r = subprocess.run([exe, "--adapt", "1e-5", "--adapt-out", "o.dlw", missing, "d"], capture_output=True, text=True,
                       timeout=60)
    assert r.returncode != 0 and "cannot open the weight file" in r.stderr, r.stderr
