"""-m "not gpu": the adapting streams on several workspaces (delora_odometry_streams_adapt_group_* and
delora_odometry_streams_push_adapt_group) without a device -- the exported symbols, the header in C, the group
workspace size against the adapting-streams size, every refusal before any launch (the update value, the group's
fields, null pointers, the identity fit, dropout), and that examples/odometry_streams.c builds with its cc line and
refuses --gpus without --adapt."""
import ctypes
import os
import shutil
import subprocess

import pytest

import odometry_harness as H
from delora_b200 import ops
from helpers import ROOT

NAME = "delora_odometry_streams_push_adapt_group"
SYMBOLS = ("delora_odometry_streams_adapt_group_workspace_bytes", "delora_odometry_streams_adapt_group_init",
           "delora_odometry_streams_push_adapt_group")
DUMMY = 16                              # never dereferenced: the calls are refused before any launch
GROUP_SECTION = 256                     # tick counter, fleet-wide count and the exchange slots, one aligned block


def _lib():
    from delora_b200 import _lib
    return _lib, _lib.lib()


def _desc(h=64, w=720, S=2, w_pre=0, n_stride=1000):
    return H.desc(H.config(h, w, device="cpu"), n_stride, S, w_pre)


def _hp(flags=ops.LOSS_PO2PL | ops.LOSS_PL2PL, lr=1e-5):
    _l, _ = _lib()
    return _l.OdometryTrainParams(lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, lambda_po2pl=1.0, loss_flags=flags,
                                  nb_h=7, nb_w=11, epsilon_range=0.5, min_neighbors=10)


def _group(world=2, rank=0, ws=48):
    _l, _ = _lib()
    g = _l.OdometryTrainGroup(rank=rank, world=world, multicast=0, n_ctas=8, n_threads=128, status=DUMMY,
                              side_stream=None, join_event=DUMMY)
    for q in range(min(world, _l.GRAD_ALLREDUCE_MAX_WORLD)):
        g.peer_ws[q] = ws if q == rank else 4096 * (q + 1)
        g.peer_flags[q] = 8192 * (q + 1)
    for k in range(_l.TRAIN_GROUP_BUCKETS):
        g.fork_events[k] = DUMMY
    return g


def _edit(**kw):
    g = _group()
    for k, v in kw.items():
        if isinstance(v, tuple):                  # (index, value) of an array field
            getattr(g, k)[v[0]] = v[1]
        else:
            setattr(g, k, v)
    return g


def _push(g=None, hp=None, update=1, desc=None, **null):
    """delora_odometry_streams_push_adapt_group with non-null dummies except where null names a pointer."""
    _, L = _lib()
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80, "losses": 96}
    args.update(null)
    g = _group() if g is None else g
    rc = L.delora_odometry_streams_push_adapt_group(ctypes.byref(desc or _desc()),
                                                    None if hp is False else ctypes.byref(hp or _hp()),
                                                    None if g is False else ctypes.byref(g), update, args["points"],
                                                    args["n_points"], None, args["workspace"], args["T"],
                                                    args["valid"], args["losses"], None)
    return rc, L.delora_last_error()


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
                "int use(const delora_odometry_desc* d, const delora_odometry_train_params* hp,\n"
                "        const delora_odometry_train_group* g, const float* w, void* ws, const float* p,\n"
                "        const int32_t* n, const int32_t* a, float* T, int32_t* valid, float* losses) {\n"
                "    if (delora_odometry_streams_adapt_group_workspace_bytes(d) < 0) return 1;\n"
                "    if (delora_odometry_streams_adapt_group_init(d, w, ws, 0)) return 1;\n"
                "    return delora_odometry_streams_push_adapt_group(d, hp, g, 1, p, n, a, ws, T, valid, losses, 0);\n"
                "}\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n")
    r = subprocess.run([build._nvcc(), "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


# the shapes of test_odometry_streams_adapt_cpu.py's layout test, and the header's table's
@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("h,w,w_pre", [(64, 720, 0), (64, 720, 2250), (16, 180, 360), (16, 259, 100), (16, 180, 0)])
def test_group_workspace_is_the_adapting_layout_plus_the_group_section(h, w, w_pre, S):
    _, L = _lib()
    dp = ctypes.byref(_desc(h, w, S, w_pre))
    adapt = L.delora_odometry_streams_adapt_workspace_bytes(dp)
    train = L.delora_odometry_train_workspace_bytes(dp)
    assert adapt > train > 0
    assert L.delora_odometry_streams_adapt_group_workspace_bytes(dp) == adapt + GROUP_SECTION


@pytest.mark.parametrize("h,w,w_pre,S,mib", [(64, 720, 0, 1, 327.3), (64, 720, 2250, 16, 1628.7),
                                             (64, 2048, 0, 16, 3006.6)])
def test_the_adapting_size_is_unchanged(h, w, w_pre, S, mib):
    _, L = _lib()
    dp = ctypes.byref(_desc(h, w, S, w_pre, 131072))
    assert round(L.delora_odometry_streams_adapt_workspace_bytes(dp) / 2 ** 20, 1) == mib


def test_invalid_descriptors_are_refused_by_name():
    _, L = _lib()
    d = _desc()
    d.act = 0
    dp = ctypes.byref(d)
    assert L.delora_odometry_streams_adapt_group_workspace_bytes(dp) == -1
    assert b"delora_odometry_streams_adapt_group_workspace_bytes: act=0" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_group_init(dp, 16, 32, None) != 0
    assert b"delora_odometry_streams_adapt_group_init: act=0" in L.delora_last_error()
    rc, err = _push(desc=d)
    assert rc != 0 and f"{NAME}: act=0".encode() in err, err
    assert L.delora_odometry_streams_adapt_group_workspace_bytes(None) == -1
    assert b"null descriptor" in L.delora_last_error()


def test_init_refuses_null_pointers():
    _, L = _lib()
    assert L.delora_odometry_streams_adapt_group_init(ctypes.byref(_desc()), None, 32, None) != 0
    assert b"delora_odometry_streams_adapt_group_init: null pointer" in L.delora_last_error()


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
    hp = _hp()
    hp.eps = 0.0
    rc, err = _push(hp=hp)
    assert rc != 0 and f"{NAME}: eps=".encode() in err, err
    rc, err = _push(hp=_hp(ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING))
    assert rc != 0 and f"{NAME}: DELORA_TRAIN_NORMALIZATION_SCALING needs w_pre > 0".encode() in err, err


@pytest.mark.parametrize("group,message", [
    (lambda: False, b"null group"),
    (lambda: _edit(world=0), b"world=0 must be in [1, 16]"),
    (lambda: _edit(world=17), b"world=17 must be in [1, 16]"),
    (lambda: _edit(rank=2), b"rank=2 outside [0, world=2)"),
    (lambda: _edit(peer_ws=(1, 0)), b"peer_ws[1] is null"),
    (lambda: _edit(peer_ws=(1, 4096 + 8)), b"peer_ws[1] is null or not 16-byte aligned"),
    (lambda: _edit(peer_ws=(0, 4096)), b"peer_ws[rank=0] is not the workspace"),
    (lambda: _edit(peer_flags=(0, 0)), b"peer_flags[0] is null"),
    (lambda: _edit(peer_flags=(1, 8194)), b"peer_flags[1] is null or not 4-byte aligned"),
    (lambda: _edit(multicast=4104), b"multicast is not 16-byte aligned"),
    (lambda: _edit(status=None), b"null status"),
    (lambda: _edit(n_ctas=0), b"n_ctas=0 outside [1, 160]"),
    (lambda: _edit(n_threads=48), b"n_threads=48 must be 32, 64, 96 or 128"),
    (lambda: _edit(fork_events=(3, None)), b"null fork_events[3]"),
    (lambda: _edit(join_event=None), b"null join_event"),
])
@pytest.mark.parametrize("update", [0, 1])
def test_group_refusals_name_the_field(group, message, update):
    rc, err = _push(g=group(), update=update)
    assert rc != 0 and NAME.encode() in err and message in err, err


def test_push_refusals_come_before_the_group_check():
    rc, err = _push(g=False, update=3)
    assert rc != 0 and f"{NAME}: update=3".encode() in err, err


def test_single_rank_group_needs_no_events():
    g = _group(world=1)
    g.join_event = None
    g.fork_events[0] = None
    rc, err = _push(g=g, T=None)                    # refused for T, not for the events
    assert rc != 0 and f"{NAME}: null T".encode() in err, err


def test_example_builds_with_its_cc_line_and_refuses_gpus_without_adapt(tmp_path):
    from delora_b200 import build
    cc = shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler named cc")
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(build._nvcc())))
    libdir = os.path.dirname(build.LIB)
    exe = str(tmp_path / "odometry_streams")
    r = subprocess.run([cc, os.path.join(ROOT, "examples", "odometry_streams.c"), "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(cuda, "include"), "-L", libdir, "-ldelora_b200", "-L",
                        os.path.join(cuda, "lib64"), "-lcudart", "-lpthread", "-Wl,-rpath," + libdir, "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    missing = str(tmp_path / "missing.dlw")
    for extra in (["--gpus", "2"], ["--gpus", "1", "--residual"]):
        r = subprocess.run([exe] + extra + [missing, "d"], capture_output=True, text=True, timeout=60)
        assert r.returncode != 0 and "--gpus adapts one model on several GPUs: it needs --adapt" in r.stderr, r.stderr
    adapt = ["--adapt", "1e-5", "--adapt-out", str(tmp_path / "o.dlw")]
    for n in ("0", "17", "x", "2x", ""):
        r = subprocess.run([exe] + adapt + ["--gpus", n, missing, "d"], capture_output=True, text=True, timeout=60)
        assert r.returncode != 0 and "--gpus must be in [1, 16]" in r.stderr, (n, r.stderr)
    # a well-formed option gets as far as the weight file
    r = subprocess.run([exe, "--gpus", "2"] + adapt + [missing, "d"], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "cannot open the weight file" in r.stderr, r.stderr
