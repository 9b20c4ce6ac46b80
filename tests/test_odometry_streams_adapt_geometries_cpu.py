"""-m "not gpu": the adapting streams of several sensor geometries (delora_odometry_streams_adapt_geometries_* and
delora_odometry_streams_push_adapt_geometries) without a device -- the exported symbols and the ABI version, the
workspace size against the sections the existing size queries imply, every refusal before any launch naming the index
and the field, and examples/odometry_streams.c's --geometry argument errors."""
import ctypes
import os
import shutil
import subprocess

import pytest

import odometry_harness as H
from delora_b200 import ops
from helpers import ROOT

NAME = "delora_odometry_streams_push_adapt_geometries"
SYMBOLS = ("delora_odometry_streams_adapt_geometries_workspace_bytes", "delora_odometry_streams_adapt_geometries_init",
           "delora_odometry_streams_push_adapt_geometries", "delora_odometry_streams_adapt_geometries_reset")


def _lib():
    from delora_b200 import _lib
    return _lib, _lib.lib()


def _arr(descs):
    _l, _ = _lib()
    return (_l.OdometryDesc * len(descs))(*descs)


def _pair(S0=2, S1=3, w0=(64, 180, 360), w1=(64, 128, 128)):
    return [H.streams_desc(w0[0], w0[1], S0, w0[2]), H.streams_desc(w1[0], w1[1], S1, w1[2])]


def _bytes(descs, n=None):
    _, L = _lib()
    return L.delora_odometry_streams_adapt_geometries_workspace_bytes(_arr(descs), len(descs) if n is None else n)


def test_symbols_are_exported_and_the_abi_stays():
    from delora_b200 import build
    lib = ctypes.CDLL(build.LIB)
    for name in SYMBOLS:
        assert hasattr(lib, name), name
    assert lib.delora_abi_version() == 3


def test_header_compiles_as_c(tmp_path):
    from delora_b200 import build
    src = os.path.join(tmp_path, "use.c")
    with open(src, "w") as f:
        f.write('#include "delora_b200.h"\n'
                "int use(const delora_odometry_desc* d, const delora_odometry_train_params* hp, const float* w,\n"
                "        void* ws, const float* const* p, const int32_t* const* n, const int32_t* a, float* T,\n"
                "        int32_t* valid, float* losses) {\n"
                "    if (delora_odometry_streams_adapt_geometries_workspace_bytes(d, 2) < 0) return 1;\n"
                "    if (delora_odometry_streams_adapt_geometries_init(d, 2, w, ws, 0)) return 1;\n"
                "    if (delora_odometry_streams_adapt_geometries_reset(d, 2, a, ws, 0)) return 1;\n"
                "    return delora_odometry_streams_push_adapt_geometries(d, 2, hp, 1, p, n, a, ws, T, valid, losses,\n"
                "                                                         0);\n"
                "}\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n")
    r = subprocess.run([build._nvcc(), "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.parametrize("h,w,w_pre,S", [(64, 720, 0, 1), (64, 720, 2250, 3), (16, 180, 360, 2), (64, 512, 512, 16)])
def test_one_geometry_is_the_adapting_workspace(h, w, w_pre, S):
    _, L = _lib()
    d = H.streams_desc(h, w, S, w_pre)
    assert _bytes([d]) == L.delora_odometry_streams_adapt_workspace_bytes(ctypes.byref(d)) > 0


@pytest.mark.parametrize("S0,S1", [(1, 1), (2, 3), (4, 4), (16, 1)])
@pytest.mark.parametrize("g1", [(64, 512, 512), (64, 128, 0), (16, 180, 360)])
def test_two_geometries_add_the_second_ones_sections(S0, S1, g1):
    _, L = _lib()
    d0, d1 = _pair(S0, S1, (64, 720, 2250), g1)
    ref = lambda f, d: int(getattr(L, f)(ctypes.byref(d)))        # noqa: E731
    adapt0 = ref("delora_odometry_streams_adapt_workspace_bytes", d0)
    train1 = ref("delora_odometry_train_workspace_bytes", d1)
    stream1 = ref("delora_odometry_streams_adapt_workspace_bytes", d1) - train1
    # d[1]'s geometry section: its training workspace after the model section (the fp32 weights, gradient, m and v,
    # the 256-byte counter slot and the bf16 filters), which the weight and trunk size queries give
    slice_ = H.align(4 * ref("delora_odometry_weight_floats", d1))
    model = 4 * slice_ + 256 + int(L.delora_trunk_weight_bytes((ctypes.c_int * 4)(*d1.layers), d1.W))
    assert int(L.delora_odometry_train_grad_offset(ctypes.byref(d1))) == slice_
    fleet = 256                             # the fleet count and geometry 1's counters, one aligned block
    assert _bytes([d0, d1]) == adapt0 + (train1 - model) + stream1 + slice_ + fleet
    assert stream1 > 0 and train1 - model > 0


def test_sizes_grow_with_each_geometry():
    d0, d1 = _pair()
    d2 = H.streams_desc(16, 180, 1, 0)
    two, three = _bytes([d0, d1]), _bytes([d0, d1, d2])
    assert three > two > _bytes([d0])


def _push(descs=None, n=None, hp=None, update=1, points=(16, 16), n_points=(32, 32), **null):
    """delora_odometry_streams_push_adapt_geometries with non-null dummies except where null names a pointer."""
    _, L = _lib()
    descs = _pair() if descs is None else descs
    n = len(descs) if n is None else n
    args = {"workspace": 48, "T": 64, "valid": 80, "losses": 96}
    args.update(null)
    pts = None if points is None else (ctypes.c_void_p * len(points))(*points)
    cnt = None if n_points is None else (ctypes.c_void_p * len(n_points))(*n_points)
    rc = L.delora_odometry_streams_push_adapt_geometries(
        _arr(descs) if descs else None, n, None if hp is False else ctypes.byref(hp or H.train_params()), update, pts,
        cnt, None, args["workspace"], args["T"], args["valid"], args["losses"], None)
    return rc, L.delora_last_error()


def test_set_refusals_name_the_index_and_field():
    _, L = _lib()
    d0, d1 = _pair()
    cases = []
    e = _pair()[1]
    e.act = 1
    cases.append(([d0, e], b"d[1].act=1 differs from d[0].act=2"))
    e = _pair()[1]
    e.layers[2] = 3
    cases.append(([d0, e], b"d[1].layers[2]=3 differs from d[0].layers[2]=2"))
    e = _pair()[1]
    e.resnet_outputs = 500
    cases.append(([d0, e], b"d[1].resnet_outputs=500 differs"))
    e = _pair()[1]
    e.single_mlp = 1
    cases.append(([d0, e], b"d[1].single_mlp=1 differs"))
    e = H.streams_desc(64, 131, 2, 0)
    cases.append(([d0, e], b"d[1].W=131 and d[0].W=180 differ in parity"))
    e = _pair()[1]
    e.max_batch = 0
    cases.append(([d0, e], b"d[1]: max_batch=0"))
    e = _pair()[1]
    e.w_pre = 1
    cases.append(([d0, e], b"d[1]: w_pre=1"))
    for descs, msg in cases:
        assert _bytes(descs) == -1
        assert msg in L.delora_last_error(), (msg, L.delora_last_error())
        rc, err = _push(descs)
        assert rc != 0 and NAME.encode() in err and msg in err, err
        assert L.delora_odometry_streams_adapt_geometries_init(_arr(descs), 2, 16, 32, None) != 0
        assert msg in L.delora_last_error()
        assert L.delora_odometry_streams_adapt_geometries_reset(_arr(descs), 2, 16, 32, None) != 0
        assert msg in L.delora_last_error()


@pytest.mark.parametrize("n,msg", [(0, b"n=0 must be >= 1"), (17, b"n=17 must be <= 16"), (-3, b"n=-3 must be >= 1")])
def test_n_is_refused(n, msg):
    _, L = _lib()
    assert L.delora_odometry_streams_adapt_geometries_workspace_bytes(_arr(_pair()), n) == -1
    assert msg in L.delora_last_error()
    rc, err = _push(n=n)
    assert rc != 0 and msg in err, err
    assert L.delora_odometry_streams_adapt_geometries_workspace_bytes(None, 2) == -1
    assert b"null descriptor" in L.delora_last_error()


@pytest.mark.parametrize("missing", ["workspace", "T", "valid", "losses"])
def test_push_refuses_null_pointers_by_name(missing):
    rc, err = _push(**{missing: None})
    assert rc != 0 and f"{NAME}: null {missing}".encode() in err, err


def test_push_refuses_null_arrays_and_entries_by_index():
    rc, err = _push(points=None)
    assert rc != 0 and f"{NAME}: null points".encode() in err, err
    rc, err = _push(n_points=None)
    assert rc != 0 and f"{NAME}: null n_points".encode() in err, err
    rc, err = _push(points=(16, None))
    assert rc != 0 and f"{NAME}: points[1] is null".encode() in err, err
    rc, err = _push(n_points=(None, 32))
    assert rc != 0 and f"{NAME}: n_points[0] is null".encode() in err, err


@pytest.mark.parametrize("update", [-1, 2])
def test_push_refuses_update(update):
    rc, err = _push(update=update)
    assert rc != 0 and f"{NAME}: update={update} must be 0 or 1".encode() in err, err


@pytest.mark.parametrize("flag,what", [(ops.LOSS_IDENTITY_FIT, b"DELORA_LOSS_IDENTITY_FIT"),
                                       (ops.TRAIN_DROPOUT, b"DELORA_TRAIN_DROPOUT")])
def test_push_refuses_identity_fit_and_dropout(flag, what):
    rc, err = _push(hp=H.train_params(ops.LOSS_PO2PL | flag))
    assert rc != 0 and NAME.encode() in err and what in err and b"loss_flags=" in err, err


def test_push_refuses_bad_params_and_mixed_w_pre_with_scaling():
    rc, err = _push(hp=False)
    assert rc != 0 and f"{NAME}: null hyperparameters".encode() in err, err
    hp = H.train_params()
    hp.eps = 0.0
    rc, err = _push(hp=hp)
    assert rc != 0 and f"{NAME}: eps=".encode() in err, err
    scaling = H.train_params(ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING)
    rc, err = _push(_pair(w1=(64, 128, 0)), hp=scaling)
    assert rc != 0 and f"{NAME}: d[1]: DELORA_TRAIN_NORMALIZATION_SCALING needs w_pre > 0".encode() in err, err
    assert b"got w_pre=0" in err
    rc, err = _push(_pair(w0=(64, 180, 0)), hp=scaling)
    assert rc != 0 and f"{NAME}: d[0]: DELORA_TRAIN_NORMALIZATION_SCALING".encode() in err, err


def test_init_and_reset_refuse_null_pointers():
    _, L = _lib()
    assert L.delora_odometry_streams_adapt_geometries_init(_arr(_pair()), 2, None, 32, None) != 0
    assert b"delora_odometry_streams_adapt_geometries_init: null pointer" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_geometries_reset(_arr(_pair()), 2, None, 32, None) != 0
    assert b"delora_odometry_streams_adapt_geometries_reset: null mask" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_geometries_reset(_arr(_pair()), 2, 16, None, None) != 0
    assert b"delora_odometry_streams_adapt_geometries_reset: null workspace" in L.delora_last_error()


def test_example_refuses_geometry_misuse(tmp_path):
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
    adapt = ["--adapt", "1e-5", "--adapt-out", str(tmp_path / "o.dlw")]
    geom = ["--geometry", "dir,64,512,-24.5,2"]

    def run(args):
        return subprocess.run([exe] + args + [missing, "d"], capture_output=True, text=True, timeout=60)

    r = run(geom)
    assert r.returncode != 0 and "--geometry adapts one model from several sensors: it needs --adapt" in r.stderr
    r = run(adapt + ["--gpus", "1"] + geom)
    assert r.returncode != 0 and "--geometry serves every sensor on one GPU" in r.stderr, r.stderr
    for bad in ("dir", "dir,64", "dir,64,512,-24.5", "dir,64,512,2,-24.5", "dir,0,512,-24.5,2", "dir,64,1,-24.5,2",
                "dir,64,512,-24.5,2,x", "dir,64,512,-24.5,2,-1", ",64,512,-24.5,2", "dir,64,512,-24.5,2,8,9"):
        r = run(adapt + ["--geometry", bad])
        assert r.returncode != 0 and "--geometry wants DIR,H,W,VFOV0,VFOV1[,W_PRE]" in r.stderr, (bad, r.stderr)
    # well-formed options get as far as the weight file
    r = run(adapt + geom + ["--geometry", "other,32,256,-15,15,512"])
    assert r.returncode != 0 and "cannot open the weight file" in r.stderr, r.stderr
