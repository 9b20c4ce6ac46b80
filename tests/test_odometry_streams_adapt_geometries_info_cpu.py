"""-m "not gpu": the information form of the adapting streams of several sensor geometries
(delora_odometry_streams_adapt_geometries_info_workspace_bytes and delora_odometry_streams_push_adapt_geometries_info)
without a device -- the exported symbols and the ABI version, the workspace size against the _adapt_geometries size plus
the information section, every refusal before any launch naming the field, and examples/odometry_streams.c accepting
--information with --geometry."""
import ctypes
import os
import shutil
import subprocess

import pytest

import odometry_harness as H
from delora_b200 import ops
from helpers import ROOT

NAME = "delora_odometry_streams_push_adapt_geometries_info"
SIZE = "delora_odometry_streams_adapt_geometries_info_workspace_bytes"


def _lib():
    from delora_b200 import _lib
    return _lib, _lib.lib()


def _arr(descs):
    _l, _ = _lib()
    return (_l.OdometryDesc * len(descs))(*descs)


def _pair(S0=2, S1=3, w0=(64, 180, 360), w1=(64, 128, 128)):
    return [H.streams_desc(w0[0], w0[1], S0, w0[2]), H.streams_desc(w1[0], w1[1], S1, w1[2])]


def test_symbols_are_exported_and_the_abi_stays():
    from delora_b200 import build
    lib = ctypes.CDLL(build.LIB)
    for name in (SIZE, NAME):
        assert hasattr(lib, name), name
    assert lib.delora_abi_version() == 3


def test_header_compiles_as_c(tmp_path):
    from delora_b200 import build
    src = os.path.join(tmp_path, "use.c")
    with open(src, "w") as f:
        f.write('#include "delora_b200.h"\n'
                "int use(const delora_odometry_desc* d, const delora_odometry_train_params* hp, void* ws,\n"
                "        const float* const* p, const int32_t* const* n, const int32_t* a, float* T, int32_t* valid,\n"
                "        float* losses, float* info) {\n"
                "    if (delora_odometry_streams_adapt_geometries_info_workspace_bytes(d, 2) < 0) return 1;\n"
                "    return delora_odometry_streams_push_adapt_geometries_info(d, 2, hp, 1, p, n, a, ws, T, valid,\n"
                "                                                              losses, info, 0);\n"
                "}\n"
                "_Static_assert(DELORA_B200_ABI_VERSION == 3, \"abi\");\n"
                "_Static_assert(sizeof(delora_odometry_desc) == 80, \"desc\");\n")
    r = subprocess.run([build._nvcc(), "-c", src, "-I", os.path.join(ROOT, "include"), "-o",
                        os.path.join(tmp_path, "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def _want(descs):
    """The _adapt_geometries size, then the rows of every stream and the largest geometry's info_scratch, aligned."""
    _, L = _lib()
    base = int(L.delora_odometry_streams_adapt_geometries_workspace_bytes(_arr(descs), len(descs)))
    rows = sum(int(d.max_batch) for d in descs) * ops.INFO_ROW * 4
    scratch = max(int(L.delora_icp_information_scratch_floats(d.max_batch, d.H, d.W)) for d in descs) * 4
    assert base > 0 and scratch > 0
    return base + H.align(rows) + H.align(scratch)


@pytest.mark.parametrize("descs", [
    [H.streams_desc(64, 720, 1, 0)],
    [H.streams_desc(64, 720, 3, 2250)],
    _pair(),
    _pair(1, 16, (64, 720, 2250), (64, 512, 512)),
    _pair(16, 1, (64, 720, 2250), (64, 512, 512)),
    _pair(4, 4, (16, 180, 360), (64, 128, 0)),
    _pair(2, 3) + [H.streams_desc(16, 180, 5, 0)],
    [H.streams_desc(16, 180, 1, 0), H.streams_desc(64, 2048, 2, 0), H.streams_desc(64, 512, 7, 512)],
], ids=["n1", "n1-pre", "n2", "n2-1-16", "n2-16-1", "n2-mixed-pre", "n3", "n3-largest-in-the-middle"])
def test_size_is_the_geometries_workspace_plus_the_information_section(descs):
    _, L = _lib()
    assert L.delora_odometry_streams_adapt_geometries_info_workspace_bytes(_arr(descs), len(descs)) == _want(descs)


def test_one_geometry_has_the_adapt_info_section():
    # n = 1: the rows and scratch of _adapt_info's information section, after _adapt's layout instead of the group one
    _, L = _lib()
    d = H.streams_desc(64, 720, 4, 2250)
    info = int(L.delora_odometry_streams_adapt_info_workspace_bytes(ctypes.byref(d)))
    group = int(L.delora_odometry_streams_adapt_group_workspace_bytes(ctypes.byref(d)))
    adapt = int(L.delora_odometry_streams_adapt_workspace_bytes(ctypes.byref(d)))
    assert L.delora_odometry_streams_adapt_geometries_info_workspace_bytes(_arr([d]), 1) == adapt + (info - group)


def _refused_sets():
    d0 = _pair()[0]
    cases = []
    e = _pair()[1]
    e.act = 1
    cases.append(([d0, e], 2, b"d[1].act=1 differs from d[0].act=2"))
    e = _pair()[1]
    e.layers[2] = 3
    cases.append(([d0, e], 2, b"d[1].layers[2]=3 differs from d[0].layers[2]=2"))
    e = _pair()[1]
    e.resnet_outputs = 500
    cases.append(([d0, e], 2, b"d[1].resnet_outputs=500 differs"))
    e = _pair()[1]
    e.single_mlp = 1
    cases.append(([d0, e], 2, b"d[1].single_mlp=1 differs"))
    cases.append(([d0, H.streams_desc(64, 131, 2, 0)], 2, b"d[1].W=131 and d[0].W=180 differ in parity"))
    e = _pair()[1]
    e.max_batch = 0
    cases.append(([d0, e], 2, b"d[1]: max_batch=0"))
    e = _pair()[1]
    e.w_pre = 1
    cases.append(([d0, e], 2, b"d[1]: w_pre=1"))
    cases.append((_pair(), 0, b"n=0 must be >= 1"))
    cases.append((_pair(), 17, b"n=17 must be <= 16"))
    cases.append((_pair(), -3, b"n=-3 must be >= 1"))
    return cases


@pytest.mark.parametrize("descs,n,msg", _refused_sets())
def test_size_refuses_what_adapt_geometries_refuses(descs, n, msg):
    _, L = _lib()
    assert L.delora_odometry_streams_adapt_geometries_workspace_bytes(_arr(descs), n) == -1
    plain = L.delora_last_error().split(b": ", 1)[1]
    assert msg in plain
    assert L.delora_odometry_streams_adapt_geometries_info_workspace_bytes(_arr(descs), n) == -1
    err = L.delora_last_error()
    assert err.startswith(SIZE.encode()) and err.split(b": ", 1)[1] == plain, (err, plain)
    assert L.delora_odometry_streams_adapt_geometries_info_workspace_bytes(None, 2) == -1
    assert b"null descriptor" in L.delora_last_error()


def _push(descs=None, n=None, hp=None, update=1, points=(16, 16), n_points=(32, 32), **null):
    """delora_odometry_streams_push_adapt_geometries_info with non-null dummies except where null names a pointer."""
    _, L = _lib()
    descs = _pair() if descs is None else descs
    n = len(descs) if n is None else n
    args = {"workspace": 48, "T": 64, "valid": 80, "losses": 96, "info": 112}
    args.update(null)
    pts = None if points is None else (ctypes.c_void_p * len(points))(*points)
    cnt = None if n_points is None else (ctypes.c_void_p * len(n_points))(*n_points)
    rc = L.delora_odometry_streams_push_adapt_geometries_info(
        _arr(descs) if descs else None, n, None if hp is False else ctypes.byref(hp or H.train_params()), update, pts,
        cnt, None, args["workspace"], args["T"], args["valid"], args["losses"], args["info"], None)
    return rc, L.delora_last_error()


@pytest.mark.parametrize("descs,n,msg", _refused_sets())
def test_push_refuses_the_geometries_sets(descs, n, msg):
    rc, err = _push(descs, n)
    assert rc != 0 and NAME.encode() in err and msg in err, err


@pytest.mark.parametrize("missing", ["workspace", "T", "valid", "losses", "info"])
def test_push_refuses_null_pointers_by_name(missing):
    rc, err = _push(**{missing: None})
    assert rc != 0 and f"{NAME}: null {missing}".encode() in err, err


def test_push_refuses_the_other_arguments_of_push_adapt_geometries():
    rc, err = _push(points=None)
    assert rc != 0 and f"{NAME}: null points".encode() in err, err
    rc, err = _push(n_points=(None, 32))
    assert rc != 0 and f"{NAME}: n_points[0] is null".encode() in err, err
    rc, err = _push(update=2)
    assert rc != 0 and f"{NAME}: update=2 must be 0 or 1".encode() in err, err
    rc, err = _push(hp=False)
    assert rc != 0 and f"{NAME}: null hyperparameters".encode() in err, err
    rc, err = _push(hp=H.train_params(ops.LOSS_PO2PL | ops.TRAIN_DROPOUT))
    assert rc != 0 and b"DELORA_TRAIN_DROPOUT" in err, err
    scaling = H.train_params(ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING)
    rc, err = _push(_pair(w1=(64, 128, 0)), hp=scaling)
    assert rc != 0 and f"{NAME}: d[1]: DELORA_TRAIN_NORMALIZATION_SCALING needs w_pre > 0".encode() in err, err


def test_example_accepts_information_with_geometry(tmp_path):
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

    # well-formed options get as far as the weight file, in either order
    for args in (adapt + geom + ["--information"], ["--information"] + geom + adapt):
        r = run(args)
        assert r.returncode != 0 and "cannot open the weight file" in r.stderr, (args, r.stderr)
    r = run(adapt + ["--gpus", "1", "--information"] + geom)
    assert r.returncode != 0 and "--geometry serves every sensor on one GPU" in r.stderr, r.stderr
    r = run(geom + ["--information"])
    assert r.returncode != 0 and "--geometry adapts one model from several sensors: it needs --adapt" in r.stderr
