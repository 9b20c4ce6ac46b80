"""-m "not gpu": one training workspace shared by several sensor geometries (delora_odometry_train_geometries_* and
delora_odometry_train_use_geometry) without a device -- the shared size against the single-geometry sizes, the model
section's gradient offset across a set, every refusal naming its index and field, and the --geometry option of
examples/odometry_train.c refusing malformed values before it touches a file or the GPU."""
import ctypes
import subprocess

import pytest

import odometry_harness as H

DUMMY = 16                              # never dereferenced: the calls are refused before any launch
KITTI, DARPA = (-24.5, 2.0), (-22.5, 22.5)


@pytest.fixture(scope="module")
def example(tmp_path_factory):
    """examples/odometry_train.c linked against the built library (the refusals below need no GPU)."""
    return H.build_example("odometry_train", str(tmp_path_factory.mktemp("example")), link=True)


def _lib():
    from delora_b200 import _lib
    return _lib, _lib.lib()


def _desc(h, w, vfov=KITTI, w_pre=0, max_batch=16, stride=131072, layers=(2, 2, 2, 2), nout=1000, single=False,
          act="tanh"):
    return H.desc(H.config(h, w, act, single, layers, nout, vfov=vfov, device="cpu"), stride, max_batch, w_pre)


def _arr(descs):
    _l, _ = _lib()
    return (_l.OdometryDesc * len(descs))(*descs)


def _single_bytes(d):
    _, L = _lib()
    return int(L.delora_odometry_train_workspace_bytes(ctypes.byref(d)))


SETS = {
    "kitti_2048+kitti_720_w2250": [_desc(64, 2048), _desc(64, 720, w_pre=2250)],
    "kitti_720_w2250+darpa_512": [_desc(64, 720, w_pre=2250), _desc(64, 512, DARPA, w_pre=512)],
    "three_batches_and_strides": [_desc(16, 180, max_batch=4, stride=4096), _desc(64, 512, DARPA, max_batch=1),
                                  _desc(32, 1024, max_batch=8, stride=65536, w_pre=1800)],
    "odd_widths": [_desc(64, 723, layers=(1, 2, 1, 1), nout=64, single=True),
                   _desc(16, 179, layers=(1, 2, 1, 1), nout=64, single=True, max_batch=2)],
    "one": [_desc(64, 720, w_pre=2250, act="relu")],
}


@pytest.mark.parametrize("name", list(SETS))
def test_shared_size_is_the_largest_single_size(name):
    _, L = _lib()
    descs = SETS[name]
    singles = [_single_bytes(d) for d in descs]
    assert min(singles) > 0
    assert L.delora_odometry_train_geometries_workspace_bytes(_arr(descs), len(descs)) == max(singles)
    # the order of the set does not matter
    assert L.delora_odometry_train_geometries_workspace_bytes(_arr(descs[::-1]), len(descs)) == max(singles)


@pytest.mark.parametrize("name", list(SETS))
def test_gradient_offset_is_the_same_on_every_geometry_of_a_set(name):
    _, L = _lib()
    offsets = {int(L.delora_odometry_train_grad_offset(ctypes.byref(d))) for d in SETS[name]}
    assert len(offsets) == 1 and min(offsets) > 0


def _edit(i, **kw):
    descs = [_desc(64, 2048), _desc(64, 720, w_pre=2250), _desc(16, 180, max_batch=2)]
    for k, v in kw.items():
        if isinstance(v, tuple):                      # (index, value) of an array field
            getattr(descs[i], k)[v[0]] = v[1]
        else:
            setattr(descs[i], k, v)
    return descs


@pytest.mark.parametrize("descs,message", [
    (lambda: _edit(1, w_pre=1), b"d[1]: w_pre=1 must be 0 or >= 2"),
    (lambda: _edit(2, max_batch=0), b"d[2]: max_batch=0 must be in"),
    (lambda: _edit(0, W=721), b"d[0]: W=721"),
    (lambda: _edit(2, act=1), b"d[2].act=1 differs from d[0].act=2"),
    (lambda: _edit(1, layers=(2, 3)), b"d[1].layers[2]=3 differs from d[0].layers[2]=2"),
    (lambda: _edit(2, resnet_outputs=999), b"d[2].resnet_outputs=999 differs from d[0].resnet_outputs=1000"),
    (lambda: _edit(1, single_mlp=1), b"d[1].single_mlp=1 differs from d[0].single_mlp=0"),
    (lambda: _edit(2, W=179), b"d[2].W=179 and d[0].W=2048 differ in parity"),
])
def test_refusals_name_the_index_and_the_field(descs, message):
    _, L = _lib()
    arr = _arr(descs())
    assert L.delora_odometry_train_geometries_workspace_bytes(arr, len(arr)) == -1
    assert message in L.delora_last_error(), L.delora_last_error()
    assert L.delora_odometry_train_geometries_init(arr, len(arr), DUMMY, DUMMY, None) != 0
    assert message in L.delora_last_error(), L.delora_last_error()
    assert L.delora_odometry_train_use_geometry(arr, len(arr), 0, DUMMY, None) != 0
    assert message in L.delora_last_error(), L.delora_last_error()


def test_parity_refusal_says_why():
    _, L = _lib()
    arr = _arr(_edit(1, W=723))
    assert L.delora_odometry_train_geometries_workspace_bytes(arr, 3) == -1
    assert b"the model section, would differ" in L.delora_last_error()


def test_set_and_argument_refusals():
    _, L = _lib()
    arr = _arr(_edit(0))
    for n in (0, -1):
        assert L.delora_odometry_train_geometries_workspace_bytes(arr, n) == -1
        assert f"n={n} must be >= 1".encode() in L.delora_last_error()
    assert L.delora_odometry_train_geometries_workspace_bytes(None, 2) == -1
    assert b"null descriptor array" in L.delora_last_error()
    for g in (3, -1):
        assert L.delora_odometry_train_use_geometry(arr, 3, g, DUMMY, None) != 0
        assert f"delora_odometry_train_use_geometry: g={g} outside [0, n=3)".encode() in L.delora_last_error()
    assert L.delora_odometry_train_use_geometry(arr, 3, 1, None, None) != 0
    assert b"null workspace" in L.delora_last_error()
    assert L.delora_odometry_train_geometries_init(arr, 3, None, DUMMY, None) != 0
    assert b"delora_odometry_train_geometries_init: null pointer" in L.delora_last_error()
    assert L.delora_odometry_train_geometries_init(arr, 3, DUMMY, None, None) != 0
    assert b"null pointer" in L.delora_last_error()


@pytest.mark.parametrize("value", ["d,64,720", "d,64,720,-24.5", "d,64,720,-24.5,2,2250,7", ",64,720,-24.5,2",
                                   "nodir", "d,64.5,720,-24.5,2", "d,0,720,-24.5,2", "d,64,1,-24.5,2",
                                   "d,64,720,2,-24.5", "d,64,720,-24.5,2x", "d,64,720,nan,2", "d,64,720,-24.5,inf",
                                   "d,64,720,-24.5,2,-1", "d,64,720,-24.5,2,1.5", "d,,720,-24.5,2", "d,64,720,,2"])
def test_train_example_refuses_malformed_geometries(example, tmp_path, value):
    exe = example
    # the input file does not exist: the option is refused before anything is read
    r = subprocess.run([exe, "--geometry", value, str(tmp_path / "missing.dlt"), str(tmp_path / "out.dlt"), "1", "1",
                        "a.bin", "b.bin"], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0
    assert "--geometry wants DIR,H,W,VFOV0,VFOV1[,W_PRE]" in r.stderr, r.stderr


def test_train_example_accepts_well_formed_geometries(example, tmp_path):
    exe = example
    for value in ("d,64,720,-24.5,2", "d,64,512,-22.5,22.5,512", "some/dir,16,180,-15,15,0"):
        r = subprocess.run([exe, "--geometry", value, "--geometry", value, str(tmp_path / "missing.dlt"),
                            str(tmp_path / "out.dlt"), "1", "1", "a.bin", "b.bin"], capture_output=True, text=True,
                           timeout=60)
        assert r.returncode != 0 and "cannot open the input file" in r.stderr, r.stderr
    r = subprocess.run([exe, "--gpus", "2", "--geometry", "d,64,720,-24.5,2", "in.dlt", "out.dlt", "1", "1", "a.bin",
                        "b.bin"], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "does not combine with --gpus" in r.stderr, r.stderr


def test_train_example_links_with_its_documented_build_line(tmp_path):
    """The Build line in the example's header (plain cc: cudart and pthread, no libm), not nvcc, whose driver adds
    libraries of its own."""
    import os
    import shutil
    from delora_b200 import build
    cc = shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler named cc")
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(build._nvcc())))
    libdir = os.path.dirname(build.LIB)
    r = subprocess.run([cc, os.path.join(H.ROOT, "examples", "odometry_train.c"), "-I", os.path.join(H.ROOT, "include"),
                        "-I", os.path.join(cuda, "include"), "-L", libdir, "-ldelora_b200", "-L",
                        os.path.join(cuda, "lib64"), "-lcudart", "-lpthread", "-Wl,-rpath," + libdir, "-o",
                        str(tmp_path / "odometry_train")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
