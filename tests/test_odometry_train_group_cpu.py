"""-m "not gpu": the data-parallel training step of the C ABI (delora_odometry_train_step_group) without a device --
every refusal names its field, the ctypes struct against the header's layout, the bucket table of the all-reduce
schedule, the gradient section's offset, and that examples/odometry_train.c compiles."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H

DUMMY = 16                              # never dereferenced: the calls are refused before any launch


def _lib():
    from delora_b200 import _lib
    return _lib, _lib.lib()


def _params():
    from delora_b200.deploy import capi
    return capi.train_params(H.config(64, 720, device="cpu"), 1e-5)


def _group(world=2, rank=0, ws=DUMMY):
    _l, _ = _lib()
    g = _l.OdometryTrainGroup(rank=rank, world=world, multicast=0, n_ctas=8, n_threads=128, status=DUMMY,
                              side_stream=None, join_event=DUMMY)
    for q in range(min(world, _l.GRAD_ALLREDUCE_MAX_WORLD)):
        g.peer_ws[q] = ws if q == rank else 4096 * (q + 1)
        g.peer_flags[q] = 8192 * (q + 1)
    for k in range(_l.TRAIN_GROUP_BUCKETS):
        g.fork_events[k] = DUMMY
    return g


def _step(g, B=1, ws=DUMMY, hp=None):
    _, L = _lib()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 2)
    hp = _params() if hp is None else hp
    return L.delora_odometry_train_step_group(ctypes.byref(d), ctypes.byref(hp), None if g is None else ctypes.byref(g),
                                              DUMMY, DUMMY, B, ws, None, None, None, None, None)


def _edit(**kw):
    g = _group()
    for k, v in kw.items():
        if isinstance(v, tuple):                  # (index, value) of an array field
            getattr(g, k)[v[0]] = v[1]
        else:
            setattr(g, k, v)
    return g


@pytest.mark.parametrize("group,message", [
    (lambda: None, b"null group"),
    (lambda: _edit(world=0), b"world=0 must be in [1, 16]"),
    (lambda: _edit(world=17), b"world=17 must be in [1, 16]"),
    (lambda: _edit(rank=2), b"rank=2 outside [0, world=2)"),
    (lambda: _edit(rank=-1), b"rank=-1 outside"),
    (lambda: _edit(peer_ws=(1, 0)), b"peer_ws[1] is null"),
    (lambda: _edit(peer_ws=(1, 4096 + 8)), b"peer_ws[1] is null or not 16-byte aligned"),
    (lambda: _edit(peer_ws=(0, 4096)), b"peer_ws[rank=0] is not the workspace"),
    (lambda: _edit(peer_flags=(0, 0)), b"peer_flags[0] is null"),
    (lambda: _edit(peer_flags=(1, 8194)), b"peer_flags[1] is null or not 4-byte aligned"),
    (lambda: _edit(multicast=4104), b"multicast is not 16-byte aligned"),
    (lambda: _edit(status=None), b"null status"),
    (lambda: _edit(n_ctas=0), b"n_ctas=0 outside [1, 160]"),
    (lambda: _edit(n_ctas=161), b"n_ctas=161 outside [1, 160]"),
    (lambda: _edit(n_threads=48), b"n_threads=48 must be 32, 64, 96 or 128"),
    (lambda: _edit(n_threads=256), b"n_threads=256"),
    (lambda: _edit(fork_events=(3, None)), b"null fork_events[3]"),
    (lambda: _edit(join_event=None), b"null join_event"),
])
def test_group_refusals_name_the_field(group, message):
    _, L = _lib()
    assert _step(group()) != 0
    assert message in L.delora_last_error(), L.delora_last_error()


def test_single_rank_group_needs_no_streams_or_events_and_keeps_the_step_refusals():
    _, L = _lib()
    g = _group(world=1)
    g.join_event = None
    g.fork_events[0] = None
    assert _step(g, B=3) != 0                     # refused for B, not for the events
    assert b"delora_odometry_train_step_group: B=3 outside [1, max_batch=2]" in L.delora_last_error()
    hp = _params()
    hp.eps = 0.0
    assert _step(g, hp=hp) != 0
    assert b"eps=" in L.delora_last_error()
    assert _step(g, ws=None) != 0
    assert b"null pointer" in L.delora_last_error()


def test_struct_layout_matches_the_header(tmp_path):
    from delora_b200 import build
    _l, _ = _lib()
    fields = [name for name, _ in _l.OdometryTrainGroup._fields_]
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"delora_b200.h\"\nint main(void) {\n"
                   "    printf(\"%zu\\n\", sizeof(delora_odometry_train_group));\n" +
                   "".join(f"    printf(\"%zu\\n\", offsetof(delora_odometry_train_group, {f}));\n" for f in fields) +
                   "    printf(\"%d %d\\n\", DELORA_GRAD_ALLREDUCE_MAX_WORLD, DELORA_TRAIN_GROUP_BUCKETS);\n"
                   "    return 0;\n}\n")
    nvcc = build._nvcc()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    exe = str(tmp_path / "layout")
    r = subprocess.run([nvcc, str(src), "-I", os.path.join(H.ROOT, "include"), "-I", cuda_inc, "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")
    assert int(out[0]) == ctypes.sizeof(_l.OdometryTrainGroup)
    for i, f in enumerate(fields):
        assert int(out[1 + i]) == getattr(_l.OdometryTrainGroup, f).offset, f
    assert out[1 + len(fields)].split() == [str(_l.GRAD_ALLREDUCE_MAX_WORLD), str(_l.TRAIN_GROUP_BUCKETS)]


def _stage_starts(cfg):
    """Float offsets in the blob (state_dict order) where layer2, layer3, layer4 and resnet.fc start, and its length."""
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(0)
    sd = OdometryModel(dict(cfg, device="cpu")).state_dict()
    starts, off = {}, 0
    for name, t in sd.items():
        for part in ("resnet.layer2", "resnet.layer3", "resnet.layer4", "resnet.fc"):
            if name.startswith(part + ".") and part not in starts:
                starts[part] = off
        off += t.numel()
    return [starts["resnet.layer2"], starts["resnet.layer3"], starts["resnet.layer4"], starts["resnet.fc"]], off


@pytest.mark.parametrize("layers,nout,single", [((2, 2, 2, 2), 1000, False), ((1, 1, 1, 1), 64, False),
                                                ((1, 2, 1, 3), 1002, False), ((2, 2, 2, 2), 1002, True),
                                                ((3, 1, 2, 1), 7, True)])
def test_bucket_table_covers_the_blob_in_production_order(layers, nout, single):
    _l, L = _lib()
    cfg = H.config(16, 720, "tanh", single, layers, nout, device="cpu")
    d = H.desc(cfg, 1000, 2)
    n = int(L.delora_odometry_weight_floats(ctypes.byref(d)))
    starts, total = _stage_starts(cfg)
    assert total == n
    K = _l.TRAIN_GROUP_BUCKETS
    off, cnt = (ctypes.c_int64 * K)(), (ctypes.c_int64 * K)()
    assert L.delora_odometry_train_group_buckets(ctypes.byref(d), off, cnt) == 0
    off, cnt = list(off), list(cnt)
    up4 = [-(-x // 4) * 4 for x in [0] + starts + [n]]         # stem, layer2, layer3, layer4, fc, end
    # launch order = production order: heads + fc, layer4, layer3, layer2, stem + layer1
    assert [(o, o + c) for o, c in zip(off, cnt)] == [(up4[4 - k], up4[5 - k]) for k in range(K)]
    assert all(o % 4 == 0 and c % 4 == 0 and c > 0 for o, c in zip(off, cnt))
    covered = np.zeros(up4[-1], dtype=np.int32)
    for o, c in zip(off, cnt):
        covered[o:o + c] += 1
    assert (covered == 1).all() and up4[-1] - n < 4                 # [0, blob) once, at most 3 floats of padding
    # no bucket reaches into a section produced after it (the sections before it in the blob)
    for k in range(K):
        assert off[k] >= ([0] + starts)[4 - k]
    if nout % 4 == 2:
        assert (starts[3] + 513 * nout) % 4 == 2                    # the heads start at 2 mod 4: inside a float4
    assert L.delora_odometry_train_group_buckets(ctypes.byref(d), None, (ctypes.c_int64 * K)()) != 0
    assert b"null pointer" in L.delora_last_error()


@pytest.mark.parametrize("max_batch,w_pre", [(1, 0), (4, 0), (2, 1440)])
def test_gradient_offset_follows_the_master_weights(max_batch, w_pre):
    _, L = _lib()
    d = H.desc(H.config(64, 720, device="cpu"), 4096, max_batch, w_pre)
    n = int(L.delora_odometry_weight_floats(ctypes.byref(d)))
    # the workspace opens with the master weights, then the gradient, each 256-byte aligned
    assert L.delora_odometry_train_grad_offset(ctypes.byref(d)) == (n * 4 + 255) // 256 * 256
    bad = H.desc(H.config(64, 720, device="cpu"), 4096, 1, w_pre=1)
    assert L.delora_odometry_train_grad_offset(ctypes.byref(bad)) == -1
    assert b"w_pre=1" in L.delora_last_error()


def test_train_example_compiles_against_the_header(tmp_path):
    H.build_example("odometry_train", tmp_path, link=False)
