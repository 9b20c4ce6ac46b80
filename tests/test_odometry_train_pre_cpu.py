"""-m "not gpu": the descriptor's w_pre field (normals at the preprocessing width for training through the C ABI).
Its place in the struct and in the .dlw header, its validation by the training size query, and the workspace sizes it
changes (training only) and does not change (inference and streams)."""
import ctypes
import struct

import pytest

import odometry_harness as H


def _cfg(h=64, w=720, w_pre=2250):
    cfg = H.config(h, w, device="cpu")
    cfg["kitti"]["horizontal_cells_preprocessing"] = w_pre
    return cfg


def _a256(n):
    return (n + 255) // 256 * 256


def _pre_growth(h, w, w_pre, max_batch):
    """What w_pre adds to the training workspace (include/delora_b200.h): the depth keys of the 2 * max_batch scans grow
    to max(W, w_pre) columns, and four H x w_pre buffers per scan follow the other sections: the image (4 fp32
    channels), the index map (int32) and the two float4 grids."""
    s, hwp = 2 * max_batch, h * w_pre
    keys = _a256(s * h * max(w, w_pre) * 8) - _a256(s * h * w * 8)
    return keys + _a256(s * 4 * hwp * 4) + _a256(s * hwp * 4) + 2 * _a256(s * hwp * 16)


def test_struct_size_and_offset():
    from delora_b200 import _lib
    assert ctypes.sizeof(_lib.OdometryDesc) == 80
    assert _lib.OdometryDesc.w_pre.offset == 76                 # header byte 16 + 76 = 92
    assert _lib.OdometryDesc.single_mlp.offset == 72


def test_header_byte_92_round_trip(tmp_path):
    import numpy as np
    from delora_b200.deploy import export
    d = export.desc_from_config(_cfg(), "kitti", 4096, 2, preprocessing_normals=True)
    assert d.w_pre == 2250
    blob = np.arange(5, dtype=np.float32)
    path = str(tmp_path / "pre.dlw")
    export.write_dlw(path, d, blob)
    raw = open(path, "rb").read()
    assert struct.unpack_from("<i", raw, 92)[0] == 2250
    h, d2, blob2 = export.read_dlw(path)
    assert h["w_pre"] == 2250 and d2.w_pre == 2250 and np.array_equal(blob2, blob)
    assert bytes(d2) == bytes(d)


def test_default_export_is_unchanged_and_reads_back_as_zero(tmp_path):
    """Without the option the header is byte for byte the one written before the field existed (zeros at 92..95)."""
    import numpy as np
    from delora_b200 import _lib
    from delora_b200.deploy import export
    d = export.desc_from_config(_cfg(), "kitti", 4096, 2)
    assert d.w_pre == 0
    blob = np.arange(5, dtype=np.float32)
    path = str(tmp_path / "plain.dlw")
    export.write_dlw(path, d, blob)
    raw = open(path, "rb").read()
    old = struct.Struct("<8sii" + "ii4d" + "iii4iii4x" + "q" + "24x")      # the layout with 4 pad bytes at 92
    want = old.pack(export.MAGIC, _lib.ABI_VERSION, 128, d.H, d.W, d.hfov0, d.hfov1, d.vfov0, d.vfov1, d.n_stride,
                    d.max_batch, d.act, *list(d.layers), d.resnet_outputs, d.single_mlp, blob.size)
    assert raw[:128] == want
    assert export.read_dlw(path)[1].w_pre == 0


@pytest.mark.parametrize("w_pre", [1, -1, -2250, (1 << 27) // 64])
def test_bad_w_pre_is_refused_by_name(w_pre):
    from delora_b200 import _lib
    L = _lib.lib()
    d = H.desc(_cfg(), 131072, 1, w_pre)
    assert L.delora_odometry_train_workspace_bytes(ctypes.byref(d)) == -1
    assert b"w_pre" in L.delora_last_error()


@pytest.mark.parametrize("w_pre", [1, -7, 2250, 1 << 30])
def test_inference_and_streams_ignore_w_pre(w_pre):
    from delora_b200 import _lib
    L = _lib.lib()
    d = H.desc(_cfg(), 131072, 4)
    want = (L.delora_odometry_workspace_bytes(ctypes.byref(d)), L.delora_odometry_streams_workspace_bytes(ctypes.byref(d)),
            L.delora_odometry_weight_floats(ctypes.byref(d)))
    d.w_pre = w_pre
    got = (L.delora_odometry_workspace_bytes(ctypes.byref(d)), L.delora_odometry_streams_workspace_bytes(ctypes.byref(d)),
           L.delora_odometry_weight_floats(ctypes.byref(d)))
    assert got == want and min(got) > 0


# 64 x 720, layers (2, 2, 2, 2), 1000 outputs, two heads, n_stride 131072: the sizes the documents quote
DOCUMENTED = {1: (340982528, 357525248), 4: (546658048, 612828928), 16: (1369363456, 1634046976)}


@pytest.mark.parametrize("h,w,w_pre,max_batch", [(64, 720, 2250, 1), (64, 720, 2250, 4), (64, 720, 2250, 16),
                                                 (16, 259, 512, 2), (64, 2048, 2048, 1), (64, 2048, 1024, 4)])
def test_training_workspace_grows_by_the_documented_section(h, w, w_pre, max_batch):
    from delora_b200 import _lib
    L = _lib.lib()
    d = H.desc(_cfg(h, w, w_pre), 131072, max_batch)
    base = L.delora_odometry_train_workspace_bytes(ctypes.byref(d))
    d.w_pre = w_pre
    grown = L.delora_odometry_train_workspace_bytes(ctypes.byref(d))
    assert base > 0 and grown - base == _pre_growth(h, w, w_pre, max_batch)
    if (h, w, w_pre) == (64, 720, 2250):
        assert (base, grown) == DOCUMENTED[max_batch]
