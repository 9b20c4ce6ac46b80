"""-m "not gpu": the ICP scratch layout (icp_layout in csrc/icp_common.cuh).  The buffer is opaque to its caller, who
allocates what delora_icp_scratch_floats returns, so its size is pinned here; the dense operator refuses a grid whose
range pyramid does not fit its section; and the constants ops.py restates match the header."""
import os
import re

import pytest

from helpers import ROOT

BATCHES = [1, 2, 3, 4, 8, 16]
STRIDES = [1, 31, 32, 33, 16 * 180, 64 * 720, 64 * 2047, 64 * 2048, 64 * 2250]


@pytest.fixture(scope="module")
def lib():
    from delora_b200 import _lib, build
    build.build()
    return _lib.lib()


def _expected_floats(b, s):
    # partial rows, column sums, finalize counters, range pyramid, row extents, extents + work-list counters, items and
    # item_done per warp, entries and results per source point
    r = (s + 31) // 32
    return (b * r * 40 + b * 40 + b + 2 + 2 * b * (s // 16 + 4096) + 4 * b * s + b + 8 + 5 * b * r + 160 * b * r)


@pytest.mark.parametrize("s", STRIDES)
@pytest.mark.parametrize("b", BATCHES)
def test_scratch_floats_are_pinned(b, s, lib):
    assert lib.delora_icp_scratch_floats(b, s) == _expected_floats(b, s)
    assert lib.delora_icp_partial_rows(s) == (s + 31) // 32


def test_dense_rejects_a_grid_whose_pyramid_does_not_fit(lib):
    # H = 30000, W = 1: ceil(H / 4) * ceil(W / 16) = 7500 blocks of 4 x 16 cells, room for 30000 // 16 + 4096 = 5971
    p = 256                                             # placeholder device pointers: the call must not reach them
    rc = lib.delora_icp_dense_fwd_bwd(p, p, p, p, p, 1, 30000, 1, -3.14, 3.14, -0.4, 0.1, 1.0, 6, p, p, p, None)
    assert rc == 1
    assert b"range-pyramid" in lib.delora_last_error()


def test_ops_constants_match_the_header():
    from delora_b200 import ops
    text = open(os.path.join(ROOT, "include", "delora_b200.h")).read()
    defines = {k: int(v) for k, v in re.findall(r"#define DELORA_(\w+)\s+(\d+)u?\b", text)}
    for name in ("LOSS_PO2PO", "LOSS_PO2PL", "LOSS_PL2PL", "NORMAL_LINEAR", "ICP_STATS", "LOSS_IDENTITY_FIT", "LOSS_ROW",
                 "ICP_PARTIAL"):
        assert getattr(ops, name) == defines[name], name
