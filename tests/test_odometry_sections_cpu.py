"""-m "not gpu": the section map of every odometry workspace kind (delora_odometry_workspace_sections) on a grid of
descriptors and geometry lists.  The pinned sizes (test_odometry_layout_cpu.py) cannot see two sections that overlap,
and the GPU tests that compare one kind with another cannot see an overlap both kinds share; this checks the layouts
themselves:
  - the sections of a kind are pairwise disjoint (the DELORA_WS_SHARED model section counted once; the training
    geometries' geometry sections share their bytes by design, so there each geometry is checked on its own);
  - every section starts on a 256-byte boundary (DELORA_WS_SUBRANGE ones lie inside an aligned allocation);
  - every section is non-empty and lies inside the kind's *_workspace_bytes;
  - a kind built by appending to another has the other's sections at the same offsets (STREAMS in RESIDUAL in INFO,
    TRAIN in ADAPT in ADAPT_GROUP in ADAPT_INFO, ADAPT_GEOMETRIES in ADAPT_GEOMETRIES_INFO);
  - in the geometries kinds the shared weight (and, training, Adam) sections are at the same offsets in every geometry.
The layouts take no normalisation input (DELORA_TRAIN_NORMALIZATION_SCALING is a per-call loss bit), so the grid
covers normalised models by construction."""
import itertools

import pytest

import odometry_harness as H
from delora_b200 import _lib

KINDS = _lib.WS_KINDS
GEOMETRY_KINDS = ("train_geometries", "adapt_geometries", "adapt_geometries_info")
PRE_KINDS = ("streams_pre", "streams_pre_info")

# kind -> its size query (the geometries kinds take (d, n))
BYTES = {
    "pairs": "delora_odometry_workspace_bytes",
    "streams": "delora_odometry_streams_workspace_bytes",
    "streams_residual": "delora_odometry_streams_residual_workspace_bytes",
    "streams_info": "delora_odometry_streams_info_workspace_bytes",
    "streams_normalized": "delora_odometry_streams_normalized_workspace_bytes",
    "streams_pre": "delora_odometry_streams_pre_workspace_bytes",
    "streams_pre_info": "delora_odometry_streams_pre_info_workspace_bytes",
    "train": "delora_odometry_train_workspace_bytes",
    "train_geometries": "delora_odometry_train_geometries_workspace_bytes",
    "adapt": "delora_odometry_streams_adapt_workspace_bytes",
    "adapt_group": "delora_odometry_streams_adapt_group_workspace_bytes",
    "adapt_info": "delora_odometry_streams_adapt_info_workspace_bytes",
    "adapt_geometries": "delora_odometry_streams_adapt_geometries_workspace_bytes",
    "adapt_geometries_info": "delora_odometry_streams_adapt_geometries_info_workspace_bytes",
}
# smaller kind -> the kind that appends to it
APPENDED = [("streams", "streams_residual"), ("streams_residual", "streams_info"), ("train", "adapt"),
            ("adapt", "adapt_group"), ("adapt_group", "adapt_info"), ("adapt_geometries", "adapt_geometries_info")]

SHAPES = ((16, 180), (16, 259), (64, 720), (64, 2048))


def _desc(h, w, w_pre=0, S=1, single=False, nout=1000):
    return H.desc(H.config(h, w, single=single, nout=nout, device="cpu"), 1000, S, w_pre)


def _grid():
    """Every descriptor of the grid: shape x w_pre x max_batch x heads x resnet_outputs."""
    return [(_desc(h, w, w_pre, S, single, nout), f"{h}x{w}/pre{w_pre}/S{S}/single{int(single)}/out{nout}")
            for (h, w), w_pre, S, single, nout in itertools.product(SHAPES, (0, 360, 2250), (1, 3, 16), (False, True),
                                                                    (1000, 1002))]


# mixed geometries, each list of one W parity (a shared model section needs it); (H, W, w_pre, S)
_EVEN = [(16, 180, 0, 1), (64, 720, 2250, 3), (16, 260, 360, 2), (64, 2048, 0, 1), (64, 512, 512, 16),
         (16, 180, 360, 3), (64, 720, 0, 2), (16, 2048, 2250, 1)]
_ODD = [(16, 259, 0, 1), (64, 2047, 360, 3), (16, 259, 2250, 2)]


def _geometry_lists():
    out = []
    for single, nout in ((False, 1000), (True, 1002)):
        def mk(specs):
            return [_desc(h, w, p, S, single, nout) for h, w, p, S in specs]
        tag = f"single{int(single)}/out{nout}"
        out.append((mk(_EVEN[:1]), f"n1/{tag}"))
        out.append((mk(_EVEN[:2]), f"n2/{tag}"))
        out.append((mk(_ODD[:3]), f"n3-odd/{tag}"))
        out.append((mk([_EVEN[(3 * g) % len(_EVEN)] for g in range(16)]), f"n16/{tag}"))
    return out


def _cases(kind):
    """(descriptor list, label) of every case of kind"""
    if kind in GEOMETRY_KINDS:
        return [([d], label) for d, label in _grid()] + _geometry_lists()
    return [([d], label) for d, label in _grid()]


def _bytes(kind, descs):
    from delora_b200 import _lib as lib_
    L = lib_.lib()
    arr = (lib_.OdometryDesc * len(descs))(*descs)
    fn = getattr(L, BYTES[kind])
    return fn(arr, len(descs)) if kind in GEOMETRY_KINDS else fn(arr)


def _overlaps(secs):
    """[(a, b)] of the sections that share a byte"""
    s = sorted(secs, key=lambda x: (x.offset, x.offset + x.bytes))
    bad, end, last = [], -1, None
    for x in s:
        if x.offset < end:
            bad.append((last, x))
        if x.offset + x.bytes > end:
            end, last = x.offset + x.bytes, x
    return bad


def _disjoint_sets(kind, secs):
    """The lists of sections that must be pairwise disjoint: the shared sections once (geometry 0's copy) with every
    other section, or for the training geometries the shared ones with each geometry's own"""
    shared = [x for x in secs if x.flags & _lib.WS_SHARED and x.geometry == 0]
    own = [x for x in secs if not x.flags & _lib.WS_SHARED]
    if kind == "train_geometries":
        return [shared + [x for x in own if x.geometry == g] for g in sorted({x.geometry for x in secs})]
    return [shared + own]


def check_layout(kind, descs):
    """Asserts every invariant of the module docstring on one kind and descriptor list -> its sections"""
    secs = H.sections(kind, descs)
    total = _bytes(kind, descs)
    if kind in PRE_KINDS and descs[0].w_pre == 0:
        assert secs is None and total == -1, "the recipe kinds refuse w_pre = 0"
        return None
    assert secs is not None and total > 0, _lib.lib().delora_last_error()
    for x in secs:
        assert x.bytes > 0, f"{x}: empty"
        assert 0 <= x.offset and x.offset + x.bytes <= total, f"{x}: outside the {total}-byte workspace"
        assert x.flags & _lib.WS_SUBRANGE or x.offset % 256 == 0, f"{x}: not 256-byte aligned"
        assert 0 <= x.geometry < len(descs), x
    for group in _disjoint_sets(kind, secs):
        bad = _overlaps(group)
        assert not bad, f"overlapping sections: {bad[:4]}"
    names = [(x.geometry, x.name) for x in secs]
    assert len(names) == len(set(names)), "a section listed twice in one geometry"
    if kind in GEOMETRY_KINDS:
        per = [{x.name: (x.offset, x.bytes, x.role) for x in secs if x.geometry == g and x.flags & _lib.WS_SHARED}
               for g in range(len(descs))]
        assert per[0] and all(p == per[0] for p in per), "the shared sections differ between geometries"
        model = {"master", "trunk.table"} | ({"adam_m", "adam_v"} if kind == "train_geometries" else set())
        assert model <= set(per[0]), f"shared sections {sorted(per[0])[:8]} lack {model}"
    return secs


@pytest.mark.parametrize("kind", KINDS)
def test_sections_are_disjoint_aligned_and_inside_the_workspace(kind):
    for descs, label in _cases(kind):
        try:
            check_layout(kind, descs)
        except AssertionError as e:
            raise AssertionError(f"{kind} {label}: {e}") from None


def _as_set(secs):
    return {(x.geometry, x.name, x.offset, x.bytes) for x in secs}


@pytest.mark.parametrize("small,large", APPENDED, ids=[f"{a}-in-{b}" for a, b in APPENDED])
def test_appended_kinds_keep_every_section_of_the_kind_they_extend(small, large):
    cases = _geometry_lists() if small in GEOMETRY_KINDS else [([d], label) for d, label in _grid()]
    for descs, label in cases:
        a, b = H.sections(small, descs), H.sections(large, descs)
        assert a is not None and b is not None, label
        missing = _as_set(a) - _as_set(b)
        assert not missing, f"{small} in {large} {label}: moved or missing {sorted(missing)[:4]}"


def test_the_map_refuses_what_the_size_queries_refuse():
    d = _desc(16, 180)
    L = _lib.lib()
    arr = (_lib.OdometryDesc * 2)(d, _desc(16, 259))
    assert L.delora_odometry_workspace_sections(len(KINDS), arr, 1, None, 0) == -1
    assert L.delora_odometry_workspace_sections(-1, arr, 1, None, 0) == -1
    assert L.delora_odometry_workspace_sections(0, arr, 2, None, 0) == -1          # n > 1 on a one-geometry kind
    assert L.delora_odometry_workspace_sections(0, arr, 1, None, 4) == -1          # cap without out
    # mixed W parities: every geometries size query refuses them, so does the map
    for kind in GEOMETRY_KINDS:
        assert H.sections(kind, [d, _desc(16, 259)]) is None and _bytes(kind, [d, _desc(16, 259)]) == -1
    # the count does not depend on cap, and a short cap writes a prefix
    full = H.sections("train", [d])
    out = (_lib.WsSection * 3)()
    assert L.delora_odometry_workspace_sections(KINDS.index("train"), arr, 1, out, 3) == len(full)
    assert [r.name.decode() for r in out] == [x.name for x in full[:3]]
