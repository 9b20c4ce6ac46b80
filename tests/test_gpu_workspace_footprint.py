"""-m gpu: where each odometry workspace kind's calls write, against its section map (delora_odometry_workspace_sections)
at 16 x 180 (w_pre 360 for the recipe kinds), S <= 3 streams, two geometries for the geometries kinds.

After init, every byte of the workspace that belongs to no section (the alignment padding) is filled with a poison
pattern, then the kind's calls run: inference pairs and push, streams ticks with an inactive stream, an idle tick and a
reset, training eval and steps, adapting ticks with update 0 and 1, information on and off, an idle geometry.  After
each call, against the bytes before it:
  - the padding keeps the poison (no call writes outside its sections);
  - the weight sections are unchanged by every call but an update, and after an update the bf16 filters are what a
    fresh delora_conv_weight_prep_multi makes of the new master weights;
  - an idle geometry's state sections (its cached frames and has_prev) are unchanged;
  - the information section is unchanged by ticks without information, and the group section by the non-group forms."""
import pytest
import torch

import odometry_harness as H
from delora_b200 import _lib, ops
from delora_b200.deploy import capi

pytestmark = pytest.mark.gpu
DEV = H.DEV
POISON = 0xA5
ICP = ops.LOSS_PO2PL | ops.LOSS_PL2PL
GEOMS = ((16, 180, 0, 2), (16, 260, 0, 3))        # H, W, w_pre, S_g of the geometries kinds
W_PRE = 360


@pytest.fixture(scope="module")
def setup(cuda_lib):
    pool = H.frames(16, 256, 8)
    n_stride = max(f.shape[1] for f in pool)
    cfg = H.config(16, 180)
    blob = H.blob(H.model(cfg, 5, near_identity=True), cfg)
    return cfg, blob, pool, n_stride


class Footprint:
    """One workspace and its section map: the padding poisoned, the bytes of the last check kept"""

    def __init__(self, kind, ws, descs):
        self.secs = H.sections(kind, descs)
        assert self.secs, kind
        self.ws = ws
        covered = torch.zeros((ws.numel(),), dtype=torch.bool)
        for x in self.secs:
            covered[x.offset:x.offset + x.bytes] = True
        self.gap = (~covered).to(DEV)
        assert int(self.gap.sum()) > 0
        self.poison()

    def poison(self):
        """The padding filled with the poison (after an init call, which zeroes it), then a snapshot"""
        torch.cuda.synchronize()
        self.ws[self.gap] = POISON
        self.snap()

    def snap(self):
        torch.cuda.synchronize()
        self.before = self.ws.clone()

    def of(self, x, t=None):
        return (self.ws if t is None else t)[x.offset:x.offset + x.bytes]

    def named(self, pred):
        return [x for x in self.secs if pred(x)]

    def check(self, what, unchanged=lambda x: False, snap=True):
        """The padding holds the poison and every section with unchanged(x) its bytes of the last check; then (snap) a
        new snapshot"""
        torch.cuda.synchronize()
        assert bool((self.ws[self.gap] == POISON).all()), f"{what}: a write into the padding between sections"
        for x in self.named(unchanged):
            assert torch.equal(self.of(x), self.of(x, self.before)), f"{what}: {x} changed"
        if snap:
            self.snap()

    def check_fresh_filters(self, what):
        """After an update: the bf16 filters equal delora_conv_weight_prep_multi of the master weights through the
        workspace's own table; the padding holds the poison"""
        torch.cuda.synchronize()
        assert bool((self.ws[self.gap] == POISON).all()), f"{what}: a write into the padding between sections"
        table = self.named(lambda x: x.name == "trunk.table" and x.geometry == 0)[0]
        filt = self.named(lambda x: x.name.startswith(("trunk.fwd", "trunk.flip")) and x.geometry == 0)
        got = [self.of(x).clone() for x in filt]
        for x in filt:
            self.of(x).zero_()
        n_conv = sum(x.name.startswith("trunk.fwd") for x in filt)
        L = _lib.lib()
        _lib.check(L.delora_conv_weight_prep_multi(self.ws.data_ptr() + table.offset, n_conv,
                                                   torch.cuda.current_stream().cuda_stream), "prep_multi")
        torch.cuda.synchronize()
        for x, g in zip(filt, got):
            assert torch.equal(self.of(x), g), f"{what}: {x} is not the prep of the master weights"
        assert not all(torch.equal(self.of(x), self.of(x, self.before)) for x in filt), f"{what}: no filter changed"
        self.snap()


WEIGHTS = lambda x: x.role == "weights"          # noqa: E731


def _ticks(pool, S, n_stride):
    act, empty, resets = H.recipe_pattern(S, 5)
    return H.recipe_ticks(pool, S, n_stride, act, empty), resets


def _run_streams(fp, ws, ticks, rows, resets, updates=None, unchanged=WEIGHTS):
    def hook(w):
        fp.check("tick", unchanged)
    H.run_streams(ws, ticks, rows, resets=resets, updates=updates, hook=hook)


def test_inference(setup):
    cfg, blob, pool, n_stride = setup
    d = H.desc(cfg, n_stride, 2)
    ws = capi.InferenceWorkspace(d, blob)
    fp = Footprint("pairs", ws.workspace, [d])
    pts, counts = H.stack_pairs(H.pairs(16, 256, 2), n_stride)
    ws.pairs(pts, counts)
    fp.check("pairs", WEIGHTS)
    T = torch.empty((16,), dtype=torch.float32, device=DEV)
    for i, T_ in enumerate((None, T)):
        p, c = H.stack([pool[i]], n_stride)
        ws.push(p, c, T_)
        fp.check("push", WEIGHTS)


@pytest.mark.parametrize("kind", ["streams", "streams_residual", "streams_info", "streams_normalized", "streams_pre",
                                  "streams_pre_info"])
def test_streams(setup, kind):
    cfg, blob, pool, n_stride = setup
    S = 3
    pre = kind in ("streams_pre", "streams_pre_info")
    d = H.desc(cfg, n_stride, S, W_PRE if pre else 0)
    rp = capi.residual_params(cfg, ICP)
    ws, rows = {
        "streams": lambda: (capi.StreamsWorkspace(d, blob), ()),
        "streams_residual": lambda: (capi.ResidualStreamsWorkspace(d, blob, rp), ("losses",)),
        "streams_info": lambda: (capi.InformationStreamsWorkspace(d, blob, rp), ("losses", "info")),
        "streams_normalized": lambda: (capi.NormalizedStreamsWorkspace(d, blob), ("factor",)),
        "streams_pre": lambda: (capi.PreStreamsWorkspace(d, blob, rp), ("losses",)),
        "streams_pre_info": lambda: (capi.PreInformationStreamsWorkspace(d, blob, rp), ("losses", "info")),
    }[kind]()
    fp = Footprint(kind, ws.workspace, [d])
    ticks, resets = _ticks(pool, S, n_stride)
    _run_streams(fp, ws, ticks, rows, resets)


def test_training(setup):
    cfg, blob, pool, n_stride = setup
    d = H.desc(cfg, n_stride, 2)
    ws = capi.TrainingWorkspace(d, blob, H.train_params(lr=1e-4))
    fp = Footprint("train", ws.workspace, [d])
    pts, counts = H.stack_pairs(H.pairs(16, 256, 2), n_stride)
    ws.eval(pts, counts)
    fp.check("eval", WEIGHTS)
    for k in range(2):
        ws.step(pts, counts)
        fp.check_fresh_filters(f"step {k}")
    ws.eval(pts[1:3], counts[1:3])                  # B = 1 after B = 2: the ICP scratch is re-armed
    fp.check("eval at B = 1", WEIGHTS)


def test_training_geometries(setup):
    cfg, blob, pool, n_stride = setup
    descs = [H.desc(H.config(h, w), n_stride, S, wp) for h, w, wp, S in GEOMS]
    ws = capi.GeometriesTrainingWorkspace(descs, blob, H.train_params(lr=1e-4))
    fp = Footprint("train_geometries", ws.workspace, descs)
    pts, counts = H.stack_pairs(H.pairs(16, 256, 2), n_stride)
    for g in (0, 1, 0):
        ws.use(g)                   # an init of geometry g's section, which zeroes its padding too
        fp.poison()
        ws.eval(pts, counts)
        fp.check(f"eval on geometry {g}", WEIGHTS)
        ws.step(pts, counts)
        fp.check_fresh_filters(f"step on geometry {g}")


def _adapt_ticks(fp, ws, ticks, resets, rows, push_rows=None):
    """Ticks with update 0, 1, 0, 1, ...: the weights unchanged by update 0, fresh filters after update 1"""
    updates = [k % 2 for k in range(len(ticks))]
    S = ws.desc.max_batch
    out = H.Outputs(S, rows)
    mask = torch.zeros((S,), dtype=torch.int32, device=DEV)
    for k, (p, c, a) in enumerate(ticks):
        if k in resets:
            mask.zero_()
            mask[list(resets[k])] = 1
            ws.reset(mask)
            fp.check("reset", lambda x: x.role != "state")
        args = (p.to(DEV), c.to(DEV), a.to(DEV)) + out.tensors
        (push_rows or ws.push)(*args, update=updates[k])
        if updates[k]:
            fp.check_fresh_filters(f"tick {k}")
        else:
            fp.check(f"tick {k}", WEIGHTS)


def test_adapt(setup):
    cfg, blob, pool, n_stride = setup
    d = H.desc(cfg, n_stride, 3)
    ws = capi.AdaptiveStreamsWorkspace(d, blob, H.train_params(lr=1e-4))
    fp = Footprint("adapt", ws.workspace, [d])
    ticks, resets = _ticks(pool, 3, n_stride)
    _adapt_ticks(fp, ws, ticks, resets, ("losses",))


def test_adapt_info(setup):
    """Ticks with information, then ticks of _push_adapt on the same workspace: the information section stays; the
    group section stays throughout"""
    cfg, blob, pool, n_stride = setup
    d = H.desc(cfg, n_stride, 3)
    ws = capi.AdaptiveInformationStreamsWorkspace(d, blob, H.train_params(lr=1e-4))
    fp = Footprint("adapt_info", ws.workspace, [d])
    group = fp.named(lambda x: x.name in ("tick", "n_fleet", "slots"))
    info = fp.named(lambda x: x.name in ("info", "info_scratch"))
    assert len(group) == 3 and len(info) == 2
    group_bytes = [fp.of(x).clone() for x in group]
    ticks, resets = _ticks(pool, 3, n_stride)
    _adapt_ticks(fp, ws, ticks, resets, ("losses", "info"))
    plain = lambda *a, update: capi.AdaptiveStreamsWorkspace.push(ws, *a, update=update)      # noqa: E731
    info_bytes = [fp.of(x).clone() for x in info]
    _adapt_ticks(fp, ws, ticks, {}, ("losses",), push_rows=plain)
    assert all(torch.equal(fp.of(x), b) for x, b in zip(info, info_bytes)), "a tick without info wrote its section"
    assert all(torch.equal(fp.of(x), b) for x, b in zip(group, group_bytes)), "a non-group tick wrote the group section"


def test_adapt_group(setup):
    """Two ranks on one device: the group ticks write the group section and nothing outside the map"""
    cfg, blob, pool, n_stride = setup
    S = 2
    d = H.desc(cfg, n_stride, S)
    wss = [capi.AdaptiveStreamsGroupWorkspace(d, blob, H.train_params(lr=1e-4)) for _ in range(2)]
    fps = [Footprint("adapt_group", w.workspace, [d]) for w in wss]
    g = capi.AdaptingStreamsGroup(wss)
    streams = [torch.cuda.Stream() for _ in wss]
    for k in range(4):
        inputs = [H.pool_tick(pool, S, n_stride, k, [1] * S, offset=r) for r in range(2)]
        u = k % 2
        H.group_tick(g, streams, inputs, [u, u])
        assert H.group_status_ok(g)
        for r, fp in enumerate(fps):
            if u:
                fp.check_fresh_filters(f"rank {r} tick {k}")
            else:
                fp.check(f"rank {r} tick {k}", WEIGHTS)


@pytest.mark.parametrize("kind", ["adapt_geometries", "adapt_geometries_info"])
def test_adapt_geometries(setup, kind):
    """Ticks over both geometries, then geometry 1 idle (its state sections stay) with update 0 and 1, a reset; the
    information form also takes ticks without information (its information section stays)"""
    cfg, blob, pool, n_stride = setup
    descs = [H.desc(H.config(h, w), n_stride, S, wp) for h, w, wp, S in GEOMS]
    info = kind == "adapt_geometries_info"
    cls = capi.GeometriesAdaptingInformationStreamsWorkspace if info else capi.GeometriesAdaptingStreamsWorkspace
    ws = cls(descs, blob, H.train_params(lr=1e-4))
    fp = Footprint(kind, ws.workspace, descs)
    S0, S1 = GEOMS[0][3], GEOMS[1][3]
    rows = ("losses", "info") if info else ("losses",)

    def tick(k, active, update, with_info=info):
        pts, counts = [], []
        for g, (_, _, _, S) in enumerate(GEOMS):
            p, c, _ = H.pool_tick(pool, S, n_stride, k, [1] * S, offset=3 * g)
            pts.append(p)
            counts.append(c)
        out = H.Outputs(S0 + S1, rows if with_info else ("losses",))
        a = torch.tensor(active, dtype=torch.int32, device=DEV)
        if with_info:
            ws.push(pts, counts, a, *out.tensors, update=update)
        else:
            capi.GeometriesAdaptingStreamsWorkspace.push(ws, pts, counts, a, *out.tensors, update=update)
        out.snapshot(k)

    def after(what, update, keep=lambda x: False):
        if update:
            fp.check(what, keep, snap=False)
            fp.check_fresh_filters(what)
        else:
            fp.check(what, lambda x: WEIGHTS(x) or keep(x))

    for k in range(3):
        tick(k, [1] * (S0 + S1), k % 2)
        after(f"tick {k}", k % 2)
    idle = lambda x: x.geometry == 1 and x.role == "state"      # noqa: E731
    for k, u in ((3, 0), (4, 1)):
        tick(k, [1] * S0 + [0] * S1, u)
        after(f"tick {k}, geometry 1 idle", u, idle)
    mask = torch.tensor([0] * S0 + [1] + [0] * (S1 - 1), dtype=torch.int32, device=DEV)
    ws.reset(mask)
    fp.check("reset", lambda x: x.role != "state" or x.geometry == 0)
    if info:
        rows_ = lambda x: x.name in ("info", "info_scratch")     # noqa: E731
        for k, u in ((5, 0), (6, 1)):
            tick(k, [1] * (S0 + S1), u, with_info=False)
            after(f"tick {k} without info", u, rows_)
