"""-m gpu: streams that adapt the model while serving it (delora_odometry_streams_push_adapt) on the H100.

- S = 1 with update = 1 is the training step: T, the loss rows and, after every tick, the _train_get_state bytes are
  bit-identical to a training workspace fed _train_step at B = 1 on (frame k-1, frame k), for a plain model at w_pre 0
  and at w_pre > 0 and for a normalised model;
- rows are independent: at S = 3 with update = 0 each row's T, loss row and valid flag are bit-identical to an S = 1
  workspace fed only that stream, across inactive ticks, resets and an empty frame;
- the update is the mean over the valid pairs: with beta1 = 0 Adam's exp_avg is the gradient, and one S = 3 tick with a
  stream on its first frame gives the mean of the other two streams' B = 1 _train_step gradients within the harness's
  bounds; changing the first-frame stream's scan leaves it byte-identical;
- a tick without a pair leaves the weights, m, v and the step count alone and serves the next tick as a workspace that
  never updated, while the cache still advances;
- one captured graph per value of update, alternated by the host, equals the eager calls bit for bit;
- _train_get_state / _set_state leave the stream section alone, and a resumed run continues bit for bit;
- AdaptiveOdometryStreams returns the workspace's bits and its state_dict loads into OdometryModel."""
import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200 import ops
from delora_b200.deploy import capi

pytestmark = pytest.mark.gpu
DEV = H.DEV
SENTINEL = 1234.5
ICP = ops.LOSS_PO2PL | ops.LOSS_PL2PL
LR = 1e-4


def _cfg(h, w, w_pre, normalized=False):
    cfg = H.config(h, w)
    cfg["kitti"]["horizontal_cells_preprocessing"] = w_pre
    cfg["normalization_scaling"] = normalized
    return cfg


def _params(cfg, normalized, lr=LR, beta1=0.9):
    return capi.train_params(cfg, lr, loss_flags=ICP | (ops.TRAIN_NORMALIZATION_SCALING if normalized else 0),
                             beta1=beta1)


def _adapt(cfg, blob, n_stride, S, w_pre, normalized=False, lr=LR, beta1=0.9):
    return capi.AdaptiveStreamsWorkspace(H.desc(cfg, n_stride, S, w_pre), blob, _params(cfg, normalized, lr, beta1))


class _Io:
    """The device arguments of one workspace's ticks."""

    def __init__(self, S, n_stride):
        self.pts = torch.zeros((S, 3, n_stride), dtype=torch.float32, device=DEV)
        self.counts = torch.zeros((S,), dtype=torch.int32, device=DEV)
        self.active = torch.zeros((S,), dtype=torch.int32, device=DEV)
        self.T = torch.full((S, 16), SENTINEL, dtype=torch.float32, device=DEV)
        self.valid = torch.full((S,), 7, dtype=torch.int32, device=DEV)
        self.losses = torch.full((S, ops.LOSS_ROW), SENTINEL, dtype=torch.float32, device=DEV)
        self.mask = torch.zeros((S,), dtype=torch.int32, device=DEV)

    def load(self, p, c, a):
        self.pts.copy_(p)
        self.counts.copy_(c)
        self.active.copy_(a)

    def args(self):
        return self.pts, self.counts, self.active, self.T, self.valid, self.losses

    def out(self):
        torch.cuda.synchronize()
        return self.T.cpu().clone(), self.valid.cpu().clone(), self.losses.cpu().clone()


def _run(ws, ticks, updates, resets=None):
    """Every tick (points [S, 3, n], counts [S], active [S]) through one workspace, eagerly -> [(T, valid, losses)]."""
    S = ws.desc.max_batch
    io = _Io(S, ticks[0][0].shape[2])
    out = []
    for k, (p, c, a) in enumerate(ticks):
        if resets and k in resets:
            io.mask.zero_()
            io.mask[resets[k]] = 1
            ws.reset(io.mask)
        io.load(p, c, a)
        ws.push(*io.args(), update=updates[k])
        out.append(io.out())
    return out


def _single_ticks(frames, n_stride, empty=()):
    out = []
    for k, f in enumerate(frames):
        p = torch.zeros((1, 3, n_stride), dtype=torch.float32)
        p[0, :, :f.shape[1]] = f
        out.append((p, torch.tensor([0 if k in empty else f.shape[1]], dtype=torch.int32),
                    torch.ones((1,), dtype=torch.int32)))
    return out


CASES = [(16, 180, 512, 0, False), (16, 180, 512, 360, False), (16, 180, 512, 360, True),
         (64, 720, 2048, 2250, True)]


@pytest.mark.parametrize("h,w,w_raw,w_pre,normalized", CASES,
                         ids=["16x180-plain", "16x180-pre360", "16x180-pre360-normalized", "64x720-pre2250-normalized"])
def test_one_stream_is_the_training_step(cuda_lib, h, w, w_raw, w_pre, normalized):
    K = 4
    cfg = _cfg(h, w, w_pre, normalized)
    frames = H.frames(h, w_raw, K)
    n_stride = max(f.shape[1] for f in frames)
    blob = H.blob(H.model(cfg, 11, near_identity=True), cfg)
    ws = _adapt(cfg, blob, n_stride, 1, w_pre, normalized)
    tr = capi.TrainingWorkspace(H.desc(cfg, n_stride, 1, w_pre), blob, _params(cfg, normalized))
    io = _Io(1, n_stride)
    for k, (p, c, a) in enumerate(_single_ticks(frames, n_stride)):
        io.load(p, c, a)
        ws.push(*io.args(), update=True)
        T, valid, losses = io.out()
        assert int(valid[0]) == (1 if k else 0), (k, int(valid[0]))
        if k:
            pts, counts = H.stack([frames[k - 1], frames[k]], n_stride)
            l_ref, t_ref, _, _ = tr.step(pts, counts)
            torch.cuda.synchronize()
            assert H.same(T[0], t_ref.reshape(16).cpu()), f"tick {k}: T differs from _train_step at B = 1"
            assert H.same(losses[0], l_ref[0].cpu()), f"tick {k}: {losses[0].tolist()} != {l_ref[0].tolist()}"
        else:
            assert float(losses[0].abs().max()) == 0.0
        assert H.same_state(H.state(ws), H.state(tr)), f"tick {k}: the training state differs from _train_step's"
    assert int(H.state(ws)[3][0]) == K - 1


def _pattern(S, ticks=7):
    act = np.ones((ticks, S), dtype=bool)
    act[1, S - 1] = False                   # an inactive stream
    act[4, :] = False                       # an idle tick
    if ticks > 6:
        act[6, 0] = False
    return act, {(2, 1 % S)}, {3: [0]}


def _ticks(pool, S, n_stride, act, empty):
    out = []
    for k in range(act.shape[0]):
        pts = torch.zeros((S, 3, n_stride), dtype=torch.float32)
        counts = torch.zeros((S,), dtype=torch.int32)
        for s in range(S):
            # an inactive stream is staged with real points and count: only the mask keeps it out
            f = pool[(3 * s + k) % len(pool)] if act[k, s] else pool[(3 * s + k + 5) % len(pool)]
            pts[s, :, :f.shape[1]] = f
            counts[s] = 0 if (k, s) in empty else f.shape[1]
        out.append((pts, counts, torch.from_numpy(act[k].astype(np.int32))))
    return out


@pytest.mark.parametrize("w_pre,normalized", [(0, False), (360, False), (360, True)],
                         ids=["plain", "pre360", "pre360-normalized"])
def test_rows_are_independent(cuda_lib, w_pre, normalized):
    h, w, w_raw, S = 16, 180, 512, 3
    cfg = _cfg(h, w, w_pre, normalized)
    pool = H.frames(h, w_raw, 8)
    n_stride = max(f.shape[1] for f in pool)
    act, empty, resets = _pattern(S)
    ticks = _ticks(pool, S, n_stride, act, empty)
    blob = H.blob(H.model(cfg, 5, near_identity=True), cfg)
    updates = [False] * len(ticks)
    out = _run(_adapt(cfg, blob, n_stride, S, w_pre, normalized), ticks, updates, resets)
    assert int(out[0][1].sum()) == 0 and sum(int(o[1].sum()) for o in out) >= 8
    for s in range(S):
        single = [(p[s:s + 1], c[s:s + 1], a[s:s + 1]) for p, c, a in ticks]
        res = {k: [0] for k, streams in resets.items() if s in streams}
        one = _run(_adapt(cfg, blob, n_stride, 1, w_pre, normalized), single, updates, res)
        for k, (e, o) in enumerate(zip(out, one)):
            assert int(e[1][s]) == int(o[1][0]), f"tick {k} stream {s}: valid differs from S = 1"
            assert H.same(e[0][s], o[0][0]), f"tick {k} stream {s}: T differs from S = 1"
            assert H.same(e[2][s], o[2][0]), f"tick {k} stream {s}: losses differ from S = 1"
            if not int(e[1][s]):
                assert float(e[2][s].abs().max()) == 0.0


def _mean_tick(cfg, blob, frames, n_stride, third):
    """S = 3, beta1 = 0: tick 0 gives streams 0 and 1 a first frame, tick 1 their second and stream 2 `third` (its
    first frame) with update = 1 -> (exp_avg, the step count)."""
    ws = _adapt(cfg, blob, n_stride, 3, 0, lr=LR, beta1=0.0)
    p0, c0 = H.stack([frames[0], frames[2], third], n_stride)
    p1, c1 = H.stack([frames[1], frames[3], third], n_stride)
    ticks = [(p0.cpu(), c0.cpu(), torch.tensor([1, 1, 0], dtype=torch.int32)),
             (p1.cpu(), c1.cpu(), torch.tensor([1, 1, 1], dtype=torch.int32))]
    out = _run(ws, ticks, [True, True])
    assert out[1][1].tolist() == [1, 1, 0]
    st = H.state(ws)
    return st[1], int(st[3][0])


def test_the_update_is_the_mean_over_the_valid_pairs(cuda_lib):
    h, w, w_raw = 16, 180, 512
    cfg = _cfg(h, w, 0)
    frames = H.frames(h, w_raw, 6)
    n_stride = max(f.shape[1] for f in frames)
    blob = H.blob(H.model(cfg, 13, near_identity=True), cfg)
    exp_avg, step = _mean_tick(cfg, blob, frames, n_stride, frames[4])
    assert step == 1
    grads = []
    for a, b in ((0, 1), (2, 3)):
        tr = capi.TrainingWorkspace(H.desc(cfg, n_stride, 1, 0), blob, _params(cfg, False, beta1=0.0))
        pts, counts = H.stack([frames[a], frames[b]], n_stride)
        grads.append(tr.step(pts, counts)[3].cpu())
    mean = H.grad_dict((grads[0] + grads[1]) * 0.5, cfg)
    tail, trunk = H.grad_spread(H.grad_dict(exp_avg, cfg), mean)
    print(f"\n[mean over valid pairs] tail {tail:.2e}  trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL and trunk <= H.TRUNK_TOL, (tail, trunk)
    # the first-frame stream adds exact zeros: another scan there gives the same bytes
    other, _ = _mean_tick(cfg, blob, frames, n_stride, frames[5])
    assert torch.equal(other.view(torch.int32), exp_avg.view(torch.int32))


@pytest.mark.parametrize("w_pre", [0, 360])
def test_no_pair_no_update(cuda_lib, w_pre):
    h, w, w_raw, S = 16, 180, 512, 2
    cfg = _cfg(h, w, w_pre)
    pool = H.frames(h, w_raw, 4)
    n_stride = max(f.shape[1] for f in pool)
    blob = H.blob(H.model(cfg, 3, near_identity=True), cfg)
    act = np.ones((3, S), dtype=bool)
    ticks = _ticks(pool, S, n_stride, act, set())
    ws = _adapt(cfg, blob, n_stride, S, w_pre)
    before = H.state(ws)
    out = _run(ws, ticks[:1], [True])
    assert int(out[0][1].sum()) == 0
    assert H.same_state(H.state(ws), before), "an update without a valid pair changed the training state"
    # the cache advanced, and the filters are the ones a workspace that never updated serves with
    ref = _run(_adapt(cfg, blob, n_stride, S, w_pre), ticks[:2], [False, False])
    nxt = _run(ws, ticks[1:2], [False])
    assert nxt[0][1].tolist() == [1] * S
    for a, b in zip(nxt[0], ref[1]):
        assert H.same(a, b)


def test_graphs_replay_the_eager_calls(cuda_lib):
    h, w, w_raw, w_pre, S = 16, 180, 512, 360, 3
    cfg = _cfg(h, w, w_pre)
    pool = H.frames(h, w_raw, 8)
    n_stride = max(f.shape[1] for f in pool)
    act, empty, _ = _pattern(S, 6)
    ticks = _ticks(pool, S, n_stride, act, empty)
    updates = [False, True, False, True, True, False]
    blob = H.blob(H.model(cfg, 8, near_identity=True), cfg)

    def warm(ws, io):
        io.active.zero_()                    # all inactive: no stream state or weight changes
        for u in (False, True):
            ws.push(*io.args(), update=u)
        torch.cuda.synchronize()

    eager_ws = _adapt(cfg, blob, n_stride, S, w_pre)
    io = _Io(S, n_stride)
    warm(eager_ws, io)
    eager = []
    for k, (p, c, a) in enumerate(ticks):
        io.load(p, c, a)
        eager_ws.push(*io.args(), update=updates[k])
        eager.append(io.out())
    g_ws = _adapt(cfg, blob, n_stride, S, w_pre)
    gio = _Io(S, n_stride)
    warm(g_ws, gio)
    graphs = {}
    for u in (False, True):
        graphs[u] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[u]):
            g_ws.push(*gio.args(), update=u)
    for k, (p, c, a) in enumerate(ticks):
        gio.load(p, c, a)
        graphs[updates[k]].replay()
        got = gio.out()
        for i, (x, y) in enumerate(zip(eager[k], got)):
            assert H.same(x, y), f"tick {k}: output {i} of the replay differs from the eager call"
    assert H.same_state(H.state(eager_ws), H.state(g_ws))
    assert int(H.state(g_ws)[3][0]) == 2          # ticks 1 and 3 update; tick 4 has no stream, so no pair


def test_state_round_trip_leaves_the_streams_and_resumes(cuda_lib):
    h, w, w_raw, w_pre, S = 16, 180, 512, 0, 2
    cfg = _cfg(h, w, w_pre)
    pool = H.frames(h, w_raw, 8)
    n_stride = max(f.shape[1] for f in pool)
    ticks = _ticks(pool, S, n_stride, np.ones((6, S), dtype=bool), set())
    blob = H.blob(H.model(cfg, 4, near_identity=True), cfg)
    a = _adapt(cfg, blob, n_stride, S, w_pre)
    _run(a, ticks[:3], [True] * 3)
    train_bytes = capi.TrainingWorkspace.workspace_bytes(a.desc)
    section = a.workspace[train_bytes:].cpu().clone()
    st = H.state(a)
    a.set_state(st[0], st[1], st[2], int(st[3][0]))
    assert torch.equal(a.workspace[train_bytes:].cpu(), section), "_train_set_state wrote into the stream section"
    assert H.same_state(H.state(a), st)
    want = _run(a, ticks[3:], [True] * 3)
    b = _adapt(cfg, blob, n_stride, S, w_pre)
    b.set_state(st[0], st[1], st[2], int(st[3][0]))
    _run(b, ticks[2:3], [False])               # the last served frame into the cache
    got = _run(b, ticks[3:], [True] * 3)
    for k, (x, y) in enumerate(zip(want, got)):
        for i, (u, v) in enumerate(zip(x, y)):
            assert H.same(u, v), f"resumed tick {k}: output {i} differs"
    assert H.same_state(H.state(a), H.state(b))


def test_python_class(cuda_lib):
    from delora_b200.deploy import export
    from delora_b200.deploy.stream import AdaptiveOdometryStreams
    from delora_b200.models.model import OdometryModel
    h, w, w_raw, w_pre, S = 16, 180, 512, 360, 2
    cfg = _cfg(h, w, w_pre)
    pool = H.frames(h, w_raw, 8)
    n_stride = max(f.shape[1] for f in pool)
    act, _, _ = _pattern(S, 5)
    act[4, :] = True
    ticks = _ticks(pool, S, n_stride, act, set())
    model = H.model(cfg, 9, near_identity=True)
    cls = AdaptiveOdometryStreams(model, cfg, "kitti", S, n_stride, LR, preprocessing_normals=True)
    ws = _adapt(cfg, H.blob(model, cfg), n_stride, S, w_pre)
    ws_out = _run(ws, ticks, [True] * len(ticks))
    served = [0] * S
    for k, (p, c, a) in enumerate(ticks):
        scans = [p[s, :, :int(c[s])].clone() if int(a[s]) else None for s in range(S)]
        got = cls.push(scans)
        for s in range(S):
            if got[s] is None:
                assert not int(ws_out[k][1][s])
                continue
            served[s] += 1
            t, losses = got[s]
            assert np.array_equal(t.reshape(16).view(np.int32), ws_out[k][0][s].numpy().view(np.int32))
            assert np.array_equal(losses.view(np.int32), ws_out[k][2][s].numpy().view(np.int32))
    for s in range(S):
        assert len(cls.relative[s]) == served[s] and len(cls.poses(s)) >= served[s]
    sd = cls.state_dict()
    m = OdometryModel(cfg).to(DEV)
    m.load_state_dict(sd)
    w_ref = ws.weights().cpu()
    assert torch.equal(torch.from_numpy(export.pack_state_dict(m.state_dict(), cfg)).view(torch.int32),
                       w_ref.view(torch.int32))
    assert not torch.equal(w_ref, H.blob(model, cfg).cpu()), "the model did not adapt"
