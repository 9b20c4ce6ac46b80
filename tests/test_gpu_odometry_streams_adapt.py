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


def _run(ws, ticks, updates, resets=None, hook=None):
    """Every tick (points [S, 3, n], counts [S], active [S]) through one workspace, eagerly -> [(T, valid, losses)]."""
    return H.run_streams(ws, ticks, ("losses",), resets=resets, updates=updates, hook=hook)


def _single_ticks(frames, n_stride):
    return H.stage_ticks(np.ones((len(frames), 1), dtype=bool), n_stride, lambda k, s: frames[k])


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
    out = _run(ws, _single_ticks(frames, n_stride), [True] * K, hook=H.state)
    for k, (T, valid, losses, state) in enumerate(out):
        assert int(valid[0]) == (1 if k else 0), (k, int(valid[0]))
        if k:
            pts, counts = H.stack([frames[k - 1], frames[k]], n_stride)
            l_ref, t_ref, _, _ = tr.step(pts, counts)
            torch.cuda.synchronize()
            assert H.same(T[0], t_ref.reshape(16).cpu()), f"tick {k}: T differs from _train_step at B = 1"
            assert H.same(losses[0], l_ref[0].cpu()), f"tick {k}: {losses[0].tolist()} != {l_ref[0].tolist()}"
        else:
            assert float(losses[0].abs().max()) == 0.0
        assert H.same_state(state, H.state(tr)), f"tick {k}: the training state differs from _train_step's"
    assert int(H.state(ws)[3][0]) == K - 1


@pytest.mark.parametrize("w_pre,normalized", [(0, False), (360, False), (360, True)],
                         ids=["plain", "pre360", "pre360-normalized"])
def test_rows_are_independent(cuda_lib, w_pre, normalized):
    h, w, w_raw, S = 16, 180, 512, 3
    cfg = _cfg(h, w, w_pre, normalized)
    pool = H.frames(h, w_raw, 8)
    n_stride = max(f.shape[1] for f in pool)
    act, empty, resets = H.recipe_pattern(S)
    ticks = H.recipe_ticks(pool, S, n_stride, act, empty)
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
    ticks = H.recipe_ticks(pool, S, n_stride, act, set())
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
    act, empty, _ = H.recipe_pattern(S, 6)
    ticks = H.recipe_ticks(pool, S, n_stride, act, empty)
    updates = [False, True, False, True, True, False]
    blob = H.blob(H.model(cfg, 8, near_identity=True), cfg)
    eager_ws, g_ws = _adapt(cfg, blob, n_stride, S, w_pre), _adapt(cfg, blob, n_stride, S, w_pre)
    eager = _run(eager_ws, ticks, updates)
    graphed = H.run_streams(g_ws, ticks, ("losses",), updates=updates, graph=True)
    for k, (e, g) in enumerate(zip(eager, graphed)):
        for i, (x, y) in enumerate(zip(e, g)):
            assert H.same(x, y), f"tick {k}: output {i} of the replay differs from the eager call"
    assert H.same_state(H.state(eager_ws), H.state(g_ws))
    assert int(H.state(g_ws)[3][0]) == 2          # ticks 1 and 3 update; tick 4 has no stream, so no pair


def test_state_round_trip_leaves_the_streams_and_resumes(cuda_lib):
    h, w, w_raw, w_pre, S = 16, 180, 512, 0, 2
    cfg = _cfg(h, w, w_pre)
    pool = H.frames(h, w_raw, 8)
    n_stride = max(f.shape[1] for f in pool)
    ticks = H.recipe_ticks(pool, S, n_stride, np.ones((6, S), dtype=bool), set())
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
    act, _, _ = H.recipe_pattern(S, 5)
    act[4, :] = True
    ticks = H.recipe_ticks(pool, S, n_stride, act, set())
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
