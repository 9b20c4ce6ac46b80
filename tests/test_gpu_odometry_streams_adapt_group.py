"""-m gpu: one model adapted from the streams of several workspaces (delora_odometry_streams_push_adapt_group) on the
H100.  The ranks are adapting-streams group workspaces on ONE device, each ticked on its own stream with its own side
stream, reaching each other's group sections, gradient sections and flag words through plain device pointers (the
unicast path).  Every rank's tick is enqueued before any host synchronisation.

  - world = 1 is _push_adapt: the same bits over a mix of update = 0 / 1 ticks (T, valid, losses and the training
    state after every tick);
  - world = 2 and 4 with S = 2 per rank against one adapting workspace of S = 2 * world fed the same frames
    (rank-major), at lr 0 and beta1 0 so that every tick serves the same weights and exp_avg is the tick's gradient:
    every row's T, valid and loss row are bit-identical; after every update tick all ranks hold bit-identical weights,
    m, v and step count; exp_avg is within the harness's gradient bounds of the single workspace's;
  - the mean is over the pairs, not over the ranks: two valid pairs on rank 0 and none on rank 1 give the update of
    those two pairs, clearly not half of it;
  - a tick without a pair on any rank changes no rank's state, and the next update tick still meets and matches a
    group that never took the empty one;
  - different numbers of serve-only ticks per rank before an update give the bits of the group without them;
  - one captured update tick per rank, replayed, equals the eager ticks bit for bit, with status 0 throughout;
  - examples/odometry_streams.c --adapt --gpus 1 writes the .dlw of a run without --gpus."""
import os
import subprocess

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
HH, WW, W_RAW = 16, 180, 512


def _params(cfg, lr=LR, beta1=0.9):
    return capi.train_params(cfg, lr, loss_flags=ICP, beta1=beta1)


def _setup(seed=3, n_frames=10):
    cfg = H.config(HH, WW)
    pool = H.frames(HH, W_RAW, n_frames)
    n_stride = max(f.shape[1] for f in pool)
    return cfg, H.blob(H.model(cfg, seed, near_identity=True), cfg), pool, n_stride


@pytest.fixture(scope="module", autouse=True)
def _kernels_loaded(cuda_lib):
    """One _push_adapt update tick at the ranks' shape loads every kernel of a group tick but the collectives, which
    _adapt_group_init loads.  The ranks here share one device and one host thread, and under lazy module loading a
    kernel's first launch waits for the device's running kernels: a first load behind a rank that spins in the count
    exchange would hold its peers until the meet's timeout."""
    cfg, blob, pool, n_stride = _setup()
    _single_tick(_single(cfg, blob, n_stride, 2), *H.pool_tick(pool, 2, n_stride, 0, [1, 1]), True)


def _group(cfg, blob, n_stride, world, S=2, lr=LR, beta1=0.9):
    ws = [capi.AdaptiveStreamsGroupWorkspace(H.desc(cfg, n_stride, S), blob, _params(cfg, lr, beta1))
          for _ in range(world)]
    return capi.AdaptingStreamsGroup(ws), [torch.cuda.Stream() for _ in range(world)]


def _single(cfg, blob, n_stride, S, lr=LR, beta1=0.9):
    return capi.AdaptiveStreamsWorkspace(H.desc(cfg, n_stride, S), blob, _params(cfg, lr, beta1))


def _single_tick(ws, pts, counts, active, update):
    return H.run_streams(ws, [(pts, counts, active)], ("losses",), updates=[update])[0]


def test_single_rank_group_is_push_adapt(cuda_lib):
    cfg, blob, pool, n_stride = _setup()
    S = 3
    g, streams = _group(cfg, blob, n_stride, 1, S)
    plain = _single(cfg, blob, n_stride, S)
    updates = [True, False, True, True, False, True]
    acts = [[1, 1, 0], [1, 1, 1], [1, 0, 1], [0, 0, 0], [1, 1, 1], [1, 1, 1]]
    for k, (u, a) in enumerate(zip(updates, acts)):
        inp = H.pool_tick(pool, S, n_stride, k, a)
        (got,) = H.group_tick(g, streams, [inp], [u])
        want = _single_tick(plain, *inp, u)
        valid = want[1]
        assert H.same(got[1], valid), f"tick {k}: valid"
        for s in range(S):
            if int(valid[s]):
                assert H.same(got[0][s], want[0][s]), f"tick {k}, stream {s}: T"
        assert H.same(got[2], want[2]), f"tick {k}: losses"
        assert H.same_state(H.state(g.workspaces[0]), H.state(plain)), f"tick {k}: the training state"
    assert int(H.state(plain)[3][0]) >= 2
    assert H.group_status_ok(g)


def _check_rows(k, outs, single, world, S):
    for r in range(world):
        for s in range(S):
            row = r * S + s
            assert int(outs[r][1][s]) == int(single[1][row]), f"tick {k}, rank {r}, stream {s}: valid"
            if int(single[1][row]):
                assert H.same(outs[r][0][s], single[0][row]), f"tick {k}, rank {r}, stream {s}: T"
            assert H.same(outs[r][2][s], single[2][row]), f"tick {k}, rank {r}, stream {s}: losses"


def _check_ranks_agree(k, g):
    states = [H.state(w) for w in g.workspaces]
    for r in range(1, len(states)):
        assert H.same_state(states[r], states[0]), f"tick {k}: rank {r}'s state differs from rank 0's"
    return states[0]


def _check_mean(k, cfg, got, want):
    tail, trunk = H.grad_spread(H.grad_dict(got, cfg), H.grad_dict(want, cfg))
    print(f"\n[tick {k}] exp_avg against the single workspace: tail {tail:.2e}  trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL and trunk <= H.TRUNK_TOL, (k, tail, trunk)


def _run_against_single(cfg, blob, pool, n_stride, world, S, extra_serve=None):
    """Ticks 0 .. 3 (update on 1, 2, 3) of a group against one S * world workspace; extra_serve[r] = the number of
    update = 0 ticks rank r takes before tick 2, re-serving its frame of tick 1 -> the group's states after tick 3."""
    g, streams = _group(cfg, blob, n_stride, world, S, lr=0.0, beta1=0.0)
    single = _single(cfg, blob, n_stride, S * world, lr=0.0, beta1=0.0)
    acts = [[1] * S, [1] * S, [1] * (S - 1) + [0], [1] * S]
    for k in range(4):
        if k == 2 and extra_serve:                  # serve-only ticks run no collective: rank by rank
            for r in range(world):
                inp = H.pool_tick(pool, S, n_stride, 1, [1] * S, r * S)
                torch.cuda.synchronize()
                for _ in range(extra_serve[r]):
                    with torch.cuda.stream(streams[r]):
                        g.push(r, *inp, update=False)
            torch.cuda.synchronize()
        inputs = [H.pool_tick(pool, S, n_stride, k, acts[k], r * S) for r in range(world)]
        update = k > 0
        outs = H.group_tick(g, streams, inputs, [update] * world)
        ref = _single_tick(single, *H.pool_tick(pool, S * world, n_stride, k, acts[k] * world), update)
        _check_rows(k, outs, ref, world, S)
        state = _check_ranks_agree(k, g)
        if update:
            assert int(state[3][0]) == k
            _check_mean(k, cfg, state[1], H.state(single)[1])
    assert H.group_status_ok(g)
    return [H.state(w) for w in g.workspaces]


@pytest.mark.parametrize("world", [2, 4])
def test_group_update_is_the_mean_over_every_ranks_pairs(cuda_lib, world):
    cfg, blob, pool, n_stride = _setup()
    _run_against_single(cfg, blob, pool, n_stride, world, 2)


def test_uneven_serve_only_ticks_change_nothing(cuda_lib):
    cfg, blob, pool, n_stride = _setup()
    want = _run_against_single(cfg, blob, pool, n_stride, 2, 2)
    got = _run_against_single(cfg, blob, pool, n_stride, 2, 2, extra_serve=[0, 3])
    for r, (a, b) in enumerate(zip(got, want)):
        assert H.same_state(a, b), f"rank {r}: serve-only ticks changed the update"


def test_the_mean_is_over_pairs_not_ranks(cuda_lib):
    cfg, blob, pool, n_stride = _setup(seed=7)
    S = 2
    g, streams = _group(cfg, blob, n_stride, 2, S, lr=0.0, beta1=0.0)
    single = _single(cfg, blob, n_stride, S, lr=0.0, beta1=0.0)
    # tick 0: rank 0's first frames, rank 1 idle; tick 1: rank 0's two pairs, rank 1 on first frames only
    for k, (a0, a1) in enumerate(([[1, 1], [0, 0]], [[1, 1], [1, 1]])):
        inputs = [H.pool_tick(pool, S, n_stride, k, a0), H.pool_tick(pool, S, n_stride, k, a1, S)]
        outs = H.group_tick(g, streams, inputs, [True, True])
        ref = _single_tick(single, *inputs[0], True)
        assert outs[0][1].tolist() == ref[1].tolist() == ([0, 0] if k == 0 else [1, 1])
        assert outs[1][1].tolist() == [0, 0]
    state = _check_ranks_agree(1, g)
    assert int(state[3][0]) == 1                    # tick 0 had no pair anywhere
    want = H.state(single)[1]
    _check_mean(1, cfg, state[1], want)
    # the mean of the ranks' means would be half of it
    tail, trunk = H.grad_spread(H.grad_dict(state[1], cfg), H.grad_dict(want * 0.5, cfg))
    assert tail > 0.5 and trunk > 0.5, (tail, trunk)
    assert H.group_status_ok(g)


def test_no_pair_on_any_rank_no_update(cuda_lib):
    cfg, blob, pool, n_stride = _setup(seed=5)
    S, world = 2, 2
    empty, e_streams = _group(cfg, blob, n_stride, world, S)      # takes the empty update tick
    plain, p_streams = _group(cfg, blob, n_stride, world, S)      # serves that tick only
    before = [H.state(w) for w in empty.workspaces]
    inputs = [H.pool_tick(pool, S, n_stride, 0, [1, 1], r * S) for r in range(world)]
    outs = H.group_tick(empty, e_streams, inputs, [True] * world)
    assert all(int(o[1].sum()) == 0 for o in outs)
    for r in range(world):
        assert H.same_state(H.state(empty.workspaces[r]), before[r]), f"rank {r}: an update without a pair"
    H.group_tick(plain, p_streams, inputs, [False] * world)
    for k in (1, 2):
        inputs = [H.pool_tick(pool, S, n_stride, k, [1, 1], r * S) for r in range(world)]
        got = H.group_tick(empty, e_streams, inputs, [True] * world)
        want = H.group_tick(plain, p_streams, inputs, [True] * world)
        for r in range(world):
            for i, (x, y) in enumerate(zip(got[r], want[r])):
                assert H.same(x, y), f"tick {k}, rank {r}: output {i}"
            assert H.same_state(H.state(empty.workspaces[r]), H.state(plain.workspaces[r])), f"tick {k}, rank {r}"
    assert int(H.state(empty.workspaces[0])[3][0]) == 2
    assert H.group_status_ok(empty) and H.group_status_ok(plain)


def test_graph_replay_of_the_group_tick_matches_eager(cuda_lib):
    cfg, blob, pool, n_stride = _setup(seed=9)
    S, world, ticks = 2, 2, 4
    acts = [[1, 1], [1, 0], [1, 1], [1, 1]]

    def warm(g, streams, bufs):
        for b in bufs:                              # all inactive: no stream state or weight changes
            b[2].zero_()
        H.group_tick(g, streams, [b[:3] for b in bufs], [True] * world)

    def buffers():
        return [[torch.zeros((S, 3, n_stride), dtype=torch.float32, device=DEV),
                 torch.zeros((S,), dtype=torch.int32, device=DEV), torch.zeros((S,), dtype=torch.int32, device=DEV),
                 torch.zeros((S, 16), dtype=torch.float32, device=DEV),
                 torch.zeros((S,), dtype=torch.int32, device=DEV),
                 torch.zeros((S, ops.LOSS_ROW), dtype=torch.float32, device=DEV)] for _ in range(world)]

    def load(bufs, k):
        for r in range(world):
            for dst, src in zip(bufs[r][:3], H.pool_tick(pool, S, n_stride, k, acts[k], r * S)):
                dst.copy_(src)

    eager, e_streams = _group(cfg, blob, n_stride, world, S)
    ebufs = buffers()
    warm(eager, e_streams, ebufs)
    want = []
    for k in range(ticks):
        load(ebufs, k)
        want.append(H.group_tick(eager, e_streams, [b[:3] for b in ebufs], [True] * world))
    graphed, streams = _group(cfg, blob, n_stride, world, S)
    bufs = buffers()
    warm(graphed, streams, bufs)
    graphs = []
    for r in range(world):
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=streams[r]):
            graphed.push(r, *bufs[r][:3], update=True, out=tuple(bufs[r][3:]))
        graphs.append(cg)
    torch.cuda.synchronize()
    for k in range(ticks):
        load(bufs, k)
        torch.cuda.synchronize()
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                graphs[r].replay()
        torch.cuda.synchronize()
        for r in range(world):
            valid = bufs[r][4].cpu()
            assert H.same(valid, want[k][r][1]), f"tick {k}, rank {r}: valid"
            for s in range(S):
                if int(valid[s]):
                    assert H.same(bufs[r][3][s].cpu(), want[k][r][0][s]), f"tick {k}, rank {r}: T"
            assert H.same(bufs[r][5].cpu(), want[k][r][2]), f"tick {k}, rank {r}: losses"
        assert H.group_status_ok(graphed), f"tick {k}: a collective timed out"
    for r in range(world):
        assert H.same_state(H.state(graphed.workspaces[r]), H.state(eager.workspaces[r])), f"rank {r}: the state"
    assert int(H.state(graphed.workspaces[0])[3][0]) == ticks - 1         # tick 0 has first frames only
    assert H.group_status_ok(eager)


def test_example_with_one_gpu_writes_the_same_file(cuda_lib, tmp_path):
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False, layers=(1, 1, 1, 1), nout=64)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    model = H.model(cfg, 6, near_identity=True)
    dlw = os.path.join(tmp_path, "m.dlw")
    export.write_dlw(dlw, export.desc_from_config(cfg, "kitti", 4096, 1), export.pack_state_dict(model.state_dict(), cfg))
    dirs = []
    for s, n in enumerate((4, 3, 2)):
        dd = os.path.join(tmp_path, f"stream{s}")
        os.makedirs(dd)
        dirs.append(dd)
        for i in range(n):
            synthetic.kitti_bin_scan(10 * s + i, vfov_deg=vfov).tofile(os.path.join(dd, f"{i:06d}.bin"))
    exe = H.build_example("odometry_streams", tmp_path, link=True)

    def run(extra, dst):
        r = subprocess.run([exe, "--adapt", "1e-4", "--adapt-out", dst] + extra + [dlw] + dirs, capture_output=True,
                           text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        return r.stdout

    plain, one = os.path.join(tmp_path, "plain.dlw"), os.path.join(tmp_path, "one.dlw")
    out = run([], plain)
    assert len(out.strip().splitlines()) == 3 + 2 + 1
    assert out == run(["--gpus", "1"], one)
    assert open(plain, "rb").read() == open(one, "rb").read()
    assert open(plain, "rb").read() != open(dlw, "rb").read(), "the model did not adapt"
