"""-m gpu: the data-parallel training step of the C ABI (delora_odometry_train_step_group) on the H100.  The ranks are
training workspaces on ONE device, each stepped on its own stream with its own side stream, that reach each other's
gradient sections and flag words through plain device pointers (the unicast path, as test_gpu_allreduce.py).

  - world = 1 launches what delora_odometry_train_step launches: the same bits (weights, m, v, step, losses, T) over
    several steps, with and without dropout, in the identity fit, with a short last batch;
  - world = 2 and 4: after every step all ranks hold bit-identical weights, m and v; the averaged gradient each rank
    reports is, bit for bit, the sum in rank order times 1 / world of the gradients plain workspaces in the same state
    compute on each rank's pairs; the Adam update of that gradient is checked against float64 (the bound is in
    _check_adam); with the same pairs on two ranks the mean is the gradient itself, and the group steps equal plain
    steps bit for bit;
  - each rank's step captured into a CUDA graph and replayed on concurrent streams gives the eager bits (the
    sequence numbers come from the workspace, so every replay waits for the peers again);
  - examples/odometry_train.c --gpus 1 writes the .dlt of a run without the option.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200 import ops

pytestmark = pytest.mark.gpu
DEV = H.DEV
LR = 1e-4


def _setup(max_batch=2, n_pairs=8):
    cfg = H.config(16, 720, "tanh", False)
    model = H.model(cfg, 21, near_identity=True)
    pairs = H.pairs(16, 1024, n_pairs)
    return cfg, H.blob(model, cfg), pairs, H.n_stride(pairs)


def _batch(pairs, first, b, n_stride):
    return H.stack_pairs([pairs[(first + j) % len(pairs)] for j in range(b)], n_stride)


def _group(cfg, blob, n_stride, world, flags=H.FLAGS):
    from delora_b200.deploy import capi
    ws = [H.trainer(cfg, n_stride, 2, blob, LR, flags=flags) for _ in range(world)]
    g = capi.TrainingGroup(ws)
    streams = [torch.cuda.Stream() for _ in range(world)]
    return g, streams


def _group_step(g, streams, batches, outputs=True):
    """Every rank's group step on its own stream (enqueued rank by rank); -> the outputs per rank."""
    torch.cuda.synchronize()
    outs = []
    for r, (pts, counts) in enumerate(batches):
        with torch.cuda.stream(streams[r]):
            outs.append(g.step(r, pts, counts, outputs))
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("flags", [H.FLAGS, H.FLAGS | ops.TRAIN_DROPOUT, H.FLAGS | ops.LOSS_IDENTITY_FIT],
                         ids=["icp", "dropout", "identity"])
def test_single_rank_group_is_the_plain_step(cuda_lib, flags):
    cfg, blob, pairs, n_stride = _setup()
    plain = H.trainer(cfg, n_stride, 2, blob, LR, flags=flags)
    g, streams = _group(cfg, blob, n_stride, 1, flags)
    for s, b in enumerate((2, 2, 1)):                        # the last batch is short
        pts, counts = _batch(pairs, 2 * s, b, n_stride)
        want = plain.step(pts, counts)
        (got,) = _group_step(g, streams, [(pts, counts)])
        for x, y, name in zip(got, want, ("losses", "T", "pooled", "grads")):
            assert torch.equal(x, y), f"step {s}: {name} differs from delora_odometry_train_step"
        for x, y, name in zip(g.workspaces[0].get_state(), plain.get_state(), ("weights", "exp_avg", "exp_avg_sq",
                                                                               "step")):
            assert torch.equal(x, y), f"step {s}: {name} differs from delora_odometry_train_step"
    assert int(g.status[0].item()) == 0


def _check_adam(before, avg, after, step):
    """The update of Adam (beta1 0.9, beta2 0.999, eps 1e-8, no weight decay) from `before` with gradient `avg` against
    float64.  m and v: one product and one fused multiply-add (two products for v) in fp32, so each is within
    2 (4 for v) units of 2^-24 of the sum of its terms' magnitudes.  The weights are checked from the step's own m and
    v: the bias corrections 1 - beta^t lose up to log2(1 / (1 - beta2)) ~ 10 bits to cancellation at small t, so the
    update is good to ~2^-14 relative; 5e-4 of the update plus one ulp of the weight."""
    w0, m0, v0 = (t.double() for t in before[:3])
    w1, m1, v1 = (t.double() for t in after[:3])
    g = avg.double()
    b1, b2, eps = float(np.float32(0.9)), float(np.float32(0.999)), float(np.float32(1e-8))
    u = 2.0 ** -24
    assert ((m1 - (b1 * m0 + (1 - b1) * g)).abs() <= 2 * u * ((b1 * m0).abs() + ((1 - b1) * g).abs()) + 1e-45).all()
    assert ((v1 - (b2 * v0 + (1 - b2) * g * g)).abs() <= 4 * u * ((b2 * v0).abs() + (1 - b2) * g * g) + 1e-45).all()
    upd = float(np.float32(LR)) / (1 - b1 ** step) * m1 / (v1.sqrt() / (1 - b2 ** step) ** 0.5 + eps)
    assert ((w1 - (w0 - upd)).abs() <= 5e-4 * upd.abs() + 2 * u * w0.abs()).all()


@pytest.mark.parametrize("world", [2, 4])
def test_group_step_averages_the_ranks_gradients(cuda_lib, world):
    cfg, blob, pairs, n_stride = _setup()
    g, streams = _group(cfg, blob, n_stride, world)
    plain = [H.trainer(cfg, n_stride, 2, blob, LR) for _ in range(world)]
    for s in range(3):
        batches = [_batch(pairs, 2 * (s * world + r), 2, n_stride) for r in range(world)]
        before = g.workspaces[0].get_state()
        ref = []
        for r in range(world):
            plain[r].set_state(*(t.cpu() for t in before[:3]), int(before[3].item()))
            ref.append(plain[r].step(*batches[r]))
        avg = torch.zeros_like(ref[0][3])
        for r in range(world):                              # the kernel adds the ranks in this order
            avg = avg + ref[r][3]
        avg = avg * (1.0 / world)
        outs = _group_step(g, streams, batches)
        states = [w.get_state() for w in g.workspaces]
        for r in range(world):
            assert torch.equal(outs[r][3], avg), f"step {s}, rank {r}: the averaged gradient"
            for x, y, name in zip(states[r], states[0], ("weights", "exp_avg", "exp_avg_sq", "step")):
                assert torch.equal(x, y), f"step {s}: rank {r}'s {name} differs from rank 0's"
            # losses, T and pooled stay the rank's own: those of a plain step on its pairs from the same state
            for x, y, name in zip(outs[r][:3], ref[r][:3], ("losses", "T", "pooled")):
                assert torch.equal(x, y), f"step {s}, rank {r}: {name}"
        assert int(states[0][3].item()) == s + 1
        _check_adam(before, avg, states[0], s + 1)
        assert all(int(st.item()) == 0 for st in g.status)


def test_equal_pairs_on_two_ranks_equal_the_plain_step(cuda_lib):
    cfg, blob, pairs, n_stride = _setup()
    g, streams = _group(cfg, blob, n_stride, 2)
    plain = H.trainer(cfg, n_stride, 2, blob, LR)
    for s in range(3):
        batch = _batch(pairs, 2 * s, 2, n_stride)
        want = plain.step(*batch)
        outs = _group_step(g, streams, [batch, batch])
        for r in range(2):
            for x, y, name in zip(outs[r], want, ("losses", "T", "pooled", "grads")):
                assert torch.equal(x, y), f"step {s}, rank {r}: {name}"
            for x, y, name in zip(g.workspaces[r].get_state(), plain.get_state(), ("weights", "m", "v", "step")):
                assert torch.equal(x, y), f"step {s}, rank {r}: {name}"
    assert all(int(st.item()) == 0 for st in g.status)


def test_graph_replay_of_the_group_step_matches_eager(cuda_lib):
    world = 2
    cfg, blob, pairs, n_stride = _setup()
    batches = [_batch(pairs, 2 * r, 2, n_stride) for r in range(world)]
    eager, e_streams = _group(cfg, blob, n_stride, world)
    for _ in range(4):
        _group_step(eager, e_streams, batches, outputs=False)
    graphed, streams = _group(cfg, blob, n_stride, world)
    _group_step(graphed, streams, batches, outputs=False)     # one eager step first, as every graph test here
    graphs = []
    for r in range(world):
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=streams[r]):
            graphed.step(r, *batches[r], outputs=False)
        graphs.append(cg)
    torch.cuda.synchronize()
    for _ in range(3):
        for r in range(world):
            with torch.cuda.stream(streams[r]):
                graphs[r].replay()
    torch.cuda.synchronize()
    assert all(int(st.item()) == 0 for st in graphed.status)
    for r in range(world):
        for x, y, name in zip(graphed.workspaces[r].get_state(), eager.workspaces[r].get_state(),
                              ("weights", "exp_avg", "exp_avg_sq", "step")):
            assert torch.equal(x, y), f"rank {r}: graph replay differs from eager stepping in {name}"


def test_train_example_with_one_gpu_writes_the_same_file(cuda_lib, tmp_path):
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False, layers=(1, 1, 1, 1), nout=64)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    init = os.path.join(tmp_path, "init.dlt")
    export.write_dlt(init, export.desc_from_config(cfg, "kitti", 4096, 2),
                     export.initial_training_state(dict(cfg, learning_rate=1e-4), 7))
    bins = []
    for i in range(4):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    exe = H.build_example("odometry_train", tmp_path, link=True)

    def run(extra, dst):
        r = subprocess.run([exe] + extra + ["--switch-below", "1e30", init, dst, "2", "2"] + bins, capture_output=True,
                           text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        return r.stdout

    plain, one = os.path.join(tmp_path, "plain.dlt"), os.path.join(tmp_path, "one.dlt")
    assert run([], plain) == run(["--gpus", "1"], one)
    assert open(plain, "rb").read() == open(one, "rb").read()
