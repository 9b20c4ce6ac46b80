"""-m gpu: one training workspace shared by several sensor geometries (delora_odometry_train_geometries_* and
delora_odometry_train_use_geometry) on the H100.

Three geometries with one model: 64 x 720 with w_pre 2250 (KITTI's vertical field of view), 64 x 512 with a +-22.5
degree one, and a small 16 x 180.  Every check is bit for bit against single-geometry workspaces, one per geometry,
that receive the state through _train_get_state -> _train_set_state (+ _train_set_dropout_seed) whenever the
geometry changes:
  - a sequence of steps that alternates geometries and varies B, with evaluations between them: losses, T, pooled and
    grads of every step, the outputs of every evaluation, the state being unchanged by an evaluation, and weights, m,
    v and step count at the end; with the ICP objective, the identity fit, dropout and normalization_scaling;
  - one CUDA graph per geometry of _use_geometry + _train_step, replayed alternately, gives the eager bits;
  - _train_step_group at world 2 with the two ranks on different geometries equals the same group of two
    single-geometry workspaces;
  - examples/odometry_train.c with a second dataset (--geometry) writes a .dlt that resumes to the bytes of an
    uninterrupted run.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200 import ops

pytestmark = pytest.mark.gpu
LR = 1e-4
LAYERS, NOUT = (1, 1, 1, 1), 64
# name -> (H, W, vfov in degrees, w_pre, synthetic scan width)
GEOMETRIES = {"64x720": (64, 720, (-24.5, 2.0), 2250, 1024), "64x512": (64, 512, (-22.5, 22.5), 0, 768),
              "16x180": (16, 180, (-15.0, 15.0), 0, 256)}
# normalization_scaling needs w_pre > 0 on every geometry
W_PRE_NORMALIZED = {"64x720": 2250, "64x512": 512, "16x180": 360}


class Geometry:
    def __init__(self, name, w_pre, max_batch=2, n_pairs=4):
        h, w, vfov, _, w_raw = GEOMETRIES[name]
        from delora_b200 import synthetic
        self.cfg = H.config(h, w, "tanh", False, LAYERS, NOUT, vfov=vfov)
        self.pairs = [synthetic.make_pair(100 * h + i, w_raw=w_raw, rings=h, vfov_deg=vfov)[:2] for i in range(n_pairs)]
        self.n_stride = H.n_stride(self.pairs)
        self.desc = H.desc(self.cfg, self.n_stride, max_batch, w_pre)

    def batch(self, first, b):
        return H.stack_pairs([self.pairs[(first + j) % len(self.pairs)] for j in range(b)], self.n_stride)


def _setup(flags, names=("64x720", "64x512", "16x180")):
    normalized = flags & ops.TRAIN_NORMALIZATION_SCALING
    geos = [Geometry(n, (W_PRE_NORMALIZED if normalized else {k: v[3] for k, v in GEOMETRIES.items()})[n])
            for n in names]
    blob = H.blob(H.model(geos[0].cfg, 31, near_identity=True), geos[0].cfg)
    return geos, blob


def _shared(geos, blob, flags):
    from delora_b200.deploy import capi
    return capi.GeometriesTrainingWorkspace([g.desc for g in geos], blob, capi.train_params(geos[0].cfg, LR,
                                                                                             loss_flags=flags))


def _single(geo, blob, flags):
    from delora_b200.deploy import capi
    return capi.TrainingWorkspace(geo.desc, blob, capi.train_params(geo.cfg, LR, loss_flags=flags))


class Reference:
    """One single-geometry workspace per geometry; the state moves to the one of the next call's geometry."""

    def __init__(self, geos, blob, flags, seed):
        self.ws = [_single(g, blob, flags) for g in geos]
        self.seed = seed
        self.cur = 0
        self.ws[0].set_dropout_seed(seed)

    def on(self, g):
        if g != self.cur:
            state = self.ws[self.cur].get_state()
            self.ws[g].set_state(*(t.cpu() for t in state[:3]), int(state[3].item()))
            self.ws[g].set_dropout_seed(self.seed)
            self.cur = g
        return self.ws[g]


def _equal_state(a, b, what):
    for x, y, name in zip(a, b, ("weights", "exp_avg", "exp_avg_sq", "step")):
        assert torch.equal(x, y), f"{what}: {name}"


# (op, geometry, B): steps alternate geometries, repeat one, vary B; evaluations sit between them
SEQUENCE = [("step", 0, 2), ("step", 1, 1), ("eval", 2, 2), ("step", 1, 2), ("step", 2, 2), ("eval", 0, 1),
            ("step", 0, 1), ("step", 2, 1), ("eval", 1, 2), ("step", 0, 2)]


@pytest.mark.parametrize("flags", [H.FLAGS, H.FLAGS | ops.LOSS_IDENTITY_FIT, H.FLAGS | ops.TRAIN_DROPOUT,
                                   H.FLAGS | ops.TRAIN_NORMALIZATION_SCALING],
                         ids=["icp", "identity", "dropout", "normalized"])
def test_alternating_geometries_match_single_geometry_workspaces(cuda_lib, flags):
    geos, blob = _setup(flags)
    seed = 0x1234567890AB
    shared = _shared(geos, blob, flags)
    shared.set_dropout_seed(seed)
    ref = Reference(geos, blob, flags, seed)
    for i, (op, g, b) in enumerate(SEQUENCE):
        pts, counts = geos[g].batch(i, b)
        if shared.geometry != g:
            shared.use(g)
        single = ref.on(g)
        what = f"{op} {i} on {list(GEOMETRIES)[g]}, B={b}"
        if op == "step":
            got, want = shared.step(pts, counts), single.step(pts, counts)
            names = ("losses", "T", "pooled", "grads")
        else:
            before = shared.get_state()
            got, want = shared.eval(pts, counts), single.eval(pts, counts)
            _equal_state(shared.get_state(), before, f"{what}: the evaluation changed the state")
            names = ("losses", "T", "pooled")
        for x, y, name in zip(got, want, names):
            assert torch.equal(x, y), f"{what}: {name}"
    _equal_state(shared.get_state(), ref.ws[ref.cur].get_state(), "end of the sequence")
    assert int(shared.get_state()[3].item()) == sum(op == "step" for op, _, _ in SEQUENCE)


def test_graph_replay_of_switch_and_step_matches_eager(cuda_lib):
    geos, blob = _setup(H.FLAGS, ("64x720", "16x180"))
    batches = [geos[0].batch(0, 2), geos[1].batch(1, 1)]
    runs = [_shared(geos, blob, H.FLAGS) for _ in range(2)]
    for ws in runs:                                   # one eager step per geometry first, as every graph test here
        for g in (0, 1):
            ws.use(g)
            ws.step(*batches[g], outputs=False)
    eager, graphed = runs
    for _ in range(3):
        for g in (0, 1):
            eager.use(g)
            eager.step(*batches[g], outputs=False)
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graphs = []
    for g in (0, 1):
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg, stream=stream):
            graphed.use(g)
            graphed.step(*batches[g], outputs=False)
        graphs.append(cg)
    for _ in range(3):
        for cg in graphs:
            cg.replay()
    torch.cuda.synchronize()
    _equal_state(graphed.get_state(), eager.get_state(), "graph replay against eager stepping")


def test_group_step_with_ranks_on_different_geometries(cuda_lib):
    from delora_b200.deploy import capi
    geos, blob = _setup(H.FLAGS, ("64x720", "16x180"))
    shared = [_shared(geos, blob, H.FLAGS) for _ in range(2)]
    shared[0].use(1)                                  # a round trip through the other geometry first
    shared[0].use(0)
    shared[1].use(1)
    single = [_single(geos[0], blob, H.FLAGS), _single(geos[1], blob, H.FLAGS)]
    groups = [capi.TrainingGroup(shared), capi.TrainingGroup(single)]
    streams = [torch.cuda.Stream() for _ in range(2)]

    def group_step(group, batches):
        torch.cuda.synchronize()
        outs = []
        for r, (pts, counts) in enumerate(batches):
            with torch.cuda.stream(streams[r]):
                outs.append(group.step(r, pts, counts))
        torch.cuda.synchronize()
        return outs

    for s in range(3):
        batches = [geos[0].batch(s, 2), geos[1].batch(s, 1 + s % 2)]
        got, want = group_step(groups[0], batches), group_step(groups[1], batches)
        for r in range(2):
            for x, y, name in zip(got[r], want[r], ("losses", "T", "pooled", "grads")):
                assert torch.equal(x, y), f"step {s}, rank {r}: {name}"
            _equal_state(shared[r].get_state(), single[r].get_state(), f"step {s}, rank {r}")
    assert all(int(st.item()) == 0 for g in groups for st in g.status)


def test_train_example_with_two_geometries_resumes_to_the_same_bytes(cuda_lib, tmp_path):
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    vfov, vfov2 = (-15.0, 15.0), (-20.0, 10.0)
    cfg = H.config(16, 720, "tanh", False, layers=LAYERS, nout=NOUT)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    init = os.path.join(tmp_path, "init.dlt")
    export.write_dlt(init, export.desc_from_config(cfg, "kitti", 4096, 2),
                     export.initial_training_state(dict(cfg, learning_rate=1e-4), 7))
    bins = []
    for i in range(5):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    second = os.path.join(tmp_path, "second")
    os.makedirs(second)
    for i in range(4):
        synthetic.kitti_bin_scan(40 + i, w_raw=96, rings=32, vfov_deg=vfov2).tofile(
            os.path.join(second, f"{i:06d}.bin"))
    exe = H.build_example("odometry_train", tmp_path, link=True)
    geometry = ["--geometry", f"{second},32,512,{vfov2[0]},{vfov2[1]}"]

    def run(src, dst, epochs):
        r = subprocess.run([exe] + geometry + ["--switch-below", "1e30", src, dst, str(epochs), "2"] + bins,
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        return r.stdout

    whole, half, resumed = (os.path.join(tmp_path, f) for f in ("whole.dlt", "half.dlt", "resumed.dlt"))
    out = run(init, whole, 2)
    assert len(out.splitlines()) == 2, out
    run(init, half, 1)
    run(half, resumed, 1)
    assert open(whole, "rb").read() == open(resumed, "rb").read()
    # the second dataset took part: the run differs from one on the listed scans alone
    alone = os.path.join(tmp_path, "alone.dlt")
    r = subprocess.run([exe, "--switch-below", "1e30", init, alone, "2", "2"] + bins, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    assert open(alone, "rb").read() != open(whole, "rb").read()
