"""-m gpu: evaluation through the C ABI on the H100 -- delora_odometry_train_eval (the ICP losses of a training
workspace's current weights, nothing updated) and delora_odometry_streams_push_residual (a per-frame ICP loss row
beside every streamed transform) -- on seeded synthetic scans, at 16 x 180 and once each at 64 x 720.

  - _train_eval returns the bits _train_step returns from the same state (losses, T, pooled), for w_pre = 0 and > 0,
    normalised or not and every ICP loss-bit combination; it leaves the master weights, the gradient, Adam's state, the
    dropout seed and the bf16 filters byte for byte; steps interleaved with evals of other batch sizes end where the
    steps alone end; the dropout and identity bits are ignored; a captured eval replays to the eager result.
  - _push_residual's T and valid are _streams_push's bytes over an activity pattern with idle ticks, a late start and
    a reset; each valid loss row is, bit for bit, the row of the dense ICP operator run alone at B = 1 on that stream's
    two frames' grids and that T (the operator's finalize sums each pair's partial rows in a fixed order that does not
    depend on the batch, and this test is what holds it to that); invalid rows are zeros; guard bytes around the
    workspace and around `losses` stay intact; one captured call serves the whole pattern.
"""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200 import _lib, ops
from delora_b200.deploy import capi

pytestmark = pytest.mark.gpu
DEV = H.DEV
ICP = ops.LOSS_PO2PL | ops.LOSS_PL2PL
ALL_ICP = ops.LOSS_PO2PO | ops.LOSS_PO2PL | ops.LOSS_PL2PL


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _batch(pairs, s, b, n_stride):
    return H.stack_pairs([pairs[(s + j) % len(pairs)] for j in range(b)], n_stride)


# ================================================================================================== _train_eval
def _setup(h=16, w=180, w_raw=256, n_pairs=4, seed=20):
    cfg = H.config(h, w, "tanh", False)
    model = H.model(cfg, seed, near_identity=True)
    pairs = H.pairs(h, w_raw, n_pairs)
    return cfg, H.blob(model, cfg), pairs, H.n_stride(pairs)


def _persistent_bytes(tr):
    """The sections of a training workspace that outlive a step, read raw: master weights, gradient, exp_avg,
    exp_avg_sq (each weight_floats floats, 256-byte aligned), then the counter slot -- the step count, the ICP
    scratch's batch size (which an eval may record) and the dropout seed -- and the bf16 filters behind it."""
    a = (tr.n * 4 + 255) // 256 * 256
    ws = tr.workspace
    layers = (ctypes.c_int * 4)(*tr.desc.layers)
    filters = int(_lib.lib().delora_trunk_weight_bytes(layers, tr.desc.W))
    assert filters > 0
    ctr = ws[4 * a:4 * a + 24].clone().view(torch.int64)
    return {"weights": ws[:a].clone(), "gradient": ws[a:2 * a].clone(), "exp_avg": ws[2 * a:3 * a].clone(),
            "exp_avg_sq": ws[3 * a:4 * a].clone(), "step count": ctr[0:1], "dropout seed": ctr[2:3],
            "bf16 filters": ws[4 * a + 256:4 * a + 256 + filters].clone()}


def _eval_then_step(tr, pairs, n_stride, b):
    """One step for a non-trivial state, then an eval and a step on the same pairs -> their outputs; asserts the eval
    left every persistent section as it was."""
    tr.set_dropout_seed(77)
    tr.step(*_batch(pairs, 1, b, n_stride), outputs=False)
    pts, counts = _batch(pairs, 0, b, n_stride)
    before = _persistent_bytes(tr)
    state = tr.get_state()
    ev = tr.eval(pts, counts)
    torch.cuda.synchronize()
    for name, was in before.items():
        assert torch.equal(_persistent_bytes(tr)[name], was), f"the eval changed the {name}"
    for x, y, name in zip(state, tr.get_state(), ("weights", "exp_avg", "exp_avg_sq", "step")):
        assert torch.equal(x, y), f"the eval changed {name} (_train_get_state)"
    st = tr.step(pts, counts)
    torch.cuda.synchronize()
    return ev, st


FLAG_SETS = [ICP, ops.LOSS_PO2PO, ops.LOSS_PO2PL, ops.LOSS_PL2PL, ALL_ICP, ALL_ICP | ops.NORMAL_LINEAR]


@pytest.mark.parametrize("flags", FLAG_SETS, ids=[f"flags{f}" for f in FLAG_SETS])
def test_eval_returns_the_steps_bits_and_updates_nothing(cuda_lib, flags):
    cfg, blob, pairs, n_stride = _setup()
    ev, st = _eval_then_step(H.trainer(cfg, n_stride, 3, blob, 1e-4, flags=flags), pairs, n_stride, 2)
    for x, y, name in zip(ev, st, ("losses", "T", "pooled")):
        assert _same(x, y), f"{name}: the eval differs from the step"
    assert float(ev[0][:, 3].min()) > 0, "no matched pairs: the comparison is empty"


@pytest.mark.parametrize("normalized", [False, True], ids=["w_pre", "w_pre-normalized"])
def test_eval_at_the_preprocessing_width(cuda_lib, normalized):
    cfg, blob, pairs, n_stride = _setup()
    flags = ICP | (ops.TRAIN_NORMALIZATION_SCALING if normalized else 0)
    ev, st = _eval_then_step(H.trainer(cfg, n_stride, 3, blob, 1e-4, w_pre=360, flags=flags), pairs, n_stride, 2)
    for x, y, name in zip(ev, st, ("losses", "T", "pooled")):
        assert _same(x, y), f"{name}: the eval differs from the step"
    assert bool((ev[0][:, 6] > 0).all()) == normalized          # the factor column


def test_eval_at_64x720(cuda_lib):
    cfg, blob, pairs, n_stride = _setup(64, 720, 1024, 3, seed=21)
    ev, st = _eval_then_step(H.trainer(cfg, n_stride, 2, blob, 1e-4), pairs, n_stride, 2)
    for x, y, name in zip(ev, st, ("losses", "T", "pooled")):
        assert _same(x, y), f"{name}: the eval differs from the step"


def test_steps_interleaved_with_evals_end_in_the_same_state(cuda_lib):
    cfg, blob, pairs, n_stride = _setup()
    bs = [2, 1, 3, 3, 2]
    plain = H.trainer(cfg, n_stride, 3, blob, 1e-4)
    mixed = H.trainer(cfg, n_stride, 3, blob, 1e-4)
    outs_p = [plain.step(*_batch(pairs, s, b, n_stride)) for s, b in enumerate(bs)]
    outs_m = []
    eval_bs = [3, 3, 1, 2, 1]            # never the neighbouring steps' batch size twice: every call re-arms the ICP
    for s, b in enumerate(bs):
        mixed.eval(*_batch(pairs, s + 2, eval_bs[s], n_stride))
        outs_m.append(mixed.step(*_batch(pairs, s, b, n_stride)))
    mixed.eval(*_batch(pairs, 1, 2, n_stride))
    torch.cuda.synchronize()
    for s, (x, y) in enumerate(zip(outs_p, outs_m)):
        for xx, yy, name in zip(x, y, ("losses", "T", "pooled", "grads")):
            assert _same(xx, yy), f"step {s + 1}: {name} differ with evals in between"
    for x, y, name in zip(plain.get_state(), mixed.get_state(), ("weights", "exp_avg", "exp_avg_sq", "step")):
        assert torch.equal(x, y), f"{name} differ with evals in between"


def test_eval_ignores_the_dropout_and_identity_bits(cuda_lib):
    cfg, blob, pairs, n_stride = _setup()
    pts, counts = _batch(pairs, 0, 2, n_stride)
    plain = H.trainer(cfg, n_stride, 2, blob, 1e-4).eval(pts, counts)
    tr = H.trainer(cfg, n_stride, 2, blob, 1e-4, flags=ICP | ops.TRAIN_DROPOUT | ops.LOSS_IDENTITY_FIT)
    tr.set_dropout_seed(5)
    flagged = tr.eval(pts, counts)
    torch.cuda.synchronize()
    for x, y, name in zip(plain, flagged, ("losses", "T", "pooled")):
        assert _same(x, y), f"{name}: the dropout / identity bits changed the eval"
    assert float(flagged[0][:, 5].abs().max()) == 0.0
    # the step they train with does apply the masks
    assert not _same(tr.step(pts, counts)[2], plain[2])


def test_eval_replays_from_a_graph(cuda_lib):
    cfg, blob, pairs, n_stride = _setup()
    tr = H.trainer(cfg, n_stride, 2, blob, 1e-4)
    pts, counts = (t.clone() for t in _batch(pairs, 0, 2, n_stride))
    tr.eval(pts, counts)                                     # warms the launchers' host-side caches
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = tr.eval(pts, counts)
    for s in (1, 2):
        p, c = _batch(pairs, s, 2, n_stride)
        pts.copy_(p)
        counts.copy_(c)
        g.replay()
        torch.cuda.synchronize()
        got = [t.clone() for t in out]
        for x, y, name in zip(got, tr.eval(p, c), ("losses", "T", "pooled")):
            assert _same(x, y), f"replay on batch {s}: {name} differ from the eager eval"


# ================================================================================================ _push_residual
TICKS = 8
SENTINEL = 1234.5


def _frame(pool, s, k):
    """Stream s's frame at tick k: consecutive pool scans, turned by a small seeded yaw per stream."""
    base = pool[(s + k) % len(pool)]
    yaw = math.radians(((s * 7919) % 7) * 0.25)
    c, si = math.cos(yaw), math.sin(yaw)
    rot = torch.tensor([[c, -si, 0.0], [si, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
    return (rot @ base).contiguous()


def _pattern(S, seed):
    rng = np.random.default_rng(seed)
    act = rng.random((TICKS, S)) < 0.75
    act[:2, S - 1] = False                  # a late start; at S = 1 tick 0 only caches the first frame later
    act[3, :] = False                       # a tick without any active stream
    act[4, :] = True                        # the tick right after the reset
    act[5, :] = True
    return act, {4: [0]}


def _ticks(pool, S, n_stride, act):
    out = []
    for k in range(act.shape[0]):
        frames = [_frame(pool, s, k) if act[k, s] else _frame(pool, s + 3, k + 2) for s in range(S)]
        pts, counts = H.stack(frames, n_stride)         # inactive streams are staged with points: `active` masks them
        out.append((pts, counts, torch.from_numpy(act[k].astype(np.int32)).to(DEV)))
    return out


def _streams_setup(S, h=16, w=180, w_raw=256, seed=30):
    cfg = H.config(h, w, "tanh", False)
    blob = H.blob(H.model(cfg, seed, near_identity=True).eval(), cfg)
    pool = H.frames(h, w_raw, 6)
    n_stride = max(s.shape[1] for s in pool) + 32
    act, resets = _pattern(S, seed + S)
    return cfg, blob, n_stride, _ticks(pool, S, n_stride, act), act, resets


def _reset(st, S, streams):
    mask = torch.zeros((S,), dtype=torch.int32, device=DEV)
    mask[list(streams)] = 1
    st.reset(mask)


def _run_plain(st, ticks, resets):
    S = st.desc.max_batch
    T = torch.full((S, 16), SENTINEL, dtype=torch.float32, device=DEV)
    valid = torch.full((S,), 7, dtype=torch.int32, device=DEV)
    out = []
    for k, (p, c, a) in enumerate(ticks):
        if k in resets:
            _reset(st, S, resets[k])
        st.push(p, c, a, T, valid)
        out.append((T.clone(), valid.clone()))
    return out


def _run_residual(st, ticks, resets, graph=False):
    """-> per tick (T, valid, losses), with guard rows around `losses` checked after every tick."""
    S = st.desc.max_batch
    pts, counts, active = (torch.zeros_like(t) for t in ticks[0])
    T = torch.full((S, 16), SENTINEL, dtype=torch.float32, device=DEV)
    valid = torch.full((S,), 7, dtype=torch.int32, device=DEV)
    guarded = torch.full((S + 2, ops.LOSS_ROW), SENTINEL, dtype=torch.float32, device=DEV)
    losses = guarded[1:S + 1]
    g = None
    if graph:
        st.push(pts, counts, active, T, valid, losses)       # all inactive: changes no stream state
        valid.fill_(7)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            st.push(pts, counts, active, T, valid, losses)
    out = []
    for k, (p, c, a) in enumerate(ticks):
        if k in resets:
            _reset(st, S, resets[k])
        pts.copy_(p)
        counts.copy_(c)
        active.copy_(a)
        if g is not None:
            g.replay()
        else:
            st.push(pts, counts, active, T, valid, losses)
        out.append((T.clone(), valid.clone(), losses.clone()))
        assert bool((guarded[0] == SENTINEL).all()) and bool((guarded[S + 1] == SENTINEL).all()), \
            f"tick {k}: a write outside losses [S, LOSS_ROW]"
    return out


def _guarded_workspace(d):
    nbytes, guard = capi.ResidualStreamsWorkspace.workspace_bytes(d), 4096
    buf = torch.empty((nbytes + 2 * guard,), dtype=torch.uint8, device=DEV)
    pattern = torch.arange(guard, device=DEV).to(torch.uint8) ^ 0xA5
    buf[:guard] = pattern
    buf[guard + nbytes:] = pattern
    return buf, buf[guard:guard + nbytes], pattern


def _reference_rows(cfg, ticks, act, resets, out, flags):
    """The dense ICP operator alone, B = 1, on each valid (tick, stream): source = this frame's grids moved by the T the
    call returned, target = the stream's previous frame's grids -> {(k, s): row}; also checks valid against the history."""
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    S = act.shape[1]
    prev = [None] * S
    rows = {}
    for k, (p, c, _) in enumerate(ticks):
        for s in resets.get(k, []):
            prev[s] = None
        T, valid, _ = out[k]
        for s in range(S):
            ok = bool(act[k, s]) and prev[s] is not None
            assert int(valid[s]) == int(ok), f"tick {k} stream {s}: valid={int(valid[s])}, expected {int(ok)}"
            if not act[k, s]:
                continue
            _, _, pg, ng = ops.project_normals(p[s:s + 1], c[s:s + 1], h, w, hf, vf, ds["neighborhood_side_length"],
                                               cfg["epsilon_range"],
                                               cfg["min_num_points_in_neighborhood_to_determine_point_class"])
            if ok:
                rows[(k, s)] = ops.icp_dense_fwd_bwd(pg, ng, T[s:s + 1, :12].contiguous(), prev[s][0], prev[s][1], h, w,
                                                     hf, vf, float(cfg["lambda_po2pl"]), flags)[0][0]
            prev[s] = (pg, ng)
    return rows


def _check_rows(out, rows, S):
    assert len(rows) > 0
    matched = 0
    for k, (_, valid, losses) in enumerate(out):
        for s in range(S):
            if (k, s) in rows:
                assert _same(losses[s], rows[(k, s)]), \
                    f"tick {k} stream {s}: {losses[s].tolist()} != the operator alone {rows[(k, s)].tolist()}"
                matched += int(losses[s][3] > 0)
            else:
                assert float(losses[s].abs().max()) == 0.0, f"tick {k} stream {s}: an invalid row is not zero"
    assert matched > 0, "no valid row matched any pair: the comparison is empty"


@pytest.mark.parametrize("S,flags", [(1, ICP), (4, ICP), (4, ALL_ICP | ops.NORMAL_LINEAR)],
                         ids=["S1", "S4", "S4-all-losses-linear"])
def test_residual_rows_and_transforms(cuda_lib, S, flags):
    cfg, blob, n_stride, ticks, act, resets = _streams_setup(S)
    d = H.desc(cfg, n_stride, S)
    plain = _run_plain(capi.StreamsWorkspace(d, blob), ticks, resets)
    buf, ws, pattern = _guarded_workspace(d)
    st = capi.ResidualStreamsWorkspace(d, blob, capi.residual_params(cfg, flags), workspace=ws)
    out = _run_residual(st, ticks, resets)
    torch.cuda.synchronize()
    assert torch.equal(buf[:4096], pattern) and torch.equal(buf[4096 + ws.numel():], pattern), \
        "a write outside delora_odometry_streams_residual_workspace_bytes"
    for k, ((tp, vp), (tr, vr, _)) in enumerate(zip(plain, out)):
        assert torch.equal(vp, vr), f"tick {k}: valid differs from _streams_push"
        assert _same(tp, tr), f"tick {k}: T differs from _streams_push"
    # the first frames, the all-inactive tick 3 and the tick after the reset leave the ICP armed: later rows still match
    _check_rows(out, _reference_rows(cfg, ticks, act, resets, out, flags), S)


def test_residual_graph_replay_matches_eager(cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _streams_setup(4)
    d = H.desc(cfg, n_stride, 4)
    rp = capi.residual_params(cfg)
    eager = _run_residual(capi.ResidualStreamsWorkspace(d, blob, rp), ticks, resets)
    graphed = _run_residual(capi.ResidualStreamsWorkspace(d, blob, rp), ticks, resets, graph=True)
    for k, (e, g) in enumerate(zip(eager, graphed)):
        assert torch.equal(e[1], g[1]), f"tick {k}: valid differs"
        assert _same(e[0], g[0]) and _same(e[2], g[2]), f"tick {k}: the replay differs from the eager call"


def test_residual_at_64x720(cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _streams_setup(2, 64, 720, 1024, seed=31)
    d = H.desc(cfg, n_stride, 2)
    plain = _run_plain(capi.StreamsWorkspace(d, blob), ticks, resets)
    out = _run_residual(capi.ResidualStreamsWorkspace(d, blob, capi.residual_params(cfg)), ticks, resets)
    for k, ((tp, vp), (tr, vr, _)) in enumerate(zip(plain, out)):
        assert torch.equal(vp, vr) and _same(tp, tr), f"tick {k}: T / valid differ from _streams_push"
    _check_rows(out, _reference_rows(cfg, ticks, act, resets, out, ICP), 2)


def test_python_class_returns_the_rows_beside_the_same_transforms(cuda_lib):
    from delora_b200.deploy.stream import OdometryStreams
    cfg = H.config(16, 180)
    model = H.model(cfg, 32, near_identity=True).eval()
    pool = H.frames(16, 256, 6)
    n_max = max(s.shape[1] for s in pool) + 32
    plain = OdometryStreams(model, cfg, "kitti", 2, n_max)
    scored = OdometryStreams(model, cfg, "kitti", 2, n_max, residual=True)
    seen = 0
    for k in range(4):
        scans = [_frame(pool, 0, k), _frame(pool, 1, k) if k != 1 else None]
        for a, b in zip(plain.push(scans), scored.push(scans)):
            assert (a is None) == (b is None)
            if a is not None:
                t, row = b
                assert t.tobytes() == a.tobytes() and row.shape == (ops.LOSS_ROW,) and row[3] > 0
                seen += 1
    assert seen == 5            # stream 0 at ticks 1..3, stream 1 (idle at tick 1) at ticks 2 and 3


# ====================================================================================================== examples
def _export(tmp_path, cfg, model, n_stride):
    ckpt = os.path.join(tmp_path, "ckpt.pth")
    torch.save({"model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, ckpt)
    dlw = os.path.join(tmp_path, "model.dlw")
    r = subprocess.run([sys.executable, os.path.join(H.ROOT, "bin", "export_odometry_weights.py"), "--checkpoint", ckpt,
                        "--out", dlw, "--n_stride", str(n_stride), "--max_batch", "2"], capture_output=True, text=True,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    return dlw


def _scan_dir(tmp_path, name, indices, vfov):
    from delora_b200 import synthetic
    dname = os.path.join(tmp_path, name)
    os.makedirs(dname)
    for i, index in enumerate(indices):
        synthetic.kitti_bin_scan(index, vfov_deg=vfov).tofile(os.path.join(dname, f"{i:06d}.bin"))
    return dname


def test_streams_example_prints_the_residual(cuda_lib, tmp_path):
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, vfov=vfov, layers=(1, 1, 1, 1))
    dlw = _export(tmp_path, cfg, H.model(cfg, 5, near_identity=True).eval(), 4096)
    dirs = [_scan_dir(tmp_path, "stream0", (0, 1, 2), vfov), _scan_dir(tmp_path, "stream1", (10, 11), vfov)]
    exe = H.build_example("odometry_streams", tmp_path, link=True)
    plain = subprocess.run([exe, dlw] + dirs, capture_output=True, text=True, timeout=300)
    scored = subprocess.run([exe, "--residual", dlw] + dirs, capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and scored.returncode == 0, plain.stderr + scored.stderr
    a = [line.split() for line in plain.stdout.strip().splitlines()]
    b = [line.split() for line in scored.stdout.strip().splitlines()]
    assert [x[:14] for x in b] == a and len(a) == 3           # the same transforms, then po2pl, pl2pl, matched pairs
    for x in b:
        assert len(x) == 17 and float(x[16]) > 0 and math.isfinite(float(x[14])) and math.isfinite(float(x[15]))


def test_train_example_scores_a_held_out_directory(cuda_lib, tmp_path):
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, vfov=vfov, layers=(1, 1, 1, 1))
    dlw = _export(tmp_path, cfg, H.model(cfg, 6, near_identity=True), 4096)
    train = _scan_dir(tmp_path, "train", (0, 1, 2), vfov)
    held = _scan_dir(tmp_path, "held", (20, 21, 22), vfov)
    exe = H.build_example("odometry_train", tmp_path, link=True)
    scans = sorted(os.path.join(train, f) for f in os.listdir(train))
    out_a, out_b = os.path.join(tmp_path, "a.dlt"), os.path.join(tmp_path, "b.dlt")
    plain = subprocess.run([exe, dlw, out_a, "2", "2"] + scans, capture_output=True, text=True, timeout=600)
    scored = subprocess.run([exe, "--eval-dir", held, dlw, out_b, "2", "2"] + scans, capture_output=True, text=True,
                            timeout=600)
    assert plain.returncode == 0 and scored.returncode == 0, plain.stderr + scored.stderr
    pl, sc = plain.stdout.strip().splitlines(), scored.stdout.strip().splitlines()
    assert len(pl) == len(sc) == 2
    for x, y in zip(pl, sc):
        assert y.startswith(x) and "held-out" in y[len(x):]
        assert math.isfinite(float(y.split()[-1]))
    # the evaluation changed nothing the training writes
    assert open(out_a, "rb").read() == open(out_b, "rb").read()
