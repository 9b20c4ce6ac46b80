"""Batched streaming of normalised models through the C ABI (delora_odometry_streams_push_normalized) on the H100.

Every valid stream's T row and factor are byte-equal to delora_odometry_pairs_normalized at B = 1 on (that stream's
previous active frame, this frame), over a seeded activity pattern with idle ticks, an all-active tick, a late start, a
reset and a count above n_stride.  Each stream's frames are scaled by a distinct factor that changes every tick, so a
row that used another stream's factor, or the previous tick's, would differ.  Inactive streams are staged with another
stream's points and a non-zero count, so the mask is what keeps them out."""
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200.deploy.capi import InferenceWorkspace, NormalizedStreamsWorkspace
from helpers import ROOT

pytestmark = pytest.mark.gpu
DEV = H.DEV
TICKS = 9
SENTINEL = H.SENTINEL


def _cfg(h, w, act="tanh", single=False, **kw):
    cfg = H.config(h, w, act, single, **kw)
    cfg["normalization_scaling"] = True
    return cfg


def _scale(s, k):
    """A distinct scale per stream and tick (not a power of two)."""
    return 0.6 + 0.37 * s + 0.11 * k


def _frame(pool, s, k):
    """Stream s's frame at tick k: a pool scan turned by a seeded yaw and scaled by _scale(s, k)."""
    base = pool[(2 * s + k) % len(pool)]
    yaw = math.radians(((s * 7919 + k * 104729) % 360) * 0.5)
    c, si = math.cos(yaw), math.sin(yaw)
    rot = torch.tensor([[c, -si, 0.0], [si, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
    return ((rot @ base) * _scale(s, k)).contiguous()


def _pattern(S, seed, empty=False):
    """active [TICKS, S] bool, per-(tick, stream) count overrides, resets {tick: [streams]} applied before the tick."""
    rng = np.random.default_rng(seed)
    act = rng.random((TICKS, S)) < 0.7
    act[:3, S - 1] = False                  # a stream that starts late
    act[2, :] = False                       # a tick without any active stream
    act[5, :] = True                        # a tick with all streams active
    override = {(6, 0): "over"}
    if empty:
        override[(3, 1 % S)] = "empty"
    for k, s in override:
        act[k, s] = True
    return act, override, {4: [0]}


def _ticks(pool, S, n_stride, act, override):
    """Host staging of every tick; inactive streams get another stream's scan and a real count."""
    def count(k, s, n):
        kind = override.get((k, s))
        return 0 if kind == "empty" else (n_stride + 1000 if kind == "over" else n)
    return H.stage_ticks(act, n_stride, lambda k, s: _frame(pool, s, k) if act[k, s] else _frame(pool, s + 11, k + 5),
                         count)


def _pairs_reference(cfg, n_stride, blobs, ticks, act, resets):
    """Per stream, delora_odometry_pairs_normalized at B = 1 on (its previous active frame, this frame), with the blob
    that is loaded at that tick (blobs: {first tick: blob}) -> {(k, s): (T [16], factor [1])}."""
    workspaces = {k0: InferenceWorkspace(H.desc(cfg, n_stride, 1), b) for k0, b in blobs.items()}
    want = {}
    for s in range(act.shape[1]):
        prev = None
        for k, (pts, counts, _) in enumerate(ticks):
            if s in resets.get(k, []):
                prev = None
            if not act[k, s]:
                continue
            if prev is not None:
                ws = workspaces[max(k0 for k0 in blobs if k0 <= k)]
                t, _, f = ws.pairs_normalized(torch.stack([prev[0], pts[s]]).to(DEV),
                                              torch.stack([prev[1], counts[s]]).to(DEV))
                want[(k, s)] = (t.reshape(16).clone(), f.clone())
            prev = (pts[s], counts[s])
    torch.cuda.synchronize()
    return {key: (t.cpu(), f.cpu()) for key, (t, f) in want.items()}


def _check(out, want, act, resets, skip=()):
    """valid, T and factor after every tick against the references; rows of (tick, stream) in skip are only checked
    for their valid flag.  -> the number of rows compared."""
    S = act.shape[1]
    expect_T = torch.full((S, 16), SENTINEL, dtype=torch.float32)
    has = [False] * S
    n = 0
    for k, (T, valid, factor) in enumerate(out):
        for s in resets.get(k, []):
            has[s] = False
        expect_f = torch.zeros((S,), dtype=torch.float32)
        for s in range(S):
            ok = bool(act[k, s]) and has[s]
            assert int(valid[s]) == int(ok), f"tick {k} stream {s}: valid={int(valid[s])}, expected {int(ok)}"
            if ok and (k, s) in skip:
                expect_T[s], expect_f[s] = T[s], factor[s]
            elif ok:
                expect_T[s], expect_f[s] = want[(k, s)][0], want[(k, s)][1][0]
                n += 1
            if act[k, s]:
                has[s] = True
        assert torch.equal(H.bits(T), H.bits(expect_T)), f"tick {k}: T differs from pairs_normalized at B = 1"
        assert torch.equal(H.bits(factor), H.bits(expect_f)), f"tick {k}: factor differs from pairs_normalized at B = 1"
    return n


def _setup(h, w, w_raw, S, act_fn="tanh", single=False, seed=0, empty=False, model_seed=0):
    cfg = _cfg(h, w, act_fn, single)
    blob = H.blob(H.model(cfg, model_seed).eval(), cfg)
    pool = H.frames(h, w_raw, 6)
    n_stride = max(s.shape[1] for s in pool) + 64
    act, override, resets = _pattern(S, seed, empty)
    return cfg, blob, n_stride, _ticks(pool, S, n_stride, act, override), act, resets


CASES = [(16, 180, 1024, "tanh", False), (16, 259, 1024, "relu", True)]    # W even / odd (channel-padded stem)


@pytest.mark.parametrize("S", [1, 3, 4])
@pytest.mark.parametrize("h,w,w_raw,act_fn,single", CASES)
def test_rows_are_bit_identical_to_pairs_normalized(cuda_lib, h, w, w_raw, act_fn, single, S):
    cfg, blob, n_stride, ticks, act, resets = _setup(h, w, w_raw, S, act_fn, single, seed=S * 31 + w)
    want = _pairs_reference(cfg, n_stride, {0: blob}, ticks, act, resets)
    out = H.run_streams(NormalizedStreamsWorkspace(H.desc(cfg, n_stride, S), blob), ticks, ("factor",), resets=resets)
    assert _check(out, want, act, resets) == len(want) > 0
    # the factors differ between streams and ticks: a row with another pair's factor could not have matched
    fs = [float(f[0]) for _, f in want.values()]
    assert len(set(fs)) == len(fs)


def test_rows_are_bit_identical_at_64x720(cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _setup(64, 720, 1024, 4, seed=3)
    want = _pairs_reference(cfg, n_stride, {0: blob}, ticks, act, resets)
    out = H.run_streams(NormalizedStreamsWorkspace(H.desc(cfg, n_stride, 4), blob), ticks, ("factor",), resets=resets)
    assert _check(out, want, act, resets) == len(want) > 0


def test_an_empty_frame_touches_only_its_own_pairs(cuda_lib):
    """Stream 1's frame at tick 3 is empty: its pairs with that frame (this one, if it has a previous frame, and the
    next one) are non-finite, as in pairs_normalized; every other row matches its reference."""
    S = 3
    cfg, blob, n_stride, ticks, act, resets = _setup(16, 180, 1024, S, seed=12, empty=True)
    want = _pairs_reference(cfg, n_stride, {0: blob}, ticks, act, resets)
    out = H.run_streams(NormalizedStreamsWorkspace(H.desc(cfg, n_stride, S), blob), ticks, ("factor",), resets=resets)
    # the pairs that hold the empty frame: tick 3 (this frame) and stream 1's next active tick (previous frame)
    nxt = next(k for k in range(4, TICKS) if act[k, 1])
    bad = {(k, 1) for k in (3, nxt) if (k, 1) in want}
    assert (nxt, 1) in bad
    for k, s in bad:
        T, valid, factor = out[k]
        assert int(valid[s]) == 1
        assert not torch.isfinite(factor[s]) and not torch.isfinite(T[s]).all(), (k, s)
    assert _check(out, want, act, resets, skip=bad) == len(want) - len(bad) > 0


def test_graph_replay_matches_the_direct_calls(cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _setup(16, 259, 1024, 4, seed=9)
    d = H.desc(cfg, n_stride, 4)
    eager = H.run_streams(NormalizedStreamsWorkspace(d, blob), ticks, ("factor",), resets=resets)
    graphed = H.run_streams(NormalizedStreamsWorkspace(d, blob), ticks, ("factor",), resets=resets, graph=True)
    for k, (e, g) in enumerate(zip(eager, graphed)):
        assert torch.equal(e[1], g[1]), f"tick {k}: valid differs"
        assert torch.equal(H.bits(e[0]), H.bits(g[0])), f"tick {k}: T differs under graph replay"
        assert torch.equal(H.bits(e[2]), H.bits(g[2])), f"tick {k}: factor differs under graph replay"


def test_load_weights_and_reset_act_as_on_the_streams_workspace(cuda_lib):
    """A second blob loaded mid-run through delora_odometry_streams_load_weights replaces the first for every later
    tick; the reset of the pattern (stream 0 before tick 4) restarts that stream."""
    S = 3
    cfg, blob, n_stride, ticks, act, resets = _setup(16, 180, 1024, S, seed=21)
    blob2 = H.blob(H.model(cfg, 7).eval(), cfg)
    want = _pairs_reference(cfg, n_stride, {0: blob, 5: blob2}, ticks, act, resets)
    out = H.run_streams(NormalizedStreamsWorkspace(H.desc(cfg, n_stride, S), blob), ticks, ("factor",), resets=resets,
                          loads={5: blob2})
    assert _check(out, want, act, resets) == len(want) > 0
    assert any(k >= 5 for k, _ in want), "no tick ran on the second blob"


def test_workspace_bounds(cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _setup(16, 259, 1024, 3, seed=8)
    d = H.desc(cfg, n_stride, 3)
    ws, intact = H.guarded_workspace(NormalizedStreamsWorkspace.workspace_bytes(d))
    H.run_streams(NormalizedStreamsWorkspace(d, blob, workspace=ws), ticks, ("factor",), resets=resets)
    assert intact(), "a call wrote outside delora_odometry_streams_normalized_workspace_bytes"


@pytest.mark.parametrize("use_graph", [True, False])
def test_python_class_returns_the_reference_transforms(cuda_lib, use_graph):
    from delora_b200.deploy.stream import NormalizedOdometryStreams
    cfg = _cfg(16, 180)
    model = H.model(cfg, 4).eval()
    blob = H.blob(model, cfg)
    pool = H.frames(16, 1024, 6)
    n_max = max(s.shape[1] for s in pool) + 64
    S = 3
    act = np.ones((6, S), dtype=bool)
    act[1, 0] = False
    act[:2, 2] = False
    resets = {4: [1]}
    streams = NormalizedOdometryStreams(model, cfg, "kitti", S, n_max, use_cuda_graph=use_graph)
    got = []
    for k in range(act.shape[0]):
        for s in resets.get(k, []):
            streams.reset(s)
        got.append(streams.push([_frame(pool, s, k) if act[k, s] else None for s in range(S)]))
    ws = InferenceWorkspace(H.desc(cfg, n_max, 1), blob)
    for s in range(S):
        prev = None
        for k in range(act.shape[0]):
            if s in resets.get(k, []):
                prev = None
            if not act[k, s]:
                assert got[k][s] is None
                continue
            cur = _frame(pool, s, k)
            if prev is None:
                assert got[k][s] is None, (k, s)
            else:
                t, _, _ = ws.pairs_normalized(*H.stack([prev, cur], n_max))
                torch.cuda.synchronize()
                assert got[k][s] is not None and got[k][s].shape == (1, 4, 4)
                assert got[k][s].tobytes() == t.cpu().numpy().tobytes(), (k, s)
            prev = cur
    for s in range(S):
        assert len(streams.poses(s)) == len(streams.relative[s]) + 1


def test_example_program_on_a_flagged_file(cuda_lib, tmp_path):
    """examples/odometry_streams.c on a .dlw exported from a normalization_scaling checkpoint, two stream directories
    of 3 and 2 KITTI .bin scans: the transforms of delora_odometry_pairs_normalized at B = 1; --residual is refused."""
    import sys
    from delora_b200 import _lib, synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = _cfg(16, 720, layers=(1, 1, 1, 1), vfov=vfov)
    model = H.model(cfg, 5).eval()
    ckpt = os.path.join(tmp_path, "ckpt.pth")
    torch.save({"model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, ckpt)
    dlw = os.path.join(tmp_path, "model.dlw")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "export_odometry_weights.py"), "--checkpoint", ckpt,
                        "--out", dlw, "--n_stride", "4096"], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    h, d, blob = export.read_dlw(dlw)
    assert h["model_flags"] == _lib.MODEL_NORMALIZATION_SCALING
    lengths = (3, 2)
    dirs, scans = [], []
    for s, n in enumerate(lengths):
        dname = os.path.join(tmp_path, f"stream{s}")
        os.makedirs(dname)
        dirs.append(dname)
        mine = []
        for i in range(n):
            path = os.path.join(dname, f"{i:06d}.bin")
            synthetic.kitti_bin_scan(10 * s + i, vfov_deg=vfov).tofile(path)
            mine.append(torch.from_numpy(np.fromfile(path, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()))
        scans.append(mine)
    exe = H.build_example("odometry_streams", tmp_path, link=True)
    r = subprocess.run([exe, dlw] + dirs, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lines = [line.split() for line in r.stdout.strip().splitlines()]
    assert [(int(x[0]), int(x[1])) for x in lines] == [(0, 1), (1, 1), (0, 2)]
    printed = np.array([[float(v) for v in x[2:]] for x in lines], dtype=np.float64).astype(np.float32)

    ws = InferenceWorkspace(H.desc(cfg, d.n_stride, 1), torch.from_numpy(blob).to(DEV))
    want = []
    for s, k in [(0, 1), (1, 1), (0, 2)]:
        t, _, _ = ws.pairs_normalized(*H.stack([scans[s][k - 1], scans[s][k]], d.n_stride))
        want.append(t[0].cpu().numpy().reshape(16)[:12])
    assert np.array_equal(printed, np.stack(want)), "the example's transforms differ from pairs_normalized"
    r = subprocess.run([exe, "--residual", dlw] + dirs, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "normalization_scaling" in r.stderr
