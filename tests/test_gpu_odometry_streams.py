"""Batched streaming odometry through the C ABI (delora_odometry_streams_*) on the H100.

Every stream's T row is byte-equal to a delora_odometry_push workspace fed only that stream's active frames, over a
seeded activity pattern with idle ticks, all-active ticks, a late start, a reset, an empty frame and a count above
n_stride.  Inactive streams are staged with another stream's points and a non-zero count, so the mask is what keeps
them out."""
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200.deploy.capi import InferenceWorkspace, StreamsWorkspace
from helpers import ROOT

pytestmark = pytest.mark.gpu
DEV = H.DEV
TICKS = 8


def _frame(pool, s, k):
    """Stream s's frame at tick k: a pool scan turned by a seeded yaw (distinct per stream and tick)."""
    base = pool[(2 * s + k) % len(pool)]
    yaw = math.radians(((s * 7919 + k * 104729) % 360) * 0.5)
    c, si = math.cos(yaw), math.sin(yaw)
    rot = torch.tensor([[c, -si, 0.0], [si, c, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
    return (rot @ base).contiguous()


def _pattern(S, seed):
    """active [TICKS, S] bool, per-(tick, stream) count overrides, resets {tick: [streams]} applied before the tick."""
    rng = np.random.default_rng(seed)
    act = rng.random((TICKS, S)) < 0.7
    act[:3, S - 1] = False                  # a stream that starts late
    act[2, :] = False                       # a tick without any active stream
    act[5, :] = True                        # a tick with all streams active
    override = {(3, 1 % S): "empty", (6, 0): "over"}
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


def _push_reference(cfg, n_stride, blob, ticks, act, resets):
    """Per stream, one delora_odometry_push workspace fed only that stream's active frames -> {(k, s): T bytes}."""
    t = torch.empty((16,), dtype=torch.float32, device=DEV)
    want = {}
    S = act.shape[1]
    for s in range(S):
        ws = InferenceWorkspace(H.desc(cfg, n_stride, 1), blob)
        has = False
        for k, (pts, counts, _) in enumerate(ticks):
            if s in resets.get(k, []):
                has = False
            if not act[k, s]:
                continue
            p = pts[s:s + 1].to(DEV)
            c = counts[s:s + 1].to(DEV)
            ws.push(p, c, t if has else None)
            if has:
                want[(k, s)] = t.clone()
            has = True
    torch.cuda.synchronize()
    return {key: v.cpu() for key, v in want.items()}


SENTINEL = H.SENTINEL


def _check_against_push(out, want, act, resets):
    S = act.shape[1]
    expect_T = torch.full((S, 16), SENTINEL, dtype=torch.float32)
    has = [False] * S
    n_valid = 0
    for k, (T, valid) in enumerate(out):
        for s in resets.get(k, []):
            has[s] = False
        for s in range(S):
            ok = bool(act[k, s]) and has[s]
            assert int(valid[s]) == int(ok), f"tick {k} stream {s}: valid={int(valid[s])}, expected {int(ok)}"
            if ok:
                expect_T[s] = want[(k, s)]
                n_valid += 1
            if act[k, s]:
                has[s] = True
        assert torch.equal(H.bits(T), H.bits(expect_T)), f"tick {k}: T differs from the per-stream pushes"
    return n_valid


SIZES = [(64, 2048, 2048), (64, 720, 1024), (64, 2047, 2048)]     # H, W, w_raw; W odd: the 64-channel stem path


@pytest.mark.parametrize("S", [1, 3, 16])
@pytest.mark.parametrize("act_fn", ["tanh", "relu"])
@pytest.mark.parametrize("h,w,w_raw", SIZES)
def test_rows_are_bit_identical_to_push(cuda_lib, h, w, w_raw, act_fn, S):
    cfg = H.config(h, w, act_fn)
    blob = H.blob(H.model(cfg).eval(), cfg)
    pool = H.frames(h, w_raw, 6)
    n_stride = max(s.shape[1] for s in pool) + 64
    act, override, resets = _pattern(S, seed=S * 31 + w)
    ticks = _ticks(pool, S, n_stride, act, override)
    want = _push_reference(cfg, n_stride, blob, ticks, act, resets)
    out = H.run_streams(StreamsWorkspace(H.desc(cfg, n_stride, S), blob), ticks, resets=resets)
    assert _check_against_push(out, want, act, resets) == len(want) > 0


@pytest.mark.parametrize("act_fn", ["tanh", "relu"])
def test_single_mlp_head_rows_are_bit_identical_to_push(cuda_lib, act_fn):
    cfg = H.config(64, 720, act_fn, single=True)
    blob = H.blob(H.model(cfg, 2).eval(), cfg)
    pool = H.frames(64, 1024, 6)
    n_stride = max(s.shape[1] for s in pool) + 64
    act, override, resets = _pattern(3, seed=5)
    ticks = _ticks(pool, 3, n_stride, act, override)
    want = _push_reference(cfg, n_stride, blob, ticks, act, resets)
    out = H.run_streams(StreamsWorkspace(H.desc(cfg, n_stride, 3), blob), ticks, resets=resets)
    assert _check_against_push(out, want, act, resets) == len(want) > 0


def _small_setup(S=4, w=720, seed=9):
    cfg = H.config(64, w)
    blob = H.blob(H.model(cfg, 1).eval(), cfg)
    pool = H.frames(64, 1024, 6)
    n_stride = max(s.shape[1] for s in pool) + 64
    act, override, resets = _pattern(S, seed=seed)
    return cfg, blob, n_stride, _ticks(pool, S, n_stride, act, override), act, resets


def test_graph_replay_matches_eager(cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _small_setup()
    eager = H.run_streams(StreamsWorkspace(H.desc(cfg, n_stride, 4), blob), ticks, resets=resets)
    graphed = H.run_streams(StreamsWorkspace(H.desc(cfg, n_stride, 4), blob), ticks, resets=resets, graph=True)
    for k, ((te, ve), (tg, vg)) in enumerate(zip(eager, graphed)):
        assert torch.equal(ve, vg), f"tick {k}: valid differs"
        assert torch.equal(H.bits(te), H.bits(tg)), f"tick {k}: graph replay differs from the eager call"


def test_deterministic(cuda_lib):
    cfg, blob, n_stride, ticks, act, resets = _small_setup(S=3, seed=4)
    a = H.run_streams(StreamsWorkspace(H.desc(cfg, n_stride, 3), blob), ticks, resets=resets)
    b = H.run_streams(StreamsWorkspace(H.desc(cfg, n_stride, 3), blob), ticks, resets=resets)
    for (ta, va), (tb, vb) in zip(a, b):
        assert torch.equal(va, vb) and torch.equal(H.bits(ta), H.bits(tb))


def test_null_active_means_all_active(cuda_lib):
    cfg, blob, n_stride, ticks, _, _ = _small_setup(S=3, seed=6)
    all_on = [(p, c, torch.ones_like(a)) for p, c, a in ticks[:3]]
    a = H.run_streams(StreamsWorkspace(H.desc(cfg, n_stride, 3), blob), all_on)
    st = StreamsWorkspace(H.desc(cfg, n_stride, 3), blob)
    T = torch.full((3, 16), SENTINEL, device=DEV)
    valid = torch.zeros((3,), dtype=torch.int32, device=DEV)
    for k, (p, c, _) in enumerate(all_on):
        st.push(p.to(DEV), c.to(DEV), None, T, valid)
        torch.cuda.synchronize()
        assert torch.equal(valid.cpu(), a[k][1]) and torch.equal(H.bits(T.cpu()), H.bits(a[k][0]))


def test_inactive_stream_keeps_its_cached_frame(cuda_lib):
    """Stream 1 sits out ticks 1..3 while the others run; at tick 4 it continues from its tick-0 frame."""
    cfg = H.config(64, 720)
    blob = H.blob(H.model(cfg, 3).eval(), cfg)
    pool = H.frames(64, 1024, 6)
    n_stride = max(s.shape[1] for s in pool) + 64
    act = np.ones((5, 3), dtype=bool)
    act[1:4, 1] = False
    ticks = _ticks(pool, 3, n_stride, act, {})
    out = H.run_streams(StreamsWorkspace(H.desc(cfg, n_stride, 3), blob), ticks)
    assert [int(v[1]) for _, v in out] == [0, 0, 0, 0, 1]
    want = _push_reference(cfg, n_stride, blob, [ticks[0], ticks[4]], act[[0, 4]], {})
    assert torch.equal(H.bits(out[4][0][1]), H.bits(want[(1, 1)]))
    assert torch.equal(H.bits(out[3][0][1]), H.bits(torch.full((16,), SENTINEL)))     # untouched while inactive


@pytest.mark.parametrize("w", [720, 2047])
def test_workspace_bounds(cuda_lib, w):
    cfg, blob, n_stride, ticks, act, resets = _small_setup(S=3, w=w, seed=8)
    d = H.desc(cfg, n_stride, 3)
    ws, intact = H.guarded_workspace(StreamsWorkspace.workspace_bytes(d))
    H.run_streams(StreamsWorkspace(d, blob, workspace=ws), ticks, resets=resets)
    assert intact(), "a streams call wrote outside delora_odometry_streams_workspace_bytes"


@pytest.mark.parametrize("use_graph", [True, False])
def test_python_class_matches_push_and_the_torch_stream(cuda_lib, use_graph):
    from delora_b200.deploy.stream import OdometryStream, OdometryStreams
    cfg = H.config(64, 720)
    model = H.model(cfg, 4).eval()
    blob = H.blob(model, cfg)
    pool = H.frames(64, 1024, 6)
    n_max = max(s.shape[1] for s in pool) + 64
    S = 3
    act = np.ones((6, S), dtype=bool)
    act[1, 0] = False
    act[:2, 2] = False
    resets = {4: [1]}
    streams = OdometryStreams(model, cfg, "kitti", S, n_max, use_cuda_graph=use_graph)
    torch_streams = [OdometryStream(model, cfg, "kitti", n_max) for _ in range(S)]
    got = []
    for k in range(act.shape[0]):
        for s in resets.get(k, []):
            streams.reset(s)
            torch_streams[s].reset()
        scans = [_frame(pool, s, k) if act[k, s] else None for s in range(S)]
        res = streams.push(scans)
        assert len(res) == S
        for s in range(S):
            ref = torch_streams[s].push(scans[s]) if scans[s] is not None else None
            assert (res[s] is None) == (ref is None), (k, s)
            if ref is not None:
                err = np.abs(res[s] - ref).max()
                assert err <= 1e-5 * max(1.0, np.abs(ref).max()), (k, s, err)
                assert res[s].shape == (1, 4, 4)
        got.append(res)
    # bit for bit against per-stream _push workspaces
    t = torch.empty((16,), dtype=torch.float32, device=DEV)
    for s in range(S):
        ws = InferenceWorkspace(H.desc(cfg, n_max, 1), blob)
        has = False
        for k in range(act.shape[0]):
            if s in resets.get(k, []):
                has = False
            if not act[k, s]:
                assert got[k][s] is None
                continue
            p, c = H.stack([_frame(pool, s, k)], n_max)
            ws.push(p, c, t if has else None)
            torch.cuda.synchronize()
            if has:
                assert got[k][s] is not None and got[k][s].tobytes() == t.cpu().numpy().tobytes(), (k, s)
            else:
                assert got[k][s] is None
            has = True
    for s in range(S):
        assert len(streams.poses(s)) == len(streams.relative[s]) + 1


def test_example_program(cuda_lib, tmp_path):
    """examples/odometry_streams.c on two stream directories of 3 and 2 KITTI .bin scans prints what _lib computes."""
    import sys
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, vfov=vfov, layers=(1, 1, 1, 1))
    model = H.model(cfg, 5).eval()
    ckpt = os.path.join(tmp_path, "ckpt.pth")
    torch.save({"model_state_dict": model.state_dict(), "parameters": dict(cfg, device="cpu")}, ckpt)
    dlw = os.path.join(tmp_path, "model.dlw")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "export_odometry_weights.py"), "--checkpoint", ckpt,
                        "--out", dlw, "--n_stride", "4096"], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
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
    printed = np.array([[float(v) for v in x[2:]] for x in lines], dtype=np.float64)

    _, d, blob = export.read_dlw(dlw)
    blob_dev = torch.from_numpy(blob).to(DEV)
    S = len(lengths)
    st = StreamsWorkspace(H.desc(cfg, d.n_stride, S), blob_dev)
    T = torch.zeros((S, 16), dtype=torch.float32, device=DEV)
    valid = torch.zeros((S,), dtype=torch.int32, device=DEV)
    want = []
    for k in range(max(lengths)):
        pts = torch.zeros((S, 3, d.n_stride), dtype=torch.float32)
        counts = torch.zeros((S,), dtype=torch.int32)
        active = torch.zeros((S,), dtype=torch.int32)
        for s in range(S):
            if k < lengths[s]:
                f = scans[s][k]
                pts[s, :, :f.shape[1]] = f
                counts[s] = f.shape[1]
                active[s] = 1
        st.push(pts.to(DEV), counts.to(DEV), active.to(DEV), T, valid)
        torch.cuda.synchronize()
        for s in range(S):
            if int(valid[s]):
                want.append(T[s].cpu().numpy()[:12].astype(np.float64))
    assert np.abs(printed - np.stack(want)).max() <= 1e-6
