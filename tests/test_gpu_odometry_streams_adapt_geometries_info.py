"""-m gpu: the adapting streams of several sensor geometries with each frame's ICP information
(delora_odometry_streams_push_adapt_geometries_info) on the H100.  The geometries of
test_gpu_odometry_streams_adapt_geometries.py: 64 x 180 (w_pre 360) with S_0 = 2 streams and 64 x 128 (w_pre 128) with
S_1 = 3, one near-identity model.

- n = 1 is _push_adapt_info: T, valid, losses, info and the training state after every tick, over update 0 / 1 ticks
  with changing `active`;
- the information adds nothing else: T, valid, losses, the training state and the gradient section after an update tick
  are a _push_adapt_geometries workspace's bytes on the same frames;
- rows per geometry (lr 0, plain and normalization_scaling): T, valid, losses and info of geometry g are bit-identical
  to a _push_adapt_info workspace of d[g] holding the same weights; invalid rows are zeros, a fully inactive geometry's
  rows too, and the other geometry's rows are unchanged;
- before the update (lr > 0, update 1): tick k's rows are the information at tick k's served T, the rows of a
  _push_adapt_info workspace holding tick k's weights before its update;
- an information section filled with 0xFF bytes after init changes no output;
- repeated runs are bit-identical, and one captured tick per update value, replayed under changing masks and a reset,
  equals the eager calls;
- GeometriesAdaptiveOdometryStreams(information=True) returns the workspace's bits, and examples/odometry_streams.c
  --adapt with --geometry and --information prints the information columns for every stream and writes the .dlw
  the run without --information writes."""
import ctypes
import gc
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
GEOMS = ((64, 180, 360, 2), (64, 128, 128, 3))       # H, W, w_pre, S_g
S_ALL = sum(g[3] for g in GEOMS)
W_RAW = 512
ROWS = ("losses", "info")


def _cfg(h, w, w_pre, normalized=False):
    cfg = H.config(h, w)
    cfg["kitti"]["horizontal_cells_preprocessing"] = w_pre
    cfg["normalization_scaling"] = normalized
    return cfg


@pytest.fixture(scope="module")
def setup(cuda_lib):
    pool = H.frames(64, W_RAW, 8)
    n_stride = max(f.shape[1] for f in pool)
    cfg = _cfg(*GEOMS[0][:3])
    blob = H.blob(H.model(cfg, 21, near_identity=True), cfg)
    yield cfg, blob, pool, n_stride
    # the workspaces here are large: hand their memory back before the next module
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()


def _params(cfg, lr=LR, normalized=False):
    return capi.train_params(cfg, lr, loss_flags=ICP | (ops.TRAIN_NORMALIZATION_SCALING if normalized else 0))


def _descs(n_stride, geoms=GEOMS):
    return [H.desc(_cfg(h, w, wp), n_stride, S, wp) for h, w, wp, S in geoms]


def _multi(blob, n_stride, cfg, lr=LR, normalized=False, geoms=GEOMS, info=True):
    kind = capi.GeometriesAdaptingInformationStreamsWorkspace if info else capi.GeometriesAdaptingStreamsWorkspace
    return kind(_descs(n_stride, geoms), blob, _params(cfg, lr, normalized))


def _single(blob, n_stride, cfg, g, lr=LR, normalized=False, geoms=GEOMS):
    return capi.AdaptiveInformationStreamsWorkspace(_descs(n_stride, geoms)[g], blob, _params(cfg, lr, normalized))


def _tick(pool, n_stride, k, active, geoms=GEOMS):
    """Tick k: per geometry (points [S_g, 3, n], counts [S_g]) on the device, and active [S_total]; stream s serves
    pool[(3 s + k) % len(pool)] (s numbered over the whole fleet)."""
    pts, counts, s0 = [], [], 0
    for _, _, _, S in geoms:
        p = torch.zeros((S, 3, n_stride), dtype=torch.float32)
        c = torch.zeros((S,), dtype=torch.int32)
        for s in range(S):
            f = pool[(3 * (s0 + s) + k) % len(pool)]
            p[s, :, :f.shape[1]] = f
            c[s] = f.shape[1]
        pts.append(p.to(DEV))
        counts.append(c.to(DEV))
        s0 += S
    return pts, counts, torch.tensor(active, dtype=torch.int32, device=DEV)


def _push_multi(ws, tick, update, rows=ROWS):
    out = H.Outputs(ws.n_streams, rows)
    ws.push(*tick, *out.tensors, update=update)
    return out.snapshot()


def _push_single(ws, tick, g, update, geoms=GEOMS):
    pts, counts, active = tick
    r = sum(S for *_, S in geoms[:g])
    return H.run_streams(ws, [(pts[g], counts[g], active[r:r + geoms[g][3]])], ROWS, updates=[update])[0]


def _same_outputs(k, got, want, r0=0, info=True):
    """got: a fleet tick's (T, valid, losses[, info]), want: the reference's, whose rows start at r0 of got."""
    S = want[1].shape[0]
    assert H.same(got[1][r0:r0 + S], want[1]), f"tick {k}: valid"
    for s in range(S):
        if int(want[1][s]):
            assert H.same(got[0][r0 + s], want[0][s]), f"tick {k}, row {r0 + s}: T"
    assert H.same(got[2][r0:r0 + S], want[2]), f"tick {k}: losses"
    if info:
        assert H.same(got[3][r0:r0 + S], want[3]), f"tick {k}: info"


def _zero_where_invalid(k, out):
    for s in range(out[1].shape[0]):
        if not int(out[1][s]):
            assert float(out[3][s].abs().max()) == 0.0, f"tick {k}, row {s}: an invalid row is not zero"


def _grad(ws):
    """The gradient section of a training-layout workspace, copied to the host."""
    torch.cuda.synchronize()
    off = int(ws._L.delora_odometry_train_grad_offset(ctypes.byref(ws.desc)))
    return ws.workspace[off:off + 4 * ws.n].view(torch.float32).cpu().clone()


def test_one_geometry_is_push_adapt_info(setup):
    cfg, blob, pool, n_stride = setup
    geoms = GEOMS[:1]
    multi = _multi(blob, n_stride, cfg, geoms=geoms)
    single = _single(blob, n_stride, cfg, 0, geoms=geoms)
    for k, (u, a) in enumerate(zip([True, False, True, True, False, True], [[1, 1], [1, 0], [1, 1], [0, 0], [1, 1],
                                                                          [0, 1]])):
        tick = _tick(pool, n_stride, k, a, geoms)
        got = _push_multi(multi, tick, u)
        want = _push_single(single, tick, 0, u, geoms)
        _same_outputs(k, got, want)
        assert H.same_state(H.state(multi), H.state(single)), f"tick {k}: the training state"
    assert int(H.state(single)[3][0]) >= 2


def test_information_adds_nothing_else(setup):
    cfg, blob, pool, n_stride = setup
    info, plain = _multi(blob, n_stride, cfg), _multi(blob, n_stride, cfg, info=False)
    acts = [[1] * 5, [1, 1, 1, 0, 1], [1, 0, 1, 1, 1], [0, 0, 1, 1, 1], [1, 1, 1, 1, 1], [1, 1, 0, 0, 0]]
    updates = [False, True, True, False, True, True]
    mask = torch.tensor([0, 1, 0, 0, 1], dtype=torch.int32, device=DEV)
    for k, (u, a) in enumerate(zip(updates, acts)):
        if k == 4:
            info.reset(mask)
            plain.reset(mask)
        tick = _tick(pool, n_stride, k, a)
        got = _push_multi(info, tick, u)
        want = _push_multi(plain, tick, u, ("losses",))
        _same_outputs(k, got, want, info=False)
        _zero_where_invalid(k, got)
        assert H.same_state(H.state(info), H.state(plain)), f"tick {k}: the training state"
        if u:
            assert H.same(_grad(info), _grad(plain)), f"tick {k}: the gradient section"
    assert int(H.state(info)[3][0]) == 4


ACTS = [[1, 1, 1, 1, 1], [1, 1, 1, 0, 1], [0, 0, 1, 1, 1], [1, 1, 0, 0, 0], [1, 1, 1, 1, 1]]


@pytest.mark.parametrize("normalized", [False, True], ids=["plain", "normalized"])
def test_rows_are_the_single_geometry_info_rows(setup, normalized):
    cfg, blob, pool, n_stride = setup
    multi = _multi(blob, n_stride, cfg, lr=0.0, normalized=normalized)
    singles = [_single(blob, n_stride, cfg, g, lr=0.0, normalized=normalized) for g in range(len(GEOMS))]
    checked = 0
    for k, u in enumerate([False, True, False, True, True]):
        tick = _tick(pool, n_stride, k, ACTS[k])
        got = _push_multi(multi, tick, u)
        r0 = 0
        for g, ws in enumerate(singles):
            want = _push_single(ws, tick, g, u)
            _same_outputs(k, got, want, r0)
            r0 += GEOMS[g][3]
        _zero_where_invalid(k, got)
        if k == 2:                          # geometry 0 fully inactive
            assert float(got[3][:2].abs().max()) == 0.0 and int(got[1][2:].sum()) >= 2
        if k == 3:                          # geometry 1 fully inactive
            assert float(got[3][2:].abs().max()) == 0.0 and int(got[1][:2].sum()) == 2
        if normalized:
            f = got[2][:, 6]
            assert bool((f[got[1] != 0] > 0).all()) and float(f[got[1] == 0].abs().sum()) == 0.0
        checked += int((got[3][:, 78] > 0).sum())
    assert checked >= 10
    assert int(H.state(multi)[3][0]) == 3


def test_rows_are_taken_before_the_update(setup):
    cfg, blob, pool, n_stride = setup
    multi = _multi(blob, n_stride, cfg)
    singles = [_single(blob, n_stride, cfg, g) for g in range(len(GEOMS))]
    acts = [[1] * 5, [1] * 5, [1, 0, 1, 1, 1], [1] * 5]
    for k, a in enumerate(acts):
        before = H.state(multi)
        tick = _tick(pool, n_stride, k, a)
        got = _push_multi(multi, tick, True)
        after = H.state(multi)
        if k:
            assert not H.same(after[0], before[0]), f"tick {k}: the update did not move the weights"
        r0 = 0
        for g, ws in enumerate(singles):
            # tick k's weights before its update, then a serve-only tick on the same stream history
            ws.set_state(before[0], before[1], before[2], int(before[3][0]))
            want = _push_single(ws, tick, g, False)
            _same_outputs(k, got, want, r0)
            r0 += GEOMS[g][3]
        _zero_where_invalid(k, got)
    assert int(H.state(multi)[3][0]) == 3


def test_uninitialised_information_section(setup):
    cfg, blob, pool, n_stride = setup
    wss = [_multi(blob, n_stride, cfg) for _ in range(2)]
    base = capi.GeometriesAdaptingStreamsWorkspace.shared_bytes(wss[0].descs)
    end = wss[0].shared_bytes(wss[0].descs)
    assert end > base
    wss[0].workspace[base:end].fill_(0xFF)
    wss[1].workspace[base:end].zero_()
    for k, u in enumerate([False, True, True, False, True]):
        tick = _tick(pool, n_stride, k, ACTS[k])
        a, b = (_push_multi(ws, tick, u) for ws in wss)
        _same_outputs(k, a, b)
        assert H.same_state(H.state(wss[0]), H.state(wss[1])), f"tick {k}: the training state"


def test_determinism_and_graphs(setup):
    cfg, blob, pool, n_stride = setup
    acts = [[1, 1, 1, 1, 1], [1, 1, 0, 1, 1], [0, 1, 1, 1, 0], [1, 1, 1, 1, 1], [1, 0, 1, 0, 1], [1, 1, 1, 1, 1]]
    updates = [False, True, True, False, True, True]
    reset_at, mask_rows = 3, [0, 3]

    def bufs():
        return ([torch.zeros((g[3], 3, n_stride), dtype=torch.float32, device=DEV) for g in GEOMS],
                [torch.zeros((g[3],), dtype=torch.int32, device=DEV) for g in GEOMS],
                torch.zeros((S_ALL,), dtype=torch.int32, device=DEV)) + H.Outputs(S_ALL, ROWS).tensors

    def load(b, k):
        pts, counts, active = _tick(pool, n_stride, k, acts[k])
        for dst, src in zip(b[0] + b[1] + [b[2]], pts + counts + [active]):
            dst.copy_(src)

    def warm(ws, b):
        b[2].zero_()                           # all inactive: no stream state or weight changes
        for u in (False, True):
            ws.push(*b, update=u)
        torch.cuda.synchronize()

    mask = torch.zeros((S_ALL,), dtype=torch.int32, device=DEV)
    mask[mask_rows] = 1

    def run(replay=None):
        out = []
        for k, u in enumerate(updates):
            if k == reset_at:
                ws.reset(mask)
            load(b, k)
            if replay:
                replay[u].replay()
            else:
                ws.push(*b, update=u)
            torch.cuda.synchronize()
            out.append(tuple(t.cpu().clone() for t in b[3:]))
        return out, H.state(ws)

    runs = []
    for _ in range(2):
        ws, b = _multi(blob, n_stride, cfg), bufs()
        warm(ws, b)
        runs.append(run())
    first, second = runs
    for k, (x, y) in enumerate(zip(first[0], second[0])):
        _same_outputs(k, x, y)
    assert H.same_state(first[1], second[1])
    ws, b = _multi(blob, n_stride, cfg), bufs()
    warm(ws, b)
    graphs = {}
    for u in (False, True):
        graphs[u] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[u]):
            ws.push(*b, update=u)
    replayed = run(graphs)
    for k, (x, y) in enumerate(zip(replayed[0], first[0])):
        _same_outputs(k, x, y)
        _zero_where_invalid(k, x)
    assert H.same_state(replayed[1], first[1])
    assert int(first[1][3][0]) == 4
    assert first[0][reset_at][1][mask_rows].tolist() == [0, 0]


def test_python_class(setup):
    from delora_b200.deploy.stream import GeometriesAdaptiveOdometryStreams
    cfg, blob, pool, n_stride = setup
    model = H.model(cfg, 21, near_identity=True)
    cfg2 = _cfg(*GEOMS[0][:3])
    cfg2["kitti2"] = dict(cfg2["kitti"], vertical_cells=GEOMS[1][0], horizontal_cells=GEOMS[1][1],
                          horizontal_cells_preprocessing=GEOMS[1][2])
    geometries = [("kitti", GEOMS[0][3]), ("kitti2", GEOMS[1][3])]
    cls = GeometriesAdaptiveOdometryStreams(model, cfg2, geometries, n_stride, LR, preprocessing_normals=True,
                                            information=True)
    plain = GeometriesAdaptiveOdometryStreams(model, cfg2, geometries, n_stride, LR, preprocessing_normals=True)
    multi = _multi(blob, n_stride, cfg)
    seen = 0
    for k in range(3):
        act = ACTS[k]
        tick = _tick(pool, n_stride, k, act)
        want = _push_multi(multi, tick, True)
        scans, s0 = [], 0
        for g, (_, _, _, S) in enumerate(GEOMS):
            for s in range(S):
                n = int(tick[1][g][s])
                scans.append(tick[0][g][s, :, :n].cpu() if act[s0 + s] else None)
            s0 += S
        got, base = cls.push(scans), plain.push(scans)
        for s, (e, p) in enumerate(zip(got, base)):
            assert (e is None) == (not int(want[1][s])) == (p is None), (k, s)
            if e is not None:
                assert len(e) == 3 and len(p) == 2
                assert np.array_equal(e[0].reshape(16).view(np.int32), want[0][s].numpy().view(np.int32))
                assert np.array_equal(e[1].view(np.int32), want[2][s].numpy().view(np.int32))
                assert np.array_equal(e[2].view(np.int32), want[3][s].numpy().view(np.int32))
                assert np.array_equal(e[0], p[0]) and np.array_equal(e[1], p[1])
                seen += 1
    assert seen >= 6
    from delora_b200.deploy import export
    adapted = torch.from_numpy(export.pack_state_dict(cls.state_dict(), cls.config))
    assert torch.equal(multi.weights().cpu().view(torch.int32), adapted.view(torch.int32))


def test_example_information_with_two_geometries(cuda_lib, tmp_path):
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 180, "tanh", False, layers=(1, 1, 1, 1), nout=64)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    model = H.model(cfg, 6, near_identity=True)
    dlw = os.path.join(tmp_path, "m.dlw")
    export.write_dlw(dlw, export.desc_from_config(cfg, "kitti", 4096, 1), export.pack_state_dict(model.state_dict(), cfg))
    dirs = []
    for s in range(3):
        dd = os.path.join(tmp_path, f"stream{s}")
        os.makedirs(dd)
        dirs.append(dd)
        for i in range(3):
            synthetic.kitti_bin_scan(10 * s + i, vfov_deg=vfov).tofile(os.path.join(dd, f"{i:06d}.bin"))
    exe = H.build_example("odometry_streams", tmp_path, link=True)

    def run(out, extra):
        r = subprocess.run([exe, "--adapt", "1e-4", "--adapt-out", out, "--geometry", f"{dirs[1]},16,128,-15,15",
                            "--geometry", f"{dirs[2]},16,128,-15,15,256"] + extra + [dlw, dirs[0]],
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        return [ln.split() for ln in r.stdout.strip().splitlines()]

    plain_out, info_out = os.path.join(tmp_path, "a.dlw"), os.path.join(tmp_path, "a-info.dlw")
    plain, with_info = run(plain_out, []), run(info_out, ["--information"])
    assert len(plain) == len(with_info) == 3 * 2
    assert sorted({int(q[0]) for q in with_info}) == [0, 1, 2]
    for p, q in zip(plain, with_info):
        assert q[:len(p)] == p and len(q) == len(p) + 8, (p, q)
        assert abs(sum(float(x) ** 2 for x in q[len(p) + 1:len(p) + 7]) - 1) < 1e-4
    assert open(plain_out, "rb").read() == open(info_out, "rb").read()
    _, desc, blob_out = export.read_dlw(info_out)
    assert desc.H == 16 and desc.W == 180
    assert not np.array_equal(np.asarray(blob_out), export.pack_state_dict(model.state_dict(), cfg)), \
        "the model did not adapt"
