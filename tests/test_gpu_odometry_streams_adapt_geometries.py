"""-m gpu: one model adapted from the streams of several sensor geometries in one workspace
(delora_odometry_streams_push_adapt_geometries) on the H100.  Two synthetic 64-ring geometries with even W, 64 x 180
(w_pre 360) with S_0 = 2 streams and 64 x 128 (w_pre 128) with S_1 = 3, one near-identity model.

- n = 1 is _push_adapt: T, valid, losses and the training state after every tick, over update = 0 / 1 ticks;
- forward: geometry g's rows of T, valid and losses are bit-identical to a _push_adapt workspace of d[g] holding the
  same weights (lr 0, so every tick serves them), with update 0 and 1, plain and with normalization_scaling (whose
  loss rows carry each pair's factor);
- update: the gradient section after one update tick is sum_g N_g G_g / N within the harness's gradient bounds, G_g
  the gradient of a _push_adapt tick of d[g] alone; the weights, m and v are torch's Adam on that gradient;
- activity: a fully inactive geometry leaves the other geometry's _push_adapt update; a tick without a valid pair
  changes no state; a reset of one stream of geometry 1 changes no other row;
- repeated runs are bit-identical, and one captured tick per update value, replayed under changing masks, equals the
  eager calls;
- GeometriesAdaptiveOdometryStreams returns the workspace's bits;
- examples/odometry_streams.c --adapt with --geometry serves two geometries and writes a .dlw export.py reads."""
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
W_RAW = 512


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


def _params(cfg, lr=LR, normalized=False, beta1=0.9):
    return capi.train_params(cfg, lr, loss_flags=ICP | (ops.TRAIN_NORMALIZATION_SCALING if normalized else 0),
                             beta1=beta1)


def _descs(n_stride, geoms=GEOMS):
    return [H.desc(_cfg(h, w, wp), n_stride, S, wp) for h, w, wp, S in geoms]


def _multi(blob, n_stride, cfg, lr=LR, normalized=False, geoms=GEOMS):
    return capi.GeometriesAdaptingStreamsWorkspace(_descs(n_stride, geoms), blob, _params(cfg, lr, normalized))


def _single(blob, n_stride, cfg, g, lr=LR, normalized=False, geoms=GEOMS):
    return capi.AdaptiveStreamsWorkspace(_descs(n_stride, geoms)[g], blob, _params(cfg, lr, normalized))


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


def _outs(S):
    return (torch.full((S, 16), 1234.5, dtype=torch.float32, device=DEV),
            torch.full((S,), 7, dtype=torch.int32, device=DEV),
            torch.full((S, ops.LOSS_ROW), 1234.5, dtype=torch.float32, device=DEV))


def _push_multi(ws, tick, update):
    pts, counts, active = tick
    out = _outs(ws.n_streams)
    ws.push(pts, counts, active, *out, update=update)
    torch.cuda.synchronize()
    return tuple(t.cpu() for t in out)


def _push_single(ws, tick, g, update, geoms=GEOMS):
    pts, counts, active = tick
    r = sum(S for *_, S in geoms[:g])
    S = geoms[g][3]
    out = _outs(S)
    ws.push(pts[g], counts[g], active[r:r + S].contiguous(), *out, update=update)
    torch.cuda.synchronize()
    return tuple(t.cpu() for t in out)


def _same_rows(k, got, want, r0, geoms=GEOMS):
    """got: a fleet tick's outputs, want: a single geometry's, whose rows start at r0."""
    S = want[1].shape[0]
    assert H.same(got[1][r0:r0 + S], want[1]), f"tick {k}: valid"
    for s in range(S):
        if int(want[1][s]):
            assert H.same(got[0][r0 + s], want[0][s]), f"tick {k}, row {r0 + s}: T"
    assert H.same(got[2][r0:r0 + S], want[2]), f"tick {k}: losses"


def _grad(ws):
    """The gradient section of a training-layout workspace, copied to the host."""
    torch.cuda.synchronize()
    off = int(ws._L.delora_odometry_train_grad_offset(ctypes.byref(ws.desc)))
    return ws.workspace[off:off + 4 * ws.n].view(torch.float32).cpu().clone()


def test_one_geometry_is_push_adapt(setup):
    cfg, blob, pool, n_stride = setup
    geoms = GEOMS[:1]
    multi = _multi(blob, n_stride, cfg, geoms=geoms)
    single = _single(blob, n_stride, cfg, 0, geoms=geoms)
    assert multi.shared_bytes(multi.descs) == capi.AdaptiveStreamsWorkspace.workspace_bytes(single.desc)
    for k, (u, a) in enumerate(zip([True, False, True, True, False, True], [[1, 1], [1, 0], [1, 1], [0, 0], [1, 1],
                                                                          [0, 1]])):
        tick = _tick(pool, n_stride, k, a, geoms)
        got = _push_multi(multi, tick, u)
        want = _push_single(single, tick, 0, u, geoms)
        _same_rows(k, got, want, 0, geoms)
        assert H.same_state(H.state(multi), H.state(single)), f"tick {k}: the training state"
    assert int(H.state(single)[3][0]) >= 2


ACTS = [[1, 1, 1, 1, 1], [1, 1, 1, 0, 1], [1, 0, 1, 1, 1], [1, 1, 1, 1, 1]]


@pytest.mark.parametrize("normalized", [False, True], ids=["plain", "normalized"])
def test_rows_are_the_single_geometry_rows(setup, normalized):
    cfg, blob, pool, n_stride = setup
    multi = _multi(blob, n_stride, cfg, lr=0.0, normalized=normalized)
    singles = [_single(blob, n_stride, cfg, g, lr=0.0, normalized=normalized) for g in range(len(GEOMS))]
    for k, u in enumerate([False, True, False, True]):
        tick = _tick(pool, n_stride, k, ACTS[k])
        got = _push_multi(multi, tick, u)
        r0 = 0
        for g, ws in enumerate(singles):
            want = _push_single(ws, tick, g, u)
            _same_rows(k, got, want, r0)
            r0 += GEOMS[g][3]
        if k:
            assert int(got[1].sum()) >= 3
        if normalized:
            f = got[2][:, 6]
            assert bool((f[got[1] != 0] > 0).all()) and float(f[got[1] == 0].abs().sum()) == 0.0
    assert int(H.state(multi)[3][0]) == 2


def test_update_is_the_fleet_mean(setup):
    cfg, blob, pool, n_stride = setup
    acts = [ACTS[0], [1, 0, 1, 1, 1]]
    singles = [_single(blob, n_stride, cfg, g, lr=0.0) for g in range(len(GEOMS))]
    multi = _multi(blob, n_stride, cfg)
    before = H.state(multi)
    want, counts = torch.zeros_like(before[0]), []
    for k in range(2):
        tick = _tick(pool, n_stride, k, acts[k])
        got = _push_multi(multi, tick, k == 1)
        for g, ws in enumerate(singles):
            one = _push_single(ws, tick, g, k == 1)
            if k == 1:
                counts.append(int(one[1].sum()))
    N = sum(counts)
    assert counts == [1, 3] and int(got[1].sum()) == N
    for g, ws in enumerate(singles):
        want += _grad(ws) * counts[g]
    want /= N
    grad = _grad(multi)
    tail, trunk = H.grad_spread(H.grad_dict(grad, cfg), H.grad_dict(want, cfg))
    print(f"\n[fleet mean] tail {tail:.2e}  trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL and trunk <= H.TRUNK_TOL, (tail, trunk)
    # torch's Adam (fp32, as the kernel) on the gradient the tick left in the gradient section
    p = torch.nn.Parameter(before[0].clone())
    opt = torch.optim.Adam([p], lr=LR, betas=(0.9, 0.999), eps=1e-8)
    p.grad = grad.clone()
    opt.step()
    w, m, v, step = H.state(multi)
    st = opt.state[p]
    assert int(step[0]) == 1
    assert torch.allclose(m, st["exp_avg"], rtol=1e-5, atol=0.0)
    # v: the kernel rounds 1 - beta2 to fp32 (0.00099998713), torch multiplies by the double 0.001: 1.3e-5 apart
    assert torch.allclose(v, st["exp_avg_sq"], rtol=5e-5, atol=1e-30)
    assert float((w - p.detach()).abs().max()) <= 1e-3 * LR
    assert float((w - before[0]).abs().max()) > 0.5 * LR


@pytest.mark.parametrize("idle", [0, 1])
def test_an_idle_geometry_leaves_the_other_ones_update(setup, idle):
    cfg, blob, pool, n_stride = setup
    other = 1 - idle
    multi = _multi(blob, n_stride, cfg)
    single = _single(blob, n_stride, cfg, other)
    r_idle = sum(S for *_, S in GEOMS[:idle])
    r_other = sum(S for *_, S in GEOMS[:other])
    for k in range(3):
        act = [1] * 5
        for s in range(GEOMS[idle][3]):
            act[r_idle + s] = 0
        tick = _tick(pool, n_stride, k, act)
        got = _push_multi(multi, tick, True)
        want = _push_single(single, tick, other, True)
        _same_rows(k, got, want, r_other)
        a, b = H.state(multi), H.state(single)
        assert H.same(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and torch.equal(a[3], b[3]), \
            f"tick {k}: the state differs from geometry {other}'s _push_adapt"
    assert int(H.state(multi)[3][0]) == 2


def test_no_pair_no_update_and_reset(setup):
    cfg, blob, pool, n_stride = setup
    multi = _multi(blob, n_stride, cfg)
    before = H.state(multi)
    out = _push_multi(multi, _tick(pool, n_stride, 0, [1] * 5), True)
    assert int(out[1].sum()) == 0
    assert H.same_state(H.state(multi), before), "an update without a valid pair changed the training state"
    # a reset of stream 1 of geometry 1 (row 3) changes only that row
    ref = _multi(blob, n_stride, cfg)
    _push_multi(ref, _tick(pool, n_stride, 0, [1] * 5), False)
    mask = torch.tensor([0, 0, 0, 1, 0], dtype=torch.int32, device=DEV)
    multi.reset(mask)
    tick = _tick(pool, n_stride, 1, [1] * 5)
    got, want = _push_multi(multi, tick, False), _push_multi(ref, tick, False)
    assert got[1].tolist() == [1, 1, 1, 0, 1] and want[1].tolist() == [1] * 5
    for s in range(5):
        if s == 3:
            assert float(got[2][s].abs().max()) == 0.0
            continue
        assert H.same(got[0][s], want[0][s]) and H.same(got[2][s], want[2][s]), f"row {s}"


def test_determinism_and_graphs(setup):
    cfg, blob, pool, n_stride = setup
    acts = [[1, 1, 1, 1, 1], [1, 1, 0, 1, 1], [0, 1, 1, 1, 0], [1, 1, 1, 1, 1], [1, 0, 1, 0, 1]]
    updates = [False, True, True, False, True]
    S = sum(g[3] for g in GEOMS)

    def bufs():
        return ([torch.zeros((g[3], 3, n_stride), dtype=torch.float32, device=DEV) for g in GEOMS],
                [torch.zeros((g[3],), dtype=torch.int32, device=DEV) for g in GEOMS],
                torch.zeros((S,), dtype=torch.int32, device=DEV)) + _outs(S)

    def load(b, k):
        pts, counts, active = _tick(pool, n_stride, k, acts[k])
        for dst, src in zip(b[0] + b[1] + [b[2]], pts + counts + [active]):
            dst.copy_(src)

    def warm(ws, b):
        b[2].zero_()                           # all inactive: no stream state or weight changes
        for u in (False, True):
            ws.push(*b, update=u)
        torch.cuda.synchronize()

    def eager():
        ws, b = _multi(blob, n_stride, cfg), bufs()
        warm(ws, b)
        out = []
        for k, u in enumerate(updates):
            load(b, k)
            ws.push(*b, update=u)
            torch.cuda.synchronize()
            out.append(tuple(t.cpu().clone() for t in b[3:]))
        return out, H.state(ws)

    first, second = eager(), eager()
    for k, (x, y) in enumerate(zip(first[0], second[0])):
        assert all(H.same(a, b) for a, b in zip(x, y)), f"tick {k}: runs differ"
    assert H.same_state(first[1], second[1])
    ws, b = _multi(blob, n_stride, cfg), bufs()
    warm(ws, b)
    graphs = {}
    for u in (False, True):
        graphs[u] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[u]):
            ws.push(*b, update=u)
    for k, u in enumerate(updates):
        load(b, k)
        graphs[u].replay()
        torch.cuda.synchronize()
        valid = b[4].cpu()
        assert H.same(valid, first[0][k][1]), f"tick {k}: valid"
        for s in range(S):
            if int(valid[s]):
                assert H.same(b[3][s].cpu(), first[0][k][0][s]), f"tick {k}, row {s}: T"
        assert H.same(b[5].cpu(), first[0][k][2]), f"tick {k}: losses"
    assert H.same_state(H.state(ws), first[1])
    assert int(first[1][3][0]) == 3           # ticks 1, 2 and 4 update


def test_python_class(setup):
    from delora_b200.deploy.stream import GeometriesAdaptiveOdometryStreams
    cfg, blob, pool, n_stride = setup
    model = H.model(cfg, 21, near_identity=True)
    cfg2 = _cfg(*GEOMS[0][:3])
    cfg2["kitti2"] = dict(cfg2["kitti"], vertical_cells=GEOMS[1][0], horizontal_cells=GEOMS[1][1],
                          horizontal_cells_preprocessing=GEOMS[1][2])
    cls = GeometriesAdaptiveOdometryStreams(model, cfg2, [("kitti", GEOMS[0][3]), ("kitti2", GEOMS[1][3])], n_stride,
                                            LR, preprocessing_normals=True)
    multi = _multi(blob, n_stride, cfg)
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
        got = cls.push(scans)
        for s, e in enumerate(got):
            assert (e is None) == (not int(want[1][s])), (k, s)
            if e is not None:
                assert np.array_equal(e[0].reshape(16).view(np.int32), want[0][s].numpy().view(np.int32))
                assert np.array_equal(e[1].view(np.int32), want[2][s].numpy().view(np.int32))
    from delora_b200.deploy import export
    adapted = torch.from_numpy(export.pack_state_dict(cls.state_dict(), cls.config))
    assert torch.equal(multi.weights().cpu().view(torch.int32), adapted.view(torch.int32))


def test_example_serves_two_geometries(cuda_lib, tmp_path):
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
    out = os.path.join(tmp_path, "a.dlw")
    r = subprocess.run([exe, "--adapt", "1e-4", "--adapt-out", out, "--geometry", f"{dirs[1]},16,128,-15,15",
                        "--geometry", f"{dirs[2]},16,128,-15,15,256", dlw, dirs[0]], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    assert len(lines) == 3 * 2, r.stdout
    assert sorted({int(line.split()[0]) for line in lines}) == [0, 1, 2]
    assert all(len(line.split()) == 2 + 12 + 3 for line in lines)
    _, desc, blob_out = export.read_dlw(out)
    assert desc.H == 16 and desc.W == 180
    assert not np.array_equal(np.asarray(blob_out), export.pack_state_dict(model.state_dict(), cfg)), \
        "the model did not adapt"
