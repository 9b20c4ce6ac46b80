"""-m gpu: streams served on the reference's two-resolution recipe (delora_odometry_streams_push_pre) on the H100.

For every valid stream and tick, over an activity pattern with a tick of first frames, an inactive stream (staged with
another stream's points and a real count, so only the mask keeps it out), an empty active frame, a reset and an idle
tick:
- T is bit-identical to delora_odometry_pairs at B = 1 on the two frames' preprocessed point lists
  (Preprocesser.preprocess_scans at w_pre: the Tester's input); for normalised models, _pairs on those lists divided by
  the call's factor, the translation multiplied back (the list factor sums in another order: it agrees within 1e-6);
- the loss row is bit-identical to delora_icp_dense_fwd_bwd at B = 1 on the grids of projection + normals at H x w_pre
  then the H x W projection (their coordinates divided by the factor for normalised models) and T's 3x4 in the model's
  units;
- rows of S = 3 equal S = 1 workspaces fed only that stream's frames, bit for bit; a graph-replayed tick equals the
  eager call; the workspace, allocated at exactly its size between guard bytes, writes nothing outside itself."""
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
SENTINEL = 1234.5
GUARD = 4096
ICP = ops.LOSS_PO2PL | ops.LOSS_PL2PL
SIZES = [(16, 180, 512, 360), (64, 720, 2048, 2250)]                   # H, W, w_raw, w_pre


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _cfg(h, w, w_pre, normalized):
    cfg = H.config(h, w)
    cfg["kitti"]["horizontal_cells_preprocessing"] = w_pre
    cfg["normalization_scaling"] = normalized
    return cfg


def _flags(normalized, flags=ICP):
    return flags | (ops.TRAIN_NORMALIZATION_SCALING if normalized else 0)


def _pattern(S):
    """active [ticks, S], the (tick, stream) with an empty frame, resets {tick: [streams]} applied before the tick."""
    act = np.ones((7, S), dtype=bool)
    act[1, S - 1] = False                   # an inactive stream
    act[4, :] = False                       # an idle tick
    act[6, 0] = False
    return act, {(2, 1 % S)}, {3: [0]}


def _ticks(pool, S, n_stride, act, empty):
    out = []
    for k in range(act.shape[0]):
        pts = torch.zeros((S, 3, n_stride), dtype=torch.float32)
        counts = torch.zeros((S,), dtype=torch.int32)
        for s in range(S):
            f = pool[(3 * s + k) % len(pool)] if act[k, s] else pool[(3 * s + k + 5) % len(pool)]
            pts[s, :, :f.shape[1]] = f
            counts[s] = 0 if (k, s) in empty else f.shape[1]
        out.append((pts, counts, torch.from_numpy(act[k].astype(np.int32))))
    return out


def _setup(h, w, w_raw, w_pre, normalized, S, seed=3):
    cfg = _cfg(h, w, w_pre, normalized)
    pool = H.frames(h, w_raw, 8)
    n_stride = max(f.shape[1] for f in pool)
    act, empty, resets = _pattern(S)
    blob = H.blob(H.model(cfg, seed, near_identity=True), cfg)
    return cfg, blob, n_stride, _ticks(pool, S, n_stride, act, empty), act, resets


def _guarded(d):
    nbytes = capi.PreStreamsWorkspace.workspace_bytes(d)
    buf = torch.full((nbytes + 2 * GUARD,), 0xFF, dtype=torch.uint8, device=DEV)      # NaN-filled floats
    return buf, buf[GUARD:GUARD + nbytes]


def _run(st, ticks, resets, normalized, graph=False):
    """Every tick through one recipe streams workspace -> [(T [S,16], valid [S], losses [S,8], factor [S] or None)]."""
    S = st.desc.max_batch
    n_stride = ticks[0][0].shape[2]
    pts = torch.zeros((S, 3, n_stride), dtype=torch.float32, device=DEV)
    counts = torch.zeros((S,), dtype=torch.int32, device=DEV)
    active = torch.zeros((S,), dtype=torch.int32, device=DEV)
    T = torch.full((S, 16), SENTINEL, dtype=torch.float32, device=DEV)
    valid = torch.full((S,), 7, dtype=torch.int32, device=DEV)
    losses = torch.full((S, ops.LOSS_ROW), SENTINEL, dtype=torch.float32, device=DEV)
    factor = torch.full((S,), SENTINEL, dtype=torch.float32, device=DEV) if normalized else None
    mask = torch.zeros((S,), dtype=torch.int32, device=DEV)
    g = None
    if graph:
        st.push(pts, counts, active, T, valid, losses, factor)        # all inactive: changes no stream's state
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            st.push(pts, counts, active, T, valid, losses, factor)
    out = []
    for k, (p, c, a) in enumerate(ticks):
        if k in resets:
            mask.zero_()
            mask[resets[k]] = 1
            st.reset(mask)
        pts.copy_(p)
        counts.copy_(c)
        active.copy_(a)
        if g is not None:
            g.replay()
        else:
            st.push(pts, counts, active, T, valid, losses, factor)
        torch.cuda.synchronize()
        out.append((T.cpu().clone(), valid.cpu().clone(), losses.cpu().clone(),
                    None if factor is None else factor.cpu().clone()))
    return out


def _history(ticks, act, resets):
    """{(k, s): (previous frame, this frame)} of every pair the streams should serve: (points [3, n], count)."""
    pairs, prev = {}, [None] * act.shape[1]
    for k, (p, c, _) in enumerate(ticks):
        for s in resets.get(k, []):
            prev[s] = None
        for s in range(act.shape[1]):
            if not act[k, s]:
                continue
            if prev[s] is not None:
                pairs[(k, s)] = (prev[s], (p[s], c[s]))
            prev[s] = (p[s], c[s])
    return pairs


def _check_against_references(cfg, blob, out, pairs, normalized, flags=ICP):
    ds = cfg["kitti"]
    h, w, w_pre = ds["vertical_cells"], ds["horizontal_cells"], ds["horizontal_cells_preprocessing"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    inf = capi.InferenceWorkspace(H.desc(cfg, h * w_pre, 1), blob)
    S = out[0][0].shape[0]
    for k, (T, valid, losses, factor) in enumerate(out):
        for s in range(S):
            want = (k, s) in pairs
            assert int(valid[s]) == int(want), f"tick {k} stream {s}: valid={int(valid[s])}, expected {int(want)}"
            if not want:
                assert float(losses[s].abs().max()) == 0.0, f"tick {k} stream {s}: an invalid loss row is not zero"
                if normalized:
                    assert float(factor[s]) == 0.0
                continue
            (p1, c1), (p2, c2) = pairs[(k, s)]
            pts, counts = H.stack([p1[:, :int(c1)], p2[:, :int(c2)]], p1.shape[1])
            plist, _, lens = H._preprocessed_lists(cfg, pts, counts, w_pre)
            lists = torch.zeros((2, 3, h * w_pre), dtype=torch.float32, device=DEV)
            lists[:, :, :plist.shape[2]] = plist
            f = float(factor[s]) if normalized else 1.0
            if normalized:
                fl = float(ops.normalization_factors(lists, lens)[0])
                assert abs(fl - f) <= 1e-6 * abs(f) or (np.isnan(fl) and np.isnan(f)), (k, s, fl, f)
                ft = torch.tensor(f, dtype=torch.float32, device=DEV)
                lists = lists / ft
            t_model, _ = inf.pairs(lists, lens)
            t_ref = t_model.clone()
            if normalized:
                t_ref[:, :3, 3] *= ft
            assert _same(T[s], t_ref.reshape(16).cpu()), \
                f"tick {k} stream {s}: T differs from delora_odometry_pairs on the preprocessed lists"
            grids = []
            for pp, cc in ((p1, c1), (p2, c2)):
                _, _, pg, ng = ops.project_normals(pp[None].to(DEV), cc.view(1).to(DEV), h, w_pre, hf, vf,
                                                   ds["neighborhood_side_length"], cfg["epsilon_range"],
                                                   cfg["min_num_points_in_neighborhood_to_determine_point_class"])
                if normalized:
                    pg = torch.cat((pg[..., :3] / ft, pg[..., 3:]), dim=-1)
                _, _, g_pts, g_nrm = ops.project_grids(pg.contiguous(), ng, h, w_pre, w, hf, vf, index_map=False)
                grids.append((g_pts, g_nrm))
            row = ops.icp_dense_fwd_bwd(grids[1][0], grids[1][1], t_model.reshape(1, 16)[:, :12].contiguous(),
                                        grids[0][0], grids[0][1], h, w, hf, vf, float(cfg["lambda_po2pl"]), flags)[0][0]
            assert _same(losses[s], row.cpu()), \
                f"tick {k} stream {s}: {losses[s].tolist()} != the operator alone {row.tolist()}"


@pytest.mark.parametrize("normalized", [False, True], ids=["plain", "normalized"])
@pytest.mark.parametrize("h,w,w_raw,w_pre", SIZES, ids=["16x180", "64x720"])
def test_rows_are_the_testers_input_and_the_operators_residual(cuda_lib, h, w, w_raw, w_pre, normalized):
    S = 3
    cfg, blob, n_stride, ticks, act, resets = _setup(h, w, w_raw, w_pre, normalized, S)
    d = H.desc(cfg, n_stride, S, w_pre)
    buf, ws = _guarded(d)
    st = capi.PreStreamsWorkspace(d, blob, capi.residual_params(cfg, _flags(normalized)), workspace=ws)
    out = _run(st, ticks, resets, normalized)
    torch.cuda.synchronize()
    assert bool((buf[:GUARD] == 0xFF).all()) and bool((buf[GUARD + ws.numel():] == 0xFF).all()), \
        "a write outside delora_odometry_streams_pre_workspace_bytes"
    pairs = _history(ticks, act, resets)
    assert len(pairs) >= 8 and int(out[0][1].sum()) == 0
    _check_against_references(cfg, blob, out, pairs, normalized)
    # rows without a transform this tick keep the T row of the tick before
    for k in range(1, len(out)):
        for s in range(S):
            if not int(out[k][1][s]):
                assert _same(out[k][0][s], out[k - 1][0][s]), f"tick {k} stream {s}: an invalid T row was written"


@pytest.mark.parametrize("normalized", [False, True], ids=["plain", "normalized"])
def test_streams_are_independent_and_the_graph_replays(cuda_lib, normalized):
    h, w, w_raw, w_pre = SIZES[0]
    S = 3
    cfg, blob, n_stride, ticks, act, resets = _setup(h, w, w_raw, w_pre, normalized, S, seed=5)
    rp = capi.residual_params(cfg, _flags(normalized))
    eager = _run(capi.PreStreamsWorkspace(H.desc(cfg, n_stride, S, w_pre), blob, rp), ticks, resets, normalized)
    graphed = _run(capi.PreStreamsWorkspace(H.desc(cfg, n_stride, S, w_pre), blob, rp), ticks, resets, normalized,
                   graph=True)
    for k, (e, g) in enumerate(zip(eager, graphed)):
        for i, (a, b) in enumerate(zip(e, g)):
            assert a is None or _same(a, b), f"tick {k}: output {i} of the replay differs from the eager call"
    for s in range(S):
        single = [(p[s:s + 1], c[s:s + 1], a[s:s + 1]) for p, c, a in ticks]
        res = {k: [0] for k, streams in resets.items() if s in streams}
        one = _run(capi.PreStreamsWorkspace(H.desc(cfg, n_stride, 1, w_pre), blob, rp), single, res, normalized)
        for k, (e, o) in enumerate(zip(eager, one)):
            assert int(e[1][s]) == int(o[1][0]), f"tick {k} stream {s}: valid differs from S = 1"
            if int(o[1][0]):
                assert _same(e[0][s], o[0][0]), f"tick {k} stream {s}: T differs from S = 1"
            assert _same(e[2][s], o[2][0]), f"tick {k} stream {s}: losses differ from S = 1"
            if normalized:
                assert _same(e[3][s], o[3][0]), f"tick {k} stream {s}: factor differs from S = 1"


@pytest.mark.parametrize("normalized", [False, True], ids=["plain", "normalized"])
def test_agrees_with_the_training_eval(cuda_lib, normalized):
    """T and the loss row against delora_odometry_train_eval at B = 1 on the same pair and descriptor: not bit-identical
    (the training forward keeps the stem's pre-activation in fp16), within 2e-3 on T's entries and 2 % on the losses
    and matched pairs; the factor is the same bits (the same grid factor kernel on the same H x w_pre grids)."""
    h, w, w_raw, w_pre = SIZES[1]
    cfg, blob, n_stride, _, _, _ = _setup(h, w, w_raw, w_pre, normalized, 1, seed=7)
    ticks = _ticks(H.frames(h, w_raw, 8), 1, n_stride, np.ones((4, 1), dtype=bool), set())
    flags = _flags(normalized)
    st = capi.PreStreamsWorkspace(H.desc(cfg, n_stride, 1, w_pre), blob, capi.residual_params(cfg, flags))
    out = _run(st, ticks, {}, normalized)
    tr = capi.TrainingWorkspace(H.desc(cfg, n_stride, 1, w_pre), blob, capi.train_params(cfg, 0.0, loss_flags=flags))
    checked = 0
    for k in range(1, 4):
        assert int(out[k][1][0]) == 1
        pts, counts = H.stack([ticks[k - 1][0][0, :, :int(ticks[k - 1][1][0])], ticks[k][0][0, :, :int(ticks[k][1][0])]],
                              n_stride)
        losses, T, _ = tr.eval(pts, counts)
        torch.cuda.synchronize()
        t_err = float((T[0].reshape(16).cpu() - out[k][0][0]).abs().max())
        l_err = float(((losses[0, :3].cpu() - out[k][2][0, :3]).abs() / losses[0, :3].cpu().abs().clamp_min(1e-12)).max())
        m_err = abs(float(losses[0, 3]) - float(out[k][2][0, 3])) / max(float(losses[0, 3]), 1.0)
        print(f"\n[64x720 w_pre 2250 {'normalized' if normalized else 'plain'} tick {k}] T {t_err:.2e}  losses "
              f"{l_err:.2e}  pairs {m_err:.2e}")
        assert t_err <= 2e-3 and l_err <= 2e-2 and m_err <= 2e-2, (t_err, l_err, m_err)
        if normalized:
            assert _same(out[k][3][0:1], losses[0, 6:7].cpu())
        checked += 1
    assert checked >= 2


def _mirror_T(model, cfg, prev, cur, normalized):
    """The reference Tester's path in Python: preprocessed lists -> ops.project at H x W -> OdometryModel ->
    GeometryHandler; normalised configs divide the lists by the pair's factor and scale the translation back."""
    from delora_b200.models.model_parts import GeometryHandler
    ds = cfg["kitti"]
    h, w, w_pre = ds["vertical_cells"], ds["horizontal_cells"], ds["horizontal_cells_preprocessing"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    pts, counts = H.stack([prev, cur], max(prev.shape[1], cur.shape[1]))
    plist, _, lens = H._preprocessed_lists(cfg, pts, counts, w_pre)
    f = ops.normalization_factors(plist, lens) if normalized else None
    if normalized:
        plist = plist / f.view(1, 1, 1)
    image, _ = ops.project(plist, lens, h, w, hf, vf)
    with torch.no_grad():
        trans, quat = model(image_1=image[0:1], image_2=image[1:2])
        t = GeometryHandler.get_transformation_matrix_quaternion(translation=trans.float(), quaternion=quat.float(),
                                                                 device=DEV)
    if normalized:
        t[:, :3, 3] *= f.view(1, 1)
    return t.cpu().numpy()


@pytest.mark.parametrize("normalized", [False, True], ids=["plain", "normalized"])
def test_python_class_returns_the_workspace_bits_and_mirrors_the_tester(cuda_lib, normalized):
    from delora_b200.deploy.stream import PreprocessedOdometryStreams
    h, w, w_raw, w_pre = SIZES[0]
    S = 2
    cfg, blob, n_stride, ticks, act, resets = _setup(h, w, w_raw, w_pre, normalized, S, seed=9)
    model = H.model(cfg, 9, near_identity=True).eval()
    cls = PreprocessedOdometryStreams(model, cfg, "kitti", S, n_stride)
    st = capi.PreStreamsWorkspace(H.desc(cfg, n_stride, S, w_pre), blob,
                                  capi.residual_params(cfg, _flags(normalized)))
    ticks = ticks[:4]
    ws_out = _run(st, ticks, {}, normalized)
    prev = [None] * S
    checked = 0
    for k, (p, c, a) in enumerate(ticks):
        scans = [p[s, :, :int(c[s])].clone() if int(a[s]) else None for s in range(S)]
        got = cls.push(scans)
        for s in range(S):
            if got[s] is None:
                assert not int(ws_out[k][1][s])
            else:
                t, losses = got[s][0], got[s][1]
                assert np.array_equal(t.reshape(16).view(np.int32), ws_out[k][0][s].numpy().view(np.int32))
                assert np.array_equal(losses.view(np.int32), ws_out[k][2][s].numpy().view(np.int32))
                if normalized:
                    assert np.float32(got[s][2]).view(np.int32) == ws_out[k][3][s].numpy().view(np.int32)
                if prev[s].shape[1] and scans[s].shape[1]:            # an empty frame has no mean range
                    mirror = _mirror_T(model, cfg, prev[s], scans[s], normalized)
                    err = float(np.abs(mirror - t).max())
                    assert err <= 1e-5, f"tick {k} stream {s}: {err:.2e} from the Tester's path"
                    checked += 1
            if scans[s] is not None:
                prev[s] = scans[s]
    assert checked >= 2 and len(cls.poses(0)) >= 2


@pytest.mark.parametrize("normalized", [False, True], ids=["plain", "normalized"])
def test_example_program_prints_the_python_class_results(cuda_lib, tmp_path, normalized):
    from delora_b200 import synthetic
    from delora_b200.deploy import export
    from delora_b200.deploy.stream import PreprocessedOdometryStreams
    vfov = (-15.0, 15.0)
    cfg = _cfg(16, 720, 1024, normalized)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    model = H.model(cfg, 6, near_identity=True).eval()
    dlw = os.path.join(tmp_path, "m.dlw")
    desc = export.desc_from_config(cfg, "kitti", 4096, 1, preprocessing_normals=True)
    export.write_dlw(dlw, desc, export.pack_state_dict(model.state_dict(), cfg), export.model_flags_from_config(cfg))
    dirs, scans = [], []
    for s, n in enumerate((4, 3)):
        dd = os.path.join(tmp_path, f"stream{s}")
        os.makedirs(dd)
        dirs.append(dd)
        scans.append([])
        for i in range(n):
            scan = synthetic.kitti_bin_scan(10 * s + i, vfov_deg=vfov)
            scan.tofile(os.path.join(dd, f"{i:06d}.bin"))
            scans[s].append(torch.from_numpy(scan[:, :3].T.copy()))
    exe = H.build_example("odometry_streams", tmp_path, link=True)
    r = subprocess.run([exe, "--preprocessing", dlw] + dirs, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lines = [ln.split() for ln in r.stdout.strip().splitlines()]
    cls = PreprocessedOdometryStreams(model, cfg, "kitti", 2, 4096)
    want = []
    for k in range(4):
        got = cls.push([sc[k] if k < len(sc) else None for sc in scans])
        for s, g in enumerate(got):
            if g is not None:
                want.append((s, k, g[0].reshape(16)[:12], g[1]))
    assert len(lines) == len(want) == 5
    for ln, (s, k, t, losses) in zip(lines, want):
        assert (int(ln[0]), int(ln[1])) == (s, k)
        assert np.array_equal(np.array(ln[2:14], dtype=np.float32), t), (ln, t)
        assert np.array_equal(np.array(ln[14:16], dtype=np.float32), losses[1:3]) and float(ln[16]) == losses[3]
    # a file without w_pre is refused, naming the exporter's option
    desc.w_pre = 0
    export.write_dlw(dlw, desc, export.pack_state_dict(model.state_dict(), cfg), export.model_flags_from_config(cfg))
    r = subprocess.run([exe, "--preprocessing", dlw] + dirs, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "--preprocessing-normals" in r.stderr
