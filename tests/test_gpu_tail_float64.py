"""The odometry tail's kernels (odometry_tail.cu: resnet.fc and the heads, the block-normalised quaternion -> T, their
backward, Adam) against the float64 reference of tail_reference.py, element by element, on the H100.

Teacher forcing: every comparison starts from bits the GPU returns, so that only the tail is under test.  pooled comes
from _pairs or _train_step; the identity fit's dL/dT is formed from the step's own T; Adam's inputs are
_train_get_state before the step and the step's returned gradient.  Every element must satisfy |got - ref| <= bound
(tail_reference's running error analysis of the kernels' arithmetic), and no NaN / Inf may appear where the reference
is finite.  Rows whose block-divided quaternion norm lies within its fp32 bound of kornia's 1e-12 clamp are excluded
(the count is printed).

Weight families (tail_reference.family_weights): torch's initialisation, near-identity heads, saturating tanh (fc and
hidden weights x 30), relu rows with a pre-activation of exactly 0, one row's quaternion dominating the block (10^3),
and rows on both sides of the 1e-12 clamp (relu: the other rows' selector unit is exactly 0; the clamp is placed in the
widest gap between rows, so none is excluded).  Shapes: resnet_outputs 1000 (float4 path), 1002 (scalar path,
misaligned in the master blob) and 3 (lanes without work, a partial dx tile), relu and tanh, both head kinds.  On the
single MLP, the worst-case propagation through four hidden layers makes the bound as large as the quaternion for
init, saturating and zero_rows; those cases print a skip, and the others (near_identity, dominance, clamp) run.

Covered: _pairs at B = 1, 2, 3, 4, 5, 7, 8, 9, 33 and 1000; _pairs_normalized with its factor; _train_step's fc and
head gradients (every element of dW and db) with the identity fit at B = 1, 3, 4, 5, 9, 64 and with the ICP objective
(icp_dense_fwd_bwd's grad_T / B on every row, after its loss rows matched the step's bit for bit) at B = 1, 5; a
DELORA_TRAIN_DROPOUT step with delora_dropout_keep_mask's fc mask; _streams_push at S = 3, 5 with an inactive stream
(per-row norm; rows that are not valid keep their sentinel); _streams_push_adapt at S = 3 with beta1 = 0 (a tick
without a valid pair leaves the state byte-identical; then exp_avg is the gradient of the mean over the valid rows,
1/n_valid, per-row norm, zeros from the first-frame row); Adam over the whole blob (n & 3 = 3 and 1) after _set_state
with step counts 0 .. 2^31 + 5, with v = 0 where g = 0, tiny v and m of the opposite sign to g, and with lr = 0.
Not covered: Adam where g * g overflows fp32; the ABI feeds Adam only the step's own gradient, and no realistic
input makes it that large.

Worst error / bound measured on an H100 SXM (700 W), largest over shapes and batch sizes:
  _pairs T: init 0.006, near_identity 0.016, saturating 0.021, zero_rows 0.005, dominance 0.014, clamp 0.009;
  identity-fit gradients: init 0.21, near_identity 0.20, saturating 0.22, zero_rows 0.22, dominance 0.22, clamp 0.21;
  ICP-objective gradients: init 0.27, near_identity 0.30, saturating 0.18, zero_rows 0.15, dominance 0.26, clamp 0.20;
  single MLP: T 0.012, gradients 0.14; dropout step 0.096; streams T 0.009; adapting streams 0.22;
  Adam: 0.994 (the last rounding of p' is up to half an ulp, which the bound takes as u |p'|: tight by construction).
"""
import numpy as np
import pytest
import torch

import odometry_harness as H
import tail_reference as R
from delora_b200 import ops
from delora_b200.deploy import export
from delora_b200.deploy.capi import InferenceWorkspace

pytestmark = pytest.mark.gpu
HW = (16, 180)
W_RAW = 512
N_DISTINCT = 40
B_INFER = [1, 2, 3, 4, 5, 7, 8, 9, 33]
B_LARGE = 1000                   # near kMaxBatch = 1024: the out kernel's single CTA and one-thread norm loop
B_TRAIN = [1, 3, 4, 5, 9, 64]
# the single-MLP cases skip, with a printed reason, the families where its bound is uninformative (see _forward)
SHAPES = [("relu", False, 1000), ("tanh", False, 1000), ("tanh", False, 1002), ("relu", False, 1002),
          ("relu", False, 3), ("tanh", False, 3), ("tanh", True, 1000), ("relu", True, 1002)]


def _batch(b):
    """b pairs (N_DISTINCT distinct ones, repeated cyclically) -> (pts, counts, n_stride)."""
    distinct = H.pairs(HW[0], W_RAW, min(b, N_DISTINCT))
    pairs = [distinct[i % len(distinct)] for i in range(b)]
    stride = H.n_stride(distinct)
    pts, counts = H.stack_pairs(pairs, stride)
    return pts, counts, stride


def _state(blob, cfg):
    return {k: v.numpy() for k, v in export.unpack_blob(blob.cpu().numpy(), cfg).items()}


def _blob(state, cfg):
    return torch.from_numpy(export.pack_state_dict({k: torch.from_numpy(np.asarray(v, np.float32))
                                                    for k, v in state.items()}, cfg)).to(H.DEV)


def _families(act, b):
    out = ["init", "near_identity", "saturating", "zero_rows"]
    if 2 <= b <= 33:
        out.append("dominance")
        if act == "relu":
            out.append("clamp")
    return out


def _check(got, ref, bound, what, skip=None):
    got = np.asarray(got, np.float64)
    ref, bound = np.broadcast_to(ref, got.shape), np.broadcast_to(bound, got.shape)
    if skip is not None:
        keep = ~np.broadcast_to(skip, got.shape)
        got, ref, bound = got[keep], ref[keep], bound[keep]
    fin = np.isfinite(ref)
    assert np.all(np.isfinite(got[fin])), f"{what}: NaN / Inf where the reference is finite"
    err = np.abs(got - ref)
    bad = err > bound
    assert not bad.any(), (f"{what}: {int(bad.sum())} elements outside the bound, worst |err| {err[bad].max():.3e} "
                           f"against {bound[bad][np.argmax(err[bad])]:.3e}")
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(r.max()) if r.size else 0.0


def _forward(pooled, w, cfg, what, **kw):
    """tail_forward, or None (printed) for a single-MLP case whose bounds say nothing: its four hidden layers compound
    the worst-case propagation until a row's quaternion bound reaches half its norm; two-head cases must never."""
    fw = R.tail_forward(pooled, w, cfg, **kw)
    if R.uninformative(fw).any():
        assert cfg["use_single_mlp_at_output"], f"{what}: a row's bound is as large as its quaternion"
        print(f"\n[{what}] skipped: the single MLP's bound is as large as the quaternion on "
              f"{int(R.uninformative(fw).sum())} rows")
        return None
    near = R.near_clamp(fw)
    assert not near.any(), f"{what}: {int(near.sum())} rows on kornia's clamp"
    return fw


def _grad_check(fw, g, eg, grads, cfg, what, valid=None):
    ref = R.tail_backward(fw, g, eg, valid)
    got = _tail_grads(grads, cfg)
    return max(_check(got[name], v, e, f"{name} {what}") for name, (v, e) in ref.items())


@pytest.mark.parametrize("act,single,nout", SHAPES)
def test_inference_T(cuda_lib, act, single, nout):
    """_pairs (block norm) at every B, and _pairs_normalized with its factor at B = 1, 5, 9."""
    cfg = H.config(*HW, act, single, nout=nout)
    base = _state(H.blob(H.model(cfg), cfg), cfg)
    bmax = B_LARGE if (act, single, nout) == ("relu", False, 1000) else max(B_INFER)
    pts_all, counts_all, stride = _batch(bmax)
    ws = InferenceWorkspace(H.desc(cfg, stride, bmax), _blob(base, cfg))
    sizes = B_INFER + ([B_LARGE] if bmax == B_LARGE else [])
    for b in sizes:
        pts, counts, _ = _batch(b)
        _, pooled = ws.pairs(pts, counts)
        pooled = pooled.cpu().numpy()
        for fam in _families(act, b):
            what = f"T {act} single={single} nout={nout} {fam} B={b}"
            w = R.family_weights(fam, base, cfg, pooled)
            ws.load_weights(_blob(w, cfg))
            T, pooled2 = ws.pairs(pts, counts)
            assert np.array_equal(pooled2.cpu().numpy(), pooled), "pooled depends on the tail weights"
            fw = _forward(pooled, w, cfg, what)
            if fw is None:
                continue
            r = _check(T.cpu().numpy(), fw["T"], fw["eT"], what)
            if b in (1, 5, 9) and fam not in ("dominance", "clamp"):   # those are fitted to _pairs' pooled
                Tn, pooled_n, f = ws.pairs_normalized(pts, counts)
                fwn = _forward(pooled_n.cpu().numpy(), w, cfg, what + " normalized", factor=f.cpu().numpy())
                r = max(r, _check(Tn.cpu().numpy(), fwn["T"], fwn["eT"], what + " normalized"))
            print(f"\n[{what}] worst {r:.3f}")


def _tail_grads(flat, cfg):
    d = _state(flat, cfg)
    return {k: d[k] for k in R.grad_names(cfg)}


def _project_normals(cfg, pts, counts):
    ds = cfg["kitti"]
    return ops.project_normals(pts, counts, *HW, cfg["horizontal_field_of_view"], ds["vertical_field_of_view"],
                               ds["neighborhood_side_length"], cfg["epsilon_range"],
                               cfg["min_num_points_in_neighborhood_to_determine_point_class"])


def _icp_grad_T(cfg, pts, counts, T, losses, src, tgt):
    """dL/dT of the ICP objective for pairs (scan src[i] -> scan tgt[i]) at the step's T: icp_dense_fwd_bwd alone on
    project_normals of the same scans.  Its loss rows must equal the step's bit for bit, the evidence that its grad_T
    is the one the step's backward read."""
    _, _, pg, ng = _project_normals(cfg, pts, counts)
    lo, gT = ops.icp_dense_fwd_bwd(pg[src].contiguous(), ng[src].contiguous(),
                                   T.reshape(-1, 16)[:, :12].contiguous(), pg[tgt].contiguous(), ng[tgt].contiguous(),
                                   *HW, cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"],
                                   float(cfg["lambda_po2pl"]), H.FLAGS)
    assert torch.equal(lo.view(torch.int32), losses.view(torch.int32)), "the ICP loss rows differ from the step's"
    return gT.cpu().numpy()


@pytest.mark.parametrize("act,single,nout", SHAPES)
def test_training_gradients(cuda_lib, act, single, nout):
    """_train_step's fc and head gradients, every element: the identity fit at every B in B_TRAIN, the ICP objective
    (dL/dT = grad_T / B on every row) at B = 1, 5."""
    cfg = H.config(*HW, act, single, nout=nout)
    base = _state(H.blob(H.model(cfg), cfg), cfg)
    for b in B_TRAIN:
        pts, counts, stride = _batch(b)
        probe = H.trainer(cfg, stride, b, _blob(base, cfg))
        pooled = probe.eval(pts, counts)[2].cpu().numpy()
        for fam in _families(act, b):
            w = R.family_weights(fam, base, cfg, pooled)
            for identity in (True, False) if b in (1, 5) else (True,):
                what = f"grads {act} single={single} nout={nout} {fam} B={b} {'identity' if identity else 'icp'}"
                flags = H.FLAGS | (ops.LOSS_IDENTITY_FIT if identity else 0)
                tr = H.trainer(cfg, stride, b, _blob(w, cfg), flags=flags)
                losses, T, pooled2, grads = tr.step(pts, counts)
                assert np.array_equal(pooled2.cpu().numpy(), pooled)
                fw = _forward(pooled, w, cfg, what)
                if fw is None:
                    continue
                Tn = T.cpu().numpy()
                worst = _check(Tn, fw["T"], fw["eT"], what)
                if identity:
                    g, eg = R.dT_identity(Tn)
                else:
                    g, eg = R.dT_scaled(_icp_grad_T(cfg, pts, counts, T, losses, slice(b, 2 * b), slice(0, b)), b)
                worst = max(worst, _grad_check(fw, g, eg, grads, cfg, what))
                print(f"\n[{what}] worst {worst:.3f}")


@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_dropout_step_gradients(cuda_lib, act):
    """A DELORA_TRAIN_DROPOUT identity-fit step: the fc output is act(keep * 1.25 * (W pooled + b)) with the mask of
    delora_dropout_keep_mask at the step count _train_get_state reports (seed 0), and its gradient is masked alike."""
    cfg = H.config(*HW, act, False, nout=1000)
    cfg["use_dropout"] = True
    base = _state(H.blob(H.model(cfg), cfg), cfg)
    b = 5
    pts, counts, stride = _batch(b)
    tr = H.trainer(cfg, stride, b, _blob(base, cfg), flags=H.FLAGS | ops.LOSS_IDENTITY_FIT)
    tr.set_state(_blob(base, cfg).cpu().numpy(), np.zeros(tr.n, np.float32), np.zeros(tr.n, np.float32), 7)
    step = int(tr.get_state()[3][0])
    keep = ops.dropout_keep_mask(0, step, ops.DROPOUT_FC, b * 1000).view(b, 1000).cpu().numpy() != 0
    _, T, pooled, grads = tr.step(pts, counts)
    what = f"dropout {act} B={b}"
    fw = _forward(pooled.cpu().numpy(), base, cfg, what, fc_keep=keep)
    Tn = T.cpu().numpy()
    worst = _check(Tn, fw["T"], fw["eT"], what)
    worst = max(worst, _grad_check(fw, *R.dT_identity(Tn), grads, cfg, what))
    print(f"\n[{what}] worst {worst:.3f}, {int((~keep).sum())} of {keep.size} fc outputs dropped")


def _pair_pooled(ws1, pair, stride):
    pts, counts = H.stack_pairs([pair], stride)
    T, pooled = ws1.pairs(pts, counts)
    return T.cpu().numpy()[0], pooled.cpu().numpy()[0]


@pytest.mark.parametrize("S", [3, 5])
def test_streams_per_row_T(cuda_lib, S):
    """_streams_push with some streams inactive: each valid row's quaternion is divided by its own norm (teacher-forced
    from _pairs at B = 1 on the same pair, whose pooled rows do not depend on B), and the other rows are not written."""
    from delora_b200.deploy.capi import StreamsWorkspace
    cfg = H.config(*HW, "relu", False, nout=1000)
    base = _state(H.blob(H.model(cfg), cfg), cfg)
    pairs = H.pairs(HW[0], W_RAW, S)
    stride = H.n_stride(pairs)
    pts_all, counts_all = H.stack_pairs(pairs, stride)
    active = torch.tensor([int(s % 3 != 1) for s in range(S)], dtype=torch.int32, device=H.DEV)
    for fam in ("init", "near_identity", "zero_rows", "dominance", "clamp"):
        ws1 = InferenceWorkspace(H.desc(cfg, stride, S), _blob(base, cfg))
        _, pooled_b = ws1.pairs(pts_all, counts_all)
        rows = [_pair_pooled(ws1, p, stride)[1] for p in pairs]
        assert np.array_equal(pooled_b.cpu().numpy(), np.stack(rows)), "_pairs' pooled rows depend on B"
        pooled = np.stack(rows)
        w = R.family_weights(fam, base, cfg, pooled)
        ws = StreamsWorkspace(H.desc(cfg, stride, S), _blob(w, cfg))
        T = torch.full((S, 16), 1234.5, dtype=torch.float32, device=H.DEV)
        valid = torch.full((S,), 7, dtype=torch.int32, device=H.DEV)
        p1, c1 = H.stack([p[0] for p in pairs], stride)
        p2, c2 = H.stack([p[1] for p in pairs], stride)
        ws.push(p1, c1, None, T, valid)
        ws.push(p2, c2, active, T, valid)
        v = valid.cpu().numpy()
        assert v.tolist() == active.cpu().numpy().tolist()
        Tn = T.cpu().numpy().reshape(S, 4, 4)
        assert np.all(Tn[v == 0] == 1234.5), "a row that is not valid was written"
        what = f"streams S={S} {fam}"
        fw = _forward(pooled[v != 0], w, cfg, what, norm="row")
        r = _check(Tn[v != 0], fw["T"], fw["eT"], what)
        print(f"\n[{what}] worst {r:.3f}")


def test_adapting_streams_gradient(cuda_lib):
    """_streams_push_adapt with update = 1 at S = 3, beta1 = 0: a tick without a valid pair changes nothing (Adam's run
    predicate at n_valid = 0); on the next, streams 0 and 1 have pairs and stream 2 its first frame, so exp_avg is the
    gradient of the mean over the two valid rows, each divided by its own norm, and row 2 contributes zeros."""
    from delora_b200.deploy import capi
    cfg = H.config(*HW, "relu", False, nout=1000)
    for fam in ("init", "near_identity", "dominance"):
        frames = H.frames(HW[0], W_RAW, 6)
        stride = max(f.shape[1] for f in frames)
        base = _state(H.blob(H.model(cfg), cfg), cfg)
        pairs = [(frames[0], frames[1]), (frames[2], frames[3])]
        # the adapting workspace runs the training forward: pooled from _train_eval on each pair alone
        probe = H.trainer(cfg, stride, 1, _blob(base, cfg))
        pooled = np.stack([probe.eval(*H.stack_pairs([p], stride))[2].cpu().numpy()[0] for p in pairs])
        w = R.family_weights(fam, base, cfg, pooled)
        ws = capi.AdaptiveStreamsWorkspace(H.desc(cfg, stride, 3), _blob(w, cfg),
                                           capi.train_params(cfg, 1e-4, loss_flags=H.FLAGS, beta1=0.0))
        T = torch.zeros((3, 16), dtype=torch.float32, device=H.DEV)
        valid = torch.zeros((3,), dtype=torch.int32, device=H.DEV)
        losses = torch.zeros((3, ops.LOSS_ROW), dtype=torch.float32, device=H.DEV)
        p0, c0 = H.stack([frames[0], frames[2], frames[4]], stride)
        p1, c1 = H.stack([frames[1], frames[3], frames[4]], stride)
        before = [a.cpu().numpy() for a in ws.get_state()]
        ws.push(p0, c0, torch.tensor([1, 1, 0], dtype=torch.int32, device=H.DEV), T, valid, losses, update=True)
        mid = [a.cpu().numpy() for a in ws.get_state()]
        assert valid.cpu().tolist() == [0, 0, 0]
        assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(before, mid)), \
            "an update without a valid pair changed the training state"
        ws.push(p1, c1, None, T, valid, losses, update=True)
        after = [a.cpu().numpy() for a in ws.get_state()]
        v = valid.cpu().numpy()
        assert v.tolist() == [1, 1, 0] and int(after[3][0]) == int(mid[3][0]) + 1
        what = f"adapt {fam}"
        fw = _forward(pooled, w, cfg, what, norm="row")
        Tn = T[:2].cpu().numpy().reshape(2, 4, 4)
        worst = _check(Tn, fw["T"], fw["eT"], what)
        pts, counts = H.stack([frames[0], frames[2], frames[1], frames[3]], stride)
        gT = _icp_grad_T(cfg, pts, counts, T[:2], losses[:2], slice(2, 4), slice(0, 2))
        g, eg = R.dT_scaled(gT, 2)
        m = after[1]                                      # beta1 = 0: exp_avg = fma(0, m, 1 * g) = g
        worst = max(worst, _grad_check(fw, g, eg, torch.from_numpy(m), cfg, what))
        print(f"\n[{what}] worst {worst:.3f}")


STEPS = [0, 1, 9, 10 ** 4, 2 ** 24 - 1, 2 ** 24, 2 ** 24 + 1, 2 ** 31 + 5]


def _adam_case(tr, pts, counts, state, lr):
    tr.set_state(*state)
    before = [a.cpu().numpy() for a in tr.get_state()]
    grads = tr.step(pts, counts)[3].cpu().numpy()
    after = [a.cpu().numpy() for a in tr.get_state()]
    t = int(before[3][0]) + 1
    assert int(after[3][0]) == t
    ref, err = R.adam_step(before[0], grads, before[1], before[2], t, lr, 0.9, 0.999, 1e-8)   # train_params' betas, eps
    return max(_check(a, r, e, f"Adam {n} t={t}") for a, r, e, n in zip(after[:3], ref, err, ("p", "m", "v"))), \
        before, grads, after


@pytest.mark.parametrize("nout", [1000, 1002])
def test_adam(cuda_lib, nout):
    cfg = H.config(*HW, "relu", False, nout=nout)
    base = _state(H.blob(H.model(cfg), cfg), cfg)
    pts, counts, stride = _batch(2)
    w = R.family_weights("zero_rows", base, cfg)           # exact zero gradients: g = 0 with v = 0 below
    blob = _blob(w, cfg)
    lr = 1e-3
    tr = H.trainer(cfg, stride, 2, blob, lr=lr, flags=H.FLAGS | ops.LOSS_IDENTITY_FIT)
    n = tr.n
    print(f"\n[Adam nout={nout}] n = {n}, n & 3 = {n & 3}")
    rng = np.random.default_rng(0)
    p0 = blob.cpu().numpy()
    m0 = (rng.standard_normal(n) * 1e-4).astype(np.float32)
    v0 = (rng.random(n) * 1e-8).astype(np.float32)
    worst = 0.0
    for step in STEPS:
        r, before, g, after = _adam_case(tr, pts, counts, (p0, m0, v0, step), lr)
        worst = max(worst, r)
        print(f"[Adam nout={nout} step {step}] worst {r:.3f}")
    # adversarial state on the gradient of this step (deterministic: the same weights give the same gradient)
    m1 = np.where(np.arange(n) % 3 == 0, -9.0 * g, m0).astype(np.float32)      # m of the opposite sign to g
    v1 = v0.copy()
    v1[g == 0] = 0                                                             # v = 0 with g = 0
    v1[1::7] = 1e-30                                                           # tiny v
    assert (g == 0).any() and ((g == 0) & (v1 == 0)).any()
    for step in (0, 10 ** 4):
        r, before, g2, after = _adam_case(tr, pts, counts, (p0, m1, v1, step), lr)
        assert np.array_equal(g2, g)
        worst = max(worst, r)
        print(f"[Adam nout={nout} adversarial m / v, step {step}] worst {r:.3f}")
    # lr = 0: the weights stay byte-identical, m and v still advance
    tr0 = H.trainer(cfg, stride, 2, blob, lr=0.0, flags=H.FLAGS | ops.LOSS_IDENTITY_FIT)
    r, before, g, after = _adam_case(tr0, pts, counts, (p0, m0, v0, 5), 0.0)
    assert np.array_equal(after[0].view(np.uint32), before[0].view(np.uint32))
    assert not np.array_equal(after[1], before[1]) and not np.array_equal(after[2], before[2])
    print(f"[Adam nout={nout}] worst over every case {max(worst, r):.3f}")
