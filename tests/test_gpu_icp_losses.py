"""The ICP operators (delora_icp_dense_fwd_bwd, delora_icp_fwd_bwd, delora_icp_point_grads) on every loss
configuration against the float64 reference (tests/icp_reference.py), on the H100.

Flag matrix: the 7 non-empty subsets of {PO2PO, PO2PL, PL2PL}, plus NORMAL_LINEAR on the 4 with PL2PL (11 sets), at
lambda_po2pl in {1, 10, 0.25}.  Inputs: synthetic scan pairs at 16x180 (W not a multiple of the 16-column range
blocks), 15x180 (H not a multiple of the 4-row blocks) and 64x720, with the normals of a seeded 25 % of the valid cells
of both scans zeroed (xyz and has-normal flag), so that po2po pairs exist.  One B = 6 call per size, one transform
per pair:
  0 identity, 1 the synthetic T_pred, 2 a misalignment of metres and 10 deg (lanes go to the block search kernel),
  3 a yaw of 178 deg (re-projections across the seam), 4 no normal anywhere (the po2po_alone configuration: M = 0),
  5 an empty source grid (M = M' = 0).
Both kernels see the same T; the CSR kernel runs on the lists of the same images (delora_lists_from_images).

Bars: M and M' exact; the CSR kernel's NN bit-identical to cKDTree's; an empty set's loss and gradient exactly 0;
losses and grad_T (relative to the pair's max-abs) within the bounds below.  Results of one pair do not depend on the
rest of the batch, on the scratch buffer's history, on the hand-over limit of the window search (up to summation
order) or on DELORA_ICP_STATS; lambda enters grad_T and nothing else.

Measured on an H100 80GB HBM3 (700 W power limit), worst over pairs, flags and lambdas, the same on both kernels:
  losses    1.0e-7 relative (16x180, 15x180 and 64x720 alike);
  grad_T    6.8e-7 of the pair's max-abs at 16x180, 4.7e-7 at 15x180, 1.5e-7 at 64x720;
  per-point gradients (64x720)  8.6e-8 (points), 1.1e-7 (normals) of their max-abs.
The bounds leave a margin of about 10x (losses, per-point gradients) and 7x (grad_T) above those.
"""
import functools
import math

import numpy as np
import pytest
import torch

import icp_reference as R
import odometry_harness as H

pytestmark = pytest.mark.gpu

DEV = "cuda"
B = 6
SIZES = [(16, 180, 192, (-15.0, 15.0)), (15, 180, 192, (-15.0, 15.0)), (64, 720, 1024, (-24.5, 2.0))]
SIZE_IDS = [f"{h}x{w}" for h, w, _, _ in SIZES]
FLAGS = R.flag_matrix()
LAMBDAS = (1.0, 10.0, 0.25)
LOSS_TOL = 1e-6         # relative to the float64 loss
GRAD_TOL = 5e-6         # relative to the pair's max-abs grad_T entry
POINT_TOL = 1e-6        # per-point gradients, relative to the tensor's max-abs
UPSTREAM = (0.7, 1.3, 2.1)
_worst = {}


def _note(key, err):
    _worst[key] = max(_worst.get(key, 0.0), err)


def _report(prefix):
    for k in sorted(k for k in _worst if k.startswith(prefix)):
        print(f"  worst {k}: {_worst[k]:.3e}", flush=True)


def transforms(t_pred):
    from delora_b200 import synthetic
    ts = [np.eye(4), t_pred.numpy().astype(np.float64),
          synthetic.transform_matrix(1.5, -0.4, 0.1, math.radians(10.0), math.radians(1.0), 0.0),
          synthetic.transform_matrix(0.5, 0.2, 0.0, math.radians(178.0)),
          t_pred.numpy().astype(np.float64), t_pred.numpy().astype(np.float64)]
    return torch.tensor(np.stack([t[:3, :] for t in ts]).reshape(B, 12), dtype=torch.float32)


class Batch:
    """Targets are rows 0..B-1, sources rows B..2B-1 of every [2B, ...] tensor."""

    def __init__(self, h, w, w_raw, vfov):
        from delora_b200 import ops, synthetic
        self.h, self.w = h, w
        cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov)
        self.hf, self.vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
        made = [synthetic.make_pair(40 + k, w_raw=w_raw, rings=h, vfov_deg=vfov) for k in range(B)]
        scans = [m[0] for m in made] + [m[1] for m in made]
        stride = max(s.shape[1] for s in scans)
        pts = torch.zeros((2 * B, 3, stride))
        for i, s in enumerate(scans):
            pts[i, :, :s.shape[1]] = s
        counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
        image, _ = ops.project(pts.to(DEV), counts.to(DEV), h, w, self.hf, self.vf)
        image[B + 5] = 0.0                                           # pair 5: empty source
        nrm_img, pg, ng = ops.normals(image, grids=True)
        valid = pg[:, :, 3].view(torch.int32) >= 0
        gen = torch.Generator(device=DEV).manual_seed(h * 100000 + w)
        drop = valid & (torch.rand(valid.shape, generator=gen, device=DEV) < 0.25)
        drop[4] = valid[4]                                           # pair 4: no normal anywhere
        drop[B + 4] = valid[B + 4]
        ng[drop] = 0.0                                               # as grids_from_projection writes it
        nrm_img.view(2 * B, 3, h * w).permute(0, 2, 1)[drop] = 0.0
        self.pg, self.ng = pg, ng
        self.pts4, self.nrm4, self.cs, self.counts = ops.lists_from_images(image, nrm_img)
        n_host = self.counts.cpu().tolist()
        for i in range(2 * B):      # the lists hold the grids' valid cells in row-major order, bit for bit
            for lst, grid in ((self.pts4, pg), (self.nrm4, ng)):
                assert torch.equal(lst[i, :n_host[i]].view(torch.int32), grid[i][valid[i]].view(torch.int32)), i
        assert n_host[B + 5] == 0 and n_host[5] > 0
        self.T = transforms(made[0][3]).to(DEV)
        # the float64 reference's flag-independent part (transform, cKDTree NN, masks), once per pair
        p4, q4 = self.pts4.cpu(), self.nrm4.cpu()
        t_host = self.T.cpu().numpy()
        self.tags, self.ref = [], []
        for k in range(B):
            ns, nt = n_host[B + k], n_host[k]
            self.ref.append(R.prepare(p4[B + k, :ns, :3].numpy(), q4[B + k, :ns, :3].numpy(), t_host[k],
                                      p4[k, :nt, :3].numpy(), q4[k, :nt, :3].numpy(), q4[k, :nt, 3].numpy() != 0))
            self.tags.append(p4[k, :nt, 3].contiguous().view(torch.int32))
        self.n_host = n_host

    def src(self, lo, hi):
        return slice(B + lo, B + hi)

    def dense(self, flags, lam, scratch=None, pairs=(0, B)):
        from delora_b200 import ops
        lo, hi = pairs
        s = self.src(lo, hi)
        return ops.icp_dense_fwd_bwd(self.pg[s].contiguous(), self.ng[s].contiguous(), self.T[lo:hi].contiguous(),
                                     self.pg[lo:hi].contiguous(), self.ng[lo:hi].contiguous(), self.h, self.w, self.hf,
                                     self.vf, lambda_po2pl=lam, flags=flags, scratch=scratch)

    def csr(self, flags, lam, scratch=None, pairs=(0, B), pointwise=False):
        from delora_b200 import ops
        lo, hi = pairs
        s = self.src(lo, hi)
        return ops.icp_fwd_bwd(self.pts4[s].contiguous(), self.nrm4[s].contiguous(), self.counts[s].contiguous(),
                               self.T[lo:hi].contiguous(), self.pts4[lo:hi].contiguous(), self.nrm4[lo:hi].contiguous(),
                               self.cs[lo:hi].contiguous(), self.h, self.w, self.hf, self.vf, lambda_po2pl=lam,
                               flags=flags, pointwise=pointwise, scratch=scratch)


@functools.lru_cache(maxsize=None)
def batch(size_index):
    return Batch(*SIZES[size_index])


def scratch(b, batch_):
    from delora_b200 import ops
    return ops.icp_scratch(b, batch_.h * batch_.w, DEV)


def check_pair(label, losses, grad_t, res):
    """One pair's losses row and grad_T against the reference's Result -> (worst loss rel err, grad err)."""
    row = losses.double().cpu().numpy()
    g = grad_t.double().cpu().numpy().reshape(3, 4)
    assert int(row[3]) == res.M and int(row[4]) == res.Mp, f"{label}: (M, M') = {row[3:5]}, want {(res.M, res.Mp)}"
    assert not row[5:].any(), label
    l_err = 0.0
    for j in range(3):
        if res.losses[j] == 0.0:
            assert row[j] == 0.0, f"{label}: loss {j} = {row[j]}, want exactly 0"
        else:
            l_err = max(l_err, abs(row[j] - res.losses[j]) / res.losses[j])
    scale = np.abs(res.grad_T).max()
    if scale == 0.0:
        assert not g.any(), f"{label}: grad_T = {g}, want exactly 0"
        g_err = 0.0
    else:
        g_err = np.abs(g - res.grad_T).max() / scale
    assert l_err <= LOSS_TOL, f"{label}: losses {row[:3]} vs float64 {res.losses}: {l_err:.3e} relative"
    assert g_err <= GRAD_TOL, f"{label}: grad_T differs from float64 by {g_err:.3e} of its max-abs"
    return l_err, g_err


@pytest.mark.parametrize("size_index", range(len(SIZES)), ids=SIZE_IDS)
def test_losses_and_grad_T_against_float64(size_index, cuda_lib):
    bt = batch(size_index)
    label0 = SIZE_IDS[size_index]
    sd, sc = scratch(B, bt), scratch(B, bt)         # one scratch per kernel, reused across the whole matrix
    nn_checked = False
    for flags in FLAGS:
        for lam in LAMBDAS:
            ld, gd = bt.dense(flags, lam, sd)
            lc, gc, nn_index, _, _ = bt.csr(flags, lam, sc, pointwise=True)
            torch.cuda.synchronize()
            if not nn_checked:
                nn_host = nn_index.cpu()
                for k in range(B):
                    ns = bt.n_host[B + k]
                    want = bt.tags[k][bt.ref[k].nn] if bt.n_host[k] else torch.full((ns,), -1, dtype=torch.int32)
                    assert torch.equal(nn_host[k, :ns], want), f"{label0} pair {k}: CSR NN differs from cKDTree"
                nn_checked = True
            for k in range(B):
                res = R.evaluate(bt.ref[k], flags, lam)
                for kern, lo, gr in (("dense", ld, gd), ("csr", lc, gc)):
                    label = f"{kern} {label0} pair {k} {R.flag_name(flags)} lambda={lam}"
                    l_err, g_err = check_pair(label, lo[k], gr[k], res)
                    _note(f"{kern} {label0} loss", l_err)
                    _note(f"{kern} {label0} grad_T", g_err)
                if k == 5:
                    assert not ld[k].any() and not gd[k].any() and not lc[k].any() and not gc[k].any()
                if k == 4:
                    assert res.M == 0 and (res.Mp > 0) == bool(flags & R.LOSS_PO2PO)
    # the batch has every kind of pair it is meant to have
    full = R.evaluate(bt.ref[2], R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL)
    assert full.M > 100 and full.Mp > 100
    print(f"\n[{label0}] against float64:", flush=True)
    _report(f"dense {label0}")
    _report(f"csr {label0}")


@pytest.mark.parametrize("size_index", range(len(SIZES)), ids=SIZE_IDS)
def test_lambda_weights_only_the_po2pl_gradient(size_index, cuda_lib):
    """grad_T(flags, lambda) - grad_T(flags, 0) = lambda grad_T(PO2PL, 1) up to fp32 rounding, and the losses rows do
    not depend on lambda at all (they are unweighted)."""
    bt = batch(size_index)
    for kern in ("dense", "csr"):
        run = (lambda f, lam: bt.dense(f, lam)) if kern == "dense" else (lambda f, lam: bt.csr(f, lam)[:2])
        _, g_pl = run(R.LOSS_PO2PL, 1.0)
        for flags in FLAGS:
            l0, g0 = run(flags, 0.0)
            for lam in LAMBDAS:
                lo, g = run(flags, lam)
                label = f"{kern} {SIZE_IDS[size_index]} {R.flag_name(flags)} lambda={lam}"
                assert torch.equal(lo.view(torch.int32), l0.view(torch.int32)), f"{label}: losses depend on lambda"
                if not flags & R.LOSS_PO2PL:
                    assert torch.equal(g, g0), f"{label}: lambda changes a gradient without po2pl"
                    continue
                want = lam * g_pl.double()
                err = ((g.double() - g0.double()) - want).abs()
                # a few roundings of the finalize's fp32 sum, each within an ulp of the larger of its terms
                bound = 8 * 2.0 ** -24 * (g.double().abs() + g0.double().abs() + want.abs()) + 1e-30
                assert bool((err <= bound).all()), f"{label}: worst {(err / bound).max().item():.2f} x the bound"
                assert float(want.abs().max()) > 0


def test_point_grads_against_float64(cuda_lib):
    """delora_icp_point_grads after a CSR call with T = None (the ICPLosses drop-in: already transformed source lists)
    at 64x720, upstream (0.7, 1.3, 2.1)."""
    from delora_b200 import ops
    bt = batch(2)
    k = 1
    ns = bt.n_host[B + k]
    p4, q4 = bt.pts4[B + k:B + k + 1].clone(), bt.nrm4[B + k:B + k + 1].clone()
    s, n_s = R.apply_rigid(bt.T[k].cpu().numpy(), p4[0, :ns, :3].cpu().numpy(), q4[0, :ns, :3].cpu().numpy())
    p4[0, :ns, :3] = torch.from_numpy(s).to(DEV)
    q4[0, :ns, :3] = torch.from_numpy(n_s).to(DEV)
    q4[0, :ns, 3] = torch.from_numpy((n_s != 0).any(axis=1).astype(np.float32)).to(DEV)
    nt = bt.n_host[k]
    tgt4 = bt.pts4[k:k + 1].cpu()
    pr = R.prepare(s, n_s, None, tgt4[0, :nt, :3].numpy(), bt.nrm4[k, :nt, :3].cpu().numpy(),
                   bt.nrm4[k, :nt, 3].cpu().numpy() != 0)
    up = torch.tensor([UPSTREAM], device=DEV)
    for flags in FLAGS:
        losses, _, nn_index, pdir, ndir = ops.icp_fwd_bwd(p4, q4, bt.counts[B + k:B + k + 1].contiguous(), None,
                                                          bt.pts4[k:k + 1].contiguous(), bt.nrm4[k:k + 1].contiguous(),
                                                          bt.cs[k:k + 1].contiguous(), bt.h, bt.w, bt.hf, bt.vf,
                                                          flags=flags, pointwise=True)
        gp, gn = ops.icp_point_grads(pdir, ndir, bt.counts[B + k:B + k + 1].contiguous(), losses, up)
        res = R.evaluate(pr, flags, 1.0, upstream=UPSTREAM)
        label = f"point grads {R.flag_name(flags)}"
        assert torch.equal(nn_index[0, :ns].cpu(), bt.tags[k][pr.nn]), label
        assert int(losses[0, 3]) == res.M and int(losses[0, 4]) == res.Mp, label
        for name, got, want in (("points", gp, res.grad_pts), ("normals", gn, res.grad_nrm)):
            got = got[0].double().cpu().numpy()
            assert not got[:, ns:].any(), f"{label}: {name} beyond the list"
            got = got[:, :ns].T
            scale = np.abs(want).max()
            if scale == 0.0:
                assert not got.any(), f"{label}: {name} want exactly 0"
                continue
            err = np.abs(got - want).max() / scale
            _note(f"point grads {name}", err)
            assert err <= POINT_TOL, f"{label}: {name} differ from float64 by {err:.3e} of their max-abs"
    print("\n[64x720] per-point gradients against float64:", flush=True)
    _report("point grads")


@pytest.mark.parametrize("size_index", range(len(SIZES)), ids=SIZE_IDS)
def test_batch_independence_and_determinism(size_index, cuda_lib):
    """Every pair of the B = 6 call is bit-identical to a B = 1 call on that pair alone (same strides, a scratch
    zeroed for each B); a repeated call is bit-identical; one scratch reused over the whole flag matrix (different
    kernel instantiations one after the other) gives the bits of a fresh one."""
    bt = batch(size_index)
    shared = {"dense": scratch(B, bt), "csr": scratch(B, bt)}
    single = {"dense": scratch(1, bt), "csr": scratch(1, bt)}
    bits = lambda t: t.view(torch.int32).cpu()          # noqa: E731
    for flags in FLAGS:
        lam = 10.0
        for kern in ("dense", "csr"):
            run = bt.dense if kern == "dense" else (lambda *a, **kw: bt.csr(*a, **kw)[:2])
            fresh = [bits(x) for x in run(flags, lam, scratch(B, bt))]
            reused = [bits(x) for x in run(flags, lam, shared[kern])]
            again = [bits(x) for x in run(flags, lam, shared[kern])]
            label = f"{kern} {SIZE_IDS[size_index]} {R.flag_name(flags)}"
            assert all(torch.equal(a, b) for a, b in zip(fresh, reused)), f"{label}: reused scratch differs"
            assert all(torch.equal(a, b) for a, b in zip(fresh, again)), f"{label}: repeated call differs"
            for k in range(B):
                one = [bits(x) for x in run(flags, lam, single[kern], pairs=(k, k + 1))]
                assert torch.equal(one[0][0], fresh[0][k]) and torch.equal(one[1][0], fresh[1][k]), \
                    f"{label}: pair {k} alone differs from pair {k} of the batch"


def test_empty_target_grid(cuda_lib):
    """B = 2, the second pair's target grid (list) empty: every lane of that pair reaches the dense path's block search
    without a candidate; losses and grad_T are 0, M = M' = 0, and the first pair is unaffected."""
    from delora_b200 import ops
    bt = batch(0)
    e = B + 5                                                 # the empty source grid of pair 5 serves as target
    src, tgt = [B + 1, B + 1], [1, e]
    T = torch.stack((bt.T[1], bt.T[1])).contiguous()
    ns = bt.n_host[B + 1]
    for flags in FLAGS + [R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL | ops.ICP_STATS]:
        if flags & ops.ICP_STATS:
            ops.icp_stats(reset=True)
        lo, g = ops.icp_dense_fwd_bwd(bt.pg[src].contiguous(), bt.ng[src].contiguous(), T, bt.pg[tgt].contiguous(),
                                      bt.ng[tgt].contiguous(), bt.h, bt.w, bt.hf, bt.vf, flags=flags)
        l1, g1 = bt.dense(flags & ~ops.ICP_STATS, 1.0, pairs=(1, 2))
        lc, gc, nn_index, _, _ = ops.icp_fwd_bwd(bt.pts4[src].contiguous(), bt.nrm4[src].contiguous(),
                                                 bt.counts[src].contiguous(), T, bt.pts4[tgt].contiguous(),
                                                 bt.nrm4[tgt].contiguous(), bt.cs[tgt].contiguous(), bt.h, bt.w, bt.hf,
                                                 bt.vf, flags=flags, pointwise=True)
        torch.cuda.synchronize()
        label = R.flag_name(flags)
        assert torch.equal(lo[0], l1[0]) and torch.equal(g[0], g1[0]), f"{label}: the first pair changed"
        for kern, x, y in (("dense", lo, g), ("csr", lc, gc)):
            assert not x[1].any() and not y[1].any(), f"{kern} {label}: {x[1].tolist()} {y[1].tolist()}"
            assert float(x[0, 3]) > 0, f"{kern} {label}: the first pair has no pairs"
        assert bool((nn_index[1, :ns] == -1).all()), f"csr {label}: NN found in an empty target"
        if flags & ops.ICP_STATS:
            st = ops.icp_stats(reset=True)
            assert st["owners_without_candidate"] >= ns, st


@pytest.mark.parametrize("flags", [R.LOSS_PO2PO, R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL | R.NORMAL_LINEAR],
                         ids=R.flag_name)
def test_po2po_kernels_under_the_hand_over_limit_and_stats(flags, cuda_lib, monkeypatch):
    """The PO2PO instantiations of the window search and of the block search (which ADDs columns 24-37 to the
    window search's partial rows) at hand-over limits 0 (every open warp goes to the block search) and 100000
    (none does), and with DELORA_ICP_STATS."""
    from delora_b200 import ops
    bt = batch(2)
    lam = 10.0
    base_l, base_g = (x.cpu() for x in bt.dense(flags, lam))
    ops.icp_stats(reset=True)
    st_l, st_g = (x.cpu() for x in bt.dense(flags | ops.ICP_STATS, lam))
    st = ops.icp_stats(reset=True)
    assert torch.equal(st_l, base_l) and torch.equal(st_g, base_g), "DELORA_ICP_STATS changes the results"
    assert st["warps_block_search"] > 0 and st["block_owners"] > 0, st
    for limit in ("0", "100000"):
        monkeypatch.setenv("DELORA_ICP_MAX_STRIPS", limit)
        lo, g = (x.cpu() for x in bt.dense(flags, lam))
        assert torch.equal(lo[:, 3:], base_l[:, 3:]), f"limit {limit}: pair counts differ"
        assert torch.allclose(lo[:, :3], base_l[:, :3], rtol=2e-6, atol=0), f"limit {limit}: losses differ"
        scale = base_g.abs().amax(dim=1, keepdim=True)
        assert bool(((g - base_g).abs() <= 1e-4 * scale).all()), f"limit {limit}: grad_T differs"
        for k in range(B):
            l_err, g_err = check_pair(f"limit {limit} pair {k}", lo[k], g[k], R.evaluate(bt.ref[k], flags, lam))
            _note("hand-over limit loss", l_err)
            _note("hand-over limit grad_T", g_err)
    monkeypatch.delenv("DELORA_ICP_MAX_STRIPS")
    print(f"\n[64x720 {R.flag_name(flags)}] hand-over limits 0 and 100000 against float64:", flush=True)
    _report("hand-over")


TRAIN_SETTINGS = [(R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL | R.NORMAL_LINEAR, 10.0), (R.LOSS_PO2PL | R.LOSS_PL2PL, 0.25)]


@pytest.mark.parametrize("h,w,w_raw", [(16, 259, 512), (64, 720, 1024)], ids=["16x259", "64x720"])
@pytest.mark.parametrize("flags,lam", TRAIN_SETTINGS, ids=["all-linear-lambda10", "po2pl+pl2pl-lambda0.25"])
def test_training_step_with_non_default_loss_settings(h, w, w_raw, flags, lam, cuda_lib):
    """delora_odometry_train_step with hp->loss_flags and hp->lambda_po2pl away from their defaults, against the Python
    training step with the same settings (the bars of test_step_matches_the_python_training_step)."""
    b = 2
    cfg = H.config(h, w)
    cfg["lambda_po2pl"] = lam
    model = H.model(cfg, near_identity=True)
    pairs = H.pairs(h, w_raw, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    tr = H.trainer(cfg, n_stride, b, H.blob(model, cfg), flags=flags)
    losses, T, pooled, grads = tr.step(pts, counts)
    py = H.python_step(model, cfg, pts, counts, flags=flags)
    torch.cuda.synchronize()
    assert torch.equal(pooled, py.pooled), "pooled features differ from TensorCoreEncoder.pooled_features"
    t_err = (T - py.T).abs().max().item()
    assert t_err <= 1e-5, f"max |T - T_py| = {t_err:.3e}"
    if flags & R.LOSS_PO2PO:
        assert bool((py.losses[:, 0] > 0).all()) and bool((py.losses[:, 4] > 0).all())
    else:
        assert not py.losses[:, 0].any() and not py.losses[:, 4].any()
    l_err = H.rel(losses[:, :3], py.losses[:, :3])
    assert l_err <= 1e-5, f"losses differ by {l_err:.3e} (relative)"
    tail, trunk = H.grad_spread(H.grad_dict(grads, cfg), py.grads)
    print(f"\n[{h}x{w} B={b} {R.flag_name(flags)} lambda={lam}] T {t_err:.2e}  losses {l_err:.2e}  grads: tail "
          f"{tail:.2e}, trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL, f"fc / head gradients differ by {tail:.3e} of their max-abs"
    assert trunk <= H.TRUNK_TOL, f"trunk gradients differ by {trunk:.3e} of their max-abs"
