"""The float64 ICP reference (tests/icp_reference.py) checked on the CPU, on the small_16x180 golden pair, for every
loss configuration the GPU tests use:
  - its losses agree with the oracle's fp32 restatement of ICPLosses (orc.icp_losses) to 1e-5 relative, with the same
    nearest neighbours and the same pair count;
  - its emulated fp32 transform is within the rounding bound of the fp32 chain of the float64 R p + t (half an ulp
    of the summed term magnitudes per rounding; measured 1.34 ulp for points);
  - its grad_T is the derivative of its objective: central finite differences in float64 with the NN held fixed."""
import os

import numpy as np
import pytest
import torch

import icp_reference as R
from helpers import GOLDEN
from oracle import delora_oracle as orc


def golden_pair():
    z = np.load(os.path.join(GOLDEN, "small_16x180.npz"))
    from delora_b200 import synthetic
    import json
    with open(os.path.join(GOLDEN, "golden.json")) as f:
        meta = json.load(f)["small_16x180"]
    t_pred = synthetic.make_pair(meta["pair_index"], w_raw=meta["w_raw"], rings=meta["rings"],
                                 vfov_deg=tuple(meta["vfov_deg"]))[3]
    # a quarter of the target's normals dropped as well, so that po2po pairs have targets without a normal
    tgt_n, tgt_has = z["normals_1"].copy(), z["has_normal_1"].copy()
    drop = np.random.default_rng(3).random(len(tgt_has)) < 0.25
    tgt_n[drop] = 0.0
    tgt_has &= ~drop
    src_n = z["normals_2"].copy()
    src_n[np.random.default_rng(4).random(len(src_n)) < 0.25] = 0.0
    return z["points_2"], src_n, t_pred[:3, :].numpy(), z["points_1"], tgt_n, tgt_has


@pytest.fixture(scope="module")
def pair():
    src_p, src_n, T, tgt_p, tgt_n, tgt_has = golden_pair()
    return R.prepare(src_p, src_n, T, tgt_p, tgt_n, tgt_has), (src_p, src_n, T, tgt_p, tgt_n, tgt_has)


@pytest.mark.parametrize("flags", R.flag_matrix(), ids=R.flag_name)
def test_losses_match_the_fp32_oracle(pair, flags):
    pr, (src_p, src_n, T, tgt_p, tgt_n, tgt_has) = pair
    t4 = torch.eye(4)
    t4[:3, :] = torch.from_numpy(T)
    t4 = t4.view(1, 4, 4)
    src = orc.transform_point_cloud(t4, torch.from_numpy(src_p).t()[None]).contiguous()
    src_nt = orc.rotate_point_cloud(t4, torch.from_numpy(src_n).t()[None]).contiguous()
    lo, aux = orc.icp_losses(src, src_nt, torch.from_numpy(tgt_p).t()[None].contiguous(),
                             torch.from_numpy(tgt_n).t()[None].contiguous(),
                             point_to_point_loss=bool(flags & R.LOSS_PO2PO),
                             point_to_plane_loss=bool(flags & R.LOSS_PO2PL),
                             plane_to_plane_loss=bool(flags & R.LOSS_PL2PL),
                             normal_loss="linear" if flags & R.NORMAL_LINEAR else "squared", return_aux=True)
    assert torch.equal(aux["nn_index"], pr.nn), "the oracle's transform gives other nearest neighbours"
    res = R.evaluate(pr, flags)
    assert res.M == aux["num_pairs"]
    if flags & R.LOSS_PO2PO:
        assert res.Mp > 100
    else:
        assert res.Mp == 0
    for j, key in enumerate(("loss_po2po", "loss_po2pl", "loss_pl2pl")):
        want = float(lo[key])
        assert (want != 0.0) == bool(flags & (R.LOSS_PO2PO, R.LOSS_PO2PL, R.LOSS_PL2PL)[j]), key
        assert res.losses[j] == pytest.approx(want, rel=1e-5, abs=0), key


def test_emulated_transform_within_one_ulp(pair):
    _, (src_p, src_n, T, _, _, _) = pair
    s, ns = R.apply_rigid(T, src_p, src_n)
    T64 = T.astype(np.float64)
    # every rounding of the chain (r0 x, two fmaf, + t for points) is at most half an ulp of the sum of the terms'
    # magnitudes: 2 ulp for points, 1.5 ulp for normals; the float64 emulation adds nothing measurable
    for got, v, t, bound in ((s, src_p, T64[:, 3], 2.0), (ns, src_n, np.zeros(3), 1.5)):
        exact = v.astype(np.float64) @ T64[:, :3].T + t
        scale = np.abs(v.astype(np.float64)) @ np.abs(T64[:, :3]).T + np.abs(t)
        err = np.abs(got.astype(np.float64) - exact)
        ulps = err / np.spacing(scale.astype(np.float32)).astype(np.float64)
        print(f"worst error {ulps.max():.3f} ulp of the summed term magnitudes (bound {bound})")
        assert ulps.max() <= bound
    # the fmaf emulation rounds once: exact on products that fit fp32, and different from mul-then-add
    a, c = np.float32(1 + 2 ** -12), np.float32(-(1 + 2 ** -11))
    assert R.fmaf(a, a, c) == np.float32(2.0 ** -24)
    assert np.float32(a * a) + c == np.float32(0.0)


@pytest.mark.parametrize("flags,lam", [(R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL, 1.0),
                                       (R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL | R.NORMAL_LINEAR, 10.0),
                                       (R.LOSS_PO2PL | R.LOSS_PL2PL, 0.25), (R.LOSS_PO2PO, 1.0)],
                         ids=["all", "all-linear-lambda10", "po2pl+pl2pl-lambda0.25", "po2po"])
def test_grad_T_matches_finite_differences(flags, lam):
    src_p, src_n, T, tgt_p, tgt_n, tgt_has = golden_pair()
    pr = R.prepare(src_p[::8], src_n[::8], T, tgt_p, tgt_n, tgt_has)     # ~330 source points
    res = R.evaluate(pr, flags, lam)
    assert res.M > 50 and (res.Mp > 20 or not flags & R.LOSS_PO2PO)
    h = 1e-4
    fd = np.zeros((3, 4))
    for i in range(3):
        for j in range(4):
            dT = torch.zeros((3, 4), dtype=torch.float64)
            dT[i, j] = h
            fd[i, j] = (float(R.objective(pr, flags, lam, dT)) - float(R.objective(pr, flags, lam, -dT))) / (2 * h)
    err = np.abs(fd - res.grad_T).max() / np.abs(res.grad_T).max()
    print(f"grad_T vs central differences: {err:.2e} of max-abs")
    assert err <= 1e-8


def test_empty_sets_give_zero():
    src_p, src_n, T, tgt_p, tgt_n, tgt_has = golden_pair()
    flags = R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL
    # no normals anywhere: M = 0, every pair is a po2po pair
    pr = R.prepare(src_p, np.zeros_like(src_n), T, tgt_p, np.zeros_like(tgt_n), np.zeros_like(tgt_has))
    res = R.evaluate(pr, flags, upstream=(0.7, 1.3, 2.1))
    assert res.M == 0 and res.Mp == len(src_p)
    assert res.losses[1] == 0.0 and res.losses[2] == 0.0 and res.losses[0] > 0.0
    assert np.isfinite(res.grad_T).all() and np.abs(res.grad_T).max() > 0
    assert not np.abs(res.grad_nrm).any()
    # empty source, and empty target: everything 0
    for pr in (R.prepare(src_p[:0], src_n[:0], T, tgt_p, tgt_n, tgt_has),
               R.prepare(src_p, src_n, T, tgt_p[:0], tgt_n[:0], tgt_has[:0])):
        res = R.evaluate(pr, flags, upstream=(0.7, 1.3, 2.1))
        assert (res.M, res.Mp) == (0, 0)
        assert not res.losses.any() and not res.grad_T.any() and not res.grad_pts.any()
