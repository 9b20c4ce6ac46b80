"""-m "not gpu": the information in metres for normalised pairs (delora_icp_dense_information_scaled) and the recipe and
adapting streams with the information (delora_odometry_streams_pre_info_*, _adapt_info_*) without a device -- the metric
form D H D against finite differences of the normalised objective, the workspace sizes as the existing layouts plus one
section, the exported symbols with the unchanged ABI, and every refusal by name."""
import ctypes

import numpy as np
import pytest

import icp_reference as R
import info_reference as IR
import odometry_harness as H
from delora_b200 import ops

NEW_SYMBOLS = ("delora_icp_dense_information_scaled", "delora_odometry_streams_pre_info_workspace_bytes",
               "delora_odometry_streams_pre_info_init", "delora_odometry_streams_push_pre_info",
               "delora_odometry_streams_adapt_info_workspace_bytes", "delora_odometry_streams_adapt_info_init",
               "delora_odometry_streams_push_adapt_info", "delora_odometry_streams_push_adapt_group_info")
ICP = ops.LOSS_PO2PL | ops.LOSS_PL2PL


def _L():
    from delora_b200 import _lib
    return _lib.lib()


def metric(Hn, f):
    """H in metres and radians of a pair whose clouds were divided by f: D H D, D = diag(1/f, 1/f, 1/f, 1, 1, 1)."""
    D = np.diag([1.0 / f] * 3 + [1.0] * 3)
    return D @ np.asarray(Hn, np.float64) @ D


def _design(seed, f, n=64):
    """A pair in metres (targets the sources moved by T, then perturbed; a quarter with a normal on neither side) and
    the same pair divided by f, with T's translation divided by f: the normalised model's ICP inputs."""
    g = np.random.default_rng(seed)
    p = g.uniform(-30, 30, (n, 3))
    m = g.normal(size=(n, 3))
    m /= np.linalg.norm(m, axis=1, keepdims=True)
    bare = np.arange(n) < n // 4
    m[bare] = 0.0
    ax = g.normal(size=3)
    T4 = IR.exp_se3(np.concatenate([g.uniform(-2, 2, 3), 0.2 * ax / np.linalg.norm(ax)]))
    tgt_p = p @ T4[:3, :3].T + T4[:3, 3] + g.normal(scale=0.05, size=(n, 3))
    tgt_n = m @ T4[:3, :3].T + g.normal(scale=0.1, size=(n, 3)) * ~bare[:, None]
    tgt_n = np.where(~bare[:, None], tgt_n / np.maximum(np.linalg.norm(tgt_n, axis=1, keepdims=True), 1e-30), 0.0)
    Tn = T4[:3, :].copy()
    Tn[:, 3] /= f
    return Tn, p / f, m, tgt_p / f, tgt_n, ~bare, np.arange(n)


@pytest.mark.parametrize("f", [0.05, 0.3, 1.0, 7.0])
@pytest.mark.parametrize("flags", R.flag_matrix(), ids=R.flag_name)
def test_metric_form_is_gauss_newton_of_the_normalised_objective_in_metres(flags, f):
    """The normalised objective as a function of the metric perturbation xi_m = (rho, phi) of the served T: its
    residuals at T_n Exp((rho / f, phi)), J by central differences in xi_m; 2 J^T J must be D H D of the normalised
    restatement (a normalised translation of rho / f is rho metres)."""
    Tn, p, m, tgt_p, tgt_n, tgt_has, nn = _design(31 + flags, f)
    lam = 0.7
    Hn, _, _, _ = IR.information(Tn, p, m, tgt_n, tgt_has, nn, flags, lam)
    kind = IR.pair_masks(Tn, p, m, tgt_n, tgt_has, nn, flags)
    scale = np.array([1.0 / f] * 3 + [1.0] * 3)
    res = lambda xi_m: IR.residuals(Tn, xi_m * scale, p, m, tgt_p, tgt_n, kind, nn, flags, lam)
    J = IR.fd_jacobian(res, h=1e-6 * min(f, 1.0))
    gn = 2.0 * J.T @ J
    Hm = metric(Hn, f)
    assert np.abs(Hm - gn).max() <= 1e-6 * np.abs(Hm).max(), np.abs(Hm - gn).max() / np.abs(Hm).max()
    if f != 1.0 and flags & (R.LOSS_PO2PO | R.LOSS_PO2PL):
        # the translation block is what changes: H itself is the Hessian in the normalised units
        assert not np.allclose(Hm[:3, :3], Hn[:3, :3])
    np.testing.assert_array_equal(Hm[3:, 3:], Hn[3:, 3:])


def test_metric_form_keeps_the_unit_factor_exact():
    g = np.random.default_rng(2)
    X = g.normal(size=(6, 6))
    Hn = X @ X.T
    np.testing.assert_array_equal(metric(Hn, 1.0), Hn)


def test_symbols_exported_and_the_abi_and_structs_stay():
    from delora_b200 import _lib
    L = _L()
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert hasattr(handle, name), name
        assert name in _lib.SIGNATURES, name
    assert L.delora_abi_version() == 3 == _lib.ABI_VERSION
    assert ctypes.sizeof(_lib.OdometryDesc) == 80
    assert ctypes.sizeof(_lib.OdometryResidualParams) == 24
    assert ctypes.sizeof(_lib.OdometryTrainParams) == 40
    assert ops.INFO_ROW == IR.INFO_ROW == 80


def _section(L, S, h, w):
    return H.align(S * IR.INFO_ROW * 4) + H.align(L.delora_icp_information_scratch_floats(S, h, w) * 4)


@pytest.mark.parametrize("h,w", [(64, 720), (64, 2048)])
@pytest.mark.parametrize("S", [1, 4, 16])
def test_pre_info_workspace_is_the_recipe_layout_plus_the_information_section(h, w, S):
    L = _L()
    dp = ctypes.byref(H.desc(H.config(h, w, device="cpu"), 131072, S, 2250))
    pre = L.delora_odometry_streams_pre_workspace_bytes(dp)
    assert pre > 0 and L.delora_odometry_streams_pre_info_workspace_bytes(dp) == pre + _section(L, S, h, w)


@pytest.mark.parametrize("w_pre", [0, 2250])
@pytest.mark.parametrize("h,w", [(64, 720), (64, 2048)])
@pytest.mark.parametrize("S", [1, 4, 16])
def test_adapt_info_workspace_is_the_group_layout_plus_the_information_section(h, w, S, w_pre):
    L = _L()
    dp = ctypes.byref(H.streams_desc(h, w, S, w_pre, 131072))
    group = L.delora_odometry_streams_adapt_group_workspace_bytes(dp)
    assert group > L.delora_odometry_streams_adapt_workspace_bytes(dp) > 0
    assert L.delora_odometry_streams_adapt_info_workspace_bytes(dp) == group + _section(L, S, h, w)


def test_queries_refuse_invalid_descriptors_by_name():
    L = _L()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 2, 0)
    dp = ctypes.byref(d)
    assert L.delora_odometry_streams_pre_info_workspace_bytes(dp) == -1
    err = L.delora_last_error()
    assert b"delora_odometry_streams_pre_info_workspace_bytes" in err and b"w_pre=0" in err, err
    assert L.delora_odometry_streams_pre_info_init(dp, 16, None) != 0
    assert b"delora_odometry_streams_pre_info_init: w_pre=0" in L.delora_last_error()
    d.w_pre = 2250
    assert L.delora_odometry_streams_pre_info_init(dp, None, None) != 0
    assert b"delora_odometry_streams_pre_info_init: null workspace" in L.delora_last_error()
    d.act = 0
    assert L.delora_odometry_streams_adapt_info_workspace_bytes(dp) == -1
    assert b"delora_odometry_streams_adapt_info_workspace_bytes: act=0" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_info_init(dp, 16, 32, None) != 0
    assert b"delora_odometry_streams_adapt_info_init: act=0" in L.delora_last_error()
    assert L.delora_odometry_streams_adapt_info_init(ctypes.byref(H.streams_desc()), None, 32, None) != 0
    assert b"delora_odometry_streams_adapt_info_init: null pointer" in L.delora_last_error()


# ------------------------------------------------------------------------------------------ the scaled operator
def _scaled(args, info=16, info_scratch=16, factor=16):
    L = _L()
    rc = L.delora_icp_dense_information_scaled(*args, info, info_scratch, factor, None)
    return rc, L.delora_last_error()


def test_scaled_operator_refuses_by_name():
    name = b"delora_icp_dense_information_scaled"
    args = [16, 16, 16, 16, 16, 1, 16, 16, -3.14, 3.14, -0.4, 0.05, 1.0, ICP, 16, 16, 16]
    rc, err = _scaled(args, factor=None)
    assert rc != 0 and name + b": null factor" in err, err
    rc, err = _scaled(args, info=None)
    assert rc != 0 and name + b": null pointer" in err, err
    rc, err = _scaled(args, info_scratch=None)
    assert rc != 0 and name + b": null pointer" in err, err
    args[13] = ICP | 256
    rc, err = _scaled(args)
    assert rc != 0 and b"DELORA_ICP_STATS" in err and name in err, err
    args[13] = ICP
    args[5] = 0
    rc, err = _scaled(args)
    assert rc != 0 and name + b": bad shape" in err, err
    args[5] = 1
    args[14] = None
    rc, err = _scaled(args)
    assert rc != 0 and name + b": null pointer" in err, err


# ------------------------------------------------------------------------------------------ _push_pre_info
PRE = "delora_odometry_streams_push_pre_info"


def _rp(flags=ICP):
    from delora_b200 import _lib
    return _lib.OdometryResidualParams(lambda_po2pl=1.0, loss_flags=flags, nb_h=7, nb_w=11, epsilon_range=0.5,
                                       min_neighbors=10)


def _push_pre(rp=None, factor=None, w_pre=2250, **null):
    L = _L()
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80, "losses": 96, "info": 112}
    args.update(null)
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 2, w_pre)
    rc = getattr(L, PRE)(ctypes.byref(d), None if rp is False else ctypes.byref(rp or _rp()), args["points"],
                         args["n_points"], None, args["workspace"], args["T"], args["valid"], args["losses"], factor,
                         args["info"], None)
    return rc, L.delora_last_error()


@pytest.mark.parametrize("missing", ["points", "n_points", "workspace", "T", "valid", "losses", "info"])
def test_push_pre_info_refuses_null_pointers_by_name(missing):
    rc, err = _push_pre(**{missing: None})
    assert rc != 0 and f"{PRE}: null {missing}".encode() in err, err


@pytest.mark.parametrize("kw,what", [
    ({"rp": False}, b"null residual_params"), ({"w_pre": 0}, b"w_pre=0"), ({"w_pre": 1}, b"w_pre=1"),
    ({"rp": _rp(ops.LOSS_PO2PL | 16)}, b"loss_flags=0x12 has a bit other"),
    ({"rp": _rp(ops.NORMAL_LINEAR)}, b"sets no loss bit"),
    ({"rp": _rp(ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING)}, b"null factor with DELORA_TRAIN_NORMALIZATION"),
    ({"rp": _rp(ops.LOSS_PO2PL), "factor": 112}, b"factor must be NULL without"),
])
def test_push_pre_info_refuses_what_push_pre_refuses(kw, what):
    rc, err = _push_pre(**kw)
    assert rc != 0 and PRE.encode() in err and what in err, err


def test_push_pre_info_checks_info_after_the_push_pre_checks():
    rc, err = _push_pre(rp=_rp(ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING), info=None)
    assert rc != 0 and f"{PRE}: null factor".encode() in err, err


# ------------------------------------------------------------------------------------------ _push_adapt(_group)_info
ADAPT = "delora_odometry_streams_push_adapt_info"
GROUP = "delora_odometry_streams_push_adapt_group_info"


def _group(world=2, rank=0, ws=48):
    from delora_b200 import _lib
    g = _lib.OdometryTrainGroup(rank=rank, world=world, multicast=0, n_ctas=8, n_threads=128, status=16,
                                side_stream=None, join_event=16)
    for q in range(world):
        g.peer_ws[q] = ws if q == rank else 4096 * (q + 1)
        g.peer_flags[q] = 8192 * (q + 1)
    for k in range(_lib.TRAIN_GROUP_BUCKETS):
        g.fork_events[k] = 16
    return g


def _push_adapt(name, hp=None, update=1, g=None, **null):
    L = _L()
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80, "losses": 96, "info": 112}
    args.update(null)
    head = [ctypes.byref(H.streams_desc()), None if hp is False else ctypes.byref(hp or H.train_params())]
    if name == GROUP:
        head.append(None if g is False else ctypes.byref(g or _group()))
    rc = getattr(L, name)(*head, update, args["points"], args["n_points"], None, args["workspace"], args["T"],
                          args["valid"], args["losses"], args["info"], None)
    return rc, L.delora_last_error()


@pytest.mark.parametrize("name", [ADAPT, GROUP])
@pytest.mark.parametrize("missing", ["points", "n_points", "workspace", "T", "valid", "losses", "info"])
def test_push_adapt_info_refuses_null_pointers_by_name(name, missing):
    rc, err = _push_adapt(name, **{missing: None})
    assert rc != 0 and f"{name}: null {missing}".encode() in err, err


@pytest.mark.parametrize("name", [ADAPT, GROUP])
@pytest.mark.parametrize("kw,what", [
    ({"update": 2}, b"update=2 must be 0 or 1"), ({"hp": False}, b"null hyperparameters"),
    ({"hp": H.train_params(ops.LOSS_PO2PL | ops.LOSS_IDENTITY_FIT)}, b"DELORA_LOSS_IDENTITY_FIT"),
    ({"hp": H.train_params(ops.LOSS_PO2PL | ops.TRAIN_DROPOUT)}, b"DELORA_TRAIN_DROPOUT"),
    ({"hp": H.train_params(ops.LOSS_PO2PL | ops.TRAIN_NORMALIZATION_SCALING)},
     b"DELORA_TRAIN_NORMALIZATION_SCALING needs w_pre > 0"),
])
def test_push_adapt_info_refuses_what_push_adapt_refuses(name, kw, what):
    rc, err = _push_adapt(name, **kw)
    assert rc != 0 and name.encode() in err and what in err, err


@pytest.mark.parametrize("g,what", [(False, b"null group"), (_group(world=0), b"world=0 must be in [1, 16]"),
                                    (_group(rank=1, ws=4096 * 2), b"peer_ws[rank=1] is not the workspace")])
def test_push_adapt_group_info_refuses_the_group_by_name(g, what):
    rc, err = _push_adapt(GROUP, g=g)
    assert rc != 0 and GROUP.encode() in err and what in err, err
