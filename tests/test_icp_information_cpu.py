"""-m "not gpu": the Gauss-Newton information of the ICP objective (delora_icp_dense_information) and the information
streams (delora_odometry_streams_info_*, _push_info) without a device -- the float64 restatement against finite
differences, the exported symbols with the unchanged ABI, the workspace as the residual layout plus one section, and
every refusal."""
import ctypes

import numpy as np
import pytest

import icp_reference as R
import info_reference as IR
import odometry_harness as H

NEW_SYMBOLS = ("delora_icp_information_scratch_floats", "delora_icp_dense_information",
               "delora_odometry_streams_info_workspace_bytes", "delora_odometry_streams_info_init",
               "delora_odometry_streams_push_info")


def _L():
    from delora_b200 import _lib
    return _lib.lib()


def _design(seed, n=64, po2po_share=0.25):
    """A smooth pair whose every residual is zero at T: targets are the sources moved by T (float64, rounded to fp32
    once), target normals the rotated source normals; a share of the pairs has a normal on neither side."""
    g = np.random.default_rng(seed)
    p = g.uniform(-8, 8, (n, 3)).astype(np.float32)
    m = g.normal(size=(n, 3))
    m = (m / np.linalg.norm(m, axis=1, keepdims=True)).astype(np.float32)
    bare = np.arange(n) < int(po2po_share * n)
    m[bare] = 0.0
    ax = g.normal(size=3)
    T4 = IR.exp_se3(np.concatenate([g.uniform(-1, 1, 3), 0.3 * ax / np.linalg.norm(ax)]))
    T = T4[:3, :].astype(np.float32)
    Rm, t = T.astype(np.float64)[:, :3], T.astype(np.float64)[:, 3]
    tgt_p = p.astype(np.float64) @ Rm.T + t
    tgt_n = m.astype(np.float64) @ Rm.T
    return T, p, m, tgt_p, tgt_n, ~bare, np.arange(n)


@pytest.mark.parametrize("flags", [f for f in R.flag_matrix() if not f & R.NORMAL_LINEAR], ids=R.flag_name)
@pytest.mark.parametrize("lam", [1.0, 0.3])
def test_reference_is_the_hessian_of_the_objective(flags, lam):
    """Where every residual is zero the Hessian of the objective in xi is exactly its Gauss-Newton approximation, so
    the restatement must equal central second differences of the float64 objective (the means included: po2po over
    3 M' coordinates)."""
    T, p, m, tgt_p, tgt_n, tgt_has, nn = _design(7 + flags)
    Hm, A, M, Mp = IR.information(T, p, m, tgt_n.astype(np.float32), tgt_has, nn, flags, lam)
    kind = IR.pair_masks(T, p, m, tgt_n, tgt_has, nn, flags)
    fd = IR.fd_hessian(lambda xi: IR.objective(T, xi, p, m, tgt_p, tgt_n, kind, nn, flags, lam))
    scale = np.abs(Hm).max()
    assert scale > 0
    # the design rounds T and n_t to fp32 once: the reference's Jacobians see those bits, the objective float64 ones
    assert np.abs(Hm - fd).max() <= 2e-5 * scale, (np.abs(Hm - fd).max(), scale)
    assert np.allclose(Hm, Hm.T)
    assert M == int(tgt_has.sum()) and Mp == (len(p) - M if flags & R.LOSS_PO2PO else 0)
    assert np.all(np.abs(Hm) <= A + 1e-12)


@pytest.mark.parametrize("flags", R.flag_matrix(), ids=R.flag_name)
def test_reference_is_gauss_newton_of_the_residuals_away_from_zero(flags):
    """With non-zero residuals (perturbed targets and normals) the restatement is 2 J^T J of the weighted residual
    vector whose squares sum to the objective, J by central differences in xi."""
    T, p, m, tgt_p, tgt_n, tgt_has, nn = _design(19 + flags)
    g = np.random.default_rng(flags)
    tgt_p = (tgt_p + g.normal(scale=0.05, size=tgt_p.shape)).astype(np.float32).astype(np.float64)
    tgt_n = tgt_n + g.normal(scale=0.1, size=tgt_n.shape) * tgt_has[:, None]
    tgt_n = np.where(tgt_has[:, None], tgt_n / np.maximum(np.linalg.norm(tgt_n, axis=1, keepdims=True), 1e-30), 0.0)
    tgt_n = tgt_n.astype(np.float32).astype(np.float64)
    lam = 0.7
    Hm, _, _, _ = IR.information(T, p, m, tgt_n, tgt_has, nn, flags, lam)
    kind = IR.pair_masks(T, p, m, tgt_n, tgt_has, nn, flags)
    res = lambda xi: IR.residuals(T, xi, p, m, tgt_p, tgt_n, kind, nn, flags, lam)
    xi = g.normal(scale=0.01, size=6)
    assert np.isclose(np.sum(res(xi) ** 2), IR.objective(T, xi, p, m, tgt_p, tgt_n, kind, nn, flags, lam), rtol=1e-12)
    J = IR.fd_jacobian(res)
    gn = 2.0 * J.T @ J
    assert np.abs(Hm - gn).max() <= 1e-6 * np.abs(Hm).max(), np.abs(Hm - gn).max() / np.abs(Hm).max()


def test_eigen_row_convention():
    g = np.random.default_rng(3)
    X = g.normal(size=(6, 6))
    ev, V = IR.eig_row(X @ X.T)
    assert np.all(np.diff(ev) >= 0)
    for k in range(6):
        big = int(np.argmax(np.abs(V[k])))
        assert V[k, big] > 0 and abs(np.linalg.norm(V[k]) - 1) < 1e-12


def test_symbols_exported_and_the_abi_version_stays():
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


@pytest.mark.parametrize("B,h,w", [(1, 64, 2048), (4, 64, 720), (3, 16, 181)])
def test_information_scratch_size(B, h, w):
    """NN ids (one int32 per source pixel), then a 64-float partial row per 32 source pixels."""
    L = _L()
    assert L.delora_icp_information_scratch_floats(B, h, w) == B * h * w + B * ((h * w + 31) // 32) * 64
    assert L.delora_icp_information_scratch_floats(0, h, w) == -1
    assert L.delora_icp_information_scratch_floats(B, 0, w) == -1


@pytest.mark.parametrize("h,w", [(64, 2048), (64, 720), (16, 180)])
@pytest.mark.parametrize("S", [1, 4, 16])
def test_info_workspace_is_the_residual_layout_plus_one_section(h, w, S):
    """The information workspace exceeds the residual workspace by exactly its appended section (S information rows,
    the operator's scratch at B = S, each 256-byte aligned), so no residual offset moves."""
    L = _L()
    dp = ctypes.byref(H.desc(H.config(h, w, device="cpu"), 131072, S))
    residual = L.delora_odometry_streams_residual_workspace_bytes(dp)
    info = L.delora_odometry_streams_info_workspace_bytes(dp)
    appended = H.align(S * IR.INFO_ROW * 4) + H.align(L.delora_icp_information_scratch_floats(S, h, w) * 4)
    assert residual > 0 and info == residual + appended


def _residual_params(**over):
    from delora_b200.deploy import capi
    rp = capi.residual_params(H.config(64, 720, device="cpu"))
    for k, v in over.items():
        setattr(rp, k, v)
    return rp


@pytest.mark.parametrize("missing", ["points", "n_points", "workspace", "T", "valid", "losses", "info"])
def test_push_info_refuses_null_pointers_by_name(missing):
    L = _L()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 3)
    args = {"points": 16, "n_points": 32, "workspace": 48, "T": 64, "valid": 80, "losses": 96, "info": 112}
    args[missing] = None
    rc = L.delora_odometry_streams_push_info(ctypes.byref(d), ctypes.byref(_residual_params()), args["points"],
                                             args["n_points"], None, args["workspace"], args["T"], args["valid"],
                                             args["losses"], args["info"], None)
    assert rc != 0
    assert f"delora_odometry_streams_push_info: null {missing}".encode() in L.delora_last_error()


@pytest.mark.parametrize("over,message", [
    ({"loss_flags": 0}, b"sets no loss bit"), ({"loss_flags": 2 | 256}, b"has a bit other than"),
    ({"nb_h": 4}, b"nb_h"), ({"epsilon_range": -1.0}, b"epsilon_range")])
def test_push_info_refuses_what_push_residual_refuses(over, message):
    L = _L()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 3)
    for name in ("delora_odometry_streams_push_residual", "delora_odometry_streams_push_info"):
        args = (16, 16, None, 16, 16, 16, 16) + ((16,) if name.endswith("info") else ()) + (None,)
        rc = getattr(L, name)(ctypes.byref(d), ctypes.byref(_residual_params(**over)), *args)
        err = L.delora_last_error()
        assert rc != 0 and message in err and name.encode() in err, err
    assert L.delora_odometry_streams_push_info(ctypes.byref(d), None, 16, 16, None, 16, 16, 16, 16, 16, None) != 0
    assert b"null residual_params" in L.delora_last_error()


def test_info_queries_refuse_invalid_descriptors():
    L = _L()
    d = H.desc(H.config(64, 720, device="cpu"), 1000, 1)
    d.max_batch = 0
    dp = ctypes.byref(d)
    assert L.delora_odometry_streams_info_workspace_bytes(dp) == -1
    assert b"delora_odometry_streams_info_workspace_bytes" in L.delora_last_error()
    assert L.delora_odometry_streams_info_init(dp, 16, None) != 0
    assert b"max_batch=0" in L.delora_last_error()
    d.max_batch = 1
    assert L.delora_odometry_streams_info_init(dp, None, None) != 0
    assert b"delora_odometry_streams_info_init: null workspace" in L.delora_last_error()


def test_operator_refuses_null_outputs_and_stats():
    L = _L()
    args = [16, 16, 16, 16, 16, 1, 16, 16, -3.14, 3.14, -0.4, 0.05, 1.0, 6, 16, 16, 16]
    assert L.delora_icp_dense_information(*args, None, 16, None) != 0
    assert b"delora_icp_dense_information: null pointer" in L.delora_last_error()
    assert L.delora_icp_dense_information(*args, 16, None, None) != 0
    args[13] = 6 | 256
    assert L.delora_icp_dense_information(*args, 16, 16, None) != 0
    assert b"DELORA_ICP_STATS" in L.delora_last_error()
    args[13] = 6
    args[5] = 0
    assert L.delora_icp_dense_information(*args, 16, 16, None) != 0
    assert b"delora_icp_dense_information: bad shape" in L.delora_last_error()
