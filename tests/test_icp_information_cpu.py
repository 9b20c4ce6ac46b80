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
import projection_reference as PR

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


def test_vectorised_restatement_is_the_sum_over_pairs():
    """information and term_sums (every pair's Jacobians at once) equal the weighted sum of each pair's `jacobians`,
    with unpaired sources, sources and targets without normals, and every flag set."""
    g = np.random.default_rng(1)
    n = 200
    T = IR.exp_se3(g.normal(size=6) * 0.3)[:3].astype(np.float32)
    p = g.uniform(-8, 8, (n, 3)).astype(np.float32)
    m = g.normal(size=(n, 3)).astype(np.float32)
    m[:50] = 0.0
    tn = g.normal(size=(n, 3)).astype(np.float32)
    has = np.ones(n, bool)
    has[40:90] = False
    tn[~has] = 0.0
    nn = g.permutation(n)
    nn[:10] = -1
    for flags in R.flag_matrix():
        Hm, _, M, Mp = IR.information(T, p, m, tn, has, nn, flags, 0.7)
        S, M2, Mp2 = IR.term_sums(T, p, m, tn, has, nn, flags)
        kind = IR.pair_masks(T, p, m, tn, has, nn, flags)
        w = dict(zip(("po2pl", "pl2pl", "po2po"), IR.weights(M, Mp, flags, 0.7)))
        H2, S2 = np.zeros((6, 6)), {k: np.zeros((6, 6)) for k in w}
        for i in np.nonzero(kind)[0]:
            for term, J in IR.jacobians(T, p[i], m[i], tn[nn[i]], kind[i], flags):
                H2 += w[term] * J.T @ J
                S2[term] += J.T @ J
        assert (M, Mp) == (M2, Mp2) == (int((kind == 1).sum()), int((kind == 2).sum()))
        assert np.allclose(Hm, H2, rtol=1e-12, atol=1e-12 * np.abs(H2).max()), R.flag_name(flags)
        for k in w:
            assert np.allclose(S[k], S2[k], rtol=1e-12, atol=1e-9), (R.flag_name(flags), k)


def _nearest_is_fma(h, a, b, c):
    from fractions import Fraction
    exact = Fraction(a) * Fraction(b) + Fraction(c)
    err = abs(Fraction(h) - exact)
    return all(err <= abs(Fraction(float(x)) - exact) for x in (np.nextafter(h, np.inf), np.nextafter(h, -np.inf)))


def test_kernel_order_evaluator():
    """kernel_order: h = fma(w_pp, S3, fma(w_nn, S2, w_pl S1)), each fma rounded once to the nearest float64, with the
    weights of the finalize (lam rounded to fp32 first, 2 lam / M, 2 / M, 2 / (3 M')); a term the flags leave out or
    whose count is 0 weighs 0; the scaled operator multiplies by 1 / f once per translation index."""
    g = np.random.default_rng(5)
    S = {k: np.zeros((6, 6)) for k in ("po2pl", "pl2pl", "po2po")}
    for k in S:
        X = g.integers(-40, 40, (6, 6)).astype(np.float64)
        S[k] = X + X.T
    every = R.LOSS_PO2PO | R.LOSS_PO2PL | R.LOSS_PL2PL
    M, Mp, lam = 37, 11, 0.3
    H, H32 = IR.kernel_order(S, M, Mp, every, lam)
    w_pl, w_nn, w_pp = 2.0 * float(np.float32(lam)) / M, 2.0 / M, 2.0 / (3.0 * Mp)
    assert IR.weights(M, Mp, every, lam) == (w_pl, w_nn, w_pp)
    fused = 0
    for i in range(6):
        for j in range(6):
            inner = IR._fma(w_nn, S["pl2pl"][i, j], w_pl * S["po2pl"][i, j])
            assert _nearest_is_fma(inner, w_nn, S["pl2pl"][i, j], w_pl * S["po2pl"][i, j])
            assert _nearest_is_fma(H[i, j], w_pp, S["po2po"][i, j], inner)
            fused += H[i, j] != (w_pl * S["po2pl"][i, j] + w_nn * S["pl2pl"][i, j]) + w_pp * S["po2po"][i, j]
    assert fused > 0, "no entry where the contraction changes the result: the evaluator is not tested"
    assert np.array_equal(H32, H.astype(np.float32)) and np.array_equal(H, H.T)
    assert IR.weights(M, Mp, R.LOSS_PO2PL, lam) == (w_pl, 0.0, 0.0)
    assert IR.weights(0, Mp, every, lam) == (0.0, 0.0, w_pp) and IR.weights(M, 0, every, lam) == (w_pl, w_nn, 0.0)
    only_pl, _ = IR.kernel_order(S, M, Mp, R.LOSS_PO2PL, lam)
    assert np.array_equal(only_pl, w_pl * S["po2pl"])
    for f in (0.25, 4.0, 0.3):
        Hs, _ = IR.kernel_order(S, M, Mp, every, lam, factor=f)
        inv = 1.0 / float(np.float32(f))
        D = np.array([inv] * 3 + [1.0] * 3)
        want = H.copy()
        for i in range(6):
            for j in range(6):
                want[i, j] = want[i, j] * D[min(i, j)] * D[max(i, j)] if min(i, j) < 3 else want[i, j]
        assert np.array_equal(Hs, want), f
        if f != 0.3:                                        # powers of two: D H D exactly
            assert np.array_equal(Hs, D[:, None] * H * D[None, :])


EXACT_DESIGNS = ("tie", "triple", "zeros", "near", "mixed")


@pytest.mark.parametrize("name", EXACT_DESIGNS)
def test_exact_designs(name):
    """Every source and every target owns its pixel; every Jacobian entry and every sum the kernels form in fp32 is an
    integer below 2^24 (so the fp32 sums are exact: the float64 sums equal their fp32 rounding); the spectrum is the
    intended one."""
    d = IR.exact_design(name)
    h, w, hf, vf = IR.DESIGN_GRID
    for pts in (d.p, d.tgt_p):
        pr = PR.project(pts.T, h, w, hf, vf)
        assert (pr["pixel"] >= 0).all() and len(np.unique(pr["pixel"])) == len(pts)
    assert np.array_equal(d.p, np.round(d.p)) and np.array_equal(d.tgt_p, np.round(d.tgt_p))
    assert np.array_equal(d.tgt_p.astype(np.float64), d.p.astype(np.float64) @ d.T[:, :3].T.astype(np.float64) + d.T[:, 3])
    for flags in (R.flag_matrix() if name == "mixed" else [d.flags]):
        kind = IR.pair_masks(d.T, d.p, d.m, d.tgt_n, d.tgt_has, np.arange(len(d.p)), flags)
        bound = np.zeros((6, 6))
        for J in IR.term_jacobians(d.T, d.p, d.m, d.tgt_n, kind, flags).values():
            assert np.array_equal(J, np.round(J))
            bound += np.einsum("nka,nkb->ab", np.abs(J), np.abs(J))
        assert bound.max() < 2 ** 24
        S, M, Mp = IR.design_sums(d, flags)
        for v in S.values():
            assert np.array_equal(v, v.astype(np.float32).astype(np.float64))
    S, M, Mp = IR.design_sums(d)
    H, H32 = IR.kernel_order(S, M, Mp, d.flags, d.lam)
    ev = np.linalg.eigvalsh(H)
    off = H - np.diag(np.diag(H))
    if name == "tie":
        b, a = H[0, 0], H[2, 2]
        assert not off.any() and H[1, 1] == b and a < b < np.diag(H)[3:].min()
    elif name == "triple":
        assert not off.any() and len(set(np.diag(H)[:3])) == 1 and len(set(np.diag(H)[3:])) == 1 and H[0, 0] < H[3, 3]
    elif name == "zeros":
        assert not H[:3].any() and not H[:, :3].any() and not off.any() and np.diag(H)[3:].min() > 0
        assert np.array_equal(ev[:3], np.zeros(3))
    elif name == "near":
        assert not H[:3, 3:].any() and H[3, 4] != 0 and S["pl2pl"][3, 3] == S["pl2pl"][4, 4] != S["pl2pl"][5, 5]
    else:
        assert M > 0 and Mp > 0 and all(np.abs(v).max() > 0 for v in S.values()) and np.abs(off).max() > 0


@pytest.mark.parametrize("ratio", (1e-3, 1e-6, 1e-9, 1e-12))
def test_near_tie_design_gaps(ratio):
    """near_tie_lambda gives the near design a pair of rotation eigenvalues whose gap is ratio (within 3x) of the
    largest, and a gap to the rest of the spectrum above 0.1 of it."""
    d = IR.exact_design("near")
    lam = IR.near_tie_lambda(d, ratio)
    S, M, Mp = IR.design_sums(d)
    H, _ = IR.kernel_order(S, M, Mp, d.flags, lam)
    ev = np.linalg.eigvalsh(H)
    gap = ev[5] - ev[4]
    assert ratio / 3 <= gap / ev[5] <= 3 * ratio, (gap / ev[5], ratio)
    assert ev[4] - ev[3] > 0.1 * ev[5]
