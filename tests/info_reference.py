"""Float64 reference of the Gauss-Newton information of delora_icp_dense_information (test infrastructure, CPU only).

For one scan pair with fixed correspondences (the exact NN of nn_reference, with the masks of the losses), H is
restated in float64 from explicit Jacobian matrices of the right perturbation T(xi) = T Exp(xi), xi = (rho, phi):
  po2pl   r = n_t^T (s - q)      J = n_t^T [R, -R [p]x]             (1 x 6)
  pl2pl   e = R m - n_t          J = [0, -R [m]x]                   (3 x 6)   squared
          o = 1 - n_t^T R m      J = [0, n_t^T R [m]x]              (1 x 6)   linear
  po2po   d = s - q              J = [R, -R [p]x]                   (3 x 6)
  H = 2 (lambda / M sum_po2pl J^T J + 1 / M sum_pl2pl J^T J + 1 / (3 M') sum_po2po J^T J)
with the losses' means (po2po over the 3 M' coordinates).  `objective` is that loss in float64 at T Exp(xi), for
checking H against finite differences where every residual is zero (there the Hessian is exactly Gauss-Newton).
"""
import numpy as np

import icp_reference as R

INFO_ROW = 80
LOSS_PO2PO, LOSS_PO2PL, LOSS_PL2PL, NORMAL_LINEAR = R.LOSS_PO2PO, R.LOSS_PO2PL, R.LOSS_PL2PL, R.NORMAL_LINEAR


def skew(v):
    x, y, z = v
    return np.array([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]])


def exp_se3(xi):
    """4 x 4 float64 Exp of xi = (rho, phi)."""
    rho, phi = np.asarray(xi[:3], np.float64), np.asarray(xi[3:], np.float64)
    th = np.linalg.norm(phi)
    K = skew(phi)
    if th < 1e-12:
        Rm, V = np.eye(3) + K, np.eye(3) + 0.5 * K
    else:
        Rm = np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K
        V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * K + (th - np.sin(th)) / th ** 3 * K @ K
    out = np.eye(4)
    out[:3, :3], out[:3, 3] = Rm, V @ rho
    return out


def pair_masks(T, p, m, tgt_n, tgt_has, nn, flags):
    """Per source: kind 0 none, 1 (normal, normal), 2 po2po, as the losses keep them (rotated source normal non-zero,
    target has-normal flag; po2po pairs only with LOSS_PO2PO)."""
    _, ns = R.apply_rigid(T, p, m)
    src_has = np.any(ns != 0, axis=1)
    paired = nn >= 0
    t_has = np.zeros(len(p), bool)
    t_has[paired] = tgt_has[nn[paired]]
    kind = np.zeros(len(p), np.int64)
    kind[paired & src_has & t_has] = 1
    if flags & LOSS_PO2PO:
        kind[paired & ~src_has & ~t_has] = 2
    return kind


def jacobians(T, p, m, n_t, kind, flags):
    """Per kept pair: list of (term, J [k, 6] float64), term in {'po2pl', 'pl2pl', 'po2po'}."""
    T = np.asarray(T, np.float32).reshape(3, 4).astype(np.float64)
    Rm = T[:, :3]
    out = []
    p, m, n_t = (np.asarray(a, np.float32).astype(np.float64) for a in (p, m, n_t))
    if kind == 1:
        if flags & LOSS_PO2PL:
            out.append(("po2pl", (n_t @ np.hstack([Rm, -Rm @ skew(p)]))[None, :]))
        if flags & LOSS_PL2PL:
            if flags & NORMAL_LINEAR:
                out.append(("pl2pl", np.hstack([np.zeros(3), n_t @ Rm @ skew(m)])[None, :]))
            else:
                out.append(("pl2pl", np.hstack([np.zeros((3, 3)), -Rm @ skew(m)])))
    elif kind == 2:
        out.append(("po2po", np.hstack([Rm, -Rm @ skew(p)])))
    return out


def information(T, p, m, tgt_n, tgt_has, nn, flags, lam=1.0):
    """-> (H [6, 6] float64, A [6, 6] float64, M, M').  A is the same weighted sum with every |J_i J_j| replaced by
    s_i s_j, s = (1, 1, 1, |p|, |p|, |p|) per Jacobian row: the magnitude the kernels' fp32 rounding is relative to."""
    p = np.asarray(p, np.float32).reshape(-1, 3)
    m = np.asarray(m, np.float32).reshape(-1, 3)
    tgt_n = np.asarray(tgt_n, np.float32).reshape(-1, 3)
    tgt_has = np.asarray(tgt_has, bool).reshape(-1)
    nn = np.asarray(nn, np.int64).reshape(-1)
    kind = pair_masks(T, p, m, tgt_n, tgt_has, nn, flags)
    M, Mp = int((kind == 1).sum()), int((kind == 2).sum())
    w = {"po2pl": 2.0 * float(np.float32(lam)) / M if M else 0.0, "pl2pl": 2.0 / M if M else 0.0,
         "po2po": 2.0 / (3.0 * Mp) if Mp else 0.0}
    H, A = np.zeros((6, 6)), np.zeros((6, 6))
    for i in np.nonzero(kind)[0]:
        sc = np.array([1, 1, 1] + [max(1.0, float(np.linalg.norm(p[i].astype(np.float64))))] * 3)
        for term, J in jacobians(T, p[i], m[i], tgt_n[nn[i]], kind[i], flags):
            H += w[term] * J.T @ J
            A += w[term] * J.shape[0] * np.outer(sc, sc)
    return H, A, M, Mp


def objective(T, xi, p, m, tgt_p, tgt_n, kind, nn, flags, lam=1.0):
    """po2po + lam po2pl + pl2pl in float64 at T Exp(xi) with the correspondences held fixed."""
    T4 = np.eye(4)
    T4[:3, :] = np.asarray(T, np.float64).reshape(3, 4)
    Tx = T4 @ exp_se3(xi)
    Rm, t = Tx[:3, :3], Tx[:3, 3]
    p, m, tgt_p, tgt_n = (np.asarray(a, np.float64) for a in (p, m, tgt_p, tgt_n))
    s = p @ Rm.T + t
    ns = m @ Rm.T
    f = 0.0
    b = kind == 1
    if b.any():
        q, n = tgt_p[nn[b]], tgt_n[nn[b]]
        M = b.sum()
        if flags & LOSS_PO2PL:
            f += lam * np.mean(np.sum((s[b] - q) * n, axis=1) ** 2)
        if flags & LOSS_PL2PL:
            if flags & NORMAL_LINEAR:
                f += np.sum((1.0 - np.sum(ns[b] * n, axis=1)) ** 2) / M
            else:
                f += np.sum((ns[b] - n) ** 2) / M
    c = kind == 2
    if c.any():
        f += np.mean((s[c] - tgt_p[nn[c]]) ** 2)
    return f


def residuals(T, xi, p, m, tgt_p, tgt_n, kind, nn, flags, lam=1.0):
    """The objective's residuals at T Exp(xi), each scaled by the square root of its weight, so that
    objective = sum(residuals ** 2) and its Gauss-Newton Hessian is 2 J^T J of this vector."""
    T4 = np.eye(4)
    T4[:3, :] = np.asarray(T, np.float64).reshape(3, 4)
    Tx = T4 @ exp_se3(xi)
    Rm, t = Tx[:3, :3], Tx[:3, 3]
    p, m, tgt_p, tgt_n = (np.asarray(a, np.float64) for a in (p, m, tgt_p, tgt_n))
    s, ns = p @ Rm.T + t, m @ Rm.T
    out = []
    b, c = kind == 1, kind == 2
    M, Mp = b.sum(), c.sum()
    if M:
        q, n = tgt_p[nn[b]], tgt_n[nn[b]]
        if flags & LOSS_PO2PL:
            out.append(np.sqrt(lam / M) * np.sum((s[b] - q) * n, axis=1))
        if flags & LOSS_PL2PL:
            if flags & NORMAL_LINEAR:
                out.append(np.sqrt(1.0 / M) * (1.0 - np.sum(ns[b] * n, axis=1)))
            else:
                out.append(np.sqrt(1.0 / M) * (ns[b] - n).reshape(-1))
    if Mp:
        out.append(np.sqrt(1.0 / (3 * Mp)) * (s[c] - tgt_p[nn[c]]).reshape(-1))
    return np.concatenate(out) if out else np.zeros(0)


def fd_jacobian(fun, h=1e-6):
    """Central first differences of fun: R^6 -> R^k at 0, as [k, 6]."""
    E = np.eye(6) * h
    return np.stack([(fun(E[i]) - fun(-E[i])) / (2 * h) for i in range(6)], axis=1)


def fd_hessian(fun, h=1e-4):
    """Central second differences of fun: R^6 -> R at 0."""
    H = np.zeros((6, 6))
    E = np.eye(6) * h
    for i in range(6):
        for j in range(i, 6):
            H[i, j] = H[j, i] = (fun(E[i] + E[j]) - fun(E[i] - E[j]) - fun(-E[i] + E[j]) + fun(-E[i] - E[j])) / (4 * h * h)
    return H


def eig_row(H):
    """Eigenvalues ascending and unit eigenvectors (rows) of H with the kernels' sign convention: each eigenvector's
    largest-magnitude component (the first of equals) positive."""
    ev, V = np.linalg.eigh(H)
    V = V.T.copy()
    for k in range(6):
        big = int(np.argmax(np.abs(V[k])))
        if V[k, big] < 0:
            V[k] = -V[k]
    return ev, V
