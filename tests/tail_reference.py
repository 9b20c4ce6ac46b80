"""Float64 restatement of the odometry tail (resnet.fc, the heads, quaternion -> T, their backward) and of Adam, each
with a per-element bound on the error of an fp32 implementation that follows odometry_tail.cu's arithmetic (test
infrastructure, imported like helpers).

The bounds are a running error analysis, with u = 2^-24 and gamma_d = d u / (1 - d u):
  - a dot product from inputs x^ with error e_x: |z^ - z| <= sum |w| e_x + gamma_d (sum |w x^| + |b|), d the longest
    chain of roundings in the kernel's summation order:
      row_dot4 (odometry_linear_kernel, the heads' last layers in odometry_out_kernel): max(ceil(K / 128) * 4,
        ceil(K / 32)) fmas per lane (float4 or scalar path), 5 butterfly adds, the bias;
      dW / db (odometry_linear_bwd_kernel, odometry_out_bwd_kernel): B fmas / adds in b order;
      dx (odometry_linear_bwd_kernel's tiles): ceil(N / 8) fmas of one warp's chunk, 8 adds of the warp partials;
      the hidden gradient of odometry_out_bwd_kernel: 7 fmas;
      the norm of the [B, 4] block (or of a row): 4B (4) fmas, then sqrtf;
  - relu is 1-Lipschitz and exact; tanhf adds 2 ulp (CUDA's documented bound); tanh' = 1 - y^2 carries
    2 |y| e_y + e_y^2 + 2u, its cancellation near saturation; relu' = [y > 0] is exact unless |z| <= e_z, where the
    bound takes the whole incoming gradient;
  - quaternion -> T (quat_to_T_row) and its backward (quat_to_T_bwd_row): the float64 Jacobian times the incoming
    bounds, plus 32u absolute on R (the per-row renormalisation, its products and sums, on entries <= 2) and
    64u * sum|g_R| / max(|p|, 1e-12) on d(quaternion) (the same, then the division by the row norm and the radial
    projection);
  - Adam: each fp32 operation of odometry_adam_kernel, (float) of the step count, and powf's 4 ulp (CUDA's documented
    bound), amplified by 1 / (1 - beta^t) in the bias corrections.

`tail_forward_fp32` / `tail_backward_fp32` / `adam_step_fp32` are numpy float32 emulations in the kernels' order; their
`mutant` argument injects one arithmetic defect, which test_tail_reference_cpu.py shows each bound to catch.

Weights are state-dict dicts (name -> array).  The tail is fc (512 -> nout), act, the hidden layers (two heads: rot.1
and trans.1 as one [200, nout] layer, the kernel's concatenated order), act, and the last layer as one [7, K_h] matrix
(two heads: block-diagonal, rows 0..3 the quaternion read hid[:, :100], rows 4..6 the translation read hid[:, 100:])."""
import math

import numpy as np
import torch

U = 2.0 ** -24
TANH_ULP = 2
POWF_ULP = 4
ULP_REL = 2 * U                     # one ulp of y is at most 2u |y| (normal range)
TINY = 2.0 ** -149
CLAMP = 1e-12


def gamma(d):
    return d * U / (1 - d * U)


def dot_chain(K):
    """row_dot4's longest rounding chain: lane fmas (float4 or scalar path), 5 butterfly adds, the bias."""
    return max(math.ceil(K / 128) * 4, math.ceil(K / 32)) + 6


# ------------------------------------------------------------------------------------------------- the model's layers
def layers(weights, cfg):
    """-> (fc (W, b), [hidden (W, b)], out (W [7, K_h], b [7]), out_K) in float64; out_K is the K of each last layer."""
    f = {k: np.asarray(v, dtype=np.float64) for k, v in weights.items()}
    fc = (f["resnet.fc.weight"], f["resnet.fc.bias"])
    if cfg["use_single_mlp_at_output"]:
        hid = [(f[f"fully_connected_rot_trans.{i}.weight"], f[f"fully_connected_rot_trans.{i}.bias"]) for i in (1, 3, 5, 7)]
        out = (f["fully_connected_rot_trans.9.weight"], f["fully_connected_rot_trans.9.bias"])
        return fc, hid, out, out[0].shape[1]
    r1, t1 = f["fully_connected_rotation.1.weight"], f["fully_connected_translation.1.weight"]
    hid = [(np.concatenate([r1, t1]), np.concatenate([f["fully_connected_rotation.1.bias"],
                                                      f["fully_connected_translation.1.bias"]]))]
    k = r1.shape[0]
    w = np.zeros((7, 2 * k))
    w[:4, :k] = f["fully_connected_rotation.3.weight"]
    w[4:, k:] = f["fully_connected_translation.3.weight"]
    b = np.concatenate([f["fully_connected_rotation.3.bias"], f["fully_connected_translation.3.bias"]])
    return fc, hid, (w, b), k


def grad_names(cfg):
    """State-dict names of the tail's parameters."""
    if cfg["use_single_mlp_at_output"]:
        heads = [f"fully_connected_rot_trans.{i}.{p}" for i in (1, 3, 5, 7, 9) for p in ("weight", "bias")]
    else:
        heads = [f"fully_connected_{h}.{i}.{p}" for h in ("rotation", "translation") for i in (1, 3)
                 for p in ("weight", "bias")]
    return ["resnet.fc.weight", "resnet.fc.bias"] + heads


def _dot(W, b, x, ex, d):
    aW = np.abs(W)
    z = x @ W.T + b
    e = ex @ aW.T + gamma(d) * ((np.abs(x) + ex) @ aW.T + np.abs(b))
    return z, e


def _act(z, ez, act):
    if act == "relu":
        y = np.maximum(z, 0.0)
        return y, np.where(z + ez > 0, ez, 0.0)
    y = np.tanh(z)
    lip = 1.0 - np.tanh(np.maximum(np.abs(z) - ez, 0.0)) ** 2
    ey = lip * ez
    return y, ey + TANH_ULP * (ULP_REL * (np.abs(y) + ey) + TINY)


def _relu_ambiguous(z, ez):
    """Where the sign of the fp32 pre-activation is not certain (z = 0 with no error is certain: y = +0, relu' = 0)."""
    return (np.abs(z) <= ez) & ~((z == 0) & (ez == 0))


def _act_bwd(s, es, y, ey, z, ez, act):
    """torch's activation backward from the stored output: tanh' = 1 - y^2, relu' = [y > 0]."""
    if act == "relu":
        amb = _relu_ambiguous(z, ez)
        g = np.where(z > 0, s, 0.0)
        e = np.where(amb, np.abs(s) + es, np.where(z > 0, es, 0.0))
        return g, e
    d = 1.0 - y * y
    g = s * d
    e_d = 2 * np.abs(y) * ey + ey * ey + 2 * U
    e = (np.abs(s) + es) * e_d + np.abs(d) * es
    return g, e + U * (np.abs(g) + e)


# ------------------------------------------------------------------------------------------------ quaternion -> T
def _rot_torch(p):
    """kornia 0.3.0 quaternion_to_rotation_matrix on (x, y, z, w) rows, L2-normalised with eps 1e-12 -> [B, 9]."""
    n = torch.linalg.vector_norm(p, dim=1, keepdim=True).clamp_min(CLAMP)
    x, y, z, w = (p / n).unbind(1)
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = torch.ones_like(x)
    return torch.stack([one - (tyy + tzz), txy - twz, txz + twy, txy + twz, one - (txx + tzz), tyz - twx,
                        txz - twy, tyz + twx, one - (txx + tyy)], 1)


def _rot_jacobian(p):
    """R(p) [B, 9] and dR/dp [B, 9, 4] in float64."""
    pt = torch.tensor(p, dtype=torch.float64, requires_grad=True)
    R = _rot_torch(pt)
    J = np.stack([torch.autograd.grad(R[:, i].sum(), pt, retain_graph=True)[0].numpy() for i in range(9)], 1)
    return R.detach().numpy(), J


def _rot_vjp(p, g9):
    """dp = J^T g [B, 4] and d(dp)/dp [B, 4, 4] in float64."""
    pt = torch.tensor(p, dtype=torch.float64, requires_grad=True)
    R = _rot_torch(pt)
    (dp,) = torch.autograd.grad(R, pt, torch.tensor(g9), create_graph=True)
    H = np.stack([torch.autograd.grad(dp[:, j].sum(), pt, retain_graph=True)[0].numpy() for j in range(4)], 1)
    return dp.detach().numpy(), H


def _norm(q, eq, rows):
    """The norm of the [B, 4] block (rows False, one ordered fma sum) or of each row -> (n [B, 1], e_n [B, 1])."""
    if rows:
        n = np.linalg.norm(q, axis=1, keepdims=True)
        en = np.linalg.norm(eq, axis=1, keepdims=True)
        d = 4
    else:
        n = np.full((q.shape[0], 1), np.linalg.norm(q))
        en = np.full_like(n, np.linalg.norm(eq))
        d = 4 * q.shape[0]
    return n, en + (n + en) * (gamma(d) + 2 * U)


# ------------------------------------------------------------------------------------------------------- forward
def tail_forward(pooled, weights, cfg, norm="block", factor=None, fc_keep=None):
    """pooled [B, 512] (the trunk's fp32 bits) -> dict with T [B, 4, 4] and its bound eT, and what tail_backward needs.
    norm: "block" (the reference's division by the norm of the whole [B, 4] quaternion block) or "row" (the streams
    kinds).  factor [B]: T[:3, 3] *= factor (normalised models).  fc_keep [B, nout] bool: the training step's fc
    dropout, act(keep * 1.25 * (W pooled + b))."""
    act = cfg["activation_fct"]
    (Wf, bf), hid, (Wo, bo), out_k = layers(weights, cfg)
    x = np.asarray(pooled, dtype=np.float64)
    z, ez = _dot(Wf, bf, x, np.zeros_like(x), dot_chain(Wf.shape[1]))
    if fc_keep is not None:
        k = np.asarray(fc_keep, dtype=np.float64) * 1.25
        z, ez = z * k, ez * k + U * np.abs(z * k)
    y, ey = _act(z, ez, act)
    acts = [(x, np.zeros_like(x), None, None), (y, ey, z, ez)]
    for W, b in hid:
        z, ez = _dot(W, b, y, ey, dot_chain(W.shape[1]))
        y, ey = _act(z, ez, act)
        acts.append((y, ey, z, ez))
    raw, eraw = _dot(Wo, bo, y, ey, dot_chain(out_k))
    q, eq = raw[:, :4], eraw[:, :4]
    n, en = _norm(q, eq, norm == "row")
    nlo = n - en
    p = q / n
    ep = (eq * n + np.abs(q) * en) / (n * nlo) + U * (np.abs(p) + eq / nlo)
    R, J = _rot_jacobian(p)
    pn = np.linalg.norm(p, axis=1, keepdims=True)
    epn = np.linalg.norm(ep, axis=1, keepdims=True)
    eR = np.einsum("bij,bj->bi", np.abs(J), ep) + 32 * U + 8 * (epn / np.maximum(pn, CLAMP)) ** 2
    t, et = raw[:, 4:], eraw[:, 4:]
    if factor is not None:
        f = np.asarray(factor, dtype=np.float64)[:, None]
        t, et = t * f, et * np.abs(f) + U * np.abs(t * f)
    B = x.shape[0]
    T = np.zeros((B, 4, 4))
    eT = np.zeros((B, 4, 4))
    T[:, :3, :3] = R.reshape(B, 3, 3)
    eT[:, :3, :3] = eR.reshape(B, 3, 3)
    T[:, :3, 3], eT[:, :3, 3] = t, et
    T[:, 3, 3] = 1.0
    return dict(T=T, eT=eT, cfg=cfg, layers=((Wf, bf), hid, (Wo, bo), out_k), acts=acts, raw=raw, eraw=eraw,
                n=n, en=en, p=p, ep=ep, rows=norm == "row", fc_keep=fc_keep, pn=pn, epn=epn)


def uninformative(fwd):
    """Rows whose quaternion bound is at least half the quaternion's norm: their T bound says nothing.  The worst-case
    propagation |W| e_x ignores the cancellation of random-signed errors, so it grows by about sqrt(K) per layer; the
    single MLP's four hidden layers take it there at torch's initialisation, the two heads' one hidden layer does not."""
    return fwd["epn"][:, 0] >= 0.5 * fwd["pn"][:, 0]


def near_clamp(fwd):
    """Rows whose float64 quaternion norm after the block division lies within its fp32 bound of kornia's 1e-12 clamp:
    the two sides of the clamp are different functions, so these rows have no bound."""
    pn, epn = fwd["pn"][:, 0], fwd["epn"][:, 0] * (1 + 1e-3)
    return (np.abs(pn - CLAMP) <= epn) & ~uninformative(fwd)


# ------------------------------------------------------------------------------------------------- dL/dT sources
def dT_identity(T_gpu):
    """The identity fit's dL/dT: 2 (T - I) / (16 B) on the 3x4 part of row B-1 (T_gpu: the step's own T) -> (g, e_g)."""
    T = np.asarray(T_gpu, dtype=np.float64).reshape(-1, 16)
    B = T.shape[0]
    g = np.zeros((B, 12))
    g[-1] = 2.0 * (T[-1, :12] - np.eye(4).reshape(16)[:12]) / (16.0 * B)
    return g, 3 * U * np.abs(g)


def dT_scaled(grad_T, scale_of, valid=None):
    """dL/dT = grad_T * scale (grad_T [B, 12] or [B, 3, 4] fp32, scale_of the integer 1/scale: B, or n_valid on the
    valid rows with zeros elsewhere) -> (g, e_g): fl(1/n) then one product."""
    g = np.asarray(grad_T, dtype=np.float64).reshape(-1, 12) / float(scale_of)
    if valid is not None:
        g = g * (np.asarray(valid) != 0)[:, None]
    return g, 2 * U * np.abs(g)


# ------------------------------------------------------------------------------------------------------ backward
def tail_backward(fwd, g, eg, valid=None):
    """dL/dT (g [B, 12], the row-major 3x4 part; bound eg) -> {name: (grad, bound)} of every fc / head tensor.  valid
    [B] (the per-row form of the adapting streams): the other rows get d(head outputs) = 0."""
    cfg = fwd["cfg"]
    act = cfg["activation_fct"]
    (Wf, bf), hid, (Wo, bo), out_k = fwd["layers"]
    B = g.shape[0]
    q, eq, n, en, p, ep = fwd["raw"][:, :4], fwd["eraw"][:, :4], fwd["n"], fwd["en"], fwd["p"], fwd["ep"]
    rows = fwd["rows"]
    gR = g[:, [0, 1, 2, 4, 5, 6, 8, 9, 10]]
    egR = eg[:, [0, 1, 2, 4, 5, 6, 8, 9, 10]]
    _, J = _rot_jacobian(p)
    dp, Hs = _rot_vjp(p, gR)
    pn = np.maximum(fwd["pn"], CLAMP)
    edp = (np.einsum("bij,bi->bj", np.abs(J), egR) + np.einsum("bjk,bk->bj", np.abs(Hs), ep)
           + 64 * U * np.abs(gR).sum(1, keepdims=True) / pn)
    # q / n backward: d n = -sum(dp q) / n^2 over the block (or the row)
    nlo = n - en
    prod, eprod = dp * q, edp * (np.abs(q) + eq) + np.abs(dp) * eq
    if rows:
        S, eS, d = prod.sum(1, keepdims=True), eprod.sum(1, keepdims=True), 4
        aS = np.abs(prod).sum(1, keepdims=True)
    else:
        S, eS, d = np.full((B, 1), prod.sum()), np.full((B, 1), eprod.sum()), 4 * B
        aS = np.full((B, 1), np.abs(prod).sum())
    eS = eS + gamma(d) * (aS + eS)
    gn = -S / n ** 2
    egn = eS / nlo ** 2 + np.abs(S) * (1 / nlo ** 2 - 1 / n ** 2) + 3 * U * (np.abs(gn) + eS / nlo ** 2)
    t1 = dp / n
    e1 = edp / nlo + np.abs(dp) * (1 / nlo - 1 / n) + U * (np.abs(dp) + edp) / nlo
    r = gn / n
    er = egn / nlo + np.abs(gn) * (1 / nlo - 1 / n) + U * (np.abs(gn) + egn) / nlo
    t2 = q * r
    e2 = eq * (np.abs(r) + er) + np.abs(q) * er + U * np.abs(t2)
    dq = t1 + t2
    edq = e1 + e2 + U * (np.abs(t1) + np.abs(t2) + e1 + e2)
    dout = np.concatenate([dq, g[:, [3, 7, 11]]], 1)
    edout = np.concatenate([edq, eg[:, [3, 7, 11]]], 1)
    if valid is not None:
        dead = np.asarray(valid) == 0
        dout[dead], edout[dead] = 0.0, 0.0

    grads = {}

    def wgrad(dz, edz, x, ex):
        ax = np.abs(x) + ex
        dW = dz.T @ x
        edW = edz.T @ ax + np.abs(dz).T @ ex + gamma(B) * (np.abs(dz) + edz).T @ ax
        db = dz.sum(0)
        edb = edz.sum(0) + gamma(B) * (np.abs(dz) + edz).sum(0)
        return (dW, edW), (db, edb)

    acts = fwd["acts"]
    y, ey, z, ez = acts[-1]
    gWo, gbo = wgrad(dout, edout, y, ey)
    s = dout @ Wo
    es = edout @ np.abs(Wo) + gamma(7) * (np.abs(dout) + edout) @ np.abs(Wo)
    dz, edz = _act_bwd(s, es, y, ey, z, ez, act)
    lin = []
    for i in range(len(hid) - 1, -1, -1):
        W, _ = hid[i]
        x, ex, zx, ezx = acts[i + 1]
        lin.append(wgrad(dz, edz, x, ex))
        N = W.shape[0]
        s = dz @ W
        es = edz @ np.abs(W) + gamma(math.ceil(N / 8) + 8) * (np.abs(dz) + edz) @ np.abs(W)
        dz, edz = _act_bwd(s, es, x, ex, zx, ezx, act)
        if i == 0 and fwd["fc_keep"] is not None:
            k = np.asarray(fwd["fc_keep"], dtype=np.float64) * 1.25
            dz, edz = dz * k, edz * k + U * np.abs(dz * k)
    lin = lin[::-1]
    gfc = wgrad(dz, edz, acts[0][0], acts[0][1])
    grads["resnet.fc.weight"], grads["resnet.fc.bias"] = gfc
    if cfg["use_single_mlp_at_output"]:
        for (gw, gb), i in zip(lin + [(gWo, gbo)], (1, 3, 5, 7, 9)):
            grads[f"fully_connected_rot_trans.{i}.weight"] = gw
            grads[f"fully_connected_rot_trans.{i}.bias"] = gb
    else:
        (hw, ehw), (hb, ehb) = lin[0]
        k = out_k
        (ow, eow), (ob, eob) = gWo, gbo
        for name, rs, orows, ocols in (("rotation", slice(0, k), slice(0, 4), slice(0, k)),
                                       ("translation", slice(k, 2 * k), slice(4, 7), slice(k, 2 * k))):
            grads[f"fully_connected_{name}.1.weight"] = (hw[rs], ehw[rs])
            grads[f"fully_connected_{name}.1.bias"] = (hb[rs], ehb[rs])
            grads[f"fully_connected_{name}.3.weight"] = (ow[orows, ocols], eow[orows, ocols])
            grads[f"fully_connected_{name}.3.bias"] = (ob[orows], eob[orows])
    return grads


# ---------------------------------------------------------------------------------------------------------- Adam
def adam_step(p, g, m, v, t, lr, beta1, beta2, eps):
    """odometry_adam_kernel's formula (torch's Adam, fused: no weight decay, no amsgrad) at step count t (after the
    increment) in float64 on fp32 inputs and hyperparameters -> ((p', m', v'), (e_p, e_m, e_v))."""
    f = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)
    p, g, m, v = f(p), f(g), f(m), f(v)
    lr, b1, b2, eps = (float(np.float32(a)) for a in (lr, beta1, beta2, eps))
    tf = float(np.float32(t))
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    ss, bc2s = lr / bc1, math.sqrt(bc2)
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    den = np.sqrt(v1) / bc2s + eps
    p1 = p - ss * m1 / den

    def pow_err(b):
        if b == 0.0:
            return 0.0
        bt = b ** t
        return bt * (POWF_ULP * ULP_REL + abs(math.log(b)) * abs(tf - t) * 2) + TINY * POWF_ULP
    e_bc1 = pow_err(b1) + U * bc1
    rho_ss = e_bc1 / (bc1 - e_bc1) + U
    rho_bc2 = (pow_err(b2) + U * bc2) / (2 * bc2 - 2 * (pow_err(b2) + U * bc2)) + U
    em = gamma(2) * (np.abs(b1 * m) + np.abs((1 - b1) * g))
    ev = gamma(3) * (b2 * v + (1 - b2) * g * g)
    rho_v = np.where(v1 > 0, ev / np.where(v1 > 0, v1, 1.0), 0.0)
    sq = np.sqrt(v1) / bc2s
    eden = sq * (rho_v / 2 + rho_v ** 2 + 2 * U + rho_bc2) + U * den
    upd = ss * m1 / den
    eupd = np.abs(upd) * (rho_ss + eden / (den - eden) + 2 * U) * (1 + 4 * U) + abs(ss) * em / (den - eden)
    ep = eupd + U * (np.abs(p1) + eupd)
    return (p1, m1, v1), (ep, em, ev)


# ------------------------------------------------------------------------------------ fp32 emulation of the kernels
F32 = np.float32


def _fma(a, b, c):
    return (a.astype(np.float64) * b + c).astype(F32)


def _row_dot4_fp32(W, x, vec, mutant=None):
    """row_dot4 for every (row of x, row of W): lane partials in the kernel's k order, the xor butterfly -> [B, N]."""
    B, K = x.shape
    N = W.shape[0]
    if vec:
        steps = [[4 * l + 128 * j + c for j in range(math.ceil(K / 128)) for c in range(4)] for l in range(32)]
    else:
        steps = [[l + 32 * j for j in range(math.ceil(K / 32))] for l in range(32)]
    idx = np.array(steps)                                   # [32, L]
    Kp = int(idx.max()) + 1
    Wp = np.zeros((N, Kp), F32)
    Wp[:, :K] = W
    xp = np.zeros((B, Kp), F32)
    xp[:, :K] = x
    acc = np.zeros((B, N, 32), F32)
    for s in range(idx.shape[1]):
        k = idx[:, s]
        acc = _fma(Wp[None, :, k], xp[:, None, k], acc)
    for o in (16, 8, 4, 2, 1):
        acc = (acc + acc[:, :, np.arange(32) ^ o]).astype(F32)
    out = acc[:, :, 0]
    if mutant == "skip_group_row":                          # row 3 of every full four-row group never written
        out = out.copy()
        out[3::4] = 0.0
    return out


def _act_fp32(z, act):
    return np.maximum(z, F32(0)) if act == "relu" else np.tanh(z).astype(F32)


def _act_bwd_fp32(g, y, act, mutant=None):
    if act == "tanh":
        return (g * (F32(1) - y * y)).astype(F32)
    if mutant == "relu_prime_0":
        return np.where(y < 0, F32(0), g).astype(F32)
    return np.where(y <= 0, F32(0), g).astype(F32)


def _quat_to_T_fp32(p, t):
    q = p.astype(F32)
    nrm = np.maximum(np.sqrt((q * q).sum(1, dtype=F32)), F32(CLAMP)).astype(F32)[:, None]
    x, y, z, w = (q / nrm).T
    tx, ty, tz = F32(2) * x, F32(2) * y, F32(2) * z
    twx, twy, twz, txx, txy, txz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = F32(1)
    R = np.stack([one - (tyy + tzz), txy - twz, txz + twy, txy + twz, one - (txx + tzz), tyz - twx,
                  txz - twy, tyz + twx, one - (txx + tyy)], 1).astype(F32)
    B = p.shape[0]
    T = np.zeros((B, 4, 4), F32)
    T[:, :3, :3] = R.reshape(B, 3, 3)
    T[:, :3, 3] = t
    T[:, 3, 3] = 1
    return T


def _quat_to_T_bwd_fp32(p, g12):
    q = p.astype(F32)
    nrm_raw = np.sqrt((q * q).sum(1, dtype=F32)).astype(F32)
    nrm = np.maximum(nrm_raw, F32(CLAMP))[:, None]
    x, y, z, w = (q / nrm).T
    g = g12.astype(F32).T
    g00, g01, g02, g10, g11, g12_, g20, g21, g22 = g[0], g[1], g[2], g[4], g[5], g[6], g[8], g[9], g[10]
    two = F32(2)
    dx = two * (y * (g01 + g10) + z * (g02 + g20) - two * x * (g11 + g22) + w * (g21 - g12_))
    dy = two * (x * (g01 + g10) + z * (g12_ + g21) - two * y * (g00 + g22) + w * (g02 - g20))
    dz = two * (x * (g02 + g20) + y * (g12_ + g21) - two * z * (g00 + g11) + w * (g10 - g01))
    dw = two * (x * (g21 - g12_) + y * (g02 - g20) + z * (g10 - g01))
    d = np.stack([dx, dy, dz, dw], 1).astype(F32)
    o = (d / nrm).astype(F32)
    u = np.stack([x, y, z, w], 1)
    dot = ((d * u).sum(1, dtype=F32) / nrm[:, 0]).astype(F32)[:, None]
    o = np.where((nrm_raw > CLAMP)[:, None], (o - dot * u).astype(F32), o)
    return o


def _sum_fp32(v, axis):
    """An ordered fp32 sum along axis (the kernels' loops)."""
    v = np.moveaxis(np.asarray(v, F32), axis, 0)
    s = np.zeros(v.shape[1:], F32)
    for row in v:
        s = (s + row).astype(F32)
    return s


def _norm_fp32(q, rows):
    if rows:
        ss = np.zeros((q.shape[0],), F32)
        for j in range(4):
            ss = _fma(q[:, j], q[:, j], ss)
        return np.sqrt(ss).astype(F32)[:, None]
    ss = np.zeros((), F32)
    for v in q.reshape(-1):
        ss = _fma(np.asarray(v), np.asarray(v), ss)
    return np.full((q.shape[0], 1), np.sqrt(ss), F32)


def tail_forward_fp32(pooled, weights, cfg, norm="block", factor=None, fc_keep=None, mutant=None):
    """The inference / training forward in fp32, in the kernels' order -> dict with T [B, 4, 4] (and the cache)."""
    act = cfg["activation_fct"]
    w = {k: np.asarray(v, F32) for k, v in weights.items()}
    (Wf, bf), hid, (Wo, bo), out_k = layers(w, cfg)
    Wf, bf, Wo, bo = Wf.astype(F32), bf.astype(F32), Wo.astype(F32), bo.astype(F32)
    hid = [(W.astype(F32), b.astype(F32)) for W, b in hid]
    x = np.asarray(pooled, F32)
    z = (_row_dot4_fp32(Wf, x, True, mutant) + bf).astype(F32)
    if fc_keep is not None:
        z = np.where(fc_keep, (z * F32(1.25)).astype(F32), F32(0))
    ys = [x, _act_fp32(z, act)]
    for W, b in hid:
        ys.append(_act_fp32((_row_dot4_fp32(W, ys[-1], True, mutant) + b).astype(F32), act))
    h = ys[-1]
    if cfg["use_single_mlp_at_output"]:
        raw = (_row_dot4_fp32(Wo, h, True) + bo).astype(F32)
    else:
        raw = np.concatenate([_row_dot4_fp32(Wo[:4, :out_k], h[:, :out_k], True),
                              _row_dot4_fp32(Wo[4:, out_k:], h[:, out_k:], True)], 1)
        raw = (raw + bo).astype(F32)
    rows = norm == "row"
    if mutant == "row_norm_for_block":
        rows = not rows
    nrm = _norm_fp32(raw[:, :4], rows)
    p = (raw[:, :4] / nrm).astype(F32)
    t = raw[:, 4:]
    if factor is not None:
        t = (t * np.asarray(factor, F32)[:, None]).astype(F32)
    return dict(T=_quat_to_T_fp32(p, t), ys=ys, raw=raw, nrm=nrm, rows=rows, weights=(Wf, hid, Wo, out_k),
                cfg=cfg, fc_keep=fc_keep)


def tail_backward_fp32(fw, g12, valid=None, mutant=None):
    """odometry_out_bwd_kernel then odometry_linear_bwd_kernel in fp32 -> {name: grad}; g12 [B, 12] is dL/dT as the
    kernel forms it (already scaled)."""
    cfg, act = fw["cfg"], fw["cfg"]["activation_fct"]
    Wf, hid, Wo, out_k = fw["weights"]
    raw, nrm, ys = fw["raw"], fw["nrm"], fw["ys"]
    B = raw.shape[0]
    g12 = np.asarray(g12, F32)
    live = np.ones(B, bool) if valid is None else np.asarray(valid) != 0
    q = raw[:, :4]
    dp = _quat_to_T_bwd_fp32((q / nrm).astype(F32), g12)
    prod = np.zeros((B,), F32) if fw["rows"] else np.zeros((), F32)
    if fw["rows"]:
        for j in range(4):
            prod = _fma(dp[:, j], q[:, j], prod)
        gn = (-prod / (nrm[:, 0] * nrm[:, 0])).astype(F32)[:, None]
    else:
        for b in range(B):
            for j in range(4):
                prod = _fma(dp[b, j], q[b, j], prod)
        gn = np.full((B, 1), -prod / (nrm[0, 0] * nrm[0, 0]), F32)
    if mutant == "drop_gn":
        gn = np.zeros_like(gn)
    dq = ((dp / nrm).astype(F32) + q * (gn / nrm).astype(F32)).astype(F32)
    d = np.concatenate([dq, g12[:, [3, 7, 11]]], 1).astype(F32)
    d[~live] = 0
    grads = {}
    y = ys[-1]

    def wgrad(dz, x):
        gw = np.zeros((dz.shape[1], x.shape[1]), F32)
        for b in range(B):
            gw = _fma(dz[b][:, None], x[b][None, :], gw)
        cnt = 4 if mutant == "db_first4" else B
        return gw, _sum_fp32(dz[:cnt], 0)

    if cfg["use_single_mlp_at_output"]:
        gWo = wgrad(d, y)
        s = np.zeros((B, y.shape[1]), F32)
        for o in range(7):
            s = _fma(Wo[o][None, :], d[:, o:o + 1], s)
        dz = _act_bwd_fp32(s, y, act, mutant)
    else:
        k = out_k
        if mutant == "hidden_ldx_100":                     # the hidden rows read with stride 100, not 200
            flat = y.reshape(-1)
            yr = flat[np.arange(B)[:, None] * k + np.arange(k)]
            yt = flat[k + np.arange(B)[:, None] * k + np.arange(k)]
        else:
            yr, yt = y[:, :k], y[:, k:]
        gr, gt = wgrad(d[:, :4], yr), wgrad(d[:, 4:], yt)
        gWo = (np.zeros((7, 2 * k), F32), np.concatenate([gr[1], gt[1]]))
        gWo[0][:4, :k], gWo[0][4:, k:] = gr[0], gt[0]
        sr = np.zeros((B, k), F32)
        for o in range(4):
            sr = _fma(Wo[o, :k][None, :], d[:, o:o + 1], sr)
        st = np.zeros((B, k), F32)
        for o in range(3):
            st = _fma(Wo[4 + o, k:][None, :], d[:, 4 + o:5 + o], st)
        dz = np.concatenate([_act_bwd_fp32(sr, yr, act, mutant), _act_bwd_fp32(st, yt, act, mutant)], 1)
    lin = []
    for i in range(len(hid) - 1, -1, -1):
        W, _ = hid[i]
        x = ys[i + 1]
        lin.append(wgrad(dz, x))
        N = W.shape[0]
        chunk = math.ceil(N / 8)
        part = np.zeros((8, B, W.shape[1]), F32)
        for w in range(8):
            for n in range(w * chunk, min(N, w * chunk + chunk)):
                part[w] = _fma(dz[:, n:n + 1], W[n][None, :], part[w])
        s = _sum_fp32(part, 0)
        if mutant == "skip_dx_row":
            s[3::4] = 0
        dz = _act_bwd_fp32(s, x, act, mutant)
        if i == 0 and fw["fc_keep"] is not None:
            dz = np.where(fw["fc_keep"], (dz * F32(1.25)).astype(F32), F32(0))
    lin = lin[::-1]
    grads["resnet.fc.weight"], grads["resnet.fc.bias"] = wgrad(dz, ys[0])
    if cfg["use_single_mlp_at_output"]:
        for (gw, gb), i in zip(lin + [gWo], (1, 3, 5, 7, 9)):
            grads[f"fully_connected_rot_trans.{i}.weight"], grads[f"fully_connected_rot_trans.{i}.bias"] = gw, gb
    else:
        k = out_k
        (hw, hb), (ow, ob) = lin[0], gWo
        for name, rs, orows, ocols in (("rotation", slice(0, k), slice(0, 4), slice(0, k)),
                                       ("translation", slice(k, 2 * k), slice(4, 7), slice(k, 2 * k))):
            grads[f"fully_connected_{name}.1.weight"] = hw[rs]
            grads[f"fully_connected_{name}.1.bias"] = hb[rs]
            grads[f"fully_connected_{name}.3.weight"] = ow[orows, ocols]
            grads[f"fully_connected_{name}.3.bias"] = ob[orows]
    return grads


def adam_step_fp32(p, g, m, v, t, lr, beta1, beta2, eps, mutant=None):
    """odometry_adam_kernel in fp32 (float4 body, then the n & 3 tail) -> (p', m', v')."""
    p, g, m, v = (np.array(a, F32) for a in (p, g, m, v))
    b1, b2, lr, eps = F32(beta1), F32(beta2), F32(lr), F32(eps)
    tt = F32(t - 1 if mutant == "adam_t_minus_1" else t)
    bc1 = F32(1) - F32(np.float64(b1) ** np.float64(tt))
    ss = F32(lr / bc1)
    bc2s = np.sqrt(F32(1) - F32(np.float64(b2) ** np.float64(F32(t))), dtype=F32)
    n = p.size
    stop = n - (n & 3) if mutant == "adam_skip_tail" else n
    sl = slice(0, stop)
    m[sl] = _fma(np.full(stop, b1), m[sl], ((F32(1) - b1) * g[sl]).astype(F32))
    v[sl] = _fma(np.full(stop, b2), v[sl], (((F32(1) - b2) * g[sl]).astype(F32) * g[sl]).astype(F32))
    den = (np.sqrt(v[sl]) / bc2s + eps).astype(F32)
    p[sl] = (p[sl] - ((ss * m[sl]).astype(F32) / den).astype(F32)).astype(F32)
    return p, m, v


# ------------------------------------------------------------------------------------------------ weight families
FAMILIES = ("init", "near_identity", "saturating", "zero_rows", "dominance", "clamp")


def _hidden_names(cfg):
    if cfg["use_single_mlp_at_output"]:
        return [f"fully_connected_rot_trans.{i}" for i in (1, 3, 5, 7)]
    return ["fully_connected_rotation.1", "fully_connected_translation.1"]


def _rot_last(cfg):
    """(name, row slice) of the quaternion rows of the last layer."""
    if cfg["use_single_mlp_at_output"]:
        return "fully_connected_rot_trans.9", slice(0, 4)
    return "fully_connected_rotation.3", slice(0, 4)


def family_weights(name, base, cfg, pooled=None, seed=0):
    """The tail weights of a family (every other tensor of `base` unchanged) -> a new state dict of fp32 arrays.
      init: base itself (torch's initialisation);
      near_identity: last layers x 0.01, the quaternion bias (0, 0, 0, 1), the translation bias 0;
      saturating: fc and hidden weights x 30 (tanh saturates);
      zero_rows: 8 fc rows and 4 rows of each hidden layer zero, bias 0 (pre-activation exactly 0: relu' = 0);
      dominance / clamp: fc unit 0 fitted on `pooled` (float64 least squares) to 1 on row 0 and -1 (relu) / 0 (tanh)
        on the others, fc unit 1 a constant 1 plus a small pooled-dependent part; each hidden layer passes units 0 and
        1 on (rows 0, 1 = e0, e1); the quaternion is d0 h0 + eps d1 h1, so row 0's quaternion dominates the block:
        eps = 1e-3 (dominance) or one that puts the other rows' block-divided norms around kornia's 1e-12 clamp."""
    rng = np.random.default_rng(seed)
    w = {k: np.array(v, dtype=np.float32, copy=True) for k, v in base.items()}
    single = cfg["use_single_mlp_at_output"]
    if name == "init":
        return w
    if name == "near_identity":
        if single:
            w["fully_connected_rot_trans.9.weight"] *= 0.01
            w["fully_connected_rot_trans.9.bias"][:] = [0, 0, 0, 1, 0, 0, 0]
        else:
            for h, b in (("rotation", [0, 0, 0, 1]), ("translation", [0, 0, 0])):
                w[f"fully_connected_{h}.3.weight"] *= 0.01
                w[f"fully_connected_{h}.3.bias"][:] = b
        return w
    if name == "saturating":
        for n in ["resnet.fc"] + _hidden_names(cfg):
            w[f"{n}.weight"] *= 30
        return w
    if name == "zero_rows":
        rows = np.arange(0, w["resnet.fc.weight"].shape[0], 7)[:8]
        w["resnet.fc.weight"][rows] = 0
        w["resnet.fc.bias"][rows] = 0
        for n in _hidden_names(cfg):
            w[f"{n}.weight"][1:5] = 0
            w[f"{n}.bias"][1:5] = 0
        return w
    assert name in ("dominance", "clamp") and pooled is not None
    P = np.asarray(pooled, dtype=np.float64)
    B = P.shape[0]
    relu = cfg["activation_fct"] == "relu"
    c = np.full(B, -1.0 if relu else 0.0)
    c[0] = 1.0
    A = np.concatenate([P, np.ones((B, 1))], 1)
    sol = np.linalg.lstsq(A, c, rcond=None)[0]
    nf = w["resnet.fc.weight"].shape[0]
    w["resnet.fc.weight"][0], w["resnet.fc.bias"][0] = sol[:-1], sol[-1]
    direction = rng.standard_normal(P.shape[1])
    spread = P @ direction
    w["resnet.fc.weight"][1] = 0.3 * direction / max(np.abs(spread - spread.mean()).max(), 1e-30)
    w["resnet.fc.bias"][1] = 1.0 - 0.3 * spread.mean() / max(np.abs(spread - spread.mean()).max(), 1e-30)
    prev = nf
    for n in _hidden_names(cfg):
        W = w[f"{n}.weight"]
        W[0:2] = 0
        W[0, 0] = W[1, 1] = 1
        w[f"{n}.bias"][0:2] = 0
        prev = W.shape[0]
    last, rs = _rot_last(cfg)
    W = w[f"{last}.weight"]
    W[rs] = 0
    d0, d1 = rng.standard_normal(4), rng.standard_normal(4)
    eps = 1e-3
    if name == "clamp":
        # |p_b| = eps |d1| h1_b / |block| on the others: 1e-12 at the geometric middle of the widest gap between their
        # sorted h1, so that rows lie on both sides of the clamp and none on it
        fw = tail_forward(pooled, {**w, f"{last}.weight": _with_cols(W, rs, d0, 0.0 * d1)}, cfg)
        h = fw["acts"][-1][0]
        h1 = np.sort(np.maximum(h[1:, 1] if B > 1 else h[:, 1], 1e-30))
        if h1.size > 1:
            i = int(np.argmax(h1[1:] / h1[:-1]))
            mid = math.sqrt(h1[i] * h1[i + 1])
        else:
            mid = 2.0 * h1[0]                               # one other row: it goes below the clamp
        eps = CLAMP * np.linalg.norm(fw["raw"][:, :4]) / (np.linalg.norm(d1) * mid)
    w[f"{last}.weight"] = _with_cols(W, rs, d0, eps * d1)
    w[f"{last}.bias"][rs] = 0
    return w


def _with_cols(W, rs, d0, d1):
    W = W.copy()
    W[rs, 0] = d0
    W[rs, 1] = d1
    return W
