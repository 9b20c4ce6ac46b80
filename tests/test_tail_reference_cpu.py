"""The float64 tail reference (tail_reference.py) on the CPU: it is OdometryModel's tail in float64 (forward and
autograd) and torch's Adam; its bounds hold for an fp32 emulation of the kernels' arithmetic on every weight family,
and each arithmetic defect below breaks them on at least one family."""
import numpy as np
import pytest
import torch

import tail_reference as R

ACTS = ("relu", "tanh")


def _cfg(act, single, nout=1000):
    return {"device": "cpu", "activation_fct": act, "use_single_mlp_at_output": single, "resnet_outputs": nout,
            "pre_feature_extraction": False, "layers": [1, 1, 1, 1], "factor_fewer_resnet_channels": 1,
            "use_dropout": False}


def _model(cfg, seed=0):
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(seed)
    return OdometryModel(cfg)


def _base(cfg, seed=0):
    return {k: v.detach().numpy().copy() for k, v in _model(cfg, seed).state_dict().items()}


def _pooled(b, seed=0):
    """Like the trunk's average-pooled relu / tanh features: non-negative, O(1)."""
    return np.random.default_rng(seed).gamma(2.0, 0.5, (b, 512)).astype(np.float32)


def test_quaternion_to_R_is_scipys():
    """_rot_torch (kornia 0.3.0's formula, (x, y, z, w) order) against scipy's Rotation.from_quat, which normalises too."""
    from scipy.spatial.transform import Rotation
    q = np.random.default_rng(8).standard_normal((64, 4)) * np.logspace(-6, 6, 64)[:, None]
    got = R._rot_torch(torch.tensor(q)).numpy().reshape(-1, 3, 3)
    np.testing.assert_allclose(got, Rotation.from_quat(q).as_matrix(), rtol=0, atol=1e-14)
    # below the clamp kornia divides by 1e-12, not by the norm: R = I + 2 [..] (q / 1e-12)^2, not a rotation
    small = np.array([[3e-13, 0.0, 0.0, 4e-13]])
    np.testing.assert_allclose(R._rot_torch(torch.tensor(small)).numpy()[0, [0, 4, 8]],
                               [1.0, 1 - 2 * 0.09, 1 - 2 * 0.09], rtol=1e-12)


def _kornia_T(trans, quat):
    B = quat.shape[0]
    T = torch.zeros((B, 4, 4), dtype=torch.float64)
    T[:, :3, :3] = R._rot_torch(quat).reshape(B, 3, 3)
    T[:, :3, 3] = trans
    T[:, 3, 3] = 1
    return T


@pytest.mark.parametrize("single", [False, True])
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("dropout", [False, True])
def test_float64_tail_is_the_model(act, single, dropout):
    cfg = _cfg(act, single, nout=40)
    m = _model(cfg, 1).double()
    w = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    B = 5
    pooled = _pooled(B, 1)
    keep = np.random.default_rng(2).random((B, 40)) >= 0.2 if dropout else None
    x = m.resnet.fc(torch.tensor(pooled, dtype=torch.float64))
    if dropout:
        x = x * torch.tensor(keep, dtype=torch.float64) * 1.25
    if single:
        y = m.fully_connected_rot_trans(x)
        rot, trans = y[:, :4], y[:, 4:]
    else:
        rot, trans = m.fully_connected_rotation(x), m.fully_connected_translation(x)
    T = _kornia_T(trans, rot / torch.norm(rot))
    G = torch.tensor(np.random.default_rng(3).standard_normal((B, 4, 4)))
    (T * G).sum().backward()
    fw = R.tail_forward(pooled, w, cfg, fc_keep=keep)
    np.testing.assert_allclose(fw["T"], T.detach().numpy(), rtol=0, atol=1e-13)
    g = G[:, :3, :].reshape(B, 12).numpy()
    grads = R.tail_backward(fw, g, np.zeros_like(g))
    params = dict(m.named_parameters())
    for name in R.grad_names(cfg):
        want = params[name].grad.numpy()
        np.testing.assert_allclose(grads[name][0], want, rtol=1e-10, atol=1e-12 * np.abs(want).max(), err_msg=name)


def test_float64_adam_is_torch():
    rng = np.random.default_rng(4)
    n = 37
    p0 = rng.standard_normal(n).astype(np.float32)
    lr, b1, b2, eps = (float(np.float32(a)) for a in (1e-3, 0.9, 0.999, 1e-8))
    p = torch.tensor(p0, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([p], lr=lr, betas=(b1, b2), eps=eps)
    pc, m, v = p0.astype(np.float64), np.zeros(n), np.zeros(n)
    for t in range(1, 5):
        g = rng.standard_normal(n).astype(np.float32)
        p.grad = torch.tensor(g, dtype=torch.float64)
        opt.step()
        (pc, m, v), _ = R.adam_step(pc, g, m, v, t, lr, b1, b2, eps)
        st = opt.state[p]
        np.testing.assert_allclose(pc, p.detach().numpy(), rtol=1e-14, atol=0)
        np.testing.assert_allclose(m, st["exp_avg"].numpy(), rtol=1e-14, atol=0)
        np.testing.assert_allclose(v, st["exp_avg_sq"].numpy(), rtol=1e-14, atol=0)
        with torch.no_grad():                              # the fp32 state the kernel keeps, on both sides
            for a in (p, st["exp_avg"], st["exp_avg_sq"]):
                a.copy_(a.float().double())
        pc, m, v = (a.astype(np.float32).astype(np.float64) for a in (pc, m, v))


# ------------------------------------------------------------------------------------------ bounds vs fp32 emulation
def _case(family, act, single, B, nout=1000, norm="block", keep=False, seed=0):
    cfg = _cfg(act, single, nout)
    pooled = _pooled(B, seed)
    w = R.family_weights(family, _base(cfg, seed), cfg, pooled, seed)
    fc_keep = np.random.default_rng(seed + 7).random((B, nout)) >= 0.2 if keep else None
    fw = R.tail_forward(pooled, w, cfg, norm=norm, fc_keep=fc_keep)
    return cfg, pooled, w, fc_keep, fw


def _worst(got, ref, bound, skip=None):
    got, ref, bound = (np.asarray(a, np.float64) for a in (got, ref, bound))
    if skip is not None:
        got, ref, bound = got[~skip], ref[~skip], bound[~skip]
    assert np.all(np.isfinite(got[np.isfinite(ref)])), "NaN / Inf where the reference is finite"
    err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.nanmax(r)) if r.size else 0.0


def _identity_g(T):
    B = T.shape[0]
    g32 = np.zeros((B, 12), np.float32)
    e = (T.reshape(B, 16)[-1, :12] - np.eye(4, dtype=np.float32).reshape(16)[:12]).astype(np.float32)
    g32[-1] = (np.float32(0.125) * e * np.float32(1.0 / B)).astype(np.float32)
    return g32


def _ratios(family, act, single, B, nout=1000, norm="block", keep=False, mutant=None, valid=None, grad="identity"):
    """Worst |emulation - reference| / bound per tensor.  grad: dL/dT of the identity fit (row B-1 only), or a given
    one on every (valid) row, as the ICP objective has."""
    cfg, pooled, w, fc_keep, fw = _case(family, act, single, B, nout, norm, keep)
    assert not R.uninformative(fw).any(), "a row's bound is as large as its quaternion"
    em = R.tail_forward_fp32(pooled, w, cfg, norm, fc_keep=fc_keep, mutant=mutant)
    skip = np.broadcast_to(R.near_clamp(fw)[:, None, None], fw["T"].shape)
    out = {"T": _worst(em["T"], fw["T"], fw["eT"], skip)}
    if R.near_clamp(fw).any():
        return out
    if grad == "identity":
        g32 = _identity_g(em["T"])
        g, eg = R.dT_identity(em["T"])
    else:
        mask = np.ones(B) if valid is None else (np.asarray(valid) != 0)
        g32 = (np.random.default_rng(5).standard_normal((B, 12)) * mask[:, None] / B).astype(np.float32)
        g, eg = g32.astype(np.float64), np.zeros((B, 12))
    ref = R.tail_backward(fw, g, eg, valid)
    got = R.tail_backward_fp32(em, g32, valid, mutant=mutant)
    for name, (v, e) in ref.items():
        out[name] = _worst(got[name], v, e)
    return out


# two heads only: on the single MLP the bounds are as large as the quaternion (tail_reference.uninformative)
CASES = [("init", "relu", False, 5), ("init", "tanh", False, 9), ("near_identity", "tanh", False, 4),
         ("near_identity", "relu", True, 3), ("saturating", "tanh", False, 5), ("zero_rows", "relu", False, 5),
         ("dominance", "relu", False, 5), ("dominance", "tanh", False, 3), ("clamp", "relu", False, 5)]


@pytest.mark.parametrize("family,act,single,B", CASES)
def test_fp32_emulation_is_inside_the_bounds(family, act, single, B):
    worst = _ratios(family, act, single, B)
    print(f"\n[{family} {act} single={single} B={B}] worst ratio {max(worst.values()):.3f}")
    assert max(worst.values()) <= 1.0, worst


def test_fp32_emulation_is_inside_the_bounds_on_other_paths():
    for kw in (dict(nout=1002), dict(nout=3), dict(keep=True), dict(norm="row", valid=[1, 0, 1, 1], grad="random"),
               dict(grad="random"), dict(family="clamp", grad="random", B=7), dict(family="zero_rows", grad="random")):
        kw = {"family": "init", "B": 4, **kw}
        worst = _ratios(act="relu", single=False, **kw)
        assert max(worst.values()) <= 1.0, (kw, worst)


MUTANTS = [
    ("row_norm_for_block", dict(family="clamp", act="relu", single=False, B=5)),
    ("row_norm_for_block", dict(family="clamp", act="relu", single=False, B=5, norm="row", grad="random")),
    ("drop_gn", dict(family="clamp", act="relu", single=False, B=5, grad="random")),
    ("skip_group_row", dict(family="init", act="tanh", single=False, B=5)),
    ("skip_dx_row", dict(family="init", act="tanh", single=False, B=5, grad="random")),
    ("db_first4", dict(family="near_identity", act="tanh", single=False, B=9)),
    ("hidden_ldx_100", dict(family="init", act="relu", single=False, B=3)),
    ("relu_prime_0", dict(family="zero_rows", act="relu", single=False, B=5)),
]


@pytest.mark.parametrize("mutant,case", MUTANTS, ids=[f"{m}-{i}" for i, (m, _) in enumerate(MUTANTS)])
def test_each_tail_mutant_breaks_a_bound(mutant, case):
    try:
        worst = _ratios(mutant=mutant, **case)
    except AssertionError:                                 # NaN / Inf where the reference is finite
        return
    assert max(worst.values()) > 1.0, f"{mutant} stays inside every bound: {worst}"


ADAM_T = [1, 2, 10, 10 ** 4 + 1, 2 ** 24, 2 ** 24 + 1, 2 ** 24 + 2, 2 ** 31 + 6]


def _adam_inputs(n=4099, seed=6):
    rng = np.random.default_rng(seed)
    p = rng.standard_normal(n).astype(np.float32)
    g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 1, n)).astype(np.float32)
    m = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    v = (rng.random(n) * 1e-6).astype(np.float32)
    g[:8], v[:8] = 0, 0                                    # v = 0 with g = 0
    v[8:16] = 1e-30                                        # tiny v
    m[16:32] = -np.sign(g[16:32]) * np.abs(g[16:32]) * 9   # m of the opposite sign: m' cancels
    return p, g, m, v


@pytest.mark.parametrize("t", ADAM_T)
def test_adam_emulation_is_inside_the_bounds(t):
    p, g, m, v = _adam_inputs()
    hp = (1e-3, 0.9, 0.999, 1e-8)
    ref, err = R.adam_step(p, g, m, v, t, *hp)
    got = R.adam_step_fp32(p, g, m, v, t, *hp)
    for a, r, e in zip(got, ref, err):
        assert _worst(a, r, e) <= 1.0


@pytest.mark.parametrize("mutant", ["adam_t_minus_1", "adam_skip_tail"])
def test_each_adam_mutant_breaks_a_bound(mutant):
    p, g, m, v = _adam_inputs()
    hp = (1e-3, 0.9, 0.999, 1e-8)
    ref, err = R.adam_step(p, g, m, v, 3, *hp)
    got = R.adam_step_fp32(p, g, m, v, 3, *hp, mutant=mutant)
    assert max(_worst(a, r, e) for a, r, e in zip(got, ref, err)) > 1.0
