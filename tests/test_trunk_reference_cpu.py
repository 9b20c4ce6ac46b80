"""-m "not gpu": the float64 trunk reference (trunk_reference.py) itself, without a device.

- With its hooks off it equals the repository's OdometryModel run in float64 (features x1 .. x4 and every trunk weight
  gradient to 1e-12 of each tensor's max-abs), so the GPU tests compare the kernels with ResNetModified's definition.
- Every exact-tier design of test_gpu_trunk_float64.py holds its premises (asserted inside exact_design: integer stores
  within bf16 / fp16, partial sums below 2^24, the average-pool backward giving back k, non-degenerate relu'), and the
  matrix gives every convolution position a nonzero weight gradient somewhere.
- Negative controls: each injected defect changes the exact tier's result, and where it applies to the Gaussian tier it
  moves the slice metric of some checked tensor above 10x that tensor kind's TAU in use there.
"""
import functools

import pytest
import torch

import trunk_reference as R
from test_gpu_trunk_float64 import EXACT_CASES, TAU


def _cfg(h, w, act, layers):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=(-24.5, 2.0), device="cpu")
    cfg.update({"activation_fct": act, "use_single_mlp_at_output": False, "layers": list(layers), "resnet_outputs": 1000,
                "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1, "use_dropout": False})
    return cfg


def _gaussian(layers, h, w, act, b=2, seed=0):
    """OdometryModel (float64, CPU) at a seed, images N(0, 25) and a Gaussian g_pooled."""
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(seed)
    model = OdometryModel(_cfg(h, w, act, layers)).double()
    g = torch.Generator().manual_seed(seed + 1)
    img1 = torch.randn((b, 4, h, w), generator=g, dtype=torch.float64) * 5.0
    img2 = torch.randn((b, 4, h, w), generator=g, dtype=torch.float64) * 5.0
    return model, img1, img2, torch.randn((b, 512), generator=g, dtype=torch.float64)


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("h,w", [(5, 24), (5, 23), (1, 8)])
def test_reference_equals_the_float64_model(h, w, act):
    layers = (1, 3, 1, 2)
    model, img1, img2, gp = _gaussian(layers, h, w, act)
    filters = R.resnet_filters(model.resnet)
    feats = model.forward_features(img1, img2)
    want_dw = torch.autograd.grad((feats[3].mean(dim=(2, 3)) * gp).sum(), filters)
    fs = [f.detach().clone().requires_grad_(True) for f in filters]
    out = R.trunk(img1, img2, fs, layers, act, hooks=False)
    worst = 0.0
    for s in range(4):
        worst = max(worst, _rel(out["x"][s].detach(), feats[s].detach()))
    worst = max(worst, _rel(out["pooled"].detach(), feats[3].mean(dim=(2, 3)).detach()))
    for c, (got, want) in enumerate(zip(R.weight_grads(out, fs, gp), want_dw)):
        assert want.abs().max().item() > 0, f"conv {c}: zero gradient in the model"
        worst = max(worst, _rel(got, want))
    print(f"\n[{h}x{w} {act}] reference vs OdometryModel float64: worst relative {worst:.2e}")
    assert worst <= 1e-12


@functools.lru_cache(maxsize=None)
def _design(layers, b, h, w):
    return R.exact_design(layers, b, h, w)


@pytest.mark.parametrize("layers,h,w,b", EXACT_CASES,
                         ids=[f"{'x'.join(map(str, c[0]))}-{c[1]}x{c[2]}-b{c[3]}" for c in EXACT_CASES])
def test_exact_design_holds_its_premises(layers, h, w, b):
    d = _design(layers, b, h, w)
    fr = d.stats["relu"]
    print(f"\n[{layers} {h}x{w} B={b}] relu'=1 fraction per activation: "
          + " ".join(f"{name} {f:.2f}" for name, f in fr))


def test_exact_matrix_covers_every_convolution_position():
    got = set()
    for layers, h, w, b in EXACT_CASES:
        got |= R.dw_coverage(layers, _design(layers, b, h, w).stats["nonzero_dw"])
    want = {"stem"} | {("first", s, p) for s in range(4) for p in ("c1", "c2")} | \
           {("first", s, "ds") for s in (1, 2, 3)} | {("later", s, p) for s in range(4) for p in ("c1", "c2")}
    assert want <= got, sorted(map(str, want - got))


# ------------------------------------------------------------------------------------------------ negative controls
CONTROL_LAYERS = (2, 2, 2, 2)


def _control_defects():
    blocks, _ = R.plan(CONTROL_LAYERS)
    first2 = next(b for b in blocks if b.stage == 2)
    return [("zero_pad", first2.c1), ("residual_from_input", 1), ("swap_blocks", 0), ("shift_pair", 1),
            ("argmax_last", None)]


def _run(img1, img2, filters, act, g_pooled, defect):
    fs = [f.detach().clone().requires_grad_(True) for f in filters]
    out = R.trunk(img1, img2, fs, CONTROL_LAYERS, act, hooks=True, saving=True, bwd_round=True, defect=defect)
    return [x.detach() for x in out["x"]], out["pooled"].detach(), R.weight_grads(out, fs, g_pooled)


@pytest.mark.parametrize("defect", _control_defects(), ids=lambda d: d[0])
def test_defect_breaks_the_exact_comparison(defect):
    d = _design(CONTROL_LAYERS, 3, 5, 23)
    xs, pooled, dw = _run(d.img1, d.img2, d.filters, "relu", d.g_pooled.double(), defect)
    same = all(torch.equal(a, b) for a, b in zip(xs, d.x)) and torch.equal(pooled, d.pooled) and \
        all(torch.equal(a, b) for a, b in zip(dw, d.dw))
    assert not same, f"{defect[0]}: the exact tier does not see it"


@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("defect", [d for d in _control_defects() if d[0] != "argmax_last"], ids=lambda d: d[0])
def test_defect_exceeds_the_gaussian_thresholds(defect, act):
    """The max-pool's tie rule has no Gaussian counterpart: ties do not occur there."""
    model, img1, img2, gp = _gaussian(CONTROL_LAYERS, 16, 180, act)
    filters = R.resnet_filters(model.resnet)
    clean = _run(img1, img2, filters, act, gp, None)
    bad = _run(img1, img2, filters, act, gp, defect)
    worst = {"x": max(R.worst_slice(a, b, R.X_AXES)[0] for a, b in zip(bad[0], clean[0])),
             "pooled": R.worst_slice(bad[1], clean[1], R.POOLED_AXES)[0],
             "dw": max(R.worst_slice(a, b, R.DW_AXES)[0] for a, b in zip(bad[2], clean[2]))}
    over = max(worst[k] / TAU[(k, act)] for k in worst)
    print(f"\n[{defect[0]} {act}] worst slice / TAU: " + "  ".join(f"{k} {worst[k] / TAU[(k, act)]:.3g}" for k in worst))
    assert over > 10, f"{defect[0]} {act}: at most {over:.3g} x TAU"
