"""-m "not gpu": the float64 trunk reference (trunk_reference.py) itself, without a device.

- With its hooks off it equals the repository's OdometryModel run in float64 (features x1 .. x4 and every trunk weight
  gradient to 1e-12 of each tensor's max-abs), so the GPU tests compare the kernels with ResNetModified's definition;
  with masks, the model whose Dropout and Dropout2d multiply by the same fixed masks times 1.25 (x3 is compared before
  the dropout, the model's x3 after it).
- Every exact-tier design of test_gpu_trunk_float64.py, with and without dropout, holds its premises (asserted inside
  exact_design: integer stores exact in bf16 / fp16, partial sums below 2^24, the average-pool backward giving back k,
  non-degenerate relu'), and the matrix gives every convolution position a nonzero weight gradient somewhere.
- Negative controls: each injected defect changes the exact tier's result, and where it applies to the Gaussian tier it
  moves the slice metric of some checked tensor above 10x that tensor kind's TAU in use there.  The dropout defects
  run on a dropout design and with the same masks; act' taken from x3d only shows with tanh (relu'(x3d) = relu'(x3)
  wherever the mask keeps), so it has no exact-tier control.
"""
import functools

import pytest
import torch

import trunk_reference as R
from test_gpu_trunk_float64 import DROPOUT_CTR, EXACT_CASES, TAU, case_id


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


class _Masked(torch.nn.Module):
    """Dropout / Dropout2d with a fixed keep mask: x * keep * 1.25 (a [B, C] mask broadcast over H x W).  The fc
    output, which dropout_values serves as well, is not the trunk's and passes unchanged."""

    def __init__(self, keep):
        super().__init__()
        self.keep = keep if keep.dim() == 4 else keep[:, :, None, None]

    def forward(self, x):
        return x if x.dim() == 2 else x * self.keep * 1.25


@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("h,w", [(5, 24), (5, 23), (1, 8)])
def test_reference_equals_the_float64_model(h, w, act):
    _equals_the_model(h, w, act, False)


@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("h,w", [(5, 24), (5, 23), (1, 8)])
def test_reference_with_masks_equals_the_masked_float64_model(h, w, act):
    _equals_the_model(h, w, act, True)


def _equals_the_model(h, w, act, dropout):
    layers = (1, 3, 1, 2)
    model, img1, img2, gp = _gaussian(layers, h, w, act)
    masks = R.dropout_masks(DROPOUT_CTR[1], DROPOUT_CTR[0], img1.shape[0], h, w) if dropout else None
    if dropout:
        model.resnet.dropout_values, model.resnet.dropout_channels = _Masked(masks[0]), _Masked(masks[1])
        assert 0 < masks[1].mean().item() < 1
    filters = R.resnet_filters(model.resnet)
    feats = model.forward_features(img1, img2)
    want_dw = torch.autograd.grad((feats[3].mean(dim=(2, 3)) * gp).sum(), filters)
    fs = [f.detach().clone().requires_grad_(True) for f in filters]
    out = R.trunk(img1, img2, fs, layers, act, hooks=False, masks=masks)
    worst = 0.0
    for s in range(4):
        want = feats[s].detach()
        if dropout and s == 2:
            want = want / 1.25                  # the model's x3 is x3d; a dropped channel is 0 in both
            assert torch.equal(want == 0, (out["x"][2].detach() * masks[1][:, :, None, None]) == 0)
            worst = max(worst, _rel(out["x"][2].detach() * masks[1][:, :, None, None], want))
            continue
        worst = max(worst, _rel(out["x"][s].detach(), want))
    worst = max(worst, _rel(out["pooled"].detach(), feats[3].mean(dim=(2, 3)).detach()))
    for c, (got, want) in enumerate(zip(R.weight_grads(out, fs, gp), want_dw)):
        assert want.abs().max().item() > 0, f"conv {c}: zero gradient in the model"
        worst = max(worst, _rel(got, want))
    print(f"\n[{h}x{w} {act} {'dropout' if dropout else 'plain'}] reference vs OdometryModel float64: worst relative "
          f"{worst:.2e}")
    assert worst <= 1e-12


@functools.lru_cache(maxsize=4)
def _design(layers, b, h, w, counter=None):
    return R.exact_design(layers, b, h, w, counter=counter)


_STATS = {}


def _stats(layers, b, h, w, counter=None):
    """A design's stats, kept for every design; the designs themselves only for the last few (their activations
    add up to gigabytes over the matrix)."""
    key = (layers, b, h, w, counter)
    if key not in _STATS:
        _STATS[key] = _design(*key).stats
    return _STATS[key]


@pytest.mark.parametrize("layers,h,w,b,counter", EXACT_CASES, ids=[case_id(*c[:3], f"b{c[3]}", c[4]) for c in EXACT_CASES])
def test_exact_design_holds_its_premises(layers, h, w, b, counter):
    d = _design(layers, b, h, w, counter)
    _STATS.setdefault((layers, b, h, w, counter), d.stats)
    fr = d.stats["relu"]
    if counter is not None:           # the masks drop something and keep something in both tensors
        for m in d.masks:
            assert 0 < m.mean().item() < 1
    print(f"\n[{layers} {h}x{w} B={b}{'' if counter is None else ' dropout'}] relu'=1 fraction per activation: "
          + " ".join(f"{name} {f:.2f}" for name, f in fr))


def test_exact_matrix_covers_every_convolution_position():
    _covers_every_position(False)


def test_dropout_matrix_covers_every_convolution_position():
    _covers_every_position(True)


def _covers_every_position(dropout):
    got = set()
    for layers, h, w, b, counter in EXACT_CASES:
        if (counter is not None) != dropout:
            continue
        got |= R.dw_coverage(layers, _stats(layers, b, h, w, counter)["nonzero_dw"])
    want = {"stem"} | {("first", s, p) for s in range(4) for p in ("c1", "c2")} | \
           {("first", s, "ds") for s in (1, 2, 3)} | {("later", s, p) for s in range(4) for p in ("c1", "c2")}
    assert want <= got, sorted(map(str, want - got))


# ------------------------------------------------------------------------------------------------ negative controls
CONTROL_LAYERS = (2, 2, 2, 2)


def _control_defects():
    blocks, _ = R.plan(CONTROL_LAYERS)
    first2 = next(b for b in blocks if b.stage == 2)
    return [("zero_pad", first2.c1), ("residual_from_input", 1), ("swap_blocks", 0), ("shift_pair", 1),
            ("argmax_last", None), ("drop_grad_unmasked", None), ("drop_stage3_shift", "pair"),
            ("drop_stage3_shift", "channel"), ("drop_input_swap", None), ("drop_act_from_x3d", None)]


def _defect_id(d):
    return d[0] + (f"-{d[1]}" if isinstance(d[1], str) else "")


def _run(img1, img2, filters, act, g_pooled, defect, masks=None):
    fs = [f.detach().clone().requires_grad_(True) for f in filters]
    out = R.trunk(img1, img2, fs, CONTROL_LAYERS, act, hooks=True, saving=True, bwd_round=True, defect=defect,
                  masks=masks)
    return [x.detach() for x in out["x"]], out["pooled"].detach(), R.weight_grads(out, fs, g_pooled)


@pytest.mark.parametrize("defect", [d for d in _control_defects() if d[0] != "drop_act_from_x3d"], ids=_defect_id)
def test_defect_breaks_the_exact_comparison(defect):
    """The dropout defects on the dropout design (an odd W: the channel-padded input conversion)."""
    d = _design(CONTROL_LAYERS, 3, 5, 23, DROPOUT_CTR if defect[0].startswith("drop_") else None)
    xs, pooled, dw = _run(d.img1, d.img2, d.filters, "relu", d.g_pooled.double(), defect, d.masks)
    same = all(torch.equal(a, b) for a, b in zip(xs, d.x)) and torch.equal(pooled, d.pooled) and \
        all(torch.equal(a, b) for a, b in zip(dw, d.dw))
    assert not same, f"{defect[0]}: the exact tier does not see it"


GAUSS_CONTROLS = [(d, act) for d in _control_defects() for act in ("relu", "tanh")
                  if d[0] != "argmax_last" and (d[0] != "drop_act_from_x3d" or act == "tanh")]


@pytest.mark.parametrize("defect,act", GAUSS_CONTROLS, ids=[f"{_defect_id(d)}-{a}" for d, a in GAUSS_CONTROLS])
def test_defect_exceeds_the_gaussian_thresholds(defect, act):
    """The max-pool's tie rule has no Gaussian counterpart: ties do not occur there; relu'(x3d) equals relu'(x3)
    wherever the mask keeps.  The dropout defects run with the masks of the dropout cases."""
    model, img1, img2, gp = _gaussian(CONTROL_LAYERS, 16, 180, act)
    filters = R.resnet_filters(model.resnet)
    masks = R.dropout_masks(DROPOUT_CTR[1], DROPOUT_CTR[0], 2, 16, 180) if defect[0].startswith("drop_") else None
    clean = _run(img1, img2, filters, act, gp, None, masks)
    bad = _run(img1, img2, filters, act, gp, defect, masks)
    worst = {"x": max(R.worst_slice(a, b, R.X_AXES)[0] for a, b in zip(bad[0], clean[0])),
             "pooled": R.worst_slice(bad[1], clean[1], R.POOLED_AXES)[0],
             "dw": max(R.worst_slice(a, b, R.DW_AXES)[0] for a, b in zip(bad[2], clean[2]))}
    over = max(worst[k] / TAU[(k, act)] for k in worst)
    print(f"\n[{defect[0]} {act}] worst slice / TAU: " + "  ".join(f"{k} {worst[k] / TAU[(k, act)]:.3g}" for k in worst))
    assert over > 10, f"{defect[0]} {act}: at most {over:.3g} x TAU"
