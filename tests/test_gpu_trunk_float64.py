"""-m gpu: the encoder trunk end to end -- delora_trunk_forward and the four delora_trunk_backward calls -- against the
float64 restatement of ResNetModified in trunk_reference.py.

Exact tier (relu): integer designs (trunk_reference.exact_design) in which every value the trunk stores is a small
integer and every fp32 sum is an exact integer, so every fp32 / bf16 result is the true one whatever the summation order.
With saving = 0 and 1, x1 .. x4 equal the reference bit for bit over the interior (zero halo rows, circular halo
columns), `pooled` is the fp32 rounding of the exact mean, and after the four backward calls every conv_dw[c] equals
float64 autograd bit for bit.  The matrix covers block counts 1 .. 64 per stage, H = 1 (stage 3's strided data gradient
with an empty odd row phase), W = 3 and 4 (stage widths of 1: a column's circular halo is itself), W = 259 (stage widths
65, 33, 17, 9), both stem routes and both data-gradient routes of the strided blocks.  Alongside: the weight and
activation buffers are exactly the queried sizes, with guard bytes behind each that no call touches; conv_dw is
NaN-filled before the backward and fully written; a second forward on the same workspace and a second backward give
the same bits.

Gaussian tier (relu and tanh; filters of OdometryModel, images N(0, 25)): per stage, teacher-forced from the kernel's own
x_{s-1}, against the reference with its bf16 rounding hooks; the weight gradients against float64 autograd through that
emulation with the backward's bf16 data-gradient stores.  Metric: every checked tensor is sliced along each of its axes
(pair, channel, row, column; output and input channel for dW) and the largest ||got - ref|| / ||ref|| over all slices
must stay below TAU[(kind, act)].  A defect confined to one column, row, channel or pair is an O(1) error in its slice.
A slice far smaller than its siblings is measured against
a quarter of the RMS slice norm (trunk_reference.slice_errors), so that a relu channel alive on a few pixels does not
turn one rounding flip into an O(1) error.  Measured on an H100 80GB HBM3 (700 W power limit) over the 18 cases, worst
slice: x relu 6.4e-3, tanh 1.1e-2; pooled relu 5.9e-3, tanh 1.4e-2; dW relu 1.4e-1, tanh 8.5e-2.  The dW slices are
the loosest: with relu, an element of a sparse output-channel gradient whose act' flips between 0 and 1 (an activation
within a rounding of zero) changes that slice by the element's whole share.  TAU leaves a margin of 2.1 .. 2.4x.

Dropout (the training step's input and stage-3 dropouts through delora_trunk_forward_dropout / _backward_dropout, at a
counter whose step and seed both have a nonzero high word; the reference with the numpy generator's masks): the exact
tier at saving 1 on designs with images in 16 x [-2, 2], so that 1.25 x and 1.25 x3 are integers (x3 is compared
before the dropout, as stage_out gives it), on both stem routes (the channel-padded conversion of an odd W, the
16-channel one of an even W) times both data-gradient routes of layer4's first block (phase at W = 23 and 180, the
zero-upsample fallback at 259, 720 and 4), each of which applies the gradient mask of x3 in its own branch; and the
Gaussian tier at the same TAU on {2,2,2,2} and {1,3,1,2} x 5x23, 16x180, 64x720, 16x259.  Measured on an H100 80GB
HBM3 (700 W power limit) over the 16 dropout cases, worst slice: x relu 7.0e-3, tanh 1.1e-2; pooled relu 7.0e-3, tanh
1.9e-2; dW relu 2.3e-1 (1x3x1x2 16x180, a relu' flip as above), tanh 1.1e-1: margins of 1.3 .. 2.4x under the same TAU.

The odometry ABI on the plans {3,4,6,3} and {1,3,1,2}, at an even and an odd W: delora_odometry_pairs' pooled equals
delora_trunk_forward's bit for bit, and one relu training step stays within odometry_harness's TAIL_TOL / TRUNK_TOL of
the Python step (measured on the H100: the trunk gradients bit-identical, the tail within 6.1e-7).  With tanh the
{3,4,6,3} step measured a trunk spread of 1.1e-2 (16 x 180) and 1.3e-2 (16 x 259), above TRUNK_TOL: its sixteen blocks
carry the tail's last-bit differences in d(pooled) through twice as many tanh' roundings as {2,2,2,2}, whose worst
was 6.0e-3.
"""
import ctypes
import zlib

import pytest
import torch

import odometry_harness as H
import trunk_reference as R
from helpers import check_exact, interior

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD = 1 << 16           # guard bytes behind the weight section and the activation workspace
GUARD_BYTE = 0xA5

TAU = {("x", "relu"): 1.5e-2, ("x", "tanh"): 2.5e-2,
       ("pooled", "relu"): 1.5e-2, ("pooled", "tanh"): 3e-2,
       ("dw", "relu"): 3e-1, ("dw", "tanh"): 2e-1}

EXACT_PLANS = [
    ((1, 1, 1, 1), [(1, 3), (1, 4), (2, 7), (3, 8), (5, 23), (16, 259)]),
    ((2, 2, 2, 2), [(1, 3), (5, 23), (16, 180), (64, 720)]),
    ((1, 3, 1, 2), [(3, 8), (16, 259)]),
    ((3, 4, 6, 3), [(5, 23), (16, 180)]),
    ((64, 1, 1, 1), [(2, 7)]),
    ((1, 1, 1, 64), [(1, 4)]),
]
# The dropout cases: every stem route (W odd: channel-padded, W even: 16-channel) with every data-gradient route of
# layer4's first block (phase when the stage-3 width is even: W = 23, 180; fallback: W = 259, 720, 4).
DROPOUT_CTR = (2 ** 32 + 7, 2 ** 40 + 0x5EED)          # (step, seed): both with a nonzero high word
DROPOUT_PLANS = [
    ((1, 1, 1, 1), [(5, 23), (16, 259), (16, 180), (16, 720), (1, 4)]),
    ((2, 2, 2, 2), [(5, 23), (16, 259), (16, 180), (64, 720)]),
    ((1, 1, 1, 64), [(5, 23), (1, 4)]),
]
EXACT_CASES = [(layers, h, w, b, None) for layers, sizes in EXACT_PLANS for h, w in sizes for b in (1, 3)] + \
    [(layers, h, w, b, DROPOUT_CTR) for layers, sizes in DROPOUT_PLANS for h, w in sizes for b in (1, 3)]
GAUSS_CASES = [(layers, h, w, act, None) for layers in ((1, 1, 1, 1), (2, 2, 2, 2), (1, 3, 1, 2))
               for h, w in ((5, 23), (16, 180), (64, 720)) for act in ("relu", "tanh")] + \
    [(layers, h, w, act, DROPOUT_CTR) for layers in ((2, 2, 2, 2), (1, 3, 1, 2))
     for h, w in ((5, 23), (16, 180), (64, 720), (16, 259)) for act in ("relu", "tanh")]


def _lib():
    from delora_b200 import _lib as L
    return L


def _id(layers):
    return "x".join(map(str, layers))


def case_id(layers, h, w, last, counter):
    return f"{_id(layers)}-{h}x{w}-{last}" + ("" if counter is None else "-dropout")


def counter_tensor(counter):
    """(step, seed) -> the device int64[3] counter of the _dropout entry points: [0] the step, [2] the seed."""
    step, seed = counter
    return torch.tensor([(v + 2 ** 63) % 2 ** 64 - 2 ** 63 for v in (step, 0, seed)], dtype=torch.int64, device=DEV)


class TrunkRun:
    """The delora_trunk_* entry points on one plan and batch, with guarded buffers of exactly the queried sizes."""

    def __init__(self, layers, b, h, w, act, filters):
        from delora_b200 import ops
        self.L, self.ops = _lib().lib(), ops
        self.layers, self.b, self.h, self.w = layers, b, h, w
        self.act = ops.ACT_RELU if act == "relu" else ops.ACT_TANH
        self.lay = (ctypes.c_int * 4)(*layers)
        self.n_conv = len(R.plan(layers)[1])
        self.nw = int(self.L.delora_trunk_weight_bytes(self.lay, w))
        assert self.nw > 0
        self.weights = torch.full((self.nw + GUARD,), GUARD_BYTE, dtype=torch.uint8, device=DEV)
        self.filters = [f.float().contiguous() for f in filters]
        ptrs = (ctypes.c_void_p * self.n_conv)(*[ops._req(f, torch.float32, "filter") for f in self.filters])
        _lib().check(self.L.delora_trunk_prep_weights(self.lay, w, ptrs, self.weights.data_ptr(), ops._stream()),
                     "delora_trunk_prep_weights")
        self.acts = {}

    def _acts(self, saving):
        if saving not in self.acts:
            n = int(self.L.delora_trunk_activation_bytes(self.lay, self.b, self.h, self.w, saving))
            assert n > 0
            buf = torch.zeros((n + GUARD,), dtype=torch.uint8, device=DEV)
            buf[n:] = GUARD_BYTE
            self.acts[saving] = (buf, n)
        return self.acts[saving][0]

    def forward(self, img1, img2, saving, ctr=None):
        """-> ([x1 .. x4] padded NHWC bf16 copies, pooled [B, 512] fp32).  ctr (counter_tensor): the dropout forward."""
        ops = self.ops
        acts = self._acts(saving)
        pooled = torch.full((self.b, 512), float("nan"), dtype=torch.float32, device=DEV)
        so = (ctypes.c_void_p * 4)()
        args = (self.lay, self.b, self.h, self.w, self.act, saving, ops._req(img1, torch.float32, "img1"),
                ops._req(img2, torch.float32, "img2"), self.weights.data_ptr(), acts.data_ptr(), pooled.data_ptr(), so)
        if ctr is None:
            _lib().check(self.L.delora_trunk_forward(*args, ops._stream()), "delora_trunk_forward")
        else:
            _lib().check(self.L.delora_trunk_forward_dropout(*args, ctr.data_ptr(), ops._stream()),
                         "delora_trunk_forward_dropout")
        xs = []
        for s, ((hs, ws), c) in enumerate(zip(R.stage_sizes(self.h, self.w), R.WIDTHS)):
            off = so[s] - acts.data_ptr()
            n = self.b * (hs + 2) * (ws + 2) * c * 2
            assert 0 <= off and off + n <= self.acts[saving][1], f"x{s + 1} outside the workspace"
            xs.append(acts[off:off + n].view(torch.bfloat16).view(self.b, hs + 2, ws + 2, c).clone())
        return xs, pooled

    def backward(self, g_pooled, ctr=None):
        """The four stage calls after a saving forward -> every conv_dw[c], each a slice of one NaN-filled buffer.
        ctr: the dropout backward, with the forward's counter."""
        ops = self.ops
        numels = [f.numel() for f in self.filters]
        flat = torch.full((sum(numels),), float("nan"), dtype=torch.float32, device=DEV)
        dws, off = [], 0
        for f, n in zip(self.filters, numels):
            dws.append(flat[off:off + n].view(f.shape))
            off += n
        ptrs = (ctypes.c_void_p * self.n_conv)(*[d.data_ptr() for d in dws])
        g = g_pooled.float().contiguous()
        for stage in (3, 2, 1, 0):
            args = (self.lay, self.b, self.h, self.w, self.act, self.weights.data_ptr(), self._acts(1).data_ptr(),
                    ops._req(g, torch.float32, "g_pooled"), ptrs, stage)
            if ctr is None:
                _lib().check(self.L.delora_trunk_backward(*args, ops._stream()), "delora_trunk_backward")
            else:
                _lib().check(self.L.delora_trunk_backward_dropout(*args, ctr.data_ptr(), ops._stream()),
                             "delora_trunk_backward_dropout")
        bad = ~torch.isfinite(flat)
        assert not bool(bad.any()), f"{int(bad.sum())} conv_dw entries not written"
        return dws

    def check_guards(self, label):
        assert bool((self.weights[self.nw:] == GUARD_BYTE).all()), f"{label}: written past the weight section"
        for saving, (buf, n) in self.acts.items():
            assert bool((buf[n:] == GUARD_BYTE).all()), f"{label}: written past the saving={saving} workspace"


def check_halo(x, label):
    """Zero halo rows; halo columns 0 and w + 1 the circular copies of columns w and 1."""
    hs, ws = x.shape[1] - 2, x.shape[2] - 2
    bits = x.view(torch.int16)
    assert not bool(bits[:, 0].any()) and not bool(bits[:, hs + 1].any()), f"{label}: halo row not zero"
    assert torch.equal(bits[:, 1:hs + 1, 0], bits[:, 1:hs + 1, ws]), f"{label}: halo column 0 differs from column w"
    assert torch.equal(bits[:, 1:hs + 1, ws + 1], bits[:, 1:hs + 1, 1]), f"{label}: halo column w+1 differs from column 1"


def nchw(x):
    return interior(x, x.shape[1] - 2, x.shape[2] - 2)


# ------------------------------------------------------------------------------------------------ exact tier
def _eligible(ci, co, wi, st):
    from delora_b200 import ops
    return ops.conv2d_dgrad_eligible(ci, co, wi, st)


def test_exact_matrix_runs_both_dgrad_routes():
    routes = {r for layers, h, w, _, _ in EXACT_CASES for _, r in R.dgrad_routes(layers, h, w, _eligible)}
    assert routes == {"phase", "fallback"}, routes


def layer4_route(layers, h, w):
    """The data-gradient route of layer4's first block, the block that reads x3d in a dropout step."""
    first4 = sum(layers[:3])
    return dict(R.dgrad_routes(layers, h, w, _eligible))[first4]


def test_dropout_matrix_runs_every_stem_and_layer4_route():
    """The masked input conversion of both stem layouts, and the stage-3 gradient mask after both data-gradient routes
    of layer4's first block (trunk.cu applies it in each route's branch)."""
    combos = {("16-channel" if w % 2 == 0 else "channel-padded", layer4_route(layers, h, w))
              for layers, h, w, _, ctr in EXACT_CASES if ctr is not None}
    print(f"\n[dropout routes] {sorted(combos)}", flush=True)
    assert combos == {(stem, r) for stem in ("16-channel", "channel-padded") for r in ("phase", "fallback")}, combos


@pytest.mark.parametrize("layers,h,w,b,counter", EXACT_CASES, ids=[case_id(*c[:3], f"b{c[3]}", c[4]) for c in EXACT_CASES])
def test_exact_integer_design(layers, h, w, b, counter, cuda_lib):
    """With a counter: saving 1 only (the dropout forward needs it); x3 is stage_out's, before the stage-3 dropout.
    The backward overwrites x3d, so the second backward follows a second forward."""
    label = f"exact {_id(layers)} {h}x{w} B={b}" + ("" if counter is None else f" dropout {counter}")
    d = R.exact_design(layers, b, h, w, device=DEV, counter=counter)
    routes = R.dgrad_routes(layers, h, w, _eligible)
    ctr = None if counter is None else counter_tensor(counter)
    tr = TrunkRun(layers, b, h, w, "relu", d.filters)
    img1, img2 = d.img1.contiguous(), d.img2.contiguous()
    h4, w4 = R.stage_sizes(h, w)[3]
    total = d.x[3].sum(dim=(2, 3))
    assert bool((total.abs() < R.SUM_MAX).all())
    want_pooled = total.float() / torch.tensor(float(h4 * w4), dtype=torch.float32, device=DEV)
    for saving in ((0, 1) if ctr is None else (1,)):
        xs, pooled = tr.forward(img1, img2, saving, ctr)
        for s in range(4):
            check_halo(xs[s], f"{label} saving={saving} x{s + 1}")
            check_exact(nchw(xs[s]), d.x[s], f"{label} saving={saving} x{s + 1}")
        assert torch.equal(pooled, want_pooled), f"{label} saving={saving}: pooled differs from the fp32 exact mean"
        xs2, pooled2 = tr.forward(img1, img2, saving, ctr)
        assert torch.equal(pooled2.view(torch.int32), pooled.view(torch.int32)), f"{label}: second forward differs"
        for a, c in zip(xs, xs2):
            assert torch.equal(a.view(torch.int16), c.view(torch.int16)), f"{label}: second forward differs"
    dws = tr.backward(d.g_pooled, ctr)
    for c, (got, ref) in enumerate(zip(dws, d.dw)):
        check_exact(got.double(), ref, f"{label} conv_dw[{c}]")
    if ctr is not None:
        tr.forward(img1, img2, 1, ctr)
    again = tr.backward(d.g_pooled, ctr)
    for c, (x, y) in enumerate(zip(dws, again)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f"{label}: second backward differs at conv {c}"
    torch.cuda.synchronize()
    tr.check_guards(label)
    fr = d.stats["relu"]
    print(f"\n[{label}] exact: x1..x4, pooled (saving {'0 / 1' if ctr is None else '1'}) and {len(dws)} conv_dw "
          f"bit-identical; {len(d.stats['nonzero_dw'])} nonzero dW; dgrad routes {routes or 'none'}; relu'=1 fraction "
          f"min {min(f for _, f in fr):.3f} max {max(f for _, f in fr):.3f} over {len(fr)} activations", flush=True)


# ------------------------------------------------------------------------------------------------ Gaussian tier
def gaussian_problem(layers, h, w, act, b=2, seed=0):
    cfg = H.config(h, w, act, layers=layers)
    model = H.model(cfg, seed)
    filters = [f.detach().float().contiguous() for f in R.resnet_filters(model.resnet)]
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(repr((layers, h, w, act, seed)).encode()))
    img1 = torch.randn((b, 4, h, w), generator=g, device=DEV) * 5.0
    img2 = torch.randn((b, 4, h, w), generator=g, device=DEV) * 5.0
    g_pooled = torch.randn((b, 512), generator=g, device=DEV)
    return filters, img1, img2, g_pooled


def gaussian_worst(layers, h, w, act, counter=None):
    """-> {kind: (worst slice ratio, where)} of the kernels against the teacher-forced, bf16-faithful reference.
    counter: the dropout entry points (saving 1) against the reference with the numpy generator's masks."""
    filters, img1, img2, g_pooled = gaussian_problem(layers, h, w, act)
    b = img1.shape[0]
    tr = TrunkRun(layers, b, h, w, act, filters)
    ctr = None if counter is None else counter_tensor(counter)
    masks = None if counter is None else R.dropout_masks(counter[1], counter[0], b, h, w, DEV)
    worst = {"x": (0.0, ""), "pooled": (0.0, ""), "dw": (0.0, "")}

    def note(kind, got, ref, axes, where):
        r, at = R.worst_slice(got, ref, axes)
        if r >= worst[kind][0]:
            worst[kind] = (r, f"{where} {at}")
    for saving in ((0, 1) if ctr is None else (1,)):
        xs, pooled = tr.forward(img1, img2, saving, ctr)
        fs = [f.double().requires_grad_(True) for f in filters]
        with torch.backends.cudnn.flags(enabled=False):
            ref = R.trunk(img1, img2, fs, layers, act, hooks=True, saving=bool(saving), bwd_round=True,
                          teacher=[nchw(x) for x in xs[:3]], masks=masks)
            for s in range(4):
                check_halo(xs[s], f"saving={saving} x{s + 1}")
                note("x", nchw(xs[s]), ref["x"][s].detach(), R.X_AXES, f"saving={saving} x{s + 1}")
            note("pooled", pooled, ref["pooled"].detach(), R.POOLED_AXES, f"saving={saving} pooled")
            if saving:
                dws = tr.backward(g_pooled, ctr)
                for c, (got, want) in enumerate(zip(dws, R.weight_grads(ref, fs, g_pooled.double()))):
                    note("dw", got, want, R.DW_AXES, f"conv_dw[{c}]")
    torch.cuda.synchronize()
    tr.check_guards(f"{_id(layers)} {h}x{w} {act}")
    return worst


@pytest.mark.parametrize("layers,h,w,act,counter", GAUSS_CASES, ids=[case_id(*c) for c in GAUSS_CASES])
def test_gaussian_slices(layers, h, w, act, counter, cuda_lib):
    worst = gaussian_worst(layers, h, w, act, counter)
    line = "  ".join(f"{k} {v[0]:.2e} ({v[1]}) / tau {TAU[(k, act)]:.1e}" for k, v in worst.items())
    print(f"\n[gauss {case_id(layers, h, w, act, counter)}] {line}", flush=True)
    for k, (r, at) in worst.items():
        assert r <= TAU[(k, act)], f"{k}: slice {at} off by {r:.3e} of its norm (tau {TAU[(k, act)]:.1e})"


# ------------------------------------------------------------------------------------------------ odometry ABI
ODO_CASES = [(layers, h, w, w_raw) for layers in ((3, 4, 6, 3), (1, 3, 1, 2)) for h, w, w_raw in
             ((16, 180, 1024), (16, 259, 512))]


@pytest.mark.parametrize("layers,h,w,w_raw", ODO_CASES, ids=[f"{_id(c[0])}-{c[1]}x{c[2]}" for c in ODO_CASES])
def test_odometry_pairs_pooled_is_the_trunk_forward(layers, h, w, w_raw, cuda_lib):
    from delora_b200 import ops
    from delora_b200.deploy.capi import InferenceWorkspace
    cfg = H.config(h, w, "relu", layers=layers)
    model = H.model(cfg, 1).eval()
    frames = H.frames(h, w_raw, 4)
    n_stride = max(s.shape[1] for s in frames)
    ws = InferenceWorkspace(H.desc(cfg, n_stride, 2), H.blob(model, cfg))
    pts, counts = H.stack([frames[0], frames[2], frames[1], frames[3]], n_stride)
    _, pooled = ws.pairs(pts, counts)
    ds = cfg["kitti"]
    img, _ = ops.project(pts, counts, h, w, cfg["horizontal_field_of_view"], ds["vertical_field_of_view"])
    with torch.no_grad():
        x4, h4, w4 = model._tensor_core_path().features(img[:2].contiguous(), img[2:].contiguous())[-1]
        want = ops.avgpool(x4, h4, w4)
    torch.cuda.synchronize()
    assert torch.equal(pooled, want), "delora_odometry_pairs' pooled differs from delora_trunk_forward's"


@pytest.mark.parametrize("layers,h,w,w_raw", ODO_CASES, ids=[f"{_id(c[0])}-{c[1]}x{c[2]}" for c in ODO_CASES])
def test_odometry_training_step_on_the_plan(layers, h, w, w_raw, cuda_lib):
    cfg = H.config(h, w, "relu", layers=layers)
    model = H.model(cfg, near_identity=True)
    pairs = H.pairs(h, w_raw, 2)
    n_stride = H.n_stride(pairs)
    pts, counts = H.stack_pairs(pairs, n_stride)
    tr = H.trainer(cfg, n_stride, 2, H.blob(model, cfg))
    _, T, pooled, grads = tr.step(pts, counts)
    py = H.python_step(model, cfg, pts, counts)
    torch.cuda.synchronize()
    assert torch.equal(pooled, py.pooled), "pooled features differ from TensorCoreEncoder.pooled_features"
    assert (T - py.T).abs().max().item() <= 1e-5
    tail, trunk = H.grad_spread(H.grad_dict(grads, cfg), py.grads)
    print(f"\n[train {_id(layers)} {h}x{w}] grads: tail {tail:.2e}, trunk {trunk:.2e}")
    assert tail <= H.TAIL_TOL and trunk <= H.TRUNK_TOL, (tail, trunk)
