"""The encoder trunk of ResNetModified -- stem, max-pool, four stages of BasicBlocks, average pool -- in float64, restated
from its definition (test infrastructure, imported like helpers).  It uses neither the kernels nor TensorCoreEncoder.

Definition (src/models/resnet_modified.py):
- stem: 3x3 convolution 8 -> 64, stride (1, 2), then the activation;
- max-pool: 3x3, stride (1, 2), circular in W, the rows beyond the image excluded;
- BasicBlock: act(conv2(act(conv1(x))) + identity), identity = x or a 1x1 downsample on the first block of a stage that
  is strided or changes the channel count; stage strides H (1, 1, 1, 2), W (1, 2, 2, 2), widths 64, 128, 256, 512;
- every 3x3 convolution pads circularly in W and with zeros in H; relu or tanh; global average pool.
Filters come in state_dict order (`plan`), the order delora_trunk_prep_weights documents.

Dropout (`masks`, a DELORA_TRAIN_DROPOUT training step; the contract of include/delora_b200.h, the Dropout paragraph
of delora_odometry_train_step): every element of cat(image_1, image_2) becomes fp32(x * 1.25f) * keep before the bf16
split; layer4's first block (its conv1, its downsample and their weight gradients) reads x3d = bf16(fp32(x3 * 1.25f))
* keep [pair, channel] while x3 (layer3's output, in "x") stays for act'; the backward takes act'(x3) first, rounds
(bwd_round), then multiplies by keep * 1.25 and rounds again (the dz2 store of layer3's last block).

Rounding hooks (`hooks=True`) round to the type the trunk stores, where it stores it: the filters and the input (bf16;
an even W keeps the rounding residual as a second bf16 term, the 16-channel layout), the stem output (fp16 on the
16-channel route in saving mode with the activation deferred to the pool, bf16 pre-activation on the other route in
saving mode, bf16 after the activation without saving), the pool, t1, the downsample, the block outputs (bf16) and
`pooled` (fp32).  act' is taken from the stored activation, as the kernels' epilogues take it.  `bwd_round` rounds the
backward's data-gradient stores to bf16: the gradient of every pre-activation, of the pool output, and the
downsample's data gradient.  With the hooks off everything is float64.

The max-pool's argmax is the FIRST strict maximum in row-major window order (the kernels' and torch's rule); ties are
common on integer inputs, so the rule is stated here, not inherited.  `teacher` runs stage s >= 1 from a given
x_{s-1} (its value; the gradient still flows into the emulated x_{s-1}).
"""
import collections

import torch
import torch.nn.functional as F

WIDTHS = (64, 128, 256, 512)
STRIDES = ((1, 1), (1, 2), (1, 2), (2, 2))

Block = collections.namedtuple("Block", "stage index cin cout stride c1 c2 ds")
DEFECTS = ("zero_pad", "residual_from_input", "swap_blocks", "shift_pair", "argmax_last", "drop_grad_unmasked",
           "drop_stage3_shift", "drop_input_swap", "drop_act_from_x3d")


def out_size(n, s):
    return (n - 1) // s + 1


def plan(layers):
    """-> (blocks in forward order, (cout, cin, k) of every filter in state_dict order: conv1, then per block conv1,
    conv2 and the downsample's conv when it has one)."""
    convs, blocks, inplanes = [(64, 8, 3)], [], 64
    for s, n in enumerate(layers):
        for bi in range(n):
            stride = STRIDES[s] if bi == 0 else (1, 1)
            cout = WIDTHS[s]
            c1, c2 = len(convs), len(convs) + 1
            convs += [(cout, inplanes, 3), (cout, cout, 3)]
            ds = -1
            if bi == 0 and (stride != (1, 1) or inplanes != cout):
                ds = len(convs)
                convs.append((cout, inplanes, 1))
            blocks.append(Block(s, bi, inplanes, cout, stride, c1, c2, ds))
            inplanes = cout
    return blocks, convs


def stage_sizes(h, w):
    """-> [(h, w)] of x1 .. x4 for an h x w image."""
    w = out_size(w, 2) // 2
    sizes = []
    for sh, sw in STRIDES:
        h, w = out_size(h, sh), out_size(w, sw)
        sizes.append((h, w))
    return sizes


def resnet_filters(resnet):
    """The trunk's filters of a ResNetModified in state_dict order."""
    f = [resnet.conv1.weight]
    for li in range(1, 5):
        for blk in getattr(resnet, f"layer{li}"):
            f += [blk.conv1.weight, blk.conv2.weight]
            if blk.downsample is not None:
                f.append(blk.downsample[0].weight)
    return f


def bf16(x):
    return x.float().bfloat16().to(x.dtype)


def fp16(x):
    return x.float().half().to(x.dtype)


def fp32(x):
    return x.float().to(x.dtype)


class _Store(torch.autograd.Function):
    """Forward: round to the storage type; backward: the gradient passes unchanged."""

    @staticmethod
    def forward(ctx, x, fn):
        return fn(x)

    @staticmethod
    def backward(ctx, g):
        return g, None


class _GradStore(torch.autograd.Function):
    """Forward: identity; backward: the data gradient as the trunk stores it (bf16 with rounding on), recorded."""

    @staticmethod
    def forward(ctx, x, name, opt):
        ctx.name, ctx.opt = name, opt
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        if ctx.opt.trace is not None:
            ctx.opt.trace["bwd"].append((ctx.name, g.detach()))
        return (bf16(g) if ctx.opt.bwd_round else g), None, None


def x3d(x3, keep, hooks):
    """The stage-3 channel dropout as the trunk stores it: bf16(fp32(x3 * 1.25f)) * keep [B, C] (the fp32 product of a
    bf16 and 1.25 is exact); x3 * 1.25 * keep without the hooks."""
    y = x3 * 1.25
    return (bf16(y) if hooks else y) * keep[:, :, None, None].to(x3)


class _Act(torch.autograd.Function):
    """y = act(x), stored (bf16 with the hooks); act' from the stored y: relu' = y > 0, tanh' = 1 - y^2.
    drop (layer3's output x3 in a dropout step): (keep3 [B, C], opt, defect name) -- the backward multiplies by
    keep * 1.25 after act', as the trunk does: bf16(act'(x3) g) with bwd_round, then keep * 1.25 (the dz2 store that
    follows rounds once more).  The forward's x3d is _Drop3's."""

    @staticmethod
    def forward(ctx, x, act, rnd, drop=None):
        y = torch.relu(x) if act == "relu" else torch.tanh(x)
        if rnd:
            y = bf16(y)
        ctx.act, ctx.drop = act, drop
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, g):
        y, = ctx.saved_tensors
        if ctx.drop is None:
            d = (y > 0).to(y.dtype) if ctx.act == "relu" else 1.0 - y * y
            return g * d, None, None, None
        keep, opt, defect = ctx.drop
        a = x3d(y, keep, opt.hooks) if defect == "drop_act_from_x3d" else y
        g = g * ((a > 0).to(a.dtype) if ctx.act == "relu" else 1.0 - a * a)
        if opt.trace is not None:
            opt.trace["bwd"].append(("g_x3", g.detach()))
        if opt.bwd_round:
            g = bf16(g)
        if defect != "drop_grad_unmasked":
            g = g * keep[:, :, None, None].to(g) * 1.25
        return g, None, None, None


class _Drop3(torch.autograd.Function):
    """Forward: x3d of x3; backward: the gradient passes unchanged (_Act applies keep * 1.25 after act')."""

    @staticmethod
    def forward(ctx, x, keep, hooks):
        return x3d(x, keep, hooks)

    @staticmethod
    def backward(ctx, g):
        return g, None, None


class _Opt:
    def __init__(self, act, hooks, saving, bwd_round, argmax, trace):
        self.act, self.hooks, self.saving, self.bwd_round, self.argmax, self.trace = \
            act, hooks, saving, bwd_round, argmax, trace

    def store(self, x, name, fn=bf16):
        if self.hooks:
            x = _Store.apply(x, fn)
        if self.trace is not None:
            self.trace["fwd"].append((name, x.detach()))
        return x

    def activation(self, x, name, drop=None):
        y = _Act.apply(x, self.act, self.hooks, drop)
        if self.trace is not None:
            self.trace["fwd"].append((name, y.detach()))
            if self.act == "relu":
                self.trace["relu"].append((name, (y > 0).double().mean().item()))
        return y


def conv(x, w, stride, circular=True):
    """The encoder's convolution: 3x3 with circular padding in W (zeros with circular=False: a defect) and zeros in H;
    1x1 without padding."""
    if w.shape[-1] == 1:
        return F.conv2d(x, w, stride=stride)
    x = F.pad(x, (1, 1, 0, 0), mode="circular") if circular else F.pad(x, (1, 1, 0, 0))
    return F.conv2d(x, w, stride=stride, padding=(1, 0))


def maxpool(z, rule="first"):
    """MaxPool2d(3, stride (1, 2)) on the W-wrapped map, rows beyond the image excluded; the winner of a window is its
    first strict maximum in row-major order (rule "last": its last maximum, a defect)."""
    b, c, h, w2 = z.shape
    w4 = w2 // 2
    zp = F.pad(F.pad(z, (1, 1, 0, 0), mode="circular"), (0, 0, 1, 1), value=float("-inf"))
    wins = torch.stack([zp[:, :, dr:dr + h, dq:dq + 2 * w4 - 1:2] for dr in range(3) for dq in range(3)])
    with torch.no_grad():
        best, arg = wins[0].clone(), torch.zeros(wins.shape[1:], dtype=torch.int64, device=z.device)
        for k in range(1, 9):
            take = wins[k] > best if rule == "first" else wins[k] >= best
            best = torch.where(take, wins[k], best)
            arg = torch.where(take, torch.full_like(arg, k), arg)
    return torch.gather(wins, 0, arg[None])[0]


def trunk_input(img1, img2, hooks, keep=None):
    """cat(image_1, image_2) as the trunk reads it: bf16, plus the bf16 rounding residual for an even W.  keep
    [B, 8, H, W] (the input dropout): fp32(x * 1.25f) * keep before the split."""
    x = torch.cat((img1, img2), dim=1).double()
    if not hooks:
        return x if keep is None else x * 1.25 * keep.to(x)
    x32 = x.float()
    if keep is not None:
        x32 = (x32 * 1.25) * keep.float()          # a float32 product, rounded as the kernels round it
    hi = x32.bfloat16().float()
    if x.shape[-1] % 2:
        return hi.double()
    return (hi + (x32 - hi).bfloat16().float()).double()


def trunk(img1, img2, filters, layers, act, hooks=True, saving=True, bwd_round=False, teacher=None, defect=None,
          trace=None, masks=None):
    """-> {"x": [x1 .. x4] NCHW, "pooled": [B, 512]} in float64, differentiable w.r.t. `filters`.

    defect (a negative control): (name, arg) with name in DEFECTS -- zero_pad: conv `arg` pads W with zeros;
    residual_from_input: the first downsampling block of stage `arg` adds its (strided, zero-channel-padded) input
    instead of the downsample; swap_blocks: conv2 of blocks 0 and 1 of stage `arg` trade filters; shift_pair: pair
    `arg` of x1 moves down one row (zero row on top); argmax_last: the pool's winner is the last maximum.  With masks:
    drop_grad_unmasked: the gradient of x3 is not multiplied by keep * 1.25; drop_stage3_shift: the stage-3 mask of
    the next pair (arg "pair") or channel (arg "channel"), cyclically; drop_input_swap: image_1 and image_2 trade
    input masks; drop_act_from_x3d: act' of x3's gradient is taken from x3d (relu cannot see it).
    masks: (keep_input [B, 8, H, W], keep_stage3 [B, 256]) 0 / 1 (dropout_masks), or None for no dropout.
    trace: a dict the design checks fill -- "fwd" / "bwd": (name, tensor) of every store, "relu": (name, fraction of
    relu' = 1), "conv": {conv index: (input, output, stride)}."""
    blocks, _ = plan(layers)
    name, arg = defect if defect else (None, None)
    opt = _Opt(act, hooks, saving, bwd_round, "last" if name == "argmax_last" else "first", trace)
    f = [_Store.apply(w, bf16) if hooks else w for w in filters]
    if name == "swap_blocks":
        bs = [b for b in blocks if b.stage == arg]
        f[bs[0].c2], f[bs[1].c2] = f[bs[1].c2], f[bs[0].c2]
    if trace is not None:
        trace.setdefault("fwd", []), trace.setdefault("bwd", []), trace.setdefault("relu", [])
        trace.setdefault("conv", {})

    def run_conv(x, c, stride):
        y = conv(x, f[c], stride, circular=not (name == "zero_pad" and arg == c))
        if trace is not None:
            trace["conv"][c] = (x.detach(), y, stride)
            y.retain_grad()
        return y

    keep_in = keep3 = None
    if masks is not None:
        keep_in, keep3 = masks
        if name == "drop_input_swap":
            keep_in = torch.cat((keep_in[:, 4:], keep_in[:, :4]), dim=1)
        if name == "drop_stage3_shift":
            keep3 = torch.roll(keep3, -1, dims=0 if arg == "pair" else 1)
    x3_block = max(i for i, b in enumerate(blocks) if b.stage == 2)
    x = opt.store(trunk_input(img1, img2, hooks, keep_in), "input", lambda v: v)
    z = run_conv(x, 0, (1, 2))
    if saving:
        z = opt.store(z, "stem", fp16 if img1.shape[-1] % 2 == 0 else bf16)
        m = maxpool(_GradStore.apply(z, "g_stem", opt), opt.argmax)
        p = torch.relu(m) if act == "relu" else torch.tanh(m)
        if trace is not None and act == "relu":
            trace["relu"].append(("stem", (z > 0).double().mean().item()))
    else:
        p = maxpool(opt.activation(z, "stem"), opt.argmax)
    cur = _GradStore.apply(opt.store(p, "pool"), "g_pool", opt)
    xs = []
    for i, b in enumerate(blocks):
        if b.index == 0 and b.stage > 0 and teacher is not None:
            cur = cur + (teacher[b.stage - 1].to(cur) - cur).detach()
        if keep3 is not None and i == x3_block + 1:
            cur = opt.store(_Drop3.apply(cur, keep3, hooks), "x3d", lambda v: v)
        t1 = opt.activation(_GradStore.apply(run_conv(cur, b.c1, b.stride), f"dz1[{i}]", opt), f"t1[{i}]")
        ident = cur
        if b.ds >= 0:
            if name == "residual_from_input" and b.stage == arg:
                ident = F.pad(cur[:, :, ::b.stride[0], ::b.stride[1]], (0, 0, 0, 0, 0, b.cout - b.cin))
            else:
                ident = opt.store(run_conv(_GradStore.apply(cur, f"gds[{i}]", opt), b.ds, b.stride), f"ds[{i}]")
        pre = run_conv(t1, b.c2, (1, 1)) + ident
        drop = (keep3, opt, name) if keep3 is not None and i == x3_block else None
        cur = opt.activation(_GradStore.apply(pre, f"dz2[{i}]", opt), f"out[{i}]", drop)
        if i + 1 == len(blocks) or blocks[i + 1].stage != b.stage:
            if name == "shift_pair" and b.stage == 0:
                cur = torch.cat((cur[:arg], F.pad(cur[arg:arg + 1, :, :-1], (0, 0, 1, 0)), cur[arg + 1:]))
            xs.append(cur)
    pooled = cur.mean(dim=(2, 3))
    if hooks:
        pooled = _Store.apply(pooled, fp32)
    return {"x": xs, "pooled": pooled}


def weight_grads(out, filters, g_pooled):
    """float64 autograd: the gradient of every filter (conv order) after backward(g_pooled) from `pooled`."""
    gs = torch.autograd.grad(out["pooled"], filters, g_pooled.to(out["pooled"]), allow_unused=True)
    return [torch.zeros_like(w) if g is None else g for w, g in zip(filters, gs)]


SLICE_FLOOR = 0.25


def slice_errors(got, ref, axes):
    """max over the slices along each named axis of ||got - ref||_2 / max(||ref||_2, floor) -> {axis: (worst, index)}.
    floor = SLICE_FLOOR x the RMS slice norm of that axis: a slice far smaller than its siblings (a relu channel alive
    on a few pixels, a channel whose mean cancels) is measured against a quarter of a typical slice, not against its
    own near-zero norm, where a rounding flip of one small element would read as an O(1) error.  A defect confined to
    one slice of typical size is still an O(1) error.  An all-zero reference counts as 0 if got is zero, else infinite."""
    d2 = (got.double() - ref.double()) ** 2
    r2 = ref.double() ** 2
    out = {}
    for k, axis in enumerate(axes):
        dims = [j for j in range(ref.dim()) if j != k]
        num, den = d2.sum(dims).sqrt(), r2.sum(dims).sqrt()
        den = den.clamp_min(SLICE_FLOOR * (den.square().mean().sqrt()).item())
        ratio = torch.where(den > 0, num / den.clamp_min(1e-300),
                            torch.where(num > 0, torch.full_like(num, float("inf")), torch.zeros_like(num)))
        j = int(ratio.argmax())
        out[axis] = (ratio[j].item(), j)
    return out


def worst_slice(got, ref, axes):
    """-> (worst ratio, "axis index") of slice_errors."""
    errs = slice_errors(got, ref, axes)
    axis = max(errs, key=lambda a: errs[a][0])
    return errs[axis][0], f"{axis} {errs[axis][1]}"


X_AXES = ("pair", "channel", "row", "column")
POOLED_AXES = ("pair", "channel")
DW_AXES = ("out", "in")


# ------------------------------------------------------------------------------------------------ exact-tier designs
Design = collections.namedtuple("Design", "layers B H W img1 img2 filters g_pooled x pooled dw stats counter masks")
SUM_MAX = 2 ** 24             # fp32 adds integers below this exactly, in any order


def dropout_masks(seed, step, B, H, W, device="cpu"):
    """The training step's input and stage-3 keep masks at (seed, step) from the numpy generator -> (keep_input
    [B, 8, H, W], keep_stage3 [B, 256]) float64 0 / 1."""
    import numpy as np
    from dropout_reference import INPUT, STAGE3, keep_mask
    k_in = keep_mask(seed, step, INPUT, B * 8 * H * W).reshape(B, 8, H, W)
    k3 = keep_mask(seed, step, STAGE3, B * WIDTHS[2]).reshape(B, WIDTHS[2])
    return tuple(torch.from_numpy(k.astype(np.float64)).to(device) for k in (k_in, k3))


def _taps(g, cout, cin, k, per_out, sign, keep=1.0):
    """A sparse integer filter: per output channel (kept with probability `keep`) `per_out` taps of +-1 at random
    (input channel, tap) positions; sign +1 / -1 forces the sign, 0 draws it."""
    w = torch.zeros((cout, cin * k * k), dtype=torch.float64)
    for o in range(cout):
        if torch.rand((), generator=g).item() >= keep:
            continue
        pos = torch.randperm(cin * k * k, generator=g)[:per_out]
        s = torch.full((per_out,), float(sign), dtype=torch.float64) if sign else \
            torch.randint(0, 2, (per_out,), generator=g).double() * 2 - 1
        w[o, pos] = s
    return w.view(cout, cin, k, k)


def _exact_in(t, fn):
    """Every element an integer that the storage type (fn: bf16 or fp16) represents exactly."""
    return bool((t == t.round()).all()) and torch.equal(fn(t), t)


def exact_design(layers, B, H, W, device="cpu", seed=0, counter=None):
    """An integer design for the exact tier and its float64 reference, with its premises asserted:
    - images of integers in [-2, 2] (the even-W layout's residual channels are exactly 0);
    - the stem and conv1 with +-1 taps of mixed sign, conv2 with -1 taps only and the downsample one +1 tap per output
      channel: t1 >= 0 and conv2(t1) <= 0, so a block's output never exceeds its residual branch and every stored value
      stays a small integer; conv2 is zero from the third block of a stage on (an identity block), so the data
      gradients of deep plans stay within bf16's integers too;
    - g_pooled = k h4 w4 with k in [-2, 2]: the average pool's backward (fp32 g * (1 / (h4 w4)), bf16) gives exactly k.
    counter (step, seed): the input and stage-3 dropouts of a training step at that counter (dropout_masks).  Then the
    images are 16 x [-2, 2] and k is 4 x [-2, 2]: the trunk has no biases and relu is homogeneous, so every value before
    x3d is a multiple of 20 (the masked input is 20 x [-2, 2]) and 1.25 x3 an integer, and every data gradient at x3d
    is a multiple of 4, so that keep * 1.25 times it is one too.
    Asserted: every bf16 store (and x3d, and the gradient of x3 before its mask) an integer that bf16 represents exactly,
    every stem value one that fp16 does on the 16-channel route, every partial sum of the forward, data-gradient and
    weight-gradient convolutions below 2^24, each relu' both 0 and 1 on >= 1 % of its elements, every stage output
    nonzero.  stats: the relu' fractions and the filters with a nonzero gradient."""
    import zlib
    key = (tuple(layers), B, H, W, seed) if counter is None else (tuple(layers), B, H, W, seed, tuple(counter))
    g = torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))
    blocks, convs = plan(layers)
    scale, gscale = (1, 1) if counter is None else (16, 4)
    img = torch.randint(-2, 3, (2, B, 4, H, W), generator=g).float() * scale
    filters = [None] * len(convs)
    filters[0] = _taps(g, 64, 8, 3, 3, 0)
    for b in blocks:
        filters[b.c1] = _taps(g, b.cout, b.cin, 3, 2, 0)
        filters[b.c2] = _taps(g, b.cout, b.cout, 3, 1, -1, keep=0.5 if b.index < 2 else 0.0)
        if b.ds >= 0:
            filters[b.ds] = _taps(g, b.cout, b.cin, 1, 1, 1)
    h4, w4 = stage_sizes(H, W)[3]
    k = torch.randint(-2, 3, (B, 512), generator=g).double() * gscale
    g_pooled = (k * (h4 * w4)).float()
    # the average pool's backward: bf16(g * fp32(1 / (h4 w4))) must be k itself
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(h4 * w4), dtype=torch.float32)
    assert torch.equal(bf16(g_pooled * inv).double(), k), "avgpool backward does not give back k"

    img1, img2 = img[0].to(device), img[1].to(device)
    masks = None if counter is None else dropout_masks(counter[1], counter[0], B, H, W, device)
    fs = [w.to(device).requires_grad_(True) for w in filters]
    trace = {}
    with torch.backends.cudnn.flags(enabled=False):
        out = trunk(img1, img2, fs, layers, "relu", hooks=True, saving=True, bwd_round=True, trace=trace, masks=masks)
        out["pooled"].backward(g_pooled.to(device).double())
    label = f"design {tuple(layers)} B={B} {H}x{W}" + ("" if counter is None else f" counter {counter}")
    for name, t in trace["fwd"]:
        fn = fp16 if name == "stem" and W % 2 == 0 else bf16
        assert _exact_in(t, fn), f"{label}: forward store {name} max {t.abs().max().item()} is not an integer " \
                                 f"exact in {fn.__name__}"
    for name, t in trace["bwd"]:
        assert _exact_in(t, bf16), f"{label}: backward store {name} max {t.abs().max().item()} is not an integer " \
                                   f"exact in bf16"
    for c, (x, y, stride) in trace["conv"].items():
        w = fs[c].detach()
        taps = (w != 0).flatten(1).sum(1).max().item()
        assert taps * x.abs().max().item() < SUM_MAX, f"{label}: conv {c} forward sums"
        dz = y.grad
        assert dz is not None, f"{label}: conv {c} got no gradient"
        taps_t = (w != 0).transpose(0, 1).flatten(1).sum(1).max().item()
        assert taps_t * dz.abs().max().item() < SUM_MAX, f"{label}: conv {c} data-gradient sums"
        # weight gradient: sum over pixels of |x| |dz| per element, bounded cheaply, exactly when the bound is loose
        cheap = x.abs().max().item() * dz.abs().sum(dim=(0, 2, 3)).max().item()
        if cheap >= SUM_MAX:
            xa = x.abs() if w.shape[-1] == 1 else F.pad(x.abs(), (1, 1, 0, 0), mode="circular")
            pad = 0 if w.shape[-1] == 1 else (1, 0)
            with torch.backends.cudnn.flags(enabled=False):
                cheap = torch.nn.grad.conv2d_weight(xa, w.shape, dz.abs(), stride=stride, padding=pad).max().item()
        assert cheap < SUM_MAX, f"{label}: conv {c} weight-gradient partial sums reach {cheap}"
    fractions = []
    for name, fr in trace["relu"]:
        assert 0.01 <= fr <= 0.99, f"{label}: relu' of {name} is 1 on {fr:.4f} of the elements"
        fractions.append((name, fr))
    for s, xs in enumerate(out["x"]):
        assert xs.abs().max().item() > 0, f"{label}: x{s + 1} is zero"
    dw = [w.grad.detach() for w in fs]
    stats = {"relu": fractions, "nonzero_dw": [c for c, d in enumerate(dw) if d.abs().max().item() > 0]}
    # the trace's graph tensors and the autograd contexts that hold the trace form reference cycles: release them now,
    # or a matrix of designs in one process keeps every design's graph until a full garbage collection
    trace.clear()
    total = out["x"][3].detach().sum(dim=(2, 3))
    assert bool((total.abs() < SUM_MAX).all()), f"{label}: the average pool's sums reach 2^24"
    return Design(tuple(layers), B, H, W, img1, img2, [w.detach() for w in fs], g_pooled.to(device),
                  [t.detach() for t in out["x"]], out["pooled"].detach(), dw, stats, counter, masks)


def dw_coverage(layers, nonzero):
    """Convolution positions of a plan with a nonzero weight gradient: "stem", ("first", stage, "c1" / "c2" / "ds"),
    ("later", stage, "c1" / "c2")."""
    blocks, _ = plan(layers)
    got = {"stem"} if 0 in nonzero else set()
    for b in blocks:
        where = "first" if b.index == 0 else "later"
        for part in ("c1", "c2", "ds"):
            c = getattr(b, part)
            if c >= 0 and c in nonzero:
                got.add((where, b.stage, part))
    return got


def dgrad_routes(layers, H, W, eligible):
    """The data-gradient route of every strided block after the first (the trunk's rule): "phase" when
    eligible(cin, cout, win, stride), else "fallback" -> [(block index, route)]."""
    blocks, _ = plan(layers)
    w = out_size(W, 2) // 2
    h = H
    routes = []
    for i, b in enumerate(blocks):
        if b.ds >= 0 and i > 0:
            routes.append((i, "phase" if eligible(b.cin, b.cout, w, b.stride) else "fallback"))
        h, w = out_size(h, b.stride[0]), out_size(w, b.stride[1])
    return routes
