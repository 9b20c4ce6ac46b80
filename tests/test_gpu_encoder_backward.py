"""-m gpu: the encoder's backward kernels layer by layer against float64 autograd on the same bf16 operands.

Covered here: the phase-decomposed data gradient of the strided 3x3 convolutions (delora_conv2d_dgrad_bf16) and its
fallback (zero-upsampled gradient through the stride-1 fprop), the act' epilogue modes of the stride-1 fprop (act 3 =
tanh', 4 = relu' of the saved forward output, with and without residual) in both kernels, the 1x1 stride-1 fprop (the
downsample's data gradient), the average-pool backward and the inference max pool.

Bar of the convolutions, per element:  |got - ref| <= 2^-8 |ref| + (n + 3) 2^-24 ref_abs,  with ref_abs the same
expression evaluated on |dz|, |w|, |residual| and |act'|, and n the products summed per output element (taps x
channels): one bf16 output rounding plus a worst-case bound on the fp32 accumulation.  It cannot flake, and one missing
or misplaced tap exceeds it by more than an order of magnitude.  Every case prints its worst err / bound (`pytest -s`);
round-to-nearest bf16 alone may use 2^-8 / (1 + 2^-8) = 0.996 of the first term, so worst ratios of 0.9 .. 0.99 are
the output rounding, and the fp32 accumulation lives in the second term's slack.

The weight gradients (delora_conv2d_wgrad_bf16: conv_wgrad.cu's wgrad2 modes 0 / 1 and conv_tc.cu's first-generation
kernel; delora_stem_wgrad_bf16: wgrad2 mode 2) are called through the C ABI, every kernel path and both reduce kernels:
- Integer operands in [-r, r] with n r^2 < 2^23 (n = products per dW element, asserted): every product is exact in
  bf16 x bf16 and every partial sum is an integer below 2^23, so any order of fp32 adds -- the wgmma accumulator even
  with a truncating adder, the split-K slices and the reduce -- gives the true sum.  The fp32 dW has no output
  rounding, so it must equal float64 autograd bit for bit: one missing, doubled or misplaced product fails at any K.
- Gaussian bf16 operands: |got - ref| <= (n + 3) 2^-23 ref_abs (2^-23, not 2^-24: the tensor-core adder need not
  round to nearest), and two calls bit-identical (the split-K reduction has a fixed order and no atomics).
- The scratch is exactly the size query's floats, NaN-filled, with a NaN guard behind it; dW is a slice of a NaN
  buffer; the output gradient's halo holds junk.  A finite dW shows every split-K slot the reduce read was written in
  that call, the untouched guards that the query covers the launch and that nothing lands outside dW, and the exact
  result that the halo is not read.  Input channels >= Cin_true hold nonzero values the reduce must drop.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from helpers import (DEV, FPROP_BWD_SHAPES, check_bound, check_exact, check_layout, conv3, conv_ref, generator,
                     interior, rand_bf16, rand_int, run_twice, sentinel_out, to_padded_nhwc)

pytestmark = pytest.mark.gpu


def saved_values(g, shape, act):
    """Saved forward outputs for act' (bf16 values): tanh outputs, some saturated to exactly +-1 (tanh' = 0); for relu'
    a signed map with exact zeros and negatives (relu' = 0 there)."""
    z = torch.randn(shape, generator=g, device=DEV, dtype=torch.float64)
    if act == 3:
        s = torch.tanh(2.5 * z)
    else:
        s = z.masked_fill(torch.rand(shape, generator=g, device=DEV) < 0.2, 0.0)
    return s.to(torch.bfloat16).double()


def act_prime(s, act):
    """act' in float64 from the bf16 saved tensor itself: 1 - s^2 (tanh') or s > 0 (relu')."""
    return 1.0 - s * s if act == 3 else (s > 0).double()


def dgrad_ref(dz, w, hin, win, stride):
    """x.grad of conv3 at an Hin x Win input after backward(dz), float64 autograd."""
    x = torch.zeros((dz.shape[0], w.shape[1], hin, win), dtype=torch.float64, device=DEV, requires_grad=True)
    conv3(x, w, stride).backward(dz)
    return x.grad


def epilogue_ref(conv, res, res_stride, d):
    """(conv + residual) * act': the residual on every pixel, or on the (sh*h, sw*w) pixels only (res_stride)."""
    out = conv.clone()
    if res is not None:
        out[..., ::res_stride[0], ::res_stride[1]] += res
    return out if d is None else out * d


# ------------------------------------------------------------------------------------------------ data gradient
DGRAD_SHAPES = [   # forward layer B, Cin, Cout, Hin, Win, stride; the data gradient maps Cout -> Cin channels
    (2, 64, 128, 8, 512, (1, 2)),      # pixel-on-M, 64 channels, two 128-pixel segments (64x2048 trunk)
    (2, 128, 256, 8, 256, (1, 2)),     # pixel-on-M, 128 channels (64x2048)
    (2, 256, 512, 9, 128, (2, 2)),     # 128-channel tiles, odd Hin (64x2048 layer shape)
    (2, 128, 256, 6, 90, (1, 2)),      # 48-pixel segments: the last 64-pixel chunk reads past the row (64x720)
    (3, 256, 512, 7, 12, (2, 2)),      # job grid 6 wide, 16-pixel segments (16x180)
    (2, 64, 128, 5, 258, (1, 2)),      # pixel-on-M with a 1-pixel second segment
    (2, 64, 128, 4, 256, (1, 2)),      # exactly 128 columns per phase
    (2, 256, 512, 1, 64, (2, 2)),      # Hin = 1
    (2, 128, 128, 3, 7, (1, 1)),       # stride 1 through the phase kernel
]
# act, residual: "grid" = the downsample's gradient on the job grid, landing on the (sh*h, sw*w) pixels (the trunk's
# mode); "full" = a residual of the output's size; None = no residual
DGRAD_CASES = [(s, a, r) for s in DGRAD_SHAPES for a, r in ((3, "grid"), (4, "grid"), (0, None))]
DGRAD_CASES += [(DGRAD_SHAPES[0], 4, "full"), (DGRAD_SHAPES[4], 3, "full")]
# the fallback route (zero_upsample + stride-1 fprop) on the same reference; the last shape has an odd width under
# stride 2, which the phase kernel does not take: its fallback runs on the first-generation kernel (conv_tc.cu)
FALLBACK_SHAPES = DGRAD_SHAPES[:3] + [(2, 64, 128, 5, 45, (1, 2))]
FALLBACK_CASES = [(s, a, r) for s in FALLBACK_SHAPES for a, r in ((3, "grid"), (4, "grid"))]
FALLBACK_CASES += [(s, 0, None) for s in DGRAD_SHAPES[:3]] + [(DGRAD_SHAPES[0], 3, "full")]


def _case_id(case):
    (b, cin, cout, h, w, st), act, res = case
    return f"{cin}x{cout}-{h}x{w}-s{st[0]}{st[1]}-b{b}-act{act}-{res or 'nores'}"


def dgrad_problem(shape, act, res):
    """bf16 operands of a data-gradient case in the kernels' layouts, and the float64 reference."""
    from delora_b200 import ops
    b, cin, cout, hin, win, stride = shape
    hout, wout = ops.conv_out_size(hin, stride[0]), ops.conv_out_size(win, stride[1])
    g = torch.Generator(device=DEV).manual_seed(cin * 7 + cout * 3 + hin * 11 + win + act * 1000)
    dz = rand_bf16(g, (b, cout, hout, wout))
    wt = rand_bf16(g, (cout, cin, 3, 3), (9 * cout) ** -0.5)
    r = None
    if res == "grid":
        r = rand_bf16(g, (b, cin, hout, wout))
    elif res == "full":
        r = rand_bf16(g, (b, cin, hin, win))
    s = saved_values(g, (b, cin, hin, win), act) if act >= 3 else None
    d = act_prime(s, act) if s is not None else None
    rs = stride if res == "grid" else (1, 1)
    ref = epilogue_ref(dgrad_ref(dz, wt, hin, win, stride), r, rs, d)
    ref_abs = epilogue_ref(dgrad_ref(dz.abs(), wt.abs(), hin, win, stride), None if r is None else r.abs(), rs,
                           None if d is None else d.abs())
    w_flip = wt.flip(2, 3).permute(1, 2, 3, 0).reshape(cin, 9, cout).contiguous().to(torch.bfloat16)
    return {"dz": to_padded_nhwc(dz), "w_flip": w_flip, "res": None if r is None else to_padded_nhwc(r),
            "saved": None if s is None else to_padded_nhwc(s), "ref": ref, "ref_abs": ref_abs, "n": 9 * cout,
            "hout": hout, "wout": wout}


@pytest.mark.parametrize("case", DGRAD_CASES, ids=_case_id)
def test_dgrad_matches_float64_autograd(case, cuda_lib):
    """delora_conv2d_dgrad_bf16 called directly: every phase, segment and the seam column against autograd."""
    from delora_b200 import ops
    shape, act, res = case
    b, cin, cout, hin, win, stride = shape
    assert ops.conv2d_dgrad_eligible(cin, cout, win, stride)
    p = dgrad_problem(shape, act, res)
    label = "dgrad " + _case_id(case)

    def call():
        out = sentinel_out(b, hin, win, cin)
        ops.conv2d_dgrad(p["dz"], p["w_flip"], hin, win, stride, act, p["res"], out, p["saved"],
                         residual_strided=(res == "grid"))
        check_layout(out, hin, win, label)
        return out
    out = run_twice(call, label)
    check_bound(interior(out, hin, win), p["ref"], p["ref_abs"], p["n"], label)


@pytest.mark.parametrize("case", FALLBACK_CASES, ids=_case_id)
def test_dgrad_fallback_matches_float64_autograd(case, cuda_lib):
    """The route of the layers the phase kernel does not take: the output gradient (and the grid residual) zero-
    upsampled, then the stride-1 fprop with the flipped filter and the same act' / residual epilogue."""
    from delora_b200 import ops
    shape, act, res = case
    b, cin, cout, hin, win, stride = shape
    p = dgrad_problem(shape, act, res)
    label = "fallback " + _case_id(case)
    up = stride != (1, 1)

    def call():
        src = ops.zero_upsample(p["dz"], p["hout"], p["wout"], stride, out_hw=(hin, win)) if up else p["dz"]
        resid = p["res"]
        if res == "grid" and up:
            resid = ops.zero_upsample(resid, p["hout"], p["wout"], stride, out_hw=(hin, win))
        out = sentinel_out(b, hin, win, cin)
        ops.conv2d_fprop(src, p["w_flip"], hin, win, 3, (1, 1), act, resid, out, saved=p["saved"])
        check_layout(out, hin, win, label)
        return out
    out = run_twice(call, label)
    check_bound(interior(out, hin, win), p["ref"], p["ref_abs"], p["n"], label)


# ------------------------------------------------------------------------------------------------ stride-1 fprop
# FPROP_BWD_SHAPES (helpers.py) are shared with the forward epilogue tests of test_gpu_encoder_forward.py
FPROP_BWD_CASES = [(s, a, r) for s in FPROP_BWD_SHAPES for a in (3, 4) for r in (False, True)]
ONE_BY_ONE_SHAPES = [          # B, Cin, Cout, H, W: the 1x1 stride-1 convolution forming the downsample's gradient
    (2, 512, 256, 4, 64),      # conv_rows, 128 output channels on M
    (2, 256, 128, 4, 128),     # conv_rows pixel-on-M
    (2, 128, 64, 5, 45),       # conv_tc
]


def _fprop_check(b, cin, cout, h, w, k, act, use_res, label):
    from delora_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(cin * 5 + cout + h * 13 + w * 3 + k + act * 100 + use_res)
    x = rand_bf16(g, (b, cin, h, w))
    wt = rand_bf16(g, (cout, cin, k, k), (k * k * cin) ** -0.5)
    r = rand_bf16(g, (b, cout, h, w)) if use_res else None
    s = saved_values(g, (b, cout, h, w), act) if act >= 3 else None
    d = act_prime(s, act) if s is not None else None
    conv = conv3 if k == 3 else (lambda xx, ww, st: F.conv2d(xx, ww))
    ref = epilogue_ref(conv(x, wt, (1, 1)), r, (1, 1), d)
    ref_abs = epilogue_ref(conv(x.abs(), wt.abs(), (1, 1)), None if r is None else r.abs(), (1, 1),
                           None if d is None else d.abs())
    wn = wt.permute(0, 2, 3, 1).reshape(cout, k * k, cin).contiguous().to(torch.bfloat16)
    xp, rp, sp = to_padded_nhwc(x), None if r is None else to_padded_nhwc(r), None if s is None else to_padded_nhwc(s)

    def call():
        out = sentinel_out(b, h, w, cout)
        ops.conv2d_fprop(xp, wn, h, w, k, (1, 1), act, rp, out, saved=sp)
        check_layout(out, h, w, label)
        return out
    out = run_twice(call, label)
    check_bound(interior(out, h, w), ref, ref_abs, k * k * cin, label)


@pytest.mark.parametrize("shape,act,use_res", FPROP_BWD_CASES,
                         ids=[f"{c[0][1]}x{c[0][2]}-{c[0][3]}x{c[0][4]}-act{c[1]}-{'res' if c[2] else 'nores'}"
                              for c in FPROP_BWD_CASES])
def test_fprop_act_prime_epilogue(shape, act, use_res, cuda_lib):
    b, cin, cout, h, w = shape
    _fprop_check(b, cin, cout, h, w, 3, act, use_res, f"fprop act{act} res={use_res} {cin}x{cout} {h}x{w}")


@pytest.mark.parametrize("shape", ONE_BY_ONE_SHAPES, ids=[f"{s[1]}x{s[2]}-{s[3]}x{s[4]}" for s in ONE_BY_ONE_SHAPES])
def test_fprop_1x1_stride1(shape, cuda_lib):
    b, cin, cout, h, w = shape
    _fprop_check(b, cin, cout, h, w, 1, 0, False, f"fprop 1x1 {cin}x{cout} {h}x{w}")


# ------------------------------------------------------------------------------------------------ weight gradient
# Forward layer (B, Cin, Cout, Hin, Win, k, stride), input channels kept (Cin_true; None = Cin), and the kernel path
# delora_conv2d_wgrad_bf16 takes for it (conv_wgrad.cu: wgrad2 mode 0 for Cout % 128 == 0, mode 1 for Cout = 64 at
# stride 1; conv_tc.cu: conv_wgrad_tc_kernel for 1x1 and for strided layers with Cout = 64)
WGRAD_CASES = [
    ("mode1", (2, 64, 64, 8, 512, 3, (1, 1)), None),        # four 128-pixel segments
    ("mode1", (1, 64, 64, 6, 180, 3, (1, 1)), None),        # ragged second segment
    ("mode1", (2, 64, 64, 3, 129, 3, (1, 1)), None),        # 1-pixel second segment
    ("mode1", (1, 128, 64, 1, 7, 3, (1, 1)), None),         # Hout = 1, NS = 16, two ci tiles, one K row: one split
    ("mode1", (1, 64, 64, 6, 180, 3, (1, 1)), 37),          # Cin_true < Cin through wgrad2_reduce_kernel
    ("mode0", (2, 128, 128, 8, 256, 3, (1, 1)), None),
    ("mode0", (2, 512, 512, 4, 64, 3, (1, 1)), None),
    ("mode0", (1, 512, 512, 5, 23, 3, (1, 1)), None),       # NS = 32, one ragged segment
    ("mode0", (2, 64, 128, 8, 512, 3, (1, 2)), None),       # strided: even / odd column tiles
    ("mode0", (1, 128, 256, 6, 90, 3, (1, 2)), None),       # NS = 48
    ("mode0", (2, 256, 512, 9, 128, 3, (2, 2)), None),      # odd Hin
    ("mode0", (1, 256, 512, 5, 45, 3, (2, 2)), None),       # odd Win, Wout = 23
    ("mode0", (2, 64, 128, 4, 130, 3, (1, 2)), None),       # 1-pixel second segment at the stride-2 cap of 64
    ("mode0", (1, 128, 256, 6, 90, 3, (1, 2)), 70),         # Cin_true < Cin, strided
    ("gen1", (2, 64, 128, 8, 512, 1, (1, 2)), None),        # 1x1 downsamples: nb = 1
    ("gen1", (1, 128, 256, 6, 90, 1, (1, 2)), None),        # nb = 2
    ("gen1", (2, 256, 512, 9, 45, 1, (2, 2)), None),        # nb = 4
    ("gen1", (2, 64, 64, 6, 90, 3, (1, 2)), None),          # 3x3, Cout 64, strided: tap group tg = 3
    ("gen1", (2, 128, 64, 5, 64, 3, (1, 2)), None),         # tg = 2: groups of taps (0, 1) and (2)
    ("gen1", (1, 256, 64, 7, 46, 3, (2, 2)), None),         # tg = 1
    ("gen1", (2, 64, 64, 5, 181, 3, (1, 2)), 8),            # the odd-width stem: 8 real channels padded to 64
]
# the stem kernel (conv_stem.cu, wgrad2 mode 2): B, H, W of the image, Cin_true
STEM_WGRAD_CASES = [
    (2, 64, 2048, 8),       # the bench shape: 8 segments per row, 132 splits
    (1, 16, 180, 8),        # one ragged segment
    (1, 1, 10, 4),          # Cin_true = 4, one K row
    (3, 5, 258, 8),         # 1-pixel second segment
]
# the Gaussian tier: a subset covering every kernel and both reduce kernels
WGRAD_GAUSS_CASES = [WGRAD_CASES[i] for i in (1, 4, 6, 10, 12, 13, 15, 18, 20)]
STEM_WGRAD_GAUSS_CASES = [STEM_WGRAD_CASES[i] for i in (0, 2, 3)]
GUARD = 4096            # fp32 NaN guard floats behind the scratch and on both sides of dW


def _wgrad_id(case):
    path, (b, cin, cout, h, w, k, st), ct = case
    return f"{path}-{cin}x{cout}-k{k}-{h}x{w}-s{st[0]}{st[1]}-b{b}" + (f"-cin{ct}" if ct else "")


def _stem_id(case):
    b, h, w, ct = case
    return f"stem-{h}x{w}-b{b}-cin{ct}"


def wgrad_ref(x, dz, k, stride):
    """w.grad of the layer's convolution (conv_ref) after backward(dz), float64 autograd."""
    w = torch.zeros((dz.shape[1], x.shape[1], k, k), dtype=torch.float64, device=DEV, requires_grad=True)
    conv_ref(x, w, stride).backward(dz)
    return w.grad


def int_range(n):
    """Largest r <= 8 with n r^2 < 2^23: every partial sum of n products of integers in [-r, r] is then an integer
    below 2^23, so fp32 adds it exactly in any order and with any rounding mode."""
    return max(1, min(8, math.isqrt((2 ** 23 - 1) // n)))


def assert_exact_premise(n, dz, x, label):
    bound = n * dz.abs().max().item() * x.abs().max().item()
    assert bound < 2 ** 23, f"{label}: n max|dz| max|x| = {bound} does not keep the partial sums exact"


def padded_grad(dz, junk):
    """The output gradient in the padded layout with `junk` in all of its halo: the weight gradients never read it
    (their dz maps stop at the last real pixel), so a halo read changes the result."""
    p = to_padded_nhwc(dz)
    p[:, 0] = junk
    p[:, -1] = junk
    p[:, :, 0] = junk
    p[:, :, -1] = junk
    return p


def guarded_wgrad(launch, n_scratch, out_shape, label):
    """launch(dw_ptr, scratch_ptr) with exactly n_scratch scratch floats (the size query's answer) pre-filled with NaN
    and followed by a NaN guard, and dW a slice in the middle of a NaN buffer.  Finite dW: every element written, and
    every split-K slot the reduce read written by this call (the scratch is reused across layers).  Unchanged guards:
    the query covers every kernel of the launch, and nothing lands outside dW."""
    numel = math.prod(out_shape)
    scratch = torch.full((n_scratch + GUARD,), float("nan"), dtype=torch.float32, device=DEV)
    buf = torch.full((GUARD + numel + GUARD,), float("nan"), dtype=torch.float32, device=DEV)
    launch(buf[GUARD:GUARD + numel].data_ptr(), scratch.data_ptr())
    nan_bits = torch.full((GUARD,), float("nan"), dtype=torch.float32, device=DEV).view(torch.int32)
    assert torch.equal(scratch[n_scratch:].view(torch.int32), nan_bits), \
        f"{label}: written past the {n_scratch} scratch floats of the size query"
    assert torch.equal(buf[:GUARD].view(torch.int32), nan_bits) and \
        torch.equal(buf[GUARD + numel:].view(torch.int32), nan_bits), f"{label}: written outside the dW slice"
    dw = buf[GUARD:GUARD + numel].view(out_shape)
    bad = ~torch.isfinite(dw)
    assert not bool(bad.any()), f"{label}: {int(bad.sum())} non-finite dW elements (unwritten, or built from a split-K " \
                                f"slot not written this call), first (co, ci, r, q) = {tuple(bad.nonzero()[0].tolist())}"
    return dw


def wgrad_problem(case, exact):
    """Operands of a delora_conv2d_wgrad_bf16 case in the kernels' layouts, the float64 reference and the launcher."""
    from delora_b200 import ops
    L = ops._lib.lib()
    _, (b, cin, cout, hin, win, k, stride), cin_true = case
    ct = cin if cin_true is None else cin_true
    hout, wout = ops.conv_out_size(hin, stride[0]), ops.conv_out_size(win, stride[1])
    n = b * hout * wout                                     # products per dW element
    g = generator("wgrad", case, exact)
    if exact:
        r = int_range(n)
        x, dz = rand_int(g, (b, cin, hin, win), r), rand_int(g, (b, cout, hout, wout), r)
        assert_exact_premise(n, dz, x, _wgrad_id(case))
    else:
        x, dz = rand_bf16(g, (b, cin, hin, win)), rand_bf16(g, (b, cout, hout, wout))
    # channels ct .. Cin of x hold nonzero values: the reduce must drop them
    ref = wgrad_ref(x[:, :ct], dz, k, stride)
    ref_abs = None if exact else wgrad_ref(x[:, :ct].abs(), dz.abs(), k, stride)
    xp, dzp = to_padded_nhwc(x), padded_grad(dz, 3.0 if exact else 1.0)
    n_scratch = int(L.delora_conv2d_wgrad_scratch_floats(b, hout, wout, cin, cout, k))

    def launch(dw_ptr, scratch_ptr):
        ops._lib.check(L.delora_conv2d_wgrad_bf16(ops._req(xp, torch.bfloat16, "x"), ops._req(dzp, torch.bfloat16, "dz"),
                                                  dw_ptr, scratch_ptr, b, hin, win, cin, ct, cout, k, stride[0], stride[1],
                                                  ops._stream()), "delora_conv2d_wgrad_bf16")
    return launch, n_scratch, (cout, ct, k, k), ref, ref_abs, n


def stem_wgrad_problem(case, exact):
    """Operands of a delora_stem_wgrad_bf16 case: the 16-channel input whose channels c and c + 8 (bf16(x) and its
    rounding residual) get independent values and share one weight, so dW = sum dz (x[c] + x[c + 8])."""
    from delora_b200 import ops
    L = ops._lib.lib()
    b, h, w, ct = case
    wout = w // 2
    n = 2 * b * h * wout
    g = generator("stem wgrad", case, exact)
    if exact:
        r = int_range(n)
        x, dz = rand_int(g, (b, 16, h, w), r), rand_int(g, (b, 64, h, wout), r)
        assert_exact_premise(n, dz, x, _stem_id(case))
    else:
        x = torch.cat([rand_bf16(g, (b, 8, h, w)), rand_bf16(g, (b, 8, h, w), 2.0 ** -8)], dim=1)
        dz = rand_bf16(g, (b, 64, h, wout))
    # channels ct .. 7 and 8 + ct .. 15 hold nonzero values: the reduce must drop them
    ref = wgrad_ref(x[:, :ct] + x[:, 8:8 + ct], dz, 3, (1, 2))
    ref_abs = None if exact else wgrad_ref(x[:, :ct].abs() + x[:, 8:8 + ct].abs(), dz.abs(), 3, (1, 2))
    xp, dzp = to_padded_nhwc(x), padded_grad(dz, 3.0 if exact else 1.0)
    n_scratch = int(L.delora_stem_wgrad_scratch_floats(b, h, w))

    def launch(dw_ptr, scratch_ptr):
        ops._lib.check(L.delora_stem_wgrad_bf16(ops._req(xp, torch.bfloat16, "x16"), ops._req(dzp, torch.bfloat16, "dz"),
                                                dw_ptr, scratch_ptr, b, h, w, ct, ops._stream()), "delora_stem_wgrad_bf16")
    return launch, n_scratch, (64, ct, 3, 3), ref, ref_abs, n


def _wgrad_exact(problem, label):
    launch, n_scratch, out_shape, ref, _, _ = problem
    check_exact(guarded_wgrad(launch, n_scratch, out_shape, label).double(), ref, label)


def _wgrad_gauss(problem, label):
    launch, n_scratch, out_shape, ref, ref_abs, n = problem
    a = guarded_wgrad(launch, n_scratch, out_shape, label)
    b = guarded_wgrad(launch, n_scratch, out_shape, label)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{label}: two calls differ"
    check_bound(a.double(), ref, ref_abs, n, label, out_unit=0.0, acc_unit=2.0 ** -23)


@pytest.mark.parametrize("case", WGRAD_CASES, ids=_wgrad_id)
def test_wgrad_exact_on_integers(case, cuda_lib):
    """delora_conv2d_wgrad_bf16 on integer operands equals float64 autograd bit for bit."""
    _wgrad_exact(wgrad_problem(case, True), "wgrad exact " + _wgrad_id(case))


@pytest.mark.parametrize("case", STEM_WGRAD_CASES, ids=_stem_id)
def test_stem_wgrad_exact_on_integers(case, cuda_lib):
    """delora_stem_wgrad_bf16 on integer operands equals float64 autograd bit for bit."""
    _wgrad_exact(stem_wgrad_problem(case, True), "wgrad exact " + _stem_id(case))


@pytest.mark.parametrize("case", WGRAD_GAUSS_CASES, ids=_wgrad_id)
def test_wgrad_gaussian(case, cuda_lib):
    """Gaussian bf16 operands: deterministic (two calls bit-identical) and within the fp32 accumulation bound."""
    _wgrad_gauss(wgrad_problem(case, False), "wgrad gauss " + _wgrad_id(case))


@pytest.mark.parametrize("case", STEM_WGRAD_GAUSS_CASES, ids=_stem_id)
def test_stem_wgrad_gaussian(case, cuda_lib):
    _wgrad_gauss(stem_wgrad_problem(case, False), "wgrad gauss " + _stem_id(case))


# ------------------------------------------------------------------------------------------------ pools
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("b,h,w,c", [(2, 32, 64, 512), (1, 32, 23, 512), (2, 4, 6, 512)])
def test_avgpool_backward_matches_float64(b, h, w, c, act, cuda_lib):
    """dz = g / (H W) * act'(a) with act' from the bf16 block output a (act 1: a > 0, act 2: 1 - a^2)."""
    from delora_b200 import ops
    L = ops._lib.lib()
    gen = torch.Generator(device=DEV).manual_seed(b * 1000 + h * 10 + w + act)
    gp = torch.randn((b, c), generator=gen, device=DEV)
    a = saved_values(gen, (b, c, h, w), 3 if act == 2 else 4)       # tanh outputs, or signed with exact zeros
    a_p = to_padded_nhwc(a)
    d = torch.ones_like(a) if act == 0 else act_prime(a, 3 if act == 2 else 4)
    ref = gp.double()[:, :, None, None] / (h * w) * d
    dz = sentinel_out(b, h, w, c)
    ops._lib.check(L.delora_avgpool_bwd_nhwc_bf16(ops._req(gp, torch.float32, "g"), a_p.data_ptr(), b, h, w, c, act,
                                                  dz.data_ptr(), ops._stream()), "delora_avgpool_bwd_nhwc_bf16")
    label = f"avgpool bwd act{act} {b}x{h}x{w}x{c}"
    check_layout(dz, h, w, label)
    got = interior(dz, h, w)
    err = (got - ref).abs()
    worst = torch.where(err == 0, torch.zeros_like(err), err / (2.0 ** -8 * ref.abs())).max().item()
    print(f"{label}: worst err/bound {worst:.4f}", flush=True)
    assert worst <= 1.0, f"{label}: err / (2^-8 |ref|) = {worst:.3g}"


@pytest.mark.parametrize("w", [1024, 360, 256, 90, 48])
def test_maxpool_w_bit_exact(w, cuda_lib):
    """The inference max pool (3x3, stride (1, 2), circular in W, rows beyond the image excluded) bit for bit against
    torch's max_pool2d on the circular / -inf padded map; its H halo rows hold junk that must not be read."""
    from delora_b200 import ops
    b, c, wo = 2, 64, w // 2
    for h in (1, 4, 7):
        g = torch.Generator(device=DEV).manual_seed(w * 10 + h)
        z = torch.randn((b, c, h, w), generator=g, device=DEV).to(torch.bfloat16).float()
        x = F.pad(F.pad(z, (1, 1, 0, 0), mode="circular"), (0, 0, 1, 1), value=100.0)
        x = x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
        zinf = F.pad(F.pad(z, (1, 1, 0, 0), mode="circular"), (0, 0, 1, 1), value=float("-inf"))
        ref = F.max_pool2d(zinf, 3, stride=(1, 2))
        assert ref.shape[-1] == wo
        y = ops.maxpool_w(x, h, w)
        got = y[:, 1:h + 1, 1:wo + 1].permute(0, 3, 1, 2).float()
        assert torch.equal(got, ref), f"maxpool {h}x{w}: {int((got != ref).sum())} outputs differ"
        yb = y.view(torch.int16)
        assert torch.equal(yb[:, 1:h + 1, 0], yb[:, 1:h + 1, wo]) and torch.equal(yb[:, 1:h + 1, wo + 1], yb[:, 1:h + 1, 1])
        assert float(y[:, 0].float().abs().max()) == 0.0 and float(y[:, h + 1].float().abs().max()) == 0.0
