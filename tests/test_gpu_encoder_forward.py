"""-m gpu: the encoder's forward convolutions layer by layer against float64 on the same bf16 operands.

Covered here: the strided 3x3 layers and the 1x1 strided downsamples on the first-generation conv_fprop_tc_kernel
(conv_tc.cu; the row kernel takes stride 1 only), the odd-width stem on the same kernel (8 real channels padded to 64),
the forward epilogues act 1 (relu) and act 2 (tanh) with and without residual at stride 1 in both kernels
(FPROP_BWD_SHAPES: conv_rows.cu and conv_tc.cu), and the stem delora_stem_fprop_bf16 (conv_stem.cu), whose 16 input
channels are bf16(x) in c and its rounding residual in c + 8, both multiplied by the weight of channel c.

Bar on Gaussian operands, per element:  |got - ref| <= 2^-8 |ref| + (n + 3) 2^-24 ref_abs  (2^-11 |ref| for the stem's
fp16 output), with ref_abs the convolution (+ residual) of the absolute values and n the products summed per output:
one output rounding plus a worst-case bound on the fp32 accumulation.  relu and tanh are 1-Lipschitz, so the
accumulation term carries through them.  act 2 runs tanh.approx.f32, for which the PTX ISA states a maximum relative
error of 2^-10.987 over the full range: its bar adds 2^-10.987 |ref|.

Exact tier (act 0 and 1): integer operands and an integer residual, |ref| <= 256 asserted (<= 2048 for the fp16
stem output).  Every product and partial sum is then an integer below 2^24 and the result is representable, so the
output must equal the float64 reference bit for bit.

Layout: every output goes into a sentinel buffer (NaN rows 1..H, HALO_ROW in rows 0 and H+1).  All three kernels'
epilogues (epilogue_store32, and the stem's own store) write the H x W interior and its circular halo columns 0 / W+1,
and never the zero halo rows: those must still hold HALO_ROW.  Two calls must agree bit for bit.
"""
import pytest
import torch

from helpers import (DEV, FPROP_BWD_SHAPES, check_bound, check_exact, check_layout, conv3, conv_ref, generator,
                     interior, rand_bf16, rand_int, run_twice, sentinel_out, to_padded_nhwc)

pytestmark = pytest.mark.gpu

TANH_APPROX_REL_ERR = 2.0 ** -10.987     # PTX ISA, tanh.approx.f32: maximum relative error over the full range

# forward layer B, Cin, Cout, Hin, Win, k, stride, Cin_true (None = Cin): all on conv_fprop_tc_kernel
STRIDED_SHAPES = [
    (2, 64, 128, 8, 512, 3, (1, 2), None),
    (1, 128, 256, 6, 90, 3, (1, 2), None),
    (2, 256, 512, 9, 128, 3, (2, 2), None),     # odd Hin
    (1, 256, 512, 5, 45, 3, (2, 2), None),      # odd Win, Wout = 23
    (2, 64, 128, 4, 130, 3, (1, 2), None),
    (2, 64, 64, 6, 90, 3, (1, 2), None),        # Cout 64: one 64-channel block of N
    (2, 128, 64, 5, 64, 3, (1, 2), None),
    (1, 256, 64, 7, 46, 3, (2, 2), None),
]
DOWNSAMPLE_SHAPES = [                           # the 1x1 strided downsamples (pad_off = 1)
    (2, 64, 128, 8, 512, 1, (1, 2), None),
    (1, 128, 256, 6, 90, 1, (1, 2), None),
    (2, 256, 512, 9, 45, 1, (2, 2), None),
]
ODD_STEM = (2, 64, 64, 5, 181, 3, (1, 2), 8)     # the stem at an odd width: 8 real channels padded to 64
EPILOGUE_SHAPES = [(b, cin, cout, h, w, 3, (1, 1), None) for b, cin, cout, h, w in FPROP_BWD_SHAPES]

# (shape, act, residual)
FPROP_GAUSS_CASES = ([(s, a, False) for s in STRIDED_SHAPES for a in (1, 2)] + [(s, 0, False) for s in DOWNSAMPLE_SHAPES]
                     + [(ODD_STEM, 2, False)] + [(s, a, r) for s in EPILOGUE_SHAPES for a in (1, 2) for r in (False, True)])
FPROP_EXACT_CASES = ([(s, a, True) for s in STRIDED_SHAPES for a in (0, 1)] + [(s, 0, True) for s in DOWNSAMPLE_SHAPES]
                     + [(ODD_STEM, 1, False)] + [(s, a, True) for s in EPILOGUE_SHAPES for a in (0, 1)])

# the stem kernel: B, H, W of the image, Cin_true
STEM_SHAPES = [
    (2, 64, 2048, 8),       # the bench shape: 8 segments of 128 output pixels per row
    (1, 16, 180, 8),        # one ragged segment
    (1, 1, 10, 4),          # Cin_true = 4 (the weights of channels 4..7 are zero)
    (3, 5, 258, 8),         # 1-pixel second segment
]
# (act, out_f16): out_f16 = training's pre-activation, fp16 bit patterns in the bf16-typed buffer
STEM_GAUSS_MODES = [(0, False), (1, False), (2, False), (0, True)]
STEM_EXACT_MODES = [(0, False), (1, False), (0, True)]


def _id(case):
    (b, cin, cout, h, w, k, st, ct), act, res = case
    return f"{cin}x{cout}-k{k}-{h}x{w}-s{st[0]}{st[1]}-b{b}" + (f"-cin{ct}" if ct else "") + \
           f"-act{act}-{'res' if res else 'nores'}"


def _stem_id(case):
    (b, h, w, ct), (act, f16) = case
    return f"stem-{h}x{w}-b{b}-cin{ct}-act{act}" + ("-f16" if f16 else "")


def act_ref(pre, act):
    return torch.relu(pre) if act == 1 else torch.tanh(pre) if act == 2 else pre


def int_filter(g, shape, n, r):
    """Integer filter in [-r, r], dense enough for ~256 / r^2 nonzero products per output (|sum| well inside 256)."""
    return rand_int(g, shape, r, density=min(1.0, 256.0 / (n * r * r)))


def run_fprop(case, exact):
    from delora_b200 import ops
    (b, cin, cout, hin, win, k, stride, cin_true), act, use_res = case
    ct = cin if cin_true is None else cin_true
    hout, wout = ops.conv_out_size(hin, stride[0]), ops.conv_out_size(win, stride[1])
    n = k * k * ct
    g = generator("fprop", case, exact)
    if exact:
        x = rand_int(g, (b, cin, hin, win), 2)
        wt = int_filter(g, (cout, cin, k, k), n, 2)
        r = rand_int(g, (b, cout, hout, wout), 4) if use_res else None
    else:
        x = rand_bf16(g, (b, cin, hin, win))
        wt = rand_bf16(g, (cout, cin, k, k), n ** -0.5)
        r = rand_bf16(g, (b, cout, hout, wout)) if use_res else None
    wt[:, ct:] = 0.0                       # padded input channels (their x values are not zero) have zero weights
    pre = conv_ref(x, wt, stride) + (0.0 if r is None else r)
    ref = act_ref(pre, act)
    wn = wt.permute(0, 2, 3, 1).reshape(cout, k * k, cin).contiguous().to(torch.bfloat16)
    xp, rp = to_padded_nhwc(x), None if r is None else to_padded_nhwc(r)
    label = ("fprop exact " if exact else "fprop gauss ") + _id(case)

    def call():
        out = sentinel_out(b, hout, wout, cout)
        ops.conv2d_fprop(xp, wn, hin, win, k, stride, act, rp, out)
        check_layout(out, hout, wout, label)
        return out
    got = interior(run_twice(call, label), hout, wout)
    if exact:
        assert ref.abs().max().item() <= 256, f"{label}: |ref| exceeds 256, the output would round"
        check_exact(got, ref, label)
    else:
        ref_abs = conv_ref(x.abs(), wt.abs(), stride) + (0.0 if r is None else r.abs())
        extra = TANH_APPROX_REL_ERR * ref.abs() if act == 2 else None
        check_bound(got, ref, ref_abs, n, label, extra=extra)


@pytest.mark.parametrize("case", FPROP_GAUSS_CASES, ids=_id)
def test_fprop_gaussian(case, cuda_lib):
    """delora_conv2d_fprop_bf16 (forward act 0 / 1 / 2, optional residual) within the rounding bound of float64."""
    run_fprop(case, False)


@pytest.mark.parametrize("case", FPROP_EXACT_CASES, ids=_id)
def test_fprop_exact_on_integers(case, cuda_lib):
    """delora_conv2d_fprop_bf16 on integer operands (act 0 / 1) equals float64 bit for bit."""
    run_fprop(case, True)


def run_stem(case, exact):
    from delora_b200 import ops
    (b, h, w, ct), (act, f16) = case
    wout = w // 2
    g = generator("stem fprop", case, exact)
    if exact:
        # fp16 output (exact to 2048): wider operands, so that outputs above 256 occur
        rx, rw = (8, 3) if f16 else (2, 1)
        x = rand_int(g, (b, 16, h, w), rx)
        wt = rand_int(g, (64, ct, 3, 3), rw)
    else:
        x = torch.cat([rand_bf16(g, (b, 8, h, w)), rand_bf16(g, (b, 8, h, w), 2.0 ** -8)], dim=1)
        wt = rand_bf16(g, (64, ct, 3, 3), (9 * ct) ** -0.5)
    # channels ct .. 7 and 8 + ct .. 15 hold nonzero values: the stem's weights are zero there
    pre = conv3(x[:, :ct] + x[:, 8:8 + ct], wt, (1, 2))
    ref = act_ref(pre, act)
    w_stem = ops.stem_weight_prep(wt.float(), torch.empty((3, 64, 64), dtype=torch.bfloat16, device=DEV))
    xp = to_padded_nhwc(x)
    label = ("stem exact " if exact else "stem gauss ") + _stem_id(case)

    def call():
        out = sentinel_out(b, h, wout, 64)
        ops.stem_fprop(xp, w_stem, h, w, act, out=out, out_f16=f16)
        check_layout(out, h, wout, label)
        return out
    out = run_twice(call, label)
    got = interior(out.view(torch.float16) if f16 else out, h, wout)
    if exact:
        lim = 2048 if f16 else 256
        assert ref.abs().max().item() <= lim, f"{label}: |ref| exceeds {lim}, the output would round"
        check_exact(got, ref, label)
    else:
        ref_abs = conv3(x[:, :ct].abs() + x[:, 8:8 + ct].abs(), wt.abs(), (1, 2))
        extra = TANH_APPROX_REL_ERR * ref.abs() if act == 2 else None
        # n = 192: the GEMM's K (3 filter rows x 4 pixels x 16 channels, the zero-weight products included)
        check_bound(got, ref, ref_abs, 192, label, out_unit=2.0 ** -11 if f16 else 2.0 ** -8, extra=extra)


@pytest.mark.parametrize("case", [(s, m) for s in STEM_SHAPES for m in STEM_GAUSS_MODES], ids=_stem_id)
def test_stem_fprop_gaussian(case, cuda_lib):
    """delora_stem_fprop_bf16 (act 0 / 1 / 2, bf16 or fp16 output) within the rounding bound of float64."""
    run_stem(case, False)


@pytest.mark.parametrize("case", [(s, m) for s in STEM_SHAPES for m in STEM_EXACT_MODES], ids=_stem_id)
def test_stem_fprop_exact_on_integers(case, cuda_lib):
    """delora_stem_fprop_bf16 on integer operands (act 0 / 1, bf16 or fp16 output) equals float64 bit for bit."""
    run_stem(case, True)
