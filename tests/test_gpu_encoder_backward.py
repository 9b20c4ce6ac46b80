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
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
HALO_ROW = 7.0          # the halo rows of an output are never written: they must still hold this after the call


def to_padded_nhwc(x):
    """[B,C,H,W] -> [B,H+2,W+2,C] bf16 with the circular W halo and the zero H halo of the encoder's layout."""
    xp = F.pad(F.pad(x, (1, 1, 0, 0), mode="circular"), (0, 0, 1, 1))
    return xp.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def interior(y, h, w):
    """padded NHWC -> [B,C,H,W] float64"""
    return y[:, 1:h + 1, 1:w + 1].permute(0, 3, 1, 2).double()


def rand_bf16(g, shape, scale=1.0):
    """float64 tensor holding bf16 values: the exact operand the kernel reads."""
    return (torch.randn(shape, generator=g, device=DEV, dtype=torch.float64) * scale).to(torch.bfloat16).double()


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


def conv3(x, w, stride):
    """The encoder's 3x3 convolution: circular padding in W, zero padding in H (src/models/resnet_modified.py)."""
    return F.conv2d(F.pad(x, (1, 1, 0, 0), mode="circular"), w, stride=stride, padding=(1, 0))


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


def check_bound(got, ref, ref_abs, n, label):
    assert bool(torch.isfinite(got).all()), f"{label}: non-finite output"
    bound = 2.0 ** -8 * ref.abs() + (n + 3) * 2.0 ** -24 * ref_abs
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    worst = ratio.max().item()
    print(f"{label}: worst err/bound {worst:.4f}", flush=True)
    if worst > 1.0:
        b, c, h, w = (int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape))
        bad = ratio > 1.0
        raise AssertionError(
            f"{label}: err/bound {worst:.3g} at (b, c, h, w) = ({b}, {c}, {h}, {w}): got {got[b, c, h, w].item():.6g}, "
            f"ref {ref[b, c, h, w].item():.6g}; {int(bad.sum())} elements over the bar, rows "
            f"{sorted(set(bad.nonzero()[:, 2].tolist()))[:16]}, columns {sorted(set(bad.nonzero()[:, 3].tolist()))[:16]}")


def sentinel_out(b, h, w, c):
    """Padded NHWC output: bf16 NaN in rows 1..H (interior and halo columns), HALO_ROW in rows 0 and H+1."""
    out = torch.full((b, h + 2, w + 2, c), float("nan"), dtype=torch.bfloat16, device=DEV)
    out[:, 0] = HALO_ROW
    out[:, h + 1] = HALO_ROW
    return out


def check_layout(out, h, w, label):
    """Every pixel of rows 1..H written, columns 0 / W+1 the circular copies of columns W / 1, halo rows untouched."""
    rows = out[:, 1:h + 1]
    nan = torch.isnan(rows)
    assert not bool(nan.any()), f"{label}: {int(nan.sum())} elements not written, first (b, h-1, w, c) = " \
                                f"{tuple(nan.nonzero()[0].tolist())}"
    bits = rows.view(torch.int16)
    assert torch.equal(bits[:, :, 0], bits[:, :, w]), f"{label}: halo column 0 differs from column W"
    assert torch.equal(bits[:, :, w + 1], bits[:, :, 1]), f"{label}: halo column W+1 differs from column 1"
    assert bool((out[:, 0] == HALO_ROW).all()) and bool((out[:, h + 1] == HALO_ROW).all()), f"{label}: halo row written"


def run_twice(fn, label):
    """Two calls into fresh sentinel outputs: both pass the layout checks and agree bit for bit."""
    a, b = fn(), fn()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{label}: two calls differ"
    return a


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
FPROP_BWD_SHAPES = [   # B, Cin, Cout, H, W at stride 1 (the backward's dz1 = conv(dz2) * act'(t1) and its residual form)
    (2, 512, 512, 4, 64),      # conv_rows, 128 output channels on M
    (2, 64, 64, 5, 180),       # conv_rows pixel-on-M, ragged second segment
    (2, 128, 128, 4, 256),     # conv_rows pixel-on-M
    (2, 64, 64, 5, 45),        # conv_tc (64 output channels on a row narrower than a segment)
]
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
