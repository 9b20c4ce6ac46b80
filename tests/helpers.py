"""Shared helpers for the parity tests and the encoder's per-layer kernel tests (test infrastructure; may import
oracle/)."""
import hashlib
import os
import zlib

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def digest(t):
    a = t.detach().cpu().contiguous().numpy() if isinstance(t, torch.Tensor) else np.ascontiguousarray(t)
    return hashlib.sha256(a.tobytes()).hexdigest()


def unsort_uv(cloud, u_sorted, v_sorted):
    """Oracle (u, v) come in stable range order; scatter them back to the original point order."""
    rng = torch.norm(cloud[None][:, :3, :], dim=1)
    order = torch.argsort(rng, dim=1, stable=True)[0]
    u = torch.empty_like(u_sorted)
    v = torch.empty_like(v_sorted)
    u[order] = u_sorted
    v[order] = v_sorted
    return u, v, rng[0]


def case_inputs(meta):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=meta["H"], w=meta["W"], vfov_deg=tuple(meta["vfov_deg"]))
    pair = synthetic.make_pair(meta["pair_index"], w_raw=meta["w_raw"], rings=meta["rings"],
                               vfov_deg=tuple(meta["vfov_deg"]))
    return cfg, pair


# ------------------------------------------------------------------------------------------------ encoder kernels
# The convolution kernels read and write padded NHWC bf16 maps [B, H+2, W+2, C]: circular halo columns, zero halo rows.
DEV = "cuda"
HALO_ROW = 7.0          # the halo rows of an output are never written: they must still hold this after the call

FPROP_BWD_SHAPES = [   # B, Cin, Cout, H, W at stride 1 (the backward's dz1 = conv(dz2) * act'(t1) and its residual form)
    (2, 512, 512, 4, 64),      # conv_rows, 128 output channels on M
    (2, 64, 64, 5, 180),       # conv_rows pixel-on-M, ragged second segment
    (2, 128, 128, 4, 256),     # conv_rows pixel-on-M
    (2, 64, 64, 5, 45),        # conv_tc (64 output channels on a row narrower than a segment)
]


def generator(*key):
    """A CUDA generator seeded from the case's parameters (stable across processes, unlike hash())."""
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


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


def rand_int(g, shape, r, density=1.0):
    """float64 tensor of integers uniform in [-r, r] (exact in bf16 for r <= 256), each kept with probability
    `density` and zero otherwise."""
    v = torch.randint(-r, r + 1, shape, generator=g, device=DEV, dtype=torch.int64).double()
    if density < 1.0:
        v = v * (torch.rand(shape, generator=g, device=DEV) < density).double()
    return v


def conv3(x, w, stride):
    """The encoder's 3x3 convolution: circular padding in W, zero padding in H (src/models/resnet_modified.py)."""
    return F.conv2d(F.pad(x, (1, 1, 0, 0), mode="circular"), w, stride=stride, padding=(1, 0))


def conv_ref(x, w, stride):
    """The encoder's 3x3 (conv3) or 1x1 (no padding) convolution, by the filter's size."""
    return conv3(x, w, stride) if w.shape[-1] == 3 else F.conv2d(x, w, stride=stride)


def check_bound(got, ref, ref_abs, n, label, out_unit=2.0 ** -8, acc_unit=2.0 ** -24, extra=None):
    """|got - ref| <= out_unit |ref| + (n + 3) acc_unit ref_abs (+ extra), element by element: one output rounding
    (out_unit 2^-8 for bf16, 2^-11 for fp16, 0 for an fp32 output) plus a worst-case bound on an accumulation of n
    products in fp32 (acc_unit 2^-24 for round-to-nearest adds, 2^-23 for adders that may truncate); `extra` is a
    further per-element term (e.g. an approximate activation's error).  Prints and returns the worst err / bound."""
    assert bool(torch.isfinite(got).all()), f"{label}: non-finite output"
    bound = out_unit * ref.abs() + (n + 3) * acc_unit * ref_abs
    if extra is not None:
        bound = bound + extra
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    worst = ratio.max().item()
    print(f"{label}: worst err/bound {worst:.4f}", flush=True)
    if worst > 1.0:
        idx = tuple(int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape))
        bad = ratio > 1.0
        raise AssertionError(
            f"{label}: err/bound {worst:.3g} at {idx}: got {got[idx].item():.6g}, ref {ref[idx].item():.6g}; "
            f"{int(bad.sum())} elements over the bar, dim-2 indices {sorted(set(bad.nonzero()[:, 2].tolist()))[:16]}, "
            f"dim-3 indices {sorted(set(bad.nonzero()[:, 3].tolist()))[:16]}")
    return worst


def check_exact(got, ref, label):
    """got == ref bit for bit (4-d tensors): on a mismatch, report the first differing element with the 3 x 3
    neighbourhood of its last two dimensions in both tensors."""
    diff = ~(got == ref)
    nd = int(diff.sum())
    print(f"{label}: {nd} differing elements", flush=True)
    if nd:
        i0, i1, i2, i3 = (int(i) for i in diff.nonzero()[0])
        s2, s3 = slice(max(i2 - 1, 0), i2 + 2), slice(max(i3 - 1, 0), i3 + 2)
        raise AssertionError(
            f"{label}: {nd} of {got.numel()} elements differ; first at {(i0, i1, i2, i3)}: got {got[i0, i1, i2, i3].item()}, "
            f"ref {ref[i0, i1, i2, i3].item()}; neighbours from ({s2.start}, {s3.start}):\n got {got[i0, i1, s2, s3].tolist()}"
            f"\n ref {ref[i0, i1, s2, s3].tolist()}")


def sentinel_out(b, h, w, c):
    """Padded NHWC output: bf16 NaN in rows 1..H (interior and halo columns), HALO_ROW in rows 0 and H+1."""
    out = torch.full((b, h + 2, w + 2, c), float("nan"), dtype=torch.bfloat16, device=DEV)
    out[:, 0] = HALO_ROW
    out[:, h + 1] = HALO_ROW
    return out


def check_layout(out, h, w, label):
    """Every pixel of rows 1..H written, columns 0 / W+1 the circular copies of columns W / 1, halo rows untouched.
    (Also right for an output holding fp16 bit patterns: no finite fp16 reads as a bf16 NaN.)"""
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
