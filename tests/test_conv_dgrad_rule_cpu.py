"""-m "not gpu": delora_conv2d_dgrad_eligible, the one statement of which layers the phase-decomposed data gradient
(delora_conv2d_dgrad_bf16) takes.  The Python trunk and the odometry training plan both route by it, and the training
plan sizes its workspace from it."""
import pytest

# Cin, Cout, Win, (stride_h, stride_w) of the forward 3x3 convolution -> eligible
TRUNK = {  # the strided blocks (stages 2-4) of the encoder at image widths 2048, 720, 512, 2047 and 180
    2048: [((64, 128, 512, (1, 2)), 1), ((128, 256, 256, (1, 2)), 1), ((256, 512, 128, (2, 2)), 1)],
    720: [((64, 128, 180, (1, 2)), 0), ((128, 256, 90, (1, 2)), 1), ((256, 512, 45, (2, 2)), 0)],
    512: [((64, 128, 128, (1, 2)), 0), ((128, 256, 64, (1, 2)), 1), ((256, 512, 32, (2, 2)), 1)],
    2047: [((64, 128, 512, (1, 2)), 1), ((128, 256, 256, (1, 2)), 1), ((256, 512, 128, (2, 2)), 1)],
    180: [((64, 128, 45, (1, 2)), 0), ((128, 256, 23, (1, 2)), 0), ((256, 512, 12, (2, 2)), 1)],
}
OFF_TRUNK = [
    ((64, 128, 254, (1, 2)), 0),      # Cin = 64: 127 columns per phase
    ((64, 128, 256, (1, 2)), 1),      # Cin = 64: 128 columns per phase
    ((64, 64, 200, (1, 1)), 1),
    ((64, 64, 100, (1, 1)), 0),
    ((128, 256, 91, (1, 2)), 0),      # odd Win at stride_w = 2
    ((256, 512, 45, (2, 2)), 0),
    ((128, 96, 256, (1, 2)), 0),      # Cout not a multiple of 64
    ((128, 32, 256, (1, 1)), 0),
    ((192, 256, 256, (1, 2)), 0),     # Cin neither 64 nor a multiple of 128
    ((128, 128, 7, (1, 1)), 1),
    ((128, 256, 256, (1, 3)), 0),     # strides outside {1, 2}
    ((128, 256, 256, (3, 1)), 0),
]
CASES = [c for w in TRUNK for c in TRUNK[w]] + OFF_TRUNK


@pytest.fixture(scope="module")
def lib():
    from delora_b200 import _lib, build
    build.build()
    return _lib.lib()


@pytest.mark.parametrize("shape,expected", CASES)
def test_dgrad_eligible(shape, expected, lib):
    from delora_b200 import ops
    cin, cout, win, (sh, sw) = shape
    assert lib.delora_conv2d_dgrad_eligible(cin, cout, win, sh, sw) == expected
    assert ops.conv2d_dgrad_eligible(cin, cout, win, (sh, sw)) == bool(expected)
    if not expected:
        # the entry point refuses the layer in its argument check, before anything reaches the device
        dummy = 256
        rc = lib.delora_conv2d_dgrad_bf16(dummy, dummy, None, None, dummy, 1, 16, win, cin, cout, sh, sw, 0, 0, None)
        assert rc != 0
        assert b"delora_conv2d_dgrad_eligible" in lib.delora_last_error()
