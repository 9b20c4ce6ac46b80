"""-m "not gpu": the encoder-trunk entry points of the C ABI without a device -- the weight-section and activation
workspace sizes against the shapes of ResNetModified, stages of up to 64 blocks, and the refusal of bad arguments by
name (every check runs before the first launch)."""
import ctypes

import pytest


def _L():
    from delora_b200 import _lib
    return _lib.lib()


def _layers(*n):
    return (ctypes.c_int * 4)(*n)


def _a256(n):
    return (n + 255) // 256 * 256


def _nhwc(b, h, w, c):
    return b * (h + 2) * (w + 2) * c * 2


def _out(n, s):
    return (n - 1) // s + 1


def _convs(layers):
    """(cout, cin, k) of every filter in state_dict order (src/models/resnet_modified.py:49-66)."""
    convs, inplanes = [(64, 8, 3)], 64
    for s, (planes, n) in enumerate(zip((64, 128, 256, 512), layers)):
        for bi in range(n):
            convs += [(planes, inplanes, 3), (planes, planes, 3)]
            if bi == 0 and (s > 0 or inplanes != planes):
                convs.append((planes, inplanes, 1))
            inplanes = planes
    return convs


@pytest.mark.parametrize("layers", [(2, 2, 2, 2), (1, 2, 1, 1), (1, 1, 17, 1)])
@pytest.mark.parametrize("w", [2048, 2047, 720, 259])
def test_weight_bytes_match_the_filter_shapes(layers, w):
    convs = _convs(layers)
    want = _a256(len(convs) * 64)                                             # the prep table
    want += _a256(3 * 64 * 64 * 2 if w % 2 == 0 else 64 * 9 * 64 * 2)         # the stem: 16- or 64-channel layout
    for cout, cin, k in convs[1:]:
        want += 2 * _a256(cout * cin * k * k * 2)                             # forward and flipped copies
    assert _L().delora_trunk_weight_bytes(_layers(*layers), w) == want


@pytest.mark.parametrize("layers", [(2, 2, 2, 2), (1, 2, 1, 1), (1, 1, 17, 1)])
@pytest.mark.parametrize("b,h,w", [(1, 64, 2048), (16, 64, 2048), (4, 64, 720), (2, 16, 259)])
def test_inference_activation_bytes_match_the_stage_shapes(layers, b, h, w):
    w2 = _out(w, 2)
    want = _a256(_nhwc(b, h, w, 16 if w % 2 == 0 else 64)) + _a256(_nhwc(b, h, w2, 64))
    sh, sw = h, w2 // 2
    for c, (st_h, st_w) in zip((64, 128, 256, 512), ((1, 1), (1, 2), (1, 2), (2, 2))):
        sh, sw = _out(sh, st_h), _out(sw, st_w)
        want += 3 * _a256(_nhwc(b, sh, sw, c))                                # three rotating buffers per stage
    L = _L()
    assert L.delora_trunk_activation_bytes(_layers(*layers), b, h, w, 0) == want
    saving = L.delora_trunk_activation_bytes(_layers(*layers), b, h, w, 1)
    assert saving > want and saving % 256 == 0


def test_stage_limits():
    L = _L()
    assert L.delora_trunk_activation_bytes(_layers(1, 1, 64, 1), 1, 16, 256, 1) > 0
    assert L.delora_trunk_activation_bytes(_layers(1, 1, 65, 1), 1, 16, 256, 1) == -1
    assert b"layers[2]=65" in L.delora_last_error()


def _last(L):
    return L.delora_last_error()


def test_size_queries_refuse_bad_arguments_by_name():
    L = _L()
    ok = _layers(2, 2, 2, 2)
    cases = [(lambda: L.delora_trunk_weight_bytes(None, 2048), b"null layers"),
             (lambda: L.delora_trunk_weight_bytes(_layers(2, 2, 0, 2), 2048), b"layers[2]=0"),
             (lambda: L.delora_trunk_weight_bytes(ok, 718), b"W=718"),
             (lambda: L.delora_trunk_activation_bytes(ok, 1, 0, 2048, 0), b"bad image size"),
             (lambda: L.delora_trunk_activation_bytes(ok, 0, 64, 2048, 0), b"B=0"),
             (lambda: L.delora_trunk_activation_bytes(ok, 1, 64, 2048, 2), b"saving=2")]
    for call, msg in cases:
        assert call() == -1
        err = _last(L)
        assert msg in err and err.startswith(b"delora_trunk_"), err


def test_launches_refuse_bad_arguments_by_name():
    L = _L()
    ok = _layers(1, 1, 1, 1)
    p = ctypes.c_void_p(256)                      # never dereferenced: every case fails a check before any launch
    n_conv = len(_convs((1, 1, 1, 1)))
    dw = (ctypes.c_void_p * n_conv)(*([256] * n_conv))
    dw_hole = (ctypes.c_void_p * n_conv)(*([256] * n_conv))
    dw_hole[0] = None
    filters_hole = (ctypes.c_void_p * n_conv)(*([256] * (n_conv - 1) + [0]))
    cases = [
        (lambda: L.delora_trunk_prep_weights(ok, 2048, None, p, None), b"null filters"),
        (lambda: L.delora_trunk_prep_weights(ok, 2048, filters_hole, p, None), b"null filters[%d]" % (n_conv - 1)),
        (lambda: L.delora_trunk_prep_weights(ok, 2048, dw, None, None), b"null weights"),
        (lambda: L.delora_trunk_forward(ok, 1, 64, 2048, 3, 0, p, p, p, p, p, None, None), b"act=3"),
        (lambda: L.delora_trunk_forward(ok, 1, 64, 2048, 1, 2, p, p, p, p, p, None, None), b"saving=2"),
        (lambda: L.delora_trunk_forward(ok, 1, 64, 2048, 1, 0, None, p, p, p, p, None, None), b"null img1"),
        (lambda: L.delora_trunk_forward(ok, 1, 64, 2048, 1, 0, p, p, p, None, p, None, None), b"null acts"),
        (lambda: L.delora_trunk_forward(ok, 1, 64, 2048, 1, 0, p, p, p, p, None, None, None), b"null pooled"),
        (lambda: L.delora_trunk_forward(ok, 1, 64, 718, 1, 0, p, p, p, p, p, None, None), b"W=718"),
        (lambda: L.delora_trunk_backward(ok, 1, 64, 2048, 1, p, p, p, dw, 4, None), b"stage=4"),
        (lambda: L.delora_trunk_backward(ok, 1, 64, 2048, 1, p, p, None, dw, 3, None), b"null g_pooled"),
        (lambda: L.delora_trunk_backward(ok, 1, 64, 2048, 1, p, p, p, None, 3, None), b"null conv_dw"),
        (lambda: L.delora_trunk_backward(ok, 1, 64, 2048, 1, p, p, p, dw_hole, 0, None), b"conv_dw[0]"),
        (lambda: L.delora_trunk_backward(ok, 1, 64, 2048, 1, None, p, p, dw, 3, None), b"null weights"),
        (lambda: L.delora_trunk_backward(ok, 0, 64, 2048, 1, p, p, p, dw, 3, None), b"B=0"),
        # the dropout variants: the same checks under their own name, and a counter only with saving = 1
        (lambda: L.delora_trunk_forward_dropout(ok, 1, 64, 2048, 1, 0, p, p, p, p, p, None, p, None),
         b"delora_trunk_forward_dropout: dropout_ctr needs saving=1"),
        (lambda: L.delora_trunk_forward_dropout(ok, 1, 64, 2047, 1, 0, p, p, p, p, p, None, p, None),
         b"delora_trunk_forward_dropout: dropout_ctr needs saving=1"),
        (lambda: L.delora_trunk_forward_dropout(ok, 1, 64, 2048, 3, 1, p, p, p, p, p, None, p, None),
         b"delora_trunk_forward_dropout: act=3"),
        (lambda: L.delora_trunk_forward_dropout(ok, 1, 64, 2048, 1, 1, p, None, p, p, p, None, p, None),
         b"delora_trunk_forward_dropout: null img2"),
        (lambda: L.delora_trunk_forward_dropout(ok, 1, 64, 2048, 1, 0, p, p, p, p, None, None, None, None),
         b"delora_trunk_forward: null pooled"),                    # no counter: the plain call
        (lambda: L.delora_trunk_backward_dropout(ok, 1, 64, 2048, 1, p, p, p, dw, -1, p, None),
         b"delora_trunk_backward_dropout: stage=-1"),
        (lambda: L.delora_trunk_backward_dropout(ok, 1, 64, 2048, 1, p, p, None, dw, 3, p, None),
         b"delora_trunk_backward_dropout: null g_pooled"),
        (lambda: L.delora_trunk_backward_dropout(ok, 1, 64, 2048, 1, p, p, p, dw_hole, 0, p, None),
         b"delora_trunk_backward_dropout: null conv_dw[0]"),
    ]
    for call, msg in cases:
        assert call() != 0
        err = _last(L)
        assert msg in err and err.startswith(b"delora_trunk_"), err
