"""CPU tests of the ResNet batch and canvas entries (include/frcnn_b200.h): NULL extents, a bad image count, a bad halving
count or a bad canvas is rejected with FRCNN_ERR_ARG and a message before anything touches the device; the per-level
extent rule is the one ResNetForwardPlan sizes its maps by; and the ResNet batch plans refuse the options they do not
support before they allocate anything."""
import ctypes

import pytest

from frcnn_b200._lib import FrcnnError


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


P = ctypes.c_void_p(256)            # never dereferenced: every call below fails its argument checks first


def _arg_error(status, words):
    from frcnn_b200 import _lib
    msg = _lib.last_error()
    return status == _lib.ERR_ARG and all(w in msg for w in words)


def test_first_layer_and_pool_entries(lib):
    assert _arg_error(lib.frcnn_pack_image_im2col_batch_ext(P, 2, 3, 64, 96, 7, 2, 3, 160, None, P, None, None), ["extents"])
    assert _arg_error(lib.frcnn_pack_image_im2col_batch_ext(P, 0, 3, 64, 96, 7, 2, 3, 160, P, P, None, None), ["N in"])
    assert _arg_error(lib.frcnn_pack_image_im2col_batch(P, 0, 3, 64, 96, 7, 2, 3, 160, P, None, None), ["N must be"])
    assert _arg_error(lib.frcnn_pack_image_im2col_batch(P, 2, 3, 64, 96, 7, 2, 3, 144, P, None, None), ["K_pad"])
    assert _arg_error(lib.frcnn_maxpool3x3s2_ceil_batch_ext(P, None, 2, 32, 48, 64, None, P, None, None), ["extents"])
    assert _arg_error(lib.frcnn_maxpool3x3s2_ceil_batch_ext(P, None, 0, 32, 48, 64, P, P, None, None), ["N in"])
    assert _arg_error(lib.frcnn_maxpool3x3s2_ceil_batch(P, None, 0, 32, 48, 64, P, None, None), ["N must be"])
    assert _arg_error(lib.frcnn_maxpool3x3s2_ceil_batch(P, None, 2, 2, 48, 64, P, None, None), ["H=2"])
    assert _arg_error(lib.frcnn_subsample2x_batch(P, None, 0, 32, 48, 64, P, None, None), ["N must be"])
    assert _arg_error(lib.frcnn_subsample2x_batch(P, None, 70000, 32, 48, 64, P, None, None), ["N must be"])


def test_residual_conv_entries(lib):
    assert _arg_error(lib.frcnn_conv2d_res_batch(P, None, 0, 8, 8, 64, P, None, P, 256, 1, 1, P, None, P, None, None), ["N must be"])
    assert _arg_error(lib.frcnn_conv2d_res_batch_ext(P, None, 2, 8, 8, 64, P, None, P, 256, 1, 1, P, None, P, None, None, 0, None),
                      ["extents"])
    assert _arg_error(lib.frcnn_conv2d_res_batch_ext(P, None, 0, 8, 8, 64, P, None, P, 256, 1, 1, P, None, P, None, P, 0, None),
                      ["N >= 1"])
    for bad in (-1, 31):
        assert _arg_error(lib.frcnn_conv2d_res_batch_ext(P, None, 2, 8, 8, 64, P, None, P, 256, 3, 1, P, None, P, None, P, bad, None),
                          ["halvings"])


def test_level_extents_entry(lib):
    assert _arg_error(lib.frcnn_resnet_level_extents(None, 2, 64, 96, P, None), ["NULL"])
    assert _arg_error(lib.frcnn_resnet_level_extents(P, 2, 64, 96, None, None), ["NULL"])
    for n, hc, wc in ((0, 64, 96), (65536, 64, 96), (2, 0, 96), (2, 64, -1)):
        assert _arg_error(lib.frcnn_resnet_level_extents(P, n, hc, wc, P, None), ["bad shape"])


def _levels(e):
    """The per-level rule of include/frcnn_b200.h (frcnn_resnet_level_extents), in Python's floor division."""
    c = (e - 1) // 2 + 1
    p = (c - 2) // 2 + 1 if c >= 2 else 0
    out = [c, p]
    for _ in range(3):
        out.append((out[-1] + 1) // 2)
    return out


class _SizeRecorder(object):
    """Stands in for a plan: ResNetForwardPlan._alloc_trunk run on it allocates (h, w, c) tuples instead of planes."""

    def __init__(self, n_layers):
        self.w = type("W", (), {"n_layers": n_layers})()

    def _act(self, h, w, c):
        return (h, w, c)


def test_level_rule_is_the_forward_plan_sizes():
    """For every h, w in 1..200: conv1, pool1, res3, res4 and res5 of ResNetForwardPlan._alloc_trunk are the level rule."""
    from frcnn_b200.resnet_engine import ResNetForwardPlan
    want = [_levels(e) for e in range(201)]
    assert want[0] == [0, 0, 0, 0, 0] and want[1] == [1, 0, 0, 0, 0] and want[3] == [2, 1, 1, 1, 1] and want[5] == [3, 1, 1, 1, 1]
    for h in range(1, 201):
        for w in range(1, 201):
            r = _SizeRecorder(50)
            feat = ResNetForwardPlan._alloc_trunk(r, h, w)
            stage_out = {B["name"].split("/")[0]: B["out"] for B in r.blocks}
            got = [r.x_col, r.p1, stage_out["res3"], stage_out["res4"], stage_out["res5"]]
            assert [g[:2] for g in got] == list(zip(want[h], want[w])) and feat == got[-1][:2], (h, w)


class _Weights(object):
    device, precision = "cpu", "bf16"
    convs = {"conv1": None}


@pytest.mark.parametrize("opt", ["raw_input", "hwc_input", "keep_rpn_debug"])
def test_resnet_batch_plans_refuse_options_up_front(opt):
    from frcnn_b200.resnet_engine import ResNetBatchPlan, ResNetCanvasBatchPlan
    for cls in (ResNetBatchPlan, ResNetCanvasBatchPlan):
        with pytest.raises(FrcnnError, match=opt):
            cls(_Weights(), 2, 64, 96, anchors=None, **{opt: True})


def test_resnet_batch_engine_plans():
    """ResNetBatchEngine builds ResNetBatchPlan / ResNetCanvasBatchPlan (cached per shape and options, with the engine's
    options and feat_stride 32); ResNetEngine keeps refusing batches."""
    from frcnn_b200 import resnet_engine as re_
    made = []

    class Eng(re_.ResNetBatchEngine):
        def _pack_weights(self, *args):
            return ("weights",) + args

        def _cached(self, kind, cls, shape, overrides):
            made.append((kind, cls, shape))
            return super(Eng, self)._cached(kind, lambda *a, **kw: (cls, a, kw), shape, overrides)

    eng = Eng({}, 50, anchors="A", post_n=100)
    b = eng.batch_plan(2, 64, 96)
    c = eng.canvas_plan(4, 192, 256, with_detect=True)
    assert made == [("batch", re_.ResNetBatchPlan, (2, 64, 96)), ("canvas", re_.ResNetCanvasBatchPlan, (4, 192, 256))]
    assert b[1:] == ((eng.weights, 2, 64, 96), dict(anchors="A", feat_stride=32, post_n=100))
    assert c[1:] == ((eng.weights, 4, 192, 256), dict(anchors="A", feat_stride=32, post_n=100, with_detect=True))
    assert eng.batch_plan(2, 64, 96) is b and len(eng.plans) == 2
    assert issubclass(re_.ResNetCanvasBatchPlan, re_.ResNetBatchPlan)

    class One(re_.ResNetEngine):
        def _pack_weights(self, *args):
            return None

    with pytest.raises(FrcnnError, match="ResNetBatchEngine"):
        One({}, 50, anchors="A").canvas_plan(2, 64, 96)
