"""CPU tests of the ResNet raw-photo canvas: frcnn_preprocess_bgr8_canvas_im2col is exported with the declared signature and
rejects every bad argument with FRCNN_ERR_ARG and a message naming it before anything touches the device; ResNetPhotoEngine
builds a ResNetRawCanvasBatchPlan for raw photos under its own cache key; and the float-input ResNet plans and engines keep
refusing raw photos."""
import ctypes
import os
import re

import numpy as np
import pytest

from frcnn_b200._lib import FrcnnError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p(256)            # never dereferenced: every call below fails its argument checks first
MEANS = (102.9801, 115.9465, 122.7717)
FN = "frcnn_preprocess_bgr8_canvas_im2col"


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def _call(lib, arena=P, arena_bytes=1 << 20, src_off=P, src_hw=P, inv_scale=P, extents=P, N=2, Hc=64, Wc=96, ksize=7, stride=2,
          pad=3, K_pad=160, y_hi=P):
    return getattr(lib, FN)(arena, arena_bytes, src_off, src_hw, inv_scale, extents, N, Hc, Wc, *MEANS, ksize, stride, pad, K_pad,
                            y_hi, None, None)


def test_symbol_and_declared_signature(lib):
    from frcnn_b200 import _lib
    res, args = _lib.SIGNATURES[FN]
    assert res is ctypes.c_int and len(args) == 19 and args[1] is ctypes.c_longlong and args[9:12] == [ctypes.c_double] * 3
    assert args[12:16] == [ctypes.c_int] * 4 and getattr(lib, FN).argtypes == args
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "frcnn_b200.h")).read(), flags=re.S)
    decl = re.search(r"int %s\((.*?)\);" % FN, hdr, flags=re.S).group(1)
    params = [" ".join(p.split()) for p in decl.split(",")]
    assert params == ["const unsigned char* arena", "long long arena_bytes", "const long long* src_off", "const int* src_hw",
                      "const double* inv_scale", "const int* extents", "int N", "int Hc", "int Wc", "double mean_b",
                      "double mean_g", "double mean_r", "int ksize", "int stride", "int pad", "int K_pad", "void* y_hi",
                      "void* y_lo", "void* stream"]


@pytest.mark.parametrize("bad,words", [
    (dict(arena=None), ["arena is NULL"]), (dict(arena_bytes=0), ["arena_bytes", "0"]), (dict(arena_bytes=-5), ["arena_bytes", "-5"]),
    (dict(src_off=None), ["src_off"]), (dict(src_hw=None), ["src_hw"]), (dict(inv_scale=None), ["inv_scale"]),
    (dict(extents=None), ["extents"]), (dict(y_hi=None), ["y_hi"]), (dict(N=0), ["N=0"]), (dict(N=65536), ["N=65536"]),
    (dict(Hc=0), ["Hc=0"]), (dict(Wc=-3), ["Wc=-3"]), (dict(ksize=0), ["ksize=0"]), (dict(ksize=46), ["ksize=46"]),
    (dict(stride=0), ["stride=0"]), (dict(pad=-1), ["pad=-1"]), (dict(pad=1 << 29), ["pad=536870912"]),
    (dict(K_pad=144), ["K_pad=144", "147"]), (dict(K_pad=164), ["K_pad=164"]), (dict(K_pad=65544), ["K_pad=65544"]),
    (dict(Hc=4, Wc=4, pad=0), ["smaller than the filter"])])
def test_argument_errors_name_the_argument(lib, bad, words):
    from frcnn_b200 import _lib
    assert _call(lib, **bad) == _lib.ERR_ARG
    msg = _lib.last_error()
    assert msg.startswith(FN) and all(w in msg for w in words), msg


class _Weights(object):
    device, precision = "cpu", "bf16"
    convs = {"conv1": None}


def test_old_plans_and_engines_still_refuse_raw_photos():
    """The float-input ResNet plans refuse raw_input=True (the message names the plan that takes raw photos);
    ResNetBatchEngine.raw_canvas_plan / detect_images raise before anything is allocated; the raw plan takes nothing else."""
    from frcnn_b200 import resnet_engine as re_
    for cls in (re_.ResNetBatchPlan, re_.ResNetCanvasBatchPlan):
        with pytest.raises(FrcnnError, match="raw_input=True .*ResNetRawCanvasBatchPlan"):
            cls(_Weights(), 2, 64, 96, anchors=None, raw_input=True)
    for opt in ("hwc_input", "keep_rpn_debug"):
        with pytest.raises(FrcnnError, match=opt):
            re_.ResNetRawCanvasBatchPlan(_Weights(), 2, 64, 96, anchors=None, **{opt: True})
    with pytest.raises(FrcnnError, match="raw_input=False"):
        re_.ResNetRawCanvasBatchPlan(_Weights(), 2, 64, 96, anchors=None, raw_input=False)

    class Batch(re_.ResNetBatchEngine):
        def _pack_weights(self, *args):
            return _Weights()

    photos = [np.zeros((120, 160, 3), np.uint8)]
    eng = Batch({}, 50, anchors="A")
    for call in (eng.raw_canvas_plan, eng.detect_images):
        with pytest.raises(FrcnnError, match="raw_input"):
            call(photos)
    assert eng.plans == {}


def test_photo_engine_plans():
    """ResNetPhotoEngine: canvas_plan(raw_input=True) is a ResNetRawCanvasBatchPlan under the key "raw_canvas" (with the
    engine's options and feat_stride 32); without raw_input it is ResNetBatchEngine's; raw_canvas_plan sizes the canvas and
    the arena as the VGG16 engine does."""
    from frcnn_b200 import resnet_engine as re_
    made = []

    class Eng(re_.ResNetPhotoEngine):
        def _pack_weights(self, *args):
            return ("weights",) + args

        def _cached(self, kind, cls, shape, overrides):
            made.append((kind, cls, shape))
            return super(Eng, self)._cached(kind, lambda *a, **kw: (cls, a, kw), shape, overrides)

    eng = Eng({}, 50, anchors="A", post_n=100)
    raw = eng.canvas_plan(4, 600, 1000, raw_input=True, arena_bytes=1 << 20)
    flt = eng.canvas_plan(4, 600, 1000)
    assert made == [("raw_canvas", re_.ResNetRawCanvasBatchPlan, (4, 600, 1000)), ("canvas", re_.ResNetCanvasBatchPlan, (4, 600, 1000))]
    assert raw[1:] == ((eng.weights, 4, 600, 1000), dict(anchors="A", feat_stride=32, post_n=100, raw_input=True, arena_bytes=1 << 20))
    assert eng.canvas_plan(4, 600, 1000, raw_input=True, arena_bytes=1 << 20) is raw and flt is not raw and len(eng.plans) == 2
    assert sorted(k[0] for k in eng.plans) == ["canvas", "raw_canvas"]
    p = eng.raw_canvas_plan([np.zeros((300, 500, 3), np.uint8), np.zeros((375, 500, 3), np.uint8)], N=4, conf=0.05)
    assert p[0] is re_.ResNetRawCanvasBatchPlan and p[1][1:] == (4, 640, 1024)
    assert p[2]["raw_input"] and p[2]["with_detect"] and p[2]["det_conf"] == 0.05 and p[2]["arena_bytes"] % (1 << 20) == 0
    assert issubclass(re_.ResNetRawCanvasBatchPlan, re_.ResNetCanvasBatchPlan)
    assert issubclass(re_.ResNetPhotoEngine, re_.ResNetBatchEngine)
