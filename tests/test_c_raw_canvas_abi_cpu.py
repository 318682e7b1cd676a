"""CPU tests of the canvas and raw-photo C entries: frcnn_forward_vgg16_canvas, frcnn_detect_vgg16_raw,
frcnn_detection_lists_batch and frcnn_raw_header_bytes are exported with their declared signatures, reject every bad
argument before anything touches the device (FRCNN_ERR_ARG, or FRCNN_ERR_WORKSPACE for a short workspace), size their
workspace as documented, and the header layout the C header declares is the one preprocess.raw_header_layout builds."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p(256)            # never dereferenced: every call below fails its argument checks first
MEANS = (102.9801, 115.9465, 122.7717)


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def _header():
    return open(os.path.join(ROOT, "include", "frcnn_b200.h")).read()


def _params(name):
    hdr = re.sub(r"/\*.*?\*/", "", _header(), flags=re.S)
    decl = re.search(r"\b%s\((.*?)\);" % name, hdr, flags=re.S).group(1)
    return [" ".join(p.split()) for p in decl.split(",")]


def _cfg(H=600, W=1000, NC=21, post=300, x3=1):
    from frcnn_b200 import _lib
    return _lib.ForwardConfig(H, W, NC, 9, 16, 6000, post, 16, 0.7, x3)


def _weights():
    from frcnn_b200 import _lib
    wt = _lib.Vgg16Weights()
    for i in range(13):
        wt.conv[i] = _lib.PackedLayer(256, 256, 256)
    return wt


def test_declared_signatures(lib):
    from frcnn_b200 import _lib
    want = {
        "frcnn_detection_lists_batch": ["int N", "const float* prob", "long prob_stride", "const float* boxes", "long boxes_stride",
                                        "const int* keep_idx", "long keep_idx_stride", "const int* conf_count",
                                        "long conf_count_stride", "const double* im_scale", "int R_cap", "int num_classes",
                                        "int* out_dets", "float* out_scores", "int* out_det_count", "void* stream"],
        "frcnn_forward_vgg16_canvas_workspace_bytes": ["const frcnn_forward_config* config", "int N"],
        "frcnn_forward_vgg16_canvas": ["const frcnn_forward_config* config", "const frcnn_vgg16_weights* weights", "int N",
                                       "const float* images_nchw", "const int* extents", "const int* im_info", "void* workspace",
                                       "size_t workspace_bytes", "float* out_prob", "float* out_boxes", "int* out_count",
                                       "void* stream"],
        "frcnn_raw_header_bytes": ["int N"],
        "frcnn_detect_vgg16_raw": ["const frcnn_forward_config* config", "const frcnn_vgg16_weights* weights", "int N",
                                   "const void* block", "long long arena_bytes", "double mean_b", "double mean_g", "double mean_r",
                                   "const double* im_scale", "double det_nms_thresh", "float det_conf", "void* workspace",
                                   "size_t workspace_bytes", "float* out_prob", "float* out_boxes", "int* out_count",
                                   "int* out_dets", "float* out_scores", "int* out_det_count", "void* stream"],
    }
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long, "long long": ctypes.c_longlong, "double": ctypes.c_double,
             "float": ctypes.c_float, "size_t": ctypes.c_size_t}
    for name, params in want.items():
        assert _params(name) == params, name
        res, args = _lib.SIGNATURES[name]
        assert getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0]
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
    assert _lib.SIGNATURES["frcnn_raw_header_bytes"][0] is ctypes.c_size_t
    assert _lib.SIGNATURES["frcnn_forward_vgg16_canvas_workspace_bytes"][0] is ctypes.c_size_t
    assert _lib.SIGNATURES["frcnn_detect_vgg16_raw"][0] is _lib.SIGNATURES["frcnn_detection_lists_batch"][0] is ctypes.c_int


# ------------------------------------------------------------------------------------------------------ detection lists
def _lists(lib, N=2, prob=P, ps=6300, boxes=P, bs=25200, keep=P, ks=6000, conf=P, cs=20, scale=P, R=300, NC=21, dets=P,
           scores=P, count=P):
    return lib.frcnn_detection_lists_batch(N, prob, ps, boxes, bs, keep, ks, conf, cs, scale, R, NC, dets, scores, count, None)


@pytest.mark.parametrize("bad,words", [
    (dict(prob=None), ["prob is NULL"]), (dict(boxes=None), ["boxes is NULL"]), (dict(keep=None), ["keep_idx is NULL"]),
    (dict(conf=None), ["conf_count is NULL"]), (dict(scale=None), ["im_scale is NULL"]), (dict(dets=None), ["out_dets is NULL"]),
    (dict(scores=None), ["out_scores is NULL"]), (dict(count=None), ["out_det_count is NULL"]), (dict(N=0), ["N=0"]),
    (dict(N=65536), ["N=65536"]), (dict(N=-1), ["N=-1"]), (dict(R=0), ["R_cap=0"]), (dict(NC=1), ["num_classes=1"]),
    (dict(NC=0), ["num_classes=0"]), (dict(ps=-1), ["stride"]), (dict(bs=-4), ["stride"]), (dict(ks=-1), ["stride"]),
    (dict(cs=-1), ["stride"]), (dict(R=1 << 20, NC=1000), ["too large"])])
def test_detection_lists_argument_errors(lib, bad, words):
    from frcnn_b200 import _lib
    assert _lists(lib, **bad) == _lib.ERR_ARG
    msg = _lib.last_error()
    assert msg.startswith("frcnn_detection_lists_batch") and all(w in msg for w in words), msg


# ------------------------------------------------------------------------------------------------------ canvas forward
def test_canvas_workspace_sizing(lib):
    """The canvas workspace is the same-size batch workspace plus frcnn_detect_batch's outputs, each 256-byte aligned;
    a bad config or N gives 0."""
    from frcnn_b200 import _lib
    al = lambda b: (b + 255) // 256 * 256                                    # noqa: E731
    for (H, W, NC, post, x3) in ((600, 1000, 21, 300, 1), (608, 1024, 21, 300, 0), (64, 96, 5, 37, 1)):
        cfg = ctypes.byref(_cfg(H, W, NC, post, x3))
        for N in (1, 2, 5):
            base = lib.frcnn_forward_batch_workspace_bytes(cfg, N)
            got = lib.frcnn_forward_vgg16_canvas_workspace_bytes(cfg, N)
            assert base > 0 and got == base + al(N * (NC - 1) * post * 4) + 2 * al(N * (NC - 1) * 4), (H, W, NC, N)
    cfg = ctypes.byref(_cfg())
    assert lib.frcnn_forward_vgg16_canvas_workspace_bytes(cfg, 4) > lib.frcnn_forward_vgg16_canvas_workspace_bytes(cfg, 3)
    for N in (0, -1, 65536):
        assert lib.frcnn_forward_vgg16_canvas_workspace_bytes(cfg, N) == 0 and "N must be" in _lib.last_error()
    assert lib.frcnn_forward_vgg16_canvas_workspace_bytes(None, 2) == 0 and "null config" in _lib.last_error()
    for bad in (_cfg(H=8), _cfg(NC=1), _cfg(post=0), _cfg(post=4096)):
        assert lib.frcnn_forward_vgg16_canvas_workspace_bytes(ctypes.byref(bad), 2) == 0
    bad = _cfg()
    bad.feat_stride = 8
    assert lib.frcnn_forward_vgg16_canvas_workspace_bytes(ctypes.byref(bad), 2) == 0 and "feat_stride" in _lib.last_error()


def _canvas(lib, cfg=None, wt=None, N=2, x=P, ext=P, info=P, ws=P, nbytes=None, prob=P, boxes=P, count=P):
    cfg = _cfg() if cfg is None else cfg
    wt = _weights() if wt is None else wt
    if nbytes is None:
        nbytes = lib.frcnn_forward_vgg16_canvas_workspace_bytes(ctypes.byref(cfg), max(1, min(N, 65535)))
    return lib.frcnn_forward_vgg16_canvas(ctypes.byref(cfg), ctypes.byref(wt), N, x, ext, info, ws, nbytes, prob, boxes, count, None)


@pytest.mark.parametrize("bad,words", [
    (dict(x=None), ["null pointer"]), (dict(ext=None), ["null pointer"]), (dict(info=None), ["null pointer"]),
    (dict(ws=None), ["null pointer"]), (dict(prob=None), ["null pointer"]), (dict(boxes=None), ["null pointer"]),
    (dict(count=None), ["null pointer"]), (dict(N=0), ["N must be", "0"]), (dict(N=65536), ["N must be", "65536"]),
    (dict(cfg=_cfg(H=15)), ["too small"]), (dict(cfg=_cfg(NC=1)), ["feat_stride"]), (dict(cfg=_cfg(post=2049)), ["top-N"])])
def test_canvas_argument_errors(lib, bad, words):
    from frcnn_b200 import _lib
    assert _canvas(lib, **bad) == _lib.ERR_ARG
    msg = _lib.last_error()
    assert msg.startswith("frcnn_forward") and all(w in msg for w in words), msg


def test_canvas_short_workspace_and_missing_weights(lib):
    from frcnn_b200 import _lib
    cfg = _cfg()
    need = lib.frcnn_forward_vgg16_canvas_workspace_bytes(ctypes.byref(cfg), 2)
    assert _canvas(lib, cfg=cfg, nbytes=need - 1) == _lib.ERR_WORKSPACE and str(need) in _lib.last_error()
    # the same-size batch workspace is not enough for a canvas call
    assert _canvas(lib, cfg=cfg, nbytes=lib.frcnn_forward_batch_workspace_bytes(ctypes.byref(cfg), 2)) == _lib.ERR_WORKSPACE
    wt = _weights()
    wt.conv[7].lo = None                                                 # bf16x3 needs the lo planes
    assert _canvas(lib, cfg=cfg, wt=wt, nbytes=need) == _lib.ERR_ARG and "trunk layer 7" in _lib.last_error()


# ------------------------------------------------------------------------------------------------------ raw photos
def _raw(lib, cfg=None, wt=None, N=2, block=P, arena=1 << 20, scale=P, ws=P, nbytes=None, prob=P, boxes=P, count=P, dets=P,
         scores=P, dcount=P):
    cfg = _cfg() if cfg is None else cfg
    wt = _weights() if wt is None else wt
    if nbytes is None:
        nbytes = lib.frcnn_forward_vgg16_canvas_workspace_bytes(ctypes.byref(cfg), max(1, min(N, 65535)))
    return lib.frcnn_detect_vgg16_raw(ctypes.byref(cfg), ctypes.byref(wt), N, block, arena, *MEANS, scale, 0.3, ctypes.c_float(0.8), ws,
                                      nbytes, prob, boxes, count, dets, scores, dcount, None)


@pytest.mark.parametrize("bad,words", [
    (dict(block=None), ["null pointer"]), (dict(scale=None), ["null pointer"]), (dict(ws=None), ["null pointer"]),
    (dict(prob=None), ["null pointer"]), (dict(boxes=None), ["null pointer"]), (dict(count=None), ["null pointer"]),
    (dict(dets=None), ["null pointer"]), (dict(scores=None), ["null pointer"]), (dict(dcount=None), ["null pointer"]),
    (dict(block=ctypes.c_void_p(260)), ["8-byte aligned"]), (dict(arena=0), ["arena_bytes", "0"]),
    (dict(arena=-7), ["arena_bytes", "-7"]), (dict(N=0), ["N must be"]), (dict(N=65536), ["N must be"]),
    (dict(cfg=_cfg(W=10)), ["too small"])])
def test_raw_argument_errors(lib, bad, words):
    from frcnn_b200 import _lib
    assert _raw(lib, **bad) == _lib.ERR_ARG
    msg = _lib.last_error()
    assert msg.startswith("frcnn_") and all(w in msg for w in words), msg


def test_raw_short_workspace(lib):
    from frcnn_b200 import _lib
    cfg = _cfg(x3=0)
    need = lib.frcnn_forward_vgg16_canvas_workspace_bytes(ctypes.byref(cfg), 3)
    assert _raw(lib, cfg=cfg, N=3, nbytes=need - 1) == _lib.ERR_WORKSPACE and str(need) in _lib.last_error()


def test_raw_header_bytes_and_declared_offsets_match_the_python_layout(lib):
    from frcnn_b200 import preprocess
    macros = dict((k, int(v)) for k, v in re.findall(r"#define FRCNN_RAW_([A-Z_]+) (\d+)", _header()))
    assert macros == {"EXTENTS": 0, "IM_INFO": 1, "SRC_HW": 2, "SRC_OFF": 3, "INV_SCALE": 4, "FIELDS": 5}
    assert macros["FIELDS"] == len(preprocess.RAW_FIELDS)
    itemsize = {"EXTENTS": (np.int32, 2), "IM_INFO": (np.int32, 2), "SRC_HW": (np.int32, 2), "SRC_OFF": (np.int64, 1),
                "INV_SCALE": (np.float64, 1)}
    for N in (1, 2, 3, 4, 7, 8, 33, 100, 65535):
        layout, hb = preprocess.raw_header_layout(N)
        assert lib.frcnn_raw_header_bytes(N) == hb and hb % 256 == 0
        for name, f in macros.items():
            if name == "FIELDS":
                continue
            off, dt, items = layout[name.lower()]
            assert off == 8 * N * f and (dt, items) == itemsize[name], (N, name)
    for N in (0, -1, 65536):
        assert lib.frcnn_raw_header_bytes(N) == 0


def test_numpy_divides_float32_boxes_by_a_python_float_in_float32():
    """The rule frcnn_detection_lists_batch restates: under the repository's NumPy (>= 2, NEP 50) a float32 row divided by a
    Python float is a float32 division by float32(im_scale) -- not a float64 division -- so the truncated ints can differ."""
    assert int(np.__version__.split(".")[0]) >= 2
    row = np.array([18.0, 30.0, 36.0, 7.5], dtype=np.float32)
    q = row / 1.2
    assert q.dtype == np.float32
    assert np.array_equal(q.view(np.uint32), (row / np.float32(1.2)).view(np.uint32))
    assert list(map(int, q)) == [14, 24, 29, 6]
    assert [int(float(v) / 1.2) for v in row] == [15, 25, 30, 6]          # what a float64 division would give
    assert not np.array_equal(q, row * np.float32(1.0 / 1.2))              # nor is it the product with the reciprocal
