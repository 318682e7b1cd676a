"""CPU tests of the raw-photo front end of canvas batches: frcnn_preprocess_bgr8_canvas is exported with the declared
signature and rejects every bad argument with FRCNN_ERR_ARG and a message naming it before anything touches the device,
and the host side of CanvasBatchPlan(raw_input=True) -- the [descriptor header | pixels] layout and the fit checks built on
preprocess.plan_size -- is plain arithmetic that runs without a GPU."""
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


def _call(lib, arena=P, arena_bytes=1 << 20, src_off=P, src_hw=P, inv_scale=P, extents=P, N=2, Hc=64, Wc=96, y_hi=P):
    return lib.frcnn_preprocess_bgr8_canvas(arena, arena_bytes, src_off, src_hw, inv_scale, extents, N, Hc, Wc, *MEANS, y_hi, None,
                                            None)


def test_symbol_and_declared_signature(lib):
    from frcnn_b200 import _lib
    res, args = _lib.SIGNATURES["frcnn_preprocess_bgr8_canvas"]
    assert res is ctypes.c_int and len(args) == 15 and args[1] is ctypes.c_longlong and args[9:12] == [ctypes.c_double] * 3
    assert lib.frcnn_preprocess_bgr8_canvas.argtypes == args
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "frcnn_b200.h")).read(), flags=re.S)
    decl = re.search(r"int frcnn_preprocess_bgr8_canvas\((.*?)\);", hdr, flags=re.S).group(1)
    params = [" ".join(p.split()) for p in decl.split(",")]
    assert params == ["const unsigned char* arena", "long long arena_bytes", "const long long* src_off", "const int* src_hw",
                      "const double* inv_scale", "const int* extents", "int N", "int Hc", "int Wc", "double mean_b",
                      "double mean_g", "double mean_r", "void* y_hi", "void* y_lo", "void* stream"]


@pytest.mark.parametrize("bad,words", [
    (dict(arena=None), ["arena is NULL"]), (dict(arena_bytes=0), ["arena_bytes", "0"]), (dict(arena_bytes=-5), ["arena_bytes", "-5"]),
    (dict(src_off=None), ["src_off"]), (dict(src_hw=None), ["src_hw"]), (dict(inv_scale=None), ["inv_scale"]),
    (dict(extents=None), ["extents"]), (dict(y_hi=None), ["y_hi"]), (dict(N=0), ["N=0"]), (dict(N=65536), ["N=65536"]),
    (dict(Hc=0), ["Hc=0"]), (dict(Wc=-3), ["Wc=-3"])])
def test_argument_errors_name_the_argument(lib, bad, words):
    from frcnn_b200 import _lib
    assert _call(lib, **bad) == _lib.ERR_ARG
    msg = _lib.last_error()
    assert msg.startswith("frcnn_preprocess_bgr8_canvas") and all(w in msg for w in words), msg


def test_header_layout():
    """Five arrays of 8 * N bytes each, 8-byte aligned, then the pixels on a 256-byte boundary."""
    from frcnn_b200 import preprocess
    for N in (1, 3, 4, 8, 33):
        layout, hb = preprocess.raw_header_layout(N)
        assert list(layout) == ["extents", "im_info", "src_hw", "src_off", "inv_scale"]
        assert [layout[k][0] for k in layout] == [0, 8 * N, 16 * N, 24 * N, 32 * N]
        assert hb % 256 == 0 and 40 * N <= hb < 40 * N + 256
        buf = np.zeros((hb,), dtype=np.uint8)
        v = preprocess.raw_header_views(buf, N)
        assert v["extents"].shape == (N, 2) and v["src_off"].dtype == np.int64 and v["inv_scale"].dtype == np.float64
        v["src_off"][N - 1] = -2
        assert buf[24 * N + 8 * (N - 1):32 * N].tolist() == [254] + [255] * 7          # a view, not a copy


def test_batch_header_contents_and_fit_checks():
    from frcnn_b200 import preprocess
    from frcnn_b200._lib import FrcnnError
    shapes = [(375, 500), (333, 500), (300, 500)]
    hdr, scales, used = preprocess.raw_batch_header(shapes, 4, 600, 1000, 1 << 21)
    v = preprocess.raw_header_views(hdr, 4)
    want = [preprocess.plan_size(h, w) for h, w in shapes]
    assert scales == [s for s, _, _ in want]
    assert v["extents"].tolist() == [[600, 800], [600, 901], [600, 1000], [0, 0]] == [list(w[1:]) for w in want] + [[0, 0]]
    assert v["im_info"].tolist() == v["extents"].tolist() and v["src_hw"].tolist() == [list(s) for s in shapes] + [[0, 0]]
    assert v["inv_scale"].tolist() == [1.0 / s for s in scales] + [0.0]
    offs = v["src_off"].tolist()
    assert offs[0] == 0 and all(o % preprocess.RAW_ALIGN == 0 for o in offs)
    assert offs[1] >= 3 * 375 * 500 and offs[2] >= offs[1] + 3 * 333 * 500 and used == offs[2] + 3 * 300 * 500
    # forward.py's clip bounds (H, H)
    hdr2, _, _ = preprocess.raw_batch_header(shapes[:2], 4, 600, 1000, 1 << 21, img_infos=[(600, 600), (600, 600)])
    assert preprocess.raw_header_views(hdr2, 4)["im_info"].tolist() == [[600, 600], [600, 600], [0, 0], [0, 0]]
    # the arena holds exactly `used` bytes, not one fewer
    preprocess.raw_batch_header(shapes, 4, 600, 1000, used)
    with pytest.raises(FrcnnError, match="arena"):
        preprocess.raw_batch_header(shapes, 4, 600, 1000, used - 1)
    with pytest.raises(FrcnnError, match="canvas"):
        preprocess.raw_batch_header([(500, 375)], 4, 600, 1000, 1 << 21)          # portrait: resizes to 800 x 600
    with pytest.raises(FrcnnError, match="canvas"):
        preprocess.raw_batch_header([(300, 500)], 4, 600, 999, 1 << 21)
    with pytest.raises(FrcnnError, match="slots"):
        preprocess.raw_batch_header(shapes, 2, 600, 1000, 1 << 21)
    with pytest.raises(FrcnnError, match="img_infos"):
        preprocess.raw_batch_header(shapes, 4, 600, 1000, 1 << 21, img_infos=[(600, 600)])
    with pytest.raises(FrcnnError, match="no pixels"):
        preprocess.raw_batch_header([(0, 500)], 4, 600, 1000, 1 << 21)
    # 720 x 1280 is scaled DOWN (long side 1000): the source is larger than its slot of the canvas
    _, s, used = preprocess.raw_batch_header([(720, 1280)], 1, 576, 1024, 3 * 720 * 1280)
    assert preprocess.plan_size(720, 1280)[1:] == (562, 1000) and used == 3 * 720 * 1280


def test_result_detections_is_the_forward_py_loop():
    """preprocess.result_detections on host arrays = forward.py:50-59 over the kept rows, boxes / im_scale truncated."""
    from frcnn_b200 import preprocess
    rng = np.random.default_rng(3)
    R, NC = 7, 4
    prob = rng.random((R, NC)).astype(np.float32)
    boxes = (rng.random((R, 4 * NC)) * 900 - 20).astype(np.float32)
    keep_idx = np.array([[3, 1, 0, 0, 0, 0, 0, 0], [0] * 8, [6, 5, 2, 0, 0, 0, 0, 0]], dtype=np.int32)
    conf_count = np.array([2, 0, 3], dtype=np.int32)
    got = preprocess.result_detections(dict(prob=prob, boxes=boxes, keep_idx=keep_idx, conf_count=conf_count), 1.6)
    want = [(c, *map(int, boxes[r, 4 * c:4 * c + 4] / 1.6), float(prob[r, c])) for c, rows in ((1, [3, 1]), (3, [6, 5, 2])) for r in rows]
    assert got == want and all(isinstance(v, int) for d in got for v in d[:5])
    boxes[3, 4] = -7.9                                                      # -4.9375 after scaling: truncated towards zero
    assert preprocess.result_detections(dict(prob=prob, boxes=boxes, keep_idx=keep_idx, conf_count=conf_count), 1.6)[0][1] == -4
