"""CPU tests of the VOC evaluation C entries: frcnn_voc_eval_workspace_bytes, frcnn_voc_eval_append_batch and frcnn_voc_eval
are exported with their declared signatures, reject every bad argument before anything touches the device (FRCNN_ERR_ARG, or
FRCNN_ERR_WORKSPACE for a short workspace), size the workspace as documented, and VocEvaluator's host-side GT validation
raises on malformed ground truth."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p(256)            # never dereferenced: every call below fails its argument checks first


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def _params(name):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "frcnn_b200.h")).read(), flags=re.S)
    decl = re.search(r"\b%s\((.*?)\);" % name, hdr, flags=re.S).group(1)
    return [" ".join(p.split()) for p in decl.split(",")]


def test_declared_signatures(lib):
    from frcnn_b200 import _lib
    want = {
        "frcnn_voc_eval_workspace_bytes": ["int num_classes", "int capacity", "int max_images", "int max_gt"],
        "frcnn_voc_eval_append_batch": ["int N", "const float* prob", "long prob_stride", "const float* boxes", "long boxes_stride",
                                        "const int* keep_idx", "long keep_idx_stride", "const int* conf_count",
                                        "long conf_count_stride", "const double* im_scale", "int R_cap", "int num_classes",
                                        "int image_base", "int capacity", "int max_images", "void* ws", "size_t ws_bytes",
                                        "void* stream"],
        "frcnn_voc_eval": ["int num_classes", "int capacity", "int max_images", "int max_gt", "int n_images",
                           "const int* gt_offsets", "const float* gt_boxes", "const int* gt_labels",
                           "const unsigned char* gt_difficult", "int n_gt", "double iou_thresh", "double* out", "void* ws",
                           "size_t ws_bytes", "void* stream"],
    }
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long, "double": ctypes.c_double, "size_t": ctypes.c_size_t}
    for name, params in want.items():
        assert _params(name) == params, name
        res, args = _lib.SIGNATURES[name]
        assert getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0]
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
    assert _lib.SIGNATURES["frcnn_voc_eval_workspace_bytes"][0] is ctypes.c_size_t
    assert _lib.SIGNATURES["frcnn_voc_eval_append_batch"][0] is _lib.SIGNATURES["frcnn_voc_eval"][0] is ctypes.c_int


def _want_bytes(NC, cap, M, G):
    """The workspace, region by region (voc_eval.cu's layout), each region 256-byte aligned: the curves tp_cum / fp_cum
    (int32 [cap] each) first, the detection counter, the segment table (int2 [NC-1][M]), the pool (float4 box + float score
    per detection), the class offsets (int [NC-1][M], int [NC-1]), the flags (uint8 [cap]), the sort's key / value double
    buffers (uint64 / int32 [cap] twice), its tile histograms (int [256][ceil(cap/2048)]) and row totals (int [256]), the
    precision envelope (double [cap]), and last the GT claim flags (uint8 [G])."""
    al = lambda b: (b + 255) // 256 * 256                                     # noqa: E731
    S, tiles = (NC - 1) * M, (cap + 2047) // 2048
    regions = [4 * cap, 4 * cap, 8, 8 * S, 16 * cap, 4 * cap, 4 * S, 4 * (NC - 1), cap, 8 * cap, 8 * cap, 4 * cap, 4 * cap,
               4 * 256 * tiles, 4 * 256, 8 * cap, G]
    return sum(al(r) for r in regions)


def test_workspace_formula(lib):
    from frcnn_b200 import _lib
    for NC, cap, M, G in ((21, 1_000_000, 4952, 14976), (2, 1, 1, 0), (21, 2049, 3, 17), (300, 123457, 10, 1000)):
        assert lib.frcnn_voc_eval_workspace_bytes(NC, cap, M, G) == _want_bytes(NC, cap, M, G), (NC, cap, M, G)
    for bad in ((1, 10, 10, 10), (0, 10, 10, 10), (65537, 10, 10, 10), (21, 0, 10, 10), (21, (1 << 30) + 1, 10, 10),
                (21, 10, 0, 10), (21, 10, 10, -1), (1 << 16, 10, 1 << 16, 0)):
        assert lib.frcnn_voc_eval_workspace_bytes(*bad) == 0 and "bad sizes" in _lib.last_error(), bad


def _append(lib, N=2, prob=P, ps=6300, boxes=P, bs=25200, keep=P, ks=6000, conf=P, cs=20, scale=P, R=300, NC=21, base=0,
            cap=1000, M=10, ws=P, nbytes=None):
    if nbytes is None:
        nbytes = lib.frcnn_voc_eval_workspace_bytes(21, 1000, 10, 0)
    return lib.frcnn_voc_eval_append_batch(N, prob, ps, boxes, bs, keep, ks, conf, cs, scale, R, NC, base, cap, M, ws, nbytes, None)


@pytest.mark.parametrize("bad,words", [
    (dict(prob=None), ["prob is NULL"]), (dict(boxes=None), ["boxes is NULL"]), (dict(keep=None), ["keep_idx is NULL"]),
    (dict(conf=None), ["conf_count is NULL"]), (dict(scale=None), ["im_scale is NULL"]), (dict(ws=None), ["ws is NULL"]),
    (dict(N=0), ["N=0"]), (dict(N=65536), ["N=65536"]), (dict(N=-1), ["N=-1"]), (dict(R=0), ["R_cap=0"]),
    (dict(NC=1), ["num_classes"]), (dict(NC=0), ["num_classes"]), (dict(ps=-1), ["stride"]), (dict(bs=-4), ["stride"]),
    (dict(ks=-1), ["stride"]), (dict(cs=-1), ["stride"]), (dict(base=-1), ["max_images"]), (dict(base=9), ["max_images = 10"]),
    (dict(N=11), ["max_images = 10"]), (dict(cap=0), ["capacity"]), (dict(M=0), ["max_images"])])
def test_append_argument_errors(lib, bad, words):
    from frcnn_b200 import _lib
    assert _append(lib, **bad) == _lib.ERR_ARG
    msg = _lib.last_error()
    assert msg.startswith("frcnn_voc_eval_append_batch") and all(w in msg for w in words), msg


def test_append_short_workspace(lib):
    from frcnn_b200 import _lib
    need = lib.frcnn_voc_eval_workspace_bytes(21, 1000, 10, 0)
    assert _append(lib, nbytes=need - 1) == _lib.ERR_WORKSPACE and "workspace" in _lib.last_error()


def _eval(lib, NC=21, cap=1000, M=10, G=64, n=10, off=P, boxes=P, labels=P, diff=P, n_gt=5, thr=0.5, out=P, ws=P, nbytes=None):
    if nbytes is None:
        nbytes = lib.frcnn_voc_eval_workspace_bytes(21, 1000, 10, 64)
    return lib.frcnn_voc_eval(NC, cap, M, G, n, off, boxes, labels, diff, n_gt, thr, out, ws, nbytes, None)


@pytest.mark.parametrize("bad,words", [
    (dict(off=None), ["gt_offsets is NULL"]), (dict(boxes=None), ["gt_boxes is NULL"]), (dict(labels=None), ["gt_labels is NULL"]),
    (dict(diff=None), ["gt_difficult is NULL"]), (dict(out=None), ["out is NULL"]), (dict(ws=None), ["ws is NULL"]),
    (dict(NC=1), ["num_classes"]), (dict(cap=0), ["capacity"]), (dict(M=0), ["max_images"]), (dict(G=-1), ["max_gt"]),
    (dict(n=11), ["n_images"]), (dict(n=-1), ["n_images"]), (dict(n_gt=65), ["n_gt"]), (dict(n_gt=-1), ["n_gt"]),
    (dict(thr=float("nan")), ["iou_thresh"]), (dict(thr=float("inf")), ["iou_thresh"]), (dict(thr=-float("inf")), ["iou_thresh"])])
def test_eval_argument_errors(lib, bad, words):
    from frcnn_b200 import _lib
    assert _eval(lib, **bad) == _lib.ERR_ARG
    msg = _lib.last_error()
    assert msg.startswith("frcnn_voc_eval") and all(w in msg for w in words), msg


def test_eval_short_workspace(lib):
    from frcnn_b200 import _lib
    need = lib.frcnn_voc_eval_workspace_bytes(21, 1000, 10, 64)
    assert _eval(lib, nbytes=need - 1) == _lib.ERR_WORKSPACE and "workspace" in _lib.last_error()


# ------------------------------------------------------------------------------------------------------ host GT validation
GOOD_B, GOOD_L = [np.array([[0, 0, 9, 9]], np.float32), np.zeros((0, 4))], [np.array([3]), np.zeros(0, np.int64)]


@pytest.mark.parametrize("boxes,labels,diff,n,words", [
    (GOOD_B, GOOD_L, None, 3, "3 were added"),
    (GOOD_B[:1], GOOD_L, None, 2, "2 were added"),
    ([np.zeros((1, 5)), GOOD_B[1]], GOOD_L, None, 2, "boxes [k,4]"),
    (GOOD_B, [np.array([3, 4]), GOOD_L[1]], None, 2, "labels [k]"),
    (GOOD_B, [np.array([0]), GOOD_L[1]], None, 2, "outside 1..20"),
    (GOOD_B, [np.array([21]), GOOD_L[1]], None, 2, "outside 1..20"),
    (GOOD_B, [np.array([1.5]), GOOD_L[1]], None, 2, "outside 1..20"),
    (GOOD_B, GOOD_L, [[True, False], []], 2, "difficult flags"),
    (GOOD_B, GOOD_L, [[True]], 2, "were added"),
])
def test_gt_validation(boxes, labels, diff, n, words):
    from frcnn_b200 import FrcnnError
    from frcnn_b200.evaluate import pack_gt
    with pytest.raises(FrcnnError, match=re.escape(words)):
        pack_gt(boxes, labels, diff, n, 21, 1000)


def test_gt_packing():
    """The CSR blob: offsets, boxes, labels and difficult flags at 16-byte aligned offsets; too many boxes raise."""
    from frcnn_b200 import FrcnnError
    from frcnn_b200.evaluate import pack_gt
    boxes = [np.array([[0, 0, 9, 9], [1, 2, 3, 4]], np.float32), np.zeros((0, 4)), np.array([[5, 6, 7, 8]], np.float32)]
    labels = [np.array([3, 1]), np.zeros(0, np.int64), np.array([20])]
    blob, G, (ob, ol, od) = pack_gt(boxes, labels, [[False, True], [], [True]], 3, 21, 3)
    assert G == 3 and ob % 16 == ol % 16 == od % 16 == 0
    assert blob[:16].view(np.int32).tolist() == [0, 2, 2, 3]
    assert blob[ob:ob + 48].view(np.float32).reshape(3, 4).tolist() == [[0, 0, 9, 9], [1, 2, 3, 4], [5, 6, 7, 8]]
    assert blob[ol:ol + 12].view(np.int32).tolist() == [3, 1, 20] and blob[od:od + 3].tolist() == [0, 1, 1]
    with pytest.raises(FrcnnError, match="max_gt"):
        pack_gt(boxes, labels, None, 3, 21, 2)
