"""CPU tests of the C entries that turn ground truth into training targets and losses (rpn_train.cu, rcnn_train.cu):
frcnn_anchor_targets, frcnn_rpn_loss, frcnn_rcnn_loss, frcnn_roi_overlaps, frcnn_roi_targets, frcnn_bbox_transform,
frcnn_keep_inside and frcnn_bbox_overlaps are exported with their declared signatures and reject every bad argument
before anything touches the device (FRCNN_ERR_ARG, or FRCNN_ERR_WORKSPACE for a short workspace).

The pointers are fake and never dereferenced.  Each call that tests one of the newer checks (num_fg against batch, the
anchor count of frcnn_rpn_loss, num_classes >= 1) is arranged so that a build without that check still stops before a
launch: at the workspace check (a zero-byte workspace) or at the kept-row check (n = 0), with another message."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p(256)            # 256-byte aligned, never dereferenced
P_ODD = ctypes.c_void_p(260)        # 4-byte aligned only


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def _params(name):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "frcnn_b200.h")).read(), flags=re.S)
    decl = re.search(r"\b%s\((.*?)\);" % name, hdr, flags=re.S).group(1)
    return [" ".join(p.split()) for p in decl.split(",")]


def _fail(status, code, words):
    from frcnn_b200 import _lib
    msg = _lib.last_error()
    assert status == code, (status, msg)
    assert all(w in msg for w in words), msg


def test_declared_signatures(lib):
    from frcnn_b200 import _lib
    names = ["frcnn_bbox_overlaps", "frcnn_anchor_targets_workspace_bytes", "frcnn_anchor_targets", "frcnn_rpn_loss_workspace_bytes",
             "frcnn_rpn_loss", "frcnn_roi_overlaps", "frcnn_roi_targets", "frcnn_bbox_transform", "frcnn_keep_inside",
             "frcnn_rcnn_loss"]
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long, "double": ctypes.c_double, "float": ctypes.c_float,
             "size_t": ctypes.c_size_t, "unsigned long long": ctypes.c_ulonglong}
    for name in names:
        params = _params(name)
        res, args = _lib.SIGNATURES[name]
        assert getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0].replace("const ", "")
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
        assert res is (ctypes.c_size_t if name.endswith("_workspace_bytes") else ctypes.c_int), name


# ------------------------------------------------------------------------------------------------------ anchor targets
def _anchor_targets(lib, anchors=P, A=9, fh=38, fw=63, stride=16, gt=P, n_gt=3, im_h=600, im_w=1000, neg=0.3, pos=0.7,
                    batch=256, num_fg=128, mode=1, seed=7, dis=None, n_dis=0, labels=P, targets=P, inds=P, counts=P, ws=P,
                    nbytes=0):
    return lib.frcnn_anchor_targets(anchors, A, fh, fw, stride, gt, n_gt, im_h, im_w, neg, pos, batch, num_fg, mode,
                                    ctypes.c_ulonglong(seed), dis, n_dis, labels, targets, inds, counts, ws, nbytes, None)


@pytest.mark.parametrize("bad,words", [
    (dict(A=0), ["bad geometry"]), (dict(A=-9), ["bad geometry"]), (dict(fh=0), ["bad geometry"]), (dict(fw=-1), ["bad geometry"]),
    (dict(stride=0), ["bad geometry"]), (dict(n_gt=0), ["at least one ground-truth"]), (dict(n_gt=-2), ["at least one"]),
    (dict(anchors=None), ["null pointer"]), (dict(gt=None), ["null pointer"]), (dict(labels=None), ["null pointer"]),
    (dict(targets=None), ["null pointer"]), (dict(inds=None), ["null pointer"]), (dict(counts=None), ["null pointer"]),
    (dict(ws=None), ["null pointer"]), (dict(mode=3), ["subsample_mode 3"]), (dict(mode=-1), ["subsample_mode -1"]),
    (dict(mode=2, n_dis=5), ["mode 2 without an index list"]), (dict(targets=P_ODD), ["16-byte aligned"]),
    (dict(A=1 << 10, fh=1 << 10, fw=1 << 10), ["too many anchors"]), (dict(A=3, fh=1 << 15, fw=1 << 15), ["too many anchors"]),
    # mode 1 with more positives allowed than the batch holds: num_bg = batch - n_fg would go negative
    (dict(num_fg=257), ["num_fg=257", "batch=256"]), (dict(num_fg=-1), ["num_fg=-1"]), (dict(batch=-1, num_fg=0), ["batch=-1"]),
    (dict(batch=0, num_fg=1), ["num_fg=1", "batch=0"])])
def test_anchor_targets_argument_errors(lib, bad, words):
    from frcnn_b200 import _lib
    _fail(_anchor_targets(lib, **bad), _lib.ERR_ARG, ["anchor_targets:"] + words)


def test_anchor_targets_num_fg_is_only_checked_where_it_is_used(lib):
    """Modes 0 and 2 ignore batch / num_fg: a short workspace, not the counts, is what stops these calls."""
    from frcnn_b200 import _lib
    for mode in (0, 2):
        _fail(_anchor_targets(lib, mode=mode, num_fg=300, batch=256), _lib.ERR_WORKSPACE, ["workspace"])
        _fail(_anchor_targets(lib, mode=mode, num_fg=-5, batch=-1), _lib.ERR_WORKSPACE, ["workspace"])
    _fail(_anchor_targets(lib, mode=1, num_fg=256, batch=256), _lib.ERR_WORKSPACE, ["workspace"])       # num_fg == batch is fine
    _fail(_anchor_targets(lib, mode=1, num_fg=0, batch=0), _lib.ERR_WORKSPACE, ["workspace"])


def test_anchor_targets_workspace(lib):
    from frcnn_b200 import _lib
    al = lambda b: (b + 255) // 256 * 256                                    # noqa: E731
    for n_all, n_gt in ((21546, 3), (1, 1), (40960, 256), (41472, 300)):
        assert lib.frcnn_anchor_targets_workspace_bytes(n_all, n_gt) == al(8 * n_all) + al(4 * n_all) + al(8 * n_gt)
    assert lib.frcnn_anchor_targets_workspace_bytes(-1, 3) == 0 and lib.frcnn_anchor_targets_workspace_bytes(5, -1) == 0
    need = lib.frcnn_anchor_targets_workspace_bytes(9 * 38 * 63, 3)
    _fail(_anchor_targets(lib, nbytes=need - 1), _lib.ERR_WORKSPACE, [str(need), str(need - 1)])


# ------------------------------------------------------------------------------------------------------ RPN loss
def _rpn_loss(lib, score=P, bbox=P, anchors=P, A=9, fh=38, fw=63, stride=16, labels=P, targets=P, counts=P, delta=3.0, lam=1.0,
              gs=1.0, losses=P, ws=P, nbytes=0):
    return lib.frcnn_rpn_loss(score, fh * fw, 1, bbox, fh * fw, 1, anchors, A, fh, fw, stride, 600, 1000, labels, targets, counts,
                              delta, lam, gs, losses, None, None, ws, nbytes, None)


@pytest.mark.parametrize("bad,words", [
    (dict(A=0), ["bad geometry"]), (dict(fh=0), ["bad geometry"]), (dict(fw=-3), ["bad geometry"]), (dict(stride=-16), ["bad geometry"]),
    (dict(score=None), ["null pointer"]), (dict(bbox=None), ["null pointer"]), (dict(anchors=None), ["null pointer"]),
    (dict(labels=None), ["null pointer"]), (dict(targets=None), ["null pointer"]), (dict(counts=None), ["null pointer"]),
    (dict(losses=None), ["null pointer"]), (dict(ws=None), ["null pointer"]), (dict(targets=P_ODD), ["16-byte aligned"]),
    (dict(delta=0.0), ["delta must be positive"]), (dict(delta=-3.0), ["delta must be positive"]),
    (dict(delta=float("nan")), ["delta must be positive"]),
    # 2^30 anchors fit an int but not the anchor-target entry that made the labels
    (dict(A=1 << 10, fh=1 << 10, fw=1 << 10), ["too many anchors"])])
def test_rpn_loss_argument_errors(lib, bad, words):
    from frcnn_b200 import _lib
    _fail(_rpn_loss(lib, **bad), _lib.ERR_ARG, ["rpn_loss:"] + words)


def test_rpn_loss_workspace(lib):
    from frcnn_b200 import _lib
    for n_all in (1, 255, 256, 257, 21546, 41472):
        assert lib.frcnn_rpn_loss_workspace_bytes(n_all) == -(-n_all // 256) * 32
    assert lib.frcnn_rpn_loss_workspace_bytes(0) == 32 and lib.frcnn_rpn_loss_workspace_bytes(-1) == 0
    need = lib.frcnn_rpn_loss_workspace_bytes(9 * 38 * 63)
    _fail(_rpn_loss(lib, nbytes=need - 1), _lib.ERR_WORKSPACE, [str(need)])


# ------------------------------------------------------------------------------------------------------ RCNN loss
def _rcnn_loss(lib, head=P, ld=128, R=300, keep=P, n=64, labels=P, ext=P, NC=21, delta=1.0, losses=P):
    return lib.frcnn_rcnn_loss(head, ld, R, keep, n, labels, ext, NC, delta, 1.0, losses, None, None)


@pytest.mark.parametrize("bad,words", [
    (dict(head=None), ["bad arguments"]), (dict(keep=None), ["bad arguments"]), (dict(labels=None), ["bad arguments"]),
    (dict(ext=None), ["bad arguments"]), (dict(losses=None), ["bad arguments"]), (dict(R=0), ["bad arguments"]),
    (dict(ld=104, NC=21), ["bad arguments"]), (dict(ld=-5, NC=21), ["bad arguments"]),
    (dict(ld=1 << 30, NC=(1 << 30) // 5 + 1), ["bad arguments"]),
    (dict(ld=0x7FFFFFFF, NC=0x7FFFFFFF // 4, n=0), ["bad arguments"]),      # 5*NC would wrap an int product
    (dict(n=0), ["1 <= kept rows", "got 0"]), (dict(n=129), ["got 129"]), (dict(n=-1), ["got -1"]),
    (dict(delta=0.0), ["delta must be positive"]), (dict(delta=float("nan")), ["delta must be positive"]),
    # no class at all: refused by the argument check itself (n=0 would stop a build without it at the row check instead)
    (dict(NC=0, n=0), ["bad arguments"]), (dict(NC=-1, n=0), ["bad arguments"]), (dict(NC=0, ld=0, n=0), ["bad arguments"])])
def test_rcnn_loss_argument_errors(lib, bad, words):
    from frcnn_b200 import _lib
    _fail(_rcnn_loss(lib, **bad), _lib.ERR_ARG, ["rcnn_loss:"] + words)


# ------------------------------------------------------------------------------------------------------ proposal targets
@pytest.mark.parametrize("args,words", [
    (dict(rois=None), []), (dict(gt=None), []), (dict(mo=None), []), (dict(am=None), []), (dict(R=0), []), (dict(R=-1), []),
    (dict(n_gt=0), []), (dict(n_gt=-1), [])])
def test_roi_overlaps_argument_errors(lib, args, words):
    from frcnn_b200 import _lib
    a = dict(rois=P, count=None, R=300, gt=P, n_gt=3, mo=P, am=P)
    a.update(args)
    _fail(lib.frcnn_roi_overlaps(a["rois"], a["count"], a["R"], a["gt"], a["n_gt"], a["mo"], a["am"], None), _lib.ERR_ARG,
          ["roi_overlaps: bad arguments"] + words)


def _roi_targets(lib, rois=P, gt=P, am=P, keep=P, n=64, NC=21, use_gt=P, ext=P, labels=P):
    return lib.frcnn_roi_targets(rois, gt, am, keep, n, NC, use_gt, ext, labels, None)


@pytest.mark.parametrize("bad", [dict(rois=None), dict(gt=None), dict(am=None), dict(keep=None), dict(use_gt=None), dict(ext=None),
                                 dict(labels=None), dict(n=-1), dict(NC=0), dict(NC=-21), dict(n=0, NC=0)])
def test_roi_targets_argument_errors(lib, bad):
    from frcnn_b200 import _lib
    _fail(_roi_targets(lib, **bad), _lib.ERR_ARG, ["roi_targets: bad arguments"])


# ------------------------------------------------------------------------------------------------------ helpers
@pytest.mark.parametrize("args,words", [
    (dict(n=-1), ["negative size"]), (dict(k=-1), ["negative size"]), (dict(boxes=None), ["null pointer"]),
    (dict(query=None), ["null pointer"]), (dict(out=None), ["null pointer"])])
def test_bbox_overlaps_argument_errors(lib, args, words):
    from frcnn_b200 import _lib
    a = dict(boxes=P, n=500, query=P, k=17, out=P)
    a.update(args)
    _fail(lib.frcnn_bbox_overlaps(a["boxes"], a["n"], a["query"], a["k"], a["out"], None), _lib.ERR_ARG, ["bbox_overlaps:"] + words)


@pytest.mark.parametrize("args,words", [
    (dict(n=-1), ["bad arguments"]), (dict(stride=3), ["bad arguments"]), (dict(stride=-5), ["bad arguments"]),
    (dict(ex=None), ["null pointer"]), (dict(gt=None), ["null pointer"]), (dict(out=None), ["null pointer"])])
def test_bbox_transform_argument_errors(lib, args, words):
    from frcnn_b200 import _lib
    a = dict(ex=P, gt=P, stride=5, n=300, out=P)
    a.update(args)
    _fail(lib.frcnn_bbox_transform(a["ex"], a["gt"], a["stride"], a["n"], a["out"], None), _lib.ERR_ARG, ["bbox_transform:"] + words)


@pytest.mark.parametrize("args,words", [(dict(n=-1), ["bad arguments"]), (dict(boxes=None), ["null pointer"]),
                                        (dict(flags=None), ["null pointer"])])
def test_keep_inside_argument_errors(lib, args, words):
    from frcnn_b200 import _lib
    a = dict(boxes=P, n=300, flags=P)
    a.update(args)
    _fail(lib.frcnn_keep_inside(a["boxes"], a["n"], 600, 1000, a["flags"], None), _lib.ERR_ARG, ["keep_inside:"] + words)


def test_empty_inputs_are_no_ops_before_the_pointer_checks(lib):
    """n == 0 (or k == 0) returns FRCNN_OK without a launch, even with null pointers: an empty batch needs no buffers."""
    from frcnn_b200 import _lib
    assert lib.frcnn_bbox_overlaps(None, 0, None, 5, None, None) == _lib.OK
    assert lib.frcnn_bbox_overlaps(None, 7, None, 0, None, None) == _lib.OK
    assert lib.frcnn_bbox_transform(None, None, 4, 0, None, None) == _lib.OK
    assert lib.frcnn_keep_inside(None, 0, 600, 1000, None, None) == _lib.OK
    assert _roi_targets(lib, n=0) == _lib.OK                       # pointers are still checked first here
    _fail(_roi_targets(lib, n=0, rois=None), _lib.ERR_ARG, ["roi_targets: bad arguments"])
