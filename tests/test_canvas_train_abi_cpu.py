"""CPU tests of the canvas training entries (frcnn_anchor_targets_batch, frcnn_rpn_loss_batch, frcnn_grad_prepare_batch):
they are exported with their declared signatures and reject every bad argument with FRCNN_ERR_ARG (or FRCNN_ERR_WORKSPACE
for a missing or short workspace) and a message, before anything touches the device.  The pointers are fake and never
dereferenced."""
import ctypes

import pytest

from test_train_targets_abi_cpu import P, P_ODD, _fail, _params

ERR_ARG, ERR_WS = -1, -3


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def test_declared_signatures(lib):
    from frcnn_b200 import _lib
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long, "double": ctypes.c_double, "float": ctypes.c_float,
             "size_t": ctypes.c_size_t}
    for name in ("frcnn_anchor_targets_batch_workspace_bytes", "frcnn_anchor_targets_batch", "frcnn_rpn_loss_batch_workspace_bytes",
                 "frcnn_rpn_loss_batch", "frcnn_grad_prepare_batch"):
        params = _params(name)
        res, args = _lib.SIGNATURES[name]
        assert getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0].replace("const ", "")
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
        assert res is (ctypes.c_size_t if name.endswith("_workspace_bytes") else ctypes.c_int), name


def test_workspace_sizes(lib):
    one = lib.frcnn_anchor_targets_workspace_bytes(9 * 38 * 63, 20)
    assert lib.frcnn_anchor_targets_batch_workspace_bytes(1, 9 * 38 * 63, 20) == one
    assert lib.frcnn_anchor_targets_batch_workspace_bytes(4, 9 * 38 * 63, 20) >= 4 * (9 * 38 * 63) * 12
    assert lib.frcnn_anchor_targets_batch_workspace_bytes(0, 100, 1) == 0
    assert lib.frcnn_rpn_loss_batch_workspace_bytes(3, 9 * 38 * 63) == 3 * lib.frcnn_rpn_loss_workspace_bytes(9 * 38 * 63)
    assert lib.frcnn_rpn_loss_batch_workspace_bytes(0, 10) == 0


def _targets(lib, N=2, A=9, fh=38, fw=63, stride=16, ext=P, halv=4, info=P, gt=P, max_gt=8, gtc=P, batch=256, num_fg=128,
             mode=1, seeds=P, dis=None, n_dis=0, offs=None, ws=P, nbytes=1 << 30, labels=P, targets=P):
    return lib.frcnn_anchor_targets_batch(P, A, fh, fw, stride, N, ext, halv, info, gt, max_gt, gtc, 0.3, 0.7, batch, num_fg, mode,
                                          seeds, dis, n_dis, offs, labels, targets, P, P, ws, nbytes, None)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N = 0"]),
    (dict(fh=0), ["bad geometry"]),
    (dict(halv=-1), ["halvings"]),
    (dict(halv=31), ["halvings"]),
    (dict(max_gt=0), ["max_gt"]),
    (dict(ext=None), ["extents"]),
    (dict(info=None), ["im_info"]),
    (dict(gtc=None), ["gt_counts"]),
    (dict(labels=None), ["null pointer"]),
    (dict(mode=3), ["subsample_mode"]),
    (dict(mode=1, seeds=None), ["seeds"]),
    (dict(mode=1, num_fg=300), ["num_fg"]),
    (dict(mode=2, offs=None), ["mode 2"]),
    (dict(mode=2, offs=P, n_dis=4, dis=None), ["mode 2"]),
    (dict(targets=P_ODD), ["16-byte"]),
    (dict(fh=40000, fw=40000), ["too many"]),
])
def test_anchor_targets_batch_argument_errors(lib, kw, words):
    _fail(_targets(lib, **kw), ERR_ARG, ["anchor_targets_batch"] + words)


def test_anchor_targets_batch_workspace_errors(lib):
    _fail(_targets(lib, ws=None), ERR_WS, ["no workspace"])
    _fail(_targets(lib, nbytes=100), ERR_WS, ["workspace"])


def _loss(lib, N=2, ld=64, A=9, fh=38, fw=63, ext=P, halv=4, info=P, head=P, delta=3.0, ws=P, nbytes=1 << 30, targets=P):
    return lib.frcnn_rpn_loss_batch(head, ld, P, A, fh, fw, 16, N, ext, halv, info, P, targets, P, delta, 1.0, 1.0, P, P, ws,
                                    nbytes, None)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N = 0"]),
    (dict(fw=0), ["bad geometry"]),
    (dict(ld=53), ["ld"]),
    (dict(halv=31), ["halvings"]),
    (dict(ext=None), ["extents"]),
    (dict(info=None), ["im_info"]),
    (dict(head=None), ["null pointer"]),
    (dict(targets=P_ODD), ["16-byte"]),
    (dict(delta=0.0), ["delta"]),
])
def test_rpn_loss_batch_argument_errors(lib, kw, words):
    _fail(_loss(lib, **kw), ERR_ARG, ["rpn_loss_batch"] + words)


def test_rpn_loss_batch_workspace_errors(lib):
    _fail(_loss(lib, ws=None), ERR_WS, ["no workspace"])
    _fail(_loss(lib, nbytes=8), ERR_WS, ["workspace"])


def _prep(lib, g=P, g32=None, ld=0, y=P, p=None, N=2, H=38, W=63, C=512, o=P, t=P, planes=1, times2=0):
    return lib.frcnn_grad_prepare_batch(g, None, g32, ld, y, None, p, None, N, H, W, C, o, None, t, None, planes, times2, None)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N = 0"]),
    (dict(C=12), ["bad shape"]),
    (dict(g=None), ["bf16 planes OR fp32"]),
    (dict(g32=P), ["bf16 planes OR fp32"]),
    (dict(g=None, g32=P, ld=0), ["fp32 source"]),
    (dict(y=None, p=P), ["pooled routing"]),
    (dict(planes=2), ["planes"]),
    (dict(o=None, t=None), ["no output"]),
    (dict(g=None, g32=P, ld=64, times2=1), ["times2"]),
    (dict(N=300, C=512 * 64), ["one launch"]),
])
def test_grad_prepare_batch_argument_errors(lib, kw, words):
    _fail(_prep(lib, **kw), ERR_ARG, ["grad_prepare_batch"] + words)
