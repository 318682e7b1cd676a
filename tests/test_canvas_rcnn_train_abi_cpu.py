"""CPU tests of the canvas RCNN-training entries (frcnn_proposal_targets_batch, frcnn_rcnn_loss_batch,
frcnn_roi_pool_backward_batch_ext, frcnn_dropout_masks_batch): they are exported with their declared signatures and
reject every bad argument with FRCNN_ERR_ARG (or FRCNN_ERR_WORKSPACE for a missing or short workspace) and a message,
before anything touches the device.  CanvasRcnnTrainer rejects bad options before it allocates anything, and put()
rejects what does not fit before it stages anything.  The pointers
are fake and never dereferenced."""
import ctypes

import pytest

from test_train_targets_abi_cpu import P, P_ODD, _fail, _params

ERR_ARG, ERR_WS = -1, -3
NAMES = ("frcnn_proposal_targets_batch", "frcnn_rcnn_loss_batch", "frcnn_roi_pool_backward_batch_workspace_bytes",
         "frcnn_roi_pool_backward_batch_ext", "frcnn_dropout_masks_batch")


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def test_declared_signatures(lib):
    from frcnn_b200 import _lib
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long, "double": ctypes.c_double, "float": ctypes.c_float,
             "size_t": ctypes.c_size_t, "unsigned long long": ctypes.c_ulonglong}
    for name in NAMES:
        params = _params(name)
        res, args = _lib.SIGNATURES[name]
        assert getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0].replace("const ", "")
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
        assert res is (ctypes.c_size_t if name.endswith("_workspace_bytes") else ctypes.c_int), name


def test_workspace_sizes(lib):
    one = lib.frcnn_roi_pool_backward_workspace_bytes(38, 63, 512)
    assert lib.frcnn_roi_pool_backward_batch_workspace_bytes(1, 38, 63, 512) == one
    assert lib.frcnn_roi_pool_backward_batch_workspace_bytes(4, 38, 63, 512) == 4 * one
    assert lib.frcnn_roi_pool_backward_batch_workspace_bytes(0, 38, 63, 512) == 0


def _targets(lib, N=2, rois=P, rs=1200, counts=P, cs=2, R_cap=300, gt=P, max_gt=8, gtc=P, nc=21, mode=1, seeds=P, klist=None,
             n_list=0, offs=None, keep=P):
    return lib.frcnn_proposal_targets_batch(N, rois, rs, counts, cs, R_cap, gt, max_gt, gtc, nc, mode, seeds, klist, n_list, offs,
                                            keep, P, P, P, P, P, P, None)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N = 0"]),
    (dict(R_cap=0), ["R_cap"]),
    (dict(R_cap=4097), ["R_cap", "4096"]),
    (dict(N=65536), ["N = 65536"]),
    (dict(max_gt=0), ["max_gt"]),
    (dict(N=65535, max_gt=1 << 16), ["N * max_gt"]),
    (dict(nc=0), ["num_classes"]),
    (dict(nc=4097), ["num_classes = 4097"]),
    (dict(rois=None), ["null pointer"]),
    (dict(gtc=None), ["null pointer"]),
    (dict(keep=None), ["null pointer"]),
    (dict(rois=P_ODD), ["16-byte"]),
    (dict(rs=1199), ["rois image stride"]),
    (dict(rs=1202), ["rois image stride"]),
    (dict(cs=-1), ["count image stride"]),
    (dict(mode=0), ["mode 0"]),
    (dict(mode=3), ["mode 3"]),
    (dict(seeds=None), ["seeds"]),
    (dict(mode=2, offs=None), ["mode 2"]),
    (dict(mode=2, offs=P, n_list=4), ["mode 2"]),
    (dict(mode=2, offs=P, n_list=-1), ["mode 2"]),
])
def test_proposal_targets_batch_errors(lib, kw, words):
    _fail(_targets(lib, **kw), ERR_ARG, ["proposal_targets_batch"] + words)


def test_proposal_targets_batch_one_slot_needs_no_stride(lib):
    from frcnn_b200 import _lib
    assert _targets(lib, N=1, rs=0, mode=0) == ERR_ARG and "mode 0" in _lib.last_error()


def _loss(lib, N=2, head=P, ld=128, R_cap=300, keep=P, counts=P, nc=21, delta=1.0, losses=P):
    return lib.frcnn_rcnn_loss_batch(N, head, ld, R_cap, keep, P, P, counts, nc, delta, 1.0, losses, None, None)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N = 0"]),
    (dict(N=65536), ["N = 65536"]),
    (dict(head=None), ["null pointer"]),
    (dict(keep=None), ["null pointer"]),
    (dict(counts=None), ["null pointer"]),
    (dict(losses=None), ["null pointer"]),
    (dict(R_cap=0), ["bad shape"]),
    (dict(nc=0), ["bad shape"]),
    (dict(ld=104), ["bad shape"]),
    (dict(delta=0.0), ["delta"]),
])
def test_rcnn_loss_batch_errors(lib, kw, words):
    _fail(_loss(lib, **kw), ERR_ARG, ["rcnn_loss_batch"] + words)


def _pool_bwd(lib, N=2, H=38, W=63, C=512, feat=P, rois=P, rs=1200, counts=P, cs=2, R_cap=300, oh=7, ow=7, ext=P, halv=4, g=P,
              dfeat=P, ws=P, nbytes=1 << 40):
    return lib.frcnn_roi_pool_backward_batch_ext(feat, None, N, H, W, C, rois, rs, counts, cs, R_cap, oh, ow, 0.0625, ext, halv, g,
                                                 None, dfeat, ws, nbytes, None)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N = 0"]),
    (dict(H=0), ["bad shape"]),
    (dict(C=12), ["bad shape"]),
    (dict(R_cap=0), ["bad shape"]),
    (dict(oh=0), ["bad shape"]),
    (dict(halv=-1), ["halvings"]),
    (dict(halv=31), ["halvings"]),
    (dict(feat=None), ["null pointer"]),
    (dict(ext=None), ["null pointer"]),
    (dict(dfeat=None), ["null pointer"]),
    (dict(rs=1196), ["rois image stride"]),
    (dict(rs=1201), ["rois image stride"]),
    (dict(cs=-2), ["count image stride"]),
])
def test_roi_pool_backward_batch_errors(lib, kw, words):
    _fail(_pool_bwd(lib, **kw), ERR_ARG, ["roi_pool_backward_batch_ext"] + words)


@pytest.mark.parametrize("kw", [dict(ws=None), dict(nbytes=2 * 38 * 63 * 512 * 8 - 1)])
def test_roi_pool_backward_batch_workspace(lib, kw):
    _fail(_pool_bwd(lib, **kw), ERR_WS, ["roi_pool_backward_batch_ext", "workspace"])


@pytest.mark.parametrize("args,words", [
    ((0, 300, 4096, P, 1, P), ["N = 0"]),
    ((65536, 300, 4096, P, 1, P), ["N = 65536"]),
    ((2, 0, 4096, P, 1, P), ["bad shape"]),
    ((2, 300, 0, P, 1, P), ["bad shape"]),
    ((2, 1 << 16, 1 << 15, P, 1, P), ["bad shape"]),
    ((2, 300, 4096, None, 1, P), ["null pointer"]),
    ((2, 300, 4096, P, 1, None), ["null pointer"]),
])
def test_dropout_masks_batch_errors(lib, args, words):
    _fail(lib.frcnn_dropout_masks_batch(*args, None), ERR_ARG, ["dropout_masks_batch"] + words)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N >= 1"]),
    (dict(N=1.5), ["N >= 1"]),
    (dict(sample="numpy"), ["sample must be one of"]),
    (dict(dropout=True), ["dropout must be one of"]),
    (dict(max_gt=0), ["max_gt"]),
    (dict(post_n=0), ["post_n"]),
    (dict(post_n=4097), ["post_n"]),
])
def test_trainer_options_are_checked_first(kw, words):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.train_engine import CanvasRcnnTrainer
    args = dict(params=None, N=2, Hc=64, Wc=64, anchors=None, device="cpu")
    args.update(kw)
    with pytest.raises(FrcnnError) as e:
        CanvasRcnnTrainer(**args)
    assert all(w in str(e.value) for w in words), str(e.value)


class _Recorder(object):
    """Stands in for the trainer's ImageInput: records whether put() reached the staging step."""

    def __init__(self):
        self.calls = 0

    def put(self, images, img_infos):
        self.calls += 1
        raise AssertionError("put() staged images although it should have refused the call")


def _bare_trainer(sample="list", dropout="explicit", N=2, max_gt=4, post_n=8):
    """A CanvasRcnnTrainer with only the attributes put() reads before it stages anything (no device, no weights)."""
    from frcnn_b200.train_engine import CanvasRcnnTrainer
    t = CanvasRcnnTrainer.__new__(CanvasRcnnTrainer)
    t.N, t.max_gt, t.post_n, t.sample, t.dropout, t.device = N, max_gt, post_n, sample, dropout, "cpu"
    t.input = _Recorder()
    return t


def _put_args(n=2, G=2, keep=None, masks=None):
    import torch
    images = [torch.zeros((3, 32, 32)) for _ in range(n)]
    gts = [torch.zeros((G, 5)) for _ in range(n)]
    return images, gts, keep, masks


def _mask_pair(rows=8, dtype=None):
    import torch
    return (torch.zeros((rows, 4096), dtype=dtype or torch.uint8), torch.zeros((rows, 4096), dtype=dtype or torch.uint8))


def _put_cases():
    import torch
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)        # noqa: E731
    ok_keep = [i32([0, 1]), i32([2])]
    return [
        ("gt count", dict(), lambda: (_put_args()[0], _put_args(n=1)[1], None, None), ["2 images and 1 ground-truth lists"]),
        ("gt columns", dict(), lambda: (_put_args()[0], [torch.zeros((2, 4))] * 2, None, None), ["ground truth of shape (2, 4)"]),
        ("no gt", dict(), lambda: _put_args(G=0), ["ground truth of shape (0, 5)", "1 <= G <= 4"]),
        ("too much gt", dict(), lambda: _put_args(G=5), ["ground truth of shape (5, 5)", "1 <= G <= 4"]),
        ("keep without list mode", dict(sample="device"), lambda: _put_args(keep=ok_keep), ["kept lists need sample='list'"]),
        ("keep count", dict(), lambda: _put_args(keep=ok_keep[:1]), ["2 images and 1 kept lists"]),
        ("keep too long", dict(), lambda: _put_args(keep=[torch.arange(129), ok_keep[1]]), ["image 0 keeps 129 rows, at most 128"]),
        ("keep repeats", dict(), lambda: _put_args(keep=[ok_keep[0], i32([3, 5, 3])]), ["image 1's kept list repeats a row"]),
        ("masks without explicit", dict(dropout="device"), lambda: _put_args(masks=[_mask_pair()] * 2),
         ["masks need dropout='explicit'"]),
        ("masks and no dropout", dict(dropout=None), lambda: _put_args(masks=[_mask_pair()] * 2), ["masks need dropout='explicit'"]),
        ("mask count", dict(), lambda: _put_args(masks=[_mask_pair()]), ["2 images and 1 mask pairs"]),
        ("mask rows", dict(), lambda: _put_args(masks=[_mask_pair(), _mask_pair(rows=7)]), ["image 1 needs two uint8 (8, 4096) masks"]),
        ("mask dtype", dict(), lambda: _put_args(masks=[_mask_pair(dtype=torch.bool), _mask_pair()]),
         ["image 0 needs two uint8 (8, 4096) masks"]),
        ("one mask", dict(), lambda: _put_args(masks=[_mask_pair()[:1], _mask_pair()]), ["image 0 needs two uint8 (8, 4096) masks"]),
    ]


@pytest.mark.parametrize("case", range(14))
def test_put_refuses_before_staging(case):
    from frcnn_b200._lib import FrcnnError
    name, kw, make, words = _put_cases()[case]
    t = _bare_trainer(**kw)
    images, gts, keep, masks = make()
    with pytest.raises(FrcnnError) as e:
        t.put(images, gts, keep_inds=keep, masks=masks)
    assert "CanvasRcnnTrainer.put" in str(e.value) and all(w in str(e.value) for w in words), (name, str(e.value))
    assert t.input.calls == 0, name
