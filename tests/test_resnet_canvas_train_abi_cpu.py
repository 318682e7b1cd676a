"""CPU tests of the ResNet canvas training step's host side.

- frcnn_maxpool3x3s2_backward_batch and frcnn_grad_prepare_stride2_batch are exported with their declared signatures
  (neither takes times2: the dropout factor has no place in these re-layouts) and reject every bad argument with
  FRCNN_ERR_ARG and a message before anything touches the device (the pointers are fake and never dereferenced);
- CanvasResNetRpnTrainer and CanvasResNetRcnnTrainer reject bad options and parameter shapes before they allocate
  anything, and put() / put_raw() refuse what does not fit before they stage anything;
- on a CPU-only box, with every launch recorded instead of run (test_trainer_launches_cpu.Recorder), the N = 1 canvas
  trainers launch the backward of ResNetRpnTrainer / ResNetRcnnTrainer entry for entry once the batch entries are mapped
  to their one-image twins, and the step's first launch derives the level extents."""
import ctypes

import pytest

from test_train_targets_abi_cpu import P, _fail, _params

ERR_ARG = -1
NAMES = ("frcnn_maxpool3x3s2_backward_batch", "frcnn_grad_prepare_stride2_batch")


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def test_declared_signatures(lib):
    from frcnn_b200 import _lib
    ctype = {"int": ctypes.c_int, "long": ctypes.c_long}
    for name in NAMES:
        params = _params(name)
        res, args = _lib.SIGNATURES[name]
        assert getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0].replace("const ", "")
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
        assert res is ctypes.c_int, name
        assert not any(p.endswith("times2") for p in params), name
        one = _params(name[:-len("_batch")])                       # the one-image entry plus N before H
        assert params == one[:one.index("int H")] + ["int N"] + one[one.index("int H"):], name


def _pool(lib, g=P, y=P, p=P, N=2, H=9, W=7, C=64, o=P, t=P):
    return lib.frcnn_maxpool3x3s2_backward_batch(g, None, y, None, p, None, N, H, W, C, o, None, t, None, None)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N = 0"]),
    (dict(N=-1), ["N = -1"]),
    (dict(N=65535, C=128), ["too many channels or images"]),
    (dict(N=32768, C=256), ["too many channels or images"]),
    (dict(H=1), ["at least 2 x 2", "H=1"]),
    (dict(W=1), ["at least 2 x 2", "W=1"]),
    (dict(C=12), ["bad shape"]),
    (dict(g=None), ["give the source"]),
    (dict(y=None), ["un-pooled forward activation"]),
    (dict(p=None), ["needs the pooled gradient, y and p"]),
    (dict(o=None, t=None), ["no output requested"]),
])
def test_pool_backward_batch_errors(lib, kw, words):
    _fail(_pool(lib, **kw), ERR_ARG, ["maxpool3x3s2_backward_batch"] + words)


def _stride2(lib, g=P, y=P, N=2, H=9, W=7, C=64, o=P, t=P, planes=1):
    return lib.frcnn_grad_prepare_stride2_batch(g, None, y, None, N, H, W, C, o, None, t, None, planes, None)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N = 0"]),
    (dict(N=65535, C=128), ["too many channels or images"]),
    (dict(H=0), ["bad shape"]),
    (dict(C=20), ["bad shape"]),
    (dict(g=None), ["give the source"]),
    (dict(planes=2), ["planes must be 1 or 3"]),
    (dict(o=None, t=None), ["no output requested"]),
])
def test_stride2_batch_errors(lib, kw, words):
    _fail(_stride2(lib, **kw), ERR_ARG, ["grad_prepare_stride2_batch"] + words)


# ------------------------------------------------------------------------------------------------ the trainers
def _anchors():
    import frcnn_oracle as orc
    return orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


@pytest.fixture
def no_alloc(monkeypatch):
    """Makes any allocation of the flat buffers fail the test: an error must come before it."""
    from frcnn_b200 import train_engine

    def alloc(*a, **k):
        raise AssertionError("the trainer allocated its buffers before it rejected the call")
    monkeypatch.setattr(train_engine._ConvTrainer, "_init_params", alloc)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N >= 1"]),
    (dict(N=2.5), ["N >= 1"]),
    (dict(subsample="numpy"), ["subsample must be one of"]),
    (dict(max_gt=0), ["max_gt"]),
    (dict(n_layers=34), ["n_layers must be one of"]),
    (dict(feat_stride=16), ["feature stride is 32"]),
    (dict(Hc=4), ["at least 5 x 5"]),
])
def test_rpn_trainer_options_are_checked_first(no_alloc, kw, words):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.resnet_train import CanvasResNetRpnTrainer
    args = dict(params={}, N=2, Hc=64, Wc=64, anchors=_anchors(), n_layers=50, device="cpu")
    args.update(kw)
    with pytest.raises(FrcnnError) as e:
        CanvasResNetRpnTrainer(**args)
    assert "CanvasResNetRpnTrainer" in str(e.value) and all(w in str(e.value) for w in words), str(e.value)


@pytest.mark.parametrize("kw,words", [
    (dict(N=0), ["N >= 1"]),
    (dict(sample="numpy"), ["sample must be one of"]),
    (dict(dropout=True), ["dropout must be one of"]),
    (dict(max_gt=0), ["max_gt"]),
    (dict(post_n=0), ["post_n"]),
    (dict(post_n=4097), ["post_n"]),
    (dict(n_layers=18), ["n_layers must be one of"]),
    (dict(feat_stride=16), ["feature stride is 32"]),
])
def test_rcnn_trainer_options_are_checked_first(no_alloc, kw, words):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer
    args = dict(params={}, N=2, Hc=64, Wc=64, anchors=_anchors(), n_layers=50, device="cpu")
    args.update(kw)
    with pytest.raises(FrcnnError) as e:
        CanvasResNetRcnnTrainer(**args)
    assert "CanvasResNetRcnnTrainer" in str(e.value) and all(w in str(e.value) for w in words), str(e.value)


def _resnet_params():
    import frcnn_oracle as orc
    return orc.make_resnet_params(50, seed=3)


_SHAPE_CASES = [(kind, name, shape) for kind in ("rpn", "rcnn") for name, shape in (
    ("trunk/conv1/W", (64, 3, 3, 3)),
    ("trunk/res3/a/bn4/avg_var", (256,)),
    ("RPN/rpn_conv_3x3/W", (512, 512, 3, 3)),                      # VGG16's RPN conv
    ("RPN/rpn_cls_score/W", None))] + [("rcnn", "fc6/W", (4096, 512 * 49))]      # VGG16's fc6


@pytest.mark.parametrize("kind,name,shape", _SHAPE_CASES)
def test_parameter_shapes_are_checked_first(no_alloc, kind, name, shape):
    import numpy as np
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer
    params = dict(_resnet_params())
    if shape is None:
        del params[name]
    else:
        params[name] = np.zeros(shape, np.float32)
    cls = CanvasResNetRpnTrainer if kind == "rpn" else CanvasResNetRcnnTrainer
    with pytest.raises(FrcnnError) as e:
        cls(params, 2, 64, 96, _anchors(), n_layers=50, device="cpu")
    assert "parameter %s must have shape" % name in str(e.value), str(e.value)


class _Recorder(object):
    """Stands in for the trainer's input: records whether put() / put_raw() reached the staging step."""

    def __init__(self):
        self.calls = 0

    def put(self, images, img_infos):
        self.calls += 1
        raise AssertionError("put() staged images although it should have refused the call")

    def upload(self, photos, boxes=None, labels=None):
        self.calls += 1
        raise AssertionError("put_raw() staged photos although it should have refused the call")


class _Targets(object):
    cap = 10


def _bare(kind, raw=False, subsample="list", sample="list", dropout="explicit", N=2, max_gt=4, post_n=8):
    """A canvas ResNet trainer with only the attributes put() / put_raw() read before staging (no device, no weights)."""
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer
    cls = CanvasResNetRpnTrainer if kind == "rpn" else CanvasResNetRcnnTrainer
    t = cls.__new__(cls)
    t.N, t.max_gt, t.post_n, t.device, t.raw_input = N, max_gt, post_n, "cpu", raw
    t.subsample, t.sample, t.dropout, t.targets = subsample, sample, dropout, _Targets()
    t.input = _Recorder()
    return t


def _images(n=2, G=2):
    import torch
    return [torch.zeros((3, 32, 32)) for _ in range(n)], [torch.zeros((G, 5)) for _ in range(n)]


def _photos(n=2):
    import numpy as np
    return [np.zeros((40, 50, 3), np.uint8) for _ in range(n)], [np.zeros((1, 4), np.float32)] * n, [np.ones(1, np.int32)] * n


def _put_cases():
    import torch
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)        # noqa: E731
    return [
        ("rpn", dict(), lambda t: t.put(_images()[0], _images(n=1)[1]), "put", ["2 images and 1 ground-truth lists"]),
        ("rpn", dict(), lambda t: t.put(*_images(G=0)), "put", ["ground truth of shape (0, 5)"]),
        ("rpn", dict(), lambda t: t.put(*_images(G=5)), "put", ["1 <= G <= 4"]),
        ("rpn", dict(subsample="device"), lambda t: t.put(*_images(), disable_pos=[i32([1])] * 2), "put",
         ["disable lists need subsample='list'"]),
        ("rpn", dict(), lambda t: t.put(*_images(), disable_pos=[i32([1])]), "put", ["2 images and 1 disable lists"]),
        ("rpn", dict(), lambda t: t.put(*_images(), disable_pos=[torch.arange(11), i32([1])]), "put",
         ["longer than 10 anchors"]),
        ("rpn", dict(raw=True), lambda t: t.put(*_images()), "put", ["raw_input=True", "put_raw"]),
        ("rpn", dict(), lambda t: t.put_raw(*_photos()), "put_raw", ["raw_input=False", "put / step"]),
        ("rpn", dict(raw=True), lambda t: t.put_raw(*_photos(), disable_pos=[i32([1])]), "put_raw",
         ["2 images and 1 disable lists"]),
        ("rcnn", dict(), lambda t: t.put(*_images(), keep_inds=[i32([0])]), "put", ["2 images and 1 kept lists"]),
        ("rcnn", dict(), lambda t: t.put(*_images(), keep_inds=[i32([0, 0]), i32([1])]), "put", ["repeats a row"]),
        ("rcnn", dict(), lambda t: t.put(*_images(), keep_inds=[torch.arange(129), i32([1])]), "put", ["at most 128"]),
        ("rcnn", dict(dropout="device"), lambda t: t.put(*_images(), masks=[(None, None)] * 2), "put",
         ["masks need dropout='explicit'"]),
        ("rcnn", dict(), lambda t: t.put(*_images(), masks=[(torch.zeros((7, 4096), dtype=torch.uint8),) * 2] * 2), "put",
         ["image 0 needs two uint8 (8, 4096) masks"]),
        ("rcnn", dict(raw=True), lambda t: t.put(*_images()), "put", ["raw_input=True"]),
        ("rcnn", dict(raw=True, sample="device"), lambda t: t.put_raw(*_photos(), keep_inds=[i32([0])] * 2), "put_raw",
         ["kept lists need sample='list'"]),
    ]


@pytest.mark.parametrize("case", range(16))
def test_put_refuses_before_staging(case):
    from frcnn_b200._lib import FrcnnError
    kind, kw, call, method, words = _put_cases()[case]
    t = _bare(kind, **kw)
    with pytest.raises(FrcnnError) as e:
        call(t)
    who = "CanvasResNetRpnTrainer" if kind == "rpn" else "CanvasResNetRcnnTrainer"
    assert "%s.%s" % (who, method) in str(e.value) and all(w in str(e.value) for w in words), (case, str(e.value))
    assert t.input.calls == 0, case


# ------------------------------------------------------------------------------------------------ launch traces
@pytest.fixture
def rec(monkeypatch):
    import test_trainer_launches_cpu as tl
    from frcnn_b200 import _lib
    r = tl.Recorder(_lib.load())
    tl._install(monkeypatch.setattr, r)
    twins = dict(tl.TWINS)
    twins.update({"frcnn_conv2d_res_batch_ext": ("frcnn_conv2d_res", (2, 16, 17)),
                  "frcnn_maxpool3x3s2_backward_batch": ("frcnn_maxpool3x3s2_backward", (6,)),
                  "frcnn_grad_prepare_stride2_batch": ("frcnn_grad_prepare_stride2", (4,))})
    monkeypatch.setattr(tl, "TWINS", twins)
    from frcnn_b200 import resnet_train
    monkeypatch.setattr(resnet_train._ResNetTrunk, "_check_input", lambda self, x, g: None)   # CPU images
    return r


@pytest.mark.parametrize("kind", ["rpn", "rcnn"])
def test_n1_canvas_backward_is_the_one_image_backward(rec, kind):
    import test_trainer_launches_cpu as tl
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer, ResNetRcnnTrainer, ResNetRpnTrainer
    params, H, W = _resnet_params(), tl.H, tl.W
    if kind == "rpn":
        one = ResNetRpnTrainer(params, H, W, tl.ANCHORS, n_layers=50, device="cpu")
        canvas = CanvasResNetRpnTrainer(params, 1, H, W, tl.ANCHORS, n_layers=50, device="cpu")
    else:
        one = ResNetRcnnTrainer(params, H, W, tl.ANCHORS, n_layers=50, post_n=tl.POST_N, device="cpu")
        canvas = CanvasResNetRcnnTrainer(params, 1, H, W, tl.ANCHORS, n_layers=50, post_n=tl.POST_N, sample="list",
                                         dropout="explicit", device="cpu")
    a, b = tl._backward_trace(rec, one), tl._backward_trace(rec, canvas)
    assert len(a) > 250
    assert a == b
    names = [c[0] for c in rec.calls]
    assert names.count("frcnn_maxpool3x3s2_backward_batch") == 1 and names.count("frcnn_grad_prepare_stride2_batch") == 3


@pytest.mark.parametrize("raw", [False, True])
def test_canvas_step_starts_with_the_level_extents(rec, raw):
    import test_trainer_launches_cpu as tl
    from frcnn_b200.resnet_train import CanvasResNetRpnTrainer
    tr = CanvasResNetRpnTrainer(_resnet_params(), 3, tl.H, tl.W, tl.ANCHORS, n_layers=50, device="cpu", raw_input=raw)
    tl._warm(tr)
    rec.reset()
    tl._forward(tr)
    names = [c[0] for c in rec.calls]
    first = "frcnn_preprocess_voc_canvas_im2col" if raw else "frcnn_pack_image_im2col_batch_ext"
    assert names[:2] == ["frcnn_resnet_level_extents", first]
    args = rec.calls[1]
    assert any(args[i:i + 4] == [7, 2, 3, 160] for i in range(len(args)))     # conv1's ksize, stride, pad, K_pad
    assert "frcnn_conv2d" not in names and "frcnn_maxpool3x3s2_ceil" not in names     # every launch a batch entry
