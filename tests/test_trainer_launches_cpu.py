"""Launch traces of the training steps on a CPU-only box.

The library is loaded but nothing reaches a device: every entry that takes a stream is recorded as (name, arguments) and
returns 0, with pointer arguments numbered in order of first use, so that a trace also shows which buffers alias which.
Every tensor passed to an entry is kept alive until the recorder is reset, so that no address is reused within a trace.
The pure-host helpers (workspace sizes, element counts, the padded pixel layout, the split-K count) run for real.  The
trainers are built on device="cpu" at a small shape; callers pass the kept lists and masks, so nothing reads a count back.

Checked here:
- the one-image and the N = 1 canvas trainers launch the same backward, entry for entry, once the batch entries are
  mapped to their one-image twins and the N, extents / halvings and m_valid arguments are dropped;
- every trainer repacks its weights in place: `packed` keeps its tensors across update(), which a captured graph and
  any caller holding the planes rely on;
- every public trainer is one trunk and one step, and a VGG16 trainer rejects a missing or misshapen parameter before
  it allocates anything, as a ResNet trainer does.

`python tests/test_trainer_launches_cpu.py out.json` dumps the forward, backward and update traces of every trainer and
mode to JSON, for comparing two builds of the trainers."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    _ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for _p in (os.path.join(_ROOT, "oracle"), os.path.join(_ROOT, "tests"), os.path.join(_ROOT, "chainer-faster-rcnn_b200")):
        sys.path.insert(0, _p)

import frcnn_oracle as orc
from test_train_targets_abi_cpu import _params

ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
H, W = 64, 96
POST_N = 64
HOST_ONLY = ("frcnn_padded_pixels", "frcnn_gemm_nt_splitk_splits")

# batch entry -> (its one-image twin, the argument positions the twin does not have)
TWINS = {"frcnn_conv2d_batch_ext": ("frcnn_conv2d", (2, 17, 18)),
         "frcnn_grad_prepare_batch": ("frcnn_grad_prepare", (8,)),
         "frcnn_roi_pool_backward_batch_ext": ("frcnn_roi_pool_backward", (2, 7, 9, 14, 15))}
ONE_IMAGE_DROP = {"frcnn_conv2d": (16,)}            # m_valid


class Recorder(object):
    """Stands in for the loaded library: records every stream entry and forwards the pure-host helpers."""

    def __init__(self, lib):
        self._lib = lib
        self.calls, self._ptrs, self._alive = [], {}, []
        self._streamed = {}

    def reset(self):
        self.calls, self._ptrs, self._alive = [], {}, []

    def pointer(self, t):
        """ops._p, holding on to the tensor."""
        if t is None:
            return None
        self._alive.append(t)
        return ctypes.c_void_p(t.data_ptr())

    def _arg(self, a):
        if a is None or isinstance(a, ctypes.c_void_p):
            v = None if a is None else a.value
            if v is None:
                return None
            return "p%d" % self._ptrs.setdefault(v, len(self._ptrs))
        if isinstance(a, ctypes._SimpleCData):
            return a.value
        if isinstance(a, (bool, int, float, np.integer, np.floating)):
            return a.item() if isinstance(a, np.generic) else a
        raise TypeError("unexpected argument %r" % (a,))

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name.endswith(("_workspace_bytes", "_elems")) or name in HOST_ONLY:
            return fn
        if name not in self._streamed:
            self._streamed[name] = _params(name)[-1].endswith("stream")
        if not self._streamed[name]:
            raise AssertionError("%s takes no stream: the trace does not expect it" % name)

        def record(*args):
            self.calls.append([name] + [self._arg(a) for a in args])
            return 0
        return record


@pytest.fixture
def rec(monkeypatch):
    from frcnn_b200 import _lib
    r = Recorder(_lib.load())
    _install(monkeypatch.setattr, r)
    return r


def _install(setattr_, r):
    from frcnn_b200 import _lib, ops, resnet_train, train_ops
    setattr_(_lib, "_lib", r)
    for m in (ops, train_ops):
        setattr_(m, "_p", r.pointer)
        setattr_(m, "_stream", lambda: None)
        setattr_(m, "_need_cuda", lambda *ts: None)
    setattr_(resnet_train._ResNetTrunk, "_check_input", lambda self, x, g: None)      # the ResNet trainers take CPU images


def _normalised(calls, names=None):
    """Batch entries as their one-image twins, without N, extents / halvings and m_valid, pointers renumbered (those in
    `names`, {recorded pointer: name}, named as given)."""
    out, ptrs, names = [], {}, names or {}
    for c in calls:
        name, args = c[0], c[1:]
        name, drop = TWINS.get(name, (name, ONE_IMAGE_DROP.get(name, ())))
        args = [a for i, a in enumerate(args) if i not in drop]
        out.append([name] + [names.get(a) or ptrs.setdefault(a, "p%d" % len(ptrs)) if isinstance(a, str) else a for a in args])
    return out


# ------------------------------------------------------------------------------------------------ inputs
def _vgg_params():
    return orc.make_params(seed=5)


def _image_and_gt():
    x = torch.zeros((3, H, W), dtype=torch.float32)
    gt = torch.tensor([[8.0, 8.0, 40.0, 30.0, 3.0], [50.0, 20.0, 90.0, 60.0, 7.0]], dtype=torch.float32)
    return x, gt


def _keep_and_masks():
    keep = torch.arange(0, 40, 3, dtype=torch.int32)
    g = torch.Generator().manual_seed(1)
    masks = [(torch.rand((POST_N, 4096), generator=g) >= 0.5).to(torch.uint8) for _ in range(2)]
    return keep, masks


def _rpn(params, **kw):
    from frcnn_b200.train_engine import RpnTrainer
    return RpnTrainer(params, H, W, ANCHORS, device="cpu", **kw)


def _rcnn(params):
    from frcnn_b200.train_engine import RcnnTrainer
    return RcnnTrainer(params, H, W, ANCHORS, post_n=POST_N, sample="numpy", dropout=True, device="cpu")


def _canvas_rpn(params, N=1, **kw):
    from frcnn_b200.train_engine import CanvasRpnTrainer
    return CanvasRpnTrainer(params, N, H, W, ANCHORS, device="cpu", **kw)


def _canvas_rcnn(params, N=1, **kw):
    from frcnn_b200.train_engine import CanvasRcnnTrainer
    return CanvasRcnnTrainer(params, N, H, W, ANCHORS, post_n=POST_N, device="cpu", **kw)


def _forward(tr):
    """One forward of any trainer on the fixed inputs (staged first for a canvas trainer)."""
    from frcnn_b200.train_engine import _CanvasSteps
    x, gt = _image_and_gt()
    keep, masks = _keep_and_masks()
    if isinstance(tr, _CanvasSteps):
        n = tr.N
        if not tr.raw_input:
            kw = {}
            if getattr(tr, "subsample", None) == "list":
                kw["disable_pos"] = [torch.arange(0, 20, 7, dtype=torch.int32)] * n
            if getattr(tr, "sample", None) == "list":
                kw["keep_inds"] = [keep] * n
            if getattr(tr, "dropout", None) == "explicit":
                kw["masks"] = [masks] * n
            tr.put([x] * n, [gt] * n, **kw)
        tr.forward()
    elif hasattr(tr, "num_classes"):
        tr.forward(x, gt, keep_inds=keep, masks=masks)
    else:
        tr.forward(x, gt)


# ------------------------------------------------------------------------------------------------ tests
def _warm(tr):
    """One forward + backward: it allocates the trainer's cached buffers and grows the process-wide zero bias that the
    weight-gradient GEMMs read (train_ops._zero_bias), so that a trace after it does not depend on what ran before."""
    _forward(tr)
    tr.backward()


def _backward_trace(rec, tr):
    _warm(tr)
    _forward(tr)
    rec.reset()
    tr.backward()
    return _normalised(rec.calls)


def test_rpn_backward_is_the_canvas_backward(rec):
    params = _vgg_params()
    one = _backward_trace(rec, _rpn(params))
    canvas = _backward_trace(rec, _canvas_rpn(params, 1))
    assert len(one) > 50
    assert one == canvas


def test_rcnn_backward_is_the_canvas_backward(rec):
    params = _vgg_params()
    one = _backward_trace(rec, _rcnn(params))
    canvas = _backward_trace(rec, _canvas_rcnn(params, 1, sample="list", dropout="explicit"))
    assert len(one) > 50
    assert one == canvas


def _planes(tr):
    out = {}
    for name, (fwd, b, dg) in tr.packed.items():
        for tag, t in (("fwd.hi", fwd[0]), ("fwd.lo", fwd[1]), ("b", b), ("dg.hi", dg and dg[0]), ("dg.lo", dg and dg[1])):
            if t is not None:
                out[(name, tag)] = t.data_ptr()
    return out


@pytest.mark.parametrize("kind", ["rpn", "rcnn", "canvas_rpn", "canvas_rcnn", "resnet"])
def test_update_repacks_in_place(rec, kind):
    if kind == "resnet":
        from frcnn_b200.resnet_train import ResNetRpnTrainer
        tr = ResNetRpnTrainer(orc.make_resnet_params(50, seed=3), H, W, ANCHORS, n_layers=50, device="cpu")
    else:
        params = _vgg_params()
        tr = dict(rpn=_rpn, rcnn=_rcnn, canvas_rpn=_canvas_rpn, canvas_rcnn=_canvas_rcnn)[kind](params)
    before = _planes(tr)
    assert len(before) >= 14 * 3
    tr.update()
    assert _planes(tr) == before


def test_each_trainer_has_one_trunk():
    from frcnn_b200 import resnet_train, train_engine
    trunks = (train_engine._Vgg16Trunk, resnet_train._ResNetTrunk)
    for trunk, module, names in ((trunks[0], train_engine, ("RpnTrainer", "RcnnTrainer", "CanvasRpnTrainer", "CanvasRcnnTrainer")),
                                 (trunks[1], resnet_train, ("ResNetRpnTrainer", "ResNetRcnnTrainer", "CanvasResNetRpnTrainer",
                                                            "CanvasResNetRcnnTrainer"))):
        for name in names:
            mro = getattr(module, name).__mro__
            assert [t for t in trunks if t in mro] == [trunk], name


@pytest.mark.parametrize("kind,name,shape", [
    ("rpn", "trunk/conv1_1/W", (64, 27)),                      # the right size: it used to be taken as it came
    ("rpn", "trunk/conv5_3/b", (256,)),
    ("rpn", "RPN/rpn_cls_score/W", None),
    ("canvas_rpn", "RPN/rpn_conv_3x3/b", None),
    ("rcnn", "fc6/W", (4096, 2048 * 49)),
    ("rcnn", "cls_score/b", None),
    ("rcnn", "RPN/rpn_conv_3x3/W", (512, 2048, 3, 3)),        # the frozen RPN the step reads
    ("canvas_rcnn", "fc7/W", (4096 * 4096,)),
])
def test_vgg16_parameters_are_checked_first(monkeypatch, kind, name, shape):
    from frcnn_b200 import train_engine
    from frcnn_b200._lib import FrcnnError

    def alloc(*a, **k):
        raise AssertionError("the trainer allocated its buffers before it rejected the parameters")
    monkeypatch.setattr(train_engine._ConvTrainer, "_init_params", alloc)
    params = _vgg_params()
    if shape is None:
        del params[name]
    else:
        params[name] = np.zeros(shape, np.float32)
    make = dict(rpn=_rpn, rcnn=_rcnn, canvas_rpn=_canvas_rpn, canvas_rcnn=_canvas_rcnn)[kind]
    with pytest.raises(FrcnnError) as e:
        make(params)
    who = dict(rpn="RpnTrainer", rcnn="RcnnTrainer", canvas_rpn="CanvasRpnTrainer", canvas_rcnn="CanvasRcnnTrainer")[kind]
    assert "%s: parameter %s must have shape" % (who, name) in str(e.value), str(e.value)


# ------------------------------------------------------------------------------------------------ the dump
def _cases():
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer, ResNetRcnnTrainer, ResNetRpnTrainer
    vgg, r50 = _vgg_params(), orc.make_resnet_params(50, seed=3)
    canvas = dict(rpn=_canvas_rpn, rcnn=_canvas_rcnn,
                  resnet50_rpn=lambda params, n, **kw: CanvasResNetRpnTrainer(params, n, H, W, ANCHORS, n_layers=50, device="cpu",
                                                                              **kw),
                  resnet50_rcnn=lambda params, n, **kw: CanvasResNetRcnnTrainer(params, n, H, W, ANCHORS, n_layers=50,
                                                                                post_n=POST_N, device="cpu", **kw))
    yield "rpn/device", lambda: _rpn(vgg, subsample="device")
    yield "rpn/none", lambda: _rpn(vgg, subsample="none")
    yield "rcnn", lambda: _rcnn(vgg)
    for trunk, params in (("", vgg), ("resnet50_", r50)):
        rpn, rcnn = canvas[trunk + "rpn"], canvas[trunk + "rcnn"]
        for n in (1, 3):
            for mode in ("device", "list", "none"):
                yield ("%scanvas_rpn/N%d/%s" % (trunk, n, mode),
                       lambda rpn=rpn, p=params, n=n, mode=mode: rpn(p, n, subsample=mode))
            yield "%scanvas_rpn/N%d/raw" % (trunk, n), lambda rpn=rpn, p=params, n=n: rpn(p, n, raw_input=True)
            for sample in ("device", "list"):
                for dropout in ("device", "explicit", None):
                    yield ("%scanvas_rcnn/N%d/%s/%s" % (trunk, n, sample, dropout),
                           lambda rcnn=rcnn, p=params, n=n, s=sample, d=dropout: rcnn(p, n, sample=s, dropout=d))
            yield "%scanvas_rcnn/N%d/raw" % (trunk, n), lambda rcnn=rcnn, p=params, n=n: rcnn(p, n, raw_input=True)
    yield "resnet50", lambda: ResNetRpnTrainer(r50, H, W, ANCHORS, n_layers=50, device="cpu")
    yield "resnet50/none", lambda: ResNetRpnTrainer(r50, H, W, ANCHORS, n_layers=50, subsample="none", device="cpu")
    yield "resnet50_rcnn", lambda: ResNetRcnnTrainer(r50, H, W, ANCHORS, n_layers=50, post_n=POST_N, device="cpu")


def dump(path):
    from frcnn_b200 import _lib
    r = Recorder(_lib.load())
    _install(setattr, r)
    out = {}
    for name, make in _cases():
        tr = make()
        _warm(tr)
        r.reset()
        _forward(tr)
        fwd = r.calls
        r.reset()
        tr.backward()
        bwd = r.calls
        r.reset()
        tr.update()
        out[name] = dict(forward=fwd, backward=bwd, update=r.calls)
        print("%-28s forward %4d  backward %4d  update %4d" % (name, len(fwd), len(bwd), len(r.calls)))
        r.reset()
        del tr
    with open(path, "w") as f:
        json.dump(out, f, indent=0)


if __name__ == "__main__":
    dump(sys.argv[1] if len(sys.argv) > 1 else "trainer_launches.json")
