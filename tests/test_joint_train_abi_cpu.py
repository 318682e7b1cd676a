"""The joint training step (JointTrainer, CanvasJointTrainer, ResNetJointTrainer, CanvasResNetJointTrainer) on a CPU-only
box, through the launch recorder of test_trainer_launches_cpu: nothing reaches a device.

Checked here:
- every joint trainer checks each parameter it reads, RPN ones included, and its options before it allocates;
- the flat layout is the union of the RPN and RCNN trainers' entries, trunk first, and export_params / optimizer_state
  round-trip;
- the forward is the RCNN trainer's trunk, one RPN forward on the trained planes, the RPN trainer's target and loss
  launches, then the RCNN trainer's proposal, target, pool, head and loss launches;
- the backward is the RCNN trainer's head and RoI launches, the RPN trainer's head and RPN-conv weight-gradient launches,
  one frcnn_conv2d_res(_batch_ext) whose residual is the split dfeat and whose output is another buffer, then the trunk;
- the one-image and the N = 1 canvas backward match entry for entry; update() repacks in place; the canvas step advances
  its seeds once and hands the same seeds to both halves' draws."""
import functools

import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import test_trainer_launches_cpu as launches
from test_trainer_launches_cpu import ANCHORS, POST_N, H, W, _forward, _planes, _warm, rec  # noqa: F401

R50 = dict(n_layers=50)


@functools.lru_cache(maxsize=None)
def _params(trunk):
    return orc.make_params(seed=5) if trunk == "vgg" else orc.make_resnet_params(50, seed=3)


def _vgg_params():
    return dict(_params("vgg"))          # a test may replace or drop entries, never change an array


def _r50_params():
    return dict(_params("r50"))


def _joint(params, **kw):
    from frcnn_b200.train_engine import JointTrainer
    return JointTrainer(params, H, W, ANCHORS, **dict(dict(post_n=POST_N, device="cpu"), **kw))


def _canvas_joint(params, N=1, **kw):
    from frcnn_b200.train_engine import CanvasJointTrainer
    return CanvasJointTrainer(params, N, H, W, ANCHORS, **dict(dict(post_n=POST_N, device="cpu"), **kw))


def _resnet_joint(params, **kw):
    from frcnn_b200.resnet_train import ResNetJointTrainer
    return ResNetJointTrainer(params, H, W, ANCHORS, **dict(dict(R50, post_n=POST_N, device="cpu"), **kw))


def _canvas_resnet_joint(params, N=1, **kw):
    from frcnn_b200.resnet_train import CanvasResNetJointTrainer
    return CanvasResNetJointTrainer(params, N, H, W, ANCHORS, **dict(dict(R50, post_n=POST_N, device="cpu"), **kw))


def _components(kind, params):
    """The RPN and RCNN trainers the joint trainer of `kind` is made of, on the same parameters."""
    from frcnn_b200 import resnet_train as rt
    from frcnn_b200 import train_engine as te
    if kind == "vgg":
        return (te.RpnTrainer(params, H, W, ANCHORS, device="cpu"),
                te.RcnnTrainer(params, H, W, ANCHORS, post_n=POST_N, device="cpu"))
    if kind == "canvas":
        return (te.CanvasRpnTrainer(params, 1, H, W, ANCHORS, device="cpu"),
                te.CanvasRcnnTrainer(params, 1, H, W, ANCHORS, post_n=POST_N, sample="list", dropout="explicit", device="cpu"))
    if kind == "resnet":
        return (rt.ResNetRpnTrainer(params, H, W, ANCHORS, device="cpu", **R50),
                rt.ResNetRcnnTrainer(params, H, W, ANCHORS, post_n=POST_N, device="cpu", **R50))
    return (rt.CanvasResNetRpnTrainer(params, 1, H, W, ANCHORS, device="cpu", **R50),
            rt.CanvasResNetRcnnTrainer(params, 1, H, W, ANCHORS, post_n=POST_N, sample="list", dropout="explicit",
                                       device="cpu", **R50))


MAKE = dict(vgg=_joint, canvas=lambda p: _canvas_joint(p, sample="list", dropout="explicit"), resnet=_resnet_joint,
            canvas_resnet=lambda p: _canvas_resnet_joint(p, sample="list", dropout="explicit"))
PARAMS = dict(vgg=_vgg_params, canvas=_vgg_params, resnet=_r50_params, canvas_resnet=_r50_params)


def _bare(calls):
    """Entries with every pointer as "p": the launch sequence and its scalar arguments."""
    return [[c[0]] + ["p" if isinstance(a, str) else a for a in c[1:]] for c in calls]


def _trace(rec, fn):
    rec.reset()
    fn()
    return list(rec.calls)


def _ptr(rec, t):
    """The recorder's name of tensor t's storage (None when the trace never used it)."""
    n = rec._ptrs.get(t.data_ptr())
    return None if n is None else "p%d" % n


# ------------------------------------------------------------------------------------------------ parameters and options
@pytest.mark.parametrize("kind,name,shape", [
    ("vgg", "RPN/rpn_cls_score/W", None),
    ("vgg", "RPN/rpn_conv_3x3/b", None),
    ("vgg", "fc6/W", (4096, 2048 * 49)),
    ("vgg", "trunk/conv5_3/b", (256,)),
    ("canvas", "RPN/rpn_bbox_pred/b", None),
    ("canvas", "cls_score/b", None),
    ("resnet", "RPN/rpn_conv_3x3/W", (512, 512, 3, 3)),
    ("resnet", "bbox_pred/W", None),
    ("canvas_resnet", "RPN/rpn_cls_score/b", None),
    ("canvas_resnet", "trunk/res5/a/bn1/gamma", None),
])
def test_parameters_are_checked_first(monkeypatch, kind, name, shape):
    from frcnn_b200 import train_engine
    from frcnn_b200._lib import FrcnnError

    def alloc(*a, **k):
        raise AssertionError("the trainer allocated its buffers before it rejected the parameters")
    monkeypatch.setattr(train_engine._ConvTrainer, "_init_params", alloc)
    params = PARAMS[kind]()
    if shape is None:
        del params[name]
    else:
        params[name] = np.zeros(shape, np.float32)
    with pytest.raises(FrcnnError) as e:
        MAKE[kind](params)
    assert "parameter %s must have shape" % name in str(e.value), str(e.value)


@pytest.mark.parametrize("kind,kw", [
    ("vgg", dict(subsample="list")), ("vgg", dict(sample="device")), ("vgg", dict(dropout="device")), ("vgg", dict(post_n=0)),
    ("canvas", dict(subsample="numpy")), ("canvas", dict(sample="numpy")), ("canvas", dict(dropout=True)),
    ("canvas", dict(post_n=4097)), ("canvas", dict(augment="host")), ("canvas", dict(augment="device")),
    ("resnet", dict(subsample="bad")), ("resnet", dict(post_n=-1)),
    ("canvas_resnet", dict(sample="bad")), ("canvas_resnet", dict(augment="list", raw_input=False)),
])
def test_bad_options_raise_before_allocation(monkeypatch, kind, kw):
    from frcnn_b200 import train_engine
    from frcnn_b200._lib import FrcnnError

    def alloc(*a, **k):
        raise AssertionError("the trainer allocated its buffers before it rejected an option")
    monkeypatch.setattr(train_engine._ConvTrainer, "_init_params", alloc)
    make = dict(vgg=_joint, canvas=_canvas_joint, resnet=_resnet_joint, canvas_resnet=_canvas_resnet_joint)[kind]
    with pytest.raises(FrcnnError):
        make(PARAMS[kind](), **kw)


# ------------------------------------------------------------------------------------------------ layout and state
@pytest.mark.parametrize("kind", ["vgg", "canvas", "resnet", "canvas_resnet"])
def test_layout_is_the_union_trunk_first(rec, kind):
    params = PARAMS[kind]()
    tr = MAKE[kind](params)
    rpn, rcnn = _components(kind, params)
    assert set(tr.index) == set(rpn.index) | set(rcnn.index)
    for n, (o, sz, shape) in tr.index.items():
        assert shape == (rpn.index.get(n) or rcnn.index[n])[2], n
    order = sorted(tr.index, key=lambda n: tr.index[n][0])
    first_step = min(i for i, n in enumerate(order) if not n.startswith("trunk/"))
    assert all(not n.startswith("trunk/") for n in order[first_step:])
    step = [n.rsplit("/", 1)[0] for n in order[first_step:]]
    assert step[:2] == ["RPN/rpn_conv_3x3"] * 2
    assert step[-4:] == ["RPN/rpn_cls_score", "RPN/rpn_bbox_pred"] * 2          # twin heads adjacent: W, W, b, b
    assert not any(s.startswith("RPN/") for s in step[2:-4])
    if kind in ("vgg", "canvas"):
        assert tr.index["trunk/conv4_1/W"][0] < tr.index[order[first_step]][0]   # the early exchange covers only the step


@pytest.mark.parametrize("kind", ["vgg", "resnet"])
def test_export_and_optimizer_state_round_trip(rec, kind):
    params = PARAMS[kind]()
    tr = MAKE[kind](params)
    g = torch.Generator().manual_seed(0)
    tr.w_flat.copy_(torch.randn(tr.w_flat.shape, generator=g))
    tr.opt_state["v"].copy_(torch.randn(tr.w_flat.shape, generator=g))
    tr.opt_t = 7
    exported, state = tr.export_params(), tr.optimizer_state()
    back = MAKE[kind](dict(params, **exported))
    assert torch.equal(back.w_flat, tr.w_flat)
    back.load_optimizer_state(state)
    assert torch.equal(back.opt_state["v"], tr.opt_state["v"]) and back.opt_t == 7
    assert set(exported) >= set(tr.index)
    if kind == "resnet":                            # a whole detector: the frozen BN constants too
        assert set(exported) == set(tr.index) | set(tr.bn_params)


@pytest.mark.parametrize("kind", ["vgg", "resnet"])
def test_export_is_a_whole_detector(rec, kind):
    """export_params() holds every parameter the detector has (oracle.make_params / make_resnet_params), in its shape."""
    params = PARAMS[kind]()
    got = MAKE[kind](params).export_params()
    assert set(got) == set(params)
    assert all(got[n].shape == np.shape(params[n]) for n in params)


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("kind", ["vgg", "canvas", "resnet", "canvas_resnet"])
def test_forward_is_the_two_steps_on_one_rpn(rec, kind):
    params = PARAMS[kind]()
    tr = MAKE[kind](params)
    rpn, rcnn = _components(kind, params)
    traces = {}
    for name, t in (("joint", tr), ("rpn", rpn), ("rcnn", rcnn)):
        _warm(t)
        traces[name] = _trace(rec, lambda t=t: _forward(t))
        n_trunk = len(_trace(rec, (lambda t=t: t._forward_trunk()) if kind.startswith("canvas") else
                             (lambda t=t: t._forward_trunk(torch.zeros((3, H, W))))))
        traces[name + "_trunk"] = n_trunk
    n = traces["rcnn_trunk"]
    assert traces["rpn_trunk"] == n == traces["joint_trunk"]
    joint, rpn_f, rcnn_f = traces["joint"], traces["rpn"], traces["rcnn"]
    want = rcnn_f[:n] + rpn_f[n:] + rcnn_f[n + 2:]          # rcnn_f[n:n+2]: the frozen RPN's conv and heads
    assert _bare(joint) == _bare(want)
    # the one RPN forward runs on the trained planes, and the proposals read its output
    _trace(rec, lambda: _forward(tr))
    R = tr.rpn_layer
    conv, heads = joint[n], joint[n + 1]
    assert conv[7 if kind.startswith("canvas") else 6] == _ptr(rec, tr.packed[R["name"]][0][0])
    assert heads[7 if kind.startswith("canvas") else 6] == _ptr(rec, tr.packed["RPN/heads"][0][0])
    props = [c for c in joint if c[0].startswith("frcnn_proposals")]
    assert len(props) == 1 and _ptr(rec, tr.rpn.head_out) in props[0][1:]
    assert sum(c[0].startswith("frcnn_conv2d") for c in joint[n:n + 2]) == 2


# ------------------------------------------------------------------------------------------------ backward
@pytest.mark.parametrize("kind", ["vgg", "canvas", "resnet", "canvas_resnet"])
def test_backward_joins_the_two_gradients_in_the_rpn_conv(rec, kind):
    from frcnn_b200.train_engine import JOIN_TAG
    params = PARAMS[kind]()
    tr = MAKE[kind](params)
    rpn, rcnn = _components(kind, params)
    bwd = {}
    for name, t in (("joint", tr), ("rpn", rpn), ("rcnn", rcnn)):
        _warm(t)
        _forward(t)
        bwd[name] = _trace(rec, t.backward)
    rcnn_b, rpn_b, joint = bwd["rcnn"], bwd["rpn"], bwd["joint"]
    pool_bwd = max(i for i, c in enumerate(rcnn_b) if c[0].startswith("frcnn_roi_pool_backward"))
    n_head = pool_bwd + 2                          # the RoI pooling backward, then the split of dfeat
    n_trunk = len(rcnn_b) - n_head
    rpn_part = rpn_b[:len(rpn_b) - n_trunk]
    assert _bare(rpn_b[len(rpn_b) - n_trunk:]) == _bare(rcnn_b[n_head:])          # the same trunk in both
    res = "frcnn_conv2d_res_batch_ext" if kind.startswith("canvas") else "frcnn_conv2d_res"
    join = n_head + len(rpn_part) - 1
    assert _bare(joint[:join]) == _bare(rcnn_b[:n_head] + rpn_part[:-1])
    assert joint[join][0] == res and rpn_part[-1][0] == res.replace("_res", "")
    assert _bare(joint[join + 1:]) == _bare(rcnn_b[n_head:])
    # the residual is the split dfeat (the output of the step's split), the output another buffer the trunk reads
    off = 1 if kind.startswith("canvas") else 0
    split = joint[n_head - 1]
    assert split[0].startswith("frcnn_grad_prepare")
    _trace(rec, tr.backward)                        # name the buffers in a fresh numbering
    fh, fw, C = tr.fh, tr.fw, tr.feat_ch
    dfeat, joined = tr._acts[(fh, fw, C, 3)], tr._acts[(fh, fw, C, JOIN_TAG)]
    call = rec.calls[join]
    res_hi, y_hi = call[12 + off], call[14 + off]
    assert res_hi == _ptr(rec, dfeat.hi) and y_hi == _ptr(rec, joined.hi)
    assert res_hi != y_hi
    assert rec.calls[join + 1][1:].count(y_hi) >= 1        # the trunk starts from the joined gradient


def test_backward_is_the_canvas_backward(rec, monkeypatch):
    monkeypatch.setitem(launches.TWINS, "frcnn_conv2d_res_batch_ext", ("frcnn_conv2d_res", (2, 16, 17)))
    params = _vgg_params()
    one = launches._backward_trace(rec, _joint(params))
    canvas = launches._backward_trace(rec, _canvas_joint(params, 1, sample="list", dropout="explicit"))
    assert len(one) > 80
    assert one == canvas


@pytest.mark.parametrize("kind", ["vgg", "canvas", "resnet"])
def test_update_repacks_in_place(rec, kind):
    tr = MAKE[kind](PARAMS[kind]())
    before = _planes(tr)
    assert ("RPN/heads", "fwd.hi") in before and ("heads", "fwd.hi") in before
    tr.update()
    assert _planes(tr) == before


def test_each_joint_trainer_has_one_trunk():
    from frcnn_b200 import resnet_train, train_engine
    trunks = (train_engine._Vgg16Trunk, resnet_train._ResNetTrunk)
    for cls, trunk in ((train_engine.JointTrainer, trunks[0]), (train_engine.CanvasJointTrainer, trunks[0]),
                       (resnet_train.ResNetJointTrainer, trunks[1]), (resnet_train.CanvasResNetJointTrainer, trunks[1])):
        assert [t for t in trunks if t in cls.__mro__] == [trunk], cls.__name__
        assert issubclass(cls, train_engine._JointStep)


# ------------------------------------------------------------------------------------------------ draws
def test_canvas_step_advances_the_seeds_once(rec):
    tr = _canvas_joint(_vgg_params(), 3, seed=11)
    assert tr.seeds.tolist() == [11, 12, 13]
    calls = _trace(rec, lambda: _forward(tr))
    assert tr.seeds.tolist() == [14, 15, 16]
    seeds = _ptr(rec, tr.seeds)
    draws = [c[0] for c in calls if seeds in c[1:]]
    assert draws == ["frcnn_anchor_targets_batch", "frcnn_proposal_targets_batch"] + ["frcnn_dropout_masks_batch"] * 2


def test_canvas_losses_are_both_steps(rec):
    tr = _canvas_joint(_vgg_params(), 2)
    _forward(tr)
    tr.rpn.targets.losses.copy_(torch.arange(8.0).view(2, 4))
    tr.ptargets.losses.copy_(torch.arange(8.0).view(2, 4) + 10)
    assert tr.step_losses.tolist() == [[0, 1, 2, 3, 10, 11, 12, 13], [4, 5, 6, 7, 14, 15, 16, 17]]


def test_pins_are_checked(rec):
    from frcnn_b200._lib import FrcnnError
    x, gt = launches._image_and_gt()
    keep, masks = launches._keep_and_masks()
    tr = _canvas_joint(_vgg_params(), 2)
    for kw in (dict(disable_pos=[torch.zeros(1, dtype=torch.int32)]), dict(keep_inds=[keep]), dict(masks=[masks])):
        with pytest.raises(FrcnnError):
            tr.put([x], [gt], **kw)
    tr = _canvas_joint(_vgg_params(), 2, subsample="list", sample="list", dropout="explicit")
    tr.put([x], [gt], disable_pos=[torch.arange(3, dtype=torch.int32)], keep_inds=[keep], masks=[masks])
    assert tr.disable_offsets.tolist() == [0, 3, 3] and tr.keep_offsets.tolist() == [0, keep.numel(), keep.numel()]
