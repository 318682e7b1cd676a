"""CPU tests of the RCNN training step with the ResNet trunk (frcnn_b200/resnet_train.py ResNetRcnnTrainer).

- the float64 reference (resnet_rcnn_train_oracle.resnet_rcnn_train_step): its unfolded frozen-BN trunk gradients equal s times
  its folded ones;
- the constructor's checks on device="cpu", every one raised before anything is allocated;
- launch traces against the recording stand-in of test_trainer_launches_cpu: on either trunk, the trunk part of the RCNN
  step's backward is, entry for entry, the RPN step's (ResNetRcnnTrainer's is ResNetRpnTrainer's bottleneck backward,
  RcnnTrainer's is RpnTrainer's 13 convolutions), and update() repacks in place.

fc6 alone is 4096 x 100,352 float32 (1.6 GB), so the trainer is built once, under the recorder, for the whole module."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import resnet_rcnn_train_oracle as rto
from test_trainer_launches_cpu import ANCHORS, POST_N, H, W, Recorder, _forward, _install, _normalised, _planes, _vgg_params

f32 = np.float32


@pytest.fixture(scope="module")
def params():
    return orc.make_resnet_params(50, seed=3)


@pytest.fixture(scope="module")
def recorder():
    from frcnn_b200 import _lib
    r = Recorder(_lib.load())
    with pytest.MonkeyPatch.context() as mp:
        _install(mp.setattr, r)
        yield r


def _warmed(rcnn, rpn):
    for tr in (rcnn, rpn):
        _forward(tr)
        tr.backward()
    return rcnn, rpn


@pytest.fixture(scope="module")
def recorded(recorder, params):
    """(recorder, ResNetRcnnTrainer, ResNetRpnTrainer) at 64 x 96, ResNet-50, built and warmed up under the recorder."""
    from frcnn_b200.resnet_train import ResNetRcnnTrainer, ResNetRpnTrainer
    return (recorder,) + _warmed(ResNetRcnnTrainer(params, H, W, ANCHORS, n_layers=50, post_n=POST_N, device="cpu"),
                                 ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50, device="cpu"))


@pytest.fixture(scope="module")
def recorded_vgg16(recorder):
    """(recorder, RcnnTrainer, RpnTrainer) at 64 x 96, built and warmed up under the recorder."""
    from frcnn_b200.train_engine import RcnnTrainer, RpnTrainer
    vgg = _vgg_params()
    return (recorder,) + _warmed(RcnnTrainer(vgg, H, W, ANCHORS, post_n=POST_N, device="cpu"),
                                 RpnTrainer(vgg, H, W, ANCHORS, device="cpu"))


def _trunk_trace(rec, tr):
    """The normalised launches of tr.backward() from its _backward_trunk call on, and the launches before it.  The
    gradient _backward_trunk receives and the trunk's own data-gradient buffer at the feature map (tag feat_grad_tag) are
    both named g: the RPN step hands the trunk its gradient in that buffer, VGG16's RCNN step in one of its own."""
    _forward(tr)
    rec.reset()
    start = []
    inner = tr._backward_trunk

    def hook(g, debug=None):
        start.append((len(rec.calls), g))
        return inner(g, debug)
    tr._backward_trunk = hook
    try:
        tr.backward()
    finally:
        del tr._backward_trunk
    assert len(start) == 1
    at, g = start[0]
    names = {}
    for act in (g, tr._gact(tr.fh, tr.fw, tr.feat_ch, tag=tr.feat_grad_tag)):
        for part, t in (("g.hi", act.hi), ("g.lo", act.lo)):
            if t is not None and t.data_ptr() in rec._ptrs:
                names["p%d" % rec._ptrs[t.data_ptr()]] = part
    return rec.calls[:at], _normalised(rec.calls[at:], names)


@pytest.mark.parametrize("trunk,C,stride,least", [("recorded", 2048, 32, 150), ("recorded_vgg16", 512, 16, 50)],
                         ids=["resnet50", "vgg16"])
def test_rcnn_trunk_backward_is_the_rpn_trunk_backward(request, trunk, C, stride, least):
    rec, rcnn, rpn = request.getfixturevalue(trunk)
    head_rcnn, trunk_rcnn = _trunk_trace(rec, rcnn)
    head_rpn, trunk_rpn = _trunk_trace(rec, rpn)
    assert len(trunk_rcnn) > least
    assert trunk_rcnn == trunk_rpn
    # what comes before it: the head and fc layers, the RoI pooling backward over the feature map's C channels and its
    # re-layout
    names = [c[0] for c in head_rcnn]
    assert names.count("frcnn_roi_pool_backward") == 1
    roi = head_rcnn[names.index("frcnn_roi_pool_backward")]
    assert roi[3:6] == [rcnn.fh, rcnn.fw, C] and roi[11] == pytest.approx(1.0 / stride)
    assert [c[0] for c in head_rpn][-1] == "frcnn_conv2d"               # the RPN 3x3 conv's data gradient


def test_update_repacks_in_place(recorded):
    rec, rcnn, _ = recorded
    before = _planes(rcnn)
    assert {"fc6", "fc7", "heads", "trunk/conv1", "trunk/res5/b2/conv3"} <= {n for n, _ in before}
    rcnn.update()
    assert _planes(rcnn) == before


def test_layout_and_export(recorded, params):
    """The flat buffer holds the trunk convolutions, trunk/conv1/b and the head, no BN and no RPN entry; fc6/W is kept in
    (h, w, c) order with c = 2048 and exported in the reference's (c, h, w) order."""
    _, rcnn, _ = recorded
    names = set(rcnn.index)
    assert "fc6/W" in names and "trunk/conv1/b" in names and "trunk/res5/a/conv4/W" in names
    assert not any("/bn" in n or n.startswith("RPN/") for n in names)
    assert set(rto.trunk_param_names(50)) <= names
    assert rcnn.index["fc6/W"][2] == (4096, 2048 * 49)
    w = rcnn.weights("fc6/W")
    assert torch.equal(w[:3, :2048 * 2].reshape(3, 2, 2048),
                       torch.from_numpy(params["fc6/W"][:3].reshape(3, 2048, 49)[:, :, :2].transpose(0, 2, 1).copy()))
    ex = rcnn.export_params()
    assert set(ex) == names and ex["fc6/W"].shape == (4096, 2048 * 49)
    assert np.array_equal(ex["fc6/W"][:7], params["fc6/W"][:7]) and np.array_equal(ex["fc6/W"][-3:], params["fc6/W"][-3:])


def test_constructor_checks(params):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.resnet_train import ResNetRcnnTrainer

    def bad(p=params, h=H, w=W, match=None, **kw):
        with pytest.raises(FrcnnError, match=match):
            ResNetRcnnTrainer(p, h, w, ANCHORS, **dict(dict(n_layers=50, device="cpu"), **kw))
    bad(n_layers=34, match="n_layers")
    bad(feat_stride=16, match="feature stride is 32")
    bad(h=4, w=4, match="at least 5 x 5")
    bad(h=64, w=3, match="at least 5 x 5")
    bad(n_layers=101, match="trunk/res4/b6/conv1/W")                      # ResNet-50 parameters for ResNet-101
    for k, v in (("fc6/W", np.zeros((4096, 512 * 49), f32)), ("trunk/res3/a/bn4/avg_var", np.ones((256,), f32)),
                 ("RPN/rpn_conv_3x3/W", np.zeros((512, 512, 3, 3), f32)), ("cls_score/W", np.zeros((20, 4096), f32))):
        p = dict(params)
        p[k] = v
        bad(p, match=k)
    for k in ("fc6/W", "RPN/rpn_cls_score/b", "trunk/res2/b1/bn2/gamma", "trunk/conv1/b"):
        p = dict(params)
        del p[k]
        bad(p, match=k)


def test_oracle_unfolded_gradients_equal_scaled_folded_ones(params):
    """resnet_rcnn_train_step with BN unfolded and with folded=True (s * dL/dWf, s * dL/dbf): the same losses and the same
    gradients to float64 rounding."""
    rng = np.random.default_rng(4)
    p = dict(params)
    p["trunk/conv1/b"] = (rng.standard_normal(64) * 0.05).astype(f32)
    x = orc.make_image(H, W, seed=2)
    rois = np.array([[4, 6, 60, 50], [20, 10, 90, 62], [0, 0, 95, 63], [40, 30, 70, 60]], f32)
    keep = np.array([2, 0, 3], np.int32)
    labels = np.array([3, 0, 7], np.int32)
    targets = np.zeros((3, 84), f32)
    targets[0, 12:16] = rng.standard_normal(4)
    targets[2, 28:32] = rng.standard_normal(4)
    masks = [(rng.random((4, 4096)) >= 0.5).astype(np.uint8) for _ in range(2)]
    a = rto.resnet_rcnn_train_step(p, x, rois, keep, labels, targets, masks, n_layers=50)
    b = rto.resnet_rcnn_train_step(p, x, rois, keep, labels, targets, masks, n_layers=50, folded=True)
    assert np.allclose(a["losses"], b["losses"], rtol=1e-12, atol=1e-14)
    assert set(a["grads"]) == set(b["grads"]) == set(rto.trunk_param_names(50)) | {
        n for n in params if n.split("/")[0] in ("fc6", "fc7", "cls_score", "bbox_pred")}
    worst = 0.0
    for k in a["grads"]:
        ga, gb = a["grads"][k], b["grads"][k]
        assert np.abs(ga).max() > 0, k
        worst = max(worst, float(np.abs(ga - gb).max() / np.abs(ga).max()))
    print("unfolded vs folded: worst gradient difference %.2e of max-norm" % worst)
    assert worst < 1e-9
