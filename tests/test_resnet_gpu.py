"""GPU parity tests of the ResNet trunk row (SURVEY.md 8f rank 2, BASELINE config #4): the added kernels one by one, then
FasterRCNN(trunk=ResNet, rpn_in_ch=2048, feat_stride=32) stage by stage against the oracle (oracle/frcnn_oracle.py
resnet_forward: the published chainer ResNetLayers structure -- UNPINNED, Chainer is absent and the reference has no test or
call site for this trunk).  Tolerances as for the VGG path: features 1e-4 of max-norm, integer / index work bit-exact."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc

pytestmark = pytest.mark.gpu
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _act(x_chw):
    """(C,H,W) float32 numpy -> ops.Act NHWC hi/lo, and the exact value it holds."""
    from frcnn_b200 import ops
    t = torch.from_numpy(np.ascontiguousarray(x_chw.transpose(1, 2, 0))).cuda()
    hi = t.to(torch.bfloat16)
    lo = (t - hi.float()).to(torch.bfloat16)
    val = (hi.float() + lo.float()).cpu().numpy().transpose(2, 0, 1)
    return ops.Act(hi.contiguous(), lo.contiguous()), val


def test_maxpool3x3s2_and_subsample_exact():
    from frcnn_b200 import ops
    rng = np.random.default_rng(0)
    for (H, W) in [(7, 9), (80, 112), (75, 101), (3, 3)]:
        x = rng.standard_normal((16, H, W)).astype(f32)
        a, val = _act(x)
        y = ops.maxpool3x3s2_ceil(a).to_chw_f32().cpu().numpy()
        want = torch.nn.functional.max_pool2d(torch.from_numpy(val)[None], 3, 2, ceil_mode=True)[0].numpy()
        assert y.shape == want.shape and np.array_equal(y, want), (H, W)
        s = ops.subsample2x(a).to_chw_f32().cpu().numpy()
        assert np.array_equal(s, val[:, ::2, ::2])


def test_conv1_7x7s2_im2col_gemm():
    """conv1 of ResNet as im2col (K = 147 -> 160) + the 1x1 tensor-core GEMM, BN folded, ReLU."""
    from frcnn_b200 import ops
    from frcnn_b200.resnet_engine import CONV1_KPAD
    rng = np.random.default_rng(1)
    for (H, W) in [(64, 96), (75, 101)]:
        x = rng.uniform(-100, 100, (3, H, W)).astype(f32)
        w = (rng.standard_normal((64, 3, 7, 7)) * 0.002).astype(f32)
        b = rng.standard_normal(64).astype(f32) * 0.1
        col = ops.pack_image_im2col_general(torch.from_numpy(x).cuda(), 7, 2, 3, CONV1_KPAD)
        hi, lo = ops.pack_conv_weights_im2col_general(torch.from_numpy(w).cuda(), CONV1_KPAD)
        y, _ = ops.conv2d(col, hi, lo, ops.pad_bias(torch.from_numpy(b).cuda(), 64), 1, True)
        want = torch.relu(torch.nn.functional.conv2d(torch.from_numpy(x).double()[None], torch.from_numpy(w).double(),
                                                     torch.from_numpy(b).double(), stride=2, padding=3))[0].numpy()
        got = y.to_chw_f32().cpu().numpy()
        assert got.shape == want.shape
        assert _rel(got, want) < 2e-5, _rel(got, want)


def test_conv_residual_epilogue():
    """frcnn_conv2d_res: relu(conv1x1(x) + bias + shortcut) in one epilogue, exact on bf16-representable data."""
    from frcnn_b200 import ops
    rng = np.random.default_rng(2)
    H, W, Cin, Cout = 20, 28, 128, 512
    x = rng.integers(-4, 5, (Cin, H, W)).astype(f32)
    r = rng.integers(-50, 50, (Cout, H, W)).astype(f32)
    w = rng.integers(-2, 3, (Cout, Cin, 1, 1)).astype(f32)
    b = rng.integers(-8, 9, Cout).astype(f32)
    xa, _ = _act(x)
    ra, _ = _act(r)
    hi, lo = ops.pack_conv_weights(torch.from_numpy(w).cuda(), cin_pad=Cin)
    y = ops.conv2d_res(xa, hi, lo, ops.pad_bias(torch.from_numpy(b).cuda(), Cout), 1, True, ra)
    want = np.maximum(np.einsum("oc,chw->ohw", w[:, :, 0, 0], x) + b[:, None, None] + r, 0)
    assert np.array_equal(y.to_chw_f32().cpu().numpy(), want)
    # random real data, 3x3 with residual, no relu
    x = rng.standard_normal((64, H, W)).astype(f32)
    r = rng.standard_normal((64, H, W)).astype(f32)
    w = (rng.standard_normal((64, 64, 3, 3)) * 0.05).astype(f32)
    xa, xv = _act(x)
    ra, rv = _act(r)
    hi, lo = ops.pack_conv_weights(torch.from_numpy(w).cuda(), cin_pad=64)
    y = ops.conv2d_res(xa, hi, lo, ops.pad_bias(torch.zeros(64).cuda(), 64), 3, False, ra)
    want = torch.nn.functional.conv2d(torch.from_numpy(xv).double()[None], torch.from_numpy(w).double(), padding=1)[0].numpy() + rv
    assert _rel(y.to_chw_f32().cpu().numpy(), want) < 2e-5


def test_bn_folding_matches_unfolded_oracle():
    p = orc.make_resnet_params(50, seed=5)
    x = orc.make_image(96, 128, seed=5)
    a = orc.resnet_forward(x, p, 50, folded=True)
    b = orc.resnet_forward(x, p, 50, folded=False)
    assert _rel(a, b) < 1e-4
    from frcnn_b200.resnet_engine import fold_batchnorm
    W, bn = p["trunk/res3/a/conv2/W"], "trunk/res3/a/bn2"
    Wf, bf = fold_batchnorm(W, p[bn + "/gamma"], p[bn + "/beta"], p[bn + "/avg_mean"], p[bn + "/avg_var"])
    Wo, bo = orc.fold_bn(W, p, bn)
    assert np.array_equal(Wf, Wo) and np.array_equal(bf, bo)


@pytest.mark.parametrize("n_layers,shape", [(50, (160, 224)), (101, (150, 201)), (152, (600, 1000))])
def test_resnet_faster_rcnn_forward_stagewise(n_layers, shape):
    """Each stage on the device's own upstream tensors.  Boxes: bbox_transform_inv makes x1 = cx + dx*w - exp(dw)*w/2 (and
    alike), so a delta error e moves a coordinate by up to e*w*(1 + exp(dw)/2); the decode amplifies the head's error by
    the exponential of the size deltas.  Each coordinate is held to 1e-4 of the image scale, or, where it is larger, to the
    deltas' own 1e-4 max-norm bound carried through that sensitivity: the synthetic head's deltas reach 7.6 on ResNet-152 at
    600x1000 (exp(7.6)/2 ~ 1000), where a 1e-5 delta error alone moves a box by 2.5e-4 of the image scale."""
    from frcnn_b200.resnet_engine import ResNetEngine
    H, W = shape
    post_n = 300 if H * W >= 600 * 1000 else 100          # the reference's test-time count where the map has the anchors
    params = orc.make_resnet_params(n_layers, seed=11)
    x = orc.make_image(H, W, seed=4)
    info = np.array([[H, W]], np.int32)
    eng = ResNetEngine(params, n_layers, precision="bf16x3", anchors=ANCHORS, keep_rpn_debug=True, use_graph=False, post_n=post_n)
    prob, boxes, plan = eng(torch.from_numpy(x[0]).cuda())
    torch.cuda.synchronize()
    R = prob.shape[0]
    # ---- trunk: res5 vs the fp32 oracle
    feat_dev = plan.acts[-1].to_chw_f32().cpu().numpy()[None]
    feat_ref = orc.resnet_forward(x, params, n_layers)
    assert feat_dev.shape == feat_ref.shape and feat_dev.shape[1] == 2048
    e = _rel(feat_dev, feat_ref)
    print("ResNet-%d res5 %s max-rel error vs fp32 oracle: %.2e (max |feat| %.1f)" % (n_layers, feat_ref.shape, e, np.abs(feat_ref).max()))
    assert e < 1e-4
    # ---- RPN on the device's own feature map, ProposalLayer bit-exact on the device's logits (feat_stride 32)
    fh, fw = plan.fh, plan.fw
    rpn = plan.rpn_out.cpu().numpy()
    logits_dev = rpn[:, :18].T.reshape(1, 18, fh, fw)
    deltas_dev = rpn[:, 18:54].T.reshape(1, 36, fh, fw)
    h_ref = orc.relu(orc.conv2d(feat_dev, params["RPN/rpn_conv_3x3/W"], params["RPN/rpn_conv_3x3/b"], 1))
    assert _rel(plan.rpn_mid.to_chw_f32().cpu().numpy()[None], h_ref) < 1e-4
    want_rois, want_fg = orc.proposal_layer(orc.softmax_axis1(logits_dev), deltas_dev, info, feat_stride=32, post_nms_top_n=post_n)
    rois_dev = plan.prop.rois.cpu().numpy()
    assert R == len(want_rois) and R > 0
    assert np.array_equal(rois_dev[:R], want_rois)
    assert np.array_equal(plan.prop.scores.cpu().numpy()[:R], want_fg.ravel())
    # ---- RoI pool (exact, scale 1/32, 2048 channels) and head on the device's feature map and RoIs
    cls_ref, box_ref, aux = orc.head_forward(feat_dev, rois_dev[:R], params, info, spatial_scale=1.0 / 32)
    pool_dev = (plan.pool5.hi.float() + plan.pool5.lo.float()).cpu().numpy().reshape(-1, 7, 7, 2048)[:R]
    assert np.array_equal(pool_dev.transpose(0, 3, 1, 2), aux["pool5"])
    # fc6 has K = 100,352: a float32 CPU dot product of that length is itself only ~1e-4 accurate, so the device is held to
    # the float64 value of the same contraction (and the fp32 oracle's own distance to it is printed)
    fc6_dev = (plan.fc6.hi.float() + plan.fc6.lo.float()).cpu().numpy()[0, :R]
    fc6_64 = np.maximum(aux["pool5"].reshape(R, -1).astype(np.float64) @ params["fc6/W"].astype(np.float64).T + params["fc6/b"], 0)
    print("fc6 (K=100352): device vs float64 %.2e, fp32 oracle vs float64 %.2e" % (_rel(fc6_dev, fc6_64), _rel(aux["fc6"], fc6_64)))
    assert _rel(fc6_dev, fc6_64) < 5e-5
    assert np.abs(prob.cpu().numpy() - cls_ref).max() < 1e-4 * cls_ref.max()
    ho = plan.head_out.cpu().numpy()[:R]
    d_dev, d_ref = ho[:, 21:105].astype(np.float64), aux["bbox_pred"].astype(np.float64)
    e_delta = _rel(d_dev, d_ref)
    assert e_delta < 1e-4
    r = rois_dev[:R].astype(np.float64)
    size = np.stack([r[:, 2] - r[:, 0] + 1, r[:, 3] - r[:, 1] + 1], 1)                          # RoI w, h
    d_size = np.maximum(np.abs(d_dev), np.abs(d_ref)).reshape(R, -1, 4)[:, :, 2:]                # dw, dh
    sens = size[:, None, :] * (1 + 0.5 * np.exp(d_size))                                        # [R, classes, (x, y)]
    sens = np.concatenate([sens, sens], axis=2).reshape(R, -1)                                  # x1, y1, x2, y2
    err = np.abs(boxes.cpu().numpy().astype(np.float64) - box_ref)
    tol = np.maximum(1e-4 * np.abs(box_ref).max(), 1e-4 * np.abs(d_ref).max() * sens)
    print("boxes: max err %.2e of scale, worst err / tol %.2f (max |delta| %.2f, deltas %.2e)" %
          (_rel(boxes.cpu().numpy(), box_ref), (err / tol).max(), np.abs(d_ref).max(), e_delta))
    assert (err <= tol).all()
    # graph replay == eager, and lanes work with the subclassed plan
    eng_g = ResNetEngine(params, n_layers, precision="bf16x3", anchors=ANCHORS, use_graph=True, post_n=post_n)
    pg, bg, plan_g = eng_g(torch.from_numpy(x[0]).cuda())
    assert torch.equal(pg, prob) and torch.equal(bg, boxes)
    assert type(plan_g.clone()) is type(plan_g)


def test_dropin_resnet_trunk_and_detector():
    """models.resnet.ResNet (the reference's trunk class name) alone and inside FasterRCNN(trunk_class=..., rpn_in_ch=2048,
    feat_stride=32): parameter paths are Chainer's (trunk/res4/b7/bn2/avg_var, ...), the forward equals the oracle's."""
    import functools
    from frcnn_b200 import dropin
    dropin.install()
    from chainer import Variable
    from models.faster_rcnn import FasterRCNN
    from models.resnet import ResNet
    np.random.seed(3)
    model = FasterRCNN(trunk_class=functools.partial(ResNet, 50), rpn_in_ch=2048, feat_stride=32)
    model.rcnn_train = False
    model.rpn_train = False
    rng = np.random.default_rng(9)
    for path, p in model.namedparams():
        if path.endswith("/avg_var"):
            p.data[...] = rng.uniform(0.8, 1.25, p.data.shape).astype(f32)
        elif path.endswith("/avg_mean") or path.endswith("/beta"):
            p.data[...] = (rng.standard_normal(p.data.shape) * 0.05).astype(f32)
        elif path == "/trunk/conv1/W":
            p.data[...] *= f32(1.0 / 64)
        elif path == "/fc6/W":
            p.data[...] *= f32(0.2)
    model._params_changed()
    params = model.param_dict()
    assert "trunk/res4/b5/bn2/avg_var" in params and "trunk/res5/a/conv4/W" in params and params["fc6/W"].shape == (4096, 2048 * 49)
    H, W = 160, 224
    x = orc.make_image(H, W, seed=6)
    feat = model.trunk(Variable(x)).data
    want = orc.resnet_forward(x, params, 50)
    assert feat.shape == want.shape == (1, 2048, 5, 7) and _rel(feat, want) < 1e-4
    info = np.array([[H, W]], np.int32)
    cls_prob, pred_boxes = model(Variable(x), Variable(info))
    R = cls_prob.data.shape[0]
    assert 0 < R <= 300 and cls_prob.data.shape == (R, 21) and pred_boxes.shape == (R, 84)
    np.testing.assert_allclose(cls_prob.data.sum(1), 1.0, rtol=1e-5)
    # the same proposals as the oracle's end-to-end run, matched by box (near-tie scores may reorder)
    want_cls, want_boxes, aux = orc.faster_rcnn_resnet_forward(x, params, info, n_layers=50, pre_nms_top_n=6000, post_nms_top_n=300)
    got_rois = model.rpn_proposals
    d = np.abs(got_rois[:, None, :] - aux["proposals"][None, :, :]).max(-1)
    matched = (d.min(1) < 0.05).mean()
    print("ResNet-50 detector: R=%d (oracle %d), proposals matched %.3f" % (R, len(aux["proposals"]), matched))
    assert matched > 0.95 and abs(R - len(aux["proposals"])) <= max(3, R // 20)
