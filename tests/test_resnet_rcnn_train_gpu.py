"""GPU tests of the RCNN training step with the ResNet trunk (frcnn_b200/resnet_train.py ResNetRcnnTrainer, frozen BN).

  (1) packing: the trainer's planes equal ResNetPackedWeights' packing of export_params() plus the BN and RPN entries, bit
      for bit, at construction and after an update (every folded trunk convolution, fc6, fc7, cls | bbox, the frozen RPN);
  (2) forward parity: the trainer and ResNetForwardPlan give bit-identical res5 maps, proposals and pool5;
  (3) layer by layer on the device's own tensors (ResNet-50 296x392, ResNet-101 600x1000): fc weight / data gradients
      within 5e-5 of max-norm of float64 products, exact ReLU + dropout masks, the RoI-pool backward at 1/32 over 2048
      channels against torchvision autograd (1e-6 of max), every bottleneck convolution's dW / db / dX within 5e-5;
  (4) end to end against resnet_rcnn_train_oracle.resnet_rcnn_train_step: the kept set, losses 2e-4, gradients 5e-2 of max-norm
      per tensor and 2e-2 in L2, the update over two steps, the loss falling on fixed kept rows and masks;
  (5) precision "bf16" against "bf16x3"; (6) alternation with ResNetRpnTrainer and loading into ResNetEngine;
  (7) the drop-in FasterRCNN(partial(ResNet, 50), 2048, 32) with rcnn_train = True; (8) bad calls."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import resnet_rcnn_train_oracle as rto
import resnet_train_ref as rtr
from test_resnet_train_gpu import _bits_equal, _case, _dev, _rel, _route_ref

pytestmark = pytest.mark.gpu
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
HEAD = ("fc6/W", "fc6/b", "fc7/W", "fc7/b", "cls_score/W", "cls_score/b", "bbox_pred/W", "bbox_pred/b")


def _rcnn_case(n_layers, H, W, seed):
    """test_resnet_train_gpu's case (livelier RPN heads, so that the proposals overlap the boxes) with head weights scaled
    so that fc6 / fc7 / the heads neither vanish nor saturate at K = 100,352."""
    params, x, gt, info = _case(n_layers, H, W, seed)
    rng = np.random.default_rng(seed + 100)
    for k, s in (("fc6/W", 0.001), ("fc7/W", 0.01), ("cls_score/W", 0.01), ("bbox_pred/W", 0.01)):
        params[k] = (rng.standard_normal(params[k].shape) * s).astype(f32)
    return params, x, gt, info


def _merged(tr, params):
    """export_params() with the constants the trainer holds (BN) and the frozen RPN, in the reference's layout."""
    m = dict(tr.export_params())
    m.update(tr.bn_params)
    m.update({k: v for k, v in params.items() if k.startswith("RPN/")})
    return m


def _trainer(params, H, W, n_layers=50, **kw):
    from frcnn_b200.resnet_train import ResNetRcnnTrainer
    return ResNetRcnnTrainer(params, H, W, ANCHORS, n_layers=n_layers, **kw)


# ------------------------------------------------------------------ (1) packing
def _same_planes(a, b):
    (hi, lo), bias = a
    rh, rl, rb = b
    return _bits_equal(hi, rh) and _bits_equal(lo, rl) and torch.equal(bias[:rb.numel()], rb) and not bool(bias[rb.numel():].any())


def test_trainer_packs_what_resnet_packed_weights_packs():
    from frcnn_b200.resnet_engine import ResNetPackedWeights
    H, W = 200, 264
    params, x, gt, _ = _rcnn_case(50, H, W, 2)
    for prec in ("bf16x3", "bf16"):
        tr = _trainer(params, H, W, precision=prec, post_n=64)
        for step in range(2 if prec == "bf16x3" else 1):
            if step:
                np.random.seed(1)
                tr.step(_dev(x[0]), _dev(gt[0]))
            ref = ResNetPackedWeights(_merged(tr, params), 50, prec, "cuda")
            for n in tr.conv:
                fwd, b, _ = tr.packed[n]
                assert _same_planes((fwd, b), ref.convs[n[len("trunk/"):]]), (prec, step, n)
            for name, want in (("fc6", ref.fc6), ("fc7", ref.fc7), ("heads", ref.head)):
                fwd, b, _ = tr.packed[name]
                assert _same_planes((fwd, b), want), (prec, step, name)
            assert _same_planes(tr.rpn3, ref.rpn3) and _same_planes(tr.rpn_heads, ref.rpn_heads), (prec, step)
        del tr


# ------------------------------------------------------------------ (2) forward parity
def test_forward_equals_resnet_forward_plan():
    from frcnn_b200.resnet_engine import ResNetEngine
    H, W = 296, 392
    params, x, gt, _ = _rcnn_case(50, H, W, 3)
    tr = _trainer(params, H, W, post_n=300)
    np.random.seed(0)
    tr.forward(_dev(x[0]), _dev(gt[0]))
    eng = ResNetEngine(_merged(tr, params), 50, precision="bf16x3", anchors=ANCHORS)
    _, _, plan = eng(_dev(x[0]), img_info=(H, W), pre_n=6000, post_n=300, nms_thresh=0.7, min_size=16)
    torch.cuda.synchronize()
    assert _bits_equal(tr.feat.hi, plan.feat.hi) and _bits_equal(tr.feat.lo, plan.feat.lo)
    R = int(tr.prop.count.item())
    assert R == int(plan.prop.count.item()) and R > 0
    assert torch.equal(tr.prop.rois[:R], plan.prop.rois[:R])
    assert _bits_equal(tr.pool5.hi[:, :R], plan.pool5.hi[:, :R]) and _bits_equal(tr.pool5.lo[:, :R], plan.pool5.lo[:, :R])
    print("forward parity: R=%d, res5 %s, pool5 %s" % (R, tuple(tr.feat.hi.shape), tuple(tr.pool5.hi.shape)))


# ------------------------------------------------------------------ (3) layer by layer
def _head_local(tr, params, dbg):
    """fc weight / data gradients against float64 products of the device's own tensors (on the GPU), exact ReLU +
    dropout masks, and the RoI-pool backward against torchvision autograd.  Returns the worst fc error."""
    import torchvision
    C, R = tr.feat_ch, int(tr.prop.count.item())
    d64 = lambda a: torch.as_tensor(a).to(device="cuda", dtype=torch.float64)           # noqa: E731
    val = lambda a: d64(a.hi.float() + a.lo.float())[0]                                 # noqa: E731  [R_cap, K]
    cols = lambda t: d64(t).reshape(t.shape[0], -1).T                                    # noqa: E731  (C,1,R_cap) -> [R_cap, C]
    rel = lambda a, b: float((d64(a) - b).abs().max() / b.abs().max().clamp_min(1e-30))  # noqa: E731
    nh = tr.n_heads
    dyh = d64(tr.head_grad)[:, :nh]
    fc7, fc6, pool5 = val(tr.fc7), val(tr.fc6), val(tr.pool5)
    Wh = d64(np.concatenate([params["cls_score/W"], params["bbox_pred/W"]], 0))
    e = [rel(torch.cat([tr.grads("cls_score/W"), tr.grads("bbox_pred/W")]), dyh.T @ fc7),
         rel(torch.cat([tr.grads("cls_score/b"), tr.grads("bbox_pred/b")]), dyh.sum(0))]
    g7 = cols(dbg["fc7"]["g_in"])
    e.append(rel(g7, dyh @ Wh))
    dy7 = cols(dbg["fc7"]["dy"])
    assert torch.equal(dy7, torch.where(fc7 > 0, 2.0 * g7, torch.zeros_like(g7)))        # ReLU + dropout backward: exact
    e += [rel(tr.grads("fc7/W"), dy7.T @ fc6), rel(tr.grads("fc7/b"), dy7.sum(0))]
    g6 = cols(dbg["fc6"]["g_in"])
    e.append(rel(g6, dy7 @ d64(params["fc7/W"])))
    dy6 = cols(dbg["fc6"]["dy"])
    assert torch.equal(dy6, torch.where(fc6 > 0, 2.0 * g6, torch.zeros_like(g6)))
    e += [rel(tr.grads("fc6/W"), dy6.T @ pool5), rel(tr.grads("fc6/b"), dy6.sum(0))]
    W6_hwc = d64(params["fc6/W"]).reshape(4096, C, 49).transpose(1, 2).reshape(4096, -1)
    dp5 = cols(dbg["roi"]["dpool5"])
    e.append(rel(dp5, dy6 @ W6_hwc))
    del W6_hwc
    print("head local errors (dWh, dbh, dX7, dW7, db7, dX6, dW6, db6, dpool5):", ["%.1e" % v for v in e])
    # the RoI pooling's backward at 1/32 over the device's res5 map
    feat = tr.feat.to_chw_f32().double()
    xf = feat[None].clone().requires_grad_(True)
    rois = tr.prop.rois[:R].double()
    br = torch.cat([torch.zeros((R, 1), dtype=torch.float64, device="cuda"), rois], 1)
    yp = torchvision.ops.roi_pool(xf, br, (7, 7), 1.0 / 32)
    yp.backward(dp5[:R].reshape(R, 7, 7, C).permute(0, 3, 1, 2))
    want_df = xf.grad[0].permute(1, 2, 0).reshape(-1, C)
    e_roi = float((d64(dbg["roi"]["dfeat"]) - want_df).abs().max() / want_df.abs().max())
    print("RoI-pool backward vs autograd: %.1e of max" % e_roi)
    assert e_roi <= 1e-6
    return max(e)


def _trunk_layerwise(tr, x, dbg):
    """Every bottleneck convolution's routed dy exactly and its dW (BN-scaled) / dX within float64 conv gradients of the
    device's own tensors, then pool1 + conv1.  Returns the worst (dW / db, dX) errors."""
    import torch.nn.grad as tg
    f64 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64, device="cuda")      # noqa: E731
    chw = lambda a: a.to_chw_f32().cpu().numpy()                                          # noqa: E731
    host = lambda t: t.cpu().numpy()                                                      # noqa: E731
    worst = dict(w=0.0, x=0.0)
    half = False
    for B in reversed(tr.blocks):
        base = B["name"]
        xin = f64(chw(tr.input_of(B)))[None]
        ins = {1: xin, 2: f64(chw(B["y1"]))[None], 3: f64(chw(B["y2"]))[None], 4: xin}
        outs = {1: chw(B["y1"]), 2: chw(B["y2"]), 3: chw(B["out"]), 4: chw(B["out"])}
        dys = {}
        for i in ((3, 4, 2, 1) if B["proj"] else (3, 2, 1)):
            n = "%s/conv%d" % (base, i)
            d, L = dbg[n], tr.conv[n]
            want = _route_ref(host(d["g_in"]), outs[i], half and i in (3, 4))
            assert np.array_equal(host(d["dy"]), want), n
            dys[i] = f64(host(d["dy"]))[None]
            s = host(L["s"])
            pad = 1 if i == 2 else 0
            Wf = f64(host(L["wf"]))
            dw_ref = host(tg.conv2d_weight(ins[i], Wf.shape, dys[i], padding=pad)) * s[:, None, None, None]
            dx_ref = tg.conv2d_input(ins[i].shape, Wf, dys[i], padding=pad)
            if i == 1:
                dx_ref = dx_ref + (tg.conv2d_input(xin.shape, f64(host(tr.conv[base + "/conv4"]["wf"])), dys[4])
                                   if B["proj"] else dys[3])
            worst["w"] = max(worst["w"], _rel(host(tr.grads(n + "/W")), dw_ref))
            worst["x"] = max(worst["x"], _rel(host(d["g_out"]), host(dx_ref)[0]))
        half = B["stride"] == 2
    d, L = dbg["trunk/conv1"], tr.conv["trunk/conv1"]
    Ho, Wo = tr.c1_hw
    g_p1 = tr._acts[(tr.p1.hi.shape[0], tr.p1.hi.shape[1], 64, 3)]
    want_hi, want_lo = rtr.maxpool3x3s2_backward(g_p1.hi, g_p1.lo, tr.c1.hi, tr.c1.lo, tr.p1.hi, tr.p1.lo)
    dz = tr._acts[(Ho, Wo, 64, 0)]
    assert _bits_equal(dz.hi, want_hi) and _bits_equal(dz.lo, want_lo), "trunk/conv1 routing"
    dzd = f64(host(d["dy"]))[None]
    s = host(L["s"])
    dw_ref = host(tg.conv2d_weight(f64(x), (64, 3, 7, 7), dzd, stride=2, padding=3)) * s[:, None, None, None]
    worst["w"] = max(worst["w"], _rel(host(tr.grads("trunk/conv1/W")), dw_ref),
                     _rel(host(tr.grads("trunk/conv1/b")), host(dzd.sum((0, 2, 3))) * s))
    print("trunk layer-wise worst: dW/db %.2e, dX %.2e" % (worst["w"], worst["x"]))
    return worst["w"], worst["x"]


def test_resnet50_step_layerwise_and_end_to_end():
    """ResNet-50 at 296 x 392 (res5 10 x 13), post_n = 64, NumPy sampling and dropout: (3) layer by layer and (4) end to
    end.  The end-to-end gradient bounds are the ResNet RPN step's (5e-2 of max-norm per tensor, 2e-2 in L2) for its
    reason: ReLU sign flips compound over 53 convolutions, and the device rounds every stored activation to 16 bits."""
    H, W = 296, 392
    params, x, gt, info = _rcnn_case(50, H, W, 5)
    tr = _trainer(params, H, W, post_n=64)
    np.random.seed(5)
    losses = tr.forward(_dev(x[0]), _dev(gt[0]))
    dbg = {}
    tr.backward(debug=dbg)
    torch.cuda.synchronize()
    R = int(tr.prop.count.item())
    keep = tr.keep.cpu().numpy()
    rois = tr.prop.rois.cpu().numpy()[:R]
    labels, ext = tr.labels.cpu().numpy(), tr.ext.cpu().numpy()
    masks = [m.cpu().numpy()[:R] for m in tr.masks]
    print("R=%d kept=%d labels=%s" % (R, len(keep), np.bincount(labels)[:8]))
    np.random.seed(5)
    ro = orc.proposal_target_layer(rois, gt)
    assert np.array_equal(ro["keep_inds"], keep) and np.array_equal(ro["use_gt_boxes"], tr.use_gt.cpu().numpy())
    fg = ro["max_overlaps"][keep] >= 0.5                       # labels are the best gt's class on background rows too
    assert fg.any() and not fg.all()
    # ---- (3) local checks
    assert _head_local(tr, params, dbg) <= 5e-5
    worst_w, worst_x = _trunk_layerwise(tr, x, dbg)
    assert worst_w <= 5e-5 and worst_x <= 5e-5
    del dbg
    # ---- (4) end to end
    want = rto.resnet_rcnn_train_step(params, x, rois, keep, labels, ext, masks, n_layers=50)
    Lv = losses.cpu().numpy()
    print("losses", Lv, "oracle", want["losses"])
    for i in (0, 1, 3):
        assert abs(Lv[i] - want["losses"][i]) <= 2e-4 * max(1.0, want["losses"][i])
    assert set(want["grads"]) == set(tr.index)
    worst, errs = 0.0, {}
    for name in tr.index:
        got = tr.grads(name).cpu().numpy()
        if name == "fc6/W":
            got = got.reshape(4096, 49, 2048).transpose(0, 2, 1).reshape(4096, -1)
        assert np.abs(want["grads"][name]).max() > 0 and np.abs(got).max() > 0, name
        errs[name] = _rel(got, want["grads"][name])
        worst = max(worst, errs[name])
    num = sum(float(np.square(tr.grads(k).cpu().numpy().astype(np.float64).reshape(-1)
                              - (want["grads"][k].reshape(4096, 2048, 49).transpose(0, 2, 1).reshape(-1) if k == "fc6/W"
                                 else want["grads"][k].reshape(-1))).sum()) for k in tr.index)
    den = sum(float(np.square(want["grads"][k]).sum()) for k in tr.index)
    l2 = (num / den) ** 0.5
    print("end-to-end worst gradient error (of max-norm): %.2e (%s), flat gradient L2 %.2e" % (worst, max(errs, key=errs.get), l2))
    print("  head:", {k: "%.1e" % errs[k] for k in HEAD})
    assert worst <= 5e-2 and l2 <= 2e-2
    del want
    # ---- the optimizer over two steps on the same kept rows and masks (momentum in play on the second)
    keep_d, masks_d = tr.keep.clone(), [m.clone() for m in tr.masks]
    lr, mom, wd = f32(0.001), f32(0.9), f32(0.0005)
    p0 = {k: tr.weights(k).cpu().numpy().copy() for k in tr.index}
    v0 = {k: np.zeros_like(p0[k]) for k in tr.index}
    for step in range(2):
        if step:
            tr.forward(_dev(x[0]), _dev(gt[0]), keep_inds=keep_d, masks=masks_d)
            tr.backward()
        g = {k: tr.grads(k).cpu().numpy().copy() for k in tr.index}
        tr.update()
        for name in tr.index:
            gi = (wd * p0[name] + g[name]).astype(f32)
            v = (mom * v0[name] - lr * gi).astype(f32)
            np.testing.assert_allclose(tr.weights(name).cpu().numpy(), (p0[name] + v).astype(f32), rtol=3e-7, atol=1e-10)
            # atol: a few float32 ulps of the largest term, for the elements where mom * v0 and lr * g cancel (fc6's
            # velocities reach 1e-11 at K = 100,352)
            np.testing.assert_allclose(tr.view(tr.v_flat, name).cpu().numpy(), v, rtol=2e-6, atol=1e-6 * float(np.abs(v).max()))
            p0[name], v0[name] = tr.weights(name).cpu().numpy().copy(), tr.view(tr.v_flat, name).cpu().numpy().copy()
        del g
    l3 = tr.forward(_dev(x[0]), _dev(gt[0]), keep_inds=keep_d, masks=masks_d).cpu().numpy()
    print("loss_rcnn after 0/2 updates: %.5f -> %.5f" % (Lv[3], l3[3]))
    assert l3[3] < Lv[3]


def test_resnet101_step_layerwise_600x1000():
    """Part (3) at the benchmarked 600 x 1000 image with ResNet-101 and 300 proposals (float64 references on the GPU)."""
    H, W = 600, 1000
    params, x, gt, _ = _rcnn_case(101, H, W, 4)
    tr = _trainer(params, H, W, n_layers=101, post_n=300)
    np.random.seed(4)
    tr.forward(_dev(x[0]), _dev(gt[0]))
    dbg = {}
    tr.backward(debug=dbg)
    torch.cuda.synchronize()
    assert _head_local(tr, params, dbg) <= 5e-5
    worst_w, worst_x = _trunk_layerwise(tr, x, dbg)
    assert worst_w <= 5e-5 and worst_x <= 5e-5


# ------------------------------------------------------------------ (5) precision
def test_bf16_against_bf16x3():
    """precision "bf16" on the kept rows and masks of a bf16x3 run: finite gradients, the loss within 0.1 of bf16x3's
    (relative), the whole flat gradient within 0.5 of it in L2 (relative) and each tensor within 0.75 of its max-norm.
    Measured on an H100: 4.6e-2, 0.28 and 0.39 (bbox_pred/W).  Looser than the ResNet RPN step's 2e-2 / 0.3 / 0.5: besides
    the ReLU signs and pool maxima that 8-bit operands move over 53 convolutions, the RPN's scores move, so the proposals
    (and the RoIs the pinned kept rows point at) are partly different boxes, and the head's losses are per RoI."""
    H, W = 296, 392
    params, x, gt, _ = _rcnn_case(50, H, W, 7)
    xd, gd = _dev(x[0]), _dev(gt[0])
    res, pins = {}, None
    for prec in ("bf16x3", "bf16"):
        tr = _trainer(params, H, W, precision=prec, post_n=64)
        np.random.seed(7)
        if pins is None:
            l = tr.forward(xd, gd)
            pins = (tr.keep.clone(), [m.clone() for m in tr.masks])
        else:
            l = tr.forward(xd, gd, keep_inds=pins[0], masks=pins[1])
        tr.backward()
        assert bool(torch.isfinite(tr.g_flat).all())
        res[prec] = (l.cpu().numpy(), {k: tr.grads(k).cpu().numpy().copy() for k in tr.index}, int(tr.prop.count.item()))
        del tr
    print("proposals: bf16x3 %d, bf16 %d" % (res["bf16x3"][2], res["bf16"][2]))
    d_loss = abs(res["bf16"][0][3] - res["bf16x3"][0][3]) / max(1.0, res["bf16x3"][0][3])
    errs = {k: _rel(res["bf16"][1][k], res["bf16x3"][1][k]) for k in res["bf16x3"][1]}
    name = max(errs, key=errs.get)
    num = sum(float(np.square(res["bf16"][1][k].astype(np.float64) - res["bf16x3"][1][k]).sum()) for k in errs)
    den = sum(float(np.square(res["bf16x3"][1][k].astype(np.float64)).sum()) for k in errs)
    l2 = (num / den) ** 0.5
    print("bf16 vs bf16x3: loss %.2e, flat gradient L2 %.2e, worst tensor %s %.2e of max-norm" % (d_loss, l2, name, errs[name]))
    assert d_loss < 0.1 and l2 < 0.5 and errs[name] < 0.75


# ------------------------------------------------------------------ (6) alternation
def test_alternation_with_the_rpn_step_and_the_engine():
    """train_rpn.py steps, export, then train_rcnn.py steps on the result: the RCNN trainer's frozen RPN planes equal the
    RPN trainer's own, and the parameters the RCNN steps export load into ResNetEngine, which runs."""
    from frcnn_b200.resnet_engine import ResNetEngine
    from frcnn_b200.resnet_train import ResNetRpnTrainer
    H, W = 200, 264
    params, x, gt, _ = _rcnn_case(50, H, W, 8)
    xd, gd = _dev(x[0]), _dev(gt[0])
    rpn = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50, subsample="device")
    for _ in range(2):
        rpn.step(xd, gd)
    p = dict(params)
    p.update(rpn.export_params())
    rcnn = _trainer(p, H, W, post_n=64)
    torch.cuda.synchronize()
    (hi, lo), b, _ = rpn.packed["RPN/rpn_conv_3x3"]
    assert _bits_equal(rcnn.rpn3[0][0], hi) and _bits_equal(rcnn.rpn3[0][1], lo) and torch.equal(rcnn.rpn3[1], b)
    (hi, lo), b, _ = rpn.packed["heads"]
    assert _bits_equal(rcnn.rpn_heads[0][0], hi) and _bits_equal(rcnn.rpn_heads[0][1], lo) and torch.equal(rcnn.rpn_heads[1], b)
    for k in rpn.conv:                                           # and the trunk the RPN step learnt
        assert _bits_equal(rcnn.packed[k][0][0], rpn.packed[k][0][0]), k
    del rpn
    np.random.seed(2)
    w0 = rcnn.w_flat.clone()
    for _ in range(2):
        l = rcnn.step(xd, gd).cpu().numpy()
        assert np.isfinite(l).all()
    assert not torch.equal(rcnn.w_flat, w0)
    eng = ResNetEngine(_merged(rcnn, p), 50, precision="bf16x3", anchors=ANCHORS)
    prob, boxes, plan = eng(xd, img_info=(H, W))
    torch.cuda.synchronize()
    assert prob.shape[0] > 0 and bool(torch.isfinite(prob).all()) and bool(torch.isfinite(boxes).all())
    # the engine's pool5 reads the same res5 the RCNN trainer computes with its updated weights
    rcnn.forward(xd, gd, keep_inds=rcnn.keep, masks=rcnn.masks)
    torch.cuda.synchronize()
    assert _bits_equal(rcnn.feat.hi, plan.feat.hi)


# ------------------------------------------------------------------ (7) drop-in
def test_dropin_faster_rcnn_resnet_rcnn_training_branch():
    import functools
    from frcnn_b200 import dropin
    from frcnn_b200.resnet_train import ResNetRcnnTrainer
    dropin.install()
    from chainer import Variable
    from models.faster_rcnn import FasterRCNN
    from models.resnet import ResNet
    np.random.seed(3)
    model = FasterRCNN(trunk_class=functools.partial(ResNet, 50), rpn_in_ch=2048, feat_stride=32)
    rng = np.random.default_rng(9)
    for path, p in model.namedparams():
        if path.endswith("/avg_var"):
            p.data[...] = rng.uniform(0.8, 1.25, p.data.shape).astype(f32)
        elif path.endswith("/avg_mean") or path.endswith("/beta"):
            p.data[...] = (rng.standard_normal(p.data.shape) * 0.05).astype(f32)
        elif path == "/trunk/conv1/W":
            p.data[...] *= f32(1.0 / 64)
        elif path in ("/RPN/rpn_cls_score/W", "/RPN/rpn_bbox_pred/W"):
            p.data[...] = (rng.standard_normal(p.data.shape) * 0.05).astype(f32)
        elif path == "/fc6/W":
            p.data[...] *= f32(0.2)
    model._params_changed()
    before = dict((k, v.data.copy()) for k, v in model.namedparams() if "/bn" in k)
    model.rcnn_train = True
    H, W = 296, 392
    x = orc.make_image(H, W, seed=5)
    gt = np.array([[[20, 30, 150, 170, 3], [100, 20, 330, 240, 7], [200, 150, 300, 280, 1]]], f32)
    info = np.array([[H, W]], np.int32)
    np.random.seed(3)
    loss = model(Variable(x), Variable(info), Variable(gt))
    assert isinstance(loss, Variable) and loss.data.shape == ()
    tr = model.rcnn_trainer
    assert isinstance(tr, ResNetRcnnTrainer) and tr.n_layers == 50
    assert abs(float(loss.data) - (float(model.loss_cls.data) + float(model.loss_bbox.data))) < 1e-5 * max(1.0, float(loss.data))
    tr.backward()
    w0 = tr.weights("fc7/W").clone()
    g = tr.grads("fc7/W").clone()
    assert float(g.abs().max()) > 0 and bool(torch.isfinite(tr.g_flat).all())
    tr.update()
    torch.testing.assert_close(tr.weights("fc7/W"), w0 + (-tr.lr * (g + tr.weight_decay * w0)), rtol=1e-6, atol=1e-9)
    named = dict(model.namedparams())                   # syncs the learnt weights back into the Link params
    fc6 = tr.weights("fc6/W").cpu().numpy().reshape(4096, 49, 2048).transpose(0, 2, 1).reshape(4096, -1)
    assert np.array_equal(named["/fc6/W"].data, fc6)
    for k in ("trunk/conv1/W", "trunk/res5/b2/conv3/W", "trunk/conv1/b", "fc7/W"):
        assert np.array_equal(named["/" + k].data, tr.weights(k).cpu().numpy()), k
    for k, v in before.items():
        assert np.array_equal(named[k].data, v), k
    # a second call on the same shape keeps the trainer; another shape builds a new one that inherits the momentum
    np.random.seed(4)
    model(Variable(x), Variable(info), Variable(gt))
    assert model.rcnn_trainer is tr
    v = tr.v_flat.clone()
    x2 = orc.make_image(264, 360, seed=6)
    np.random.seed(4)
    model(Variable(x2), Variable(np.array([[264, 360]], np.int32)), Variable(gt))
    assert model.rcnn_trainer is not tr and torch.equal(model.rcnn_trainer.v_flat, v)


# ------------------------------------------------------------------ (8) bad calls
def test_bad_calls_raise_before_queueing():
    from frcnn_b200._lib import FrcnnError
    H, W = 128, 160
    params, x, gt, _ = _rcnn_case(50, H, W, 1)
    torch.cuda.synchronize()
    mem = torch.cuda.memory_allocated()
    for kw, p in ((dict(n_layers=34), params), (dict(feat_stride=16), params), (dict(), dict(params, **{"fc6/W": params["fc7/W"]}))):
        with pytest.raises(FrcnnError):
            _trainer(p, H, W, **dict(dict(n_layers=50), **kw))
    with pytest.raises(FrcnnError):
        _trainer(params, 4, 64)
    assert torch.cuda.memory_allocated() == mem
    tr = _trainer(params, H, W, post_n=32)
    state = tr.gen.get_state()
    for xx, gg in ((_dev(x[0][:, :-1]), _dev(gt[0])), (_dev(x[0]), _dev(gt[0][:, :4])), (_dev(x[0]), _dev(gt[0][:0])),
                   (torch.from_numpy(x[0]), _dev(gt[0])), (_dev(x[0][None]), _dev(gt[0]))):
        with pytest.raises(FrcnnError):
            tr.forward(xx, gg)
    assert tr.last_losses is None and torch.equal(tr.gen.get_state(), state)
