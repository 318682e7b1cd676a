"""The joint training step (JointTrainer, CanvasJointTrainer, CanvasResNetJointTrainer) against its two parts and float64.

Bit-identity against RpnTrainer / RcnnTrainer (and their canvas and ResNet versions) is the bar everywhere except where the
two gradients of the feature map meet: the joined gradient (the RPN conv's data gradient with the split dfeat added in its
epilogue) is checked elementwise against the float64 sum of the two trainers' gradients, and the trunk's gradients against
the float64 sum of theirs."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_aug_train_gpu import SCALES, _run_pair
from test_canvas_rcnn_train_gpu import MIX, _masks_ref, _rcnn_params
from test_canvas_train_gpu import ANCHORS, _flat_equal, _images
from test_raw_canvas_train_gpu import HC, WC
from test_train_gpu import _rel, _train_case

pytestmark = pytest.mark.gpu
f32 = np.float32
HEAD = ("fc6/", "fc7/", "cls_score/", "bbox_pred/")


def _f64(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _dfeat_chw(dfeat, fh, fw):
    """RcnnTrainer's fp32 dfeat [fh*fw, C] as (C, fh, fw)."""
    return dfeat.view(fh, fw, -1).permute(2, 0, 1)


def _pins(jt, x, gt, post_n, seed):
    """A disable list (the reference's NumPy subsampling), a kept list (the reference's NumPy sampling on the joint
    trainer's own proposals) and explicit masks for one image."""
    h, w = int(x.shape[1]), int(x.shape[2])
    np.random.seed(seed)
    dis = jt._numpy_subsample(gt, h, w)
    jt.forward(x, gt, disable_pos=dis)                       # numpy sampling draws the kept rows
    torch.cuda.synchronize()
    keep = jt.keep.clone()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    masks = [(torch.rand((post_n, 4096), device="cuda", generator=gen) >= 0.5).to(torch.uint8) for _ in range(2)]
    return dis, keep, masks


def _labels_equal(a, b):
    """The anchor labels of two AnchorTargetsBatch, slot by slot over each slot's inside anchors."""
    if not torch.equal(a.counts, b.counts):
        return False
    for n in range(a.N):
        inds = a.inds_inside[n, :int(a.counts[n, 0])].long()
        if not (torch.equal(inds, b.inds_inside[n, :inds.numel()].long())
                and torch.equal(a.labels_full[n][inds], b.labels_full[n][inds])):
            return False
    return True


# ------------------------------------------------------------------------------------------------ (1) the two parts
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_joint_step_is_its_two_parts(precision):
    from frcnn_b200.train_engine import JointTrainer, RcnnTrainer, RpnTrainer
    H, W, post_n = 296, 392, 120
    params = _rcnn_params(H, W, 3)
    xs, gts = _images([(H, W)], 4)
    x, gt = xs[0], gts[0]
    jt = JointTrainer(params, H, W, ANCHORS, precision=precision, post_n=post_n)
    pt = RpnTrainer(params, H, W, ANCHORS, precision=precision)
    rt = RcnnTrainer(params, H, W, ANCHORS, precision=precision, post_n=post_n)
    dis, keep, masks = _pins(jt, x, gt, post_n, 10)
    lj = jt.forward(x, gt, disable_pos=dis, keep_inds=keep, masks=masks).clone()
    dj = {}
    jt.backward(debug=dj)
    lp = pt.forward(x, gt, disable_pos=dis).clone()
    dp = {}
    pt.backward(debug=dp)
    lr_ = rt.forward(x, gt, keep_inds=keep, masks=masks).clone()
    dr = {}
    rt.backward(debug=dr)
    torch.cuda.synchronize()
    assert lj.shape == (8,)
    assert _flat_equal(lj[:4], lp) and _flat_equal(lj[4:], lr_)
    assert _flat_equal(jt.rpn.head_out, rt.rpn_out)                     # one RPN output for both halves
    R = int(rt.prop.count.item())
    assert int(jt.prop.count.item()) == R and _flat_equal(jt.prop.rois[:R].contiguous(), rt.prop.rois[:R].contiguous())
    assert _flat_equal(jt.rpn.head_grad, pt.head_grad) and _flat_equal(jt.head_grad, rt.head_grad)
    assert _flat_equal(jt.dfeat, rt.dfeat)
    for name in jt.index:
        if name.startswith("RPN/"):
            assert _flat_equal(jt.grads(name), pt.grads(name)), name
        elif name.startswith(HEAD):
            assert _flat_equal(jt.grads(name), rt.grads(name)), name
    # the joined gradient of the feature map, elementwise against the float64 sum of its two parts
    g_rpn = _f64(dp["RPN/rpn_conv_3x3"]["g_out"])
    g_roi = _f64(_dfeat_chw(dr["roi"]["dfeat"], jt.fh, jt.fw))
    joined = _f64(dj["RPN/rpn_conv_3x3"]["g_out"])
    bar = 2.0 ** (-15 if precision == "bf16x3" else -7)
    ratio = np.abs(joined - (g_rpn + g_roi)) / np.maximum(np.abs(g_rpn) + np.abs(g_roi), 1e-300)
    print("%s joined-gradient worst error (of |g_rpn| + |dfeat|): %.2e (bar %.2e)" % (precision, ratio.max(), bar))
    assert bool((np.abs(joined - (g_rpn + g_roi)) <= bar * (np.abs(g_rpn) + np.abs(g_roi))).all())
    assert np.abs(g_rpn).max() > 0 and np.abs(g_roi).max() > 0
    if precision == "bf16x3":
        worst = max(_rel(_f64(jt.grads(n)), _f64(pt.grads(n)) + _f64(rt.grads(n))) for n in jt.index if n.startswith("trunk/"))
        print("trunk-gradient worst error (of max-norm): %.2e" % worst)
        assert worst <= 1e-4
    jt.update()
    pt.update()
    rt.update()
    torch.cuda.synchronize()
    for name in jt.index:
        ref = pt if name.startswith("RPN/") else rt if name.startswith(HEAD) else None
        if ref is not None:
            assert _flat_equal(jt.weights(name), ref.weights(name)), name
            assert _flat_equal(jt.view(jt.v_flat, name), ref.view(ref.v_flat, name)), name


def test_export_is_a_detector_the_engine_loads():
    from frcnn_b200.engine import Engine
    from frcnn_b200.train_engine import JointTrainer
    H, W = 160, 224
    params = _rcnn_params(H, W, 2)
    xs, gts = _images([(H, W)], 3)
    jt = JointTrainer(params, H, W, ANCHORS, post_n=64)
    jt.step(xs[0], gts[0])
    torch.cuda.synchronize()
    eng = Engine(jt.export_params(), precision="bf16x3", anchors=ANCHORS, with_detect=True)
    prob, boxes, _ = eng(xs[0])
    torch.cuda.synchronize()
    assert prob.shape[0] > 0 and bool(torch.isfinite(prob).all()) and bool(torch.isfinite(boxes).all())


# ------------------------------------------------------------------------------------------------ (2) full-size canvas
def test_full_size_canvas_is_the_one_image_step():
    from frcnn_b200.train_engine import CanvasJointTrainer, JointTrainer
    H, W, post_n = 296, 392, 120
    params = _rcnn_params(H, W, 4)
    xs, gts = _images([(H, W)] * 2, 5)
    jt = JointTrainer(params, H, W, ANCHORS, post_n=post_n)
    ct = CanvasJointTrainer(params, 1, H, W, ANCHORS, post_n=post_n, subsample="list", sample="list", dropout="explicit")
    for k in range(2):
        dis, keep, masks = _pins(jt, xs[k], gts[k], post_n, 20 + k)
        lj = jt.forward(xs[k], gts[k], disable_pos=dis, keep_inds=keep, masks=masks).clone()
        jt.backward()
        ct.put([xs[k]], [gts[k]], disable_pos=[dis], keep_inds=[keep], masks=[masks])
        lc = ct.forward().clone()
        ct.backward()
        torch.cuda.synchronize()
        assert lc.shape == (1, 8) and _flat_equal(lc[0], lj), k
        assert _flat_equal(ct.g_flat, jt.g_flat), k
        jt.update()
        ct.update()
        torch.cuda.synchronize()
        assert _flat_equal(ct.w_flat, jt.w_flat) and _flat_equal(ct.v_flat, jt.v_flat), k


# ------------------------------------------------------------------------------------------------ (3) mixed sizes
def test_mixed_sizes_equal_per_image_steps():
    from frcnn_b200.train_engine import CanvasJointTrainer, JointTrainer
    Hc, Wc, post_n = 296, 392, 100
    params = _rcnn_params(Hc, Wc, 5)
    xs, gts = _images(MIX, 6)
    refs, pins = [], []
    for n, (h, w) in enumerate(MIX):
        jt = JointTrainer(params, h, w, ANCHORS, post_n=post_n)
        pins.append(_pins(jt, xs[n], gts[n], post_n, 30 + n))
        refs.append(jt)
    ct = CanvasJointTrainer(params, 4, Hc, Wc, ANCHORS, post_n=post_n, subsample="list", sample="list", dropout="explicit")
    ct.put(xs, gts, disable_pos=[p[0] for p in pins], keep_inds=[p[1] for p in pins], masks=[p[2] for p in pins])
    losses = ct.forward().clone()
    dbg = {}
    ct.backward(debug=dbg)
    torch.cuda.synchronize()
    assert losses[3].cpu().numpy().tolist() == [0.0] * 8                       # the empty slot
    gsum = {k: np.zeros(ct.index[k][2], np.float64) for k in ct.index}
    for n, jt in enumerate(refs):
        dis, keep, masks = pins[n]
        lo = jt.forward(xs[n], gts[n], disable_pos=dis, keep_inds=keep, masks=masks)
        rd = {}
        jt.backward(debug=rd)
        torch.cuda.synchronize()
        assert _flat_equal(losses[n], lo), n
        R = int(jt.prop.count.item())
        assert int(ct.head_ext[n, 1]) == R, n
        assert _flat_equal(ct.prop.rois[n, :R].contiguous(), jt.prop.rois[:R].contiguous()), n
        for a, b in ((ct.fc6, jt.fc6), (ct.fc7, jt.fc7), (ct.pool5, jt.pool5)):
            assert torch.equal(a.hi[n, 0, :R], b.hi[0, :R]) and torch.equal(a.lo[n, 0, :R], b.lo[0, :R]), n
        rows = slice(n * post_n, (n + 1) * post_n)
        assert _flat_equal(ct.head_grad[rows].contiguous(), jt.head_grad), n
        fh, fw = jt.fh, jt.fw
        rpn_grad = ct.rpn.head_grad.view(4, ct.fh, ct.fw, -1)[n, :fh, :fw].contiguous()
        assert _flat_equal(rpn_grad, jt.rpn.head_grad.view(fh, fw, -1)), n
        for key, d in rd.items():
            if not (key.startswith("trunk/") or key.startswith("RPN/")):
                continue
            for f, v in d.items():
                c = dbg[key][f][n]
                _, hh, ww = v.shape
                assert _flat_equal(c[:, :hh, :ww].contiguous(), v), (key, f, n)
                out = c.clone()
                out[:, :hh, :ww] = 0
                assert bool((out == 0).all()), (key, f, n)
        for k in ct.index:
            gsum[k] += jt.grads(k).cpu().numpy()
    worst = max(_rel(ct.grads(k).cpu().numpy(), gsum[k]) for k in ct.index)
    print("summed-gradient worst error (of max-norm): %.2e" % worst)
    assert worst <= 5e-5


# ------------------------------------------------------------------------------------------------ (4) draws and replay
def test_step0_draws_are_the_component_trainers():
    from frcnn_b200.train_engine import CanvasJointTrainer, CanvasRcnnTrainer, CanvasRpnTrainer
    Hc, Wc, N, post_n, s = 296, 392, 3, 100, 41
    params = _rcnn_params(Hc, Wc, 7)
    xs, gts = _images(MIX, 8)
    kw = dict(post_n=post_n, sample="device", dropout="device", seed=s)
    ct = CanvasJointTrainer(params, N, Hc, Wc, ANCHORS, subsample="device", **kw)
    cp = CanvasRpnTrainer(params, N, Hc, Wc, ANCHORS, subsample="device", seed=s)
    cr = CanvasRcnnTrainer(params, N, Hc, Wc, ANCHORS, **kw)
    for t in (ct, cp, cr):
        t.put(xs, gts)
        t.forward()
    torch.cuda.synchronize()
    assert _labels_equal(ct.rpn.targets, cp.targets)
    assert torch.equal(ct.head_ext, cr.head_ext) and torch.equal(ct.prop.rois, cr.prop.rois)
    assert torch.equal(ct.ptargets.keep, cr.ptargets.keep) and torch.equal(ct.ptargets.counts, cr.ptargets.counts)
    assert torch.equal(ct.masks, cr.masks)
    assert torch.equal(ct.seeds, cp.seeds) and torch.equal(ct.seeds, cr.seeds)       # advanced once, by N


@pytest.mark.parametrize("rule", ["MomentumSGD", "Adam"])
def test_graph_replay_equals_eager_run_and_follows_lr(rule):
    from frcnn_b200 import optimizers
    from frcnn_b200.train_engine import CanvasJointTrainer
    Hc, Wc, N, post_n, s = 296, 392, 3, 100, 31
    params = _rcnn_params(Hc, Wc, 9)
    xs, gts = _images(MIX, 10)
    opt = lambda: optimizers.MomentumSGD(lr=0.001) if rule == "MomentumSGD" else optimizers.Adam(alpha=1e-4)   # noqa: E731
    kw = dict(post_n=post_n, subsample="device", sample="device", dropout="device", seed=s)
    a = CanvasJointTrainer(params, N, Hc, Wc, ANCHORS, optimizer=opt(), **kw)
    b = CanvasJointTrainer(params, N, Hc, Wc, ANCHORS, optimizer=opt(), **kw)
    masks = []
    for it in range(3):
        if it == 2:                                          # a learning-rate drop after the capture reaches the replay
            a.lr, b.lr = a.lr * 0.1, b.lr * 0.1
        la = a.step(xs, gts)                                 # eager, then capture, then replays
        masks.append(a.masks.clone())
        b.put(xs, gts)
        b.run()
        torch.cuda.synchronize()
        assert la.shape == (N, 8) and _flat_equal(la, b.step_losses), it
        assert torch.equal(a.masks, b.masks) and torch.equal(a.ptargets.keep, b.ptargets.keep), it
        assert _labels_equal(a.rpn.targets, b.rpn.targets), it
        assert _flat_equal(a.g_flat, b.g_flat) and _flat_equal(a.w_flat, b.w_flat), it
        for k in a.opt_state:
            assert _flat_equal(a.opt_state[k], b.opt_state[k]), (it, k)
    assert a.graph is not None and a.n_updates == 3
    assert not torch.equal(masks[1], masks[2])              # replays draw fresh masks
    for n in range(N):                                       # step 2, slot n: seed + 2N + n
        for j in range(2):
            np.testing.assert_array_equal(masks[2][j, n].cpu().numpy(), _masks_ref(s + 2 * N + n, j + 1, post_n, 4096))


# ------------------------------------------------------------------------------------------------ (5) raw photos
def test_raw_augmented_step_equals_float_step():
    from frcnn_b200.train_engine import CanvasJointTrainer
    N = 2
    params = _rcnn_params(HC, WC, 7)
    kw = dict(post_n=300, seed=11, subsample="device", sample="device", dropout="device")
    raw = CanvasJointTrainer(params, N, HC, WC, ANCHORS, raw_input=True, augment="device", scales=SCALES, **kw)
    flt = CanvasJointTrainer(params, N, HC, WC, ANCHORS, **kw)
    seen = _run_pair(raw, flt, N, 710)
    assert len(set(seen)) > 1, seen
    assert torch.equal(raw.masks, flt.masks) and torch.equal(raw.seeds, flt.seeds)
    assert _labels_equal(raw.rpn.targets, flt.rpn.targets)


# ------------------------------------------------------------------------------------------------ (6) ResNet-50 canvas
def test_resnet50_canvas_is_its_two_parts():
    from test_resnet_train_gpu import _case
    from frcnn_b200.resnet_train import CanvasResNetJointTrainer, CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer
    Hc, Wc, N, post_n, s = 256, 320, 2, 64, 3
    params = _case(50, Hc, Wc, 3)[0]
    rng = np.random.default_rng(4)
    for k in ("cls_score/W", "bbox_pred/W"):
        params[k] = (rng.standard_normal(params[k].shape) * 0.02).astype(f32)
    xs, gts = _images([(256, 320), (200, 288)], 12)
    kw = dict(n_layers=50, post_n=post_n, sample="device", dropout="device", seed=s)
    ct = CanvasResNetJointTrainer(params, N, Hc, Wc, ANCHORS, **kw)
    cp = CanvasResNetRpnTrainer(params, N, Hc, Wc, ANCHORS, n_layers=50, seed=s)
    cr = CanvasResNetRcnnTrainer(params, N, Hc, Wc, ANCHORS, **kw)
    for t in (ct, cp, cr):
        t.put(xs, gts)
        t.forward()
        t.backward()
    torch.cuda.synchronize()
    lc = ct.step_losses
    assert _flat_equal(lc[:, :4].contiguous(), cp.step_losses) and _flat_equal(lc[:, 4:].contiguous(), cr.step_losses)
    for name in ct.index:
        if name.startswith("RPN/"):
            assert _flat_equal(ct.grads(name), cp.grads(name)), name
        elif name.startswith(HEAD):
            assert _flat_equal(ct.grads(name), cr.grads(name)), name
    worst = max(_rel(_f64(ct.grads(n)), _f64(cp.grads(n)) + _f64(cr.grads(n))) for n in ct.index if n.startswith("trunk/"))
    print("ResNet-50 trunk-gradient worst error (of max-norm): %.2e" % worst)
    assert worst <= 1e-4
    assert set(ct.export_params()) == set(params)


# ------------------------------------------------------------------------------------------------ (7) headline size
def test_headline_size_float64_check():
    """600x1000, N = 1, 300 proposals, the reference's kept set in list mode, explicit masks: the losses and every gradient
    against orc.rpn_train_step + orc.rcnn_train_step in float64 on the same parameters, labels and kept set."""
    from frcnn_b200.train_engine import CanvasJointTrainer
    H, W, post_n = 600, 1000, 300
    params, x, gt, info = _train_case(H, W, 5)
    rng = np.random.default_rng(12)
    for k in ("fc6/W", "fc7/W", "cls_score/W", "bbox_pred/W"):
        params[k] = (rng.standard_normal(params[k].shape) * (0.002 if k == "fc6/W" else 0.01)).astype(f32)
    gt[0, :, 4] = [3, 7, 1]
    xd, gd = torch.from_numpy(np.ascontiguousarray(x[0])).cuda(), torch.from_numpy(gt[0]).cuda()
    ct = CanvasJointTrainer(params, 1, H, W, ANCHORS, post_n=post_n, subsample="device", sample="list", dropout="explicit",
                            seed=2)
    ct.put([xd], [gd], keep_inds=[torch.zeros((0,), dtype=torch.int32)])
    ct.forward()                                             # the proposals, to draw the kept set from
    torch.cuda.synchronize()
    R = int(ct.head_ext[0, 1])
    rois = ct.prop.rois[0, :R].cpu().numpy()
    np.random.seed(5)
    ro = orc.proposal_target_layer(rois, gt)                 # the reference's draw on these proposals
    keep = ro["keep_inds"]
    gen = torch.Generator(device="cuda").manual_seed(3)
    mk = [(torch.rand((post_n, 4096), device="cuda", generator=gen) >= 0.5).to(torch.uint8) for _ in range(2)]
    ct.seeds.sub_(1)                                         # the same anchor draw as the first forward
    ct.put([xd], [gd], keep_inds=[torch.from_numpy(keep)], masks=[mk])
    losses = ct.forward().clone()[0]
    ct.backward()
    torch.cuda.synchronize()
    assert np.array_equal(ct.prop.rois[0, :R].cpu().numpy(), rois)
    tg = ct.rpn.targets
    n_in = int(tg.counts[0, 0])
    inds = tg.inds_inside[0, :n_in].cpu().numpy().astype(np.int64)
    labels, targets = tg.labels_full[0].cpu().numpy()[inds], tg.targets_full[0].cpu().numpy()[inds]
    pt = ct.ptargets
    n_keep = int(pt.counts[0, 0])
    assert n_keep == len(keep) and np.array_equal(pt.keep[0, :n_keep].cpu().numpy(), keep)
    rlabels, ext = pt.labels[0, :n_keep].cpu().numpy(), pt.bbox_reg_targets[0, :n_keep].cpu().numpy()
    masks = [m.cpu().numpy()[:R] for m in mk]
    want_rpn = orc.rpn_train_step(params, x, labels, targets, inds)
    want_rcnn = orc.rcnn_train_step(params, x, rois, keep, rlabels, ext, masks)
    Lv = losses.cpu().numpy()
    want_l = list(want_rpn["losses"]) + list(want_rcnn["losses"])
    print("R=%d kept=%d losses" % (R, n_keep), Lv, "oracle", want_l)
    for i in (0, 1, 3, 4, 5, 7):
        assert abs(Lv[i] - want_l[i]) <= 2e-4 * max(1.0, abs(want_l[i])), i
    assert abs(Lv[6] - want_l[6]) <= 1.0 / len(keep) + 1e-6
    worst = 0.0
    for name in ct.index:
        gdev = ct.grads(name).cpu().numpy()
        if name == "fc6/W":
            gdev = gdev.reshape(4096, 49, 512).transpose(0, 2, 1).reshape(4096, -1)
        want = want_rpn["grads"].get(name, 0.0) + want_rcnn["grads"].get(name, 0.0)
        assert np.abs(want).max() > 0, name
        worst = max(worst, _rel(gdev, want))
    print("end-to-end worst gradient error (of max-norm): %.2e" % worst)
    assert worst <= 3e-2
    ct.update()
    ct.put([xd], [gd], keep_inds=[torch.zeros((0,), dtype=torch.int32)])
    ct.seeds.sub_(1)
    ct.forward()                                             # the updated RPN's proposals: the same draw on them
    torch.cuda.synchronize()
    R2 = int(ct.head_ext[0, 1])
    np.random.seed(5)
    keep2 = orc.proposal_target_layer(ct.prop.rois[0, :R2].cpu().numpy(), gt)["keep_inds"]
    ct.put([xd], [gd], keep_inds=[torch.from_numpy(keep2)], masks=[mk])
    ct.seeds.sub_(1)
    l2 = ct.forward().clone()[0].cpu().numpy()
    print("rpn_loss + loss_rcnn %.5f -> %.5f" % (Lv[3] + Lv[7], l2[3] + l2[7]))
    assert l2[3] + l2[7] < Lv[3] + Lv[7]
