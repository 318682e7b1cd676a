"""The float64 reference of one RCNN training update with the ResNet trunk and frozen BatchNorm, the restatement that
tests/test_resnet_rcnn_train_cpu.py and tests/test_resnet_rcnn_train_gpu.py hold
frcnn_b200.resnet_train.ResNetRcnnTrainer to.  Its trunk restates resnet_train_oracle.resnet_rpn_train_step's (the
oracle's ResNet structure, every BN frozen, unfolded or folded); its head is frcnn_oracle.rcnn_train_step's, with the RoI
pooling at 1/32 over res5's 2048 channels."""
import numpy as np

from frcnn_oracle import BN_EPS, resnet_block_names


def _frozen_bn_trunk(params, x, n_layers, folded, P, T):
    """The trunk forward in float64 autograd with every BN frozen.  P: the trainable leaves by name (every trunk
    convolution's W and trunk/conv1/b); folded=True differentiates the folded convolutions instead.  Returns (res5, grad)
    where grad(k) is dL/d(k) after backward: s * dL/dWf, s * dL/dbf for a folded convolution, which equal the unfolded
    gradients by the chain rule."""
    import torch
    import torch.nn.functional as F
    blocks = resnet_block_names(n_layers)
    convs = [("trunk/conv1", "trunk/bn1")]
    for stage, blk, cin, mid, cout, stride, proj in blocks:
        base = "trunk/%s/%s" % (stage, blk)
        convs += [(base + "/conv%d" % i, base + "/bn%d" % i) for i in ((1, 2, 3, 4) if proj else (1, 2, 3))]
    S = {c: T(params[bn + "/gamma"]) / torch.sqrt(T(params[bn + "/avg_var"]) + BN_EPS) for c, bn in convs}
    leaf = {}
    if folded:
        for c, bn in convs:
            b0 = T(params["trunk/conv1/b"]) if c == "trunk/conv1" else torch.zeros_like(S[c])
            leaf[c] = ((T(params[c + "/W"]) * S[c].view(-1, 1, 1, 1)).requires_grad_(True),
                       (T(params[bn + "/beta"]) + (b0 - T(params[bn + "/avg_mean"])) * S[c]).requires_grad_(True))
    bn_of = dict(convs)

    def cbn(h, conv, stride=1, pad=0, relu_=True):
        if folded:
            Wf, bf = leaf[conv]
            y = F.conv2d(h, Wf, bf, stride=stride, padding=pad)
        else:
            bn = bn_of[conv]
            y = F.conv2d(h, P[conv + "/W"], P.get(conv + "/b"), stride=stride, padding=pad)
            g, b_, m, v = (T(params[bn + "/" + k]).view(1, -1, 1, 1) for k in ("gamma", "beta", "avg_mean", "avg_var"))
            y = g * (y - m) / torch.sqrt(v + BN_EPS) + b_
        return F.relu(y) if relu_ else y
    h = cbn(T(x), "trunk/conv1", stride=2, pad=3)
    h = F.max_pool2d(h, 3, 2, ceil_mode=True)
    for stage, blk, cin, mid, cout, stride, proj in blocks:
        base = "trunk/%s/%s" % (stage, blk)
        y = cbn(h, base + "/conv1", stride=stride)
        y = cbn(y, base + "/conv2", pad=1)
        y = cbn(y, base + "/conv3", relu_=False)
        sc = cbn(h, base + "/conv4", stride=stride, relu_=False) if proj else h
        h = F.relu(y + sc)

    def grad(k):
        c = k.rsplit("/", 1)[0]
        if folded and c in leaf:
            Wf, bf = leaf[c]
            return Wf.grad * S[c].view(-1, 1, 1, 1) if k.endswith("/W") else bf.grad * S[c]
        return P[k].grad
    return h, grad


def trunk_param_names(n_layers):
    """The trainable trunk parameters: every convolution's W, then trunk/conv1/b."""
    names = ["trunk/conv1/W"]
    for stage, blk, cin, mid, cout, stride, proj in resnet_block_names(n_layers):
        base = "trunk/%s/%s" % (stage, blk)
        names += [base + "/conv%d/W" % i for i in ((1, 2, 3, 4) if proj else (1, 2, 3))]
    return names + ["trunk/conv1/b"]


def _momentum_update(params, grads, names, velocity, lr, momentum, weight_decay):
    vel = {k: (np.zeros_like(grads[k]) if velocity is None else np.asarray(velocity[k], np.float64)) for k in names}
    new_p, new_v = {}, {}
    for k in names:
        w = np.asarray(params[k], np.float64)
        v = momentum * vel[k] - lr * (grads[k] + weight_decay * w)
        new_v[k] = v
        new_p[k] = w + v
    return new_p, new_v


def resnet_rcnn_train_step(params, x, rois, keep_inds, labels, bbox_reg_targets, masks=None, n_layers=101, lr=0.001,
                           momentum=0.9, weight_decay=0.0005, velocity=None, delta=1.0, folded=False):
    """One train_rcnn.py update of FasterRCNN(trunk_class=ResNet, rpn_in_ch=2048, feat_stride=32) in RCNN mode with FROZEN
    BatchNorm: frcnn_oracle.rcnn_train_step's head on resnet_rpn_train_step's trunk, restated in float64 with torch-CPU
    autograd (UNPINNED: Chainer is absent).  rois (R,4): the proposals of the frozen test-mode RPN (plain arrays: no
    gradient reaches the RPN); keep_inds / labels / bbox_reg_targets: a ProposalTargetLayer result; masks: the two dropout
    keep-masks (R,4096) or None, applied as x*mask*2.  RoI pooling at 1/32 over res5's 2048 channels; fc6/W in the
    reference's (c, h, w) column order.  Trainable: every trunk convolution's W, trunk/conv1/b, fc6, fc7, cls_score and
    bbox_pred.  folded=True differentiates the folded trunk convolutions (see _frozen_bn_trunk).
    Returns dict(losses=(cls, bbox, acc, total), grads, params, velocity, head=(R, 5*num_classes))."""
    import torch
    import torch.nn.functional as F
    import torchvision
    td = torch.float64
    names = trunk_param_names(n_layers) + [k for k in params if k.split("/")[0] in ("fc6", "fc7", "cls_score", "bbox_pred")]
    T = lambda a: torch.tensor(np.asarray(a, np.float64), dtype=td)          # noqa: E731
    P = {k: T(params[k]).requires_grad_(True) for k in names}
    h, grad = _frozen_bn_trunk(params, x, n_layers, folded, P, T)
    R = len(rois)
    brois = torch.cat([torch.zeros((R, 1), dtype=td), T(rois)], dim=1)
    pool5 = torchvision.ops.roi_pool(h, brois, (7, 7), 1.0 / 32)
    a6 = F.relu(F.linear(pool5.reshape(R, -1), P["fc6/W"], P["fc6/b"]))
    if masks is not None:
        a6 = a6 * T(masks[0]) * 2.0
    a7 = F.relu(F.linear(a6, P["fc7/W"], P["fc7/b"]))
    if masks is not None:
        a7 = a7 * T(masks[1]) * 2.0
    cls = F.linear(a7, P["cls_score/W"], P["cls_score/b"])
    bb = F.linear(a7, P["bbox_pred/W"], P["bbox_pred/b"])
    keep = torch.from_numpy(np.asarray(keep_inds, dtype=np.int64))
    t = torch.from_numpy(np.asarray(labels, dtype=np.int64))
    loss_cls = F.cross_entropy(cls[keep], t)
    loss_bbox = F.huber_loss(bb[keep], T(bbox_reg_targets), reduction="sum", delta=float(delta)) / len(keep)
    loss = loss_cls + loss_bbox
    loss.backward()
    acc = float((cls[keep].argmax(1) == t).double().mean())
    grads = {k: grad(k).detach().numpy().astype(np.float64) for k in names}
    new_p, new_v = _momentum_update(params, grads, names, velocity, lr, momentum, weight_decay)
    return dict(losses=(float(loss_cls.detach()), float(loss_bbox.detach()), acc, float(loss.detach())), grads=grads,
                params=new_p, velocity=new_v, head=torch.cat([cls, bb], 1).detach().numpy())
