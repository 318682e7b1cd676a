"""The float64 reference of one RPN training update with the ResNet trunk and frozen BatchNorm, the restatement that
tests/test_resnet_train_abi_cpu.py and tests/test_resnet_train_gpu.py hold frcnn_b200.resnet_train.ResNetRpnTrainer to.
It builds on the oracle's ResNet structure (resnet_block_names, BN_EPS) and its RPN label map-up (rpn_labels_mapped)."""
import numpy as np

from frcnn_oracle import BN_EPS, resnet_block_names, rpn_labels_mapped


def resnet_rpn_train_step(params, x, labels, targets, inds_inside, n_layers=101, lr=0.001, momentum=0.9, weight_decay=0.0005,
                          velocity=None, loss_lambda=1.0, delta=3.0, A=9, folded=False):
    """One train_rpn.py update of FasterRCNN(trunk_class=ResNet, rpn_in_ch=2048, feat_stride=32) in RPN mode with FROZEN
    BatchNorm, restated in float64 with torch-CPU autograd (UNPINNED: Chainer is absent).  Every BN applies its stored
    statistics and affine as constants, unfolded: gamma * (conv(x) + b - mean) / sqrt(var + eps) + beta; the pool is
    F.max_pool2d(3, 2, ceil_mode=True) (Chainer's cover_all at pad 0).  Trainable: every trunk convolution's W,
    trunk/conv1/b and RPN/*; BN parameters get no gradient and no weight decay.  labels / targets / inds_inside: an
    AnchorTargetLayer result.  folded=True differentiates the folded convolutions instead (Wf = W*s, bf = beta + (b-mean)*s
    in float64) and returns s * dL/dWf, s * dL/dbf: by the chain rule these equal the unfolded gradients.
    Returns dict(losses=(cls, bbox, acc, total), grads, params, velocity) as rpn_train_step does."""
    import torch
    import torch.nn.functional as F
    td = torch.float64
    blocks = resnet_block_names(n_layers)
    convs = [("trunk/conv1", "trunk/bn1")]
    for stage, blk, cin, mid, cout, stride, proj in blocks:
        base = "trunk/%s/%s" % (stage, blk)
        convs += [(base + "/conv%d" % i, base + "/bn%d" % i) for i in ((1, 2, 3, 4) if proj else (1, 2, 3))]
    names = [c + "/W" for c, _ in convs] + ["trunk/conv1/b"] + [k for k in params if k.startswith("RPN/")]
    T = lambda a: torch.tensor(np.asarray(a, np.float64), dtype=td)          # noqa: E731
    P = {k: T(params[k]).requires_grad_(True) for k in names}
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
    mid = F.relu(F.conv2d(h, P["RPN/rpn_conv_3x3/W"], P["RPN/rpn_conv_3x3/b"], padding=1))
    score = F.conv2d(mid, P["RPN/rpn_cls_score/W"], P["RPN/rpn_cls_score/b"])
    pred = F.conv2d(mid, P["RPN/rpn_bbox_pred/W"], P["RPN/rpn_bbox_pred/b"])
    _, _, fh, fw = score.shape
    t = torch.from_numpy(rpn_labels_mapped(labels, inds_inside, A * fh * fw, A, fh, fw)).long()
    z = score.reshape(1, 2, A, fh, fw)
    valid = t != -1
    loss_cls = F.cross_entropy(z, t, ignore_index=-1) if bool(valid.any()) else z.sum() * 0
    acc = float((z.argmax(1)[valid] == t[valid]).double().mean()) if bool(valid.any()) else 0.0
    p4 = pred.reshape(4, A, -1).permute(2, 1, 0).reshape(-1, 4)
    sel = p4[torch.from_numpy(np.asarray(inds_inside, dtype=np.int64))]
    loss_bbox = F.huber_loss(sel, T(targets), reduction="sum", delta=float(delta)) / p4.shape[0]
    loss = loss_cls + loss_lambda * loss_bbox
    loss.backward()
    grads = {}
    for k in names:
        c = k.rsplit("/", 1)[0]
        if folded and c in leaf:
            Wf, bf = leaf[c]
            src = Wf.grad * S[c].view(-1, 1, 1, 1) if k.endswith("/W") else bf.grad * S[c]
        else:
            src = P[k].grad
        grads[k] = src.detach().numpy().astype(np.float64)
    vel = {k: (np.zeros_like(grads[k]) if velocity is None else np.asarray(velocity[k], np.float64)) for k in names}
    new_p, new_v = {}, {}
    for k in names:
        w = np.asarray(params[k], np.float64)
        v = momentum * vel[k] - lr * (grads[k] + weight_decay * w)
        new_v[k] = v
        new_p[k] = w + v
    return dict(losses=(float(loss_cls.detach()), float(loss_bbox.detach()), acc, float(loss.detach())), grads=grads,
                params=new_p, velocity=new_v)
