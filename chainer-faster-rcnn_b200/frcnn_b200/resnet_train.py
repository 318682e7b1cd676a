"""The train_rpn.py and train_rcnn.py steps with the ResNet-50/101/152 trunk: `FasterRCNN(trunk_class=ResNet,
rpn_in_ch=2048, feat_stride=32)` with `rpn_train = True` or `rcnn_train = True` (the reference's utils/prepare_train.py
offers --trunk_model ResNet50/101/152).

ResNetRpnTrainer -- forward (conv1 7x7/2 + pool 3x3/2 + bottleneck blocks + RPN) -> AnchorTargetLayer -> rpn_loss -> backward
through the RPN heads, the RPN 3x3 conv and every trunk convolution -> [gradient all-reduce] -> WeightDecay + MomentumSGD.

BatchNorm is FROZEN: every BN layer applies its stored statistics and affine (gamma, beta, avg_mean, avg_var are constants,
not in the flat parameter buffer and not weight-decayed).  The reasons: the reference never ran a batch-statistics ResNet
detector (FasterRCNN calls trunk_class() without n_layers), per-image batch statistics with one image per update would be a
different model from the test-mode BN the forward engines define, and frozen BN is how ResNet Faster R-CNN is trained in
practice (py-faster-rcnn's use_global_stats with the scale layers at lr_mult 0).  Trainable: every trunk convolution's W,
trunk/conv1/b, and the RPN's parameters.

A convolution and its frozen BN are then the folded convolution Wf = W*s, bf = beta + (b - mean)*s, s = gamma/sqrt(var+eps):
    forward          the folded weights, rebuilt from the fp32 masters at every repack (frcnn_fold_batchnorm, the float64
                     arithmetic of resnet_engine.fold_batchnorm) and packed by the forward engines' packers, so the planes
                     equal ResNetPackedWeights' of the exported parameters; the launches are ResNetForwardPlan._run_trunk's
    data gradient    frcnn_conv2d on the folded weights' dgrad planes; the residual sums are the epilogue of
                     frcnn_conv2d_res with relu = 0 (identity block: dgrad_conv1(dy1) + dy3; projection block:
                     dgrad_conv1(dy1) + dgrad_conv4(dy3))
    weight gradient  dW = s[co] * sum dz (x) x, d(conv1/b) = s * sum dz: the split-K GEMM of the folded convolution, reduced
                     in fixed order and scaled per output channel (frcnn_wgrad_reduce_scaled)
    re-layouts       the 3x3/2 cover_all max-pool backward fused with conv1's ReLU mask (frcnn_maxpool3x3s2_backward), and the
                     backward of the stride-2 subsample fused with the ReLU mask of the block output it reads
                     (frcnn_grad_prepare_stride2)
Everything else -- the flat buffers, the RPN step, the loss, the optimizer and the gradient exchange (one bucket, after
backward) -- is shared with the VGG16 trainers (train_engine's _ConvTrainer and _RpnStep).

ResNetRcnnTrainer -- RcnnTrainer's step on the same trunk: trunk -> frozen test-mode RPN (2048 -> 512 3x3, twin heads) ->
ProposalLayer -> ProposalTargetLayer -> RoI pool 7x7 at 1/32 over 2048 channels -> fc6 (K = 2048*49) / fc7 with dropout ->
cls_score | bbox_pred -> losses -> backward through the head, the RoI pooling and every bottleneck -> WeightDecay +
MomentumSGD.  The head, its losses and backward are RcnnTrainer's step (_RcnnStep) with feat_ch = 2048; the trunk
(_ResNetTrunk) is ResNetRpnTrainer's, launch for launch.  Trainable: every trunk convolution's W, trunk/conv1/b, fc6, fc7,
cls_score and bbox_pred; the RPN is packed once and gets no gradient, the BN entries stay constant.

ResNetJointTrainer / CanvasResNetJointTrainer -- JointTrainer's and CanvasJointTrainer's approximate joint training step
(train_engine._JointStep) on the same trunk: the RPN and the head trained together, the feature map's two gradients joined in
the epilogue of the RPN conv's data gradient, then every bottleneck; export_params() adds the BN constants, so it is a
whole detector.
"""
import numpy as np
import torch

from . import ops, train_ops
from ._lib import FrcnnError
from .resnet_engine import BN_EPS, CONV1_KPAD, RESNET_BLOCKS, block_list, fold_batchnorm
from .train_engine import _CanvasJointStep, _CanvasRcnnStep, _CanvasRpnStep, _JointStep, _RcnnStep, _RpnStep

SUBSAMPLE_MODES = ("device", "numpy", "none")
BN_FIELDS = ("gamma", "beta", "avg_mean", "avg_var")


def bn_scale(params, bn):
    """s = gamma / sqrt(var + eps) in float64, as resnet_engine.fold_batchnorm computes it."""
    return np.asarray(params[bn + "/gamma"], np.float64) / np.sqrt(np.asarray(params[bn + "/avg_var"], np.float64) + BN_EPS)


def trunk_convs(n_layers):
    """[(conv name, bn name, cin, cout, k)] of the trunk in flat-buffer order: conv1, then per block conv1..conv3 (+ conv4)."""
    out = [("trunk/conv1", "trunk/bn1", 3, 64, 7)]
    for stage, blk, cin, mid, cout, stride, proj in block_list(n_layers):
        base = "trunk/%s/%s" % (stage, blk)
        out += [(base + "/conv1", base + "/bn1", cin, mid, 1), (base + "/conv2", base + "/bn2", mid, mid, 3),
                (base + "/conv3", base + "/bn3", mid, cout, 1)]
        if proj:
            out.append((base + "/conv4", base + "/bn4", cin, cout, 1))
    return out


class _ResNetTrunk(object):
    """The ResNet trunk with frozen BatchNorm, the trunk of the four ResNet trainers: the layer table and BN constants, the
    activations, the forward launches, the fold + repack, and the bottleneck backward (_backward_trunk, from the gradient
    of the feature map).  Every launch goes through the trainer's launch layer (_conv, _res_conv, _pool3, _subsample,
    _prep, _pool3_backward, _prep_stride2, _pack_input), so the same code runs one image and, with _CanvasSteps' launches,
    a canvas.  A trunk level is an index into frcnn_resnet_level_extents' five: 0 conv1, 1 pool1 / res2, 2 res3, 3 res4,
    4 res5.  The trainer sets n_layers before it is built."""
    feat_ch = 2048
    halvings = 4                        # the feature map's level (res5)
    first_layer = (7, 2, 3, CONV1_KPAD)
    early_exchange = None               # no early bucket: a multi-rank exchange is one bucket after backward
    feat_grad_tag = 3                   # the _gact tag of res5's input gradients, which the RPN conv's data gradient shares

    def _trunk_table(self, H, W, feat_stride):
        """Checks the trunk's options (FrcnnError); returns the trunk convolutions in flat-buffer order and the frozen-BN
        constants [(name, shape)] they read."""
        who, n_layers = type(self).__name__, self.n_layers
        if n_layers not in RESNET_BLOCKS:
            raise FrcnnError("%s: n_layers must be one of %s (got %r)" % (who, sorted(RESNET_BLOCKS), n_layers))
        if feat_stride != 32:
            raise FrcnnError("%s: the ResNet trunk's feature stride is 32 (got feat_stride=%r)" % (who, feat_stride))
        if min((H - 1) // 2 + 1, (W - 1) // 2 + 1) < 3:          # conv1 7x7/2 pad 3
            raise FrcnnError("%s: the image must be at least 5 x 5 (got %d x %d)" % (who, H, W))
        convs = trunk_convs(n_layers)
        layers = [dict(name=n, bn=bn, cin=ci, cout=co, k=k, bias=n == "trunk/conv1") for n, bn, ci, co, k in convs]
        return layers, [("%s/%s" % (bn, f), (co,)) for _, bn, _, co, _ in convs for f in BN_FIELDS]

    def _init_trunk(self, params, H, W, lead):
        """The frozen-BN constants and the trunk activations; on a canvas (lead (N,)) also the per-level extents."""
        dev = self.device
        # ---- frozen BN: s (float64) per conv, the constant folded bias of every conv but conv1, the folded-weight buffers
        T = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dt)     # noqa: E731
        self.conv = {L["name"]: L for L in self.layers if "bn" in L}
        for n, L in self.conv.items():
            bn = L["bn"]
            L["s"] = T(bn_scale(params, bn), torch.float64)
            L["wf"] = torch.empty((L["cout"], L["cin"], L["k"], L["k"]), dtype=torch.float32, device=dev)
            if L["bias"]:
                L["beta"], L["mean"] = T(params[bn + "/beta"]), T(params[bn + "/avg_mean"])
                L["bf"] = torch.empty((L["cout"],), dtype=torch.float32, device=dev)
            else:
                L["bf"] = T(fold_batchnorm(params[n + "/W"], params[bn + "/gamma"], params[bn + "/beta"], params[bn + "/avg_mean"],
                                           params[bn + "/avg_var"])[1])
        self.bn_params = {k: np.asarray(params[k]).copy() for k in ("%s/%s" % (L["bn"], f) for L in self.conv.values()
                                                                    for f in BN_FIELDS)}
        # ---- activations (ResNetForwardPlan._alloc_trunk's, every one kept for backward)
        act = self._act
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        self.x_col = act(Ho, Wo, CONV1_KPAD)
        self.c1 = act(Ho, Wo, 64)
        h, w = (Ho - 2) // 2 + 1, (Wo - 2) // 2 + 1
        self.p1 = act(h, w, 64)
        self.c1_hw = (Ho, Wo)
        self.blocks = []
        x, level = self.p1, 1
        for stage, blk, cin, mid, cout, stride, proj in block_list(self.n_layers):
            B = dict(name="trunk/%s/%s" % (stage, blk), x=x, stride=stride, proj=proj, cin=cin, mid=mid, cout=cout)
            if stride == 2:
                h, w, level = (h + 1) // 2, (w + 1) // 2, level + 1
                B["xs"] = act(h, w, cin)
            B["H"], B["W"], B["level"] = h, w, level
            B["y1"], B["y2"] = act(h, w, mid), act(h, w, mid)
            if proj:
                B["sc"] = act(h, w, cout)
            B["out"] = act(h, w, cout)
            self.blocks.append(B)
            x = B["out"]
        self.fh, self.fw = h, w
        self.db_raw = torch.empty((64,), dtype=torch.float32, device=dev)
        if lead:
            self.level_ext = torch.zeros((5, lead[0], 2), dtype=torch.int32, device=dev)

    def _check_input(self, x_chw, gt_boxes):
        who = type(self).__name__
        if not (torch.is_tensor(x_chw) and x_chw.is_cuda and tuple(x_chw.shape) == (3, self.H, self.W)):
            raise FrcnnError("%s.forward: x_chw must be a (3, %d, %d) CUDA tensor" % (who, self.H, self.W))
        if not (torch.is_tensor(gt_boxes) and gt_boxes.is_cuda and gt_boxes.dim() == 2 and gt_boxes.shape[1] == 5
                and gt_boxes.shape[0] >= 1):
            raise FrcnnError("%s.forward: gt_boxes must be a (G >= 1, 5) CUDA tensor" % who)

    # ---------------------------------------------------------------- weights: fold, then the forward engines' packers
    def _pack_image_layer(self, w, out=None):
        return ops.pack_conv_weights_im2col_general(w, CONV1_KPAD, precision=self.precision, out=out)

    def _pack_image(self, x, out):
        ops.pack_image_im2col_general(x, *self.first_layer, out=out)

    def _repack_trunk(self):
        """Folds and repacks every trunk convolution."""
        for n, L in self.conv.items():
            first = n == "trunk/conv1"
            train_ops.fold_batchnorm(self.weights(n + "/W"), L["s"], L["wf"], b=self.weights(n + "/b") if first else None,
                                     beta=L.get("beta"), mean=L.get("mean"), bf=L["bf"] if first else None)
            self._repack(n, L["wf"], L["bf"], L["cout"], first=first, cin_pad=L["cin"])

    def folded_params(self):
        """{conv name: (Wf, bf)} float32 numpy: the folded weights the device packed at the last repack."""
        return {n: (L["wf"].cpu().numpy().copy(), L["bf"].cpu().numpy().copy()) for n, L in self.conv.items()}

    # ---------------------------------------------------------------- forward
    def _forward_trunk(self, x_chw=None):
        """ResNetForwardPlan._run_trunk's launches (ResNetBatchPlan's on a canvas) on the folded weights, with every
        activation kept."""
        pk = self.packed
        self._pack_input(x_chw)
        fwd, b, _ = pk["trunk/conv1"]
        self._conv(self.x_col, fwd, b, 1, True, 0, out=self.c1)
        self._pool3(self.c1, self.p1, 0)
        for B in self.blocks:
            x, lv = B["x"], B["level"]
            if B["stride"] == 2:
                self._subsample(x, B["xs"])
                x = B["xs"]
            fwd, b, _ = pk[B["name"] + "/conv1"]
            self._conv(x, fwd, b, 1, True, lv, out=B["y1"])
            fwd, b, _ = pk[B["name"] + "/conv2"]
            self._conv(B["y1"], fwd, b, 3, True, lv, out=B["y2"])
            if B["proj"]:
                fwd, b, _ = pk[B["name"] + "/conv4"]
                self._conv(x, fwd, b, 1, False, lv, out=B["sc"])
                res = B["sc"]
            else:
                res = B["x"]
            fwd, b, _ = pk[B["name"] + "/conv3"]
            self._res_conv(B["y2"], fwd, b, 1, True, res, lv, B["out"])
        self.feat = self.blocks[-1]["out"]
        return self.feat

    def input_of(self, B):
        """The activation block B's conv1 and conv4 read: the subsampled input of a stride-2 block, else its input."""
        return B["xs"] if B["stride"] == 2 else B["x"]

    # ---------------------------------------------------------------- backward
    def _dgrad(self, name, dy, ksize, cin, tag, level, res=None):
        """The data gradient of `name` (its folded weights) at trunk level `level`, plus `res` (frcnn_conv2d_res,
        relu = 0) when given."""
        dg = self.packed[name][2]
        h, w, _ = dy.hi.shape[-3:]
        g = self._gact(h, w, cin, tag=tag)
        if res is None:
            self._conv(dy, dg, self.zero_bias, ksize, False, level, out=g)
        else:
            self._res_conv(dy, dg, self.zero_bias, ksize, False, res, level, g)
        return g

    def _backward_trunk(self, g, debug=None):
        """Backward through the bottleneck blocks (last first), pool1 and conv1 from g, the gradient of the feature map
        (ops.Act [fh, fw, 2048]).  debug: receives, per conv name, the incoming gradient ("g_in": w.r.t. the conv's
        post-ReLU output, or w.r.t. the block output for conv3 / conv4, at the subsampled resolution when the next block
        reads it through the stride-2 subsample), the masked / routed gradient w.r.t. the (folded) conv output ("dy") and
        the data gradient the conv passes on ("g_out"; for a block's conv1 the summed gradient of the block input, residual
        included; none for trunk/conv1)."""
        dbg = (lambda a: self._chw(a).clone()) if debug is not None else None        # noqa: E731
        # ---- the bottleneck blocks, last first; `half`: g is w.r.t. the stride-2 subsample of this block's output
        half = False
        for B in reversed(self.blocks):
            g = self._backward_block(B, g, half, debug)
            half = B["stride"] == 2
        # ---- pool1 + conv1: g is w.r.t. p1
        Ho, Wo = self.c1_hw
        dz = self._gact(Ho, Wo, 64)
        dzT = self._tbuf(1, 64, Ho, Wo)
        self._pool3_backward(g, self.c1, self.p1, dz, dzT)
        L = self.conv["trunk/conv1"]
        self._first_layer_wgrad(dzT, Ho, Wo, 64, self.grads("trunk/conv1/W"), scale=L["s"])
        train_ops.bias_grad(dzT, 64, self.db_raw)
        train_ops.wgrad_reduce_scaled(self.db_raw.view(1, 1, 64, 1), 64, 1, L["s"], self.grads("trunk/conv1/b"))
        if debug is not None:
            debug["trunk/conv1"] = dict(g_in=dbg(g), dy=dbg(dz))

    def _backward_block(self, B, g, half, debug):
        """One bottleneck block's backward; g: gradient w.r.t. B["out"] (or its stride-2 subsample when `half`).  Returns
        the gradient w.r.t. the block's conv input (B["xs"] for a stride-2 block, else B["x"])."""
        dbg = lambda a: self._chw(a).clone()          # noqa: E731
        h, w, cin, mid, cout, lv = B["H"], B["W"], B["cin"], B["mid"], B["cout"], B["level"]
        base = B["name"]
        s = lambda i: self.conv["%s/conv%d" % (base, i)]["s"]       # noqa: E731
        # dz: w.r.t. conv3's (folded) output and the shortcut, = g * (out > 0)
        dz = self._gact(h, w, cout)
        dzT = self._tbuf(1, cout, h, w, tag=1)
        if half:
            self._prep_stride2(h, w, cout, g, B["out"], dz, dzT)
        else:
            self._prep(h, w, cout, g=g, y=B["out"], out=dz, tbuf=dzT)
        # conv3 (1x1, mid -> cout)
        y2T = self._tbuf(1, mid, h, w, tag=2)
        self._prep(h, w, mid, g=B["y2"], tbuf=y2T)
        self._wgrad(dzT, y2T, cout, mid, 1, self.grads(base + "/conv3/W"), scale=s(3))
        g2 = self._dgrad(base + "/conv3", dz, 1, mid, 1, lv)
        if debug is not None:
            debug[base + "/conv3"] = dict(g_in=dbg(g), dy=dbg(dz), g_out=dbg(g2))
        # conv2 (3x3, mid -> mid)
        dy2 = self._gact(h, w, mid)
        dyT = self._tbuf(1, mid, h, w)
        self._prep(h, w, mid, g=g2, y=B["y2"], out=dy2, tbuf=dyT)
        if debug is not None:                              # g2's buffer receives g1 below
            debug[base + "/conv2"] = dict(g_in=dbg(g2), dy=dbg(dy2))
        y1T = self._tbuf(3, mid, h, w)
        self._prep(h, w, mid, g=B["y1"], tbuf=y1T)
        self._wgrad(dyT, y1T, mid, mid, 9, self.grads(base + "/conv2/W"), scale=s(2))
        g1 = self._dgrad(base + "/conv2", dy2, 3, mid, 1, lv)
        if debug is not None:
            debug[base + "/conv2"]["g_out"] = dbg(g1)
        # conv1 (1x1, cin -> mid) and conv4 (1x1, cin -> cout) on the same input
        dy1 = self._gact(h, w, mid)
        self._prep(h, w, mid, g=g1, y=B["y1"], out=dy1, tbuf=dyT)
        if debug is not None:
            debug[base + "/conv1"] = dict(g_in=dbg(g1), dy=dbg(dy1))
        xT = self._tbuf(1, cin, h, w, tag=3)
        self._prep(h, w, cin, g=self.input_of(B), tbuf=xT)
        self._wgrad(dyT, xT, mid, cin, 1, self.grads(base + "/conv1/W"), scale=s(1))
        if B["proj"]:
            self._wgrad(dzT, xT, cout, cin, 1, self.grads(base + "/conv4/W"), scale=s(4))
            res = self._dgrad(base + "/conv4", dz, 1, cin, 2, lv)
            if debug is not None:
                debug[base + "/conv4"] = dict(g_in=dbg(g), dy=dbg(dz), g_out=dbg(res))
        else:
            res = dz
        gx = self._dgrad(base + "/conv1", dy1, 1, cin, 3, lv, res=res)
        if debug is not None:
            debug[base + "/conv1"]["g_out"] = dbg(gx)
        return gx


class ResNetRpnTrainer(_ResNetTrunk, _RpnStep):
    """Weights, optimizer state and buffers of the RPN-mode training step with the ResNet trunk for one image shape.  The
    surface is RpnTrainer's: forward / backward(debug) / update / step / weights / grads / export_params, subsample modes
    "device", "numpy" and "none", disable_pos.  `params` follows oracle.make_resnet_params / models.resnet.ResNet naming;
    its BN entries are read once and stay constant."""

    def __init__(self, params, H, W, anchors, n_layers=101, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=32, loss_lambda=1.0, delta=3.0, subsample="device", seed=0, device="cuda", process_group=None,
                 optimizer=None):
        if subsample not in SUBSAMPLE_MODES:
            raise FrcnnError("ResNetRpnTrainer: subsample must be one of %s (got %r)" % (SUBSAMPLE_MODES, subsample))
        self.n_layers = n_layers
        self._init_rpn(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                       loss_lambda, delta, subsample, seed, optimizer=optimizer)

    def forward(self, x_chw, gt_boxes, im_info=None, disable_pos=None):
        """x_chw (3,H,W) float32 CUDA; gt_boxes [G,5] float32 CUDA.  Returns losses float32[4] (device), as RpnTrainer."""
        self._check_input(x_chw, gt_boxes)
        return super(ResNetRpnTrainer, self).forward(x_chw, gt_boxes, im_info, disable_pos)


class ResNetRcnnTrainer(_ResNetTrunk, _RcnnStep):
    """Weights, optimizer state and buffers of the RCNN-mode training step (train_rcnn.py) with the ResNet trunk for one
    image shape.  The surface is RcnnTrainer's: forward(x, gt, im_info, keep_inds, masks) / backward(debug) / update / step
    / weights / grads / export_params, sample="numpy" (a seeded run draws the reference's kept set), keep_inds= and masks=
    pins.  backward(debug=...) fills RcnnTrainer's head entries ("heads", "fc7", "fc6", "roi") and ResNetRpnTrainer's
    per-convolution entries.  `params` follows oracle.make_resnet_params / models.resnet.ResNet naming; the BN entries and
    the RPN are read once and stay constant.  fc6/W is held in the (h, w, c) column order the RoI pool emits, c = 2048;
    export_params returns the reference's (c, h, w)."""

    def __init__(self, params, H, W, anchors, n_layers=101, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=32, num_classes=21, delta=1.0, post_n=300, pre_n=6000, nms_thresh=0.7, min_size=16,
                 sample="numpy", seed=0, dropout=True, device="cuda", process_group=None, optimizer=None):
        self.n_layers = n_layers
        self._init_rcnn(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                        num_classes, delta, post_n, pre_n, nms_thresh, min_size, sample, seed, dropout, optimizer=optimizer)

    def forward(self, x_chw, gt_boxes, im_info=None, keep_inds=None, masks=None):
        """x_chw (3,H,W) float32 CUDA; gt_boxes [G,5] float32 CUDA.  Returns losses float32[4] (device), as RcnnTrainer."""
        self._check_input(x_chw, gt_boxes)
        return super(ResNetRcnnTrainer, self).forward(x_chw, gt_boxes, im_info, keep_inds, masks)


class CanvasResNetRpnTrainer(_ResNetTrunk, _CanvasRpnStep):
    """CanvasRpnTrainer's step with the ResNet trunk: N images of different sizes per update (put / put_raw / forward /
    backward(debug) / update / run / step / step_raw, per-slot losses [N, 4]), one set of weights with ResNetRpnTrainer's
    parameters, frozen BatchNorm and folded_params().

    The trunk is _ResNetTrunk's, launch for launch, through _CanvasSteps' launches: the first launch of the step derives
    the extents of the five levels from the staged sizes (frcnn_resnet_level_extents, as ResNetCanvasBatchPlan does),
    every convolution, pool and RPN / target / loss launch reads its level's [N][2] extents with halvings 0, and the
    backward runs the _batch re-layouts (frcnn_maxpool3x3s2_backward_batch, frcnn_grad_prepare_stride2_batch,
    frcnn_grad_prepare_batch) and weight-gradient GEMMs over K = N*Kp.  So the gradient is the SUM of the N per-image
    gradients, followed by one WeightDecay + MomentumSGD update; inside each image every activation, masked gradient and
    data gradient equals ResNetRpnTrainer's on that image alone, bit for bit.

    subsample "device": slot n of step t draws with seed + t*N + n; "list": put() takes per-image disable lists; "none":
    labels before subsampling.  raw_input=True: put_raw takes raw photos and the VOC transform runs on the device,
    straight into conv1's 7x7/2 im2col planes, augmented as CanvasRpnTrainer's augment / scales / flip describe.  The step is captured after the first call in a single process and runs
    eagerly with a process group of more than one rank; the gradient exchange is then one bucket after backward (the
    ResNet trunk names no early-exchange layer)."""

    def __init__(self, params, N, Hc, Wc, anchors, n_layers=101, precision="bf16x3", lr=0.001, momentum=0.9,
                 weight_decay=0.0005, feat_stride=32, loss_lambda=1.0, delta=3.0, subsample="device", seed=0, max_gt=256,
                 device="cuda", process_group=None, raw_input=False, optimizer=None, augment=None, scales=(600,), flip=True):
        self.n_layers = n_layers
        self._init_canvas_rpn(params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, loss_lambda,
                              delta, subsample, seed, max_gt, device, process_group, raw_input, optimizer=optimizer,
                              augment=augment, scales=scales, flip=flip)


class CanvasResNetRcnnTrainer(_ResNetTrunk, _CanvasRcnnStep):
    """CanvasRcnnTrainer's step with the ResNet trunk: N images of different sizes per update, with ResNetRcnnTrainer's
    parameters (the head on res5's 2048-channel RoIs, fc6 with K = 2048*49; the RPN frozen and packed once; frozen
    BatchNorm) and CanvasRcnnTrainer's surface, sample ("device" | "list") and dropout ("device" | "explicit" | None)
    modes.  The trunk runs as in CanvasResNetRpnTrainer; RoI pooling and its backward read res5's level extents.  Inside
    each image every activation and data gradient equals ResNetRcnnTrainer's on that image with the same kept rows and
    masks, bit for bit; the gradient is the sum over the slots, then one WeightDecay + MomentumSGD update.  The gradient
    exchange of a multi-rank run is one bucket after backward, as in CanvasResNetRpnTrainer."""

    def __init__(self, params, N, Hc, Wc, anchors, n_layers=101, precision="bf16x3", lr=0.001, momentum=0.9,
                 weight_decay=0.0005, feat_stride=32, num_classes=21, delta=1.0, post_n=300, pre_n=6000, nms_thresh=0.7,
                 min_size=16, sample="device", dropout="device", seed=0, max_gt=256, device="cuda", process_group=None,
                 raw_input=False, optimizer=None, augment=None, scales=(600,), flip=True):
        self.n_layers = n_layers
        self._init_canvas_rcnn(params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, num_classes,
                               delta, post_n, pre_n, nms_thresh, min_size, sample, dropout, seed, max_gt, device,
                               process_group, raw_input, optimizer=optimizer, augment=augment, scales=scales, flip=flip)


def _export_detector(self):
    """export_params() with the frozen BatchNorm constants: a whole detector, which ResNetEngine loads as it stands."""
    return dict(self.bn_params, **_JointStep.export_params(self))


class ResNetJointTrainer(_ResNetTrunk, _JointStep):
    """JointTrainer's approximate joint training step with the ResNet trunk for one image shape: one trunk forward, the
    trained RPN (2048 -> 512 3x3, twin heads) once, rpn_loss and ProposalLayer from its output, the head on res5's RoIs and
    loss_rcnn; backward of their sum, the feature map's two gradients joined in the epilogue of the RPN conv's data
    gradient, through every bottleneck.  The surface is JointTrainer's (forward(x, gt, im_info, disable_pos, keep_inds,
    masks) -> float32[8], backward(debug), update, step, export_params), with folded_params(); the arguments are
    ResNetRpnTrainer's and ResNetRcnnTrainer's, rpn_delta and rcnn_delta being their deltas.  The BN entries stay constant;
    export_params() holds every parameter of the detector: the trunk's, the RPN's, the head's and the BN constants."""
    export_params = _export_detector

    def __init__(self, params, H, W, anchors, n_layers=101, precision="bf16x3", lr=0.001, momentum=0.9, weight_decay=0.0005,
                 feat_stride=32, loss_lambda=1.0, rpn_delta=3.0, subsample="device", num_classes=21, rcnn_delta=1.0,
                 post_n=300, pre_n=6000, nms_thresh=0.7, min_size=16, sample="numpy", seed=0, dropout=True, device="cuda",
                 process_group=None, optimizer=None):
        self.n_layers = n_layers
        self._init_joint(params, H, W, anchors, precision, lr, momentum, weight_decay, feat_stride, device, process_group,
                         loss_lambda, rpn_delta, subsample, num_classes, rcnn_delta, post_n, pre_n, nms_thresh, min_size,
                         sample, seed, dropout, optimizer=optimizer)

    def forward(self, x_chw, gt_boxes, im_info=None, disable_pos=None, keep_inds=None, masks=None):
        """x_chw (3,H,W) float32 CUDA; gt_boxes [G,5] float32 CUDA.  Returns losses float32[8] (device), as JointTrainer."""
        self._check_input(x_chw, gt_boxes)
        return super(ResNetJointTrainer, self).forward(x_chw, gt_boxes, im_info, disable_pos, keep_inds, masks)


class CanvasResNetJointTrainer(_ResNetTrunk, _CanvasJointStep):
    """CanvasJointTrainer's step with the ResNet trunk: N images of different sizes per update, per-slot losses [N, 8], one
    set of weights with ResNetJointTrainer's parameters, frozen BatchNorm and folded_params().  The trunk runs as in
    CanvasResNetRpnTrainer, the RPN half as there and the head half as in CanvasResNetRcnnTrainer; draws, pins, raw input
    and augmentation are CanvasJointTrainer's.  A multi-rank run stays eager with one exchange bucket after backward.
    export_params() is ResNetJointTrainer's."""
    export_params = _export_detector

    def __init__(self, params, N, Hc, Wc, anchors, n_layers=101, precision="bf16x3", lr=0.001, momentum=0.9,
                 weight_decay=0.0005, feat_stride=32, loss_lambda=1.0, rpn_delta=3.0, subsample="device", num_classes=21,
                 rcnn_delta=1.0, post_n=300, pre_n=6000, nms_thresh=0.7, min_size=16, sample="device", dropout="device",
                 seed=0, max_gt=256, device="cuda", process_group=None, raw_input=False, optimizer=None, augment=None,
                 scales=(600,), flip=True):
        self.n_layers = n_layers
        self._init_canvas_joint(params, N, Hc, Wc, anchors, precision, lr, momentum, weight_decay, feat_stride, loss_lambda,
                                rpn_delta, subsample, num_classes, rcnn_delta, post_n, pre_n, nms_thresh, min_size, sample,
                                dropout, seed, max_gt, device, process_group, raw_input, optimizer=optimizer, augment=augment,
                                scales=scales, flip=flip)
