"""ResNet-50/101/152 trunk for the forward engine (SURVEY.md 8f rank 2, BASELINE config #4).

The reference's trunk class is /root/reference models/resnet.py:11-45: a thin subclass of the un-vendored
chainer.links.model.vision.resnet.ResNetLayers that returns 'res5' (stride 32, 2048 channels), so the detector is
`FasterRCNN(trunk_class=ResNet, rpn_in_ch=2048, feat_stride=32)` with fc6 reading 2048*7*7 inputs.  Restated structure:

    conv1 7x7/2 p3 (+bias) - bn1 - relu - max_pooling_2d(3, stride=2)      [pad 0, cover_all]
    res2 (64-64-256, stride 1) x3, res3 (128-128-512, /2) x4, res4 (256-256-1024, /2) x23 (101), res5 (512-512-2048, /2) x3
    block 'a'  (BottleneckA): conv1 1x1/s - bn - relu - conv2 3x3 - bn - relu - conv3 1x1 - bn;  shortcut conv4 1x1/s - bn4
    block 'bN' (BottleneckB): same main path, identity shortcut;  out = relu(main + shortcut)

On the device every BatchNormalization (test mode) is folded into the preceding convolution at pack time, every
convolution is the tcgen05 kernel of the VGG path (1x1 = plain GEMM tiles, 3x3 = shared-halo implicit GEMM), conv1 is an
im2col GEMM (K = 147 -> 160), the residual add + ReLU is the epilogue of conv3 (frcnn_conv2d_res), and a stride-2 1x1
convolution is frcnn_subsample2x (shared by conv1 and the projection shortcut) followed by a stride-1 GEMM.

Engines: ResNetEngine runs one image at a time; ResNetBatchEngine adds same-size batches (ResNetBatchPlan) and canvases of
images of different sizes (ResNetCanvasBatchPlan); ResNetPhotoEngine adds raw uint8 photos on a canvas
(ResNetRawCanvasBatchPlan, whose first launch frcnn_preprocess_bgr8_canvas_im2col resizes the photos straight into conv1's
im2col planes), so detect_images and engine.CanvasStreamRunner serve the ResNet detector as they serve VGG16.
"""
import numpy as np
import torch

from . import ops
from ._lib import FrcnnError
from .engine import BatchPlan, CanvasBatchPlan, Engine, ForwardPlan, PackedWeights, _t

RESNET_BLOCKS = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}
RESNET_STAGES = (("res2", 64, 64, 256, 1), ("res3", 256, 128, 512, 2), ("res4", 512, 256, 1024, 2), ("res5", 1024, 512, 2048, 2))
BN_EPS = 2e-5                  # chainer.links.BatchNormalization default
CONV1_KPAD = 160               # 7*7*3 = 147 -> 160 (16-byte rows)


def block_list(n_layers):
    out = []
    for (stage, cin, mid, cout, stride), n in zip(RESNET_STAGES, RESNET_BLOCKS[n_layers]):
        out.append((stage, "a", cin, mid, cout, stride, True))
        for i in range(1, n):
            out.append((stage, "b%d" % i, cout, mid, cout, 1, False))
    return out


def fold_batchnorm(W, gamma, beta, mean, var, bias=None, eps=BN_EPS):
    """Test-mode BN after a convolution == the convolution with W*s and bias beta + (b - mean)*s, s = gamma/sqrt(var+eps).
    float64 host arithmetic (one-time, at weight-pack time), float32 results."""
    s = np.asarray(gamma, np.float64) / np.sqrt(np.asarray(var, np.float64) + eps)
    b0 = np.zeros_like(s) if bias is None else np.asarray(bias, np.float64)
    Wf = (np.asarray(W, np.float64) * s[:, None, None, None]).astype(np.float32)
    bf = (np.asarray(beta, np.float64) + (b0 - np.asarray(mean, np.float64)) * s).astype(np.float32)
    return Wf, bf


class ResNetPackedWeights(PackedWeights):
    def __init__(self, params, n_layers=101, precision="bf16x3", device="cuda", num_classes=21, n_anchors=9):
        self.n_layers = n_layers
        super(ResNetPackedWeights, self).__init__(params, precision, device, num_classes, n_anchors, pool_chw=(2048, 7, 7))

    def _folded(self, params, conv, bn, bias=None):
        return fold_batchnorm(params[conv + "/W"], params[bn + "/gamma"], params[bn + "/beta"], params[bn + "/avg_mean"],
                              params[bn + "/avg_var"], bias)

    def _pack_trunk(self, params, P):
        dev = self.device
        Wf, bf = self._folded(params, "trunk/conv1", "trunk/bn1", params.get("trunk/conv1/b"))
        hi, lo = ops.pack_conv_weights_im2col_general(_t(Wf, dev), CONV1_KPAD, precision=self.precision)
        self.convs["conv1"] = (hi, lo, ops.pad_bias(_t(bf, dev), 64))
        for stage, blk, cin, mid, cout, stride, proj in block_list(self.n_layers):
            base = "trunk/%s/%s" % (stage, blk)
            for ci in ((1, 2, 3, 4) if proj else (1, 2, 3)):
                Wf, bf = self._folded(params, base + "/conv%d" % ci, base + "/bn%d" % ci)
                self.convs["%s/%s/conv%d" % (stage, blk, ci)] = self._pack(_t(Wf, dev), _t(bf, dev), cin_pad=Wf.shape[1])


class ResNetForwardPlan(ForwardPlan):
    """ForwardPlan with the ResNet trunk (the RPN / ProposalLayer / RoI pool / head part is inherited unchanged)."""

    def _alloc_trunk(self, H, W):
        act = self._act
        Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
        self.x_col = act(Ho, Wo, CONV1_KPAD)
        self.c1 = act(Ho, Wo, 64)
        h, w = (Ho - 2) // 2 + 1, (Wo - 2) // 2 + 1
        self.p1 = act(h, w, 64)
        self.blocks = []
        x = self.p1
        for stage, blk, cin, mid, cout, stride, proj in block_list(self.w.n_layers):
            B = dict(name="%s/%s" % (stage, blk), x=x, stride=stride, proj=proj)
            if stride == 2:
                h, w = (h + 1) // 2, (w + 1) // 2
                B["xs"] = act(h, w, cin)                 # the stride-2 1x1 convs read pixels (2h, 2w)
            B["y1"], B["y2"] = act(h, w, mid), act(h, w, mid)
            if proj:
                B["sc"] = act(h, w, cout)
            B["out"] = act(h, w, cout)
            self.blocks.append(B)
            x = B["out"]
        self.acts = [self.x_col, x]                      # acts[-1] is the feature map ('res5')
        return h, w

    def _run_trunk(self):
        cv = self.w.convs
        n = 0
        ops.pack_image_im2col_general(self.x_in, 7, 2, 3, CONV1_KPAD, out=self.x_col)
        hi, lo, b = cv["conv1"]
        ops.conv2d(self.x_col, hi, lo, b, 1, True, out=self.c1)
        ops.maxpool3x3s2_ceil(self.c1, out=self.p1)
        n += 3
        for B in self.blocks:
            x = B["x"]
            if B["stride"] == 2:
                ops.subsample2x(x, out=B["xs"])
                x = B["xs"]
                n += 1
            hi, lo, b = cv[B["name"] + "/conv1"]
            ops.conv2d(x, hi, lo, b, 1, True, out=B["y1"])
            hi, lo, b = cv[B["name"] + "/conv2"]
            ops.conv2d(B["y1"], hi, lo, b, 3, True, out=B["y2"])
            if B["proj"]:
                hi, lo, b = cv[B["name"] + "/conv4"]
                ops.conv2d(x, hi, lo, b, 1, False, out=B["sc"])
                res = B["sc"]
                n += 1
            else:
                res = B["x"]
            hi, lo, b = cv[B["name"] + "/conv3"]
            ops.conv2d_res(B["y2"], hi, lo, b, 1, True, res, out=B["out"])
            n += 3
        return self.blocks[-1]["out"], n


class ResNetBatchPlan(BatchPlan):
    """BatchPlan with the ResNet trunk: N images of one shape in ONE CUDA graph, every launch of ResNetForwardPlan's trunk
    once over all N (frcnn_pack_image_im2col_batch, frcnn_maxpool3x3s2_ceil_batch, frcnn_subsample2x_batch,
    frcnn_conv2d_batch, frcnn_conv2d_res_batch), then BatchPlan's RPN / ProposalLayer / RoI pool / head.  Every image's
    results are bit-identical to a ResNetForwardPlan's on that image.  Takes ForwardPlan's keyword options except
    hwc_input (the 7x7 first layer reads dense (C,H,W) images) and keep_rpn_debug."""
    _trunk_name, _trunk_layer = "ResNet", "conv1"
    _alloc_trunk = ResNetForwardPlan._alloc_trunk      # activations through self._act: [N, ...] planes in a batch
    _takes_raw_input = False                           # ResNetRawCanvasBatchPlan: raw photos on a canvas

    def __init__(self, weights, N, H, W, **options):
        for opt, why in (("raw_input", "raw photos need ResNetRawCanvasBatchPlan"),
                         ("hwc_input", "the 7x7 first layer reads dense (3,H,W) images"),
                         ("keep_rpn_debug", "no RPN debug outputs")):
            if options.get(opt) and not (opt == "raw_input" and self._takes_raw_input):
                raise FrcnnError("%s: %s=True is not supported (%s)" % (type(self).__name__, opt, why))
        super(ResNetBatchPlan, self).__init__(weights, N, H, W, **options)
        # a canvas batch: the extents of conv1, pool1, res3, res4 and res5, derived on the device by the first launch
        self.level_ext = None if self.extents is None else torch.zeros((5, self.N, 2), dtype=torch.int32, device=weights.device)

    def _run_trunk(self):
        cv, lv = self.w.convs, self.level_ext
        ext = lambda k: None if lv is None else lv[k]          # noqa: E731  (level k's [N, 2] extents, halvings 0)
        n = 0
        if lv is not None:
            ops.resnet_level_extents(self.extents, self.H, self.W, out=lv)
            n += 1
        self.input.pack_im2col(self.x_col, 7, 2, 3, CONV1_KPAD)
        hi, lo, b = cv["conv1"]
        ops.conv2d_batch(self.x_col, hi, lo, b, 1, True, out=self.c1, extents=ext(0))
        ops.maxpool3x3s2_ceil_batch(self.c1, out=self.p1, extents=ext(0))
        n += 3
        level = 1
        for B in self.blocks:
            x = B["x"]
            if B["stride"] == 2:
                ops.subsample2x_batch(x, out=B["xs"])
                x = B["xs"]
                level += 1
                n += 1
            e = ext(level)
            hi, lo, b = cv[B["name"] + "/conv1"]
            ops.conv2d_batch(x, hi, lo, b, 1, True, out=B["y1"], extents=e)
            hi, lo, b = cv[B["name"] + "/conv2"]
            ops.conv2d_batch(B["y1"], hi, lo, b, 3, True, out=B["y2"], extents=e)
            if B["proj"]:
                hi, lo, b = cv[B["name"] + "/conv4"]
                ops.conv2d_batch(x, hi, lo, b, 1, False, out=B["sc"], extents=e)
                res = B["sc"]
                n += 1
            else:
                res = B["x"]
            hi, lo, b = cv[B["name"] + "/conv3"]
            ops.conv2d_res_batch(B["y2"], hi, lo, b, 1, True, res, out=B["out"], extents=e)
            n += 3
        return self.blocks[-1]["out"], n

    def _feature_extents(self):
        return (None if self.level_ext is None else self.level_ext[4]), 0


class ResNetCanvasBatchPlan(ResNetBatchPlan, CanvasBatchPlan):
    """CanvasBatchPlan with the ResNet trunk: N images of different sizes, each at the top-left of its Hc x Wc slot, in ONE
    captured graph.  The first launch derives every level's extents from the per-image sizes (frcnn_resnet_level_extents);
    each later launch reads its level's and writes 0 outside every image, so each image's results are bit-identical to a
    ResNetForwardPlan's on that image alone.  Preprocessed float images only: raw photos take ResNetRawCanvasBatchPlan."""


class ResNetRawCanvasBatchPlan(ResNetCanvasBatchPlan):
    """ResNetCanvasBatchPlan on RAW uint8 (h0,w0,3) BGR photos: CanvasBatchPlan(raw_input=True)'s static input (one device
    block [descriptor header | pixels], forward_raw, raw_batch_header, fetch_result), with the ResNet trunk behind it.  After
    the level extents, the first launch (frcnn_preprocess_bgr8_canvas_im2col) resizes every photo as forward.py does,
    subtracts pixel_means and writes conv1's 7x7/2 im2col planes straight from the photos, so the plan holds no float32
    images and one host-to-device copy of the block delivers a whole batch.  The launch count is the float canvas plan's.
    Every image's results are bit-identical to a ResNetForwardPlan's on preprocess.img_preprocessing of that photo alone."""
    _takes_raw_input = True

    def __init__(self, weights, N, Hc, Wc, raw_input=True, **options):
        if not raw_input:
            raise FrcnnError("ResNetRawCanvasBatchPlan takes raw photos only (raw_input=False: use ResNetCanvasBatchPlan)")
        super(ResNetRawCanvasBatchPlan, self).__init__(weights, N, Hc, Wc, raw_input=True, **options)


class ResNetEngine(Engine):
    """`Engine` for FasterRCNN(trunk_class=ResNet, rpn_in_ch=2048, feat_stride=32)."""
    supports_hwc_input = False         # the 7x7 first layer's im2col kernel reads dense (C,H,W) only
    plan_class = ResNetForwardPlan

    def __init__(self, params, n_layers=101, precision="bf16x3", device="cuda", anchors=None, num_classes=21, n_anchors=9,
                 feat_stride=32, **plan_kwargs):
        self.n_layers = n_layers
        super(ResNetEngine, self).__init__(params, precision, device, anchors, num_classes, n_anchors, feat_stride, **plan_kwargs)

    def _pack_weights(self, params, precision, device, num_classes, n_anchors):
        return ResNetPackedWeights(params, self.n_layers, precision, device, num_classes, n_anchors)

    def batch_plan(self, N, H, W, **overrides):
        raise FrcnnError("ResNetEngine runs one image at a time: batches (BatchPlan) need the VGG16 trunk or ResNetBatchEngine")

    def canvas_plan(self, N, Hc, Wc, **overrides):
        raise FrcnnError("ResNetEngine runs one image at a time: canvas batches (CanvasBatchPlan) need the VGG16 trunk or "
                         "ResNetBatchEngine")


class ResNetBatchEngine(ResNetEngine):
    """ResNetEngine that also runs batches: batch_plan() is a ResNetBatchPlan and canvas_plan() a ResNetCanvasBatchPlan, so
    Engine.forward_batch (N same-size images) and Engine.forward_images (images of different sizes on a canvas) run N images
    per graph replay, each image bit-identical to ResNetForwardPlan on it.  Preprocessed float images only: detect_images
    (raw photos) raises FrcnnError before anything is allocated; ResNetPhotoEngine takes raw photos.  ResNetEngine itself
    keeps running one image at a time."""

    def batch_plan(self, N, H, W, **overrides):
        """The ResNetBatchPlan for N images of H x W (cached per shape and options)."""
        return self._cached("batch", ResNetBatchPlan, (N, H, W), overrides)

    def canvas_plan(self, N, Hc, Wc, **overrides):
        """The ResNetCanvasBatchPlan of N slots of Hc x Wc (cached per canvas and options)."""
        return self._cached("canvas", ResNetCanvasBatchPlan, (N, Hc, Wc), overrides)


class ResNetPhotoEngine(ResNetBatchEngine):
    """ResNetBatchEngine that also detects on raw photos: canvas_plan(..., raw_input=True) is a ResNetRawCanvasBatchPlan, so
    Engine.raw_canvas_plan, Engine.detect_images (forward.py's detection lists from uint8 BGR photos of any sizes, N per
    graph replay) and engine.CanvasStreamRunner work as they do for the VGG16 detector."""

    def canvas_plan(self, N, Hc, Wc, **overrides):
        """raw_input=True: the ResNetRawCanvasBatchPlan of N slots of Hc x Wc (cached under its own key); otherwise
        ResNetBatchEngine.canvas_plan."""
        if overrides.get("raw_input"):
            return self._cached("raw_canvas", ResNetRawCanvasBatchPlan, (N, Hc, Wc), overrides)
        return super(ResNetPhotoEngine, self).canvas_plan(N, Hc, Wc, **overrides)


class TrunkOnly(object):
    """The trunk alone (models.resnet.ResNet.__call__): packs only trunk/* and runs ResNetForwardPlan's trunk hooks."""

    class _W(ResNetPackedWeights):
        def __init__(self, params, n_layers, precision, device):        # no RPN / head parameters here
            self.n_layers, self.precision, self.device = n_layers, precision, device
            self.convs = {}
            self._pack_trunk(params, None)

    class _Plan(ResNetForwardPlan):
        def __init__(self, weights, H, W):
            self.w, self.H, self.W = weights, H, W
            dev = weights.device
            x3 = weights.precision == "bf16x3"

            def act(h, w, c):
                hi = torch.empty((h, w, c), dtype=torch.bfloat16, device=dev)
                return ops.Act(hi, torch.empty_like(hi) if x3 else None)
            self._act = act
            self.x_in = torch.zeros((3, H, W), dtype=torch.float32, device=dev)
            self._alloc_trunk(H, W)

    def __init__(self, params, n_layers, precision, device):
        self.weights = self._W(params, n_layers, precision, device)
        self.plans = {}

    def run(self, x_chw):
        _, H, W = x_chw.shape
        if (H, W) not in self.plans:
            self.plans[(H, W)] = self._Plan(self.weights, H, W)
        p = self.plans[(H, W)]
        p.x_in.copy_(x_chw)
        feat, _ = p._run_trunk()
        return feat
