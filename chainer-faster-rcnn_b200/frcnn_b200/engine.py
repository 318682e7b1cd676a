"""The whole Faster R-CNN forward detection path as one replayable CUDA graph.

Mirrors FasterRCNN.__call__ (inference branch, /root/reference models/faster_rcnn.py:92-134,175-178):

    input                                    frcnn_pack_image_im2col3x3 (float CHW) or frcnn_preprocess_bgr8 (raw uint8)
    trunk (models/vgg16.py:38-82)            13x frcnn_conv2d(3x3)+ReLU (first layer = K=32 GEMM over the im2col image),
                                             the 4 ceil-mode 2x2 max-pools fused into the producing conv's epilogue
    RPN   (models/region_proposal_network.py:117-124)
                                             frcnn_conv2d(3x3)+ReLU, ONE frcnn_conv2d(1x1) for the twin
                                             heads (18 cls + 36 bbox -> fp32 [H*W, 64])
    ProposalLayer (models/proposal_layer.py:102-198)
                                             frcnn_proposals (18-way softmax fused, NHWC logits in)
    RoI pool + head (models/faster_rcnn.py:123-134)
                                             frcnn_roi_pool, frcnn_conv2d as GEMM for fc6 / fc7 /
                                             (cls_score | bbox_pred merged: 105 -> fp32 [R, 128])
    tail  (models/faster_rcnn.py:175-178)    frcnn_head_decode (softmax + decode + clip)
    caller's per-class NMS (forward.py:48-57) frcnn_detect (optional)

All buffers are allocated once per (image shape, mode); the data-dependent RoI count stays on the
device (rows past it are zero) so the launch sequence is static and is captured into a CUDA graph.
"""
import collections
import threading
import time

import numpy as np
import torch

from . import ops, preprocess
from ._lib import FrcnnError

_CAPTURE_LOCK = threading.Lock()
# diagnostic hook: a list that receives, per ForwardPlan.forward_host call, the host-side milliseconds of
# (pageable->pinned copy, H2D enqueue, graph replay enqueue, D2H enqueue + wait for the result); None = off
HOST_PROFILE = None

VGG16_LAYERS = [
    ("conv1_1", 3, 64), ("conv1_2", 64, 64), "pool",
    ("conv2_1", 64, 128), ("conv2_2", 128, 128), "pool",
    ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), "pool",
    ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3", 512, 512), "pool",
    ("conv5_1", 512, 512), ("conv5_2", 512, 512), ("conv5_3", 512, 512),
]

# one VGG16 conv layer of a plan: `halvings` 2x2 pools precede its input, fused_pool = the following pool runs in its
# epilogue, pool_after = it runs as a stand-alone max-pool; (out_h, out_w) is the layer's output (after a fused pool)
TrunkStep = collections.namedtuple("TrunkStep", "name cin cout halvings fused_pool pool_after out_h out_w")


def vgg16_schedule(H, W, fuse_pool):
    """The VGG16 trunk on an H x W image: ([TrunkStep] per conv layer, feature-map (h, w)).  Every 2x2 pool is ceil-mode."""
    steps, h, w, k = [], H, W, 0
    for i, item in enumerate(VGG16_LAYERS):
        if item == "pool":
            continue
        pooled = i + 1 < len(VGG16_LAYERS) and VGG16_LAYERS[i + 1] == "pool"
        fused = fuse_pool and pooled
        if fused:
            h, w = (h + 1) // 2, (w + 1) // 2
        steps.append(TrunkStep(item[0], item[1], item[2], k, fused, pooled and not fused, h, w))
        if pooled:
            k += 1
            if not fused:
                h, w = (h + 1) // 2, (w + 1) // 2
    return steps, (h, w)


def _t(a, device):
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=torch.float32)
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)


class PackedWeights(object):
    """Reference-named fp32 parameters (trunk/conv1_1/W ... bbox_pred/b, SURVEY.md 5) repacked once
    into the kernels' layouts: [taps, Cout, Cin] bf16 hi(/lo) + padded fp32 bias."""

    def __init__(self, params, precision="bf16x3", device="cuda", num_classes=21, n_anchors=9,
                 pool_chw=(512, 7, 7)):
        if precision not in ops.PRECISIONS:
            raise FrcnnError("unknown precision %r" % (precision,))
        self.precision, self.device = precision, device
        self.num_classes, self.n_anchors = num_classes, n_anchors
        P = lambda k: _t(params[k], device)
        self.convs = {}
        self._pack_trunk(params, P)
        self.rpn3 = self._pack(P("RPN/rpn_conv_3x3/W"), P("RPN/rpn_conv_3x3/b"))
        # twin 1x1 heads merged along Cout: rows [0,2A) = rpn_cls_score, [2A,6A) = rpn_bbox_pred
        wh = torch.cat([P("RPN/rpn_cls_score/W"), P("RPN/rpn_bbox_pred/W")], dim=0)
        bh = torch.cat([P("RPN/rpn_cls_score/b"), P("RPN/rpn_bbox_pred/b")], dim=0)
        self.rpn_ld = ops.round_up(6 * n_anchors, 32)
        self.rpn_heads = self._pack(wh, bh, n_bias=self.rpn_ld)
        self.fc6 = self._pack(P("fc6/W"), P("fc6/b"), perm_chw=pool_chw)
        self.fc7 = self._pack(P("fc7/W"), P("fc7/b"))
        wc = torch.cat([P("cls_score/W"), P("bbox_pred/W")], dim=0)
        bc = torch.cat([P("cls_score/b"), P("bbox_pred/b")], dim=0)
        self.head_ld = ops.round_up(5 * num_classes, 32)
        self.head = self._pack(wc, bc, n_bias=self.head_ld)
        torch.cuda.synchronize(device)

    def _pack_trunk(self, params, P):
        """VGG16 (models/vgg16.py:38-69); subclasses pack another trunk (resnet_engine.ResNetPackedWeights)."""
        for item in VGG16_LAYERS:
            if item == "pool":
                continue
            name, cin, cout = item
            w = P("trunk/%s/W" % name)
            if cin <= 3:
                # first layer as a K = 3 x 32 GEMM over the compact [H][W+2][8] image (ops.pack_image_c8 / conv3x3_c8)
                hi, lo = ops.pack_conv_weights_c8(w, precision=self.precision)
                b = P("trunk/%s/b" % name)
                self.convs[name] = (hi, lo, ops.pad_bias(b, b.numel()))
            else:
                self.convs[name] = self._pack(w, P("trunk/%s/b" % name), cin_pad=cin)

    def _pack(self, w, b, cin_pad=None, perm_chw=None, n_bias=0):
        hi, lo = ops.pack_conv_weights(w, cin_pad=cin_pad, precision=self.precision, perm_chw=perm_chw)
        return hi, lo, ops.pad_bias(b, max(n_bias, b.numel()))


def _result_layout(post_n, NC):
    """Every per-image result lives in ONE device block (4-byte words) so that a host caller gets all of it with a single
    D2H transfer: [count | prob | boxes | rois | scores | keep_count | conf_count | keep_idx].  Returns ({name: (offset,
    words)}, block words)."""
    sizes = [("count", 4), ("prob", post_n * NC), ("boxes", post_n * 4 * NC), ("rois", post_n * 4), ("scores", post_n),
             ("keep_count", NC - 1), ("conf_count", NC - 1), ("keep_idx", (NC - 1) * post_n)]
    layout, off = {}, 0
    for name, n_ in sizes:
        layout[name] = (off, n_)
        off += (n_ + 3) // 4 * 4
    return layout, off


def _unpack_block(words, L, post_n, NC, with_detect):
    f = words.view(np.float32)
    R = int(words[L["count"][0]])
    sl = lambda a, name: a[L[name][0]: L[name][0] + L[name][1]]          # noqa: E731
    out = dict(count=R, prob=sl(f, "prob").reshape(post_n, NC)[:R], boxes=sl(f, "boxes").reshape(post_n, 4 * NC)[:R],
               rois=sl(f, "rois").reshape(post_n, 4)[:R], scores=sl(f, "scores")[:R])
    if with_detect:
        out.update(keep_idx=sl(words, "keep_idx").reshape(NC - 1, post_n), keep_count=sl(words, "keep_count"),
                   conf_count=sl(words, "conf_count"))
    return out


class _PlanBase(object):
    """What ForwardPlan (one image) and BatchPlan (N images of one shape) share: the keyword options, the VGG16 trunk's
    activations, the result blocks and the host-array front end.  Each keeps its own launch sequence (_run)."""
    _lead = ()          # leading dimensions of every activation and of the result blocks: (N,) in a BatchPlan

    def __init__(self, weights, H, W, pre_n=6000, post_n=300, nms_thresh=0.7, min_size=16, feat_stride=16, anchors=None,
                 with_detect=False, det_nms_thresh=0.3, det_conf=0.8, use_graph=True, keep_rpn_debug=False, fuse_pool=True,
                 hwc_input=False):
        if anchors is None:
            raise FrcnnError("%s needs the [A,4] float64 anchor table" % type(self).__name__)
        self.w, self.H, self.W = weights, H, W
        self._ctor = dict(pre_n=pre_n, post_n=post_n, nms_thresh=nms_thresh, min_size=min_size, feat_stride=feat_stride,
                          anchors=anchors, with_detect=with_detect, det_nms_thresh=det_nms_thresh, det_conf=det_conf,
                          use_graph=use_graph, keep_rpn_debug=keep_rpn_debug, fuse_pool=fuse_pool, hwc_input=hwc_input)
        self.pre_n, self.post_n, self.nms_thresh, self.min_size, self.feat_stride = pre_n, post_n, nms_thresh, min_size, feat_stride
        self.with_detect, self.det_nms_thresh, self.det_conf = with_detect, det_nms_thresh, det_conf
        self.use_graph, self.keep_rpn_debug, self.fuse_pool = use_graph, keep_rpn_debug, fuse_pool
        # hwc_input: the static input holds the bytes of dense (H,W,3) float32 images (what a forward.py-style caller's
        # `img.transpose(2,0,1).astype(np.float32)` really is in memory); the first kernel reads them with HWC strides
        self.hwc_input = bool(hwc_input)
        self.anchors = torch.from_numpy(np.ascontiguousarray(anchors, dtype=np.float64)).to(weights.device)
        self._host = None
        self.graph = None
        self.im_h, self.im_w = H, W
        self.n_launches = 0

    def _act(self, *shape, zero=False):
        """Activation planes of `shape` behind the plan's leading dimensions: bf16 hi, and lo in bf16x3."""
        new, like = (torch.zeros, torch.zeros_like) if zero else (torch.empty, torch.empty_like)
        hi = new(self._lead + shape, dtype=torch.bfloat16, device=self.w.device)
        return ops.Act(hi, like(hi) if self.w.precision == "bf16x3" else None)

    def _alloc_trunk(self, H, W):
        """VGG16 activations; returns the feature-map size.  (resnet_engine.ResNetForwardPlan overrides both trunk hooks.)"""
        self.acts = [self._act(ops._lib.load().frcnn_image_c8_elems(H, W))]     # compact first-layer input: [H][W+2][8] (+ slack)
        self.trunk, feat_hw = vgg16_schedule(H, W, self.fuse_pool)
        self.trunk_steps = [(s.name, s.fused_pool, s.pool_after) for s in self.trunk]
        for s in self.trunk:
            self.acts.append(self._act(s.out_h, s.out_w, s.cout))
            if s.pool_after:
                self.acts.append(self._act((s.out_h + 1) // 2, (s.out_w + 1) // 2, s.cout))
        return feat_hw

    def _alloc_result(self, n):
        """n result blocks (_result_layout) in ONE int32 buffer, so a host caller gets everything with one D2H; prob, boxes
        and det are [n, ...] views into them.  Returns the (rois, scores, count) views that ProposalLayer writes."""
        post_n, NC = self.post_n, self.w.num_classes
        L, bw = self.result_layout, self.block_words = _result_layout(post_n, NC)
        self.result_words_nodetect = L["keep_count"][0]
        self.result = torch.zeros((n * bw,), dtype=torch.int32, device=self.w.device)
        blocks = self.result.view(n, bw)
        bf = blocks.view(torch.float32)
        seg = lambda t, name: t[:, L[name][0]: L[name][0] + L[name][1]]      # noqa: E731
        self.prob = seg(bf, "prob").view(n, post_n, NC)
        self.boxes = seg(bf, "boxes").view(n, post_n, 4 * NC)
        self.det = (seg(blocks, "keep_idx").view(n, NC - 1, post_n), seg(blocks, "keep_count"), seg(blocks, "conf_count"))
        return seg(bf, "rois").view(n, post_n, 4), seg(bf, "scores"), seg(blocks, "count")[:, 0]

    def clone(self):
        """A second set of buffers (and its own graph) over the SAME packed weights: lets another image or batch be in flight."""
        p = type(self)(self.w, *(self._lead + (self.H, self.W)), **self._ctor)
        p.set_clip(self.im_h, self.im_w)
        return p

    def set_clip(self, im_h, im_w):
        """img_info as the caller passes it (forward.py:93 passes (H, H), SURVEY.md Q7).  Changing it
        invalidates a captured graph (the bounds are kernel arguments)."""
        if (im_h, im_w) != (self.im_h, self.im_w):
            self.im_h, self.im_w = int(im_h), int(im_w)
            self.graph = None

    # -- host-array front end (the reference's model-input interface: a float32 HOST array in, host results out)
    def result_words(self):
        """Words of the result buffer a host caller needs: every block, the last one without the NMS lists when they are off."""
        n = int(self.result.numel())
        return n if self.with_detect else n - self.block_words + self.result_words_nodetect

    def host_io(self):
        """Pinned staging for one synchronous host call at a time: the input and a mirror of the result blocks."""
        if self._host is None:
            dev = self.x_in.device
            self._host = dict(x=ops.PinnedBlock(tuple(self.x_in.shape), np.float32),
                              res=ops.PinnedBlock((int(self.result.numel()),), np.int32),
                              stream=torch.cuda.Stream(device=dev))
        return self._host

    def forward_host(self, x_np):
        """x_np: a float32 numpy array of x_in's shape ((3,H,W), or (1,3,H,W), for a ForwardPlan; (N,3,H,W) for a BatchPlan).
        Copies it into pinned staging (multi-threaded host copy), uploads, replays the graph and brings the result blocks
        back with ONE D2H; blocks until they are there.  Returns unpack_result's numpy VIEWS into the pinned mirror (valid
        until the next forward_host on this plan)."""
        io = self.host_io()
        prof = HOST_PROFILE
        t0 = time.perf_counter() if prof is not None else 0.0
        n = self.result_words()
        st = io["stream"]
        t1 = t0
        io["x"].upload(x_np, self.x_in, st)                        # pageable -> pinned -> device, chunk-pipelined (one C call)
        t2 = time.perf_counter() if prof is not None else 0.0
        with torch.cuda.stream(st):
            self.forward(None)
        t3 = time.perf_counter() if prof is not None else 0.0
        io["res"].d2h(self.result, st, nbytes=4 * n)               # D2H: everything the caller can ask for, one transfer
        ops.stream_synchronize(st)
        if prof is not None:
            t4 = time.perf_counter()
            prof.append((1e3 * (t1 - t0), 1e3 * (t2 - t1), 1e3 * (t3 - t2), 1e3 * (t4 - t3)))
        return self.unpack_result(io["res"].np)


class ForwardPlan(_PlanBase):
    """Buffers + launch sequence for one image shape.  Takes _PlanBase's keyword options."""

    def __init__(self, weights, H, W, **options):
        super(ForwardPlan, self).__init__(weights, H, W, **options)
        dev, post_n = weights.device, self.post_n
        self.x_in = torch.zeros((3, H, W), dtype=torch.float32, device=dev)      # static input (C,H,W)
        h, w_ = self.fh, self.fw = self._alloc_trunk(H, W)
        self.rpn_mid = self._act(h, w_, weights.rpn3[0].shape[1])
        self.rpn_out = torch.empty((h * w_, weights.rpn_ld), dtype=torch.float32, device=dev)
        rois, scores, count = self._alloc_result(1)
        self.prob, self.boxes, self.det = self.prob[0], self.boxes[0], tuple(t[0] for t in self.det)
        self.prop = ops.ProposalWorkspace(weights.n_anchors, h, w_, self.pre_n, post_n, dev, debug=self.keep_rpn_debug,
                                          outputs=(rois[0], scores[0], count))
        C = self.acts[-1].hi.shape[2]
        self.pool5 = self._act(1, post_n, 49 * C)
        self.fc6 = self._act(1, post_n, 4096)
        self.fc7 = self._act(1, post_n, 4096)
        self.head_out = torch.empty((post_n, weights.head_ld), dtype=torch.float32, device=dev)
        # split-K slabs of the swapped-operand head GEMMs (ops.linear); one buffer sized for the largest layer
        self.fc_work = max((ops.linear_workspace(post_n, k_, c_, dev) for k_, c_ in
                            ((49 * C, 4096), (4096, 4096), (4096, 5 * weights.num_classes))), key=lambda t: t.numel())

    def _run_trunk(self):
        """Launches the trunk; returns (feature map Act, number of launches)."""
        acts = iter(self.acts)
        x = next(acts)
        ops.pack_image_c8(self.x_in, out=x, hwc_memory=self.hwc_input)
        n = 1
        for s in self.trunk:
            hi, lo, b = self.w.convs[s.name]
            y = next(acts)
            if s.cin <= 3:                      # conv1_1: sliding-window reads of the compact image, K = 3 x 32
                ops.conv3x3_c8(x, self.H, self.W, hi, lo, b, True, out=y)
            else:
                ops.conv2d(x, hi, lo, b, 3, True, out=y, fuse_pool=s.fused_pool)
            x = y
            n += 1
            if s.pool_after:
                x = next(acts)
                ops.maxpool2x2_ceil(y, out=x)
                n += 1
        return x, n

    # -- the launch sequence (static; safe to capture)
    def _run(self):
        w = self.w
        feat, n = self._run_trunk()
        self.feat = feat
        hi, lo, b = w.rpn3
        ops.conv2d(feat, hi, lo, b, 3, True, out=self.rpn_mid)
        hi, lo, b = w.rpn_heads
        ops.conv2d(self.rpn_mid, hi, lo, b, 1, False, out_act=False, ld_f32=w.rpn_ld, out_f32=self.rpn_out)
        ops.proposals(self.rpn_out, None, self.anchors, w.n_anchors, self.fh, self.fw, self.feat_stride,
                      self.im_h, self.im_w, self.min_size, self.pre_n, self.post_n, self.nms_thresh,
                      layout="nhwc", ld=w.rpn_ld, cls_is_logits=True, work=self.prop,
                      debug=self.prop.dbg_dets is not None)
        n += 2 + 5          # rpn 3x3, rpn heads; decode, select, rank/scatter, IoU mask, mask scan
        ops.roi_pool(feat, self.prop.rois, self.prop.count, 7, 7, 1.0 / self.feat_stride, out=self.pool5)
        n += 1
        hi, lo, b = w.fc6
        ops.linear(self.pool5, hi, lo, b, True, m_valid=self.prop.count, out=self.fc6, work=self.fc_work)
        hi, lo, b = w.fc7
        ops.linear(self.fc6, hi, lo, b, True, m_valid=self.prop.count, out=self.fc7, work=self.fc_work)
        hi, lo, b = w.head
        ops.linear(self.fc7, hi, lo, b, False, m_valid=self.prop.count, out_f32=self.head_out, ld_f32=w.head_ld,
                   work=self.fc_work, want_act=False)
        n += 3 * 2          # each head layer = the split-K GEMM + its reduction
        ops.head_decode(self.head_out, w.head_ld, self.prop.rois, self.prop.count, w.num_classes, self.im_h, self.im_w,
                        out_prob=self.prob, out_boxes=self.boxes)
        n += 1
        if self.with_detect:
            ops.detect(self.prob, self.boxes, self.prop.count, self.det_nms_thresh, self.det_conf, out=self.det)
            n += 1
        self.n_launches = n

    def unpack_result(self, words):
        """numpy int32 words of a result block -> dict of views (count int, prob [R,NC], boxes [R,4NC], rois, scores, detect lists)."""
        return _unpack_block(words, self.result_layout, self.post_n, self.w.num_classes, self.with_detect)

    def forward(self, x_chw=None):
        """Run one image.  x_chw: (3,H,W) float32 CUDA tensor (copied into the static input) or None
        to reuse the current contents of `self.x_in`.  Returns (prob, boxes, count) device tensors."""
        if x_chw is not None:
            self.x_in.copy_(x_chw, non_blocking=True)
        _launch(self)
        return self.prob, self.boxes, self.prop.count


def _launch(plan):
    """Runs plan._run(): eagerly, or by replaying its CUDA graph (captured on first use)."""
    if not plan.use_graph:
        plan._run()
        return
    if plan.graph is None:
        # one capture at a time in the process (torch's capture stream is shared), and thread-local capture mode so
        # that other host threads (each running its own plan) may keep calling CUDA meanwhile
        with _CAPTURE_LOCK:
            plan._run()                   # warm-up outside capture (func attributes, lazy init)
            torch.cuda.current_stream().synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                plan._run()
            plan.graph = g
    plan.graph.replay()


class BatchPlan(_PlanBase):
    """Buffers + launch sequence for N images of one shape (VGG16 trunk), all in ONE CUDA graph.

    Every stage runs once over all N images: the trunk, the RPN convolutions and the fc6 / fc7 / head GEMMs
    (frcnn_conv2d_batch, frcnn_conv3x3_c8_batch, frcnn_linear_batch: the one-image plan with N times the tiles), and
    ProposalLayer, RoI pooling, the head decode, the per-class NMS and the stand-alone max-pools (frcnn_proposals_batch,
    frcnn_roi_pool_batch, frcnn_head_decode_batch, frcnn_detect_batch, frcnn_maxpool2x2_ceil_batch: the image is a grid
    dimension), so the number of launches does not grow with N.  Every image's results are bit-identical to a
    ForwardPlan's on that image.  The result buffer holds N consecutive blocks in ForwardPlan's layout, so the host gets
    everything with one D2H; the batched post-processing reads and writes those blocks in place at a stride of one block.
    Takes ForwardPlan's keyword options."""
    _trunk_name, _trunk_layer = "VGG16", "conv1_1"        # the trunk the launch sequence runs, and a layer only it has

    def __init__(self, weights, N, H, W, **options):
        if int(N) != N or N < 1:
            raise FrcnnError("BatchPlan needs N >= 1 images (got %r)" % (N,))
        super(BatchPlan, self).__init__(weights, H, W, **options)
        if self._trunk_layer not in weights.convs:
            raise FrcnnError("%s runs the %s trunk only" % (type(self).__name__, self._trunk_name))
        N = self.N = int(N)
        self._lead = (N,)
        dev, post_n = weights.device, self.post_n
        # the static input that the first launch reads; extents / im_info: per-image device int32 [N, 2] sizes and clip
        # bounds on a canvas, None when every image fills the H x W slot and (im_h, im_w) clips all of them
        self.input = self._new_input(dev)
        self.x_in, self.extents, self.im_info = self.input.x_in, self.input.extents, self.input.im_info
        h, w_ = self.fh, self.fw = self._alloc_trunk(H, W)
        self.rpn_mid = self._act(h, w_, weights.rpn3[0].shape[1])
        self.rpn_out = torch.empty((N * h * w_, weights.rpn_ld), dtype=torch.float32, device=dev)
        # every per-image result as ONE [N, ...] view of the N blocks (image stride = block_words): the batched entries
        # write straight into the blocks
        outputs = self._alloc_result(N)
        self.prop = ops.ProposalBatchWorkspace(N, weights.n_anchors, h, w_, self.pre_n, post_n, dev, debug=self.keep_rpn_debug,
                                               outputs=outputs)
        self.images = [dict(prob=self.prob[n], boxes=self.boxes[n], det=tuple(t[n] for t in self.det)) for n in range(N)]
        # the RoI counts for frcnn_linear_batch: word `count` of every block, block_words apart
        self.counts = self.result[self.result_layout["count"][0]:]
        # head activations: one segment of ld1 rows per image; rows [post_n, ld1) of pool5 stay zero
        self.ld1 = ops.round_up(post_n, 32)
        C = self.acts[-1].hi.shape[-1]
        self.pool5 = self._act(self.ld1, 49 * C, zero=True)
        self.fc6 = self._act(self.ld1, 4096)
        self.fc7 = self._act(self.ld1, 4096)
        self.head_out = torch.empty((N, self.ld1, weights.head_ld), dtype=torch.float32, device=dev)
        self.fc_work = max((ops.linear_batch_workspace(N, post_n, k_, c_, dev) for k_, c_ in
                            ((49 * C, 4096), (4096, 4096), (4096, 5 * weights.num_classes))), key=lambda t: t.numel())

    def _new_input(self, dev):
        return ImageInput(self.N, self.H, self.W, dev, hwc_memory=self.hwc_input)

    def _run_trunk(self):
        """Launches the input stage and the trunk; returns (feature map Act, number of launches)."""
        w, N, ext = self.w, self.N, self.extents
        self.input.pack_c8(self.acts[0])
        n = 1
        acts = iter(self.acts)
        x = next(acts)
        for s in self.trunk:            # a layer's extents are ceil(extent / 2^halvings)
            hi, lo, b = w.convs[s.name]
            y = next(acts)
            if s.cin <= 3:
                ops.conv3x3_c8_batch(x, N, self.H, self.W, hi, lo, b, True, out=y, extents=ext)
            else:
                ops.conv2d_batch(x, hi, lo, b, 3, True, out=y, fuse_pool=s.fused_pool, extents=ext, halvings=s.halvings)
            x = y
            n += 1
            if s.pool_after:
                x = next(acts)
                ops.maxpool2x2_ceil_batch(y, out=x)
                n += 1
        return x, n

    def _feature_extents(self):
        """(extents, halvings) of the feature map for the RPN, ProposalLayer and RoI pooling launches: the image extents
        after the trunk's four ceil-mode pools (None: every image fills its slot)."""
        return self.extents, VGG16_LAYERS.count("pool")

    def _run(self):
        w, N, post_n = self.w, self.N, self.post_n
        feat, n = self._run_trunk()
        self.feat = feat
        ext, k = self._feature_extents()
        hi, lo, b = w.rpn3
        ops.conv2d_batch(feat, hi, lo, b, 3, True, out=self.rpn_mid, extents=ext, halvings=k)
        hi, lo, b = w.rpn_heads
        ops.conv2d_batch(self.rpn_mid, hi, lo, b, 1, False, out_act=False, ld_f32=w.rpn_ld, out_f32=self.rpn_out, extents=ext,
                         halvings=k)
        n += 2
        ops.proposals_batch(self.rpn_out.view(N, self.fh * self.fw, w.rpn_ld), None, self.anchors, w.n_anchors, self.fh, self.fw,
                            self.feat_stride, self.im_h, self.im_w, self.min_size, self.pre_n, post_n, self.nms_thresh,
                            layout="nhwc", ld=w.rpn_ld, cls_is_logits=True, work=self.prop, debug=self.prop.dbg_dets is not None,
                            extents=ext, halvings=k, im_info=self.im_info)
        p5 = self.pool5
        ops.roi_pool_batch(feat, self.prop.rois, self.prop.count, 7, 7, 1.0 / self.feat_stride,
                           out=ops.Act(p5.hi[:, :post_n], None if p5.lo is None else p5.lo[:, :post_n]), extents=ext, halvings=k)
        n += 5 + 1          # decode, select, rank/scatter, IoU mask, mask scan; RoI pool
        cnt, bw = self.counts, self.block_words
        hi, lo, b = w.fc6
        ops.linear_batch(self.pool5, hi, lo, b, True, post_n, counts=cnt, count_stride=bw, out=self.fc6, work=self.fc_work)
        hi, lo, b = w.fc7
        ops.linear_batch(self.fc6, hi, lo, b, True, post_n, counts=cnt, count_stride=bw, out=self.fc7, work=self.fc_work)
        hi, lo, b = w.head
        ops.linear_batch(self.fc7, hi, lo, b, False, post_n, counts=cnt, count_stride=bw, out_f32=self.head_out,
                         ld_f32=w.head_ld, work=self.fc_work, want_act=False)
        n += 3 * 2
        ops.head_decode_batch(self.head_out[:, :post_n], w.head_ld, self.prop.rois, self.prop.count, w.num_classes,
                              self.im_h, self.im_w, out_prob=self.prob, out_boxes=self.boxes, im_info=self.im_info)
        n += 1
        if self.with_detect:
            ops.detect_batch(self.prob, self.boxes, self.prop.count, self.det_nms_thresh, self.det_conf, out=self.det)
            n += 1
        self.n_launches = n

    def unpack_result(self, words):
        """numpy int32 words of the result buffer -> list of N dicts as ForwardPlan.unpack_result returns them."""
        bw = self.block_words
        return [_unpack_block(words[k * bw:(k + 1) * bw], self.result_layout, self.post_n, self.w.num_classes, self.with_detect)
                for k in range(self.N)]

    def forward(self, x_nchw=None):
        """Run the batch.  x_nchw: (N,3,H,W) float32 CUDA tensor (copied into the static input) or None to reuse the
        current contents of `self.x_in`.  Returns (list of prob [post_n,NC], list of boxes [post_n,4NC], counts [N] int32
        device view); rows past an image's count are zero."""
        if x_nchw is not None:
            if tuple(x_nchw.shape) != tuple(self.x_in.shape):
                raise FrcnnError("BatchPlan: input of shape %s, the plan is for %s" % (tuple(x_nchw.shape), tuple(self.x_in.shape)))
            self.x_in.copy_(x_nchw, non_blocking=True)
        _launch(self)
        counts = self.result.view(self.N, self.block_words)[:, self.result_layout["count"][0]]
        return [im["prob"] for im in self.images], [im["boxes"] for im in self.images], counts


class CanvasBatchPlan(BatchPlan):
    """A BatchPlan whose N images may have different sizes: each sits at the top-left of its Hc x Wc canvas slot, and its
    true size and clip bounds are int32 [N, 2] device arrays that every kernel reads at run time (the *_batch_ext entries:
    pixels outside an image are computed as zeros, its proposals, RoI bins and clips are its own).  So ONE captured graph
    serves any mix of sizes up to the canvas, and an unused slot (extent 0 x 0) costs nothing but its share of the tiles.
    Every image's results are bit-identical to a ForwardPlan's on that image alone.  Takes ForwardPlan's keyword options
    except keep_rpn_debug (the debug rows would carry canvas anchor indices) and hwc_input.

    raw_input=True: the plan takes RAW uint8 (h0,w0,3) BGR photos (forward_raw) instead of preprocessed float32 tensors, in
    a RawPhotoInput (pixel_means, arena_bytes): one host-to-device copy of its block delivers a whole batch."""

    def __init__(self, weights, N, Hc, Wc, raw_input=False, pixel_means=None, arena_bytes=None, **kw):
        if kw.get("keep_rpn_debug"):
            raise FrcnnError("CanvasBatchPlan has no RPN debug outputs (keep_rpn_debug=True)")
        if kw.get("hwc_input"):
            raise FrcnnError("CanvasBatchPlan takes (3,H,W) images (hwc_input=True)")
        self.raw_input = bool(raw_input)
        self._raw_options = dict(pixel_means=pixel_means, arena_bytes=arena_bytes)
        super(CanvasBatchPlan, self).__init__(weights, N, Hc, Wc, **kw)
        if self.raw_input:
            inp = self.input
            self.block, self.arena, self.header_bytes = inp.block, inp.arena, inp.header_bytes
            self.pixel_means, self.arena_bytes = inp.pixel_means, inp.arena_bytes
            self._ctor.update(raw_input=True, pixel_means=self.pixel_means, arena_bytes=self.arena_bytes)
        self.image_sizes = [(0, 0)] * self.N
        self._res_host = None       # pinned mirror of the result blocks (fetch_result)

    def _new_input(self, dev):
        if self.raw_input:
            return RawPhotoInput(self.N, self.H, self.W, dev, **self._raw_options)
        return ImageInput(self.N, self.H, self.W, dev, canvas=True)

    def _raw(self):
        if not self.raw_input:
            raise FrcnnError("CanvasBatchPlan: raw photos need a plan built with raw_input=True")
        return self.input

    def raw_batch_header(self, shapes, img_infos=None):
        """RawPhotoInput.header of this plan's input."""
        return self._raw().header(shapes, img_infos)

    def forward_raw(self, images, img_infos=None):
        """images: a list of at most N RAW uint8 (h0,w0,3) BGR photos of any sizes -- all numpy arrays (copied into a pinned
        mirror of the block and uploaded with ONE host-to-device copy, header included) or all CUDA tensors (copied into the
        arena on the device).  Each is resized as forward.py:34-45 does (preprocess.plan_size) inside the first launch.
        img_infos: optional per-image clip bounds, default the resized (H_n, W_n); forward.py passes (H_n, H_n) (SURVEY.md
        Q7).  Raises FrcnnError before anything is queued if a resized image does not fit the canvas or the photos do not
        fit the arena.  Returns BatchPlan.forward's (list of prob, list of boxes, counts) and the list of im_scale."""
        hdr, scales = self._raw().upload(list(images), img_infos)
        self.image_sizes = [tuple(int(v) for v in e) for e in preprocess.raw_header_views(hdr, self.N)["extents"]]
        return self.forward(None) + (scales,)

    def fetch_result(self):
        """ONE device-to-host copy of all N result blocks on the current stream, waited for: unpack_result's list (numpy
        views into a pinned block, valid until the next fetch)."""
        if self._res_host is None:
            self._res_host = ops.PinnedBlock((int(self.result.numel()),), np.int32)
        cur = torch.cuda.current_stream()
        self._res_host.d2h(self.result, cur, nbytes=4 * self.result_words())
        ops.stream_synchronize(cur)
        return self.unpack_result(self._res_host.np)

    def forward(self, images=None, img_infos=None):
        """images: a list of at most N (3,H_n,W_n) float32 CUDA tensors with H_n <= Hc and W_n <= Wc, copied into the
        top-left of slots 0, 1, ...; the remaining slots are empty (count 0).  img_infos: optional per-image clip bounds
        (im_h, im_w) (forward.py passes (H, H), SURVEY.md Q7); default (H_n, W_n).  None reuses the current slots, sizes and
        clip bounds.  Returns BatchPlan.forward's (list of prob, list of boxes, counts)."""
        if images is not None:
            if self.raw_input:
                raise FrcnnError("CanvasBatchPlan(raw_input=True) takes raw photos through forward_raw")
            sizes = self.input.put(list(images), img_infos)
            self.image_sizes = [tuple(int(v) for v in e) for e in sizes[0]]
        return super(CanvasBatchPlan, self).forward(None)


class ImageInput(object):
    """Float32 images x_in [N,3,H,W] (hwc_memory: the bytes of (N,H,W,3) images), and on a canvas the int32 [2,N,2] `sizes`
    whose rows `extents` and `im_info` are each slot's image size and clip bounds (None in a same-size batch).  pack_c8 /
    pack_im2col: the first launch of the VGG16 / ResNet trunk, into the first layer's planes `out`."""

    def __init__(self, N, H, W, device, canvas=False, hwc_memory=False):
        self.x_in = torch.zeros((N, 3, H, W), dtype=torch.float32, device=device)
        self.hwc_memory = bool(hwc_memory)
        self.sizes = torch.zeros((2, N, 2), dtype=torch.int32, device=device) if canvas else None
        self.extents, self.im_info = (None, None) if self.sizes is None else (self.sizes[0], self.sizes[1])

    def put(self, images, img_infos=None):
        """A list of float (3,H_n,W_n) CUDA images into the top-left of the canvas slots 0, 1, ..., and their extents and clip
        bounds into `sizes` (preprocess.canvas_sizes, which raises first if they do not fit).  Returns the host sizes."""
        N, _, Hc, Wc = self.x_in.shape
        sizes = preprocess.canvas_sizes([tuple(x.shape) for x in images], N, Hc, Wc, img_infos)
        for n, x in enumerate(images):
            self.x_in[n, :, :x.shape[1], :x.shape[2]].copy_(x, non_blocking=True)
        # a pageable source: the copy is staged before copy_ returns, so `sizes` may go out of scope at once
        self.sizes.copy_(torch.from_numpy(sizes), non_blocking=True)
        return sizes

    def pack_c8(self, out):
        ops.pack_image_c8_batch(self.x_in, out=out, hwc_memory=self.hwc_memory, extents=self.extents)

    def pack_im2col(self, out, ksize, stride, pad, k_pad):
        ops.pack_image_im2col_batch(self.x_in, ksize, stride, pad, k_pad, out=out, extents=self.extents)


class RawPhotoInput(object):
    """RAW uint8 (h0,w0,3) BGR photos on a canvas: one device block [header | pixels] (preprocess.raw_header_layout) whose
    header holds each slot's extents, clip bounds, source size, pixel offset and 1 / im_scale, and whose `arena` of
    arena_bytes (default: N sources of Hc x Wc) the photos.  pack_c8 / pack_im2col (frcnn_preprocess_bgr8_canvas[_im2col])
    resize, subtract pixel_means and pack every slot straight into the first layer's planes: there is no x_in.

    max_gt (a training canvas): the photos are the VOC training dataset's, so the block also carries a ground-truth section
    (preprocess.voc_gt_layout) between the header and the pixels, pixel_means default to preprocess.VOC_MEANS, pack_im2col
    resizes bicubically as the dataset does (frcnn_preprocess_voc_canvas_im2col) and scale_gt writes the scaled boxes.

    scales (a training canvas that augments): the training short-side targets.  An augmentation section
    (preprocess.voc_aug_layout) follows the ground-truth section; augment() selects each slot's flip and scale on the device
    (frcnn_voc_augment_batch) and pack_im2col / scale_gt apply the flip (the _flip entries)."""
    x_in = None

    def __init__(self, N, Hc, Wc, device, pixel_means=None, arena_bytes=None, max_gt=None, scales=None):
        self.N, self.H, self.W = int(N), int(Hc), int(Wc)
        self.max_gt = None if max_gt is None else int(max_gt)
        self.scales = None if scales is None else tuple(int(s) for s in scales)
        if self.scales is not None and (self.max_gt is None or not 1 <= len(self.scales) <= preprocess.AUG_MAX_SCALES
                                        or min(self.scales) < 1):
            raise FrcnnError("raw batch: augmentation needs a training canvas and 1 to %d positive scales (got %r)"
                             % (preprocess.AUG_MAX_SCALES, scales))
        if pixel_means is None:
            pixel_means = preprocess.PIXEL_MEANS if self.max_gt is None else preprocess.VOC_MEANS
        self.pixel_means = tuple(float(v) for v in np.asarray(pixel_means, dtype=np.float64).reshape(-1)[:3])
        self.arena_bytes = self.N * 3 * self.H * self.W if arena_bytes is None else int(arena_bytes)
        if self.arena_bytes < 1:
            raise FrcnnError("raw batch: arena_bytes must be positive (got %d)" % self.arena_bytes)
        layout, self.header_bytes = preprocess.raw_header_layout(self.N)
        gt_at = self.header_bytes
        if self.max_gt is not None:
            gt_layout, gt_bytes = preprocess.voc_gt_layout(self.N, self.max_gt)
            self.header_bytes += gt_bytes
        aug_at = self.header_bytes
        if self.scales is not None:
            aug_layout, aug_bytes = preprocess.voc_aug_layout(self.N, len(self.scales))
            self.header_bytes += aug_bytes
        self.block = torch.zeros((self.header_bytes + self.arena_bytes,), dtype=torch.uint8, device=device)
        self.arena = self.block[self.header_bytes:]
        tdt = {np.int32: torch.int32, np.int64: torch.int64, np.float64: torch.float64, np.float32: torch.float32}
        h = {name: self.block[off:off + 8 * self.N].view(tdt[dt]).view((self.N, 2) if items == 2 else (self.N,))
             for name, (off, dt, items) in layout.items()}
        self.extents, self.im_info = h["extents"], h["im_info"]
        # what both first-layer kernels read from the block
        self.descriptors = (self.arena, h["src_off"], h["src_hw"], h["inv_scale"], h["extents"])
        if self.max_gt is not None:
            self.gt_fields = tuple(self.block[gt_at + off:gt_at + off + int(np.prod(shape)) * 4].view(tdt[dt]).view(shape)
                                   for off, dt, shape in (gt_layout[k] for k in ("scale", "count", "raw_gt")))
        self.aug = None
        if self.scales is not None:
            self.aug = {k: self.block[aug_at + off:aug_at + off + int(np.prod(shape)) * np.dtype(dt).itemsize].view(tdt[dt]).view(shape)
                        for k, (off, dt, shape) in aug_layout.items()}
        self._stage = None          # pinned host mirror of the block + the event of its last upload

    def header(self, shapes, img_infos=None):
        """preprocess.raw_batch_header for these slots, canvas and arena (raises FrcnnError when something does not fit)."""
        return preprocess.raw_batch_header(shapes, self.N, self.H, self.W, self.arena_bytes, img_infos)

    def upload(self, images, img_infos=None, boxes=None, labels=None, flips=None, scale_index=None):
        """A list of photos into the block on the current stream, as CanvasBatchPlan.forward_raw describes; on a training
        canvas also their boxes (source-photo coordinates) and labels (preprocess.voc_gt_section).  On an augmenting canvas
        also every photo's candidate sizes (preprocess.voc_aug_section) and, when given, the choice: flips [bool] and
        scale_index [int] per photo (omitted: no flip, index 0; augment(draw != 0) overwrites them).  Raises FrcnnError before
        anything is queued when something does not fit.  Returns (host header, [im_scale]); on an augmenting canvas
        [im_scale] holds each photo's tuple of candidate im_scale, and the header's sizes are those of the smallest scale
        until augment() selects."""
        on_host = all(isinstance(x, np.ndarray) for x in images)
        if not on_host and not all(isinstance(x, torch.Tensor) and x.is_cuda for x in images):
            raise FrcnnError("forward_raw: the images must be all numpy arrays or all CUDA tensors")
        for n, x in enumerate(images):
            if x.dtype != (np.uint8 if on_host else torch.uint8) or len(x.shape) != 3 or x.shape[2] != 3:
                raise FrcnnError("forward_raw: image %d is not a uint8 (h, w, 3) array" % n)
        shapes = [x.shape[:2] for x in images]
        aug = None
        if self.scales is not None:
            aug, cands = preprocess.voc_aug_section(shapes, self.N, self.H, self.W, self.scales)
            choice = preprocess.voc_aug_views(aug, self.N, len(self.scales))["choice"]
            for col, vals, name, top in ((0, flips, "flips", 2), (1, scale_index, "scale_index", len(self.scales))):
                if vals is None:
                    continue
                vals = [int(v) for v in vals]
                if len(vals) != len(images) or any(not 0 <= v < top for v in vals):
                    raise FrcnnError("raw training batch: %s needs one value in [0, %d) per photo (got %r for %d photos)"
                                     % (name, top, vals, len(images)))
                choice[:len(vals), col] = vals
        elif flips is not None or scale_index is not None:
            raise FrcnnError("raw batch: flips and scale_index need an augmenting input (scales=...)")
        if aug is None:
            hdr, scales, _ = self.header(shapes, img_infos)
        else:
            hdr, scales, _ = preprocess.raw_batch_header(shapes, self.N, self.H, self.W, self.arena_bytes, img_infos,
                                                         scale=min(self.scales))
        block_hdr = hdr
        if self.max_gt is not None:
            if boxes is None or labels is None:
                raise FrcnnError("raw training batch: the photos need their boxes and labels")
            block_hdr = np.concatenate([hdr, preprocess.voc_gt_section(list(boxes), list(labels), scales, self.N, self.max_gt)]
                                       + ([] if aug is None else [aug]))
        cur = torch.cuda.current_stream()
        if self._stage is None:
            self._stage = (ops.PinnedBlock((self.block.numel(),), np.uint8), torch.cuda.Event())
        pin, done = self._stage
        done.synchronize()                    # the previous upload has left the pinned mirror
        pin.h2d(self.block, cur, nbytes=preprocess.fill_raw_block(pin.np, block_hdr, images if on_host else [], self.N))
        if not on_host:
            offs = preprocess.raw_header_views(hdr, self.N)["src_off"]
            for n, x in enumerate(images):
                self.arena[int(offs[n]):int(offs[n]) + x.numel()].copy_(x.contiguous().view(-1), non_blocking=True)
        done.record(cur)
        return hdr, (scales if aug is None else cands)

    def augment(self, seeds, draw):
        """frcnn_voc_augment_batch on the block: draw 1 (flip and scale) or 2 (scale only) from seeds (int64 [N]), 0 (the
        uploaded choice); the chosen candidates become the slots' extents, clip bounds, inv_scale and box scale."""
        h = self.descriptors
        ops.voc_augment(seeds if draw else None, self.aug["cand_hw"], self.aug["cand_inv"], self.aug["cand_scale"], h[2],
                        self.aug["choice"], self.aug["flip"], self.extents, self.im_info, h[3], self.gt_fields[0], draw)

    def pack_c8(self, out):
        if self.max_gt is not None:
            raise FrcnnError("raw batch: a training canvas packs im2col planes only")
        ops.preprocess_pack_canvas(*self.descriptors, self.H, self.W, self.pixel_means, out=out)

    def pack_im2col(self, out, ksize, stride, pad, k_pad):
        if self.aug is not None:
            ops.preprocess_voc_im2col_canvas_flip(*self.descriptors, self.aug["flip"], self.H, self.W, self.pixel_means, ksize,
                                                  stride, pad, k_pad, out=out)
            return
        pack = ops.preprocess_im2col_canvas if self.max_gt is None else ops.preprocess_voc_im2col_canvas
        pack(*self.descriptors, self.H, self.W, self.pixel_means, ksize, stride, pad, k_pad, out=out)

    def scale_gt(self, gt, gt_counts):
        """A training canvas's boxes (mirrored first where the slot flips) times each slot's im_scale, labels and counts into
        gt [N, max_gt, 5] / gt_counts [N]."""
        if self.aug is not None:
            ops.voc_flip_scale_gt(*self.gt_fields, self.descriptors[2], self.aug["flip"], gt, gt_counts)
            return
        ops.voc_scale_gt(*self.gt_fields, gt, gt_counts)


class LanePool(object):
    """`lanes` independent images in flight on one GPU: one ForwardPlan (buffers + CUDA graph) and one CUDA stream
    per lane over shared weights.  The reference processes one image per call (batch hard-wired to 1, SURVEY.md
    Q10); images are independent, so a second/third image's tensor-core layers fill the SMs that image one's
    single-CTA steps (radix select, NMS scan) and ragged last waves leave idle.  Each image still runs the whole
    path; nothing is batched or skipped, and results are bit-identical to the single-lane run (tests)."""

    def __init__(self, plan, lanes=3):
        self.plans = [plan] + [plan.clone() for _ in range(max(1, int(lanes)) - 1)]
        dev = plan.w.device
        self.streams = [torch.cuda.Stream(device=dev) for _ in self.plans]
        for p, st in zip(self.plans, self.streams):
            if p.use_graph and p.graph is None:
                with torch.cuda.stream(st):
                    p.forward(None)
        torch.cuda.synchronize(dev)

    def __len__(self):
        return len(self.plans)

    def fork(self):
        """Lane streams start after everything queued so far on the current stream."""
        ev = torch.cuda.Event()
        ev.record()
        for st in self.streams:
            st.wait_event(ev)

    def submit(self, i, x_chw=None):
        """Queue image number i on lane i % lanes.  Returns that lane's plan (its outputs are valid once the lane's
        stream reaches this point; the next image on the same lane overwrites them)."""
        k = i % len(self.plans)
        with torch.cuda.stream(self.streams[k]):
            self.plans[k].forward(x_chw)
        return self.plans[k]

    def join(self):
        """The current stream waits for every lane."""
        cur = torch.cuda.current_stream()
        for st in self.streams:
            cur.wait_stream(st)


class StreamRunner(object):
    """Host-to-host streaming front end of a ForwardPlan: images come from (pinned) HOST memory and results go
    back to pinned HOST memory, for every image.  A ring of `depth` slots on two CUDA streams: the H2D copy of a
    later image runs on the copy stream while earlier images' graphs run on the compute stream; the D2H of
    (prob, boxes, count) is queued behind each graph.  Nothing is skipped per image -- the copies are overlapped,
    not removed -- so the steady-state rate is max(H2D, graph), not their sum.  The host only blocks when it
    reuses a slot (image i waits for image i-depth), so a stalled driver call (some hosts block cudaMemcpyAsync
    for tens of ms) does not drain the GPU queue."""

    def __init__(self, plan, src_hw=None, pixel_means=None, depth=8, lanes=1):
        """lanes: images in flight on the compute side (LanePool; lane = image index % lanes).
        src_hw=None: host images are the preprocessed (3,H,W) float32 tensors forward.py uploads.
        src_hw=(h0,w0): host images are RAW uint8 (h0,w0,3) BGR images; mean subtraction + bilinear resize run
        on the device (frcnn_preprocess_bgr8) -- 4x+ fewer H2D bytes."""
        self.pool = plan if isinstance(plan, LanePool) else LanePool(plan, lanes)
        self.plan = plan = self.pool.plans[0]
        dev = plan.x_in.device
        self.depth = D = max(2, int(depth), 2 * len(self.pool))
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.src_hw, self.pixel_means = src_hw, pixel_means
        if src_hw is None:
            self.stage = [torch.empty_like(plan.x_in) for _ in range(D)]
        else:
            from . import preprocess
            s, H, W = preprocess.plan_size(src_hw[0], src_hw[1])
            if (H, W) != (plan.H, plan.W):
                raise FrcnnError("source %s resizes to %s, but the plan is for %s" % (src_hw, (H, W), (plan.H, plan.W)))
            self.stage = [torch.empty((src_hw[0], src_hw[1], 3), dtype=torch.uint8, device=dev) for _ in range(D)]
        self.h2d_done = [torch.cuda.Event() for _ in range(D)]
        self.step_done = [torch.cuda.Event() for _ in range(D)]
        self.n_words = plan.result_words()
        self.res = [ops.PinnedBlock((self.n_words,), np.int32) for _ in range(D)]
        self.h2d_bytes = self.stage[0].numel() * self.stage[0].element_size()
        self.d2h_bytes = 4 * self.n_words

    def _deliver(self, i, counts, on_result):
        s = i % self.depth
        self.step_done[s].synchronize()
        counts.append(int(self.res[s].np[self.plan.result_layout["count"][0]]))
        if on_result is not None:
            on_result(i, self.plan.unpack_result(self.res[s].np))

    def run(self, host_images, on_result=None):
        """host_images: sequence of pinned host tensors ((3,H,W) float32, or (h0,w0,3) uint8 with src_hw).
        Calls on_result(i, res) in order with the unpacked result of image i (ForwardPlan.unpack_result: numpy views
        into the pinned block, valid until image i+depth is submitted).  Returns the proposal counts."""
        n, D, L = len(host_images), self.depth, len(self.pool)
        self.pool.fork()
        counts = []
        for i in range(n):
            s = i % D
            plan, cur = self.pool.plans[i % L], self.pool.streams[i % L]
            if i >= D:
                self._deliver(i - D, counts, on_result)         # slot reuse: image i-D must be finished and handed over
            # H2D on the copy stream (overlaps earlier images' graphs): cudaMemcpyAsync straight from the caller's buffer
            # -- asynchronous when that buffer is pinned (ops.PinnedBlock, tensor.pin_memory()), staged by the driver if not
            src = host_images[i]
            src = src.t if isinstance(src, ops.PinnedBlock) else (torch.from_numpy(src) if isinstance(src, np.ndarray) else src)
            if src.numel() * src.element_size() != self.h2d_bytes:
                raise FrcnnError("StreamRunner: host image %d has %d bytes, expected %d" %
                                 (i, src.numel() * src.element_size(), self.h2d_bytes))
            if not src.is_contiguous():
                src = src.contiguous()             # a strided view (e.g. an HWC->CHW transpose): densify on the host first
                host_images = list(host_images)
                host_images[i] = src               # keep it alive until the copy has been consumed
            ops.memcpy_h2d_async(self.stage[s], src.data_ptr(), self.h2d_bytes, self.copy_stream)
            self.h2d_done[s].record(self.copy_stream)
            with torch.cuda.stream(cur):
                cur.wait_event(self.h2d_done[s])
                if self.src_hw is None:
                    plan.x_in.copy_(self.stage[s], non_blocking=True)           # D2D into the graph's static input
                else:
                    from . import preprocess
                    if self.pixel_means is None:
                        preprocess.img_preprocessing(self.stage[s], out=plan.x_in)
                    else:
                        preprocess.img_preprocessing(self.stage[s], self.pixel_means, out=plan.x_in)
                plan.forward(None)
                # ONE D2H: count, class probabilities, boxes, proposals (+ the per-class NMS keep lists and counts)
                self.res[s].d2h(plan.result, cur, nbytes=4 * self.n_words)
                self.step_done[s].record(cur)
        for i in range(max(0, n - D), n):
            self._deliver(i, counts, on_result)
        self.pool.join()
        return counts


class CanvasStreamRunner(object):
    """Host-to-host streaming front end of a CanvasBatchPlan(raw_input=True, with_detect=True): RAW uint8 photos of mixed
    sizes come from host memory, N per graph replay, and every image's detections (preprocess.result_detections, boxes in
    source-image coordinates) go back to the host.  A ring of `depth` slots, each a pinned mirror of the plan's [header |
    pixels] block and a pinned result block.  Per batch the host copies the photos and the header into the mirror, and the
    GPU gets ONE H2D copy on the copy stream (straight into the lane plan's block, once that lane's previous replay is
    over: the header is read throughout the graph), the graph on the lane's compute stream and ONE D2H of the result blocks.
    With lanes > 1 a batch's upload and graph overlap the other lanes' graphs.  The host blocks only when it reuses a slot."""

    def __init__(self, plan, depth=2, lanes=1):
        base = plan.plans[0] if isinstance(plan, LanePool) else plan
        if not (isinstance(base, CanvasBatchPlan) and base.raw_input and base.with_detect):
            raise FrcnnError("CanvasStreamRunner needs a CanvasBatchPlan(raw_input=True, with_detect=True)")
        self.pool = plan if isinstance(plan, LanePool) else LanePool(plan, lanes)
        self.plan = plan = base
        self.depth = D = max(2, int(depth), 2 * len(self.pool))
        self.copy_stream = torch.cuda.Stream(device=plan.w.device)
        self.stage = [ops.PinnedBlock((plan.block.numel(),), np.uint8) for _ in range(D)]
        self.n_words = plan.result_words()
        self.res = [ops.PinnedBlock((self.n_words,), np.int32) for _ in range(D)]
        self.h2d_done = [torch.cuda.Event() for _ in range(D)]
        self.step_done = [torch.cuda.Event() for _ in range(D)]
        self.lane_done = [torch.cuda.Event() for _ in self.pool.plans]
        self.h2d_copies = self.h2d_bytes = 0          # totals over run() calls

    def _deliver(self, b, batches, results, on_result):
        s, N = b % self.depth, self.plan.N
        self.step_done[s].synchronize()
        res = self.plan.unpack_result(self.res[s].np)
        for n, im_scale in enumerate(batches[b][1]):
            dets = preprocess.result_detections(res[n], im_scale)
            results.append(dets)
            if on_result is not None:
                on_result(b * N + n, dets, im_scale)

    def run(self, raw_images, on_result=None, img_infos=None):
        """raw_images: sequence of uint8 (h0,w0,3) numpy arrays (pageable or pinned).  Every batch is checked against the
        canvas and the arena first: FrcnnError is raised before anything is queued.  Calls on_result(i, detections,
        im_scale) in image order and returns the list of detections; a last partial batch runs with its other slots empty."""
        plan, D, L, N = self.plan, self.depth, len(self.pool), self.plan.N
        raw_images = list(raw_images)
        shapes = preprocess.raw_photo_shapes(raw_images)
        batches = [plan.raw_batch_header(shapes[s0:s0 + N], None if img_infos is None else img_infos[s0:s0 + N])
                   for s0 in range(0, len(raw_images), N)]
        results = []
        self.pool.fork()
        self.copy_stream.wait_stream(torch.cuda.current_stream())
        for b, (hdr, _, _) in enumerate(batches):
            s, k = b % D, b % L
            lane, cur = self.pool.plans[k], self.pool.streams[k]
            if b >= D:
                self._deliver(b - D, batches, results, on_result)         # slot reuse: batch b-D is finished and handed over
            nbytes = preprocess.fill_raw_block(self.stage[s].np, hdr, raw_images[b * N:b * N + N], N)
            if b >= L:
                self.copy_stream.wait_event(self.lane_done[k])            # the lane's previous replay no longer reads its block
            self.stage[s].h2d(lane.block, self.copy_stream, nbytes=nbytes)
            self.h2d_done[s].record(self.copy_stream)
            self.h2d_copies += 1
            self.h2d_bytes += nbytes
            with torch.cuda.stream(cur):
                cur.wait_event(self.h2d_done[s])
                lane.forward(None)
                self.lane_done[k].record(cur)
                self.res[s].d2h(lane.result, cur, nbytes=4 * self.n_words)
                self.step_done[s].record(cur)
        for b in range(max(0, len(batches) - D), len(batches)):
            self._deliver(b, batches, results, on_result)
        self.pool.join()
        return results


class _PlanLease(object):
    """Thread-local handle of a checked-out ForwardPlan: returns the plan to its engine's pool when the owning thread's
    thread-local storage is torn down."""

    def __init__(self, engine, key, plan):
        self.engine, self.key, self.plan = engine, key, plan

    def __del__(self):
        try:
            self.engine._return_plan(self.key, self.plan)
        except Exception:          # noqa: BLE001  (interpreter shutdown)
            pass


class Engine(object):
    """Weights + per-shape plans.  `engine(x)` -> (prob [R,21], boxes [R,84]) device tensors, R synced."""
    supports_hwc_input = True          # the VGG16 plan's first kernel takes source strides (ForwardPlan(hwc_input=True))
    plan_class = ForwardPlan           # the one-image plan of plan() / thread_plan()

    def __init__(self, params, precision="bf16x3", device="cuda", anchors=None, num_classes=21, n_anchors=9,
                 feat_stride=16, **plan_kwargs):
        self.weights = self._pack_weights(params, precision, device, num_classes, n_anchors)
        self.anchors, self.feat_stride = anchors, feat_stride
        self.plan_kwargs = plan_kwargs
        self.plans = {}
        self._tls, self._lock = threading.local(), threading.Lock()
        self._plan_pool = {}               # thread_plan: the plans handed back, per base plan

    def _pack_weights(self, params, precision, device, num_classes, n_anchors):
        return PackedWeights(params, precision, device, num_classes, n_anchors)

    def _cached(self, kind, cls, shape, overrides):
        """The cls plan of `shape` with the engine's plan options updated by `overrides`, built on first use; cached under
        (kind, *shape, options), or (*shape, options) when kind is None."""
        kw = dict(self.plan_kwargs)
        kw.update(overrides)
        key = (() if kind is None else (kind,)) + tuple(shape) + (tuple(sorted(kw.items())),)
        if key not in self.plans:
            self.plans[key] = cls(self.weights, *shape, anchors=self.anchors, feat_stride=self.feat_stride, **kw)
        return self.plans[key]

    def plan(self, H, W, **overrides):
        return self._cached(None, self.plan_class, (H, W), overrides)

    def thread_plan(self, H, W, **overrides):
        """A plan private to the calling thread (buffers, graph, stream over the shared weights): several host threads may
        call the model concurrently, one image each, and their graphs overlap on the GPU.  Plans live in a pool per (shape,
        options): a thread checks one out on its first call and a finalizer on its thread-local state hands it back when
        the thread ends, so the next thread reuses the captured graph and the pinned staging -- nothing is freed at thread
        exit (cudaFree / cudaFreeHost there would stall every other caller)."""
        held = self._tls.__dict__.setdefault("plans", {})
        call = (H, W, tuple(sorted(overrides.items())))
        lease = held.get(call)
        if lease is None:
            with self._lock:
                base = self.plan(H, W, **overrides)
                pool = self._plan_pool.setdefault(base, [])
                p = pool.pop() if pool else (base.clone() if getattr(base, "_leased", False) else base)
                p._leased = True
            lease = held[call] = _PlanLease(self, base, p)
        return lease.plan

    def _return_plan(self, base, plan):
        with self._lock:
            self._plan_pool.setdefault(base, []).append(plan)

    def call_host(self, x_np, img_info=None, **overrides):
        """Host-array call: x_np float32 (3,H,W) numpy -> dict of numpy results (ForwardPlan.forward_host).  A C-contiguous
        array is uploaded as it is; so is the transposed view of a dense (H,W,3) array (forward.py:45 produces exactly that:
        `img.transpose([2, 0, 1]).astype(np.float32)` keeps the HWC memory) -- the first kernel then reads it with HWC
        strides; any other striding is densified on the host first."""
        H, W = int(x_np.shape[-2]), int(x_np.shape[-1])
        if x_np.dtype != np.float32:
            x_np = np.ascontiguousarray(x_np, dtype=np.float32)
        if x_np.flags.c_contiguous:
            dense = x_np
        elif self.supports_hwc_input and x_np.ndim == 3 and x_np.transpose(1, 2, 0).flags.c_contiguous:
            dense = x_np.transpose(1, 2, 0)             # the (H,W,3) memory itself, no copy
            overrides = dict(overrides, hwc_input=True)
        else:
            dense = np.ascontiguousarray(x_np)
        x_np = dense
        p = self.thread_plan(H, W, **overrides)
        if img_info is not None:
            p.set_clip(int(img_info[0]), int(img_info[1]))
        return p.forward_host(x_np), p

    def __call__(self, x_chw, img_info=None, **overrides):
        _, H, W = x_chw.shape
        p = self.plan(H, W, **overrides)
        if img_info is not None:
            p.set_clip(int(img_info[0]), int(img_info[1]))
        prob, boxes, count = p.forward(x_chw)
        R = int(count.item())           # the one documented D2H sync (SURVEY.md Q11)
        return prob[:R], boxes[:R], p

    def batch_plan(self, N, H, W, **overrides):
        """The BatchPlan for N images of H x W (cached per shape and options)."""
        return self._cached("batch", BatchPlan, (N, H, W), overrides)

    def forward_batch(self, x_nchw, img_info=None, **overrides):
        """N same-size images (N,3,H,W) float32 CUDA -> list of per-image (prob [R_n,NC], boxes [R_n,4NC]) device tensors,
        after one sync for the N counts."""
        if x_nchw.dim() != 4 or x_nchw.shape[1] != 3:
            raise FrcnnError("forward_batch: expected (N,3,H,W) images, got %s" % (tuple(x_nchw.shape),))
        N, _, H, W = x_nchw.shape
        p = self.batch_plan(N, H, W, **overrides)
        if img_info is not None:
            p.set_clip(int(img_info[0]), int(img_info[1]))
        probs, boxes, counts = p.forward(x_nchw)
        R = counts.cpu().tolist()
        return [(pr[:r], bx[:r]) for pr, bx, r in zip(probs, boxes, R)]

    def canvas_plan(self, N, Hc, Wc, **overrides):
        """The CanvasBatchPlan of N slots of Hc x Wc (cached per canvas and options)."""
        return self._cached("canvas", CanvasBatchPlan, (N, Hc, Wc), overrides)

    def forward_images(self, images, img_infos=None, N=None, canvas=None, **overrides):
        """Images of any sizes, a list of (3,H_n,W_n) float32 CUDA tensors -> list of per-image (prob [R_n,NC], boxes
        [R_n,4NC]) device tensors, N images per graph replay (default: all of them) on a canvas of (Hc, Wc) (default: the
        largest H and W, each rounded up to a multiple of 64, so that a stream of photos reuses a few canvases).
        img_infos: optional per-image clip bounds (im_h, im_w).  With more than N images the results are copies; otherwise
        views into the plan's buffers, valid until its next call."""
        images = list(images)
        if not images:
            return []
        for x in images:
            if x.dim() != 3 or x.shape[0] != 3:
                raise FrcnnError("forward_images: expected (3,H,W) images, got %s" % (tuple(x.shape),))
        N = len(images) if N is None else int(N)
        if canvas is None:
            canvas = (ops.round_up(max(int(x.shape[1]) for x in images), 64), ops.round_up(max(int(x.shape[2]) for x in images), 64))
        p = self.canvas_plan(N, int(canvas[0]), int(canvas[1]), **overrides)
        out = []
        for s in range(0, len(images), N):
            chunk = images[s:s + N]
            probs, boxes, counts = p.forward(chunk, None if img_infos is None else img_infos[s:s + N])
            R = counts.cpu().tolist()
            res = [(probs[n][:R[n]], boxes[n][:R[n]]) for n in range(len(chunk))]
            out += [(a.clone(), b.clone()) for a, b in res] if len(images) > N else res
        return out

    def raw_canvas_plan(self, raw_images, N=None, canvas=None, nms_thresh=0.3, conf=0.8, **overrides):
        """The CanvasBatchPlan(raw_input=True, with_detect=True) that serves `raw_images` N per replay: the canvas defaults
        to the largest resized H and W, each rounded up to a multiple of 64, and the arena to N times the largest photo,
        rounded up to 1 MiB."""
        shapes = [tuple(int(v) for v in x.shape[:2]) for x in raw_images]
        N = len(shapes) if N is None else int(N)
        if canvas is None:
            sizes = [preprocess.plan_size(h0, w0)[1:] for h0, w0 in shapes]
            canvas = (ops.round_up(max(s[0] for s in sizes), 64), ops.round_up(max(s[1] for s in sizes), 64))
        arena = N * ops.round_up(max(3 * h0 * w0 for h0, w0 in shapes), preprocess.RAW_ALIGN)
        kw = dict(raw_input=True, arena_bytes=ops.round_up(arena, 1 << 20), with_detect=True, det_nms_thresh=nms_thresh,
                  det_conf=conf)
        kw.update(overrides)
        return self.canvas_plan(N, int(canvas[0]), int(canvas[1]), **kw)

    def detect_images(self, raw_images, N=None, canvas=None, nms_thresh=0.3, conf=0.8, img_infos=None, **overrides):
        """forward.py's whole loop on RAW photos of any sizes: a list of uint8 (h0,w0,3) BGR arrays -> for each image the list
        preprocess.detections gives, (cls_id, x1, y1, x2, y2, score) in source-image coordinates.  N images per graph
        replay (default: all of them), one upload and one download per replay; the canvas as raw_canvas_plan picks it.
        img_infos: optional per-image clip bounds (forward.py passes the resized (H, H))."""
        raw_images = list(raw_images)
        if not raw_images:
            return []
        p = self.raw_canvas_plan(raw_images, N, canvas, nms_thresh, conf, **overrides)
        out = []
        for s in range(0, len(raw_images), p.N):
            chunk = raw_images[s:s + p.N]
            scales = p.forward_raw(chunk, None if img_infos is None else img_infos[s:s + p.N])[3]
            res = p.fetch_result()
            out += [preprocess.result_detections(res[n], scales[n]) for n in range(len(chunk))]
        return out

    def evaluate_images(self, raw_images, gt_boxes, gt_labels, gt_difficult=None, N=None, canvas=None, nms_thresh=0.3, conf=0.05,
                        img_infos=None, iou_thresh=0.5, **overrides):
        """PASCAL VOC average precision of the model on RAW photos (evaluate.VocEvaluator): detect_images' plan and batching,
        but the detections stay on the device -- per replay one upload of the photos and the evaluator's append, no download;
        the im_scale of every photo goes up in one copy first, and the result comes back in one download at the end.
        gt_boxes / gt_labels / gt_difficult: per-photo ground truth in source-photo coordinates (VocEvaluator.evaluate).
        conf: the detection threshold (0.05, the usual evaluation setting).  Returns the VocEvalResult."""
        from .evaluate import VocEvaluator
        raw_images = list(raw_images)
        if not raw_images:
            raise FrcnnError("evaluate_images: no images")
        p = self.raw_canvas_plan(raw_images, N, canvas, nms_thresh, conf, **overrides)
        M, NC = len(raw_images), self.weights.num_classes
        ev = VocEvaluator(NC, max_images=M, capacity=M * (NC - 1) * p.post_n,
                          max_gt=max(1, sum(len(b) for b in gt_boxes)), device=self.weights.device)
        infos = lambda s: None if img_infos is None else img_infos[s:s + p.N]      # noqa: E731
        shapes = preprocess.raw_photo_shapes(raw_images)
        ev.put_scales([v for s in range(0, M, p.N) for v in p.raw_batch_header(shapes[s:s + p.N], infos(s))[1]])
        for s in range(0, M, p.N):
            chunk = raw_images[s:s + p.N]
            p.forward_raw(chunk, infos(s))
            keep_idx, _, conf_count = p.det
            n = len(chunk)
            ev._append(p.prob[:n], p.boxes[:n], keep_idx[:n], conf_count[:n])
        return ev.evaluate(gt_boxes, gt_labels, gt_difficult, iou_thresh)


def _c_structs(weights, H, W, anchors, pre_n, post_n, nms_thresh, min_size, feat_stride):
    """(device anchor table, frcnn_forward_config, frcnn_vgg16_weights) of the whole-graph C entries, filled from a
    PackedWeights; the structs point into the weights' and the anchor table's device memory."""
    from . import _lib
    anchors = torch.from_numpy(np.ascontiguousarray(anchors, dtype=np.float64)).to(weights.device)
    cfg = _lib.ForwardConfig(H, W, weights.num_classes, weights.n_anchors, feat_stride, pre_n, post_n, min_size,
                             float(nms_thresh), 1 if weights.precision == "bf16x3" else 0)
    p = lambda t: None if t is None else t.data_ptr()                     # noqa: E731
    layer = lambda hi, lo, b: _lib.PackedLayer(p(hi), p(lo), p(b))         # noqa: E731
    wt = _lib.Vgg16Weights()
    for i, s in enumerate(vgg16_schedule(H, W, True)[0]):
        wt.conv[i] = layer(*weights.convs[s.name])
    wt.rpn3, wt.rpn_heads = layer(*weights.rpn3), layer(*weights.rpn_heads)
    wt.fc6, wt.fc7, wt.head = layer(*weights.fc6), layer(*weights.fc7), layer(*weights.head)
    wt.anchors = anchors.data_ptr()
    return anchors, cfg, wt


class CForward(object):
    """frcnn_forward_vgg16: the whole forward path behind the single C-ABI entry (include/frcnn_b200.h) -- what a caller
    without Python binds.  Same kernels, same order as BatchPlan._run; this wrapper only fills the C structs from a
    PackedWeights and owns the workspace / output tensors.  N > 1: frcnn_forward_vgg16_batch over N images per call."""

    def __init__(self, weights, H, W, anchors, pre_n=6000, post_n=300, nms_thresh=0.7, min_size=16, feat_stride=16, N=1):
        import ctypes
        from . import _lib
        if int(N) != N or N < 1:
            raise FrcnnError("CForward needs N >= 1 images (got %r)" % (N,))
        self._lib, self._ct = _lib.load(), ctypes
        self.w, self.H, self.W, self.post_n, self.N = weights, H, W, post_n, int(N)
        dev = weights.device
        self.anchors, self.cfg, self.wt = _c_structs(weights, H, W, anchors, pre_n, post_n, nms_thresh, min_size, feat_stride)
        cfg = self.cfg
        if self.N == 1:
            nbytes = self._lib.frcnn_forward_workspace_bytes(ctypes.byref(cfg))
        else:
            nbytes = self._lib.frcnn_forward_batch_workspace_bytes(ctypes.byref(cfg), self.N)
        if nbytes == 0:
            raise FrcnnError("frcnn_forward_workspace_bytes: %s" % _lib.last_error())
        self.ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        lead = () if self.N == 1 else (self.N,)
        self.prob = torch.empty(lead + (post_n, weights.num_classes), dtype=torch.float32, device=dev)
        self.boxes = torch.empty(lead + (post_n, 4 * weights.num_classes), dtype=torch.float32, device=dev)
        self.count = torch.zeros((self.N,), dtype=torch.int32, device=dev)

    def forward(self, x, im_info=None):
        """x: (3,H,W) float32 CUDA for N = 1, (N,3,H,W) otherwise.  Returns (prob, boxes, count) device tensors
        ([N, ...] for N > 1; rows past an image's count are zero)."""
        from . import _lib
        im_h, im_w = (self.H, self.W) if im_info is None else (int(im_info[0]), int(im_info[1]))
        want = (3, self.H, self.W) if self.N == 1 else (self.N, 3, self.H, self.W)
        if tuple(x.shape) != want:
            raise FrcnnError("CForward: input of shape %s, expected %s" % (tuple(x.shape), want))
        x = x.contiguous().float()
        ct = self._ct
        args = (ct.c_void_p(x.data_ptr()), im_h, im_w, ct.c_void_p(self.ws.data_ptr()), self.ws.numel(),
                ct.c_void_p(self.prob.data_ptr()), ct.c_void_p(self.boxes.data_ptr()), ct.c_void_p(self.count.data_ptr()),
                ct.c_void_p(torch.cuda.current_stream().cuda_stream))
        if self.N == 1:
            _lib.check(self._lib.frcnn_forward_vgg16(ct.byref(self.cfg), ct.byref(self.wt), *args), "frcnn_forward_vgg16")
        else:
            _lib.check(self._lib.frcnn_forward_vgg16_batch(ct.byref(self.cfg), ct.byref(self.wt), self.N, *args),
                       "frcnn_forward_vgg16_batch")
        return self.prob, self.boxes, self.count


class CCanvasForward(object):
    """frcnn_forward_vgg16_canvas / frcnn_detect_vgg16_raw: a canvas batch -- N images of different sizes, each at the top-left
    of its Hc x Wc slot -- behind the single C-ABI call a caller without Python binds.  Same kernels, same order as
    CanvasBatchPlan._run; this wrapper fills the C structs from a PackedWeights and owns the workspace, the static inputs and
    the outputs, so launch() can be captured into a CUDA graph and replayed for any mix of sizes.

    raw_input=False: the input is an ImageInput canvas, (N,3,Hc,Wc) float32 images plus the int32 [N, 2] extents and clip
    bounds (forward).  raw_input=True: the input is a RawPhotoInput, the device block [header | pixels] of raw uint8 BGR
    photos (pixel_means, arena_bytes), and the float64 [N] im_scale; the call also runs the per-class
    NMS (det_nms_thresh, det_conf) and writes forward.py's detection lists into ONE int32 buffer `lists`
    [det_count (N, padded to 64 words) | dets [N][cap][5] | scores [N][cap] (float32)], cap = (NC-1) * post_n, so a host
    caller gets them with one device-to-host copy (detect_raw)."""

    def __init__(self, weights, N, Hc, Wc, anchors, pre_n=6000, post_n=300, nms_thresh=0.7, min_size=16, feat_stride=16,
                 raw_input=False, pixel_means=None, arena_bytes=None, det_nms_thresh=0.3, det_conf=0.8):
        import ctypes
        from . import _lib
        if int(N) != N or N < 1:
            raise FrcnnError("CCanvasForward needs N >= 1 images (got %r)" % (N,))
        self._lib, self._ct = _lib.load(), ctypes
        self.w, self.N, self.H, self.W, self.post_n = weights, int(N), int(Hc), int(Wc), post_n
        self.raw_input = bool(raw_input)
        self.det_nms_thresh, self.det_conf = float(det_nms_thresh), float(det_conf)
        dev = weights.device
        self.anchors, self.cfg, self.wt = _c_structs(weights, self.H, self.W, anchors, pre_n, post_n, nms_thresh, min_size,
                                                     feat_stride)
        nbytes = self._lib.frcnn_forward_vgg16_canvas_workspace_bytes(ctypes.byref(self.cfg), self.N)
        if nbytes == 0:
            raise FrcnnError("frcnn_forward_vgg16_canvas_workspace_bytes: %s" % _lib.last_error())
        self.ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        NC = weights.num_classes
        self.prob = torch.zeros((self.N, post_n, NC), dtype=torch.float32, device=dev)
        self.boxes = torch.zeros((self.N, post_n, 4 * NC), dtype=torch.float32, device=dev)
        self.count = torch.zeros((self.N,), dtype=torch.int32, device=dev)
        if not self.raw_input:
            self.input = ImageInput(self.N, self.H, self.W, dev, canvas=True)
            return
        inp = self.input = RawPhotoInput(self.N, self.H, self.W, dev, pixel_means, arena_bytes)
        self.block, self.header_bytes, self.arena_bytes = inp.block, inp.header_bytes, inp.arena_bytes
        self.im_scale = torch.zeros((self.N,), dtype=torch.float64, device=dev)
        self.cap = (NC - 1) * post_n
        self.lists_layout = dict(det_count=0, dets=ops.round_up(self.N, 64), scores=ops.round_up(self.N, 64) + self.N * self.cap * 5)
        self.lists = torch.zeros((self.lists_layout["scores"] + self.N * self.cap,), dtype=torch.int32, device=dev)
        L = self.lists_layout
        self.det_count = self.lists[:self.N]
        self.dets = self.lists[L["dets"]:L["scores"]].view(self.N, self.cap, 5)
        self.scores = self.lists[L["scores"]:].view(torch.float32).view(self.N, self.cap)
        # pinned mirror of im_scale + the event of its last upload (stage_raw)
        self._scale_stage = (ops.PinnedBlock((self.N,), np.float64), torch.cuda.Event())
        self._res_host = None       # pinned mirror of `lists` (fetch_detections)

    def launch(self):
        """Enqueue the C call on the current stream over the current contents of the static inputs (capturable)."""
        from . import _lib
        inp, ct, p = self.input, self._ct, lambda t: self._ct.c_void_p(t.data_ptr())          # noqa: E731
        st = ct.c_void_p(torch.cuda.current_stream().cuda_stream)
        if self.raw_input:
            m = inp.pixel_means
            _lib.check(self._lib.frcnn_detect_vgg16_raw(ct.byref(self.cfg), ct.byref(self.wt), self.N, p(inp.block), inp.arena_bytes,
                                                        m[0], m[1], m[2], p(self.im_scale), self.det_nms_thresh,
                                                        ct.c_float(self.det_conf), p(self.ws), self.ws.numel(), p(self.prob),
                                                        p(self.boxes), p(self.count), p(self.dets), p(self.scores),
                                                        p(self.det_count), st), "frcnn_detect_vgg16_raw")
        else:
            _lib.check(self._lib.frcnn_forward_vgg16_canvas(ct.byref(self.cfg), ct.byref(self.wt), self.N, p(inp.x_in), p(inp.extents),
                                                            p(inp.im_info), p(self.ws), self.ws.numel(), p(self.prob),
                                                            p(self.boxes), p(self.count), st), "frcnn_forward_vgg16_canvas")

    def set_images(self, images, img_infos=None):
        """Float input: at most N (3,H_n,W_n) float32 CUDA tensors with H_n <= Hc and W_n <= Wc into the top-left of slots
        0, 1, ...; the other slots are empty.  img_infos: optional per-image clip bounds (im_h, im_w), default (H_n, W_n)."""
        if self.raw_input:
            raise FrcnnError("CCanvasForward(raw_input=True) takes raw photos (stage_raw / detect_raw)")
        self.input.put(list(images), img_infos)

    def forward(self, images, img_infos=None):
        """set_images + launch.  Returns (prob [N,post_n,NC], boxes [N,post_n,4NC], count [N]) device tensors; rows past an
        image's count are zero."""
        self.set_images(images, img_infos)
        self.launch()
        return self.prob, self.boxes, self.count

    def stage_raw(self, photos, img_infos=None):
        """Raw input: at most N uint8 (h0,w0,3) BGR numpy photos and their header (preprocess.raw_batch_header) into the block
        with one host-to-device copy, and their im_scale into `im_scale`.  Returns the list of im_scale."""
        if not self.raw_input:
            raise FrcnnError("CCanvasForward: raw photos need raw_input=True")
        photos = list(photos)
        preprocess.raw_photo_shapes(photos)             # numpy photos only
        _, scales = self.input.upload(photos, img_infos)
        cur = torch.cuda.current_stream()
        pin, done = self._scale_stage
        done.synchronize()                    # the previous upload has left the pinned mirror
        pin.np[:] = 0.0
        pin.np[:len(scales)] = scales
        pin.h2d(self.im_scale, cur)
        done.record(cur)
        return scales

    def fetch_detections(self, n_images=None):
        """ONE device-to-host copy of `lists` on the current stream, waited for: for each of the first n_images slots (default
        N) its list of (cls_id, x1, y1, x2, y2, score), preprocess.result_detections' tuples."""
        if self._res_host is None:
            self._res_host = ops.PinnedBlock((int(self.lists.numel()),), np.int32)
        cur = torch.cuda.current_stream()
        self._res_host.d2h(self.lists, cur)
        ops.stream_synchronize(cur)
        return self.unpack_lists(self._res_host.np, n_images)

    def unpack_lists(self, words, n_images=None):
        """Host int32 words of `lists` -> for each of the first n_images slots (default N) its list of detections."""
        L = self.lists_layout
        dets = words[L["dets"]:L["scores"]].reshape(self.N, self.cap, 5)
        scores = words[L["scores"]:].view(np.float32).reshape(self.N, self.cap)
        return [[(*(int(v) for v in dets[n, k]), float(scores[n, k])) for k in range(int(words[n]))]
                for n in range(self.N if n_images is None else int(n_images))]

    def detect_raw(self, photos, img_infos=None):
        """forward.py's whole loop on at most N raw photos in one C call: stage_raw + launch + fetch_detections."""
        photos = list(photos)
        self.stage_raw(photos, img_infos)
        self.launch()
        return self.fetch_detections(len(photos))
