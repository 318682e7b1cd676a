"""torch-tensor front end of the RPN-training entry points of the C ABI (include/frcnn_b200.h:
frcnn_bbox_overlaps, frcnn_anchor_targets, frcnn_rpn_loss and their canvas forms), of the RCNN-head training entries and
their canvas forms (frcnn_proposal_targets_batch, frcnn_rcnn_loss_batch, frcnn_roi_pool_backward_batch_ext,
frcnn_dropout_masks_batch).  Like ops.py: device pointers + the current
stream in, tensors out, no CPU path.

Replaces models/bbox.pyx:16-56, models/anchor_target_layer.py:66-198 and the two loss functions of
models/region_proposal_network.py:160-204 (all under /root/reference); the second half wraps the conv-backward entry
points (frcnn_gemm_nt_splitk, frcnn_grad_prepare, frcnn_wgrad_reduce, frcnn_bias_grad, frcnn_optimizer_update,
frcnn_sgd_momentum, frcnn_pack_conv_weights_dgrad) used by train_engine.py, and those the ResNet trunk adds
(frcnn_maxpool3x3s2_backward, frcnn_grad_prepare_stride2 and their _batch forms, frcnn_fold_batchnorm,
frcnn_wgrad_reduce_scaled) used by resnet_train.py.
"""
import ctypes

import torch

from . import _lib
from ._lib import FrcnnError, check
from .ops import _need_cuda, _p, _stream

RPN_NEGATIVE_OVERLAP, RPN_POSITIVE_OVERLAP = 0.3, 0.7       # models/anchor_target_layer.py:44-45
RPN_FG_FRACTION, RPN_BATCHSIZE = 0.5, 256                   # :46-47
SUBSAMPLE_NONE, SUBSAMPLE_DEVICE, SUBSAMPLE_LIST = 0, 1, 2
ROIS_PER_IMAGE = 128                                        # models/proposal_target_layer.py:49


def bbox_overlaps(boxes, query):
    """boxes [N,4], query [K,4] float64 CUDA tensors -> overlaps [N,K] float64 (bbox.pyx:16-56)."""
    _need_cuda(boxes, query)
    b = boxes.contiguous().double()
    q = query.contiguous().double()
    if b.ndim != 2 or q.ndim != 2 or b.shape[1] != 4 or q.shape[1] != 4:
        raise FrcnnError("bbox_overlaps: expected (N,4) and (K,4), got %s and %s" % (tuple(b.shape), tuple(q.shape)))
    out = torch.zeros((b.shape[0], q.shape[0]), dtype=torch.float64, device=b.device)
    check(_lib.load().frcnn_bbox_overlaps(_p(b), b.shape[0], _p(q), q.shape[0], _p(out), _stream()), "frcnn_bbox_overlaps")
    return out


class AnchorTargets(object):
    """Device buffers of one feature-map shape: labels_full [n_all] int32, targets_full [n_all,4] float32,
    inds_inside [n_all] int32 (first counts[0] valid), counts int32 [8]."""

    def __init__(self, A, H, W, device, max_gt=256):
        self.shape = (A, H, W)
        self.n_all = n = A * H * W
        self.labels_full = torch.empty((n,), dtype=torch.int32, device=device)
        self.targets_full = torch.empty((n, 4), dtype=torch.float32, device=device)
        self.inds_inside = torch.empty((n,), dtype=torch.int32, device=device)
        self.counts = torch.zeros((8,), dtype=torch.int32, device=device)
        self.max_gt = max_gt
        lib = _lib.load()
        self.ws = torch.empty((lib.frcnn_anchor_targets_workspace_bytes(n, max_gt),), dtype=torch.uint8, device=device)
        self.loss_ws = torch.empty((lib.frcnn_rpn_loss_workspace_bytes(n),), dtype=torch.uint8, device=device)
        self.losses = torch.zeros((4,), dtype=torch.float32, device=device)

    def compact(self):
        """The reference's return values (anchor_target_layer.py:120): labels [n_inside], targets [n_inside,4],
        inds_inside [n_inside], n_all.  One D2H read of the inside count."""
        n = int(self.counts[0].item())
        idx = self.inds_inside[:n].long()
        return self.labels_full[idx], self.targets_full[idx], idx, self.n_all


def anchor_targets(anchors, A, H, W, feat_stride, gt_boxes, im_h, im_w, mode=SUBSAMPLE_DEVICE, seed=0, disable_pos=None,
                   work=None, neg_thr=RPN_NEGATIVE_OVERLAP, pos_thr=RPN_POSITIVE_OVERLAP, batch=RPN_BATCHSIZE,
                   num_fg=int(RPN_FG_FRACTION * RPN_BATCHSIZE)):
    """frcnn_anchor_targets.  anchors [A,4] float64 CUDA; gt_boxes [G,5] float32 CUDA.  Returns the AnchorTargets."""
    _need_cuda(anchors, gt_boxes)
    gt = gt_boxes.contiguous().float()
    if gt.ndim != 2 or gt.shape[1] != 5 or gt.shape[0] < 1:
        raise FrcnnError("anchor_targets: gt_boxes must be (G>=1, 5), got %s" % (tuple(gt.shape),))
    G = gt.shape[0]
    if work is None or work.shape != (A, H, W) or work.max_gt < G:
        work = AnchorTargets(A, H, W, gt.device, max_gt=max(256, G))
    dp, nd = None, 0
    if mode == SUBSAMPLE_LIST:
        dp = (disable_pos if disable_pos is not None else torch.zeros((0,), dtype=torch.int32, device=gt.device))
        dp = dp.to(device=gt.device, dtype=torch.int32).contiguous()
        nd = dp.numel()
    check(_lib.load().frcnn_anchor_targets(
        _p(anchors), A, H, W, int(feat_stride), _p(gt), G, int(im_h), int(im_w), float(neg_thr), float(pos_thr),
        int(batch), int(num_fg), int(mode), ctypes.c_ulonglong(int(seed) & (2 ** 64 - 1)), _p(dp) if nd else None, nd,
        _p(work.labels_full), _p(work.targets_full), _p(work.inds_inside), _p(work.counts), _p(work.ws), work.ws.numel(),
        _stream()), "frcnn_anchor_targets")
    return work


def rpn_loss(score, bbox, anchors, A, H, W, feat_stride, im_h, im_w, work, delta=3.0, loss_lambda=1.0, grad_scale=1.0,
             layout="nchw", ld=0, want_grads=True):
    """frcnn_rpn_loss.  layout "nchw": score (2A,H,W), bbox (4A,H,W) planar float32 (the reference's);
    layout "nhwc": ONE float32 matrix [H*W, ld] (score in columns [0,2A), bbox in [2A,6A)) passed as `score`.
    Returns (losses float32[4] = cls, bbox, accuracy, total; dscore; dbbox) -- gradients in the inputs' layout
    (for "nhwc" a single [H*W, ld] matrix, returned as dscore, dbbox None)."""
    _need_cuda(score, bbox)
    if layout == "nchw":
        score = score.contiguous().float()
        bbox = bbox.contiguous().float()
        cs, ps, bcs, bps = H * W, 1, H * W, 1
        bbox_ptr = _p(bbox)
        ds = torch.empty_like(score) if want_grads else None
        db = torch.empty_like(bbox) if want_grads else None
        ds_ptr, db_ptr = _p(ds), _p(db)
    else:
        if score.dtype != torch.float32 or not score.is_contiguous() or score.shape != (H * W, ld):
            raise FrcnnError("rpn_loss: nhwc layout needs a contiguous float32 [H*W, ld] matrix")
        cs, ps, bcs, bps = 1, ld, 1, ld
        bbox_ptr = ctypes.c_void_p(score.data_ptr() + 4 * 2 * A)
        ds = torch.zeros_like(score) if want_grads else None           # pad columns stay zero
        db = None
        ds_ptr = _p(ds)
        db_ptr = ctypes.c_void_p(ds.data_ptr() + 4 * 2 * A) if want_grads else None
    check(_lib.load().frcnn_rpn_loss(_p(score), cs, ps, bbox_ptr, bcs, bps, _p(anchors), A, H, W, int(feat_stride),
                                     int(im_h), int(im_w), _p(work.labels_full), _p(work.targets_full), _p(work.counts),
                                     float(delta), float(loss_lambda), float(grad_scale), _p(work.losses), ds_ptr, db_ptr,
                                     _p(work.loss_ws), work.loss_ws.numel(), _stream()), "frcnn_rpn_loss")
    return work.losses.clone(), ds, db          # a fresh tensor per call: the workspace buffer is overwritten by the next step


class AnchorTargetsBatch(object):
    """Device buffers of frcnn_anchor_targets_batch / frcnn_rpn_loss_batch for N slots of an H x W canvas feature map: slot
    n's labels_full [n][cap] int32, targets_full [n][cap,4] float32, inds_inside [n][cap] int32, counts [n][8] int32 and
    losses [n][4] float32, cap = A*H*W."""

    def __init__(self, N, A, H, W, max_gt, device):
        self.shape, self.N, self.max_gt = (A, H, W), int(N), int(max_gt)
        self.cap = n = A * H * W
        self.labels_full = torch.empty((N, n), dtype=torch.int32, device=device)
        self.targets_full = torch.empty((N, n, 4), dtype=torch.float32, device=device)
        self.inds_inside = torch.empty((N, n), dtype=torch.int32, device=device)
        self.counts = torch.zeros((N, 8), dtype=torch.int32, device=device)
        self.losses = torch.zeros((N, 4), dtype=torch.float32, device=device)
        lib = _lib.load()
        self.ws = torch.empty((lib.frcnn_anchor_targets_batch_workspace_bytes(N, n, max_gt),), dtype=torch.uint8, device=device)
        self.loss_ws = torch.empty((lib.frcnn_rpn_loss_batch_workspace_bytes(N, n),), dtype=torch.uint8, device=device)


def _slot_array(t, dtype, shape, what):
    _need_cuda(t)
    if t.dtype != dtype or tuple(t.shape) != tuple(shape) or not t.is_contiguous():
        raise FrcnnError("%s: expected a dense %s %s CUDA tensor, got %s %s" % (what, dtype, tuple(shape), t.dtype, tuple(t.shape)))
    return _p(t)


def anchor_targets_batch(anchors, A, feat_stride, extents, im_info, gt, gt_counts, work, halvings=4, mode=SUBSAMPLE_DEVICE,
                         seeds=None, disable_pos=None, disable_offsets=None, neg_thr=RPN_NEGATIVE_OVERLAP,
                         pos_thr=RPN_POSITIVE_OVERLAP, batch=RPN_BATCHSIZE, num_fg=int(RPN_FG_FRACTION * RPN_BATCHSIZE)):
    """frcnn_anchor_targets_batch into `work` (AnchorTargetsBatch).  extents / im_info int32 [N, 2]; gt float32
    [N, max_gt, 5]; gt_counts int32 [N]; mode 1: seeds uint64 (torch.int64) [N]; mode 2: disable_pos int32 [n] and
    disable_offsets int32 [N+1].  All device tensors, read when the kernels run."""
    _need_cuda(anchors)
    N, (_, H, W) = work.N, work.shape
    args = [_slot_array(extents, torch.int32, (N, 2), "extents"), int(halvings), _slot_array(im_info, torch.int32, (N, 2), "im_info"),
            _slot_array(gt, torch.float32, (N, work.max_gt, 5), "gt"), work.max_gt, _slot_array(gt_counts, torch.int32, (N,), "gt_counts")]
    sp, dp, nd, do = None, None, 0, None
    if mode == SUBSAMPLE_DEVICE:
        sp = _slot_array(seeds, torch.int64, (N,), "seeds")
    elif mode == SUBSAMPLE_LIST:
        nd = int(disable_pos.numel())
        dp = _slot_array(disable_pos, torch.int32, (nd,), "disable_pos") if nd else None
        do = _slot_array(disable_offsets, torch.int32, (N + 1,), "disable_offsets")
    check(_lib.load().frcnn_anchor_targets_batch(
        _p(anchors), A, H, W, int(feat_stride), N, *args, float(neg_thr), float(pos_thr), int(batch), int(num_fg), int(mode), sp, dp,
        nd, do, _p(work.labels_full), _p(work.targets_full), _p(work.inds_inside), _p(work.counts), _p(work.ws), work.ws.numel(),
        _stream()), "frcnn_anchor_targets_batch")
    return work


def rpn_loss_batch(head, ld, anchors, A, feat_stride, extents, im_info, work, halvings=4, delta=3.0, loss_lambda=1.0,
                   grad_scale=1.0, dhead=None):
    """frcnn_rpn_loss_batch on the NHWC head matrix head [N*H*W, ld] float32; dhead (same shape, optional) receives the
    gradient in every element.  Returns work.losses ([N, 4], overwritten by the next call)."""
    N, (_, H, W) = work.N, work.shape
    for t in (head, dhead):
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != (N * H * W, ld)):
            raise FrcnnError("rpn_loss_batch: head / dhead must be contiguous float32 [%d, %d]" % (N * H * W, ld))
    check(_lib.load().frcnn_rpn_loss_batch(
        _p(head), int(ld), _p(anchors), A, H, W, int(feat_stride), N, _slot_array(extents, torch.int32, (N, 2), "extents"),
        int(halvings), _slot_array(im_info, torch.int32, (N, 2), "im_info"), _p(work.labels_full), _p(work.targets_full),
        _p(work.counts), float(delta), float(loss_lambda), float(grad_scale), _p(work.losses), _p(dhead), _p(work.loss_ws),
        work.loss_ws.numel(), _stream()), "frcnn_rpn_loss_batch")
    return work.losses


def split_bf16(x):
    """float32 CUDA tensor -> (hi, lo) bf16 planes with x ~= hi + lo (the kernels' "bf16x3" operand format)."""
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


_ZERO_BIAS = {}


def _zero_bias(device, n):
    z = _ZERO_BIAS.get(device)
    if z is None or z.numel() < n:
        z = _ZERO_BIAS[device] = torch.zeros((max(n, 1024),), dtype=torch.float32, device=device)
    return z


def gemm_nt_splitk(a_hi, a_lo, b_hi, b_lo, groups=1, row_stride=0, splits=1, out=None):
    """frcnn_gemm_nt_splitk: A [M,K]; B [N,K] (groups=1) or [3,N,K] pre-shifted planes (groups=9); bf16 planes (lo may
    be None for both) -> parts [groups, S, M, ld] fp32, ld = N rounded up to 32.  See include/frcnn_b200.h."""
    _need_cuda(a_hi, b_hi)
    M, K = a_hi.shape
    N = b_hi.shape[-2]
    want_b = (3, N, K) if groups == 9 else (N, K)
    if tuple(b_hi.shape) != want_b or K % 64:
        raise FrcnnError("gemm_nt_splitk: A [M,K], B %s with K %% 64 == 0 (got %s, %s)" % (want_b, tuple(a_hi.shape), tuple(b_hi.shape)))
    lib = _lib.load()
    S = lib.frcnn_gemm_nt_splitk_splits(K, int(splits))
    ld = (N + 31) // 32 * 32
    if out is not None:          # groups == S == 1 and ld == N: the single slab IS the result (e.g. a weight gradient view)
        if groups != 1 or S != 1 or ld != N or out.numel() != M * N or out.dtype != torch.float32 or not out.is_contiguous():
            raise FrcnnError("gemm_nt_splitk: `out` needs groups = splits = 1, N %% 32 == 0 and a contiguous fp32 [M*N] target")
        parts = out.view(1, 1, M, ld)
    else:
        parts = torch.empty((groups, S, M, ld), dtype=torch.float32, device=a_hi.device)
    zero = _zero_bias(a_hi.device, ld)
    check(lib.frcnn_gemm_nt_splitk(_p(a_hi), _p(a_lo), M, K, _p(b_hi), _p(b_lo), N, int(groups), int(row_stride), int(splits),
                                   _p(zero), _p(parts), ld, _stream()), "frcnn_gemm_nt_splitk")
    return parts


def padded_pixels(H, W):
    """(Kp, Wp) of the transposed padded layout of an H x W map (include/frcnn_b200.h)."""
    wp = ctypes.c_int(0)
    kp = _lib.load().frcnn_padded_pixels(int(H), int(W), ctypes.byref(wp))
    return int(kp), int(wp.value)


class TBuf(object):
    """Transposed padded planes [planes, C, N*Kp] bf16 hi (+ lo), zeroed once (the kernels write the interior only); image n
    of a batch in columns [n*Kp, (n+1)*Kp)."""

    def __init__(self, planes, C, H, W, device, x3=True, N=1):
        self.Kp, self.Wp = padded_pixels(H, W)
        self.planes, self.C, self.H, self.W, self.N = planes, C, H, W, N
        self.hi = torch.zeros((planes, C, N * self.Kp), dtype=torch.bfloat16, device=device)
        self.lo = torch.zeros_like(self.hi) if x3 else None


def grad_prepare(H, W, C, g=None, g_f32=None, y=None, p=None, out=None, tbuf=None, times2=False):
    """frcnn_grad_prepare.  g: ops.Act source (NHWC, or pooled size when p is given) or g_f32 [H*W, ld] fp32;
    y / p: forward activation / its pooled map (ops.Act) for the ReLU mask / max-pool routing;
    out: ops.Act [H,W,C] to receive the NHWC result (optional); tbuf: TBuf to receive the transposed planes (optional)."""
    ld = int(g_f32.shape[1]) if g_f32 is not None else 0
    check(_lib.load().frcnn_grad_prepare(
        _p(g.hi) if g is not None else None, _p(g.lo) if g is not None else None, _p(g_f32), ld,
        _p(y.hi) if y is not None else None, _p(y.lo) if y is not None else None,
        _p(p.hi) if p is not None else None, _p(p.lo) if p is not None else None, int(H), int(W), int(C),
        _p(out.hi) if out is not None else None, _p(out.lo) if out is not None else None,
        _p(tbuf.hi) if tbuf is not None else None, _p(tbuf.lo) if tbuf is not None else None,
        tbuf.planes if tbuf is not None else 1, 1 if times2 else 0, _stream()), "frcnn_grad_prepare")


def grad_prepare_batch(N, H, W, C, g=None, g_f32=None, y=None, p=None, out=None, tbuf=None, times2=False):
    """frcnn_grad_prepare_batch: grad_prepare over N images; every Act is [N, ...], g_f32 [N*H*W, ld], tbuf a TBuf of N
    blocks."""
    if tbuf is not None and tbuf.N != N:
        raise FrcnnError("grad_prepare_batch: the transposed buffer holds %d images, not %d" % (tbuf.N, N))
    ld = int(g_f32.shape[1]) if g_f32 is not None else 0
    check(_lib.load().frcnn_grad_prepare_batch(
        _p(g.hi) if g is not None else None, _p(g.lo) if g is not None else None, _p(g_f32), ld,
        _p(y.hi) if y is not None else None, _p(y.lo) if y is not None else None,
        _p(p.hi) if p is not None else None, _p(p.lo) if p is not None else None, int(N), int(H), int(W), int(C),
        _p(out.hi) if out is not None else None, _p(out.lo) if out is not None else None,
        _p(tbuf.hi) if tbuf is not None else None, _p(tbuf.lo) if tbuf is not None else None,
        tbuf.planes if tbuf is not None else 1, 1 if times2 else 0, _stream()), "frcnn_grad_prepare_batch")


def maxpool3x3s2_backward(g, y, p, out=None, tbuf=None):
    """frcnn_maxpool3x3s2_backward: the pooled gradient g and pooled map p (Acts [h, w, C]) routed back to the 3x3/2
    cover_all windows of y (Act [H, W, C], the post-ReLU pool input) and masked by y > 0; out: Act [H, W, C] (optional),
    tbuf: TBuf with planes = 1 (optional)."""
    H, W, C = y.hi.shape
    ph, pw = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    for name, a in (("g", g), ("p", p)):
        if tuple(a.hi.shape) != (ph, pw, C):
            raise FrcnnError("maxpool3x3s2_backward: %s must be [%d, %d, %d], got %s" % (name, ph, pw, C, tuple(a.hi.shape)))
    if tbuf is not None and tbuf.planes != 1:
        raise FrcnnError("maxpool3x3s2_backward: the transposed buffer must have 1 plane")
    check(_lib.load().frcnn_maxpool3x3s2_backward(
        _p(g.hi), _p(g.lo), _p(y.hi), _p(y.lo), _p(p.hi), _p(p.lo), int(H), int(W), int(C),
        _p(out.hi) if out is not None else None, _p(out.lo) if out is not None else None,
        _p(tbuf.hi) if tbuf is not None else None, _p(tbuf.lo) if tbuf is not None else None, _stream()),
        "frcnn_maxpool3x3s2_backward")


def grad_prepare_stride2(H, W, C, g, y=None, out=None, tbuf=None):
    """frcnn_grad_prepare_stride2: g (Act [ceil(H/2), ceil(W/2), C]) placed at the even pixels of an H x W map, zero
    elsewhere, masked by y > 0 when y (Act [H, W, C]) is given; out / tbuf as in grad_prepare."""
    if tuple(g.hi.shape) != ((H + 1) // 2, (W + 1) // 2, C):
        raise FrcnnError("grad_prepare_stride2: g must be [%d, %d, %d], got %s" % ((H + 1) // 2, (W + 1) // 2, C, tuple(g.hi.shape)))
    check(_lib.load().frcnn_grad_prepare_stride2(
        _p(g.hi), _p(g.lo), _p(y.hi) if y is not None else None, _p(y.lo) if y is not None else None, int(H), int(W), int(C),
        _p(out.hi) if out is not None else None, _p(out.lo) if out is not None else None,
        _p(tbuf.hi) if tbuf is not None else None, _p(tbuf.lo) if tbuf is not None else None,
        tbuf.planes if tbuf is not None else 1, _stream()), "frcnn_grad_prepare_stride2")


def _check_batch_tbuf(what, tbuf, N, planes=None):
    if tbuf is not None and tbuf.N != N:
        raise FrcnnError("%s: the transposed buffer holds %d images, not %d" % (what, tbuf.N, N))
    if tbuf is not None and planes is not None and tbuf.planes != planes:
        raise FrcnnError("%s: the transposed buffer must have %d plane" % (what, planes))


def maxpool3x3s2_backward_batch(N, g, y, p, out=None, tbuf=None):
    """frcnn_maxpool3x3s2_backward_batch: maxpool3x3s2_backward over N images; g, p Acts [N, h, w, C], y Act [N, H, W, C],
    out Act [N, H, W, C] (optional), tbuf a TBuf of N blocks with planes = 1 (optional)."""
    _, H, W, C = y.hi.shape
    ph, pw = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    for name, a in (("y", y), ("g", g), ("p", p)):
        want = (N, H, W, C) if name == "y" else (N, ph, pw, C)
        if tuple(a.hi.shape) != want:
            raise FrcnnError("maxpool3x3s2_backward_batch: %s must be %s, got %s" % (name, list(want), tuple(a.hi.shape)))
    _check_batch_tbuf("maxpool3x3s2_backward_batch", tbuf, N, planes=1)
    check(_lib.load().frcnn_maxpool3x3s2_backward_batch(
        _p(g.hi), _p(g.lo), _p(y.hi), _p(y.lo), _p(p.hi), _p(p.lo), int(N), int(H), int(W), int(C),
        _p(out.hi) if out is not None else None, _p(out.lo) if out is not None else None,
        _p(tbuf.hi) if tbuf is not None else None, _p(tbuf.lo) if tbuf is not None else None, _stream()),
        "frcnn_maxpool3x3s2_backward_batch")


def grad_prepare_stride2_batch(N, H, W, C, g, y=None, out=None, tbuf=None):
    """frcnn_grad_prepare_stride2_batch: grad_prepare_stride2 over N images; g Act [N, ceil(H/2), ceil(W/2), C], y / out Acts
    [N, H, W, C] (optional), tbuf a TBuf of N blocks (optional)."""
    want = (N, (H + 1) // 2, (W + 1) // 2, C)
    if tuple(g.hi.shape) != want:
        raise FrcnnError("grad_prepare_stride2_batch: g must be %s, got %s" % (list(want), tuple(g.hi.shape)))
    _check_batch_tbuf("grad_prepare_stride2_batch", tbuf, N)
    check(_lib.load().frcnn_grad_prepare_stride2_batch(
        _p(g.hi), _p(g.lo), _p(y.hi) if y is not None else None, _p(y.lo) if y is not None else None, int(N), int(H), int(W),
        int(C), _p(out.hi) if out is not None else None, _p(out.lo) if out is not None else None,
        _p(tbuf.hi) if tbuf is not None else None, _p(tbuf.lo) if tbuf is not None else None,
        tbuf.planes if tbuf is not None else 1, _stream()), "frcnn_grad_prepare_stride2_batch")


def fold_batchnorm(w, s, wf, b=None, beta=None, mean=None, bf=None):
    """frcnn_fold_batchnorm: wf = f32(f64(w) * s[co]) (w, wf float32 [Cout, ...], s float64 [Cout]); bf (optional, float32
    [Cout]) = f32(f64(beta) + (f64(b) - f64(mean)) * s), b = 0 when None."""
    Cout = int(w.shape[0])
    per_out = w.numel() // Cout
    if wf.shape != w.shape or wf.dtype != torch.float32 or s.dtype != torch.float64 or s.numel() != Cout:
        raise FrcnnError("fold_batchnorm: w / wf float32 of one shape and s float64 [Cout] needed")
    check(_lib.load().frcnn_fold_batchnorm(_p(w), _p(s), Cout, per_out, _p(b), _p(beta), _p(mean), _p(wf), _p(bf), _stream()),
          "frcnn_fold_batchnorm")
    return wf


def wgrad_reduce_scaled(parts, M, N, s, dw):
    """parts [groups, S, M_parts, ld] -> dw (flat fp32 view, OIHW order) = f32(s[m] * fixed-order split sum), s float64 [>= M]."""
    groups, S, Mp, ld = parts.shape
    check(_lib.load().frcnn_wgrad_reduce_scaled(_p(parts), groups, S, Mp, int(M), ld, int(N), _p(s), _p(dw), _stream()),
          "frcnn_wgrad_reduce_scaled")


def wgrad_reduce(parts, M, N, dw, scale=1.0):
    """parts [groups, S, M_parts, ld] -> dw (flat fp32 view of M*N*groups elements, OIHW order)."""
    groups, S, Mp, ld = parts.shape
    check(_lib.load().frcnn_wgrad_reduce(_p(parts), groups, S, Mp, int(M), ld, int(N), float(scale), _p(dw), _stream()),
          "frcnn_wgrad_reduce")


def bias_grad(tbuf, C, db, scale=1.0):
    """db = scale * the sum over all N*Kp columns of the transposed dY."""
    check(_lib.load().frcnn_bias_grad(_p(tbuf.hi), _p(tbuf.lo), int(C), tbuf.N * tbuf.Kp, float(scale), _p(db), _stream()),
          "frcnn_bias_grad")


def sgd_momentum(w, v, g, lr, momentum, weight_decay):
    check(_lib.load().frcnn_sgd_momentum(_p(w), _p(v), _p(g), w.numel(), float(lr), float(momentum), float(weight_decay),
                                         _stream()), "frcnn_sgd_momentum")


def cast_f32_bf16(src, dst):
    """frcnn_cast_f32_bf16: round a (16-byte aligned) slice of the fp32 gradient bucket into the bf16 bucket."""
    check(_lib.load().frcnn_cast_f32_bf16(_p(src), _p(dst), src.numel(), _stream()), "frcnn_cast_f32_bf16")


def sgd_momentum_bf16g(w, v, g_bf16, lr, momentum, weight_decay):
    check(_lib.load().frcnn_sgd_momentum_bf16g(_p(w), _p(v), _p(g_bf16), w.numel(), float(lr), float(momentum),
                                               float(weight_decay), _stream()), "frcnn_sgd_momentum_bf16g")


def optimizer_update(rule, w, s0, s1, g, hyper):
    """frcnn_optimizer_update: WeightDecay + the rule (optimizers.RULES) on the flat fp32 masters w with state s0 (s1: Adam's
    second state, else None), from the fp32 or bf16 gradient g, with the hyper-parameters in the device array `hyper`."""
    check(_lib.load().frcnn_optimizer_update(int(rule), _p(w), _p(s0), _p(s1), _p(g), int(g.dtype == torch.bfloat16), w.numel(),
                                             _p(hyper), _stream()), "frcnn_optimizer_update")


def pack_conv_weights_dgrad(w, cout_pad=None, x3=True, out=None):
    """OIHW float32 CUDA weights -> ([taps, Cin, cout_pad] bf16 hi, lo or None): the filter of the data-gradient conv.
    out: an earlier result to overwrite in place."""
    w = w.contiguous().float()
    if w.dim() == 2:
        w = w[:, :, None, None]
    Cout, Cin, kh, kw = w.shape
    cout_pad = cout_pad or (Cout + 7) // 8 * 8
    hi, lo = out if out is not None else (torch.empty((kh * kw, Cin, cout_pad), dtype=torch.bfloat16, device=w.device), None)
    if out is None and x3:
        lo = torch.empty_like(hi)
    check(_lib.load().frcnn_pack_conv_weights_dgrad(_p(w), Cout, Cin, kh, kw, cout_pad, _p(hi), _p(lo), _stream()),
          "frcnn_pack_conv_weights_dgrad")
    return hi, lo


# ---------------------------------------------------------------------------------------------- RCNN-head training
def roi_overlaps(rois, count, gt_boxes):
    """frcnn_roi_overlaps: rois [R_cap,4] fp32, count int32[1] or None, gt [G,5] -> (max_overlaps float64 [R_cap], argmax int32)."""
    R = rois.shape[0]
    gt = gt_boxes.contiguous().float()
    mo = torch.empty((R,), dtype=torch.float64, device=rois.device)
    am = torch.empty((R,), dtype=torch.int32, device=rois.device)
    check(_lib.load().frcnn_roi_overlaps(_p(rois), _p(count), R, _p(gt), gt.shape[0], _p(mo), _p(am), _stream()), "frcnn_roi_overlaps")
    return mo, am


def roi_targets(rois, gt_boxes, argmax, keep_inds, num_classes=21):
    """frcnn_roi_targets -> (use_gt_boxes [n,5], bbox_reg_targets [n,4*num_classes], labels int32 [n])."""
    n = keep_inds.numel()
    gt = gt_boxes.contiguous().float()
    keep = keep_inds.to(dtype=torch.int32).contiguous()
    use_gt = torch.empty((n, 5), dtype=torch.float32, device=rois.device)
    ext = torch.empty((n, 4 * num_classes), dtype=torch.float32, device=rois.device)
    labels = torch.empty((n,), dtype=torch.int32, device=rois.device)
    check(_lib.load().frcnn_roi_targets(_p(rois), _p(gt), _p(argmax), _p(keep), n, num_classes, _p(use_gt), _p(ext), _p(labels),
                                        _stream()), "frcnn_roi_targets")
    return use_gt, ext, labels


def rcnn_loss(head_out, keep_inds, labels, bbox_reg_targets, num_classes=21, delta=1.0, grad_scale=1.0, want_grad=True):
    """frcnn_rcnn_loss -> (losses float32[4] = cls, bbox, accuracy, total; dhead like head_out or None)."""
    R, ld = head_out.shape
    keep = keep_inds.to(dtype=torch.int32).contiguous()
    losses = torch.empty((4,), dtype=torch.float32, device=head_out.device)
    dh = torch.empty_like(head_out) if want_grad else None
    check(_lib.load().frcnn_rcnn_loss(_p(head_out), ld, R, _p(keep), keep.numel(), _p(labels), _p(bbox_reg_targets), num_classes,
                                      float(delta), float(grad_scale), _p(losses), _p(dh), _stream()), "frcnn_rcnn_loss")
    return losses, dh


def dropout_(act, mask, scale=2.0):
    """In-place F.dropout with an explicit uint8 mask (same number of elements as the activation)."""
    n = act.hi.numel()
    if mask.numel() != n or mask.dtype != torch.uint8:
        raise FrcnnError("dropout_: mask must be uint8 with %d elements" % n)
    check(_lib.load().frcnn_dropout(_p(act.hi), _p(act.lo), _p(mask), n, float(scale), _stream()), "frcnn_dropout")
    return act


def roi_pool_backward(feat, rois, count, g, outh=7, outw=7, scale=1.0 / 16, out=None, ws=None):
    """frcnn_roi_pool_backward: feat Act [H,W,C], g Act [1,R_cap,outh*outw*C] -> dfeat fp32 [H*W, C]."""
    H, W, C = feat.hi.shape
    R = rois.shape[0]
    lib = _lib.load()
    if ws is None:
        ws = torch.empty((lib.frcnn_roi_pool_backward_workspace_bytes(H, W, C),), dtype=torch.uint8, device=feat.hi.device)
    if out is None:
        out = torch.empty((H * W, C), dtype=torch.float32, device=feat.hi.device)
    check(lib.frcnn_roi_pool_backward(_p(feat.hi), _p(feat.lo), H, W, C, _p(rois), _p(count), R, outh, outw, float(scale),
                                      _p(g.hi), _p(g.lo), _p(out), _p(ws), ws.numel(), _stream()), "frcnn_roi_pool_backward")
    return out


def bbox_transform(ex_rois, gt_rois):
    """frcnn_bbox_transform: ex [n,4], gt [n,>=4] float32 CUDA -> targets [n,4] (models/bbox_transform.py:18-38)."""
    _need_cuda(ex_rois, gt_rois)
    e, g = ex_rois.contiguous().float(), gt_rois.contiguous().float()
    if e.shape[0] != g.shape[0] or e.shape[1] != 4 or g.shape[1] < 4:
        raise FrcnnError("bbox_transform: expected (n,4) and (n,>=4), got %s and %s" % (tuple(e.shape), tuple(g.shape)))
    out = torch.empty((e.shape[0], 4), dtype=torch.float32, device=e.device)
    check(_lib.load().frcnn_bbox_transform(_p(e), _p(g), g.shape[1], e.shape[0], _p(out), _stream()), "frcnn_bbox_transform")
    return out


def keep_inside_flags(boxes, im_h, im_w):
    """frcnn_keep_inside: boxes [n,4] float32 CUDA -> uint8 [n] (1 = fully inside the image)."""
    _need_cuda(boxes)
    b = boxes.contiguous().float()
    flags = torch.empty((b.shape[0],), dtype=torch.uint8, device=b.device)
    check(_lib.load().frcnn_keep_inside(_p(b), b.shape[0], int(im_h), int(im_w), _p(flags), _stream()), "frcnn_keep_inside")
    return flags


# ---------------------------------------------------------------------------------------------- RCNN-head training on a canvas
class ProposalTargetsBatch(object):
    """Device buffers of frcnn_proposal_targets_batch / frcnn_rcnn_loss_batch for N slots of R_cap proposals: keep, labels
    int32 [N][128], use_gt [N][128][5], bbox_reg_targets [N][128][4*num_classes] fp32, max_overlaps float64 [N][R_cap],
    argmax int32 [N][R_cap], counts int32 [N][8] and losses fp32 [N][4]."""

    def __init__(self, N, R_cap, num_classes, device):
        self.N, self.R_cap, self.num_classes = N, R_cap, num_classes = int(N), int(R_cap), int(num_classes)
        K = ROIS_PER_IMAGE
        self.keep = torch.empty((N, K), dtype=torch.int32, device=device)
        self.labels = torch.empty((N, K), dtype=torch.int32, device=device)
        self.use_gt = torch.empty((N, K, 5), dtype=torch.float32, device=device)
        self.bbox_reg_targets = torch.empty((N, K, 4 * num_classes), dtype=torch.float32, device=device)
        self.max_overlaps = torch.empty((N, R_cap), dtype=torch.float64, device=device)
        self.argmax = torch.empty((N, R_cap), dtype=torch.int32, device=device)
        self.counts = torch.zeros((N, 8), dtype=torch.int32, device=device)
        self.losses = torch.zeros((N, 4), dtype=torch.float32, device=device)


def proposal_targets_batch(rois, counts, gt, gt_counts, work, mode=SUBSAMPLE_DEVICE, seeds=None, keep_list=None,
                           list_offsets=None):
    """frcnn_proposal_targets_batch into `work` (ProposalTargetsBatch).  rois [N, R_cap, 4] fp32 (each slot's block dense);
    counts: int32 with one entry per slot (e.g. a column of an [N, 2] array) or None; gt fp32 [N, max_gt, 5]; gt_counts
    int32 [N]; mode 1: seeds uint64 (torch.int64) [N]; mode 2: keep_list int32 [n] and list_offsets int32 [N+1]."""
    from .ops import _counts_stride, _image_stride
    N, R_cap = work.N, work.R_cap
    rs = _image_stride(rois, (R_cap, 4), "proposal_targets_batch rois")
    cs = _counts_stride(counts, N, "proposal_targets_batch")
    _need_cuda(gt)
    if gt.dim() != 3 or gt.shape[0] != N or gt.shape[2] != 5 or gt.dtype != torch.float32 or not gt.is_contiguous():
        raise FrcnnError("proposal_targets_batch: gt must be a dense float32 [%d, max_gt, 5] CUDA tensor" % N)
    sp, kp, nl, lo = None, None, 0, None
    if mode == SUBSAMPLE_DEVICE:
        sp = _slot_array(seeds, torch.int64, (N,), "seeds")
    elif mode == SUBSAMPLE_LIST:
        nl = int(keep_list.numel())
        kp = _slot_array(keep_list, torch.int32, (nl,), "keep_list") if nl else None
        lo = _slot_array(list_offsets, torch.int32, (N + 1,), "list_offsets")
    check(_lib.load().frcnn_proposal_targets_batch(
        N, _p(rois), rs, _p(counts), cs, R_cap, _p(gt), int(gt.shape[1]), _slot_array(gt_counts, torch.int32, (N,), "gt_counts"),
        work.num_classes, int(mode), sp, kp, nl, lo, _p(work.keep), _p(work.labels), _p(work.use_gt), _p(work.bbox_reg_targets),
        _p(work.max_overlaps), _p(work.argmax), _p(work.counts), _stream()), "frcnn_proposal_targets_batch")
    return work


def rcnn_loss_batch(head, work, delta=1.0, grad_scale=1.0, dhead=None):
    """frcnn_rcnn_loss_batch on head [N*R_cap, ld] fp32 with the kept rows of `work`; dhead (same shape, optional) receives
    the gradient in every element.  Returns work.losses ([N, 4], overwritten by the next call)."""
    N, R_cap = work.N, work.R_cap
    ld = int(head.shape[1])
    for t in (head, dhead):
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != (N * R_cap, ld)):
            raise FrcnnError("rcnn_loss_batch: head / dhead must be contiguous float32 [%d, %d]" % (N * R_cap, ld))
    check(_lib.load().frcnn_rcnn_loss_batch(N, _p(head), ld, R_cap, _p(work.keep), _p(work.labels), _p(work.bbox_reg_targets),
                                            _p(work.counts), work.num_classes, float(delta), float(grad_scale), _p(work.losses),
                                            _p(dhead), _stream()), "frcnn_rcnn_loss_batch")
    return work.losses


def roi_pool_backward_batch(feat, rois, counts, g, extents, halvings, outh=7, outw=7, scale=1.0 / 16, out=None, ws=None):
    """frcnn_roi_pool_backward_batch_ext: feat Act [N,H,W,C], rois [N,R_cap,4], counts int32 per slot (or None), g Act
    [N,...,R_cap*outh*outw*C], extents int32 [N, 2] -> dfeat fp32 [N*H*W, C] (0 outside each image)."""
    from .ops import _counts_stride, _image_stride, _per_image_pairs
    N, H, W, C = feat.hi.shape
    R_cap = rois.shape[1]
    rs = _image_stride(rois, (R_cap, 4), "roi_pool_backward_batch rois")
    cs = _counts_stride(counts, N, "roi_pool_backward_batch")
    if g.hi.numel() != N * R_cap * outh * outw * C or not g.hi.is_contiguous():
        raise FrcnnError("roi_pool_backward_batch: g must be a dense [N, R_cap, %d] gradient" % (outh * outw * C))
    lib = _lib.load()
    if ws is None:
        ws = torch.empty((lib.frcnn_roi_pool_backward_batch_workspace_bytes(N, H, W, C),), dtype=torch.uint8, device=feat.hi.device)
    if out is None:
        out = torch.empty((N * H * W, C), dtype=torch.float32, device=feat.hi.device)
    check(lib.frcnn_roi_pool_backward_batch_ext(_p(feat.hi), _p(feat.lo), N, H, W, C, _p(rois), rs, _p(counts), cs, R_cap, outh, outw,
                                                float(scale), _per_image_pairs(extents, N, "extents"), int(halvings), _p(g.hi),
                                                _p(g.lo), _p(out), _p(ws), ws.numel(), _stream()), "frcnn_roi_pool_backward_batch_ext")
    return out


def dropout_masks_batch(seeds, salt, out):
    """frcnn_dropout_masks_batch: seeds uint64 (torch.int64) [N] device -> out uint8 [N, rows, cols] (written in place)."""
    _need_cuda(out)
    N, rows, cols = out.shape
    if out.dtype != torch.uint8 or not out.is_contiguous():
        raise FrcnnError("dropout_masks_batch: out must be a dense uint8 [N, rows, cols] CUDA tensor")
    check(_lib.load().frcnn_dropout_masks_batch(N, rows, cols, _slot_array(seeds, torch.int64, (N,), "seeds"),
                                                ctypes.c_ulonglong(int(salt) & (2 ** 64 - 1)), _p(out), _stream()),
          "frcnn_dropout_masks_batch")
    return out
