"""torch-tensor front end of the C ABI: PyTorch is only the device-memory / stream vehicle.

Every function takes CUDA tensors, passes raw device pointers and the current torch stream to
libfrcnn_b200.so, and returns tensors.  Nothing here computes on the CPU and nothing falls back
to torch operators: a failing native call raises `FrcnnError`.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import FrcnnError, check

PRECISIONS = ("bf16x3", "bf16")


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise FrcnnError("expected CUDA tensors (the library has no CPU path)")


def round_up(v, m):
    return (v + m - 1) // m * m


class Act(object):
    """An NHWC activation: bf16 `hi` plane and optional `lo` plane (value = hi + lo)."""

    __slots__ = ("hi", "lo")

    def __init__(self, hi, lo=None):
        self.hi, self.lo = hi, lo

    @property
    def shape(self):
        return tuple(self.hi.shape)

    def to_chw_f32(self):
        """(C,H,W) float32 view of the value, the reference's feature-map layout."""
        H, W, C = self.hi.shape
        out = torch.empty((C, H, W), dtype=torch.float32, device=self.hi.device)
        check(_lib.load().frcnn_unpack_nhwc(_p(self.hi), _p(self.lo), H, W, C, _p(out), _stream()), "frcnn_unpack_nhwc")
        return out


def pack_image(x_chw, c_pad=16, precision="bf16x3"):
    """(C,H,W) float32 CUDA image -> Act [H,W,c_pad]."""
    _need_cuda(x_chw)
    x = x_chw.contiguous().float()
    C, H, W = x.shape
    hi = torch.empty((H, W, c_pad), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi) if precision == "bf16x3" else None
    check(_lib.load().frcnn_pack_image(_p(x), C, H, W, c_pad, _p(hi), _p(lo), _stream()), "frcnn_pack_image")
    return Act(hi, lo)


def pack_conv_weights(w, cin_pad=None, precision="bf16x3", perm_chw=None, out=None):
    """OIHW (or (Cout, K)) float32 weights -> ([taps, Cout, cin_pad] bf16 hi, lo or None).  out: an earlier result of the
    same shape to overwrite in place (a captured graph keeps reading it)."""
    _need_cuda(w)
    w = w.contiguous().float()
    if w.dim() == 2:
        w = w[:, :, None, None]
    Cout, Cin, kh, kw = w.shape
    cin_pad = cin_pad or round_up(Cin, 8)
    hi, lo = out if out is not None else (torch.empty((kh * kw, Cout, cin_pad), dtype=torch.bfloat16, device=w.device), None)
    if out is None and precision == "bf16x3":
        lo = torch.empty_like(hi)
    pc, ph, pw = perm_chw if perm_chw else (0, 0, 0)
    check(_lib.load().frcnn_pack_conv_weights(_p(w), Cout, Cin, kh, kw, cin_pad, _p(hi), _p(lo),
                                              1 if perm_chw else 0, pc, ph, pw, _stream()), "frcnn_pack_conv_weights")
    return hi, lo


def pack_image_im2col(x_chw, precision="bf16x3", out=None, hwc_memory=False):
    """(C<=3,H,W) float32 CUDA image -> Act [H,W,32]: every pixel's zero-padded 3x3xC neighbourhood.
    hwc_memory: `x_chw` is a (C,H,W)-shaped buffer whose BYTES are the dense (H,W,C) image (a host caller's transposed
    view uploaded as it was); the kernel reads it with (1, W*C, C) strides."""
    _need_cuda(x_chw)
    x = x_chw.contiguous().float()
    C, H, W = x.shape
    if out is None:
        hi = torch.empty((H, W, 32), dtype=torch.bfloat16, device=x.device)
        out = Act(hi, torch.empty_like(hi) if precision == "bf16x3" else None)
    sc, sh, sw = (1, W * C, C) if hwc_memory else (H * W, W, 1)
    check(_lib.load().frcnn_pack_image_im2col3x3_strided(_p(x), C, H, W, sc, sh, sw, _p(out.hi), _p(out.lo), _stream()),
          "frcnn_pack_image_im2col3x3_strided")
    return out


def pack_image_c8(x_chw, precision="bf16x3", out=None, hwc_memory=False):
    """(C<=3,H,W) float32 CUDA image -> compact first-layer input: Act of flat planes holding [H][W+2][8] (+ slack).
    hwc_memory as in pack_image_im2col."""
    _need_cuda(x_chw)
    x = x_chw.contiguous().float()
    C, H, W = x.shape
    if out is None:
        n = _lib.load().frcnn_image_c8_elems(H, W)
        hi = torch.empty((n,), dtype=torch.bfloat16, device=x.device)
        out = Act(hi, torch.empty_like(hi) if precision == "bf16x3" else None)
    sc, sh, sw = (1, W * C, C) if hwc_memory else (H * W, W, 1)
    check(_lib.load().frcnn_pack_image_c8(_p(x), C, H, W, sc, sh, sw, _p(out.hi), _p(out.lo), _stream()), "frcnn_pack_image_c8")
    return out


def pack_conv_weights_c8(w, precision="bf16x3"):
    """OIHW (Cout, Cin<=3, 3, 3) float32 -> ([3, Cout, 32] bf16 hi, lo or None) for conv3x3_c8."""
    _need_cuda(w)
    w = w.contiguous().float()
    Cout, Cin, kh, kw = w.shape
    if (kh, kw) != (3, 3):
        raise FrcnnError("pack_conv_weights_c8: 3x3 kernels only")
    hi = torch.empty((3, Cout, 32), dtype=torch.bfloat16, device=w.device)
    lo = torch.empty_like(hi) if precision == "bf16x3" else None
    check(_lib.load().frcnn_pack_conv_weights_c8(_p(w), Cout, Cin, _p(hi), _p(lo), _stream()), "frcnn_pack_conv_weights_c8")
    return hi, lo


def conv3x3_c8(x_c8, H, W, w_hi, w_lo, bias, relu=True, out=None):
    """frcnn_conv3x3_c8: conv1_1 over the compact image (pack_image_c8) -> Act [H,W,Cout]."""
    taps, Cout, k = w_hi.shape
    if (taps, k) != (3, 32):
        raise FrcnnError("conv3x3_c8: weights must be [3, Cout, 32] (pack_conv_weights_c8)")
    if (x_c8.lo is None) != (w_lo is None):
        raise FrcnnError("conv3x3_c8: activation and weight precision modes differ")
    if out is None:
        yh = torch.empty((H, W, Cout), dtype=torch.bfloat16, device=x_c8.hi.device)
        out = Act(yh, torch.empty_like(yh) if x_c8.lo is not None else None)
    check(_lib.load().frcnn_conv3x3_c8(_p(x_c8.hi), _p(x_c8.lo), H, W, _p(w_hi), _p(w_lo), _p(bias), Cout, 1 if relu else 0,
                                       _p(out.hi), _p(out.lo), _stream()), "frcnn_conv3x3_c8")
    return out


def pack_conv_weights_im2col(w, precision="bf16x3", out=None):
    """OIHW (Cout, Cin<=3, 3, 3) float32 -> ([1, Cout, 32] bf16 hi, lo or None), K order of pack_image_im2col.  out: an
    earlier result to overwrite in place."""
    _need_cuda(w)
    w = w.contiguous().float()
    Cout, Cin, kh, kw = w.shape
    if (kh, kw) != (3, 3):
        raise FrcnnError("pack_conv_weights_im2col: 3x3 kernels only")
    hi, lo = out if out is not None else (torch.empty((1, Cout, 32), dtype=torch.bfloat16, device=w.device), None)
    if out is None and precision == "bf16x3":
        lo = torch.empty_like(hi)
    check(_lib.load().frcnn_pack_conv_weights_im2col3x3(_p(w), Cout, Cin, _p(hi), _p(lo), _stream()),
          "frcnn_pack_conv_weights_im2col3x3")
    return hi, lo


def pad_bias(b, n, out=None):
    if out is None:
        out = torch.zeros(round_up(max(n, b.numel()), 32), dtype=torch.float32, device=b.device)
    out[: b.numel()] = b.float()
    return out


def conv2d(x, w_hi, w_lo, bias, ksize, relu, out_act=True, ld_f32=0, m_valid=None, out=None, out_f32=None,
           fuse_pool=False):
    """frcnn_conv2d: x Act [H,W,Cin]; returns (Act or None, fp32 [H*W, ld_f32] or None).
    fuse_pool: the Act output is the 2x2 ceil-mode max-pooled map [ceil(H/2), ceil(W/2), Cout]."""
    H, W, Cin = x.hi.shape
    taps, Cout, cin_w = w_hi.shape
    if cin_w != Cin or taps != ksize * ksize:
        raise FrcnnError("conv2d: weight shape %s does not match input channels %d / ksize %d" % (tuple(w_hi.shape), Cin, ksize))
    if (x.lo is None) != (w_lo is None):
        raise FrcnnError("conv2d: activation and weight precision modes differ")
    y = out
    if out_act and y is None:
        oh, ow = ((H + 1) // 2, (W + 1) // 2) if fuse_pool else (H, W)
        yh = torch.empty((oh, ow, Cout), dtype=torch.bfloat16, device=x.hi.device)
        y = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    y32 = out_f32
    if ld_f32 and y32 is None:
        y32 = torch.empty((H * W, ld_f32), dtype=torch.float32, device=x.hi.device)
    need = round_up(max(Cout, ld_f32), 32)
    if bias.numel() < need:
        raise FrcnnError("conv2d: bias has %d entries, needs %d (use pad_bias)" % (bias.numel(), need))
    check(_lib.load().frcnn_conv2d(_p(x.hi), _p(x.lo), H, W, Cin, _p(w_hi), _p(w_lo), _p(bias), Cout, ksize,
                                   1 if relu else 0, 1 if fuse_pool else 0, _p(y.hi) if y else None, _p(y.lo) if y else None,
                                   _p(y32), ld_f32, _p(m_valid), _stream()), "frcnn_conv2d")
    return y, y32


def linear_workspace(R_cap, K, Cout, device):
    n = _lib.load().frcnn_linear_workspace_bytes(int(R_cap), int(K), int(Cout))
    if n == 0:
        raise FrcnnError("frcnn_linear_workspace_bytes: bad shape R_cap=%d K=%d Cout=%d" % (R_cap, K, Cout))
    return torch.empty((n,), dtype=torch.uint8, device=device)


def linear(x, w_hi, w_lo, bias, relu, m_valid=None, out=None, out_f32=None, ld_f32=0, work=None, want_act=True):
    """frcnn_linear: x Act [1,R_cap,K] (one RoI per row); w [1,Cout,K] packed planes; bias fp32 [>= Cout].
    Returns (Act [1,R_cap,Cout] or None, fp32 [R_cap, ld_f32] or None).  `work`: uint8 workspace (linear_workspace)."""
    _, R_cap, K = x.hi.shape
    taps, Cout, kw = w_hi.shape
    if taps != 1 or kw != K:
        raise FrcnnError("linear: weight shape %s does not match K = %d" % (tuple(w_hi.shape), K))
    if (x.lo is None) != (w_lo is None):
        raise FrcnnError("linear: activation and weight precision modes differ")
    dev = x.hi.device
    y = out
    if want_act and y is None:
        yh = torch.empty((1, R_cap, Cout), dtype=torch.bfloat16, device=dev)
        y = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    y32 = out_f32
    if ld_f32 and y32 is None:
        y32 = torch.empty((R_cap, ld_f32), dtype=torch.float32, device=dev)
    if work is None:
        work = linear_workspace(R_cap, K, Cout, dev)
    check(_lib.load().frcnn_linear(_p(x.hi), _p(x.lo), R_cap, K, _p(w_hi), _p(w_lo), _p(bias), Cout, 1 if relu else 0,
                                   _p(m_valid), _p(y.hi) if y else None, _p(y.lo) if y else None, _p(y32), int(ld_f32),
                                   _p(work), work.numel(), _stream()), "frcnn_linear")
    return y, y32


def _per_image_pairs(t, N, what):
    """A canvas batch's per-image (height, width) extents or (im_h, im_w) clip bounds: dense int32 CUDA [N, 2]."""
    _need_cuda(t)
    if t.dtype != torch.int32 or tuple(t.shape) != (N, 2) or not t.is_contiguous():
        raise FrcnnError("%s: expected a dense int32 [%d, 2] CUDA tensor, got %s %s" % (what, N, t.dtype, tuple(t.shape)))
    return _p(t)


def pack_image_c8_batch(x_nchw, precision="bf16x3", out=None, hwc_memory=False, extents=None):
    """(N,C<=3,H,W) float32 CUDA images -> Act of planes [N, frcnn_image_c8_elems(H,W)]: pack_image_c8 of every image.
    hwc_memory: the buffer's BYTES are dense (N,H,W,C) images.  extents: int32 [N, 2] device (height, width) of each image
    in its H x W canvas slot (frcnn_pack_image_c8_batch_ext: everything outside is packed as 0)."""
    _need_cuda(x_nchw)
    x = x_nchw.contiguous().float()
    N, C, H, W = x.shape
    lib = _lib.load()
    n = lib.frcnn_image_c8_elems(H, W)
    if out is None:
        hi = torch.empty((N, n), dtype=torch.bfloat16, device=x.device)
        out = Act(hi, torch.empty_like(hi) if precision == "bf16x3" else None)
    if out.hi.numel() < N * n:
        raise FrcnnError("pack_image_c8_batch: output holds %d elements, needs %d" % (out.hi.numel(), N * n))
    sc, sh, sw = (1, W * C, C) if hwc_memory else (H * W, W, 1)
    if extents is not None:
        check(lib.frcnn_pack_image_c8_batch_ext(_p(x), N, C, H, W, C * H * W, sc, sh, sw, _per_image_pairs(extents, N, "extents"),
                                                _p(out.hi), _p(out.lo), _stream()), "frcnn_pack_image_c8_batch_ext")
        return out
    check(lib.frcnn_pack_image_c8_batch(_p(x), N, C, H, W, C * H * W, sc, sh, sw, _p(out.hi), _p(out.lo), _stream()),
          "frcnn_pack_image_c8_batch")
    return out


def preprocess_pack_canvas(arena, src_off, src_hw, inv_scale, extents, Hc, Wc, pixel_means, precision="bf16x3", out=None):
    """frcnn_preprocess_bgr8_canvas: raw uint8 BGR photos -> the compact first-layer planes of an N-slot Hc x Wc canvas, Act
    [N, frcnn_image_c8_elems(Hc,Wc)], in one launch (resize + mean subtraction + pack; 0 outside every image).  arena: dense
    uint8 CUDA tensor holding image n's (h0,w0,3) pixels at byte src_off[n] (int64 [N]); src_hw: int32 [N, 2] (h0, w0), <= 0
    = empty slot; inv_scale: float64 [N] = 1 / im_scale; extents: int32 [N, 2] resized (H, W).  All of them device tensors
    read when the kernel runs."""
    N = _raw_descriptors("preprocess_pack_canvas", arena, src_off, src_hw, inv_scale, extents)
    lib = _lib.load()
    n = lib.frcnn_image_c8_elems(Hc, Wc)
    if out is None:
        hi = torch.empty((N, n), dtype=torch.bfloat16, device=arena.device)
        out = Act(hi, torch.empty_like(hi) if precision == "bf16x3" else None)
    if out.hi.numel() < N * n:
        raise FrcnnError("preprocess_pack_canvas: output holds %d elements, needs %d" % (out.hi.numel(), N * n))
    m = np.asarray(pixel_means, dtype=np.float64).reshape(-1)
    check(lib.frcnn_preprocess_bgr8_canvas(_p(arena), arena.numel(), _p(src_off), _per_image_pairs(src_hw, N, "src_hw"),
                                           _p(inv_scale), _per_image_pairs(extents, N, "extents"), N, int(Hc), int(Wc),
                                           float(m[0]), float(m[1]), float(m[2]), _p(out.hi), _p(out.lo), _stream()),
          "frcnn_preprocess_bgr8_canvas")
    return out


def _raw_descriptors(what, arena, src_off, src_hw, inv_scale, extents):
    """The dtype / shape checks of a raw-photo canvas's arena and descriptors; returns the slot count N."""
    _need_cuda(arena, src_off, src_hw, inv_scale, extents)
    N = int(extents.shape[0])
    if arena.dtype != torch.uint8 or not arena.is_contiguous():
        raise FrcnnError("%s: arena must be a dense uint8 CUDA tensor" % what)
    for t, dt, name in ((src_off, torch.int64, "src_off"), (inv_scale, torch.float64, "inv_scale")):
        if t.dtype != dt or tuple(t.shape) != (N,) or not t.is_contiguous():
            raise FrcnnError("%s: %s must be a dense %s [%d] CUDA tensor" % (what, name, dt, N))
    return N


def preprocess_im2col_canvas(arena, src_off, src_hw, inv_scale, extents, Hc, Wc, pixel_means, ksize, stride, pad, k_pad,
                             precision="bf16x3", out=None):
    """frcnn_preprocess_bgr8_canvas_im2col: raw uint8 BGR photos -> the first-layer im2col planes of an N-slot Hc x Wc canvas,
    Act [N, Ho, Wo, k_pad] (pack_image_im2col_batch's layout), in one launch (resize + mean subtraction + im2col; 0 outside
    every image's output extent).  The descriptors are preprocess_pack_canvas's, all device tensors read when the kernel
    runs."""
    return _preprocess_im2col(_lib.load().frcnn_preprocess_bgr8_canvas_im2col, "frcnn_preprocess_bgr8_canvas_im2col", arena, src_off, src_hw, inv_scale, extents, Hc, Wc,
                              pixel_means, ksize, stride, pad, k_pad, precision, out)


def preprocess_voc_im2col_canvas(arena, src_off, src_hw, inv_scale, extents, Hc, Wc, pixel_means, ksize, stride, pad, k_pad,
                                 precision="bf16x3", out=None):
    """frcnn_preprocess_voc_canvas_im2col: preprocess_im2col_canvas with the VOC training dataset's bicubic resize (OpenCV's
    float INTER_CUBIC) in place of forward.py's bilinear."""
    return _preprocess_im2col(_lib.load().frcnn_preprocess_voc_canvas_im2col, "frcnn_preprocess_voc_canvas_im2col", arena, src_off, src_hw, inv_scale, extents, Hc, Wc,
                              pixel_means, ksize, stride, pad, k_pad, precision, out)


def preprocess_voc_im2col_canvas_flip(arena, src_off, src_hw, inv_scale, extents, flip, Hc, Wc, pixel_means, ksize, stride, pad,
                                      k_pad, precision="bf16x3", out=None):
    """frcnn_preprocess_voc_canvas_im2col_flip: preprocess_voc_im2col_canvas where a slot whose flip[n] (dense int32 [N] CUDA
    tensor, read when the kernel runs) is nonzero is resized from its mirrored photo p[:, ::-1]."""
    N = int(extents.shape[0])
    _need_cuda(flip)
    if flip.dtype != torch.int32 or tuple(flip.shape) != (N,) or not flip.is_contiguous():
        raise FrcnnError("frcnn_preprocess_voc_canvas_im2col_flip: flip must be a dense int32 [%d] CUDA tensor" % N)
    lib = _lib.load()
    return _preprocess_im2col(lambda *a: lib.frcnn_preprocess_voc_canvas_im2col_flip(*a[:6], _p(flip), *a[6:]),
                              "frcnn_preprocess_voc_canvas_im2col_flip", arena, src_off, src_hw, inv_scale, extents, Hc, Wc,
                              pixel_means, ksize, stride, pad, k_pad, precision, out)


def _preprocess_im2col(fn, entry, arena, src_off, src_hw, inv_scale, extents, Hc, Wc, pixel_means, ksize, stride, pad, k_pad, precision,
                       out):
    N = _raw_descriptors(entry, arena, src_off, src_hw, inv_scale, extents)
    Ho, Wo = (Hc + 2 * pad - ksize) // stride + 1, (Wc + 2 * pad - ksize) // stride + 1
    if out is None:
        hi = torch.empty((N, Ho, Wo, k_pad), dtype=torch.bfloat16, device=arena.device)
        out = Act(hi, torch.empty_like(hi) if precision == "bf16x3" else None)
    if tuple(out.hi.shape) != (N, Ho, Wo, k_pad) or (out.lo is not None and out.lo.shape != out.hi.shape):
        raise FrcnnError("%s: output %s, expected %s" % (entry, tuple(out.hi.shape), (N, Ho, Wo, k_pad)))
    _dense_planes(entry, out)
    m = np.asarray(pixel_means, dtype=np.float64).reshape(-1)
    check(fn(
        _p(arena), arena.numel(), _p(src_off), _per_image_pairs(src_hw, N, "src_hw"), _p(inv_scale),
        _per_image_pairs(extents, N, "extents"), N, int(Hc), int(Wc), float(m[0]), float(m[1]), float(m[2]), int(ksize),
        int(stride), int(pad), int(k_pad), _p(out.hi), _p(out.lo), _stream()), entry)
    return out


def voc_scale_gt(scale, count, raw_gt, gt, gt_counts):
    """frcnn_voc_scale_gt_batch: gt [N, max_gt, 5] float32 <- the raw boxes of raw_gt [N, max_gt, 5] times scale[n] (float32
    [N]), labels copied, 0 after count[n] (int32 [N]) rows; gt_counts [N] int32 <- the clamped counts.  Device tensors."""
    _need_cuda(scale, count, raw_gt, gt, gt_counts)
    N, max_gt = int(gt.shape[0]), int(gt.shape[1])
    for t, dt, shape, name in ((scale, torch.float32, (N,), "scale"), (count, torch.int32, (N,), "count"),
                               (raw_gt, torch.float32, (N, max_gt, 5), "raw_gt"), (gt, torch.float32, (N, max_gt, 5), "gt"),
                               (gt_counts, torch.int32, (N,), "gt_counts")):
        if t.dtype != dt or tuple(t.shape) != shape or not t.is_contiguous():
            raise FrcnnError("voc_scale_gt: %s must be a dense %s %s CUDA tensor" % (name, dt, shape))
    check(_lib.load().frcnn_voc_scale_gt_batch(_p(scale), _p(count), _p(raw_gt), N, max_gt, _p(gt), _p(gt_counts), _stream()),
          "frcnn_voc_scale_gt_batch")


def voc_flip_scale_gt(scale, count, raw_gt, src_hw, flip, gt, gt_counts):
    """frcnn_voc_flip_scale_gt_batch: voc_scale_gt where a slot whose flip[n] (int32 [N]) is nonzero first mirrors its boxes
    in its photo's src_hw[n, 1] columns (x1' = (w0 - x2) - 1, x2' = (w0 - x1) - 1, float32).  Device tensors."""
    _need_cuda(scale, count, raw_gt, src_hw, flip, gt, gt_counts)
    N, max_gt = int(gt.shape[0]), int(gt.shape[1])
    for t, dt, shape, name in ((scale, torch.float32, (N,), "scale"), (count, torch.int32, (N,), "count"),
                               (raw_gt, torch.float32, (N, max_gt, 5), "raw_gt"), (src_hw, torch.int32, (N, 2), "src_hw"),
                               (flip, torch.int32, (N,), "flip"), (gt, torch.float32, (N, max_gt, 5), "gt"),
                               (gt_counts, torch.int32, (N,), "gt_counts")):
        if t.dtype != dt or tuple(t.shape) != shape or not t.is_contiguous():
            raise FrcnnError("voc_flip_scale_gt: %s must be a dense %s %s CUDA tensor" % (name, dt, shape))
    check(_lib.load().frcnn_voc_flip_scale_gt_batch(_p(scale), _p(count), _p(raw_gt), _p(src_hw), _p(flip), N, max_gt, _p(gt),
                                                    _p(gt_counts), _stream()), "frcnn_voc_flip_scale_gt_batch")


def voc_augment(seeds, cand_hw, cand_inv, cand_scale, src_hw, choice, flip, extents, im_info, inv_scale, scale, draw):
    """frcnn_voc_augment_batch: draw 1 (flip and scale) or 2 (scale only) writes each slot's draw from seeds (int64 [N], read
    as uint64) into choice [N, 2]; draw 0 reads choice as staged.  Then each slot's chosen candidate (cand_hw [N, S, 2],
    cand_inv [N, S], cand_scale [N, S]) becomes its extents / im_info [N, 2], inv_scale [N] and scale [N], and flip [N]
    its flip bit.  Device tensors; seeds may be None when draw is 0."""
    _need_cuda(seeds, cand_hw, cand_inv, cand_scale, src_hw, choice, flip, extents, im_info, inv_scale, scale)
    N, S = int(cand_hw.shape[0]), int(cand_hw.shape[1])
    for t, dt, shape, name in ((seeds, torch.int64, (N,), "seeds"), (cand_hw, torch.int32, (N, S, 2), "cand_hw"),
                               (cand_inv, torch.float64, (N, S), "cand_inv"), (cand_scale, torch.float32, (N, S), "cand_scale"),
                               (src_hw, torch.int32, (N, 2), "src_hw"), (choice, torch.int32, (N, 2), "choice"),
                               (flip, torch.int32, (N,), "flip"), (extents, torch.int32, (N, 2), "extents"),
                               (im_info, torch.int32, (N, 2), "im_info"), (inv_scale, torch.float64, (N,), "inv_scale"),
                               (scale, torch.float32, (N,), "scale")):
        if t is None and name == "seeds" and not draw:
            continue
        if t is None or t.dtype != dt or tuple(t.shape) != shape or not t.is_contiguous():
            raise FrcnnError("voc_augment: %s must be a dense %s %s CUDA tensor" % (name, dt, shape))
    check(_lib.load().frcnn_voc_augment_batch(_p(seeds), N, S, _p(cand_hw), _p(cand_inv), _p(cand_scale), _p(src_hw), int(draw),
                                              _p(choice), _p(flip), _p(extents), _p(im_info), _p(inv_scale), _p(scale), _stream()),
          "frcnn_voc_augment_batch")


def conv3x3_c8_batch(x_c8, N, H, W, w_hi, w_lo, bias, relu=True, out=None, extents=None):
    """frcnn_conv3x3_c8_batch: conv1_1 over N compact images (pack_image_c8_batch) -> Act [N,H,W,Cout].  extents: int32
    [N, 2] device image sizes in H x W canvas slots (frcnn_conv3x3_c8_batch_ext: pixels outside are written as 0)."""
    taps, Cout, k = w_hi.shape
    if (taps, k) != (3, 32):
        raise FrcnnError("conv3x3_c8_batch: weights must be [3, Cout, 32] (pack_conv_weights_c8)")
    if (x_c8.lo is None) != (w_lo is None):
        raise FrcnnError("conv3x3_c8_batch: activation and weight precision modes differ")
    if x_c8.hi.numel() < N * _lib.load().frcnn_image_c8_elems(H, W):
        raise FrcnnError("conv3x3_c8_batch: input holds fewer than %d compact images of %dx%d" % (N, H, W))
    if out is None:
        yh = torch.empty((N, H, W, Cout), dtype=torch.bfloat16, device=x_c8.hi.device)
        out = Act(yh, torch.empty_like(yh) if x_c8.lo is not None else None)
    if extents is not None:
        check(_lib.load().frcnn_conv3x3_c8_batch_ext(_p(x_c8.hi), _p(x_c8.lo), N, H, W, _p(w_hi), _p(w_lo), _p(bias), Cout,
                                                     1 if relu else 0, _per_image_pairs(extents, N, "extents"), _p(out.hi),
                                                     _p(out.lo), _stream()), "frcnn_conv3x3_c8_batch_ext")
        return out
    check(_lib.load().frcnn_conv3x3_c8_batch(_p(x_c8.hi), _p(x_c8.lo), N, H, W, _p(w_hi), _p(w_lo), _p(bias), Cout,
                                             1 if relu else 0, _p(out.hi), _p(out.lo), _stream()), "frcnn_conv3x3_c8_batch")
    return out


def conv2d_batch(x, w_hi, w_lo, bias, ksize, relu, out_act=True, ld_f32=0, out=None, out_f32=None, fuse_pool=False,
                 extents=None, halvings=0):
    """frcnn_conv2d_batch: x Act [N,H,W,Cin]; returns (Act [N,H,W,Cout] (pooled: [N,ceil(H/2),ceil(W/2),Cout]) or None,
    fp32 [N*H*W, ld_f32] or None).  Each image's output equals conv2d on that image, bit for bit.
    extents: int32 [N, 2] device image sizes (input pixels) in H x W canvas slots, ceil(extent / 2^halvings) at this layer
    (frcnn_conv2d_batch_ext: every output pixel outside is written as 0)."""
    N, H, W, Cin = x.hi.shape
    taps, Cout, cin_w = w_hi.shape
    if cin_w != Cin or taps != ksize * ksize:
        raise FrcnnError("conv2d_batch: weight shape %s does not match input channels %d / ksize %d" % (tuple(w_hi.shape), Cin, ksize))
    if (x.lo is None) != (w_lo is None):
        raise FrcnnError("conv2d_batch: activation and weight precision modes differ")
    y = out
    if out_act and y is None:
        oh, ow = ((H + 1) // 2, (W + 1) // 2) if fuse_pool else (H, W)
        yh = torch.empty((N, oh, ow, Cout), dtype=torch.bfloat16, device=x.hi.device)
        y = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    y32 = out_f32
    if ld_f32 and y32 is None:
        y32 = torch.empty((N * H * W, ld_f32), dtype=torch.float32, device=x.hi.device)
    need = round_up(max(Cout, ld_f32), 32)
    if bias.numel() < need:
        raise FrcnnError("conv2d_batch: bias has %d entries, needs %d (use pad_bias)" % (bias.numel(), need))
    if extents is not None:
        check(_lib.load().frcnn_conv2d_batch_ext(_p(x.hi), _p(x.lo), N, H, W, Cin, _p(w_hi), _p(w_lo), _p(bias), Cout, ksize,
                                                 1 if relu else 0, 1 if fuse_pool else 0, _p(y.hi) if y else None,
                                                 _p(y.lo) if y else None, _p(y32), ld_f32, _per_image_pairs(extents, N, "extents"),
                                                 int(halvings), _stream()), "frcnn_conv2d_batch_ext")
        return y, y32
    check(_lib.load().frcnn_conv2d_batch(_p(x.hi), _p(x.lo), N, H, W, Cin, _p(w_hi), _p(w_lo), _p(bias), Cout, ksize,
                                         1 if relu else 0, 1 if fuse_pool else 0, _p(y.hi) if y else None,
                                         _p(y.lo) if y else None, _p(y32), ld_f32, _stream()), "frcnn_conv2d_batch")
    return y, y32


def linear_batch_workspace(N, R_cap, K, Cout, device):
    n = _lib.load().frcnn_linear_batch_workspace_bytes(int(N), int(R_cap), int(K), int(Cout))
    if n == 0:
        raise FrcnnError("frcnn_linear_batch_workspace_bytes: bad shape N=%d R_cap=%d K=%d Cout=%d" % (N, R_cap, K, Cout))
    return torch.empty((n,), dtype=torch.uint8, device=device)


def linear_batch(x, w_hi, w_lo, bias, relu, R_cap, counts=None, count_stride=1, out=None, out_f32=None, ld_f32=0, work=None,
                 want_act=True):
    """frcnn_linear_batch: x Act [N, ld1, K] with ld1 = round_up(R_cap, 32) rows per image; counts: device int32 holding image
    n's RoI count at counts[n * count_stride] (None: R_cap each).  Returns (Act [N, ld1, Cout] or None, fp32 [N, ld1, ld_f32] or
    None); each image's rows equal linear on that image, bit for bit, and rows past its count are zero."""
    N, ld1, K = x.hi.shape
    taps, Cout, kw = w_hi.shape
    if taps != 1 or kw != K:
        raise FrcnnError("linear_batch: weight shape %s does not match K = %d" % (tuple(w_hi.shape), K))
    if ld1 != round_up(R_cap, 32):
        raise FrcnnError("linear_batch: %d rows per image, expected round_up(R_cap=%d, 32)" % (ld1, R_cap))
    if (x.lo is None) != (w_lo is None):
        raise FrcnnError("linear_batch: activation and weight precision modes differ")
    dev = x.hi.device
    y = out
    if want_act and y is None:
        yh = torch.empty((N, ld1, Cout), dtype=torch.bfloat16, device=dev)
        y = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    y32 = out_f32
    if ld_f32 and y32 is None:
        y32 = torch.empty((N, ld1, ld_f32), dtype=torch.float32, device=dev)
    if work is None:
        work = linear_batch_workspace(N, R_cap, K, Cout, dev)
    check(_lib.load().frcnn_linear_batch(_p(x.hi), _p(x.lo), N, R_cap, K, _p(w_hi), _p(w_lo), _p(bias), Cout, 1 if relu else 0,
                                         _p(counts), int(count_stride), _p(y.hi) if y else None, _p(y.lo) if y else None,
                                         _p(y32), int(ld_f32), _p(work), work.numel(), _stream()), "frcnn_linear_batch")
    return y, y32


def conv2d_res(x, w_hi, w_lo, bias, ksize, relu, res, out=None):
    """frcnn_conv2d_res: y = act(conv(x) + bias + res); res an Act of the output shape (ResNet shortcut add)."""
    H, W, Cin = x.hi.shape
    taps, Cout, cin_w = w_hi.shape
    if cin_w != Cin or taps != ksize * ksize or tuple(res.hi.shape) != (H, W, Cout):
        raise FrcnnError("conv2d_res: shapes do not match (x %s, w %s, res %s)" % (tuple(x.hi.shape), tuple(w_hi.shape), tuple(res.hi.shape)))
    if out is None:
        yh = torch.empty((H, W, Cout), dtype=torch.bfloat16, device=x.hi.device)
        out = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    check(_lib.load().frcnn_conv2d_res(_p(x.hi), _p(x.lo), H, W, Cin, _p(w_hi), _p(w_lo), _p(bias), Cout, ksize, 1 if relu else 0,
                                       _p(res.hi), _p(res.lo), _p(out.hi), _p(out.lo), _stream()), "frcnn_conv2d_res")
    return out


def pack_image_im2col_general(x_chw, ksize, stride, pad, k_pad, precision="bf16x3", out=None):
    """(C,H,W) float32 CUDA image -> Act [Ho,Wo,k_pad]: the zero-padded ksize x ksize x C neighbourhood of every
    stride-th pixel (K index (r*ksize+s)*C + c)."""
    _need_cuda(x_chw)
    x = x_chw.contiguous().float()
    C, H, W = x.shape
    Ho, Wo = (H + 2 * pad - ksize) // stride + 1, (W + 2 * pad - ksize) // stride + 1
    if out is None:
        hi = torch.empty((Ho, Wo, k_pad), dtype=torch.bfloat16, device=x.device)
        out = Act(hi, torch.empty_like(hi) if precision == "bf16x3" else None)
    check(_lib.load().frcnn_pack_image_im2col(_p(x), C, H, W, ksize, stride, pad, k_pad, _p(out.hi), _p(out.lo), _stream()),
          "frcnn_pack_image_im2col")
    return out


def pack_conv_weights_im2col_general(w, k_pad, precision="bf16x3", out=None):
    """OIHW float32 -> ([1, Cout, k_pad] bf16 hi, lo or None) in the K order of pack_image_im2col_general.  out: an earlier
    result to overwrite in place."""
    w = w.contiguous().float()
    Cout, Cin, kh, kw = w.shape
    hi, lo = out if out is not None else (torch.empty((1, Cout, k_pad), dtype=torch.bfloat16, device=w.device), None)
    if out is None and precision == "bf16x3":
        lo = torch.empty_like(hi)
    check(_lib.load().frcnn_pack_conv_weights_im2col(_p(w), None, Cout, Cin, kh, k_pad, _p(hi), _p(lo), _stream()),
          "frcnn_pack_conv_weights_im2col")
    return hi, lo


def maxpool3x3s2_ceil(x, out=None):
    H, W, C = x.hi.shape
    Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
    if out is None:
        yh = torch.empty((Ho, Wo, C), dtype=torch.bfloat16, device=x.hi.device)
        out = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    check(_lib.load().frcnn_maxpool3x3s2_ceil(_p(x.hi), _p(x.lo), H, W, C, _p(out.hi), _p(out.lo), _stream()), "frcnn_maxpool3x3s2_ceil")
    return out


def subsample2x(x, out=None):
    H, W, C = x.hi.shape
    if out is None:
        yh = torch.empty(((H + 1) // 2, (W + 1) // 2, C), dtype=torch.bfloat16, device=x.hi.device)
        out = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    check(_lib.load().frcnn_subsample2x(_p(x.hi), _p(x.lo), H, W, C, _p(out.hi), _p(out.lo), _stream()), "frcnn_subsample2x")
    return out


def _dense_planes(what, *acts):
    for a in acts:
        for t in (a.hi, a.lo):
            if t is not None and not t.is_contiguous():
                raise FrcnnError("%s: planes must be dense [N,H,W,C]" % what)


def resnet_level_extents(extents, Hc, Wc, out=None):
    """frcnn_resnet_level_extents: int32 [N, 2] device image sizes in Hc x Wc canvas slots -> int32 [5, N, 2] device extents of
    the ResNet levels conv1, pool1, res3, res4, res5 (each clamped to that level's canvas)."""
    N = int(extents.shape[0])
    ext = _per_image_pairs(extents, N, "extents")
    if out is None:
        out = torch.empty((5, N, 2), dtype=torch.int32, device=extents.device)
    if out.dtype != torch.int32 or tuple(out.shape) != (5, N, 2) or not out.is_contiguous():
        raise FrcnnError("resnet_level_extents: out must be a dense int32 [5, %d, 2] CUDA tensor" % N)
    check(_lib.load().frcnn_resnet_level_extents(ext, N, int(Hc), int(Wc), _p(out), _stream()), "frcnn_resnet_level_extents")
    return out


def pack_image_im2col_batch(x_nchw, ksize, stride, pad, k_pad, precision="bf16x3", out=None, extents=None):
    """(N,C,H,W) float32 CUDA images -> Act [N,Ho,Wo,k_pad]: pack_image_im2col_general of every image.  extents: int32 [N, 2]
    device image sizes in the H x W slots (frcnn_pack_image_im2col_batch_ext: taps outside an image read as the zero padding,
    output pixels outside its own output size are written as 0)."""
    _need_cuda(x_nchw)
    x = x_nchw.contiguous().float()
    N, C, H, W = x.shape
    Ho, Wo = (H + 2 * pad - ksize) // stride + 1, (W + 2 * pad - ksize) // stride + 1
    if out is None:
        hi = torch.empty((N, Ho, Wo, k_pad), dtype=torch.bfloat16, device=x.device)
        out = Act(hi, torch.empty_like(hi) if precision == "bf16x3" else None)
    if tuple(out.hi.shape) != (N, Ho, Wo, k_pad):
        raise FrcnnError("pack_image_im2col_batch: output %s, expected %s" % (tuple(out.hi.shape), (N, Ho, Wo, k_pad)))
    _dense_planes("pack_image_im2col_batch", out)
    lib = _lib.load()
    if extents is not None:
        check(lib.frcnn_pack_image_im2col_batch_ext(_p(x), N, C, H, W, ksize, stride, pad, k_pad, _per_image_pairs(extents, N, "extents"),
                                                    _p(out.hi), _p(out.lo), _stream()), "frcnn_pack_image_im2col_batch_ext")
        return out
    check(lib.frcnn_pack_image_im2col_batch(_p(x), N, C, H, W, ksize, stride, pad, k_pad, _p(out.hi), _p(out.lo), _stream()),
          "frcnn_pack_image_im2col_batch")
    return out


def maxpool3x3s2_ceil_batch(x, out=None, extents=None):
    """frcnn_maxpool3x3s2_ceil_batch: Act [N,H,W,C] -> Act [N,ceil((H-3)/2)+1,...,C], one launch.  extents: int32 [N, 2] device
    image sizes at THIS map's resolution (frcnn_maxpool3x3s2_ceil_batch_ext: windows clipped at each image's border, output
    pixels outside the image's pooled size written as 0)."""
    N, H, W, C = x.hi.shape
    if out is None:
        yh = torch.empty((N, (H - 2) // 2 + 1, (W - 2) // 2 + 1, C), dtype=torch.bfloat16, device=x.hi.device)
        out = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    _dense_planes("maxpool3x3s2_ceil_batch", x, out)
    lib = _lib.load()
    if extents is not None:
        check(lib.frcnn_maxpool3x3s2_ceil_batch_ext(_p(x.hi), _p(x.lo), N, H, W, C, _per_image_pairs(extents, N, "extents"), _p(out.hi),
                                                    _p(out.lo), _stream()), "frcnn_maxpool3x3s2_ceil_batch_ext")
        return out
    check(lib.frcnn_maxpool3x3s2_ceil_batch(_p(x.hi), _p(x.lo), N, H, W, C, _p(out.hi), _p(out.lo), _stream()),
          "frcnn_maxpool3x3s2_ceil_batch")
    return out


def subsample2x_batch(x, out=None):
    """frcnn_subsample2x_batch: Act [N,H,W,C] -> Act [N,ceil(H/2),ceil(W/2),C], one launch.  On a canvas the input must be 0
    outside every image; the output then is too."""
    N, H, W, C = x.hi.shape
    if out is None:
        yh = torch.empty((N, (H + 1) // 2, (W + 1) // 2, C), dtype=torch.bfloat16, device=x.hi.device)
        out = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    _dense_planes("subsample2x_batch", x, out)
    check(_lib.load().frcnn_subsample2x_batch(_p(x.hi), _p(x.lo), N, H, W, C, _p(out.hi), _p(out.lo), _stream()),
          "frcnn_subsample2x_batch")
    return out


def conv2d_res_batch(x, w_hi, w_lo, bias, ksize, relu, res, out=None, extents=None, halvings=0):
    """frcnn_conv2d_res_batch: conv2d_res over x Act [N,H,W,Cin] with res an Act [N,H,W,Cout]; each image equals conv2d_res on
    it, bit for bit.  extents: int32 [N, 2] device image sizes, ceil(extent / 2^halvings) at this layer
    (frcnn_conv2d_res_batch_ext: every output pixel outside is written as 0)."""
    N, H, W, Cin = x.hi.shape
    taps, Cout, cin_w = w_hi.shape
    if cin_w != Cin or taps != ksize * ksize or tuple(res.hi.shape) != (N, H, W, Cout) or \
            (res.lo is not None and tuple(res.lo.shape) != (N, H, W, Cout)):
        raise FrcnnError("conv2d_res_batch: shapes do not match (x %s, w %s, res %s)" % (tuple(x.hi.shape), tuple(w_hi.shape),
                                                                                          tuple(res.hi.shape)))
    if (x.lo is None) != (w_lo is None):
        raise FrcnnError("conv2d_res_batch: activation and weight precision modes differ")
    if out is None:
        yh = torch.empty((N, H, W, Cout), dtype=torch.bfloat16, device=x.hi.device)
        out = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    _dense_planes("conv2d_res_batch", res, out)
    lib = _lib.load()
    if extents is not None:
        check(lib.frcnn_conv2d_res_batch_ext(_p(x.hi), _p(x.lo), N, H, W, Cin, _p(w_hi), _p(w_lo), _p(bias), Cout, ksize,
                                             1 if relu else 0, _p(res.hi), _p(res.lo), _p(out.hi), _p(out.lo),
                                             _per_image_pairs(extents, N, "extents"), int(halvings), _stream()),
              "frcnn_conv2d_res_batch_ext")
        return out
    check(lib.frcnn_conv2d_res_batch(_p(x.hi), _p(x.lo), N, H, W, Cin, _p(w_hi), _p(w_lo), _p(bias), Cout, ksize, 1 if relu else 0,
                                     _p(res.hi), _p(res.lo), _p(out.hi), _p(out.lo), _stream()), "frcnn_conv2d_res_batch")
    return out


def set_conv_tile(block_n=0, tile_h=0, tile_w=0):
    _lib.load().frcnn_conv2d_set_tile(block_n, tile_h, tile_w)


def set_conv_cta_group(cta_group=0):
    """0 = automatic (single CTAs), 1 = single CTAs, 2 = CTA pairs (a 2-CTA cluster sharing the weight tile) wherever the layer allows."""
    _lib.load().frcnn_conv2d_set_cta_group(cta_group)


class PinnedBlock(object):
    """A pinned host block owned by the library (frcnn_host_alloc), exposed as a numpy array and a CPU torch tensor that
    share its memory.  Uploads / downloads go through h2d() / d2h(): cudaMemcpyAsync on the given torch stream."""

    def __init__(self, shape, dtype):
        self.shape, self.dtype = tuple(int(v) for v in shape), np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        lib = _lib.load()
        self.ptr = lib.frcnn_host_alloc(self.nbytes)
        if not self.ptr:
            raise FrcnnError("frcnn_host_alloc(%d) failed: %s" % (self.nbytes, _lib.last_error()))
        buf = (ctypes.c_char * self.nbytes).from_address(self.ptr)
        self.np = np.frombuffer(buf, dtype=self.dtype).reshape(self.shape)
        self.t = torch.from_numpy(self.np)

    def fill_from(self, arr):
        """Copy a C-contiguous numpy array of the same byte size into the block (frcnn_host_copy: a few sleeping worker
        threads -- no framework thread pool is woken per image)."""
        if arr.nbytes != self.nbytes or not arr.flags.c_contiguous:
            raise FrcnnError("PinnedBlock.fill_from: need a C-contiguous array of %d bytes" % self.nbytes)
        check(_lib.load().frcnn_host_copy(self.ptr, arr.ctypes.data, self.nbytes), "frcnn_host_copy")

    def upload(self, arr, dst, stream):
        """frcnn_upload_pageable: a C-contiguous numpy array -> device tensor `dst` through this pinned block, the host copy
        of one 1 MB chunk overlapping the DMA of the previous one."""
        if arr.nbytes != self.nbytes or not arr.flags.c_contiguous:
            raise FrcnnError("PinnedBlock.upload: need a C-contiguous array of %d bytes" % self.nbytes)
        check(_lib.load().frcnn_upload_pageable(dst.data_ptr(), arr.ctypes.data, self.ptr, self.nbytes, stream.cuda_stream),
              "frcnn_upload_pageable")

    def h2d(self, dst, stream, nbytes=None):
        check(_lib.load().frcnn_memcpy_h2d_async(ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(self.ptr),
                                                 int(self.nbytes if nbytes is None else nbytes),
                                                 ctypes.c_void_p(stream.cuda_stream)), "frcnn_memcpy_h2d_async")

    def d2h(self, src, stream, nbytes=None):
        check(_lib.load().frcnn_memcpy_d2h_async(ctypes.c_void_p(self.ptr), ctypes.c_void_p(src.data_ptr()),
                                                 int(self.nbytes if nbytes is None else nbytes),
                                                 ctypes.c_void_p(stream.cuda_stream)), "frcnn_memcpy_d2h_async")

    def __del__(self):
        try:
            if self.ptr:
                self.np = self.t = None
                _lib.load().frcnn_host_free(ctypes.c_void_p(self.ptr))
                self.ptr = None
        except Exception:          # noqa: BLE001  (interpreter shutdown)
            pass


def host_copy(dst_ptr, arr):
    """frcnn_host_copy: a C-contiguous numpy array -> host memory at address dst_ptr (e.g. inside a PinnedBlock)."""
    if not arr.flags.c_contiguous:
        raise FrcnnError("host_copy: need a C-contiguous array")
    check(_lib.load().frcnn_host_copy(ctypes.c_void_p(int(dst_ptr)), ctypes.c_void_p(arr.ctypes.data), arr.nbytes), "frcnn_host_copy")


def memcpy_h2d_async(dst, src_ptr, nbytes, stream):
    """cudaMemcpyAsync(dst tensor <- host pointer) on a torch stream."""
    check(_lib.load().frcnn_memcpy_h2d_async(ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(int(src_ptr)), int(nbytes),
                                             ctypes.c_void_p(stream.cuda_stream)), "frcnn_memcpy_h2d_async")


def stream_synchronize(stream):
    check(_lib.load().frcnn_stream_synchronize(ctypes.c_void_p(stream.cuda_stream)), "frcnn_stream_synchronize")


def set_programmatic_launch(on=-1):
    """Programmatic dependent launch of the forward-path kernels for the calling thread: 1 on, 0 off, -1 = the
    FRCNN_PDL environment default (off).  Read at launch time, i.e. baked into a CUDA graph at capture."""
    _lib.load().frcnn_set_programmatic_launch(int(on))


def set_conv_smem_reserve(nbytes=0):
    """Shared memory per SM that later conv launches of this thread leave free for other streams' small kernels."""
    _lib.load().frcnn_conv2d_set_smem_reserve(int(nbytes))


def set_conv_max_ctas(max_ctas=0):
    """Cap the persistent grid of later conv launches (0 = all SMs); baked into CUDA graphs at capture time."""
    _lib.load().frcnn_conv2d_set_max_ctas(int(max_ctas))


CONV_PLAN_FIELDS = ("BN", "BK", "x3", "promote", "CG", "TH", "TW", "stages", "grid", "num_tiles", "n_parts", "splits")


def conv_last_plan():
    """The plan of this thread's last conv / GEMM launch (frcnn_conv2d_last_plan) as a dict of CONV_PLAN_FIELDS."""
    buf = (ctypes.c_int * len(CONV_PLAN_FIELDS))()
    n = _lib.load().frcnn_conv2d_last_plan(buf, len(buf))
    if n != len(CONV_PLAN_FIELDS):
        raise FrcnnError("frcnn_conv2d_last_plan: %d fields, expected %d" % (n, len(CONV_PLAN_FIELDS)))
    return dict(zip(CONV_PLAN_FIELDS, buf))


def maxpool2x2_ceil(x, out=None):
    H, W, C = x.hi.shape
    if out is None:
        yh = torch.empty(((H + 1) // 2, (W + 1) // 2, C), dtype=torch.bfloat16, device=x.hi.device)
        out = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    check(_lib.load().frcnn_maxpool2x2_ceil(_p(x.hi), _p(x.lo), H, W, C, _p(out.hi), _p(out.lo), _stream()),
          "frcnn_maxpool2x2_ceil")
    return out


def roi_pool(feat, rois, count=None, outh=7, outw=7, scale=1.0 / 16, want_f32=False, out=None):
    """feat Act [H,W,C]; rois [R_cap,4] f32; count int32[1] or None.
    Returns (Act [R_cap, outh*outw*C] viewed as [1? no: R_cap rows], fp32 copy or None)."""
    H, W, C = feat.hi.shape
    R_cap = rois.shape[0]
    if out is None:
        oh = torch.empty((1, R_cap, outh * outw * C), dtype=torch.bfloat16, device=rois.device)
        out = Act(oh, torch.empty_like(oh) if feat.lo is not None else None)
    o32 = torch.empty((R_cap, outh * outw, C), dtype=torch.float32, device=rois.device) if want_f32 else None
    check(_lib.load().frcnn_roi_pool(_p(feat.hi), _p(feat.lo), H, W, C, _p(rois), _p(count), R_cap, outh, outw,
                                     ctypes.c_float(scale), _p(out.hi), _p(out.lo), _p(o32), _stream()), "frcnn_roi_pool")
    return out, o32


def head_decode(scores_deltas, ld, rois, count, num_classes, im_h, im_w, out_prob=None, out_boxes=None):
    """scores_deltas fp32 [R_cap, ld]: columns [0,NC) scores, [NC, 5NC) deltas."""
    R_cap = rois.shape[0]
    dev = rois.device
    if out_prob is None:
        out_prob = torch.empty((R_cap, num_classes), dtype=torch.float32, device=dev)
    if out_boxes is None:
        out_boxes = torch.empty((R_cap, 4 * num_classes), dtype=torch.float32, device=dev)
    deltas_ptr = ctypes.c_void_p(scores_deltas.data_ptr() + 4 * num_classes)
    check(_lib.load().frcnn_head_decode(_p(scores_deltas), deltas_ptr, ld, _p(rois), _p(count), R_cap, num_classes,
                                        int(im_h), int(im_w), _p(out_prob), _p(out_boxes), _stream()), "frcnn_head_decode")
    return out_prob, out_boxes


def bbox_decode(boxes, trans, clip_to=None, min_size=None):
    """frcnn_bbox_decode: boxes [N,4], trans [N,4K] CUDA fp32 -> out [N,4K] (+ uint8 ok flags if min_size)."""
    _need_cuda(boxes, trans)
    boxes = boxes.contiguous().float()
    trans = trans.contiguous().float() if trans is not None else None
    N, K = boxes.shape[0], (trans if trans is not None else boxes).shape[1] // 4
    out = torch.empty_like(trans if trans is not None else boxes)
    flags = torch.empty((N,), dtype=torch.uint8, device=boxes.device) if min_size is not None else None
    im_h, im_w = (int(clip_to[0]), int(clip_to[1])) if clip_to is not None else (0, 0)
    check(_lib.load().frcnn_bbox_decode(_p(boxes), _p(trans), N, max(K, 1), 1 if clip_to is not None else 0, im_h, im_w,
                                        int(min_size or 0), _p(out), _p(flags), _stream()), "frcnn_bbox_decode")
    return out, flags


def detect(prob, boxes, count=None, nms_thresh=0.3, conf=0.8, out=None):
    """frcnn_detect.  out: optional pre-allocated (keep_idx [NC-1,R_cap], keep_count [NC-1], conf_count [NC-1]) int32."""
    R_cap, NC = prob.shape
    dev = prob.device
    if out is not None:
        keep_idx, keep_count, conf_count = out
    else:
        keep_idx = torch.empty((NC - 1, R_cap), dtype=torch.int32, device=dev)
        keep_count = torch.empty((NC - 1,), dtype=torch.int32, device=dev)
        conf_count = torch.empty((NC - 1,), dtype=torch.int32, device=dev)
    check(_lib.load().frcnn_detect(_p(prob), _p(boxes), _p(count), R_cap, NC, float(nms_thresh), ctypes.c_float(conf),
                                   _p(keep_idx), _p(keep_count), _p(conf_count), _stream()), "frcnn_detect")
    return keep_idx, keep_count, conf_count


class ProposalWorkspace(object):
    """Pre-allocated scratch + outputs of frcnn_proposals for one (A,H,W,pre,post) shape."""

    def __init__(self, A, H, W, pre_n, post_n, device, debug=False, outputs=None):
        """outputs: optional pre-allocated (rois [post_n,4] f32, scores [post_n] f32, count [1] i32) -- e.g. views of one
        result block that is copied to the host in a single transfer."""
        lib = _lib.load()
        self.shape = (A, H, W, pre_n, post_n)
        nbytes = lib.frcnn_proposals_workspace_bytes(A, H, W, pre_n)
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        if outputs is not None:
            self.rois, self.scores, self.count = outputs
        else:
            self.rois = torch.zeros((post_n, 4), dtype=torch.float32, device=device)
            self.scores = torch.zeros((post_n,), dtype=torch.float32, device=device)
            self.count = torch.zeros((1,), dtype=torch.int32, device=device)
        k_cap = min(pre_n, A * H * W)
        self.dbg_dets = torch.zeros((k_cap, 5), dtype=torch.float32, device=device) if debug else None
        self.dbg_idx = torch.zeros((k_cap,), dtype=torch.int32, device=device) if debug else None
        self.dbg_num = torch.zeros((1,), dtype=torch.int32, device=device) if debug else None


def proposals(cls, bbox, anchors, A, H, W, feat_stride, im_h, im_w, min_size, pre_n, post_n, nms_thresh,
              layout="nchw", ld=0, cls_is_logits=False, work=None, debug=False):
    """frcnn_proposals.  layout "nchw": cls (2A,H,W), bbox (4A,H,W) planar (the reference's);
    layout "nhwc": one fp32 matrix [H*W, ld] with cls in columns [0,2A) and bbox in [2A,6A)."""
    dev = cls.device
    if work is None or work.shape != (A, H, W, pre_n, post_n) or (debug and work.dbg_dets is None):
        work = ProposalWorkspace(A, H, W, pre_n, post_n, dev, debug)
    if layout == "nchw":
        cs, ps, bcs, bps = H * W, 1, H * W, 1
        bbox_ptr = _p(bbox)
    else:
        cs, ps, bcs, bps = 1, ld, 1, ld
        bbox_ptr = ctypes.c_void_p(cls.data_ptr() + 4 * 2 * A) if bbox is None else _p(bbox)
    check(_lib.load().frcnn_proposals(_p(cls), cs, ps, 1 if cls_is_logits else 0, bbox_ptr, bcs, bps, _p(anchors),
                                      A, H, W, feat_stride, int(im_h), int(im_w), int(min_size), pre_n, post_n,
                                      float(nms_thresh), _p(work.rois), _p(work.scores), _p(work.count),
                                      _p(work.dbg_dets), _p(work.dbg_idx), _p(work.dbg_num),
                                      _p(work.ws), work.ws.numel(), _stream()), "frcnn_proposals")
    return work


# ---- batched post-processing: N images in one launch per kernel.  Every per-image array is a tensor whose dim 0 is the
# image: each image's block must be dense, the blocks may sit any distance apart (e.g. views of BatchPlan's result blocks),
# and that distance -- the tensor's stride(0) -- is the image stride handed to the library.
def _image_stride(t, inner, what):
    """t: [N, *inner] with each image's block dense (row-major); returns the image stride in elements."""
    if t is None:
        return 0
    _need_cuda(t)
    if tuple(t.shape[1:]) != tuple(inner):
        raise FrcnnError("%s: per-image shape %s, expected %s" % (what, tuple(t.shape[1:]), tuple(inner)))
    want = 1
    for d, st in zip(reversed(inner), reversed(t.stride()[1:])):
        if d > 1 and st != want:
            raise FrcnnError("%s: each image's block must be dense (strides %s)" % (what, tuple(t.stride())))
        want *= d
    return int(t.stride(0))


def _counts_stride(counts, N, what):
    """counts: None (R_cap each) or an int32 tensor whose dim 0 is the image (e.g. one word of every result block)."""
    if counts is None:
        return 0
    _need_cuda(counts)
    if counts.dtype != torch.int32 or counts.shape[0] != N:
        raise FrcnnError("%s: counts must be int32 with one entry per image" % what)
    return int(counts.stride(0))


def maxpool2x2_ceil_batch(x, out=None):
    """frcnn_maxpool2x2_ceil_batch: Act [N,H,W,C] -> Act [N,ceil(H/2),ceil(W/2),C], one launch."""
    N, H, W, C = x.hi.shape
    if out is None:
        yh = torch.empty((N, (H + 1) // 2, (W + 1) // 2, C), dtype=torch.bfloat16, device=x.hi.device)
        out = Act(yh, torch.empty_like(yh) if x.lo is not None else None)
    for t in (x.hi, x.lo, out.hi, out.lo):
        if t is not None and not t.is_contiguous():
            raise FrcnnError("maxpool2x2_ceil_batch: planes must be dense [N,H,W,C]")
    check(_lib.load().frcnn_maxpool2x2_ceil_batch(_p(x.hi), _p(x.lo), N, H, W, C, _p(out.hi), _p(out.lo), _stream()),
          "frcnn_maxpool2x2_ceil_batch")
    return out


def roi_pool_batch(feat, rois, counts=None, outh=7, outw=7, scale=1.0 / 16, want_f32=False, out=None, out_f32=None,
                   extents=None, halvings=0):
    """frcnn_roi_pool_batch: feat Act [N,H,W,C] (dense); rois [N,R_cap,4]; counts [N] int32 (or None).  Returns (Act
    [N,R_cap,outh*outw*C], fp32 [N,R_cap,outh*outw,C] or None).  `out` / `out_f32` may be strided views (image blocks
    apart); the library takes one image stride for all outputs, so given both, their strides must agree.
    extents: int32 [N, 2] device image sizes (input pixels); image n's map is the top-left ceil(extent / 2^halvings) of
    its slot and its bins are clamped to it (frcnn_roi_pool_batch_ext)."""
    N, H, W, C = feat.hi.shape
    R_cap = rois.shape[1]
    K = outh * outw * C
    if not feat.hi.is_contiguous() or (feat.lo is not None and not feat.lo.is_contiguous()):
        raise FrcnnError("roi_pool_batch: feature planes must be dense [N,H,W,C]")
    rs = _image_stride(rois, (R_cap, 4), "roi_pool_batch rois")
    cs = _counts_stride(counts, N, "roi_pool_batch")
    if out is None:
        oh = torch.empty((N, R_cap, K), dtype=torch.bfloat16, device=rois.device)
        out = Act(oh, torch.empty_like(oh) if feat.lo is not None else None)
    os_ = _image_stride(out.hi, (R_cap, K), "roi_pool_batch out")
    if out.lo is not None and _image_stride(out.lo, (R_cap, K), "roi_pool_batch out") != os_:
        raise FrcnnError("roi_pool_batch: hi and lo outputs need the same image stride")
    o32 = out_f32
    if want_f32 and o32 is None:          # image blocks as far apart as the bf16 output's
        o32 = torch.empty((N, os_), dtype=torch.float32, device=rois.device)[:, :K].view(N, R_cap, outh * outw, C)
    if o32 is not None and _image_stride(o32, (R_cap, outh * outw, C), "roi_pool_batch out_f32") != os_ and N > 1:
        raise FrcnnError("roi_pool_batch: the bf16 and fp32 outputs need the same image stride")
    if extents is not None:
        check(_lib.load().frcnn_roi_pool_batch_ext(_p(feat.hi), _p(feat.lo), N, H, W, C, _p(rois), rs, _p(counts), cs, R_cap, outh,
                                                   outw, ctypes.c_float(scale), _per_image_pairs(extents, N, "extents"),
                                                   int(halvings), _p(out.hi), _p(out.lo), _p(o32), os_, _stream()),
              "frcnn_roi_pool_batch_ext")
        return out, o32
    check(_lib.load().frcnn_roi_pool_batch(_p(feat.hi), _p(feat.lo), N, H, W, C, _p(rois), rs, _p(counts), cs, R_cap, outh, outw,
                                           ctypes.c_float(scale), _p(out.hi), _p(out.lo), _p(o32), os_, _stream()),
          "frcnn_roi_pool_batch")
    return out, o32


def head_decode_batch(scores_deltas, ld, rois, counts, num_classes, im_h, im_w, out_prob=None, out_boxes=None, im_info=None):
    """frcnn_head_decode_batch: scores_deltas fp32 [N,R_cap,ld] (columns [0,NC) scores, [NC,5NC) deltas), rois [N,R_cap,4],
    counts [N] int32 or None; out_prob [N,R_cap,NC], out_boxes [N,R_cap,4NC] (may be strided views).
    im_info: int32 [N, 2] device clip bounds (im_h, im_w) per image, in place of (im_h, im_w) (frcnn_head_decode_batch_ext)."""
    N, R_cap = rois.shape[0], rois.shape[1]
    dev = rois.device
    if out_prob is None:
        out_prob = torch.empty((N, R_cap, num_classes), dtype=torch.float32, device=dev)
    if out_boxes is None:
        out_boxes = torch.empty((N, R_cap, 4 * num_classes), dtype=torch.float32, device=dev)
    ins = _image_stride(scores_deltas, (R_cap, ld), "head_decode_batch scores")
    rs = _image_stride(rois, (R_cap, 4), "head_decode_batch rois")
    cs = _counts_stride(counts, N, "head_decode_batch")
    ps = _image_stride(out_prob, (R_cap, num_classes), "head_decode_batch out_prob")
    bs = _image_stride(out_boxes, (R_cap, 4 * num_classes), "head_decode_batch out_boxes")
    deltas_ptr = ctypes.c_void_p(scores_deltas.data_ptr() + 4 * num_classes)
    if im_info is not None:
        check(_lib.load().frcnn_head_decode_batch_ext(N, _p(scores_deltas), deltas_ptr, ld, ins, _p(rois), rs, _p(counts), cs, R_cap,
                                                      num_classes, _per_image_pairs(im_info, N, "im_info"), _p(out_prob), ps,
                                                      _p(out_boxes), bs, _stream()), "frcnn_head_decode_batch_ext")
        return out_prob, out_boxes
    check(_lib.load().frcnn_head_decode_batch(N, _p(scores_deltas), deltas_ptr, ld, ins, _p(rois), rs, _p(counts), cs, R_cap, num_classes,
                                              int(im_h), int(im_w), _p(out_prob), ps, _p(out_boxes), bs, _stream()),
          "frcnn_head_decode_batch")
    return out_prob, out_boxes


def detect_batch(prob, boxes, counts=None, nms_thresh=0.3, conf=0.8, out=None):
    """frcnn_detect_batch: prob [N,R_cap,NC], boxes [N,R_cap,4NC], counts [N] int32 or None.  out: optional (keep_idx
    [N,NC-1,R_cap], keep_count [N,NC-1], conf_count [N,NC-1]) int32, possibly strided views."""
    N, R_cap, NC = prob.shape
    dev = prob.device
    if out is not None:
        keep_idx, keep_count, conf_count = out
    else:
        keep_idx = torch.empty((N, NC - 1, R_cap), dtype=torch.int32, device=dev)
        keep_count = torch.empty((N, NC - 1), dtype=torch.int32, device=dev)
        conf_count = torch.empty((N, NC - 1), dtype=torch.int32, device=dev)
    ps = _image_stride(prob, (R_cap, NC), "detect_batch prob")
    bs = _image_stride(boxes, (R_cap, 4 * NC), "detect_batch boxes")
    cs = _counts_stride(counts, N, "detect_batch")
    ks = _image_stride(keep_idx, (NC - 1, R_cap), "detect_batch keep_idx")
    kc = _image_stride(keep_count, (NC - 1,), "detect_batch keep_count")
    cc = _image_stride(conf_count, (NC - 1,), "detect_batch conf_count")
    check(_lib.load().frcnn_detect_batch(N, _p(prob), ps, _p(boxes), bs, _p(counts), cs, R_cap, NC, float(nms_thresh),
                                         ctypes.c_float(conf), _p(keep_idx), ks, _p(keep_count), kc, _p(conf_count), cc, _stream()),
          "frcnn_detect_batch")
    return keep_idx, keep_count, conf_count


def detection_lists_batch(prob, boxes, keep_idx, conf_count, im_scale, out=None):
    """frcnn_detection_lists_batch: the lists forward.py:50-59 draws (preprocess.result_detections), built on the device.
    prob [N,R_cap,NC], boxes [N,R_cap,4NC] fp32 and keep_idx [N,NC-1,R_cap] / conf_count [N,NC-1] int32 (detect_batch's
    outputs), each possibly a strided view; im_scale float64 [N] device.  out: optional dense (dets int32 [N,cap,5], scores
    fp32 [N,cap], det_count int32 [N]), cap = (NC-1)*R_cap.  Returns that triple; rows past det_count[n] are not written."""
    N, R_cap, NC = prob.shape
    dev = prob.device
    cap = (NC - 1) * R_cap
    if out is None:
        out = (torch.empty((N, cap, 5), dtype=torch.int32, device=dev), torch.empty((N, cap), dtype=torch.float32, device=dev),
               torch.empty((N,), dtype=torch.int32, device=dev))
    dets, scores, det_count = out
    _need_cuda(im_scale, dets, scores, det_count)
    for t, dt, shape, what in ((im_scale, torch.float64, (N,), "im_scale"), (dets, torch.int32, (N, cap, 5), "dets"),
                               (scores, torch.float32, (N, cap), "scores"), (det_count, torch.int32, (N,), "det_count")):
        if t.dtype != dt or tuple(t.shape) != shape or not t.is_contiguous():
            raise FrcnnError("detection_lists_batch: %s must be a dense %s %s CUDA tensor" % (what, dt, list(shape)))
    ps = _image_stride(prob, (R_cap, NC), "detection_lists_batch prob")
    bs = _image_stride(boxes, (R_cap, 4 * NC), "detection_lists_batch boxes")
    ks = _image_stride(keep_idx, (NC - 1, R_cap), "detection_lists_batch keep_idx")
    cc = _image_stride(conf_count, (NC - 1,), "detection_lists_batch conf_count")
    check(_lib.load().frcnn_detection_lists_batch(N, _p(prob), ps, _p(boxes), bs, _p(keep_idx), ks, _p(conf_count), cc, _p(im_scale),
                                                  R_cap, NC, _p(dets), _p(scores), _p(det_count), _stream()),
          "frcnn_detection_lists_batch")
    return dets, scores, det_count


def voc_eval_workspace_bytes(num_classes, capacity, max_images, max_gt):
    """frcnn_voc_eval_workspace_bytes; raises on bad sizes."""
    n = _lib.load().frcnn_voc_eval_workspace_bytes(int(num_classes), int(capacity), int(max_images), int(max_gt))
    if n == 0:
        raise FrcnnError("voc_eval_workspace_bytes: %s" % _lib.last_error())
    return int(n)


def voc_eval_append_batch(prob, boxes, keep_idx, conf_count, im_scale, image_base, capacity, max_images, ws):
    """frcnn_voc_eval_append_batch: appends images image_base .. image_base+N-1 of a dataset to the evaluation workspace `ws`
    (a uint8 CUDA tensor of voc_eval_workspace_bytes, zeroed before the dataset's first append).  prob / boxes / keep_idx /
    conf_count as detection_lists_batch takes them; im_scale float64 [N] device, this batch's scales."""
    N, R_cap, NC = prob.shape
    _need_cuda(im_scale, ws)
    for t, dt, what in ((prob, torch.float32, "prob"), (boxes, torch.float32, "boxes"), (keep_idx, torch.int32, "keep_idx"),
                        (conf_count, torch.int32, "conf_count"), (ws, torch.uint8, "ws")):
        if t.dtype != dt:
            raise FrcnnError("voc_eval_append_batch: %s must be %s (got %s)" % (what, dt, t.dtype))
    if im_scale.dtype != torch.float64 or tuple(im_scale.shape) != (N,) or not im_scale.is_contiguous():
        raise FrcnnError("voc_eval_append_batch: im_scale must be a dense float64 [%d] CUDA tensor" % N)
    ps = _image_stride(prob, (R_cap, NC), "voc_eval_append_batch prob")
    bs = _image_stride(boxes, (R_cap, 4 * NC), "voc_eval_append_batch boxes")
    ks = _image_stride(keep_idx, (NC - 1, R_cap), "voc_eval_append_batch keep_idx")
    cc = _image_stride(conf_count, (NC - 1,), "voc_eval_append_batch conf_count")
    check(_lib.load().frcnn_voc_eval_append_batch(N, _p(prob), ps, _p(boxes), bs, _p(keep_idx), ks, _p(conf_count), cc, _p(im_scale),
                                                  R_cap, NC, int(image_base), int(capacity), int(max_images), _p(ws), ws.numel(),
                                                  _stream()),
          "frcnn_voc_eval_append_batch")


def voc_eval(num_classes, capacity, max_images, max_gt, gt_offsets, gt_boxes, gt_labels, gt_difficult, iou_thresh, ws, out=None,
             n_gt=None):
    """frcnn_voc_eval over the detections appended to `ws`: the GT as a device CSR (gt_offsets int32 [n_images+1], gt_boxes
    float32 [G,4], gt_labels int32 [G], gt_difficult uint8 [G]; n_gt: the boxes in use, default G -- a caller without GT
    passes one-row arrays and n_gt = 0, since an empty tensor has no device pointer).  Returns `out`, the float64
    [3 + 6*(num_classes-1)] device result (status, mAP07, mAP, then per class npos, n_det, tp, fp, ap07, ap)."""
    _need_cuda(gt_offsets, gt_boxes, gt_labels, gt_difficult, ws)
    G = int(gt_labels.shape[0])
    n_gt = G if n_gt is None else int(n_gt)
    if not 0 <= n_gt <= G:
        raise FrcnnError("voc_eval: n_gt = %d outside [0, %d]" % (n_gt, G))
    for t, dt, shape, what in ((gt_boxes, torch.float32, (G, 4), "gt_boxes"), (gt_labels, torch.int32, (G,), "gt_labels"),
                               (gt_difficult, torch.uint8, (G,), "gt_difficult")):
        if t.dtype != dt or tuple(t.shape) != shape or not t.is_contiguous():
            raise FrcnnError("voc_eval: %s must be a dense %s %s CUDA tensor" % (what, dt, list(shape)))
    if gt_offsets.dtype != torch.int32 or gt_offsets.dim() != 1 or not gt_offsets.is_contiguous():
        raise FrcnnError("voc_eval: gt_offsets must be a dense int32 [n_images+1] CUDA tensor")
    if out is None:
        out = torch.empty((3 + 6 * (num_classes - 1),), dtype=torch.float64, device=ws.device)
    check(_lib.load().frcnn_voc_eval(int(num_classes), int(capacity), int(max_images), int(max_gt), int(gt_offsets.shape[0]) - 1,
                                     _p(gt_offsets), _p(gt_boxes), _p(gt_labels), _p(gt_difficult), n_gt, float(iou_thresh), _p(out),
                                     _p(ws), ws.numel(), _stream()),
          "frcnn_voc_eval")
    return out


class ProposalBatchWorkspace(object):
    """Scratch + outputs of frcnn_proposals_batch for N images of one (A,H,W,pre,post) shape: N workspace slices in one
    buffer, rois [N,post_n,4], scores [N,post_n], count [N] int32 and, with debug, dbg_dets [N,k,5], dbg_idx [N,k],
    dbg_num [N] (k = min(pre_n, A*H*W))."""

    def __init__(self, N, A, H, W, pre_n, post_n, device, debug=False, outputs=None):
        """outputs: optional pre-allocated (rois [N,post_n,4], scores [N,post_n], count [N]) -- e.g. strided views of N result
        blocks."""
        lib = _lib.load()
        self.N, self.shape = int(N), (A, H, W, pre_n, post_n)
        nbytes = lib.frcnn_proposals_batch_workspace_bytes(int(N), A, H, W, pre_n)
        if nbytes == 0:
            raise FrcnnError("frcnn_proposals_batch_workspace_bytes: bad shape N=%r A=%d H=%d W=%d pre=%d" % (N, A, H, W, pre_n))
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        if outputs is not None:
            self.rois, self.scores, self.count = outputs
        else:
            self.rois = torch.zeros((N, post_n, 4), dtype=torch.float32, device=device)
            self.scores = torch.zeros((N, post_n), dtype=torch.float32, device=device)
            self.count = torch.zeros((N,), dtype=torch.int32, device=device)
        k_cap = min(pre_n, A * H * W)
        self.dbg_dets = torch.zeros((N, k_cap, 5), dtype=torch.float32, device=device) if debug else None
        self.dbg_idx = torch.zeros((N, k_cap), dtype=torch.int32, device=device) if debug else None
        self.dbg_num = torch.zeros((N,), dtype=torch.int32, device=device) if debug else None


def proposals_batch(cls, bbox, anchors, A, H, W, feat_stride, im_h, im_w, min_size, pre_n, post_n, nms_thresh,
                    layout="nchw", ld=0, cls_is_logits=False, work=None, debug=False, extents=None, halvings=0, im_info=None):
    """frcnn_proposals_batch over N images (one clip bound for all).  layout "nchw": cls (N,2A,H,W), bbox (N,4A,H,W) planar;
    layout "nhwc": cls one fp32 tensor [N,H*W,ld] with cls in columns [0,2A) and bbox in [2A,6A) (bbox None).  Returns the
    ProposalBatchWorkspace holding the outputs.
    A canvas batch (frcnn_proposals_batch_ext): extents int32 [N, 2] device image sizes in input pixels, the feature-map
    extent being ceil(extent / 2^halvings) of the H x W slot; im_info int32 [N, 2] device clip bounds per image, in place of
    (im_h, im_w).  Both are required together; no debug outputs."""
    _need_cuda(cls)
    N = cls.shape[0]
    dev = cls.device
    if work is None or work.N != N or work.shape != (A, H, W, pre_n, post_n) or (debug and work.dbg_dets is None):
        work = ProposalBatchWorkspace(N, A, H, W, pre_n, post_n, dev, debug)
    if layout == "nchw":
        cs, ps, bcs, bps = H * W, 1, H * W, 1
        cis = _image_stride(cls, (2 * A, H, W), "proposals_batch cls")
        bis = _image_stride(bbox, (4 * A, H, W), "proposals_batch bbox")
        bbox_ptr = _p(bbox)
    else:
        cs, ps, bcs, bps = 1, ld, 1, ld
        cis = _image_stride(cls, (H * W, ld), "proposals_batch cls")
        bis = cis if bbox is None else _image_stride(bbox, (H * W, ld), "proposals_batch bbox")
        bbox_ptr = ctypes.c_void_p(cls.data_ptr() + 4 * 2 * A) if bbox is None else _p(bbox)
    k_cap = min(pre_n, A * H * W)
    rs = _image_stride(work.rois, (post_n, 4), "proposals_batch rois")
    ss = _image_stride(work.scores, (post_n,), "proposals_batch scores")
    cnt = _counts_stride(work.count, N, "proposals_batch")
    dd = _image_stride(work.dbg_dets, (k_cap, 5), "proposals_batch dbg_dets") if debug else 0
    di = _image_stride(work.dbg_idx, (k_cap,), "proposals_batch dbg_idx") if debug else 0
    dn = _counts_stride(work.dbg_num, N, "proposals_batch dbg_num") if debug else 0
    if extents is not None or im_info is not None:
        if extents is None or im_info is None or debug:
            raise FrcnnError("proposals_batch: a canvas batch needs both extents and im_info, and has no debug outputs")
        check(_lib.load().frcnn_proposals_batch_ext(N, _p(cls), cs, ps, cis, 1 if cls_is_logits else 0, bbox_ptr, bcs, bps, bis,
                                                    _p(anchors), A, H, W, feat_stride, _per_image_pairs(extents, N, "extents"),
                                                    int(halvings), _per_image_pairs(im_info, N, "im_info"), int(min_size), pre_n,
                                                    post_n, float(nms_thresh), _p(work.rois), rs, _p(work.scores), ss,
                                                    _p(work.count), cnt, _p(work.ws), work.ws.numel(), _stream()),
              "frcnn_proposals_batch_ext")
        return work
    check(_lib.load().frcnn_proposals_batch(N, _p(cls), cs, ps, cis, 1 if cls_is_logits else 0, bbox_ptr, bcs, bps, bis, _p(anchors),
                                            A, H, W, feat_stride, int(im_h), int(im_w), int(min_size), pre_n, post_n,
                                            float(nms_thresh), _p(work.rois), rs, _p(work.scores), ss, _p(work.count), cnt,
                                            _p(work.dbg_dets) if debug else None, dd, _p(work.dbg_idx) if debug else None, di,
                                            _p(work.dbg_num) if debug else None, dn, _p(work.ws), work.ws.numel(), _stream()),
          "frcnn_proposals_batch")
    return work


def nms(dets, thresh, mode=_lib.NMS_GE_DOUBLE, max_keep=0):
    """Device greedy NMS over unsorted dets [n,5] (CUDA fp32).  Returns (keep int32[n], count int32[1])."""
    _need_cuda(dets)
    dets = dets.contiguous().float()
    n = dets.shape[0]
    lib = _lib.load()
    ws = torch.empty(lib.frcnn_nms_workspace_bytes(n), dtype=torch.uint8, device=dets.device)
    keep = torch.empty((max(n, 1),), dtype=torch.int32, device=dets.device)
    count = torch.zeros((1,), dtype=torch.int32, device=dets.device)
    check(lib.frcnn_nms(_p(dets), n, float(thresh), mode, max_keep, _p(keep), _p(count), _p(ws), ws.numel(), _stream()),
          "frcnn_nms")
    return keep, count


_nms_tls = None


def cpu_nms_host(dets_np, thresh, device_id=-1):
    """Host-array entry (frcnn_cpu_nms_host): numpy f32 [n,5] in, list[int] out -- the drop-in
    behind models.cpu_nms.cpu_nms (the arithmetic runs on the GPU).  Called 20 times per image by forward.py's loop, so
    the wrapper itself is kept lean: a per-thread output buffer, raw addresses instead of ctypes casts."""
    global _nms_tls
    d = dets_np if (dets_np.dtype == np.float32 and dets_np.flags.c_contiguous) else np.ascontiguousarray(dets_np, dtype=np.float32)
    if d.ndim != 2 or d.shape[1] != 5:
        raise FrcnnError("cpu_nms: dets must be (N,5), got %s" % (d.shape,))
    n = d.shape[0]
    if _nms_tls is None:
        import threading
        _nms_tls = threading.local()
    keep = getattr(_nms_tls, "keep", None)
    if keep is None or keep.shape[0] < n:
        keep = _nms_tls.keep = np.empty(max(n, 1024), dtype=np.int32)
        _nms_tls.fn = _lib.load().frcnn_cpu_nms_host
    r = _nms_tls.fn(d.ctypes.data, n, float(thresh), keep.ctypes.data, device_id)
    if r < 0:
        raise FrcnnError("frcnn_cpu_nms_host failed (status %d): %s" % (r, _lib.last_error()))
    return keep[:r].tolist()


def gpu_nms_host(sorted_dets_np, thresh, device_id=0):
    """The reference FFI `_nms` (models/gpu_nms.hpp:9-10): pre-sorted host boxes, `>` comparison."""
    d = np.ascontiguousarray(sorted_dets_np, dtype=np.float32)
    n, dim = d.shape
    keep = np.empty(max(n, 1), dtype=np.int32)
    num = ctypes.c_int(0)
    _lib.load()._nms(keep.ctypes.data_as(ctypes.c_void_p), ctypes.cast(ctypes.pointer(num), ctypes.c_void_p),
                     d.ctypes.data_as(ctypes.c_void_p), n, dim, ctypes.c_float(thresh), device_id)
    if num.value < 0:
        raise FrcnnError("_nms failed: %s" % _lib.last_error())
    return keep[: num.value].copy()
