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


def pack_conv_weights(w, cin_pad=None, precision="bf16x3", perm_chw=None):
    """OIHW (or (Cout, K)) float32 weights -> ([taps, Cout, cin_pad] bf16 hi, lo or None)."""
    _need_cuda(w)
    w = w.contiguous().float()
    if w.dim() == 2:
        w = w[:, :, None, None]
    Cout, Cin, kh, kw = w.shape
    cin_pad = cin_pad or round_up(Cin, 8)
    hi = torch.empty((kh * kw, Cout, cin_pad), dtype=torch.bfloat16, device=w.device)
    lo = torch.empty_like(hi) if precision == "bf16x3" else None
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


def pack_conv_weights_im2col(w, precision="bf16x3"):
    """OIHW (Cout, Cin<=3, 3, 3) float32 -> ([1, Cout, 32] bf16 hi, lo or None), K order of pack_image_im2col."""
    _need_cuda(w)
    w = w.contiguous().float()
    Cout, Cin, kh, kw = w.shape
    if (kh, kw) != (3, 3):
        raise FrcnnError("pack_conv_weights_im2col: 3x3 kernels only")
    hi = torch.empty((1, Cout, 32), dtype=torch.bfloat16, device=w.device)
    lo = torch.empty_like(hi) if precision == "bf16x3" else None
    check(_lib.load().frcnn_pack_conv_weights_im2col3x3(_p(w), Cout, Cin, _p(hi), _p(lo), _stream()),
          "frcnn_pack_conv_weights_im2col3x3")
    return hi, lo


def pad_bias(b, n):
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


def pack_conv_weights_im2col_general(w, k_pad, precision="bf16x3"):
    """OIHW float32 -> ([1, Cout, k_pad] bf16 hi, lo or None) in the K order of pack_image_im2col_general."""
    w = w.contiguous().float()
    Cout, Cin, kh, kw = w.shape
    hi = torch.empty((1, Cout, k_pad), dtype=torch.bfloat16, device=w.device)
    lo = torch.empty_like(hi) if precision == "bf16x3" else None
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
