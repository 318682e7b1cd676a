"""Caller-side pre/post-processing of the reference's forward.py on the device ("next" row, SURVEY.md 8f rank 4).

  img_preprocessing(orig_img, pixel_means, max_size=1000, scale=600)   forward.py:34-45, same signature/returns
  detections(cls_prob, pred_boxes, im_scale, nms_thresh=0.3, conf=0.8)  the numeric part of draw_result, forward.py:48-59

The raw uint8 BGR image is uploaded (4x+ fewer H2D bytes than the float32 tensor forward.py uploads) and mean
subtraction + OpenCV-compatible bilinear resize + HWC->CHW run in frcnn_preprocess_bgr8; per-class NMS + confidence
filter run in frcnn_detect.  Drawing (cv.rectangle / putText) stays out of scope.
"""
import numpy as np
import torch

from . import _lib, ops
from ._lib import check

PIXEL_MEANS = np.array([[[102.9801, 115.9465, 122.7717]]])     # forward.py:22 (BGR)


def plan_size(h0, w0, scale=600, max_size=1000):
    """(im_scale, H, W): forward.py:38-41 + cv.resize's output-size rounding (half to even)."""
    im_scale = float(scale) / float(min(h0, w0))
    if np.round(im_scale * max(h0, w0)) > max_size:
        im_scale = float(max_size) / float(max(h0, w0))
    return im_scale, int(np.rint(h0 * im_scale)), int(np.rint(w0 * im_scale))


def img_preprocessing(orig_img, pixel_means=PIXEL_MEANS, max_size=1000, scale=600, out=None):
    """uint8 (h0,w0,3) BGR image (numpy or CUDA tensor) -> ((3,H,W) float32 CUDA tensor, im_scale)."""
    if isinstance(orig_img, np.ndarray):
        if orig_img.dtype != np.uint8 or orig_img.ndim != 3 or orig_img.shape[2] != 3:
            raise _lib.FrcnnError("img_preprocessing expects a uint8 (h, w, 3) BGR image")
        img = torch.from_numpy(np.ascontiguousarray(orig_img)).cuda(non_blocking=True)
    else:
        img = orig_img.contiguous()
        if img.dtype != torch.uint8 or not img.is_cuda:
            raise _lib.FrcnnError("img_preprocessing expects a uint8 image (numpy, or a CUDA tensor)")
    h0, w0, _ = img.shape
    im_scale, H, W = plan_size(h0, w0, scale, max_size)
    if out is None:
        out = torch.empty((3, H, W), dtype=torch.float32, device=img.device)
    m = np.asarray(pixel_means, dtype=np.float64).reshape(-1)
    check(_lib.load().frcnn_preprocess_bgr8(ops._p(img), h0, w0, float(m[0]), float(m[1]), float(m[2]), float(im_scale),
                                            H, W, ops._p(out), ops._stream()), "frcnn_preprocess_bgr8")
    return out, im_scale


def result_detections(res, im_scale):
    """The list forward.py:50-59 draws, from host arrays: res holds prob [R,NC], boxes [R,4NC] and the per-class NMS lists
    keep_idx [NC-1, >=R] / conf_count [NC-1] (an unpacked result block of a with_detect plan, or detections() below).
    Boxes are divided by im_scale and truncated like `map(int, dets[i, :4] / im_scale)`; (cls_id, x1, y1, x2, y2, score)
    in the reference's iteration order."""
    prob, boxes, keep_idx, conf_count = res["prob"], res["boxes"], res["keep_idx"], res["conf_count"]
    out = []
    for c in range(1, prob.shape[1]):
        for r in keep_idx[c - 1, :conf_count[c - 1]]:
            x1, y1, x2, y2 = map(int, boxes[r, 4 * c:4 * c + 4] / im_scale)
            out.append((c, x1, y1, x2, y2, float(prob[r, c])))
    return out


def detections(cls_prob, pred_boxes, im_scale, nms_thresh=0.3, conf=0.8, count=None):
    """forward.py:48-59 without the drawing: for every foreground class, per-class NMS (device), confidence
    filter, boxes divided by im_scale and truncated to int like `map(int, dets[i, :4] / im_scale)`.
    Returns a list of (cls_id, x1, y1, x2, y2, score) in the reference's iteration order."""
    keep_idx, keep_count, conf_count = ops.detect(cls_prob, pred_boxes, count, nms_thresh, conf)
    return result_detections(dict(prob=cls_prob.detach().cpu().numpy(), boxes=pred_boxes.detach().cpu().numpy(),
                                  keep_idx=keep_idx.cpu().numpy(), conf_count=conf_count.cpu().numpy()), im_scale)


# ---- raw photos into a canvas batch (engine.CanvasBatchPlan(raw_input=True)): one block [descriptor header | pixels]
# The header holds, for the N slots, the five arrays frcnn_preprocess_bgr8_canvas and the later *_batch_ext kernels read;
# the pixels follow at header_bytes.  Host and device copies share the layout, so one H2D copy delivers a whole batch.
RAW_FIELDS = (("extents", np.int32, 2), ("im_info", np.int32, 2), ("src_hw", np.int32, 2), ("src_off", np.int64, 1),
              ("inv_scale", np.float64, 1))
RAW_ALIGN = 64          # images start on 64-byte boundaries of the pixel area (the kernel itself reads single bytes)


def raw_header_layout(N):
    """({name: (byte offset, dtype, per-slot items)}, header_bytes): every array takes 8 * N bytes, and the pixels start at
    header_bytes, a multiple of 256."""
    return ({name: (8 * N * k, dt, items) for k, (name, dt, items) in enumerate(RAW_FIELDS)},
            ops.round_up(8 * N * len(RAW_FIELDS), 256))


def raw_header_views(buf, N):
    """numpy views of the header arrays inside `buf`, a uint8 array that starts with a header for N slots."""
    layout, _ = raw_header_layout(N)
    return {name: buf[off:off + 8 * N].view(dt).reshape((N, 2) if items == 2 else (N,)) for name, (off, dt, items) in layout.items()}


def canvas_sizes(shapes, N, Hc, Wc, img_infos=None):
    """The int32 [2, N, 2] extents (row 0) and clip bounds (row 1) of one canvas batch of float images: shapes = the
    (3, H, W) of at most N images, each at the top-left of its Hc x Wc slot; the remaining slots are empty (0 x 0).
    img_infos: per-image clip bounds, default (H, W).  Raises FrcnnError when there are too many images or an image does
    not fit the canvas."""
    if len(shapes) > N or (img_infos is not None and len(img_infos) != len(shapes)):
        raise _lib.FrcnnError("canvas batch: %d images (%s img_infos) for %d slots" %
                              (len(shapes), "no" if img_infos is None else len(img_infos), N))
    sizes = np.zeros((2, N, 2), dtype=np.int32)
    for n, shape in enumerate(shapes):
        if len(shape) != 3 or shape[0] != 3 or not (0 < shape[1] <= Hc and 0 < shape[2] <= Wc):
            raise _lib.FrcnnError("canvas batch: image %d of shape %s does not fit a (3,%d,%d) canvas" % (n, tuple(shape), Hc, Wc))
        sizes[0, n] = shape[1:]
        sizes[1, n] = shape[1:] if img_infos is None else (int(img_infos[n][0]), int(img_infos[n][1]))
    return sizes


def raw_photo_shapes(photos):
    """The (h0, w0) of raw photos; raises FrcnnError unless every one is a uint8 (h, w, 3) numpy array."""
    for n, x in enumerate(photos):
        if not isinstance(x, np.ndarray) or x.dtype != np.uint8 or x.ndim != 3 or x.shape[2] != 3:
            raise _lib.FrcnnError("raw batch: photo %d is not a uint8 (h, w, 3) numpy array" % n)
    return [x.shape[:2] for x in photos]


def fill_raw_block(buf, hdr, photos, N):
    """Writes one batch into `buf`, a uint8 numpy view of a host [header | pixels] block for N slots: the header that
    raw_batch_header made for `photos` (raw_photo_shapes' photos), then each photo at its src_off.  Returns the bytes to
    upload, header included."""
    offs = raw_header_views(hdr, N)["src_off"]
    nbytes = hdr.size + max([int(offs[n]) + x.nbytes for n, x in enumerate(photos)], default=0)
    if nbytes > buf.size:
        raise _lib.FrcnnError("raw batch: %d bytes for a block of %d" % (nbytes, buf.size))
    buf[:hdr.size] = hdr
    for n, x in enumerate(photos):
        ops.host_copy(buf.ctypes.data + hdr.size + int(offs[n]), np.ascontiguousarray(x))
    return nbytes


def raw_batch_header(shapes, N, Hc, Wc, arena_bytes, img_infos=None, scale=600, max_size=1000):
    """The header of one batch of raw images: shapes = the (h0, w0) of at most N uint8 BGR images, laid out one after the
    other (RAW_ALIGN) in a pixel area of arena_bytes; the remaining slots are empty.  img_infos: per-image clip bounds,
    default the resized (H, W).  Returns (uint8 header array, [im_scale], pixel bytes used).  Raises FrcnnError when there
    are too many images, a resized image does not fit the Hc x Wc canvas, or the pixels do not fit the arena."""
    shapes = [(int(h0), int(w0)) for h0, w0 in shapes]
    if len(shapes) > N:
        raise _lib.FrcnnError("raw batch: %d images for %d slots" % (len(shapes), N))
    if img_infos is not None and len(img_infos) != len(shapes):
        raise _lib.FrcnnError("raw batch: %d img_infos for %d images" % (len(img_infos), len(shapes)))
    hdr = np.zeros((raw_header_layout(N)[1],), dtype=np.uint8)
    v = raw_header_views(hdr, N)
    scales, used = [], 0
    for n, (h0, w0) in enumerate(shapes):
        if h0 < 1 or w0 < 1:
            raise _lib.FrcnnError("raw batch: image %d has no pixels (%d x %d)" % (n, h0, w0))
        im_scale, H, W = plan_size(h0, w0, scale, max_size)
        if not (0 < H <= Hc and 0 < W <= Wc):
            raise _lib.FrcnnError("raw batch: image %d (%d x %d) resizes to %d x %d, which does not fit a %d x %d canvas" %
                                  (n, h0, w0, H, W, Hc, Wc))
        off = ops.round_up(used, RAW_ALIGN)
        used = off + 3 * h0 * w0
        if used > arena_bytes:
            raise _lib.FrcnnError("raw batch: images 0..%d need %d bytes, the arena holds %d" % (n, used, arena_bytes))
        v["extents"][n] = (H, W)
        v["im_info"][n] = (H, W) if img_infos is None else (int(img_infos[n][0]), int(img_infos[n][1]))
        v["src_hw"][n] = (h0, w0)
        v["src_off"][n] = off
        v["inv_scale"][n] = 1.0 / im_scale
        scales.append(im_scale)
    return hdr, scales, used


# ---- raw photos into a training canvas (CanvasRpnTrainer / CanvasRcnnTrainer(raw_input=True)): one block
# [raw header | ground-truth section | pixels].  The raw header is raw_header_layout's, unchanged; the ground-truth section
# carries each slot's float32 im_scale, box count and raw boxes + labels, so photos and boxes travel in one H2D copy.
VOC_MEANS = (103.939, 116.779, 123.68)    # datasets/pascal_voc_dataset.py VOC.mean (BGR)


def voc_gt_layout(N, max_gt):
    """({name: (byte offset inside the section, dtype, shape)}, section bytes, a multiple of 256): "scale" float32 [N],
    "count" int32 [N], "raw_gt" float32 [N, max_gt, 5] (x1, y1, x2, y2 in source-photo coordinates, label)."""
    off_count = ops.round_up(4 * N, 16)
    off_gt = off_count + ops.round_up(4 * N, 16)
    return ({"scale": (0, np.float32, (N,)), "count": (off_count, np.int32, (N,)),
             "raw_gt": (off_gt, np.float32, (N, max_gt, 5))}, ops.round_up(off_gt + 20 * N * max_gt, 256))


def voc_gt_section(boxes, labels, scales, N, max_gt):
    """The uint8 ground-truth section for the photos whose im_scale are `scales`: boxes[n] (G_n, 4) and labels[n] (G_n,)
    with 1 <= G_n <= max_gt.  Raises FrcnnError when a list does not fit."""
    if len(boxes) != len(scales) or len(labels) != len(scales):
        raise _lib.FrcnnError("raw training batch: %d photos, %d box lists and %d label lists" % (len(scales), len(boxes), len(labels)))
    layout, nbytes = voc_gt_layout(N, max_gt)
    sec = np.zeros((nbytes,), dtype=np.uint8)
    v = {name: sec[off:off + int(np.prod(shape)) * 4].view(dt).reshape(shape) for name, (off, dt, shape) in layout.items()}
    for n, (b, l) in enumerate(zip(boxes, labels)):
        b, l = np.asarray(b), np.asarray(l)
        G = b.shape[0] if b.ndim == 2 else -1
        if b.ndim != 2 or b.shape[1] != 4 or l.shape != (G,) or not 1 <= G <= max_gt:
            raise _lib.FrcnnError("raw training batch: photo %d has boxes of shape %s and labels of shape %s, needs (G, 4) and "
                                  "(G,) with 1 <= G <= %d" % (n, b.shape, l.shape, max_gt))
        v["raw_gt"][n, :G, :4] = b
        v["raw_gt"][n, :G, 4] = l
        v["count"][n] = G
        v["scale"][n] = scales[n]
    return sec


# ---- augmentation (CanvasRpnTrainer / CanvasRcnnTrainer(augment=...)): a section after the ground-truth section holds
# each slot's S candidate sizes, from plan_size at every training scale, and its choice (flip, scale index); the first
# launch of the step (frcnn_voc_augment_batch) draws or reads the choice and writes the chosen candidate into the header.
AUG_MAX_SCALES = 8


def voc_aug_layout(N, S):
    """({name: (byte offset inside the section, dtype, shape)}, section bytes, a multiple of 256): "cand_inv" float64 [N, S]
    (1 / im_scale), "cand_hw" int32 [N, S, 2] (the resized H, W), "cand_scale" float32 [N, S] (im_scale), "choice" int32
    [N, 2] (flip, scale index) and "flip" int32 [N] (the flip the step applies)."""
    fields = (("cand_inv", np.float64, (N, S)), ("cand_hw", np.int32, (N, S, 2)), ("cand_scale", np.float32, (N, S)),
              ("choice", np.int32, (N, 2)), ("flip", np.int32, (N,)))
    layout, off = {}, 0
    for name, dt, shape in fields:
        layout[name] = (off, dt, shape)
        off = ops.round_up(off + int(np.prod(shape)) * np.dtype(dt).itemsize, 16)
    return layout, ops.round_up(off, 256)


def voc_aug_views(sec, N, S):
    """numpy views of the augmentation arrays inside `sec`, a uint8 array that starts with the section."""
    layout, _ = voc_aug_layout(N, S)
    return {k: sec[o:o + int(np.prod(sh)) * np.dtype(dt).itemsize].view(dt).reshape(sh) for k, (o, dt, sh) in layout.items()}


def voc_aug_section(shapes, N, Hc, Wc, scales, max_size=1000):
    """The uint8 augmentation section for photos of source sizes `shapes` ((h0, w0) each, at most N) at the training
    `scales` (short-side targets): candidate k of photo n is plan_size(h0, w0, scales[k], max_size); the remaining slots
    and the choice are 0.  Returns (section, [tuple of im_scale per photo]).  Raises FrcnnError when a candidate of a photo
    does not fit the Hc x Wc canvas."""
    S = len(scales)
    sec = np.zeros((voc_aug_layout(N, S)[1],), dtype=np.uint8)
    v = voc_aug_views(sec, N, S)
    out = []
    for n, (h0, w0) in enumerate(shapes):
        cands = []
        for k, s in enumerate(scales):
            im_scale, H, W = plan_size(h0, w0, s, max_size)
            if not (0 < H <= Hc and 0 < W <= Wc):
                raise _lib.FrcnnError("raw batch: image %d (%d x %d) at scale %d resizes to %d x %d, which does not fit a %d x %d "
                                      "canvas" % (n, h0, w0, s, H, W, Hc, Wc))
            v["cand_hw"][n, k] = (H, W)
            v["cand_inv"][n, k] = 1.0 / im_scale
            v["cand_scale"][n, k] = im_scale
            cands.append(im_scale)
        out.append(tuple(cands))
    return sec, out


def voc_scale_boxes(boxes, im_scale):
    """The reference's `bbox *= im_scale` on float32 boxes, as NumPy >= 2 computes it: f32(box) * f32(im_scale), float32."""
    return np.asarray(boxes, dtype=np.float32) * np.float32(im_scale)
