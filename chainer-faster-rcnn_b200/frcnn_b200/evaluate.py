"""PASCAL VOC detection metric on the device: per-class average precision (VOC07 11-point and area) and mAP over a dataset.

A VocEvaluator keeps the dataset's detections in device memory: after each `with_detect` batch or canvas plan has run, `add`
appends the plan's keep lists (frcnn_voc_eval_append_batch) without a download, and `evaluate` uploads the ground truth once,
runs the metric (frcnn_voc_eval) and downloads one small result.  The metric is the devkit's; include/frcnn_b200.h states it.
"""
import numpy as np
import torch

from . import ops
from ._lib import FrcnnError


class VocEvalResult(object):
    """The metric over a dataset.  Per-class arrays are indexed by class - 1 (classes 1 .. num_classes-1): ap07 / ap float64
    (NaN for a class without non-difficult GT), npos / n_det / tp / fp int64.  map07 / map: the means over the classes with
    npos > 0 (NaN if none)."""

    def __init__(self, out, evaluator):
        self.status = int(out[0])
        self.map07, self.map = float(out[1]), float(out[2])
        rows = out[3:].reshape(-1, 6)
        self.npos, self.n_det, self.tp, self.fp = (rows[:, q].astype(np.int64) for q in range(4))
        self.ap07, self.ap = rows[:, 4].copy(), rows[:, 5].copy()
        self._ev, self._epoch = evaluator, evaluator._epoch

    def curve(self, c):
        """(tp_cum, fp_cum) int32 numpy arrays of class c in rank order: one download from the evaluator's workspace, which
        holds them until its next add, evaluate or reset."""
        ev = self._ev
        if ev._epoch != self._epoch:
            raise FrcnnError("VocEvalResult.curve: the evaluator has changed since this result")
        if not 1 <= c < ev.num_classes:
            raise FrcnnError("VocEvalResult.curve: class %r outside 1..%d" % (c, ev.num_classes - 1))
        b, n = int(self.n_det[:c - 1].sum()), int(self.n_det[c - 1])
        return ev._tp_cum[b:b + n].cpu().numpy(), ev._fp_cum[b:b + n].cpu().numpy()


class VocEvaluator(object):
    """Device-side VOC evaluation of up to `max_images` images and `capacity` detections (over all classes), with up to
    `max_gt` ground-truth boxes (default 64 per image).  Images are numbered in the order they are added."""

    def __init__(self, num_classes=21, max_images=5000, capacity=None, max_gt=None, device="cuda"):
        self.num_classes, self.max_images = int(num_classes), int(max_images)
        self.capacity = 1000 * self.max_images if capacity is None else int(capacity)
        self.max_gt = 64 * self.max_images if max_gt is None else int(max_gt)
        self.device = torch.device(device)
        nbytes = ops.voc_eval_workspace_bytes(self.num_classes, self.capacity, self.max_images, self.max_gt)
        self.ws = torch.empty((nbytes,), dtype=torch.uint8, device=self.device)
        cap = self.capacity
        self._tp_cum = self.ws[:4 * cap].view(torch.int32)
        fp_at = (4 * cap + 255) // 256 * 256
        self._fp_cum = self.ws[fp_at:fp_at + 4 * cap].view(torch.int32)
        self.im_scale = torch.empty((self.max_images,), dtype=torch.float64, device=self.device)
        self.out = torch.empty((3 + 6 * (self.num_classes - 1),), dtype=torch.float64, device=self.device)
        self.reset()

    def reset(self):
        """Forget every image added (on the current stream)."""
        self.ws.zero_()
        self.n_images = 0
        self._epoch = getattr(self, "_epoch", 0) + 1

    def _check_room(self, n):
        if self.n_images + n > self.max_images:
            raise FrcnnError("VocEvaluator: %d images added, %d more exceed max_images = %d" % (self.n_images, n, self.max_images))

    def put_scales(self, scales, first=None):
        """Uploads im_scale values of images first, first+1, ... (default: the next images to be added) in one copy."""
        first = self.n_images if first is None else int(first)
        s = torch.from_numpy(np.asarray(scales, dtype=np.float64).reshape(-1))
        if first < 0 or first + s.numel() > self.max_images:
            raise FrcnnError("VocEvaluator: scales of images [%d, %d) exceed max_images = %d" % (first, first + s.numel(),
                                                                                                   self.max_images))
        self.im_scale[first:first + s.numel()].copy_(s, non_blocking=True)

    def _append(self, prob, boxes, keep_idx, conf_count):
        """Appends the next N images; their scales must already be in im_scale."""
        n = int(prob.shape[0])
        self._check_room(n)
        ops.voc_eval_append_batch(prob, boxes, keep_idx, conf_count, self.im_scale[self.n_images:self.n_images + n], self.n_images,
                                  self.capacity, self.max_images, self.ws)
        self.n_images += n
        self._epoch += 1

    def add_arrays(self, prob, boxes, keep_idx, conf_count, im_scale):
        """Appends N images from detect_batch-style device tensors: prob [N,R_cap,NC], boxes [N,R_cap,4NC], keep_idx
        [N,NC-1,R_cap], conf_count [N,NC-1] (strided views allowed), and their N im_scale values (host sequence)."""
        if int(prob.shape[-1]) != self.num_classes:
            raise FrcnnError("VocEvaluator: prob has %d classes, the evaluator %d" % (int(prob.shape[-1]), self.num_classes))
        n = int(prob.shape[0])
        if len(im_scale) != n:
            raise FrcnnError("VocEvaluator: %d images but %d scales" % (n, len(im_scale)))
        self._check_room(n)
        self.put_scales(im_scale)
        self._append(prob, boxes, keep_idx, conf_count)

    def add(self, plan, scales):
        """Appends the occupied slots of a `with_detect` batch or canvas plan after it has run: slot n holds the image of
        scale scales[n] (what forward_raw returns), slots past len(scales) are ignored."""
        if not getattr(plan, "with_detect", False):
            raise FrcnnError("VocEvaluator.add: the plan was built without with_detect")
        n = len(scales)
        if not 1 <= n <= plan.N:
            raise FrcnnError("VocEvaluator.add: %d scales for a plan of %d slots" % (n, plan.N))
        keep_idx, _, conf_count = plan.det
        self.add_arrays(plan.prob[:n], plan.boxes[:n], keep_idx[:n], conf_count[:n], scales)

    def evaluate(self, gt_boxes, gt_labels, gt_difficult=None, iou_thresh=0.5):
        """The metric over every image added, against per-image GT: gt_boxes[i] float [k_i,4] (x1,y1,x2,y2 in source-photo
        coordinates), gt_labels[i] int [k_i] in 1..num_classes-1, gt_difficult[i] bool [k_i] (default all False).  One upload, the
        launches, one download.  Raises FrcnnError on malformed GT, a GT image count other than the number of images
        added, or more detections than `capacity`."""
        if not np.isfinite(iou_thresh):
            raise FrcnnError("VocEvaluator.evaluate: iou_thresh must be finite (got %r)" % (iou_thresh,))
        blob, G, (o_box, o_lab, o_dif) = pack_gt(gt_boxes, gt_labels, gt_difficult, self.n_images, self.num_classes, self.max_gt)
        dev = torch.from_numpy(blob).to(self.device, non_blocking=True)
        n, g = self.n_images, max(G, 1)           # the blob has room for one row past an empty GT
        ops.voc_eval(self.num_classes, self.capacity, self.max_images, self.max_gt, dev[:4 * (n + 1)].view(torch.int32),
                     dev[o_box:o_box + 16 * g].view(torch.float32).view(g, 4), dev[o_lab:o_lab + 4 * g].view(torch.int32),
                     dev[o_dif:o_dif + g], iou_thresh, self.ws, out=self.out, n_gt=G)
        self._epoch += 1
        res = VocEvalResult(self.out.cpu().numpy(), self)
        if res.status != 0:
            raise FrcnnError("VocEvaluator.evaluate: more than capacity = %d detections were added" % self.capacity)
        return res


def pack_gt(gt_boxes, gt_labels, gt_difficult, n, num_classes, max_gt):
    """Validates the per-image GT lists of n images and packs them into one host blob: offsets int32 [n+1] | boxes float32
    [G,4] | labels int32 [G] | difficult uint8 [G] (each 16-byte aligned, with room for one row when G = 0).  Returns
    (blob, G, byte offsets)."""
    if len(gt_boxes) != n or len(gt_labels) != n or (gt_difficult is not None and len(gt_difficult) != n):
        raise FrcnnError("VocEvaluator.evaluate: ground truth for %d / %d / %s images, %d were added" % (
            len(gt_boxes), len(gt_labels), "-" if gt_difficult is None else len(gt_difficult), n))
    boxes, labels, diff, counts = [], [], [], np.zeros(n + 1, dtype=np.int64)
    for i in range(n):
        b = np.asarray(gt_boxes[i], dtype=np.float32)
        lab = np.asarray(gt_labels[i])
        if b.size == 0 and lab.size == 0:
            b, lab = b.reshape(0, 4), lab.reshape(0)
        if b.ndim != 2 or b.shape[1] != 4 or lab.shape != (b.shape[0],):
            raise FrcnnError("VocEvaluator.evaluate: image %d needs boxes [k,4] and labels [k] (got %s and %s)" % (
                i, b.shape, lab.shape))
        if lab.size and (not np.issubdtype(lab.dtype, np.integer) or lab.min() < 1 or lab.max() >= num_classes):
            raise FrcnnError("VocEvaluator.evaluate: image %d has labels outside 1..%d" % (i, num_classes - 1))
        d = np.zeros(b.shape[0], dtype=bool) if gt_difficult is None else np.asarray(gt_difficult[i]).reshape(-1)
        if d.shape != (b.shape[0],):
            raise FrcnnError("VocEvaluator.evaluate: image %d has %d difficult flags for %d boxes" % (i, d.size, b.shape[0]))
        boxes.append(b)
        labels.append(lab.astype(np.int32))
        diff.append(d.astype(np.uint8))
        counts[i + 1] = b.shape[0]
    offsets = np.cumsum(counts)
    G = int(offsets[-1])
    if G > max_gt:
        raise FrcnnError("VocEvaluator.evaluate: %d GT boxes exceed max_gt = %d" % (G, max_gt))
    a16 = lambda v: (v + 15) // 16 * 16        # noqa: E731
    o_box = a16(4 * (n + 1))
    g = max(G, 1)
    o_lab = a16(o_box + 16 * g)
    o_dif = a16(o_lab + 4 * g)
    blob = np.zeros(a16(o_dif + g), dtype=np.uint8)
    blob[:4 * (n + 1)] = offsets.astype(np.int32).view(np.uint8)
    if G:
        blob[o_box:o_box + 16 * G] = np.concatenate(boxes).view(np.uint8).reshape(-1)
        blob[o_lab:o_lab + 4 * G] = np.concatenate(labels).view(np.uint8)
        blob[o_dif:o_dif + G] = np.concatenate(diff)
    return blob, G, (o_box, o_lab, o_dif)
