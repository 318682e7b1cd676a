"""Float64 NumPy restatement of the PASCAL VOC detection metric as include/frcnn_b200.h (frcnn_voc_eval) states it: the oracle
of the device evaluator.  Written from the definition: the rank order is a np.lexsort on (score key, image, keep-list
position) with the project's score order (-0.0 == +0.0, NaN after every number), matching and the curve are plain loops,
and the area AP is summed left to right."""
import numpy as np

f32 = np.float32
EPS = np.finfo(np.float64).eps


def score_key(scores):
    """uint32 keys, larger = earlier in the score order: -0.0 and +0.0 share a key, every NaN gets key 1 (below -inf)."""
    s = np.ascontiguousarray(scores, dtype=f32)
    b = s.view(np.uint32).copy()
    b[b == 0x80000000] = 0
    key = np.where(b & 0x80000000, ~b, b | 0x80000000).astype(np.uint32)
    key[np.isnan(s)] = 1
    return key


def detections_from_lists(prob, boxes, keep_idx, conf_count, im_scale, image_base=0):
    """The detections a batch contributes: for image n, class c = 1..NC-1, the first conf_count[n][c-1] entries r of
    keep_idx[n][c-1] (clamped to [0, R_cap]); score prob[n][r][c], box boxes[n][r][4c:4c+4] / float32(im_scale[n]) in float32
    (an r outside [0, R_cap): a zero box of score 0).  Returns dict of arrays cls, img, pos, score (f32), box (f32 [D,4])."""
    N, R_cap, NC = prob.shape
    cls, img, pos, score, box = [], [], [], [], []
    for n in range(N):
        s = f32(im_scale[n])
        for c in range(1, NC):
            k = min(max(int(conf_count[n][c - 1]), 0), R_cap)
            for j in range(k):
                r = int(keep_idx[n][c - 1][j])
                cls.append(c)
                img.append(image_base + n)
                pos.append(j)
                if 0 <= r < R_cap:
                    score.append(prob[n, r, c])
                    box.append(boxes[n, r, 4 * c:4 * c + 4] / s)
                else:
                    score.append(f32(0))
                    box.append(np.zeros(4, dtype=f32))
    return dict(cls=np.array(cls, dtype=np.int64), img=np.array(img, dtype=np.int64), pos=np.array(pos, dtype=np.int64),
                score=np.array(score, dtype=f32).reshape(-1), box=np.array(box, dtype=f32).reshape(-1, 4))


def concat(dets_list):
    return {k: np.concatenate([d[k] for d in dets_list]) for k in ("cls", "img", "pos", "score", "box")}


def overlaps(bb, gt):
    """The devkit's overlaps of one detection box bb (float64 [4]) with GT boxes gt (float64 [k,4])."""
    ixmin = np.maximum(gt[:, 0], bb[0])
    iymin = np.maximum(gt[:, 1], bb[1])
    ixmax = np.minimum(gt[:, 2], bb[2])
    iymax = np.minimum(gt[:, 3], bb[3])
    iw = np.maximum(ixmax - ixmin + 1., 0.)
    ih = np.maximum(iymax - iymin + 1., 0.)
    inters = iw * ih
    uni = ((bb[2] - bb[0] + 1.) * (bb[3] - bb[1] + 1.) + (gt[:, 2] - gt[:, 0] + 1.) * (gt[:, 3] - gt[:, 1] + 1.) - inters)
    with np.errstate(divide="ignore", invalid="ignore"):
        return inters / uni


def ap07(rec, prec):
    ap = 0.0
    for k in range(11):
        t = k * 0.1
        sel = prec[rec >= t]
        p = np.max(sel) if sel.size else 0.0
        ap = ap + p / 11.0
    return ap


def ap_area(rec, prec):
    mrec = np.concatenate(([0.], rec, [1.]))
    mpre = np.concatenate(([0.], prec, [0.]))
    for i in range(mpre.size - 1, 0, -1):
        mpre[i - 1] = np.maximum(mpre[i - 1], mpre[i])
    ap = 0.0
    for i in np.where(mrec[1:] != mrec[:-1])[0]:
        ap = ap + (mrec[i + 1] - mrec[i]) * mpre[i + 1]
    return ap


def voc_eval(dets, gt_boxes, gt_labels, gt_difficult, num_classes, iou_thresh=0.5):
    """dets: detections_from_lists' dict (over the whole set); gt_*: per-image lists.  Returns dict with per-class arrays
    (index class-1) npos, n_det, tp, fp, ap07, ap, the per-class curves tp_cum / fp_cum (int32) and map07 / map."""
    n_images = len(gt_boxes)
    gtb = [np.asarray(b, dtype=f32).reshape(-1, 4).astype(np.float64) for b in gt_boxes]
    gtl = [np.asarray(lab, dtype=np.int64).reshape(-1) for lab in gt_labels]
    gtd = [np.zeros(len(lab), dtype=bool) if gt_difficult is None else np.asarray(d, dtype=bool).reshape(-1)
           for lab, d in zip(gtl, gt_difficult if gt_difficult is not None else gtl)]
    K = num_classes - 1
    res = dict(npos=np.zeros(K, np.int64), n_det=np.zeros(K, np.int64), tp=np.zeros(K, np.int64), fp=np.zeros(K, np.int64),
               ap07=np.full(K, np.nan), ap=np.full(K, np.nan), tp_cum=[], fp_cum=[])
    keys = score_key(dets["score"])
    for c in range(1, num_classes):
        sel = np.nonzero(dets["cls"] == c)[0]
        order = sel[np.lexsort((dets["pos"][sel], dets["img"][sel], np.uint32(0xFFFFFFFF) - keys[sel]))]
        npos = sum(int(np.sum((lab == c) & ~d)) for lab, d in zip(gtl, gtd))
        claimed = [np.zeros(int(np.sum(lab == c)), dtype=bool) for lab in gtl]
        nd = order.size
        tp, fp = np.zeros(nd), np.zeros(nd)
        for d, e in enumerate(order):
            n = int(dets["img"][e])
            m = gtl[n] == c if n < n_images else None
            if m is None or not m.any():
                fp[d] = 1.
                continue
            ov = overlaps(dets["box"][e].astype(np.float64), gtb[n][m])
            ovmax = np.max(ov)
            jmax = int(np.argmax(ov))
            if ovmax > iou_thresh:
                if not gtd[n][m][jmax]:
                    if not claimed[n][jmax]:
                        tp[d] = 1.
                        claimed[n][jmax] = True
                    else:
                        fp[d] = 1.
            else:
                fp[d] = 1.
        fp, tp = np.cumsum(fp), np.cumsum(tp)
        res["tp_cum"].append(tp.astype(np.int32))
        res["fp_cum"].append(fp.astype(np.int32))
        k = c - 1
        res["npos"][k], res["n_det"][k] = npos, nd
        res["tp"][k], res["fp"][k] = (int(tp[-1]), int(fp[-1])) if nd else (0, 0)
        if npos > 0:
            rec = tp / float(npos)
            prec = tp / np.maximum(tp + fp, EPS)
            res["ap07"][k], res["ap"][k] = ap07(rec, prec), ap_area(rec, prec)
    valid = res["npos"] > 0
    m = int(valid.sum())
    s07 = s = 0.0
    for k in np.nonzero(valid)[0]:
        s07, s = s07 + res["ap07"][k], s + res["ap"][k]
    res["map07"], res["map"] = (s07 / m, s / m) if m else (np.nan, np.nan)
    return res
