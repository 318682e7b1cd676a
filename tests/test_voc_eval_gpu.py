"""GPU tests of the device VOC evaluator (voc_eval.cu through ops.voc_eval_append_batch / ops.voc_eval, evaluate.VocEvaluator
and Engine.evaluate_images) against the NumPy oracle tests/voc_eval_ref.py: every count, every tp_cum / fp_cum curve and
every 11-point AP bit for bit, the area AP within 1e-12, on fabricated keep lists with tied, signed-zero and NaN scores,
NaN boxes, IoUs exactly at the threshold, difficult GT, empty slots and images without GT, split over several batches; on a
VOC07-test-sized set of more than a million detections; at the capacity limit; and end to end from raw photos on VGG16 and
ResNet-50 with random weights."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import voc_eval_ref as ref
from test_batch_gpu import ANCHORS

pytestmark = pytest.mark.gpu
f32 = np.float32
TIES = np.array([0.5, 0.25, -0.0, 0.0, 0.75], f32)
SCALES = np.array([1.0, 2.0, 1.6, 0.75, 1.2], np.float64)


def fabricate(seed, n_images, R, NC, mean_dets):
    """Keep lists of n_images images as frcnn_detect_batch leaves them, but in arbitrary order: prob [M,R,NC], boxes [M,R,4NC]
    (scaled by im_scale), keep_idx [M,NC-1,R] (random permutations, a few entries outside [0,R)), conf_count [M,NC-1]
    (some negative, some past R); and integer GT (0-4 boxes per image, labels 1..NC-1, 20% difficult).  Half the boxes are
    jittered GT boxes, 5% of those exactly IoU 0.5 to their GT (on exactly representable scales); scores have ties, -0.0 /
    +0.0 and NaN; boxes a few NaN."""
    rng = np.random.default_rng(seed)
    M = n_images
    k = rng.integers(0, 5, M)
    k[rng.random(M) < 0.2] = 0
    gt_pad = np.zeros((M, 4, 4), np.int32)
    x1, y1 = rng.integers(0, 400, (M, 4)), rng.integers(0, 300, (M, 4))
    gt_pad[..., 0], gt_pad[..., 1] = x1, y1
    gt_pad[..., 2], gt_pad[..., 3] = x1 + rng.integers(8, 150, (M, 4)), y1 + rng.integers(8, 150, (M, 4))
    lab_pad = rng.integers(1, NC, (M, 4))
    dif_pad = rng.random((M, 4)) < 0.2
    gt_boxes = [gt_pad[n, :k[n]].astype(f32) for n in range(M)]
    gt_labels = [lab_pad[n, :k[n]] for n in range(M)]
    gt_diff = [dif_pad[n, :k[n]] for n in range(M)]
    scale = SCALES[rng.integers(0, len(SCALES), M)]
    prob = rng.random((M, R, NC)).astype(f32)
    tie = rng.random(prob.shape) < 0.15
    prob[tie] = TIES[rng.integers(0, len(TIES), int(tie.sum()))]
    prob[rng.random(prob.shape) < 0.005] = np.nan
    bx = np.empty((M, R, NC, 4), f32)
    rx, ry = rng.integers(0, 450, (M, R, NC)), rng.integers(0, 350, (M, R, NC))
    bx[..., 0], bx[..., 1] = rx, ry
    bx[..., 2], bx[..., 3] = rx + rng.integers(4, 160, (M, R, NC)), ry + rng.integers(4, 160, (M, R, NC))
    g = gt_pad[np.arange(M)[:, None, None], rng.integers(0, np.maximum(k, 1)[:, None, None], (M, R, NC))]
    src = (rng.random((M, R, NC)) < 0.5) & (k > 0)[:, None, None]
    jit = g + rng.integers(-3, 4, g.shape) * (rng.random((M, R, NC)) < 0.7)[..., None]
    exact = g.copy()
    exact[..., 2] = g[..., 0] + 2 * (g[..., 2] - g[..., 0] + 1) - 1
    use_exact = src & (rng.random((M, R, NC)) < 0.05) & np.isin(scale, (1.0, 2.0))[:, None, None]
    bx[src] = jit[src]
    bx[use_exact] = exact[use_exact]
    bx = (bx * scale.astype(f32)[:, None, None, None]).astype(f32)
    bx[rng.random(bx.shape) < 0.001] = np.nan
    boxes = bx.reshape(M, R, 4 * NC)
    keep = rng.permuted(np.tile(np.arange(R, dtype=np.int32), (M, NC - 1, 1)), axis=2)
    bad = rng.random(keep.shape) < 0.002
    keep[bad] = rng.choice(np.array([-1, R, R + 7], np.int32), int(bad.sum()))
    conf = np.minimum(rng.poisson(mean_dets / (NC - 1), (M, NC - 1)), R).astype(np.int32)
    conf[rng.random(conf.shape) < 0.05] = 0
    conf[rng.random(conf.shape) < 0.01] = -3
    conf[rng.random(conf.shape) < 0.01] = R + 5
    return dict(prob=prob, boxes=boxes, keep=keep, conf=conf, scale=scale, gt=(gt_boxes, gt_labels, gt_diff))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def add_batches(ev, data, splits):
    """VocEvaluator.add_arrays over consecutive batches of the sizes in splits"""
    s = 0
    for n in splits:
        sl = slice(s, s + n)
        ev.add_arrays(_cuda(data["prob"][sl]), _cuda(data["boxes"][sl]), _cuda(data["keep"][sl]), _cuda(data["conf"][sl]),
                      data["scale"][sl].tolist())
        s += n
    assert s == len(data["scale"])


def oracle(data, NC, iou_thresh=0.5):
    d = ref.detections_from_lists(data["prob"], data["boxes"], data["keep"], data["conf"], data["scale"])
    return ref.voc_eval(d, *data["gt"], NC, iou_thresh=iou_thresh)


def _same_float(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def assert_matches(res, want, NC, curves=True):
    for f in ("npos", "n_det", "tp", "fp"):
        assert np.array_equal(getattr(res, f), want[f]), (f, getattr(res, f), want[f])
    assert _same_float(res.ap07, want["ap07"]), (res.ap07, want["ap07"])
    assert np.array_equal(np.isnan(res.ap), np.isnan(want["ap"]))
    ok = ~np.isnan(want["ap"])
    assert np.all(np.abs(res.ap[ok] - want["ap"][ok]) <= 1e-12), np.abs(res.ap[ok] - want["ap"][ok]).max()
    assert _same_float(res.map07, want["map07"]) and (np.isnan(want["map"]) or abs(res.map - want["map"]) <= 1e-12)
    if curves:
        for c in range(1, NC):
            tp, fp = res.curve(c)
            assert np.array_equal(tp, want["tp_cum"][c - 1]) and np.array_equal(fp, want["fp_cum"][c - 1]), c


def _evaluator(NC, M, capacity=None, max_gt=None):
    from frcnn_b200.evaluate import VocEvaluator
    return VocEvaluator(NC, max_images=M, capacity=capacity, max_gt=max_gt)


@pytest.mark.parametrize("NC,R,M,mean,splits", [(4, 40, 24, 30, (5, 1, 8, 10)), (21, 300, 16, 150, (4, 4, 4, 4)),
                                                (2, 64, 9, 20, (9,))])
def test_fabricated_lists_equal_oracle(NC, R, M, mean, splits):
    """Ties within and across images, -0.0 / +0.0, NaN scores and boxes, IoU exactly 0.5, difficult GT, empty slots, images
    without GT and classes without GT or detections, several add calls: the device result equals the oracle; a second
    evaluation and another split of the same images give bitwise the same result."""
    data = fabricate(100 + NC + M, M, R, NC, mean)
    want = oracle(data, NC)
    assert want["tp"].sum() > 0 and want["fp"].sum() > 0 and want["n_det"].sum() > 0
    ev = _evaluator(NC, M + 3)
    add_batches(ev, data, splits)
    res = ev.evaluate(*data["gt"])
    assert_matches(res, want, NC)
    again = ev.evaluate(*data["gt"])
    assert _same_float(np.r_[again.ap07, again.ap, again.map07, again.map], np.r_[res.ap07, res.ap, res.map07, res.map])
    ev.reset()
    add_batches(ev, data, (M,))
    other = ev.evaluate(*data["gt"])
    assert _same_float(np.r_[other.ap07, other.ap, other.map07, other.map], np.r_[res.ap07, res.ap, res.map07, res.map])
    # the strict threshold: one double below 0.5 the exact-0.5 overlaps become matches
    below = float(np.nextafter(0.5, 0.0))
    assert_matches(ev.evaluate(*data["gt"], iou_thresh=below), oracle(data, NC, below), NC, curves=False)


def test_ops_entries_directly():
    """ops.voc_eval_append_batch / ops.voc_eval on raw tensors: the result vector's layout (status, mAP07, mAP, then six
    values per class) and an empty dataset (every class NaN or 0)."""
    from frcnn_b200 import ops
    NC, R, M = 3, 16, 4
    data = fabricate(7, M, R, NC, 10)
    nb = ops.voc_eval_workspace_bytes(NC, 1000, M, 64)
    ws = torch.zeros((nb,), dtype=torch.uint8, device="cuda")
    ops.voc_eval_append_batch(_cuda(data["prob"]), _cuda(data["boxes"]), _cuda(data["keep"]), _cuda(data["conf"]),
                              _cuda(data["scale"]), 0, 1000, M, ws)
    from frcnn_b200.evaluate import pack_gt
    blob, G, (ob, ol, od) = pack_gt(*data["gt"], M, NC, 64)
    b = _cuda(blob)
    out = ops.voc_eval(NC, 1000, M, 64, b[:4 * (M + 1)].view(torch.int32), b[ob:ob + 16 * G].view(torch.float32).view(G, 4),
                       b[ol:ol + 4 * G].view(torch.int32), b[od:od + G], 0.5, ws).cpu().numpy()
    want = oracle(data, NC)
    assert out[0] == 0 and _same_float(out[1], want["map07"])
    rows = out[3:].reshape(NC - 1, 6)
    assert np.array_equal(rows[:, 0], want["npos"]) and np.array_equal(rows[:, 1], want["n_det"])
    assert _same_float(rows[:, 4], want["ap07"])
    ev = _evaluator(NC, M)
    ev.add_arrays(_cuda(data["prob"][:1]), _cuda(data["boxes"][:1]), _cuda(np.zeros_like(data["keep"][:1])),
                  _cuda(np.zeros_like(data["conf"][:1])), [1.0])
    empty = ev.evaluate([np.zeros((0, 4))], [np.zeros(0, np.int64)])
    assert np.all(empty.n_det == 0) and np.all(np.isnan(empty.ap)) and np.isnan(empty.map07)


def test_voc07_sized_set():
    """4,952 images, 20 classes, more than a million detections: the sort, the scans and the reductions across many CTAs."""
    NC, R, M = 21, 150, 4952
    data = fabricate(2007, M, R, NC, 240)
    want = oracle(data, NC)
    assert want["n_det"].sum() > 1_000_000
    ev = _evaluator(NC, M, capacity=int(want["n_det"].sum()) + 1000)
    add_batches(ev, data, [64] * (M // 64) + [M % 64])
    assert_matches(ev.evaluate(*data["gt"]), want, NC)


def test_capacity_limit():
    """Exactly `capacity` detections evaluate normally; one more makes evaluate raise."""
    from frcnn_b200 import FrcnnError
    NC, R, M = 5, 32, 6
    data = fabricate(11, M, R, NC, 20)
    want = oracle(data, NC)
    D = int(want["n_det"].sum())
    ev = _evaluator(NC, M, capacity=D)
    add_batches(ev, data, (3, 3))
    assert_matches(ev.evaluate(*data["gt"]), want, NC)
    ev = _evaluator(NC, M, capacity=D - 1)
    add_batches(ev, data, (3, 3))
    with pytest.raises(FrcnnError, match="capacity"):
        ev.evaluate(*data["gt"])
    with pytest.raises(FrcnnError, match="were added"):
        ev.evaluate(*(g[:-1] for g in data["gt"]))


# ------------------------------------------------------------------------------------------------------ end to end
VOC_SHAPES = [(375, 500), (500, 375), (333, 500), (500, 334), (281, 500), (375, 500)]


def _photos(seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in VOC_SHAPES]


def _gt_from_first_pass(dets_per_image, seed):
    """GT from jittered copies of each image's top detections (so TP, FP, duplicate and difficult paths occur), plus a
    random box; the last image gets none."""
    rng = np.random.default_rng(seed)
    boxes, labels, diff = [], [], []
    for i, dets in enumerate(dets_per_image):
        top = sorted(dets, key=lambda d: -d[5])[:6] if i < len(dets_per_image) - 1 else []
        b = [np.array(d[1:5], np.float64) + rng.uniform(-3, 3, 4) for d in top] + ([[10, 10, 120, 90]] if top else [])
        lab = [d[0] for d in top] + ([int(rng.integers(1, 21))] if top else [])
        boxes.append(np.array(b, f32).reshape(-1, 4))
        labels.append(np.array(lab, np.int64))
        diff.append(rng.random(len(lab)) < 0.25)
    return boxes, labels, diff


def _end_to_end(eng):
    from frcnn_b200 import preprocess
    photos = _photos(5)
    first = eng.detect_images(photos, N=4, conf=0.05)
    assert sum(len(d) for d in first) > 0
    gt = _gt_from_first_pass(first, 6)
    res = eng.evaluate_images(photos, *gt, N=4, conf=0.05)
    # the oracle on the same plan's keep lists, divided by the same scales
    p = eng.raw_canvas_plan(photos, 4, None, 0.3, 0.05)
    NC, post = eng.weights.num_classes, p.post_n
    dets = []
    for s in range(0, len(photos), 4):
        chunk = photos[s:s + 4]
        scales = p.forward_raw(chunk)[3]
        blocks = p.fetch_result()
        for n in range(len(chunk)):
            r = blocks[n]
            prob = np.zeros((1, post, NC), f32)
            boxes = np.zeros((1, post, 4 * NC), f32)
            prob[0, :r["count"]], boxes[0, :r["count"]] = r["prob"], r["boxes"]
            d = ref.detections_from_lists(prob, boxes, r["keep_idx"][None], r["conf_count"][None], [scales[n]], s + n)
            lists = preprocess.result_detections(r, scales[n])
            assert [(int(c), *np.trunc(b).astype(np.int64).tolist()) for c, b in zip(d["cls"], d["box"])] == \
                [t[:5] for t in lists]
            assert d["score"].tolist() == [t[5] for t in lists]
            dets.append(d)
    want = ref.voc_eval(ref.concat(dets), *gt, NC)
    assert want["tp"].sum() > 0 and want["fp"].sum() > 0
    assert_matches(res, want, NC, curves=False)


def test_engine_evaluate_images_vgg16():
    from frcnn_b200.engine import Engine
    _end_to_end(Engine(orc.make_params(seed=1234), precision="bf16x3", anchors=ANCHORS, with_detect=True))


def test_engine_evaluate_images_resnet50():
    from frcnn_b200.resnet_engine import ResNetPhotoEngine
    _end_to_end(ResNetPhotoEngine(orc.make_resnet_params(50, seed=21), 50, precision="bf16x3", anchors=ANCHORS, with_detect=True))
