"""CPU tests of the VOC metric's oracle (tests/voc_eval_ref.py) on cases worked out by hand: both AP variants, the strict IoU
threshold, difficult GT, duplicates, classes without GT or without detections, the rank order's tie rules, and the 11 recall
thresholds."""
import numpy as np
import pytest

import voc_eval_ref as ref

A, B = (0, 0, 9, 9), (20, 20, 29, 29)          # two 10 x 10 GT boxes (+1 convention)


def _dets(rows):
    """rows: (cls, img, pos, score, box) -> the oracle's detection dict"""
    cls, img, pos, score, box = zip(*rows)
    return dict(cls=np.array(cls, np.int64), img=np.array(img, np.int64), pos=np.array(pos, np.int64),
                score=np.array(score, np.float32), box=np.array(box, np.float32).reshape(-1, 4))


def test_two_gt_three_detections_by_hand():
    """TP, FP, TP: tp_cum [1,1,2], fp_cum [0,1,1]; rec [.5,.5,1], prec [1,.5,2/3].  11-point: t <= 0.5 sees precision 1, t >= 0.6
    only the last point (2/3): (6 + 5 * 2/3) / 11 = 28/33.  Area: 0.5 * 1 + 0.5 * 2/3 = 5/6."""
    d = _dets([(1, 0, 0, 0.9, A), (1, 0, 1, 0.8, (50, 50, 59, 59)), (1, 0, 2, 0.7, B)])
    r = ref.voc_eval(d, [[A, B]], [[1, 1]], None, 2)
    assert r["tp_cum"][0].tolist() == [1, 1, 2] and r["fp_cum"][0].tolist() == [0, 1, 1]
    assert (r["npos"][0], r["n_det"][0], r["tp"][0], r["fp"][0]) == (2, 3, 2, 1)
    assert r["ap07"][0] == pytest.approx(28 / 33, abs=1e-15) and r["ap"][0] == pytest.approx(5 / 6, abs=1e-15)
    assert r["map07"] == r["ap07"][0] and r["map"] == r["ap"][0]


def test_iou_exactly_at_threshold_is_not_a_match():
    """(0,0,19,9) against (0,0,9,9): intersection 100, union 200, IoU exactly 0.5 in float64 -- not above 0.5, so an FP; with
    the threshold one double below 0.5 the same IoU is above it and the detection is a TP."""
    box = (0, 0, 19, 9)
    assert ref.overlaps(np.array(box, np.float64), np.array([A], np.float64))[0] == 0.5
    d = _dets([(1, 0, 0, 0.9, box)])
    at = ref.voc_eval(d, [[A]], [[1]], None, 2, iou_thresh=0.5)
    below = ref.voc_eval(d, [[A]], [[1]], None, 2, iou_thresh=np.nextafter(0.5, 0.0))
    assert (at["tp"][0], at["fp"][0], at["ap"][0]) == (0, 1, 0.0)
    assert (below["tp"][0], below["fp"][0], below["ap"][0]) == (1, 0, 1.0)


def test_difficult_best_overlap_ignores_the_detection():
    """GT 0 difficult and the best overlap (IoU 1), GT 1 non-difficult and unclaimed (IoU 0.81 > 0.5): the detection takes
    the first maximum, the difficult box, and is neither TP nor FP; GT 1 stays unclaimed for the next detection."""
    g1 = (1, 0, 9, 9)
    d = _dets([(1, 0, 0, 0.9, A), (1, 0, 1, 0.8, g1)])
    r = ref.voc_eval(d, [[A, g1]], [[1, 1]], [[True, False]], 2)
    assert r["npos"][0] == 1 and r["tp_cum"][0].tolist() == [0, 1] and r["fp_cum"][0].tolist() == [0, 0]
    eleven = 0.0
    for _ in range(11):
        eleven = eleven + 1.0 / 11.0          # left to right: 1 + 2**-52
    assert r["ap07"][0] == eleven and r["ap"][0] == 1.0


def test_duplicates_and_rank_ties():
    """Two identical detections of one GT: the first in rank order is the TP, the duplicate an FP.  Equal scores rank by
    image, then by keep-list position, and -0.0 ties +0.0 -- whatever order the detections are stored in."""
    rows = [(1, 1, 0, 0.5, B), (1, 0, 1, 0.5, A), (1, 0, 0, 0.5, A), (1, 1, 1, -0.0, B), (1, 1, 2, 0.0, B), (1, 1, 3, np.nan, B)]
    r = ref.voc_eval(_dets(rows), [[A], [B]], [[1], [1]], None, 2)
    # rank: (img0,pos0) TP, (img0,pos1) FP dup, (img1,pos0) TP, (img1,pos1) FP, (img1,pos2) FP, NaN last FP
    assert r["tp_cum"][0].tolist() == [1, 1, 2, 2, 2, 2] and r["fp_cum"][0].tolist() == [0, 1, 1, 2, 3, 4]
    r2 = ref.voc_eval(_dets(rows[::-1]), [[A], [B]], [[1], [1]], None, 2)
    assert r2["tp_cum"][0].tolist() == r["tp_cum"][0].tolist() and r2["ap"][0] == r["ap"][0]


def test_classes_without_gt_or_without_detections():
    """Class 1: GT, no detection -> AP 0.  Class 2: detections, no GT -> AP NaN, all FP, left out of the mean.  Class 3:
    neither -> NaN.  mAP = class 1's 0."""
    d = _dets([(2, 0, 0, 0.9, A)])
    r = ref.voc_eval(d, [[A]], [[1]], None, 4)
    assert (r["ap07"][0], r["ap"][0]) == (0.0, 0.0) and r["n_det"][0] == 0
    assert np.isnan(r["ap07"][1]) and np.isnan(r["ap"][1]) and (r["fp"][1], r["npos"][1]) == (1, 0)
    assert np.isnan(r["ap"][2]) and r["map07"] == 0.0 and r["map"] == 0.0
    none = ref.voc_eval(d, [[]], [[]], None, 4)
    assert np.isnan(none["map07"]) and np.isnan(none["map"])


def test_nan_overlap_is_a_false_positive():
    d = _dets([(1, 0, 0, 0.9, (0, np.nan, 9, 9))])
    r = ref.voc_eval(d, [[A]], [[1]], None, 2)
    assert (r["tp"][0], r["fp"][0]) == (0, 1)


def test_eleven_point_thresholds_are_arange():
    """t = k * 0.1 in float64 is exactly np.arange(0., 1.1, 0.1)[k] (the devkit's loop), for all 11 points."""
    ts = np.arange(0., 1.1, 0.1)
    assert ts.size == 11 and all(k * 0.1 == ts[k] for k in range(11))


def test_score_key_order():
    s = np.array([1.0, -0.0, 0.0, np.nan, -np.inf, np.inf, -1.0], np.float32)
    k = ref.score_key(s)
    assert k[1] == k[2] and k[3] == 1 and k[3] < k[4] < k[6] < k[1] < k[0] < k[5]
