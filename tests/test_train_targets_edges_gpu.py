"""Edge cases of the kernels that turn ground truth into training targets and losses (rpn_train.cu; the target, helper
and loss kernels of rcnn_train.cu), each against an exact reference.

References:
* labels, IoUs and indices: the oracle (orc.bbox_overlaps restates bbox.pyx, orc.anchor_target_layer and
  orc.proposal_target_layer the two target layers); `_targets_ref` restates anchor_target_layer.py:131-168 for other
  thresholds, batch and num_fg and is pinned to the oracle at the reference's own values;
* device subsampling (mode 1): the counter hash restated in NumPy uint64 and handed to the oracle as `choice=`;
* losses and gradients: float64 restatements below, pinned once to torch float64 cross_entropy / huber_loss.

Bars: labels, indices, counts and IoUs bit-exact; anchor regression targets within 1 float32 ulp (float64 arithmetic,
CUDA's log against NumPy's); proposal targets within 2 ulp (float32 logf) with inf / NaN at the same places; every loss,
accuracy and gradient within 1 float32 ulp of the float64 reference, plus, on the extreme-logit sets only, the absolute
allowance derived at `_allowances`.  The worst ulp of each bar is printed ("BAR ...")."""
import math

import numpy as np
import pytest
import torch

import frcnn_oracle as orc

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
# 15 anchors.  0-6 share a height of 20 and are nested in anchor 0 (40 wide), so a gt box equal to anchor 0 overlaps
# 1-6 at IoU w/40 exactly: 28 -> 0.7, 29 -> 0.725, 27 -> 0.675, 12 -> 0.3, 13 -> 0.325, 11 -> 0.275.
ANCHORS15 = np.array([[-20, -10, 19, 9], [-14, -10, 13, 9], [-14, -10, 14, 9], [-13, -10, 13, 9], [-6, -10, 5, 9],
                      [-6, -10, 6, 9], [-5, -10, 5, 9], [-32, -32, 31, 31], [-64, -64, 63, 63], [-16, -48, 15, 47],
                      [-48, -16, 47, 15], [-90, -45, 89, 44], [-8, -8, 7, 7], [-100, -100, 99, 99], [-24, -24, 24, 24]], f64)
ANCHORS4 = ANCHORS[[0, 3, 4, 6]]
BG_SEED_XOR = 0xA5A5A5A5DEADBEEF
EPS = 2.0 ** -52


@pytest.fixture(scope="module")
def tops():
    from frcnn_b200 import train_ops
    return train_ops


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ulp(got, want):
    """float32 ulp distance; inf must meet the same inf and NaN a NaN (distance 0 there, asserted)."""
    g = np.ascontiguousarray(got, f32)
    w = np.ascontiguousarray(want, f32)
    assert g.shape == w.shape
    assert np.array_equal(np.isnan(g), np.isnan(w)), "NaN positions differ"
    fin = np.isfinite(w)
    assert np.array_equal(g[~fin & ~np.isnan(w)], w[~fin & ~np.isnan(w)]), "inf positions differ"
    assert np.isfinite(g[fin]).all(), "finite reference, non-finite result"

    def key(a):
        i = a.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    d = np.zeros(g.shape, np.int64)
    d[fin] = np.abs(key(g[fin]) - key(w[fin]))
    return d


def _close(what, got, want64, allow=0.0):
    """got (float32) within 1 ulp of float32(want64), or within `allow` of want64 in absolute terms."""
    got = np.asarray(got, f32)
    want64 = np.asarray(want64, f64)
    with np.errstate(over="ignore"):
        u = _ulp(got, want64.astype(f32))
    with np.errstate(invalid="ignore"):
        in_allow = np.abs(got.astype(f64) - want64) <= allow
    ok = (u <= 1) | in_allow
    print("BAR %s: max ulp %d, %d beyond 1 ulp inside the allowance %s" % (what, u.max(initial=0), int(((u > 1) & in_allow).sum()),
                                                                          np.max(allow)))
    bad = np.flatnonzero(~ok)[:4]
    assert ok.all(), (what, bad, got.ravel()[bad], want64.ravel()[bad])


# ================================================================================================ A. anchor targets
def _targets_ref(anchors, fh, fw, stride, gt, im_h, im_w, neg=0.3, pos=0.7, batch=256, num_fg=128, choice=None):
    """anchor_target_layer.py:108-168 with the thresholds, batch and num_fg as parameters (orc.bbox_overlaps for the IoU).
    choice(inds, size) picks the positions to disable, as in orc.anchor_target_layer."""
    allb = orc.all_anchor_boxes_f64(fh, fw, stride, anchors)
    inds, inside = orc.keep_inside(allb, (im_h, im_w))
    ov = orc.bbox_overlaps(inside, gt[:, :4])
    argmax = ov.argmax(axis=1)
    max_ov = ov[np.arange(len(inds)), argmax]
    gt_max = ov[ov.argmax(axis=0), np.arange(ov.shape[1])]
    gt_rows = np.where(ov == gt_max)[0]
    labels = np.full((len(inds),), -1, np.int32)
    labels[max_ov < neg] = 0
    labels[gt_rows] = 1
    labels[max_ov >= pos] = 1
    labels[max_ov < neg] = 0
    before = labels.copy()
    fg = np.where(labels == 1)[0]
    if len(fg) > num_fg:
        labels[np.asarray(choice(fg, len(fg) - num_fg), np.int64)] = -1
    num_bg = batch - int((labels == 1).sum())
    bg = np.where(labels == 0)[0]
    if len(bg) > num_bg:
        labels[np.asarray(choice(bg, len(bg) - num_bg), np.int64)] = -1
    targets = orc.bbox_transform(inside, gt[argmax]).astype(f32)
    return dict(labels=labels, targets=targets, inds_inside=inds, n_all=len(allb), labels_before_subsample=before,
                max_overlaps=max_ov, overlaps=ov, gt_rows=gt_rows)


def _first(inds, size):
    return inds[:size]


def _device_targets(tops, anchors, fh, fw, stride, gt, im_h, im_w, mode=0, **kw):
    if "disable_pos" in kw:
        kw["disable_pos"] = _dev(np.asarray(kw["disable_pos"], np.int32))
    w = tops.anchor_targets(_dev(anchors.astype(f64)), len(anchors), fh, fw, stride, _dev(gt.astype(f32)), im_h, im_w,
                            mode=mode, **kw)
    c = w.counts.cpu().numpy().copy()
    return dict(work=w, counts=c, labels=w.labels_full.cpu().numpy().copy(), targets=w.targets_full.cpu().numpy().copy(),
                inds=w.inds_inside[:int(c[0])].cpu().numpy().copy())


def _assert_targets(d, r, labels_key="labels_before_subsample"):
    n_all, inds = r["n_all"], r["inds_inside"]
    assert np.array_equal(d["inds"], inds)
    assert d["labels"].shape == (n_all,)
    assert np.array_equal(d["labels"][inds], r[labels_key])
    outside = np.ones(n_all, bool)
    outside[inds] = False
    assert (d["labels"][outside] == -1).all() and (d["targets"][outside] == 0).all()
    lab, before = r[labels_key], r["labels_before_subsample"]
    want = [len(inds), int((lab == 1).sum()), int((lab == 0).sum()), int((before == 1).sum()), int((before == 0).sum()), n_all, 0, 0]
    assert d["counts"].tolist() == want, (d["counts"].tolist(), want)
    u = _ulp(d["targets"][inds], r["targets"])
    print("BAR anchor targets: max ulp %d over %d anchors" % (u.max(initial=0), len(inds)))
    assert u.max(initial=0) <= 1


def _gt_at(box, gw, gh, iw, ih, cls=1):
    """An integer gt box gw x gh whose intersection with `box` is iw x ih (it hangs over the box's right and bottom)."""
    x1, y1 = box[2] - iw + 1, box[3] - ih + 1
    return [x1, y1, x1 + gw - 1, y1 + gh - 1, cls]


def _shifted(anchors, a, px, py, stride):
    return anchors[a] + np.array([px, py, px, py], f64) * stride


def _random_gt(rng, n, im_h, im_w, lo=16, hi=None):
    hi = hi or 0.5 * min(im_h, im_w)
    w, h = rng.uniform(lo, hi, n), rng.uniform(lo, hi, n)
    x1, y1 = np.floor(rng.uniform(0, im_w - w)), np.floor(rng.uniform(0, im_h - h))
    return np.stack([x1, y1, np.floor(x1 + w - 1), np.floor(y1 + h - 1), rng.integers(1, 21, n)], 1).astype(f32)


def _case(name):
    """-> anchors, fh, fw, stride, gt [G,5] float32, im_h, im_w."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("a9_s16"):
        # n_all = 9*37*61 = 20313: not a multiple of 32, 256 or 1024
        fh, fw, stride, im_h, im_w, anchors = 37, 61, 16, 592, 976, ANCHORS
        # integer gt boxes at IoU exactly 7/10 and 3/10 with one anchor (sizes from solving 17*I = 7*(A+G), 13*I = 3*(A+G)),
        # far enough apart that nothing else overlaps those anchors more
        exact = [_gt_at(_shifted(ANCHORS, 3, 10, 8, 16), 93, 128, 91, 128), _gt_at(_shifted(ANCHORS, 3, 30, 8, 16), 41, 128, 39, 128),
                 _gt_at(_shifted(ANCHORS, 0, 12, 25, 16), 138, 93, 138, 91), _gt_at(_shifted(ANCHORS, 6, 45, 22, 16), 29, 176, 27, 176),
                 _gt_at(_shifted(ANCHORS, 0, 50, 6, 16), 63, 96, 57, 96), _gt_at(_shifted(ANCHORS, 6, 28, 27, 16), 64, 183, 64, 175)]
        gt = np.vstack([np.array(exact, f32), _random_gt(rng, 3, im_h, im_w)]) if name == "a9_s16_rand" else np.array(exact, f32)
    elif name == "a9_s32":
        fh, fw, stride, im_h, im_w, anchors = 19, 31, 32, 600, 1000, ANCHORS          # the ResNet geometry: 5301 anchors
        gt = _random_gt(rng, 7, im_h, im_w, 40, 500)
    elif name.startswith("a15"):
        fh, fw, stride, im_h, im_w, anchors = 23, 29, 16, 368, 464, ANCHORS15           # 10005 anchors
        if name == "a15_exact":
            gt = np.array([list(_shifted(ANCHORS15, 0, px, py, 16)) + [3] for px, py in ((3, 2), (12, 2), (22, 3), (5, 12), (17, 15))], f32)
        else:
            a = _shifted(ANCHORS15, 8, 8, 8, 16)                                          # 128x128 at (128, 128)
            mirror = [[a[0] + 24, a[1], a[2] + 24, a[3], 4], [a[0] - 24, a[1], a[2] - 24, a[3], 5]]   # same IoU with a
            tie = [[200 + 8, 40, 200 + 8 + 63, 40 + 63, 6]]                               # halfway between two 64x64 anchors
            dup = [list(_shifted(ANCHORS15, 13, 20, 14, 16)) + [7]] * 2 + [list(_shifted(ANCHORS15, 13, 20, 14, 16)) + [9]]
            gt = np.array(mirror + tie + dup, f32)
    elif name == "a9_degenerate":
        fh, fw, stride, im_h, im_w, anchors = 38, 63, 16, 600, 1000, ANCHORS
        gt = np.array([[100, 100, 99, 300, 1],                       # zero width: x2 = x1 - 1
                       [400, 200, 600, 199, 2],                      # zero height
                       [700, 100, 650, 90, 3],                       # negative width and height
                       [1200, 700, 1400, 900, 4],                    # entirely outside the image
                       [-300, -200, -10, -5, 5],                     # outside, to the top left
                       [0, 0, 999, 599, 6],                          # the whole image
                       [300, 250, 520, 430, 7]], f32)
    else:
        raise KeyError(name)
    return anchors, fh, fw, stride, gt, im_h, im_w


THRESHOLDS = {"a9_s16_exact": (0.3, 0.7), "a9_s16_rand": (0.3, 0.7), "a9_s32": (0.3, 0.7), "a15_exact": (0.3, 0.7),
              "a15_dup": (0.3, 0.7), "a9_degenerate": (0.3, 0.7), "a9_s16_rand@0.2/0.6": (0.2, 0.6),
              "a9_s32@0.5/0.9": (0.5, 0.9), "a15_exact@0.45/0.45": (0.45, 0.45), "a15_dup@0.1/0.5": (0.1, 0.5)}


def test_targets_ref_matches_the_oracle_at_the_reference_values():
    """The parametrised restatement is the oracle's anchor_target_layer at 0.3 / 0.7 / 256 / 128."""
    for name in ("a9_s16_rand", "a15_dup"):
        anchors, fh, fw, stride, gt, im_h, im_w = _case(name)
        mine = _targets_ref(anchors, fh, fw, stride, gt, im_h, im_w, choice=_first)
        r = orc.anchor_target_layer(fh, fw, gt[None], np.array([[im_h, im_w]]), anchors=anchors, feat_stride=stride, choice=_first)
        for k in ("labels", "inds_inside", "labels_before_subsample", "max_overlaps"):
            assert np.array_equal(mine[k], r[k]), k
        assert mine["n_all"] == r["n_all"] and np.array_equal(mine["targets"], r["targets"])


@pytest.mark.parametrize("case", list(THRESHOLDS))
def test_anchor_targets_geometry_and_thresholds(tops, case):
    name = case.split("@")[0]
    neg, pos = THRESHOLDS[case]
    anchors, fh, fw, stride, gt, im_h, im_w = _case(name)
    r = _targets_ref(anchors, fh, fw, stride, gt, im_h, im_w, neg, pos, choice=_first)
    d = _device_targets(tops, anchors, fh, fw, stride, gt, im_h, im_w, mode=0, neg_thr=neg, pos_thr=pos)
    _assert_targets(d, r)
    mo, before, ov = r["max_overlaps"], r["labels_before_subsample"], r["overlaps"]
    assert (ov >= 0).all() and not np.signbit(ov).any()
    if case in ("a9_s16_exact", "a15_exact"):
        # the thresholds are met exactly, by anchors that are not the best anchor of any gt: only >= / < decide them
        not_best = np.ones(len(mo), bool)
        not_best[r["gt_rows"]] = False
        assert ((mo == 0.7) & not_best & (before == 1)).any()
        assert ((mo == 0.3) & not_best & (before == -1)).any()
        if case == "a15_exact":
            assert ((mo == 0.725) & (before == 1)).sum() == 5 and ((mo == 0.675) & (before == -1)).sum() == 5
            assert ((mo == 0.275) & (before == 0)).sum() == 5 and ((mo == 0.325) & (before == -1)).sum() == 5
    if name == "a15_dup":
        # mirrored gt boxes: equal IoU, the first column wins the arg-max (and so the regression target)
        ties = np.where((ov[:, 0] == ov[:, 1]) & (ov[:, 0] == mo) & (mo > 0))[0]
        assert ties.size and (ov[ties].argmax(1) == 0).all()
        # a gt whose best IoU several anchors share: every such row is a positive unless the background rule clobbers it
        counts = (ov == ov.max(0)).sum(0)
        assert counts.max() > 1
        assert (before[r["gt_rows"]][mo[r["gt_rows"]] >= neg] == 1).all()
    if name == "a9_degenerate":
        # a gt no inside anchor overlaps has gt_max == 0: every inside row with IoU 0 to it counts as its best
        assert (ov[:, :5] == 0).all()


def test_bbox_overlaps_is_never_negative_on_degenerate_boxes(tops):
    anchors, fh, fw, stride, gt, im_h, im_w = _case("a9_degenerate")
    allb = orc.all_anchor_boxes_f64(fh, fw, stride, anchors)
    q = gt[:, :4].astype(f64)
    got = tops.bbox_overlaps(_dev(allb), _dev(q)).cpu().numpy()
    assert np.array_equal(got, orc.bbox_overlaps(allb, q))
    assert (got >= 0).all() and not np.signbit(got).any()
    # and against each other: inverted boxes on both sides
    inv = np.vstack([q, q[:, [2, 3, 0, 1]]])
    got = tops.bbox_overlaps(_dev(inv), _dev(inv)).cpu().numpy()
    assert np.array_equal(got, orc.bbox_overlaps(inv, inv)) and not np.signbit(got).any()


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_no_anchor_inside_the_image(tops, mode):
    """The reference raises on its empty arg-max; the device returns an empty target set and rpn_loss zeros."""
    A, fh, fw, im_h, im_w = 9, 5, 7, 64, 96                     # every anchor of this set is wider than 64 pixels
    gt = np.array([[10, 10, 40, 50, 1]], f32)
    kw = dict(disable_pos=[0, 1, -1]) if mode == 2 else dict(seed=3)
    d = _device_targets(tops, ANCHORS, fh, fw, 16, gt, im_h, im_w, mode=mode, **kw)
    n_all = A * fh * fw
    assert d["counts"].tolist() == [0, 0, 0, 0, 0, n_all, 0, 0]
    assert (d["labels"] == -1).all() and (d["targets"] == 0).all()
    rng = np.random.default_rng(1)
    score = rng.standard_normal((2 * A, fh, fw)).astype(f32)
    pred = rng.standard_normal((4 * A, fh, fw)).astype(f32)
    losses, ds, db = tops.rpn_loss(_dev(score), _dev(pred), _dev(ANCHORS), A, fh, fw, 16, im_h, im_w, d["work"])
    assert (losses.cpu().numpy() == 0).all() and not ds.cpu().numpy().any() and not db.cpu().numpy().any()


# ================================================================================================ B. device subsampling
def _mix64(x):
    x = x + np.uint64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def _sample_key(seed, idx):
    """rpn_train.cu sample_key: (top 32 bits of mix64(seed ^ i*0xD6E8FEB86659FD93)) << 32 | i, in uint64."""
    i = np.asarray(idx, np.int64).astype(np.uint64)
    with np.errstate(over="ignore"):
        h = _mix64(np.uint64(seed & (2 ** 64 - 1)) ^ (i * np.uint64(0xD6E8FEB86659FD93)))
    return (h & np.uint64(0xFFFFFFFF00000000)) | i


def _hash_choice(seed, inds_inside, before):
    """The device's mode-1 rule as an oracle `choice`: disable the `size` candidates with the smallest key; positives
    are keyed by `seed`, negatives by seed ^ 0xA5A5A5A5DEADBEEF."""
    def choice(pos, size):
        s = seed if before[pos[0]] == 1 else seed ^ BG_SEED_XOR
        return pos[np.argsort(_sample_key(s, inds_inside[pos]), kind="stable")[:size]]
    return choice


def test_sample_key_restatement_known_values():
    """Two values of the splitmix64 finaliser (seed 0's first output is the published 0xE220A8397B1DCDAF)."""
    assert int(_mix64(np.array([0], np.uint64))[0]) == 0xE220A8397B1DCDAF
    k = _sample_key(0, [0, 5])
    assert int(k[0]) == 0xE220A8397B1DCDAF & 0xFFFFFFFF00000000 and int(k[1]) & 0xFFFFFFFF == 5


@pytest.mark.parametrize("regime", ["headline_38x63", "exactly_40960", "uncached_64x72"])
def test_device_subsampling_disables_the_smallest_keys(tops, regime):
    rng = np.random.default_rng(41)
    if regime == "headline_38x63":
        anchors, fh, fw, im_h, im_w, pos = ANCHORS, 38, 63, 600, 1000, 0.7
        gt = _random_gt(rng, 40, im_h, im_w, 100, 300)
    elif regime == "exactly_40960":
        anchors, fh, fw, im_h, im_w, pos = ANCHORS4, 80, 128, 1280, 2048, 0.5      # 4*80*128 = 40960: the last cached size
        gt = _random_gt(rng, 60, im_h, im_w, 100, 400)
    else:
        anchors, fh, fw, im_h, im_w, pos = ANCHORS, 64, 72, 1024, 1152, 0.5         # 41472 anchors: keys are not cached
        gt = _random_gt(rng, 60, im_h, im_w, 100, 400)
    seed = 0x1234_5678_9ABC_DEF0
    r0 = _targets_ref(anchors, fh, fw, 16, gt, im_h, im_w, pos=pos, choice=_first)
    assert (r0["labels_before_subsample"] == 1).sum() > 128 and (r0["labels_before_subsample"] == 0).sum() > 256
    choice = _hash_choice(seed, r0["inds_inside"], r0["labels_before_subsample"])
    if pos == 0.7:
        r = orc.anchor_target_layer(fh, fw, gt[None], np.array([[im_h, im_w]]), anchors=anchors, choice=choice)
    else:
        r = _targets_ref(anchors, fh, fw, 16, gt, im_h, im_w, pos=pos, choice=choice)
    d = _device_targets(tops, anchors, fh, fw, 16, gt, im_h, im_w, mode=1, seed=seed, pos_thr=pos)
    _assert_targets(d, r, labels_key="labels")
    assert int(d["counts"][1]) == 128 and int(d["counts"][2]) == 128


def _tie(idx, seed_xor):
    """First seed s >= 1 for which two of the candidate anchor indices `idx` share the 32-bit hash: -> (s, rank of the
    lower-index member in (hash, index) order, the two indices)."""
    for s in range(1, 20000):
        k = _sample_key(s ^ seed_xor, idx)
        order = np.argsort(k, kind="stable")
        h = (k[order] >> np.uint64(32))
        eq = np.flatnonzero(h[1:] == h[:-1])
        if eq.size:
            j = int(eq[0])
            return s, j, int(idx[order[j]]), int(idx[order[j + 1]])
    raise AssertionError("no hash tie among %d candidates" % len(idx))


@pytest.mark.parametrize("which", ["fg", "bg"])
@pytest.mark.parametrize("regime", ["cached_38x63", "uncached_64x72"])
def test_device_subsampling_breaks_hash_ties_toward_the_lower_index(tops, regime, which):
    fh, fw, im_h, im_w = (38, 63, 600, 1000) if regime.startswith("cached") else (64, 72, 1024, 1152)
    gt = np.array([[100, 100, 300, 260, 1], [500, 300, 760, 520, 2]], f32)
    # every inside anchor a positive (both thresholds 0) or a negative (both above 1) candidate
    thr = 0.0 if which == "fg" else 2.0
    r0 = _targets_ref(ANCHORS, fh, fw, 16, gt, im_h, im_w, thr, thr, choice=_first)
    inds = r0["inds_inside"]
    assert (r0["labels_before_subsample"] == (1 if which == "fg" else 0)).all()
    s, rank, lo, hi = _tie(inds, 0 if which == "fg" else BG_SEED_XOR)
    n_dis = rank + 1                                             # the cut-off falls between the two tied anchors
    keep = len(inds) - n_dis
    batch, num_fg = (keep, keep) if which == "fg" else (keep, 0)
    choice = _hash_choice(s, inds, r0["labels_before_subsample"])
    r = _targets_ref(ANCHORS, fh, fw, 16, gt, im_h, im_w, thr, thr, batch=batch, num_fg=num_fg, choice=choice)
    d = _device_targets(tops, ANCHORS, fh, fw, 16, gt, im_h, im_w, mode=1, seed=s, neg_thr=thr, pos_thr=thr, batch=batch,
                        num_fg=num_fg)
    print("tie %s %s: seed %d, anchors %d and %d share the hash at rank %d of %d" % (regime, which, s, lo, hi, rank, len(inds)))
    assert d["labels"][lo] == -1 and d["labels"][hi] == (1 if which == "fg" else 0)
    _assert_targets(d, r, labels_key="labels")


def test_device_subsampling_refuses_more_positives_than_the_batch(tops):
    """num_fg > batch used to leave counts[2] = batch - num_fg < 0, the loss normaliser with it."""
    from frcnn_b200._lib import FrcnnError
    anchors, fh, fw, stride, gt, im_h, im_w = _case("a9_s32")
    for batch, num_fg in ((256, 300), (64, 65), (0, 1), (256, -1)):
        with pytest.raises(FrcnnError, match="num_fg"):
            _device_targets(tops, anchors, fh, fw, stride, gt, im_h, im_w, mode=1, batch=batch, num_fg=num_fg)
    d = _device_targets(tops, anchors, fh, fw, stride, gt, im_h, im_w, mode=1, batch=256, num_fg=256, seed=5)
    assert (d["counts"] >= 0).all()


def test_list_subsampling_ignores_bad_positions(tops):
    """Mode 2 disables each valid position once and ignores duplicates, negatives and positions >= n_inside."""
    anchors, fh, fw, stride, gt, im_h, im_w = _case("a9_s16_rand")
    r0 = _targets_ref(anchors, fh, fw, stride, gt, im_h, im_w, choice=_first)
    n_in = len(r0["inds_inside"])
    rng = np.random.default_rng(8)
    valid = rng.choice(n_in, 300, replace=False)
    pos = np.concatenate([valid, valid[:50], [-1, -7, -(1 << 31), n_in, n_in + 1, 1 << 30, n_in - 1, n_in - 1]])
    rng.shuffle(pos)
    d = _device_targets(tops, anchors, fh, fw, stride, gt, im_h, im_w, mode=2, disable_pos=pos)
    lab = r0["labels_before_subsample"].copy()
    lab[np.concatenate([valid, [n_in - 1]])] = -1
    r = dict(r0, labels=lab)
    _assert_targets(d, r, labels_key="labels")


# ================================================================================================ C. RPN loss
def _allowances(m_abs, scale):
    """Extra absolute allowance on the extreme-logit sets.  The kernels form lse = m + log(sum exp(z - m)) and
    ce = lse - z in double: every double operation is within 1 ulp (2^-52 relative) and the operands are at most
    |m| + log(#classes) + 1 in size, so ce carries at most 4 ulps of that size, 4 * 2^-52 * (|m| + log C + 1), summed over
    the rows it averages.  A gradient is (p - [c == t]) * scale with p in [0, 1] from an exp and a division: at most
    4 * 2^-52 * |scale| absolute.  Both only matter where the exact value cancels to far below that size (a loss of
    exp(-80), a gradient of 1 - p ~ 0); anywhere else they are below half a float32 ulp."""
    return 4 * EPS * float(np.sum(m_abs)), 4 * EPS * abs(scale)


def _softplus(x):
    return np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x)))


def _sigmoid(x):
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, 1 / (1 + e), e / (1 + e))


def rpn_ref(z0, z1, lab, pred, tgt, inside, n_all, delta, lam, gs):
    """float64 restatement of region_proposal_network.py:160-204 per anchor i (z0/z1 = bg/fg logit, pred/tgt [n_all, 4]):
    -> (losses [4], dz0, dz1, dpred [n_all,4]) as float64; gradients of gs * (loss_cls + lam * loss_bbox)."""
    valid = lab >= 0
    nv = int(valid.sum())
    cnt = max(nv, 1)
    zl, zo = np.where(lab == 1, z1, z0), np.where(lab == 1, z0, z1)
    x = zo - zl                                                  # ce = log(1 + e^x), p_other = sigmoid(x)
    ce = np.where(valid, _softplus(x), 0.0)
    po = np.where(valid, _sigmoid(x), 0.0)
    s = gs / cnt
    g_lab, g_oth = -po * s, po * s
    dz0, dz1 = np.where(lab == 1, g_oth, g_lab), np.where(lab == 1, g_lab, g_oth)
    correct = valid & ((z1 > z0).astype(np.int32) == lab)
    d = pred - tgt
    ad = np.abs(d)
    hub = np.where(ad < delta, 0.5 * d * d, delta * (ad - 0.5 * delta)) * inside[:, None]
    dp = np.where(ad < delta, d, np.sign(d) * delta) * (lam * gs / n_all) * inside[:, None]
    lc = math.fsum(ce) / cnt
    lb = math.fsum(hub.ravel()) / n_all
    acc = int(correct.sum()) / nv if nv else 0.0
    return np.array([lc, lb, acc, lc + lam * lb]), dz0, dz1, dp


def test_float64_references_match_torch():
    """rpn_ref and rcnn_ref against torch float64 cross_entropy(ignore_index=-1) and huber_loss, values and gradients."""
    import torch.nn.functional as F
    rng = np.random.default_rng(3)
    n = 500
    z = rng.standard_normal((n, 2)) * 3
    lab = rng.integers(-1, 2, n)
    pred, tgt = rng.standard_normal((n, 4)) * 3, rng.standard_normal((n, 4))
    inside = rng.random(n) < 0.8
    L, dz0, dz1, dp = rpn_ref(z[:, 0], z[:, 1], lab, pred, tgt, inside, n, 3.0, 1.5, 0.5)
    zt = torch.tensor(z, requires_grad=True)
    pt = torch.tensor(pred, requires_grad=True)
    lc = F.cross_entropy(zt, torch.tensor(lab), ignore_index=-1)
    msk = torch.tensor(inside)
    lb = F.huber_loss(pt[msk], torch.tensor(tgt)[msk], reduction="sum", delta=3.0) / n
    (0.5 * (lc + 1.5 * lb)).backward()
    np.testing.assert_allclose(L[:2], [lc.item(), lb.item()], rtol=1e-14)
    np.testing.assert_allclose(np.stack([dz0, dz1], 1), zt.grad.numpy(), rtol=1e-12, atol=1e-17)
    np.testing.assert_allclose(dp, pt.grad.numpy(), rtol=1e-12, atol=1e-17)
    # rcnn
    R, NC = 40, 7
    head = rng.standard_normal((R, 5 * NC)) * 2
    keep = rng.permutation(R)[:25]
    labels = rng.integers(0, NC, 25)
    ext = rng.standard_normal((25, 4 * NC))
    L, dh = rcnn_ref(head, keep, labels, ext, NC, 1.0, 0.7)
    ht = torch.tensor(head, requires_grad=True)
    kt = torch.tensor(keep)
    lc = F.cross_entropy(ht[kt, :NC], torch.tensor(labels))
    lb = F.huber_loss(ht[kt, NC:], torch.tensor(ext), reduction="sum", delta=1.0) / 25
    (0.7 * (lc + lb)).backward()
    np.testing.assert_allclose(L[[0, 1, 3]], [lc.item(), lb.item(), (lc + lb).item()], rtol=1e-14)
    np.testing.assert_allclose(dh, ht.grad.numpy(), rtol=1e-12, atol=1e-17)


def _rpn_inputs(kind, A, fh, fw, inside, rng):
    """-> score [2A,HW], pred [4A,HW], labels [n_all], targets [n_all,4] (float32 / int32), delta."""
    n_all, HW = A * fh * fw, fh * fw
    lab = np.where(inside, rng.integers(-1, 2, n_all), -1).astype(np.int32)
    score = (rng.standard_normal((2 * A, HW)) * 2).astype(f32)
    pred = (rng.standard_normal((4 * A, HW)) * 2.5).astype(f32)
    tgt = np.where(inside[:, None], rng.standard_normal((n_all, 4)) * 0.5, 0).astype(f32)
    delta = 3.0
    if kind == "ties":
        t = rng.random(HW) < 0.5
        score[A:, :] = np.where(t[None], score[:A, :], score[A:, :])
    elif kind in ("gap80", "gap1e4"):
        g = 80.0 if kind == "gap80" else 1e4
        score[A:, :] = score[:A, :] + (rng.choice([-g, g], (A, HW))).astype(f32)
    elif kind == "huber_edges":
        # |d| exactly delta and one float32 ulp either side, on both signs: targets 0.5, pred 0.5 +- {3, 3 +- ulp}
        tgt = np.where(inside[:, None], f32(0.5), f32(0)).astype(f32)
        vals = np.array([3.5, np.nextafter(f32(3.5), f32(4)), np.nextafter(f32(3.5), f32(3)), -2.5, np.nextafter(f32(-2.5), f32(-3)),
                         np.nextafter(f32(-2.5), f32(-2)), 0.5, 1.25], f32)
        pred = rng.choice(vals, (4 * A, HW)).astype(f32)
    elif kind == "all_ignored":
        lab[:] = -1
    return score, pred, lab, tgt, delta


RPN_CASES = [  # (kind, A-set, fh, fw, layout, ld, lam, gs)
    ("nominal", "a9", 37, 61, "nchw", 0, 1.0, 1.0),          # 20313 anchors: a partial last 256-block
    ("nominal", "a9", 37, 61, "nhwc", 54, 1.0, 1.0),          # ld = 6A exactly
    ("nominal", "a9", 37, 61, "nhwc", 64, 1.5, 1.0),          # padded rows
    ("nominal", "a15", 23, 29, "nchw", 0, 1.0, 1.0),
    ("nominal", "a4", 9, 13, "nhwc", 32, 1.0, 1.0),           # 468 anchors
    ("ties", "a9", 19, 23, "nchw", 0, 1.0, 1.0),
    ("gap80", "a9", 19, 23, "nchw", 0, 1.0, 1.0),
    ("gap1e4", "a15", 23, 29, "nhwc", 96, 1.0, 1.0),
    ("huber_edges", "a9", 19, 23, "nchw", 0, 1.0, 1.0),
    ("nominal", "a9", 19, 23, "nchw", 0, 0.0, 1.0),           # lambda = 0
    ("nominal", "a9", 19, 23, "nhwc", 64, 2.0, 0.37),         # grad_scale != 1
    ("all_ignored", "a9", 19, 23, "nchw", 0, 1.0, 1.0),
]
ASETS = {"a9": ANCHORS, "a15": ANCHORS15, "a4": ANCHORS4}


@pytest.mark.parametrize("case", RPN_CASES, ids=["%s-%s-%dx%d-%s%d-l%g-g%g" % c for c in RPN_CASES])
def test_rpn_loss_against_float64(tops, case):
    kind, aset, fh, fw, layout, ld, lam, gs = case
    anchors = ASETS[aset]
    A, stride = len(anchors), 16
    im_h, im_w = fh * stride, fw * stride
    n_all, HW = A * fh * fw, fh * fw
    allb = orc.all_anchor_boxes_f64(fh, fw, stride, anchors)
    inside = np.zeros(n_all, bool)
    inside[orc.keep_inside(allb, (im_h, im_w))[0]] = True
    rng = np.random.default_rng(len(kind) * 1000 + fh + ld)
    score, pred, lab, tgt, delta = _rpn_inputs(kind, A, fh, fw, inside, rng)
    # labels, targets and counts go in through the AnchorTargets buffers
    w = tops.AnchorTargets(A, fh, fw, "cuda")
    w.labels_full.copy_(_dev(lab))
    w.targets_full.copy_(_dev(tgt))
    w.counts.copy_(_dev(np.array([inside.sum(), (lab == 1).sum(), (lab == 0).sum(), 0, 0, n_all, 0, 0], np.int32)))
    an = _dev(anchors)

    def run(want_grads=True):
        if layout == "nchw":
            L, ds, db = tops.rpn_loss(_dev(score), _dev(pred), an, A, fh, fw, stride, im_h, im_w, w, delta=delta, loss_lambda=lam,
                                      grad_scale=gs, want_grads=want_grads)
            return L.cpu().numpy(), (ds.cpu().numpy() if want_grads else None), (db.cpu().numpy() if want_grads else None)
        m = np.zeros((HW, ld), f32)
        m[:, :2 * A], m[:, 2 * A:6 * A] = score.T, pred.T
        m[:, 6 * A:] = 7.0                                       # padding must neither be read nor written
        L, dm, _ = tops.rpn_loss(_dev(m), None, an, A, fh, fw, stride, im_h, im_w, w, delta=delta, loss_lambda=lam, grad_scale=gs,
                                 layout="nhwc", ld=ld, want_grads=want_grads)
        if not want_grads:
            return L.cpu().numpy(), None, None
        dm = dm.cpu().numpy()
        assert not dm[:, 6 * A:].any()
        return L.cpu().numpy(), dm[:, :2 * A].T.copy(), dm[:, 2 * A:6 * A].T.copy()

    L, ds, db = run()
    # anchor order i = k*A + a: score channel a / A+a, bbox channel j*A + a, at pixel k
    z0 = score[:A].T.reshape(-1).astype(f64)
    z1 = score[A:].T.reshape(-1).astype(f64)
    p4 = pred.reshape(4, A, HW).transpose(2, 1, 0).reshape(-1, 4).astype(f64)
    WL, dz0, dz1, dp = rpn_ref(z0, z1, lab, p4, tgt.astype(f64), inside, n_all, delta, lam, gs)
    extreme = kind.startswith("gap")
    cnt = max(int((lab >= 0).sum()), 1)
    ce_allow, g_allow = _allowances(np.abs(np.maximum(z0, z1))[lab >= 0] + 1, gs / cnt) if extreme else (0.0, 0.0)
    _close("rpn losses %s" % kind, L, WL, np.array([ce_allow / cnt, 0, 0, ce_allow / cnt]))
    want_ds = np.concatenate([dz0.reshape(HW, A).T, dz1.reshape(HW, A).T])
    want_db = dp.reshape(HW, A, 4).transpose(2, 1, 0).reshape(4 * A, HW)
    _close("rpn dscore %s" % kind, ds, want_ds, g_allow)
    _close("rpn dbbox %s" % kind, db, want_db)
    assert not ds[np.concatenate([lab.reshape(HW, A).T] * 2) < 0].any()             # exactly zero where no loss term applies
    assert not db[~np.concatenate([inside.reshape(HW, A).T] * 4)].any()
    if kind == "all_ignored":
        assert L[0] == 0 and L[2] == 0 and not ds.any()
    if kind == "ties":
        tied = (z0 == z1) & (lab >= 0)
        assert tied.any()
    # without gradients: the same losses; repeated: bit-identical (fixed-order reduction)
    L2, _, _ = run(False)
    L3, ds3, db3 = run()
    assert np.array_equal(L2.view(np.int32), L.view(np.int32))
    assert np.array_equal(L3.view(np.int32), L.view(np.int32)) and np.array_equal(ds3, ds) and np.array_equal(db3, db)


# ================================================================================================ D. RCNN loss
def rcnn_ref(head, keep, labels, ext, NC, delta, gs):
    """float64 restatement of faster_rcnn.py:151-165 on the merged head rows: -> (losses [4], dhead like head)."""
    head = np.asarray(head, f64)
    n = len(keep)
    z = head[keep, :NC]
    m = z.max(1, keepdims=True)
    e = np.exp(z - m)
    S = e.sum(1, keepdims=True)
    ok = (labels >= 0) & (labels < NC)
    t = np.where(ok, labels, 0)
    zt = z[np.arange(n), t]
    # ce = lse - z_t = (m - z_t) + log S; NaN for a label outside [0, NC)
    ce = np.where(ok, (m[:, 0] - zt) + np.log(S[:, 0]), np.nan)
    p = e / S
    onehot = np.zeros_like(p)
    onehot[np.arange(n)[ok], t[ok]] = 1.0
    g = p - onehot
    # p_t - 1 without cancellation: minus the other classes' share of the sum
    others = np.where(onehot > 0, 0.0, e).sum(1)
    g[np.arange(n)[ok], t[ok]] = -(others / S[:, 0])[ok]
    d = head[keep, NC:5 * NC] - np.asarray(ext, f64)
    ad = np.abs(d)
    hub = np.where(ad < delta, 0.5 * d * d, delta * (ad - 0.5 * delta))
    gd = np.where(ad < delta, d, np.sign(d) * delta)
    acc = float((z.argmax(1) == labels).sum()) / n
    lc = math.fsum(ce) / n if ok.all() else float("nan")
    lb = math.fsum(hub.ravel()) / n
    dh = np.zeros(head.shape, f64)
    dh[keep, :NC] = g * gs / n
    dh[keep, NC:5 * NC] = gd * gs / n
    return np.array([lc, lb, acc, lc + lb]), dh


def _rcnn_case(tops, n, NC, ld, kind, rng, gs=1.0, delta=1.0):
    R = 300
    head = np.full((R, ld), 5.0, f32)                            # padding columns: a nonzero value that must not leak
    head[:, :NC] = rng.standard_normal((R, NC)) * 2
    head[:, NC:5 * NC] = rng.standard_normal((R, 4 * NC)) * 0.8
    keep = rng.permutation(R)[:n].astype(np.int32)               # scattered and unsorted
    labels = rng.integers(0, NC, n).astype(np.int32)
    labels[0] = NC - 1
    if n > 1:
        labels[1] = 0
    ext = (rng.standard_normal((n, 4 * NC)) * 0.5).astype(f32)
    ext[rng.random((n, 4 * NC)) < 0.7] = 0
    if kind == "ties":
        for i, r in enumerate(keep):
            c1, c2 = sorted(rng.choice(NC, 2, replace=False))
            head[r, c1] = head[r, c2] = head[r, :NC].max() + 1
            labels[i] = c2 if i % 2 == 0 else c1                 # the first maximum is c1: accuracy counts only odd rows
    elif kind in ("big1e30", "big3e38"):
        v = f32(1e30) if kind == "big1e30" else f32(3e38)
        head[:, :NC] = rng.choice([-v, v], (R, NC))
        head[keep[::3], :NC] = -v
        head[keep[::3], labels[::3]] = v                         # a unique maximum on every third row
    elif kind == "bad_label":
        labels[n // 2] = NC if n % 2 else -1
    L, dh = tops.rcnn_loss(_dev(head), _dev(keep), _dev(labels), _dev(ext), NC, delta, grad_scale=gs)
    WL, wdh = rcnn_ref(head, keep, labels, ext, NC, delta, gs)
    return L.cpu().numpy(), dh.cpu().numpy(), WL, wdh, head, keep, labels


RCNN_SHAPES = [(n, NC) for n in (1, 31, 32, 33, 64, 127, 128) for NC in (2, 21, 32, 33, 81)]


@pytest.mark.parametrize("n,NC", RCNN_SHAPES)
def test_rcnn_loss_rows_and_classes(tops, n, NC):
    rng = np.random.default_rng(n * 100 + NC)
    for ld in (5 * NC, (5 * NC + 31) // 32 * 32 + 32):
        L, dh, WL, wdh, head, keep, labels = _rcnn_case(tops, n, NC, ld, "nominal", rng, gs=0.75 if ld % 2 else 1.0)
        _close("rcnn losses n=%d NC=%d ld=%d" % (n, NC, ld), L, WL)
        _close("rcnn dhead n=%d NC=%d ld=%d" % (n, NC, ld), dh, wdh)
        not_kept = np.ones(300, bool)
        not_kept[keep] = False
        assert not dh[not_kept].any() and not dh[:, 5 * NC:].any()      # exactly zero, not just small


@pytest.mark.parametrize("kind", ["ties", "big1e30", "big3e38", "bad_label"])
@pytest.mark.parametrize("n,NC", [(1, 2), (33, 21), (128, 81)])
def test_rcnn_loss_edges(tops, kind, n, NC):
    rng = np.random.default_rng(7 + n + NC)
    ld = 5 * NC + 3
    L, dh, WL, wdh, head, keep, labels = _rcnn_case(tops, n, NC, ld, kind, rng)
    extreme = kind.startswith("big")
    z = head[keep, :NC].astype(f64)
    ce_allow, g_allow = _allowances(np.abs(z.max(1)) + math.log(NC) + 1, 1.0 / n) if extreme else (0.0, 0.0)
    if kind == "bad_label":
        assert np.isnan(L[0]) and np.isnan(L[3]) and np.isfinite(L[1])
        _close("rcnn losses %s" % kind, L[[1, 2]], WL[[1, 2]])
    else:
        with np.errstate(over="ignore"):
            _close("rcnn losses %s n=%d NC=%d" % (kind, n, NC), L, WL, np.array([ce_allow / n, 0, 0, ce_allow / n]))
    _close("rcnn dhead %s n=%d NC=%d" % (kind, n, NC), dh, wdh, g_allow)
    if kind == "ties":
        assert L[2] == f32(float(np.sum(np.arange(n) % 2 == 1)) / n)


# ================================================================================================ E. proposal targets and helpers
def _gt_ptl():
    return np.array([[40, 40, 79, 59, 1], [200, 100, 299, 139, 2], [200, 100, 299, 139, 3],      # a duplicate box, other class
                     [320, 20, 359, 119, 20], [100, 200, 199, 249, 0]], f32)


@pytest.mark.parametrize("count", [None, 0, 137, 300, 1000, -5])
def test_roi_overlaps_against_bbox_overlaps(tops, count):
    rng = np.random.default_rng(12)
    gt = _gt_ptl()
    R = 300
    rois = np.empty((R, 4), f32)
    src = gt[rng.integers(0, len(gt), R), :4]
    rois[:] = src + rng.integers(-12, 13, (R, 4))
    rois[:20] = gt[[1, 2] * 10, :4]                               # IoU 1 with two equal gt rows: the first wins
    rois[20:30, 2] = rois[20:30, 0] - 1                           # zero width
    c = None if count is None else _dev(np.array([count], np.int32))
    mo, am = tops.roi_overlaps(_dev(rois), c, _dev(gt))
    mo, am = mo.cpu().numpy(), am.cpu().numpy()
    Rv = R if count is None else max(0, min(count, R))
    ov = orc.bbox_overlaps(rois[:Rv], gt[:, :4])
    assert np.array_equal(mo[:Rv], ov.max(1)) and np.array_equal(am[:Rv], ov.argmax(1).astype(np.int32))
    assert (mo[Rv:] == -1.0).all() and (am[Rv:] == -1).all()
    if Rv >= 20:
        assert (am[:20] == 1).all() and (mo[:20] == 1.0).all()


def test_sampling_at_the_exact_thresholds_keeps_what_the_reference_keeps(tops):
    """Proposals nested in a gt at IoU exactly 0.5 and 0.1 (and one pixel either side): the host sampling keeps the set
    orc.proposal_target_layer keeps under the same NumPy seed."""
    from frcnn_b200.train_engine import RcnnTrainer
    gt = np.array([[100, 100, 139, 119, 4], [300, 300, 339, 319, 9]], f32)         # 40 x 20
    rows = []
    for g in gt:
        for w in (20, 21, 19, 4, 5, 3, 40, 30):                                    # IoU w/40: 0.5, .525, .475, 0.1, .125, .075
            rows.append([g[0], g[1], g[0] + w - 1, g[3]])
    props = np.array(rows * 3, f32)
    mo, am = tops.roi_overlaps(_dev(props), None, _dev(gt))
    mo_h = mo.cpu().numpy()
    assert (mo_h == 0.5).sum() == 6 and (mo_h == 0.1).sum() == 6
    for seed in (0, 1, 2):
        np.random.seed(seed)
        got = RcnnTrainer._sample(None, mo, len(props))
        np.random.seed(seed)
        r = orc.proposal_target_layer(props, gt[None])
        assert np.array_equal(got, r["keep_inds"])
        kept = set(got.tolist())
        assert all(i in kept for i in np.flatnonzero(mo_h == 0.5)) and all(i in kept for i in np.flatnonzero(mo_h == 0.1))
        assert not any(i in kept for i in np.flatnonzero(mo_h == 0.075))
        fg = set(np.flatnonzero(mo_h >= 0.5).tolist())
        assert set(got[:r["n_fg"]].tolist()) == fg


@pytest.mark.parametrize("NC", [2, 21, 81])
def test_roi_targets_classes_and_degenerate_proposals(tops, NC):
    rng = np.random.default_rng(NC)
    G = 8
    gt = _random_gt(rng, G, 600, 1000)
    gt[:, 4] = [0, NC - 1, NC, NC + 5, 1, min(3, NC - 1), -1, NC - 1]            # class 0, last, >= NC, negative
    R = 200
    rois = _random_gt(rng, R, 600, 1000)[:, :4].copy()
    rois[:10, 2] = rois[:10, 0] - 1                                               # zero width: ew = 0
    rois[10:15, 3] = rois[10:15, 1] - 1                                           # zero height
    rois[15:18] = rois[15:18, [2, 3, 0, 1]]                                       # inverted: negative sizes
    argmax = rng.integers(0, G, R).astype(np.int32)
    argmax[:G] = np.arange(G)
    keep = rng.permutation(R)[:150].astype(np.int32)
    keep[:18] = np.arange(18)
    use_gt, ext, labels = tops.roi_targets(_dev(rois), _dev(gt), _dev(argmax), _dev(keep), NC)
    want_gt = gt[argmax[keep]]
    assert np.array_equal(use_gt.cpu().numpy(), want_gt)
    assert np.array_equal(labels.cpu().numpy(), want_gt[:, 4].astype(np.int32))
    with np.errstate(all="ignore"):
        reg = orc.bbox_transform(rois[keep], want_gt)                             # float32 in, float32 arithmetic
    want = np.zeros((len(keep), 4 * NC), f32)
    for i, c in enumerate(want_gt[:, 4]):
        if c > 0 and int(c) < NC:
            want[i, 4 * int(c):4 * int(c) + 4] = reg[i]
    got = ext.cpu().numpy()
    assert np.array_equal(got == 0, want == 0)
    u = _ulp(got, want)
    print("BAR roi targets NC=%d: max ulp %d, %d non-finite" % (NC, u.max(), int((~np.isfinite(want)).sum())))
    assert u.max() <= 2 and (~np.isfinite(want)).any()


@pytest.mark.parametrize("gt_stride", [4, 5])
def test_bbox_transform_gt_stride(tops, gt_stride):
    rng = np.random.default_rng(gt_stride)
    ex = _random_gt(rng, 333, 600, 1000)[:, :4].copy()
    gt = _random_gt(rng, 333, 600, 1000)[:, :gt_stride].copy()
    ex[:3] = [[0, 0, 0, 0], [5.5, 2.25, 9.75, 4.5], [0, 0, 1e6, 1e6]]
    got = tops.bbox_transform(_dev(ex), _dev(gt)).cpu().numpy()
    want = orc.bbox_transform(ex, gt[:, :4])
    assert np.array_equal(got[:, :2], want[:, :2])                                # the same float32 operations
    assert _ulp(got[:, 2:], want[:, 2:]).max() <= 2                               # logf


def test_keep_inside_boundaries(tops):
    im_h, im_w = 600, 1000
    inf = np.inf
    xs = [im_w - 1, im_w - 0.5, np.nextafter(f32(im_w), f32(0)), im_w, im_w + 0.5, inf, -inf]
    rows = [[0, 0, x, 10] for x in xs] + [[0, 0, 10, y] for y in [im_h - 1, im_h - 0.5, im_h, inf, -inf]]
    rows += [[-0.0, -0.0, 5, 5], [-0.0, 0, 5, 5], [0, -0.0, 5, 5], [np.nextafter(f32(0), f32(-1)), 0, 5, 5], [-inf, 0, 5, 5],
             [inf, 0, 5, 5], [0, inf, 5, 5], [0, -inf, 5, 5]]
    boxes = np.array(rows * 37, f32)                                               # 37 * 20 rows: not a multiple of 256
    got = tops.keep_inside_flags(_dev(boxes), im_h, im_w).cpu().numpy()
    want = np.zeros(len(boxes), np.uint8)
    want[orc.keep_inside(boxes, (im_h, im_w))[0]] = 1
    assert np.array_equal(got, want)
    assert want[:12].tolist() == [1, 1, 1, 0, 0, 0, 1, 1, 1, 0, 0, 1] and want[12:16].tolist() == [1, 1, 1, 0]


def test_bbox_overlaps_touching_half_pixel_identical(tops):
    b = np.array([[0, 0, 9, 9], [10, 0, 19, 9], [0, 10, 9, 19], [0.5, 0.5, 9.5, 9.5], [4.5, 0, 14.5, 9], [0, 0, 9, 9],
                  [3, 3, 3, 3], [2.25, 7.75, 30.5, 8.25]], f64)
    rng = np.random.default_rng(2)
    extra = np.floor(rng.uniform(0, 40, (29, 2))) / 2
    extra = np.hstack([extra, extra + np.floor(rng.uniform(0, 20, (29, 2))) / 2])
    boxes = np.vstack([b, extra])                                                  # 37 boxes
    q = np.vstack([b, extra[:21]])                                                 # 29 queries: 37*29 = 1073 pairs
    got = tops.bbox_overlaps(_dev(boxes), _dev(q)).cpu().numpy()
    want = orc.bbox_overlaps(boxes, q)
    assert np.array_equal(got, want)
    assert got[0, 1] == 0 and got[0, 2] == 0                                       # touching: iw == 0 under the +1 rule
    assert got[0, 5] == 1.0 and (np.diag(got[:8, :8]) == 1.0).all()                # identical boxes: exactly 1
    assert 0 < got[0, 3] < 1 and 0 < got[0, 4] < 1
