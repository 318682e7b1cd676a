"""GPU tests of the float32 decode arithmetic against the CPU oracle where such kernels go wrong: every float32 input of
det_expf, and deltas, logits, scores and boxes that are NaN, infinite, huge, subnormal, signed zeros or on the exp clamps.

Kernels: bbox_decode_kernel (frcnn_bbox_decode: decode, clip, min-size flags), head_decode_kernel (frcnn_head_decode and
frcnn_head_decode_batch: class softmax, decode, clip) and rpn_decode_kernel (frcnn_proposals and frcnn_proposals_batch,
planar probabilities and NHWC logits), and after them the per-class NMS (frcnn_detect) and the ProposalLayer's sort and
NMS, fed the decoded rows.  The claim under test is DESIGN §2's: every float is bit-identical to the oracle.
"""
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import frcnn_oracle as orc

pytestmark = pytest.mark.gpu
f32 = np.float32
A = 9
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def assert_f32_equal(got, want, what, zero_sign=False):
    """float32 arrays equal bit for bit, with two exceptions.

    NaN is compared by position only: the device's arithmetic makes the canonical NaN and x86 makes 0xFFC00000, and
    which operand's payload survives an operation differs between the two.  With `zero_sign` (clipped coordinates),
    +0.0 and -0.0 compare equal: NumPy's maximum returns a zero's sign depending on its SIMD path (one build gave -0.0
    for np.maximum(+0.0, -0.0) and +0.0 for np.maximum(-0.0, 0)), so the oracle's sign of a clipped zero is not a
    property of clip_boxes.
    """
    g = np.ascontiguousarray(got, dtype=f32)
    w = np.ascontiguousarray(want, dtype=f32)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    gn, wn = np.isnan(g), np.isnan(w)
    bad = (gn != wn) | (~gn & (g.view(np.uint32) != w.view(np.uint32)))
    if zero_sign:
        bad &= ~((g == 0) & (w == 0))
    if bad.any():
        at = np.argwhere(bad)[:6]
        show = ["%s: got %08x want %08x" % (tuple(int(i) for i in ix), g.view(np.uint32)[tuple(ix)],
                                            w.view(np.uint32)[tuple(ix)]) for ix in at]
        raise AssertionError("%s: %d of %d values differ; %s" % (what, int(bad.sum()), bad.size, "; ".join(show)))


@pytest.fixture(scope="module")
def ops():
    from frcnn_b200 import ops as _ops
    return _ops


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(*u):
    return np.array(u, np.uint32).view(f32)


QNAN, NQNAN = _bits(0x7FC00000, 0xFFC00000)
TINY = _bits(1)[0]                                       # smallest subnormal
# Deltas (and logits, scores, coordinates): signed zeros, subnormals, ordinary values, det_expf's subnormal and zero
# thresholds (-87.33655 = ln 2^-126; -103.97208 / -103.972084 straddle ln 2^-150) and its -104 clamp, the band where
# 2 exp(v) overflows (from 88.03), exp's overflow point (88.72283 finite, 88.72284 inf), the 88.8 clamp, huge and
# infinite values, and NaN of both signs.
EDGE_VALUES = np.concatenate([
    np.array([0.0, -0.0, TINY, -TINY, 1e-30, -1e-30, 0.5, -0.5, 1, -1, 4.135, -4.135, 60, -60,
              -87.33655, -103.97208, -103.972084, -104, -104.1, 88.02, 88.72283, 88.72284, 88.8, 88.81, 100,
              1e30, -1e30, 3.4e38, -3.4e38, np.inf, -np.inf], f32),
    np.array([QNAN, NQNAN], f32)])
EDGE_BOXES = np.array([
    [10, 20, 110, 220],                  # ordinary
    [0.25, 3.5, 47.75, 15.125],          # ordinary, fractional
    [50, 60, 49, 59],                    # zero width and height: x2 = x1 - 1
    [300, 400, 120, 150],                # inverted
    [-1e30, -1e30, 1e30, 1e30],          # huge
    [1e30, 1e30, -1e30, -1e30],          # huge, inverted
    [-0.0, 0.0, -0.0, 0.0],              # signed zeros
    [0.0, -0.0, -1.0, -1.0],             # signed zeros, zero width
    [2000, 1500, 2100, 1600],            # right of and below a 600 x 1000 image
    [-300, -200, -100, -50],             # left of and above it
], f32)


def _value_matrix(K, seed=0):
    """(boxes [N,4], trans [N,4K]): every (dx, dw) pair of EDGE_VALUES with dy, dh drawn from them, on every EDGE_BOXES
    box (K = 1), or the same 4-tuples 21 to a row on the boxes in turn (K = 21)."""
    rng = np.random.default_rng(seed)
    V = EDGE_VALUES
    ix, iw = np.meshgrid(np.arange(len(V)), np.arange(len(V)), indexing="ij")
    n = ix.size
    d = np.stack([V[ix.ravel()], V[rng.integers(0, len(V), n)], V[iw.ravel()], V[rng.integers(0, len(V), n)]], 1)
    nb = len(EDGE_BOXES)
    if K == 1:
        return np.repeat(EDGE_BOXES, n, axis=0), np.tile(d, (nb, 1))
    d = np.tile(d, (nb, 1))
    rows = -(-len(d) // K)
    d = np.concatenate([d, np.zeros((rows * K - len(d), 4), f32)]).reshape(rows, 4 * K)
    return EDGE_BOXES[np.arange(rows) % nb], d


def _ok_flags(boxes, min_size):
    flags = np.zeros(len(boxes), np.uint8)
    flags[orc.filter_boxes(boxes, min_size)] = 1
    return flags


# ------------------------------------------------------------------------------------------------ a. every exp input
CHUNK = 1 << 24


def _check_exp_slice(got, start, lo, hi):
    """Rows [lo, hi) of a chunk whose row i decoded the bit pattern start + i as (dw, dh) on the box (-1, -0.5, 0, -0.5):
    bw = 2, bh = 1, cx = cy = 0, so x2 = 0 + 0.5 (2 e) and y2 = 0 + 0.5 e with e = orc_expf(v), each step exact while
    2 e is finite resp. e >= 2^-125."""
    v = np.arange(start + lo, start + hi, dtype=np.uint64).astype(np.uint32).view(f32)
    e = orc.expf(v)
    g = got[lo:hi]
    half, zero = f32(0.5), f32(0)
    with np.errstate(over="ignore", invalid="ignore"):
        pw, ph = e * f32(2), e * f32(1)
        want = np.stack([zero - half * pw, zero - half * ph, zero + half * pw, zero + half * ph], 1)
    assert_f32_equal(g, want, "bbox_decode of patterns %#x + [%d, %d)" % (start, lo, hi))
    # the same, stated on orc_expf itself: x2 = e wherever 2 e is finite (below ~88.03), y2 = e / 2 wherever e >= 2^-125;
    # between them they cover every input but NaN
    fin = np.isfinite(pw)
    big = e >= f32(2.0 ** -125)
    assert np.array_equal(g[fin, 2].view(np.uint32), e[fin].view(np.uint32))
    assert np.array_equal(g[big, 3].view(np.uint32), (e[big] * half).view(np.uint32))
    assert (fin | big | np.isnan(v)).all()
    return hi - lo


def test_every_exp_input(ops):
    """All 2^32 float32 bit patterns through det_expf in bbox_decode_kernel, each compared with orc_expf (NaN, +-inf,
    subnormal results and both clamps included).  On the way, the oracle's own accuracy claim, < 2 ulp from the
    correctly rounded exp on [-87, 88], is checked on every float in that interval against a float64 exp."""
    t0 = time.time()
    box = torch.tensor([-1.0, -0.5, 0.0, -0.5], device="cuda").expand(CHUNK, 4).contiguous()
    trans = torch.zeros((CHUNK, 4), dtype=torch.float32, device="cuda")
    nthreads = os.cpu_count() or 1
    slices = [(k * CHUNK // nthreads, (k + 1) * CHUNK // nthreads) for k in range(nthreads)]
    box_np = np.tile(np.array([[-1.0, -0.5, 0.0, -0.5]], f32), (CHUNK, 1))
    seen, in_range, worst = 0, 0, 0.0
    with ThreadPoolExecutor(nthreads) as pool:
        for c in range((1 << 32) // CHUNK):
            start = c * CHUNK
            base = start if start < 1 << 31 else start - (1 << 32)        # the same 32 bits as a signed int
            v = torch.arange(base, base + CHUNK, dtype=torch.int64, device="cuda").to(torch.int32).view(torch.float32)
            trans[:, 2] = v
            trans[:, 3] = v
            out, _ = ops.bbox_decode(box, trans)
            sel = (v >= -87.0) & (v <= 88.0)
            n_sel = int(sel.sum().item())
            if n_sel:
                ref = torch.exp(v[sel].double())
                r32 = ref.float()
                ulp = (torch.nextafter(r32, torch.full_like(r32, float("inf"))) - r32).double()
                worst = max(worst, ((out[:, 2][sel].double() - ref).abs() / ulp).max().item())
                in_range += n_sel
            got = out.cpu().numpy()
            seen += sum(pool.map(lambda s: _check_exp_slice(got, start, *s), slices))
            if c % 64 == 0:            # tie the restatement above to the oracle's bbox_transform_inv
                tr = np.zeros((CHUNK, 4), f32)
                tr[:, 2] = tr[:, 3] = np.arange(start, start + CHUNK, dtype=np.uint64).astype(np.uint32).view(f32)
                assert_f32_equal(got, orc.bbox_transform_inv(box_np, tr), "orc.bbox_transform_inv chunk %d" % c)
    assert seen == 1 << 32
    # [0, 88] and [-87, -0] as bit patterns
    assert in_range == (int(f32(88.0).view(np.uint32)) + 1) + (int(f32(-87.0).view(np.uint32)) - 0x80000000 + 1)
    assert worst < 2.0, worst
    print("every exp input: %d patterns, max error on [-87, 88] %.4f ulp, %.1f s on %d threads"
          % (seen, worst, time.time() - t0, nthreads))


# ------------------------------------------------------------------------------------------------ b. frcnn_bbox_decode
@pytest.mark.parametrize("K", [1, 21])
@pytest.mark.parametrize("clip", [None, (600, 1000), (1, 1)], ids=["noclip", "600x1000", "1x1"])
def test_bbox_decode_value_matrix(ops, K, clip):
    """Decode (and clip) of the value matrix: bit-exact against orc.bbox_transform_inv (+ orc.clip_boxes); with K = 1 the
    min-size flags at 0, 1 and 16 equal orc.filter_boxes (a NaN box fails every min size)."""
    boxes, trans = _value_matrix(K)
    with np.errstate(over="ignore", invalid="ignore"):
        want = orc.bbox_transform_inv(boxes, trans)
        if clip is not None:
            want = orc.clip_boxes(want, clip)
        for m in (0, 1, 16) if K == 1 else (None,):
            out, flags = ops.bbox_decode(dev(boxes), dev(trans), clip_to=clip, min_size=m)
            assert_f32_equal(out.cpu().numpy(), want, "bbox_decode K=%d clip=%s" % (K, clip), zero_sign=clip is not None)
            if m is not None:
                assert np.array_equal(flags.cpu().numpy(), _ok_flags(want, m)), m


@pytest.mark.parametrize("K", [1, 21])
@pytest.mark.parametrize("clip", [(600, 1000), (1, 1)], ids=["600x1000", "1x1"])
def test_clip_only_value_matrix(ops, K, clip):
    """trans = NULL (clip and flags only) on unclipped decodes of the value matrix and on boxes whose coordinates are the
    edge values themselves: equal to orc.clip_boxes, flags to orc.filter_boxes."""
    boxes, trans = _value_matrix(K, seed=1)
    V = EDGE_VALUES
    a, b = np.meshgrid(V, V, indexing="ij")
    raw = np.stack([a.ravel(), b.ravel(), b.ravel(), a.ravel()], 1)
    raw = np.concatenate([raw, np.zeros((-len(raw) % K, 4), f32)]).reshape(-1, 4 * K)
    with np.errstate(over="ignore", invalid="ignore"):
        inp = np.concatenate([orc.bbox_transform_inv(boxes, trans), raw])
        want = orc.clip_boxes(inp.copy(), clip)
        for m in (0, 1, 16) if K == 1 else (None,):
            out, flags = ops.bbox_decode(dev(inp), None, clip_to=clip, min_size=m)
            assert_f32_equal(out.cpu().numpy(), want, "clip only K=%d clip=%s" % (K, clip), zero_sign=True)
            if m is not None:
                assert np.array_equal(flags.cpu().numpy(), _ok_flags(want, m)), m


# ------------------------------------------------------------------------------------------------ c. head decode, detect
R_CAP = 300
NAN_CLASS_ROWS = 6          # rows of one class with NaN dx on one roi: NaN boxes, which suppress nothing


def _special_logit_rows(rng, NC):
    """One row of NC logits per kind: all equal, one +inf, one -inf, all -inf, a NaN of each sign, a spread above 104
    (every exp but the row maximum's underflows), +-3e38, mixed +-0.0, and edge values."""
    ar = np.arange(NC)

    def base():
        return (rng.standard_normal(NC) * 2).astype(f32)

    rows = [np.full(NC, 0.75, f32), np.full(NC, -np.inf, f32)]
    for pos, val in ((1, np.inf), (2, -np.inf), (3, QNAN), (0, NQNAN)):
        r = base()
        r[pos % NC] = val
        rows.append(r)
    r = (-105.0 - 7.0 * ar).astype(f32)
    r[NC // 2] = 20.0
    rows.append(r)
    rows.append(np.where(ar % 2 == 1, f32(3e38), f32(-3e38)).astype(f32))
    rows.append(np.where(ar % 3 == 0, f32(0.0), f32(-0.0)).astype(f32))
    rows.append(EDGE_VALUES[rng.integers(0, len(EDGE_VALUES), NC)])
    rows.append(-np.abs(EDGE_VALUES[rng.integers(0, 19, NC)]))
    return np.stack(rows)


def _head_inputs(NC, ld, special, seed):
    """scores | deltas [R_CAP, ld] and rois [R_CAP, 4].  special: the special logit rows first, deltas with 30% edge
    values, the edge boxes among the rois, and NAN_CLASS_ROWS rows of class min(1, NC-1) with NaN dx on one roi."""
    rng = np.random.default_rng(seed)
    mat = np.zeros((R_CAP, ld), f32)
    mat[:, :NC] = rng.standard_normal((R_CAP, NC)) * 2
    deltas = (rng.standard_normal((R_CAP, 4 * NC)) * 0.3).astype(f32)
    xy = rng.uniform(-50, 900, size=(R_CAP, 2))
    rois = np.hstack([xy, xy + rng.uniform(-5, 300, size=(R_CAP, 2))]).astype(f32)
    if special:
        sp = _special_logit_rows(rng, NC)
        mat[:len(sp), :NC] = sp
        pick = rng.random(deltas.shape) < 0.3
        deltas[pick] = EDGE_VALUES[rng.integers(0, len(EDGE_VALUES), int(pick.sum()))]
        rois[1:1 + 2 * len(EDGE_BOXES):2] = EDGE_BOXES
        c = min(1, NC - 1)
        lo = len(sp) + 2 * len(EDGE_BOXES) + 3
        rows = slice(lo, lo + NAN_CLASS_ROWS)
        mat[rows, :NC] = 0.0
        mat[rows, c] = 3.0                                  # ordinary, equal probabilities
        deltas[rows] = (rng.standard_normal((NAN_CLASS_ROWS, 4 * NC)) * 0.1).astype(f32)
        deltas[rows, 4 * c] = QNAN
        rois[rows] = rois[lo]
    mat[:, NC:5 * NC] = deltas
    return mat, rois


def _want_head(mat, rois, NC, R, im):
    with np.errstate(over="ignore", invalid="ignore"):
        p = orc.softmax_axis1(mat[:R, :NC])
        b = orc.clip_boxes(orc.bbox_transform_inv(rois[:R], mat[:R, NC:5 * NC]), im)
    return p, b


def _check_head(p, b, want_p, want_b, R, what):
    assert_f32_equal(p[:R], want_p, what + " prob")
    assert_f32_equal(b[:R], want_b, what + " boxes", zero_sign=True)
    assert not p[R:].view(np.uint32).any() and not b[R:].view(np.uint32).any(), what + ": rows past the count"


def _check_detect(keep_idx, keep_count, conf_count, want_p, want_b, conf, what):
    for c, keep_conf, _ in orc.detect(want_p, want_b, nms_thresh=0.3, conf=conf):
        dets = np.hstack((want_b[:, 4 * c:4 * c + 4], want_p[:, c:c + 1])).astype(f32)
        keep = orc.cpu_nms(dets, 0.3)
        n = int(keep_count[c - 1])
        assert keep_idx[c - 1, :n].tolist() == keep, (what, c)
        assert int(conf_count[c - 1]) == len(keep_conf), (what, c)
        assert keep_idx[c - 1, :len(keep_conf)].tolist() == keep_conf.tolist(), (what, c)


HEAD_CASES = [(1, 128), (2, 128), (21, 128), (81, 408)]


@pytest.mark.parametrize("count", ["zero", "one", "ragged", "full"])
@pytest.mark.parametrize("NC,ld", HEAD_CASES, ids=["nc1", "nc2", "nc21", "nc81"])
def test_head_decode_and_detect_edges(ops, NC, ld, count):
    """head_decode on the special logit rows, edge-value deltas and edge boxes: softmax bit-exact against
    orc.softmax_axis1, boxes against orc.clip_boxes(orc.bbox_transform_inv), zeros past the count; then the decoded
    rows through frcnn_detect against orc.detect, NaN boxes of one class included."""
    R = {"zero": 0, "one": 1, "ragged": R_CAP - 37, "full": R_CAP}[count]
    im = (600, 1000)
    mat, rois = _head_inputs(NC, ld, True, seed=NC)
    want_p, want_b = _want_head(mat, rois, NC, R, im)
    cnt = dev(np.array([R], np.int32))
    p, b = ops.head_decode(dev(mat), ld, dev(rois), cnt, NC, im[0], im[1])
    _check_head(p.cpu().numpy(), b.cpu().numpy(), want_p, want_b, R, "head_decode NC=%d R=%d" % (NC, R))
    if NC >= 2:
        conf = 0.05
        keep_idx, keep_count, conf_count = ops.detect(p, b, cnt, nms_thresh=0.3, conf=conf)
        _check_detect(keep_idx.cpu().numpy(), keep_count.cpu().numpy(), conf_count.cpu().numpy(), want_p, want_b, conf,
                      "detect NC=%d R=%d" % (NC, R))


@pytest.mark.parametrize("NC,ld", HEAD_CASES, ids=["nc1", "nc2", "nc21", "nc81"])
def test_head_decode_batch_edges(ops, NC, ld):
    """head_decode_batch and detect_batch at N = 2, an ordinary image 0 and the special image 1 (ragged count), each
    image against the oracle."""
    im = (600, 1000)
    ins = [_head_inputs(NC, ld, False, seed=100 + NC), _head_inputs(NC, ld, True, seed=NC)]
    Rs = [R_CAP, R_CAP - 37]
    mat = dev(np.stack([m for m, _ in ins]))
    rois = dev(np.stack([r for _, r in ins]))
    counts = dev(np.array(Rs, np.int32))
    p, b = ops.head_decode_batch(mat, ld, rois, counts, NC, im[0], im[1])
    det = ops.detect_batch(p, b, counts, nms_thresh=0.3, conf=0.05) if NC >= 2 else None
    p, b = p.cpu().numpy(), b.cpu().numpy()
    for n, ((m, r), R) in enumerate(zip(ins, Rs)):
        want_p, want_b = _want_head(m, r, NC, R, im)
        _check_head(p[n], b[n], want_p, want_b, R, "head_decode_batch image %d NC=%d" % (n, NC))
        if det is not None:
            _check_detect(*(t[n].cpu().numpy() for t in det), want_p, want_b, 0.05, "detect_batch image %d" % n)


# ------------------------------------------------------------------------------------------------ d. ProposalLayer
H, W = 30, 60                # 16,200 anchors
IM = (H * 16, W * 16)
PRE = 16384                  # above the anchor count: every survivor of the min-size test is in the debug lists
SCORE_SPECIALS = np.concatenate([np.array([QNAN, NQNAN], f32),
                                 np.array([np.inf, -np.inf, 0.0, -0.0, TINY, -TINY, 2.0 ** -140, 1e-30], f32)])


def _rpn_inputs(seed, special, nan_share=0.0):
    """prob (1,18,H,W) on 32 levels (ties), deltas (1,36,H,W) N(0, 0.2) and logits (1,18,H,W) N(0, 2).  special: 20% of
    the deltas from EDGE_VALUES, 10% of the probabilities from SCORE_SPECIALS (NaN of both signs, +-inf, +-0.0,
    subnormals), every 7th pixel's logits one of the special logit rows; nan_share: that share of fg scores NaN."""
    rng = np.random.default_rng(seed)
    prob = (rng.integers(0, 32, size=(1, 2 * A, H, W)) / 32.0).astype(f32)
    pred = (rng.standard_normal((1, 4 * A, H, W)) * 0.2).astype(f32)
    logits = (rng.standard_normal((1, 2 * A, H, W)) * 2).astype(f32)
    if special:
        pick = rng.random(pred.shape) < 0.2
        pred[pick] = EDGE_VALUES[rng.integers(0, len(EDGE_VALUES), int(pick.sum()))]
        pick = rng.random(prob.shape) < 0.1
        prob[pick] = SCORE_SPECIALS[rng.integers(0, len(SCORE_SPECIALS), int(pick.sum()))]
        sp = _special_logit_rows(rng, 2 * A)
        flat = logits[0].reshape(2 * A, -1)
        for k, pix in enumerate(range(0, H * W, 7)):
            flat[:, pix] = sp[k % len(sp)]
    if nan_share:
        pick = rng.random((A, H, W)) < nan_share
        prob[0, A:][pick] = np.where(rng.random(int(pick.sum())) < 0.5, QNAN, NQNAN)
    return prob, pred, logits


def _nhwc(logits, pred, ld=64):
    mat = np.zeros((H * W, ld), f32)
    mat[:, :2 * A] = logits[0].reshape(2 * A, -1).T
    mat[:, 2 * A:6 * A] = pred[0].reshape(4 * A, -1).T
    return mat


def _want_proposals(prob, pred, min_size, post):
    dbg = {}
    with np.errstate(over="ignore", invalid="ignore"):
        rois, fg = orc.proposal_layer(prob, pred, IM, anchors=ANCHORS, pre_nms_top_n=PRE, post_nms_top_n=post,
                                      nms_thresh=0.7, min_size=min_size, debug=dbg)
    return rois, fg.ravel(), dbg


def _check_proposals(rois, scores, count, dbg_dets, dbg_idx, dbg_num, want, what):
    want_rois, want_fg, dbg = want
    assert dbg_num == len(dbg["dets"]), what
    assert np.array_equal(dbg_idx[:dbg_num], dbg["anchor_index"]), what
    assert_f32_equal(dbg_dets[:dbg_num, :4], dbg["dets"][:, :4], what + " dbg boxes", zero_sign=True)
    assert_f32_equal(dbg_dets[:dbg_num, 4], dbg["dets"][:, 4], what + " dbg scores")
    assert count == len(want_rois), what
    assert_f32_equal(rois[:count], want_rois, what + " rois", zero_sign=True)
    assert_f32_equal(scores[:count], want_fg, what + " scores")


def _run_proposals(ops, form, prob, pred, logits, min_size, post):
    """The one-image entry on one image; returns the host outputs."""
    anchors = dev(ANCHORS)
    if form == "probs":
        w = ops.proposals(dev(prob[0]), dev(pred[0]), anchors, A, H, W, 16, IM[0], IM[1], min_size, PRE, post, 0.7,
                          debug=True)
    else:
        w = ops.proposals(dev(_nhwc(logits, pred)), None, anchors, A, H, W, 16, IM[0], IM[1], min_size, PRE, post, 0.7,
                          layout="nhwc", ld=64, cls_is_logits=True, debug=True)
    return (w.rois.cpu().numpy(), w.scores.cpu().numpy(), int(w.count.item()), w.dbg_dets.cpu().numpy(),
            w.dbg_idx.cpu().numpy(), int(w.dbg_num.item()))


def _oracle_prob(form, prob, logits):
    with np.errstate(over="ignore", invalid="ignore"):
        return prob if form == "probs" else orc.softmax_axis1(logits)


CASES = [("probs", 0, 300, 0.0), ("probs", 1, 300, 0.0), ("probs", 16, 300, 0.0), ("probs", 16, 2000, 0.95),
         ("logits", 0, 300, 0.0), ("logits", 1, 300, 0.0), ("logits", 16, 300, 0.0)]
CASE_IDS = ["probs-min0", "probs-min1", "probs-min16", "probs-min16-nan95", "logits-min0", "logits-min1", "logits-min16"]


@pytest.mark.parametrize("form,min_size,post,nan_share", CASES, ids=CASE_IDS)
def test_proposal_layer_edges(ops, form, min_size, post, nan_share):
    """frcnn_proposals on edge-value deltas and special scores (planar probabilities) or special logit rows (NHWC,
    softmax on device): debug lists, rois, scores and count against orc.proposal_layer.  NaN-score anchors stay, ranked
    after every number; in the 95%-NaN case fewer finite rows survive than post_nms_top_n, so NaN rows fill the rest."""
    prob, pred, logits = _rpn_inputs(seed=7 + min_size, special=True, nan_share=nan_share)
    want = _want_proposals(_oracle_prob(form, prob, logits), pred, min_size, post)
    got = _run_proposals(ops, form, prob, pred, logits, min_size, post)
    _check_proposals(*got, want, "proposals %s min_size=%d" % (form, min_size))
    assert np.isnan(want[2]["dets"][:, 4]).any()           # NaN-score rows survive the min-size test
    if nan_share:
        assert np.isnan(want[1]).any() and want[0].shape[0] <= post


@pytest.mark.parametrize("form,min_size,post,nan_share", CASES, ids=CASE_IDS)
def test_proposals_batch_edges(ops, form, min_size, post, nan_share):
    """frcnn_proposals_batch at N = 2: an ordinary image 0 and the special image 1, each against orc.proposal_layer."""
    imgs = [_rpn_inputs(seed=50 + min_size, special=False),
            _rpn_inputs(seed=7 + min_size, special=True, nan_share=nan_share)]
    anchors = dev(ANCHORS)
    if form == "probs":
        cls = dev(np.concatenate([p for p, _, _ in imgs]))
        bbox = dev(np.concatenate([d for _, d, _ in imgs]))
        w = ops.proposals_batch(cls, bbox, anchors, A, H, W, 16, IM[0], IM[1], min_size, PRE, post, 0.7, debug=True)
    else:
        mat = dev(np.stack([_nhwc(lg, d) for _, d, lg in imgs]))
        w = ops.proposals_batch(mat, None, anchors, A, H, W, 16, IM[0], IM[1], min_size, PRE, post, 0.7, layout="nhwc",
                                ld=64, cls_is_logits=True, debug=True)
    host = [t.cpu().numpy() for t in (w.rois, w.scores, w.count, w.dbg_dets, w.dbg_idx, w.dbg_num)]
    for n, (prob, pred, logits) in enumerate(imgs):
        want = _want_proposals(_oracle_prob(form, prob, logits), pred, min_size, post)
        _check_proposals(host[0][n], host[1][n], int(host[2][n]), host[3][n], host[4][n], int(host[5][n]), want,
                         "proposals_batch image %d %s min_size=%d" % (n, form, min_size))
