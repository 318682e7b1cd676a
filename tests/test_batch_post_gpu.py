"""GPU tests of the batched post-processing: frcnn_proposals_batch, frcnn_roi_pool_batch, frcnn_head_decode_batch,
frcnn_detect_batch, frcnn_maxpool2x2_ceil_batch, engine.BatchPlan on top of them, and the one-call batch forward
frcnn_forward_vgg16_batch.  Every image's outputs must be bit-identical (int32 views of the floats) to the one-image entry
point on that image, and nothing may be written between one image's outputs and the next: every per-image output block
below is followed by a run of sentinel words that must survive."""
import ctypes

import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_nms_paths_gpu import GENERATORS

pytestmark = pytest.mark.gpu
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
A = 9
SENTINEL = -12345
PAD = 40                  # sentinel words after every image's block (a multiple of 8: keeps 16-byte rows aligned)
_INT = {torch.float32: torch.int32, torch.int32: torch.int32, torch.bfloat16: torch.int16}


@pytest.fixture(scope="module")
def ops():
    from frcnn_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def params():
    return orc.make_params(seed=1234)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Padded(object):
    """N per-image blocks of `inner` elements, `stride` elements apart (default: PAD sentinel words after every block):
    .t is the [N, *inner] view."""

    def __init__(self, N, inner, dtype, stride=None):
        self.n = int(np.prod(inner))
        self.buf = torch.full((N, stride or self.n + PAD), SENTINEL, dtype=_INT[dtype], device="cuda")
        self.t = self.buf.view(dtype)[:, :self.n].view((N,) + tuple(inner))

    def intact(self):
        return bool((self.buf[:, self.n:] == SENTINEL).all().item())


def bits(t):
    return t.contiguous().view(_INT[t.dtype])


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


# ------------------------------------------------------------------------------------------------ proposals_batch
def _rpn_maps(N, H, W, seed, levels=16):
    """(N,18,H,W) probabilities on `levels` values, (N,36,H,W) small deltas, (N,H*W,64) NHWC rows of logits | deltas."""
    rng = np.random.default_rng(seed)
    prob = (rng.integers(0, levels, size=(N, 2 * A, H, W)) / float(levels)).astype(f32)
    pred = (rng.standard_normal((N, 4 * A, H, W)) * 0.1).astype(f32)
    logits = (rng.standard_normal((N, 2 * A, H, W)) * 2).astype(f32)
    return prob, pred, logits


def _special_images(prob, pred, logits):
    """Image 1: every box collapses below min_size (count 0).  Image 2: every score tied."""
    N = prob.shape[0]
    if N > 1:
        pred[1, 2::4] = -8.0
        pred[1, 3::4] = -8.0
    if N > 2:
        prob[2] = 0.5
        logits[2] = 0.25


def _nhwc(logits, pred, ld=64):
    N, _, H, W = logits.shape
    mat = np.zeros((N, H * W, ld), f32)
    mat[:, :, :2 * A] = logits.reshape(N, 2 * A, -1).transpose(0, 2, 1)
    mat[:, :, 2 * A:6 * A] = pred.reshape(N, 4 * A, -1).transpose(0, 2, 1)
    return mat


def _proposals_padded(ops, N, H, W, pre, post):
    k = min(pre, A * H * W)
    outs = dict(rois=Padded(N, (post, 4), torch.float32), scores=Padded(N, (post,), torch.float32),
                count=Padded(N, (1,), torch.int32), dets=Padded(N, (k, 5), torch.float32), idx=Padded(N, (k,), torch.int32),
                num=Padded(N, (1,), torch.int32))
    work = ops.ProposalBatchWorkspace(N, A, H, W, pre, post, "cuda", debug=True,
                                      outputs=(outs["rois"].t, outs["scores"].t, outs["count"].t[:, 0]))
    work.dbg_dets, work.dbg_idx, work.dbg_num = outs["dets"].t, outs["idx"].t, outs["num"].t[:, 0]
    return work, outs


def _check_proposals(ops, layout, prob, pred, logits, im, pre, post, thr=0.7):
    N, _, H, W = prob.shape
    anchors = dev(ANCHORS)
    work, outs = _proposals_padded(ops, N, H, W, pre, post)
    if layout == "nchw":
        cls_b, bbox_b = dev(prob), dev(pred)
        ops.proposals_batch(cls_b, bbox_b, anchors, A, H, W, 16, im[0], im[1], 16, pre, post, thr, work=work, debug=True)
    else:
        mat = dev(_nhwc(logits, pred))
        ops.proposals_batch(mat, None, anchors, A, H, W, 16, im[0], im[1], 16, pre, post, thr, layout="nhwc", ld=64,
                            cls_is_logits=True, work=work, debug=True)
    torch.cuda.synchronize()
    counts = []
    for n in range(N):
        if layout == "nchw":
            one = ops.proposals(cls_b[n], bbox_b[n], anchors, A, H, W, 16, im[0], im[1], 16, pre, post, thr, debug=True)
        else:
            one = ops.proposals(mat[n], None, anchors, A, H, W, 16, im[0], im[1], 16, pre, post, thr, layout="nhwc", ld=64,
                                cls_is_logits=True, debug=True)
        torch.cuda.synchronize()
        assert same(work.rois[n], one.rois) and same(work.scores[n], one.scores), n
        assert int(work.count[n]) == int(one.count.item()), n
        ns = int(one.dbg_num.item())           # the debug lists hold dbg_num entries; the rest is not written
        assert int(work.dbg_num[n]) == ns, n
        assert same(work.dbg_dets[n, :ns], one.dbg_dets[:ns]) and same(work.dbg_idx[n, :ns], one.dbg_idx[:ns]), n
        counts.append(int(one.count.item()))
    for name, p in outs.items():
        assert p.intact(), name
    return counts


@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("N", [1, 2, 3, 5])
def test_proposals_batch_small_ragged_maps(ops, N, layout):
    """Small odd maps (the pre_nms_top_n cut falls inside tie groups of the 16 score levels); image 1 keeps no box,
    image 2 has every score tied."""
    H, W = 7 + N, 11 + 2 * N
    prob, pred, logits = _rpn_maps(N, H, W, seed=N)
    _special_images(prob, pred, logits)
    counts = _check_proposals(ops, layout, prob, pred, logits, (H * 16, W * 16), 600, 100)
    if N > 1:
        assert counts[1] == 0
    assert counts[0] > 0


@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
@pytest.mark.parametrize("pre,post", [(6000, 300), (12000, 2000)], ids=["test", "train"])
def test_proposals_batch_600x1000(ops, pre, post, layout):
    """N = 4 on the 38 x 63 map of a 600 x 1000 image, test mode (keys in shared memory) and train mode (keys in global
    memory, cut inside a tie group); one image without proposals and one with every score tied."""
    prob, pred, logits = _rpn_maps(4, 38, 63, seed=11)
    _special_images(prob, pred, logits)
    counts = _check_proposals(ops, layout, prob, pred, logits, (600, 1000), pre, post)
    assert counts[1] == 0 and min(counts[0], counts[2], counts[3]) > 0


def test_proposals_batch_into_result_blocks(ops):
    """Outputs written straight into BatchPlan-style result blocks (count, rois, scores at their offsets, block_words
    apart): equal to ForwardPlan-style per-image calls, and every other word of the blocks untouched."""
    from frcnn_b200.engine import _result_layout
    N, H, W, pre, post = 3, 38, 63, 6000, 300
    L, bw = _result_layout(post, 21)
    res = torch.full((N, bw), SENTINEL, dtype=torch.int32, device="cuda")
    rf = res.view(torch.float32)
    seg = lambda t, name: t[:, L[name][0]:L[name][0] + L[name][1]]      # noqa: E731
    work = ops.ProposalBatchWorkspace(N, A, H, W, pre, post, "cuda",
                                      outputs=(seg(rf, "rois").view(N, post, 4), seg(rf, "scores"), seg(res, "count")[:, 0]))
    prob, pred, logits = _rpn_maps(N, H, W, seed=21)
    mat = dev(_nhwc(logits, pred))
    ops.proposals_batch(mat, None, dev(ANCHORS), A, H, W, 16, 600, 1000, 16, pre, post, 0.7, layout="nhwc", ld=64,
                        cls_is_logits=True, work=work)
    torch.cuda.synchronize()
    written = torch.zeros(bw, dtype=torch.bool, device="cuda")
    for name in ("rois", "scores"):
        written[L[name][0]:L[name][0] + L[name][1]] = True
    written[L["count"][0]] = True
    assert bool((res[:, ~written] == SENTINEL).all().item())
    for n in range(N):
        one = ops.proposals(mat[n], None, dev(ANCHORS), A, H, W, 16, 600, 1000, 16, pre, post, 0.7, layout="nhwc", ld=64,
                            cls_is_logits=True)
        assert same(work.rois[n], one.rois) and same(work.scores[n], one.scores)
        assert int(res[n, L["count"][0]]) == int(one.count.item()) > 0


# ------------------------------------------------------------------------------------------------ roi_pool_batch
def _feat(N, H, W, C, x3, seed):
    g = torch.Generator().manual_seed(seed)
    v = torch.relu(torch.randn((N, H, W, C), generator=g)).cuda()
    hi = v.to(torch.bfloat16)
    return hi.contiguous(), ((v - hi.float()).to(torch.bfloat16).contiguous() if x3 else None)


def _rois(N, R_cap, H, W, seed):
    rng = np.random.default_rng(seed)
    x1 = rng.uniform(-40, W * 16, size=(N, R_cap))
    y1 = rng.uniform(-40, H * 16, size=(N, R_cap))
    w = rng.uniform(0, W * 12, size=(N, R_cap))
    h = rng.uniform(0, H * 12, size=(N, R_cap))
    return np.stack([x1, y1, x1 + w, y1 + h], axis=2).astype(f32)


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
@pytest.mark.parametrize("H,W,C,R_cap", [(19, 31, 512, 300), (9, 13, 2048, 40)])
def test_roi_pool_batch_equals_per_image(ops, H, W, C, R_cap, x3):
    """Counts 0, 1 and R_cap in one batch; bf16 and fp32 outputs at a padded image stride; C = 512 and 2048."""
    N, K = 3, 49 * C
    hi, lo = _feat(N, H, W, C, x3, seed=C + R_cap)
    feat = ops.Act(hi, lo)
    rois = Padded(N, (R_cap, 4), torch.float32)
    rois.t.copy_(dev(_rois(N, R_cap, H, W, seed=C)))
    cnt = Padded(N, (1,), torch.int32)
    cnt.t[:, 0] = torch.tensor([0, 1, R_cap], dtype=torch.int32, device="cuda")
    # one image stride (in elements) for the bf16 and fp32 outputs
    o32 = Padded(N, (R_cap, 49, C), torch.float32)
    oh = Padded(N, (R_cap, K), torch.bfloat16, stride=o32.n + PAD)
    ol = Padded(N, (R_cap, K), torch.bfloat16, stride=o32.n + PAD) if x3 else None
    out, y32 = ops.roi_pool_batch(feat, rois.t, cnt.t[:, 0], 7, 7, 1.0 / 16, out=ops.Act(oh.t, ol.t if x3 else None),
                                  out_f32=o32.t)
    torch.cuda.synchronize()
    for n in range(N):
        one, one32 = ops.roi_pool(ops.Act(hi[n], None if lo is None else lo[n]), rois.t[n], cnt.t[n], 7, 7, 1.0 / 16,
                                  want_f32=True)
        assert same(out.hi[n], one.hi[0]) and same(y32[n], one32), n
        if x3:
            assert same(out.lo[n], one.lo[0]), n
    assert not y32[0].any().item() and y32[2].any().item()
    for p in (rois, cnt, oh, o32) + ((ol,) if x3 else ()):
        assert p.intact()


# ------------------------------------------------------------------------------------------------ head decode, detect
def _head_inputs(N, R_cap, NC, seed, ld=128):
    rng = np.random.default_rng(seed)
    sd = np.zeros((N, R_cap, ld), f32)
    sd[:, :, :NC] = rng.integers(0, 4, size=(N, R_cap, NC)) * 0.5          # tied scores
    sd[:, ::7, 1] = np.nan                                                 # NaN rows
    sd[:, :, NC:5 * NC] = rng.standard_normal((N, R_cap, 4 * NC)) * 0.2
    return sd, _rois(N, R_cap, 38, 63, seed + 1)


@pytest.mark.parametrize("R_cap", [300, 2048])
def test_head_decode_batch_equals_per_image(ops, R_cap):
    """Counts 0 / 1 / R_cap, tied and NaN scores; outputs at a padded image stride."""
    N, NC, ld = 3, 21, 128
    sd, rois = _head_inputs(N, R_cap, NC, seed=R_cap)
    sd_t, rois_t = dev(sd), dev(rois)
    cnt = dev(np.array([0, 1, R_cap], np.int32))
    prob, boxes = Padded(N, (R_cap, NC), torch.float32), Padded(N, (R_cap, 4 * NC), torch.float32)
    ops.head_decode_batch(sd_t, ld, rois_t, cnt, NC, 600, 1000, out_prob=prob.t, out_boxes=boxes.t)
    torch.cuda.synchronize()
    for n in range(N):
        p1, b1 = ops.head_decode(sd_t[n], ld, rois_t[n], cnt[n:n + 1], NC, 600, 1000)
        assert same(prob.t[n], p1) and same(boxes.t[n], b1), n
    assert not prob.t[0].any().item() and prob.t[1, 0].any().item() and not prob.t[1, 1:].any().item()
    assert prob.intact() and boxes.intact()


def _detect_inputs(N, R_cap, NC, thr, seed):
    rng = np.random.default_rng(seed)
    gens = list(GENERATORS)
    prob = np.zeros((N, R_cap, NC), f32)
    boxes = np.zeros((N, R_cap, 4 * NC), f32)
    for n in range(N):
        for c in range(1, NC):
            d = GENERATORS[gens[(c + n + seed) % len(gens)]](R_cap, rng, thr)
            prob[n, :, c] = d[:, 4]
            boxes[n, :, 4 * c:4 * c + 4] = d[:, :4]
    return prob, boxes


@pytest.mark.parametrize("R_cap", [300, 1152, 1153, 2048])
def test_detect_batch_equals_per_image(ops, R_cap):
    """Counts 0 / 1 / R_cap on both sides of the detect_kernel / detect_barrier_kernel switch (1152 | 1153), every class a
    different input generator of test_nms_paths_gpu (ties, equal, signed zeros, NaN, threshold-exact IoUs, degenerate
    boxes); outputs at padded image strides."""
    N, NC, thr = 3, 21, 0.3
    prob, boxes = _detect_inputs(N, R_cap, NC, thr, seed=R_cap)
    prob_t, boxes_t = dev(prob), dev(boxes)
    cnt = dev(np.array([0, 1, R_cap], np.int32))
    ki, kc, cc = Padded(N, (NC - 1, R_cap), torch.int32), Padded(N, (NC - 1,), torch.int32), Padded(N, (NC - 1,), torch.int32)
    ops.detect_batch(prob_t, boxes_t, cnt, thr, 0.5, out=(ki.t, kc.t, cc.t))
    torch.cuda.synchronize()
    for n in range(N):
        k1, c1, f1 = ops.detect(prob_t[n], boxes_t[n], cnt[n:n + 1], thr, 0.5)
        assert same(ki.t[n], k1) and same(kc.t[n], c1) and same(cc.t[n], f1), n
    assert not kc.t[0].any().item() and bool((kc.t[1] == 1).all().item())
    assert ki.intact() and kc.intact() and cc.intact()


# ------------------------------------------------------------------------------------------------ maxpool
@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
@pytest.mark.parametrize("H,W", [(37, 63), (19, 32), (75, 125)])
def test_maxpool_batch_equals_per_image(ops, H, W, x3):
    N, C = 3, 64
    hi, lo = _feat(N, H, W, C, x3, seed=H * W)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    yh = Padded(1, (N, Ho, Wo, C), torch.bfloat16)
    yl = Padded(1, (N, Ho, Wo, C), torch.bfloat16) if x3 else None
    y = ops.maxpool2x2_ceil_batch(ops.Act(hi, lo), out=ops.Act(yh.t[0], yl.t[0] if x3 else None))
    torch.cuda.synchronize()
    for n in range(N):
        y1 = ops.maxpool2x2_ceil(ops.Act(hi[n], None if lo is None else lo[n]))
        assert same(y.hi[n], y1.hi) and (not x3 or same(y.lo[n], y1.lo)), n
    assert yh.intact() and (not x3 or yl.intact())


# ------------------------------------------------------------------------------------------------ BatchPlan
FIELDS = ("prob", "boxes", "rois", "scores", "keep_count", "conf_count", "keep_idx")


def _images(N, H, W, seed):
    return torch.from_numpy(np.stack([orc.make_image(H, W, seed=seed + n)[0] for n in range(N)]).astype(f32)).cuda()


def _assert_same(got, want, what):
    assert got["count"] == want["count"], what
    for f in FIELDS:
        a, b = np.asarray(got[f]), np.asarray(want[f])
        assert a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32)), (what, f)


def _per_image(plan1, x):
    out = []
    for n in range(x.shape[0]):
        plan1.forward(x[n])
        torch.cuda.synchronize()
        r = plan1.unpack_result(plan1.result.cpu().numpy())
        out.append(({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in r.items()},
                    int(plan1.prop.dbg_num.item()), plan1.prop.dbg_dets.cpu().clone(), plan1.prop.dbg_idx.cpu().clone()))
    return out


def test_batch_plan_all_options_equals_forward_plan(params):
    """with_detect, keep_rpn_debug and fuse_pool=False (stand-alone batched max-pools): every image equals ForwardPlan
    with the same options, debug lists included; the post-processing launches do not grow with N; a graph replay with a
    second input set gives the second set's results."""
    from frcnn_b200.engine import BatchPlan, ForwardPlan, PackedWeights
    H, W, N = 150, 201, 3
    opts = dict(anchors=ANCHORS, with_detect=True, det_conf=0.05, keep_rpn_debug=True, fuse_pool=False)
    wts = PackedWeights(params, "bf16x3")
    plan1 = ForwardPlan(wts, H, W, **opts)
    bplan = BatchPlan(wts, N, H, W, **opts)
    first, second = _images(N, H, W, seed=40), _images(N, H, W, seed=60)
    want1, want2 = _per_image(plan1, first), _per_image(plan1, second)
    for x, want in ((first, want1), (second, want2), (first, want1)):
        bplan.forward(x)
        torch.cuda.synchronize()
        got = bplan.unpack_result(bplan.result.cpu().numpy())
        for n, (g, (w, ns, dd, di)) in enumerate(zip(got, want)):
            assert w["count"] > 0
            _assert_same(g, w, n)
            assert int(bplan.prop.dbg_num[n]) == ns
            assert torch.equal(bplan.prop.dbg_dets[n, :ns].cpu().view(torch.int32), dd[:ns].view(torch.int32))
            assert torch.equal(bplan.prop.dbg_idx[n, :ns].cpu(), di[:ns])
    assert bplan.graph is not None
    b1 = BatchPlan(wts, 1, H, W, use_graph=False, **opts)
    b4 = BatchPlan(wts, 4, H, W, use_graph=False, **opts)
    b1.forward(first[:1])
    b4.forward(torch.cat([first, first[:1]]))
    assert b1.n_launches == b4.n_launches == bplan.n_launches > 0


# ------------------------------------------------------------------------------------------------ frcnn_forward_vgg16_batch
def _cforward_case(params, N, H, W, precision):
    from frcnn_b200.engine import BatchPlan, CForward, PackedWeights
    wts = PackedWeights(params, precision)
    x = _images(N, H, W, seed=70 + N)
    cfb = CForward(wts, H, W, ANCHORS, N=N)
    pb, bb, cb = cfb.forward(x if N > 1 else x[0])
    torch.cuda.synchronize()
    pb, bb, cb = pb.clone().view(N, *pb.shape[-2:]), bb.clone().view(N, *bb.shape[-2:]), cb.clone()
    cf1 = CForward(wts, H, W, ANCHORS)
    bplan = BatchPlan(wts, N, H, W, anchors=ANCHORS, use_graph=False)
    bprob, bboxes, bcounts = bplan.forward(x)
    torch.cuda.synchronize()
    for n in range(N):
        p1, b1, c1 = cf1.forward(x[n])
        torch.cuda.synchronize()
        assert int(cb[n]) == int(c1.item()) == int(bcounts[n]) > 0, n
        assert same(pb[n], p1) and same(bb[n], b1), n
        assert same(pb[n], bprob[n]) and same(bb[n], bboxes[n]), n
    return wts, cfb, x, (pb, bb, cb)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("N", [1, 3])
def test_forward_vgg16_batch_150x201(params, N, precision):
    """One C call for N images = frcnn_forward_vgg16 per image = BatchPlan, bit for bit."""
    _cforward_case(params, N, 150, 201, precision)


def test_forward_vgg16_batch_600x1000_graph(params):
    """N = 4 at the benchmarked size; the call captured into a CUDA graph replays to the same results, also after the
    input changed and changed back."""
    wts, cfb, x, (pb, bb, cb) = _cforward_case(params, 4, 600, 1000, "bf16x3")
    static = x.clone()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="thread_local"):
        cfb.forward(static)
    for rep in range(2):
        cfb.prob.zero_()
        cfb.count.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert same(cfb.prob, pb) and same(cfb.boxes, bb) and same(cfb.count, cb), rep
        static.copy_(torch.flip(x, dims=[0]))
        g.replay()
        torch.cuda.synchronize()
        assert same(cfb.prob[0], pb[3]) and same(cfb.count[1:2], cb[2:3])
        static.copy_(x)


def test_forward_vgg16_batch_errors(params, lib):
    """N = 0 and a workspace one byte short return the documented statuses."""
    from frcnn_b200 import _lib
    from frcnn_b200.engine import CForward, PackedWeights
    wts = PackedWeights(params, "bf16")
    H, W = 64, 96
    cf = CForward(wts, H, W, ANCHORS, N=2)
    cfg, wt = ctypes.byref(cf.cfg), ctypes.byref(cf.wt)
    assert lib.frcnn_forward_batch_workspace_bytes(cfg, 0) == 0
    need = lib.frcnn_forward_batch_workspace_bytes(cfg, 2)
    assert need == cf.ws.numel() > lib.frcnn_forward_batch_workspace_bytes(cfg, 1) == lib.frcnn_forward_workspace_bytes(cfg)
    x = torch.zeros((2, 3, H, W), device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())                              # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = lambda N, nbytes: (cfg, wt, N, p(x), H, W, p(cf.ws), nbytes, p(cf.prob), p(cf.boxes), p(cf.count), st)   # noqa: E731
    assert lib.frcnn_forward_vgg16_batch(*args(0, need)) == _lib.ERR_ARG and "N must be" in _lib.last_error()
    assert lib.frcnn_forward_vgg16_batch(*args(2, need - 1)) == _lib.ERR_WORKSPACE
    assert lib.frcnn_forward_vgg16_batch(cfg, wt, 2, None, H, W, p(cf.ws), need, p(cf.prob), p(cf.boxes), p(cf.count), st) == _lib.ERR_ARG
    assert lib.frcnn_forward_vgg16_batch(*args(2, need)) == _lib.OK
    torch.cuda.synchronize()
    with pytest.raises(_lib.FrcnnError):
        CForward(wts, H, W, ANCHORS, N=0)


# ------------------------------------------------------------------------------------------------ error paths
def test_batch_post_errors(lib):
    """N < 1, NULL pointers, output strides that would overlap two images and a short workspace: status and message, no
    launch."""
    from frcnn_b200 import _lib
    ERR, WS = _lib.ERR_ARG, _lib.ERR_WORKSPACE
    buf = torch.zeros(1 << 22, dtype=torch.float32, device="cuda")
    P = ctypes.c_void_p(buf.data_ptr())
    st = None
    H, W, pre, post = 8, 10, 600, 100
    k = min(pre, A * H * W)
    ws1 = lib.frcnn_proposals_workspace_bytes(A, H, W, pre)
    assert lib.frcnn_proposals_batch_workspace_bytes(3, A, H, W, pre) == 3 * ws1 and ws1 % 256 == 0
    assert lib.frcnn_proposals_batch_workspace_bytes(0, A, H, W, pre) == 0
    anchors = dev(ANCHORS)
    AP = ctypes.c_void_p(anchors.data_ptr())
    ws = torch.zeros(3 * ws1, dtype=torch.uint8, device="cuda")
    WP = ctypes.c_void_p(ws.data_ptr())

    def prop(N=3, rois_is=4 * post, scores_is=post, count_is=1, dd_is=5 * k, di_is=k, dn_is=1, nbytes=3 * ws1, cls=P):
        return lib.frcnn_proposals_batch(N, cls, H * W, 1, 18 * H * W, 0, P, H * W, 1, 36 * H * W, AP, A, H, W, 16, 128, 160, 16,
                                         pre, post, 0.7, P, rois_is, P, scores_is, P, count_is, P, dd_is, P, di_is, P, dn_is,
                                         WP, nbytes, st)
    assert prop(N=0) == ERR and "N must be" in _lib.last_error()
    assert prop(cls=None) == ERR and "NULL" in _lib.last_error()
    for kw in (dict(rois_is=4 * post - 4), dict(rois_is=4 * post + 2), dict(scores_is=post - 1), dict(count_is=0),
               dict(dd_is=5 * k - 1), dict(di_is=k - 1), dict(dn_is=0)):
        assert prop(**kw) == ERR and "overlap" in _lib.last_error(), kw
    assert prop(nbytes=3 * ws1 - 1) == WS
    torch.cuda.synchronize()

    R, NC, C = 50, 21, 64
    assert lib.frcnn_roi_pool_batch(P, None, 0, H, W, C, P, 4 * R, P, 1, R, 7, 7, ctypes.c_float(1 / 16), P, None, None,
                                    R * 49 * C, st) == ERR
    assert lib.frcnn_roi_pool_batch(None, None, 2, H, W, C, P, 4 * R, P, 1, R, 7, 7, ctypes.c_float(1 / 16), P, None, None,
                                    R * 49 * C, st) == ERR
    assert lib.frcnn_roi_pool_batch(P, None, 2, H, W, C, P, 4 * R, P, 1, R, 7, 7, ctypes.c_float(1 / 16), P, None, None,
                                    R * 49 * C - 8, st) == ERR and "overlap" in _lib.last_error()
    dargs = lambda N, ps, bs: (N, P, P, 128, 0, P, 0, P, 1, R, NC, 600, 1000, P, ps, P, bs, st)     # noqa: E731
    assert lib.frcnn_head_decode_batch(*dargs(0, R * NC, 4 * R * NC)) == ERR
    assert lib.frcnn_head_decode_batch(*dargs(2, R * NC - 1, 4 * R * NC)) == ERR and "overlap" in _lib.last_error()
    assert lib.frcnn_head_decode_batch(*dargs(2, R * NC, 4 * R * NC - 4)) == ERR and "overlap" in _lib.last_error()
    assert lib.frcnn_head_decode_batch(2, None, P, 128, 0, P, 0, P, 1, R, NC, 600, 1000, P, R * NC, P, 4 * R * NC, st) == ERR
    targs = lambda N, ks, kc, cc, kp=P: (N, P, 0, P, 0, P, 1, R, NC, 0.3, ctypes.c_float(0.5), kp, ks, P, kc, P, cc, st)  # noqa: E731
    assert lib.frcnn_detect_batch(*targs(0, R * (NC - 1), NC - 1, NC - 1)) == ERR
    assert lib.frcnn_detect_batch(*targs(2, R * (NC - 1), NC - 1, NC - 1, kp=None)) == ERR
    for bad in ((R * (NC - 1) - 1, NC - 1, NC - 1), (R * (NC - 1), NC - 2, NC - 1), (R * (NC - 1), NC - 1, 0)):
        assert lib.frcnn_detect_batch(*targs(2, *bad)) == ERR and "overlap" in _lib.last_error(), bad
    assert lib.frcnn_maxpool2x2_ceil_batch(P, None, 0, H, W, C, P, None, st) == ERR
    assert lib.frcnn_maxpool2x2_ceil_batch(P, P, 2, H, W, C, P, None, st) == ERR
    torch.cuda.synchronize()
