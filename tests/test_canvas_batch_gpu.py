"""GPU tests of canvas batches: N images of DIFFERENT sizes, each at the top-left of its Hc x Wc slot, with their sizes and
clip bounds in device arrays (the *_batch_ext entries and engine.CanvasBatchPlan).  Every image's result must be
bit-identical to the one-image entry point (or ForwardPlan) on that image alone -- including where the canvas launch picks
another N tile or pixel tile than the image alone would -- every output pixel outside an image must be exactly 0, and
whatever lies outside an image in the canvas (large values, NaN, a previous larger image) must never reach its results."""
import ctypes

import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_batch_gpu import ANCHORS, _act, _assert_same, _bits, _per_image, _weights

pytestmark = pytest.mark.gpu
POISON = (3.0e38, float("nan"), -1.0e30)


@pytest.fixture(scope="module")
def params():
    return orc.make_params(seed=1234)


def _ops():
    from frcnn_b200 import ops
    return ops


def _ext(sizes):
    return torch.tensor(sizes, dtype=torch.int32, device="cuda").view(-1, 2).contiguous()


def _poison_like(t):
    """t filled with a cycle of huge values and NaN (a stale or foreign canvas)."""
    v = torch.tensor(POISON, dtype=torch.float32)
    return v.repeat(t.numel() // len(POISON) + 1)[:t.numel()].view(t.shape).to(device=t.device, dtype=t.dtype)


def _layer_ext(e, k):
    return -(-e // (1 << k))


# ------------------------------------------------------------------------------------------------ 1: convolutions
# (Hc, Wc, Cin, Cout, ksize, relu, fused pool, bf16 out, ld_f32, halvings, image sizes in input pixels,
#  whether some image's one-image plan must differ from the canvas plan)
CONV_CASES = {
    # BN: 256 (bf16) / 128 (bf16x3) for the canvas, 64 alone; pixel tile: 1x128 for the canvas, 4x32 for the 20x30 image
    "3x3_bn_and_tile": (75, 125, 128, 256, 3, True, False, True, 0, 0, [(75, 125), (20, 30), (5, 120), (0, 0)], True),
    "3x3_pool_odd": (38, 66, 256, 512, 3, True, True, True, 0, 0, [(37, 65), (13, 7), (38, 66)], True),
    "1x1_f32_halvings": (19, 31, 512, 54, 1, False, False, False, 64, 4, [(304, 496), (100, 129), (1, 1)], True),
    "3x3_relu_off_bf16_and_f32": (13, 21, 64, 64, 3, False, False, True, 64, 0, [(13, 21), (12, 3), (0, 0)], False),
}
PLAN_KEYS = ("BN", "TH", "TW")


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv2d_batch_ext_equals_per_image_conv(case, x3):
    """frcnn_conv2d_batch_ext over a canvas = frcnn_conv2d on each image alone, bit for bit, and exactly 0 at every output
    pixel outside an image (the output buffers are poisoned first).  The canvas input is zero outside the images, as the
    previous canvas layer leaves it."""
    ops = _ops()
    Hc, Wc, Cin, Cout, k, relu, pool, out_bf16, ld, halv, sizes, differs = CONV_CASES[case]
    N = len(sizes)
    lsz = [(_layer_ext(h, halv), _layer_ext(w, halv)) for h, w in sizes]
    g = torch.Generator().manual_seed(len(case) + 7 * x3)
    x = torch.zeros((N, Hc, Wc, Cin))
    for n, (h, w) in enumerate(lsz):
        x[n, :h, :w] = torch.randn((h, w, Cin), generator=g) + 0.2
    x = x.cuda()
    xa = _act(x, x3)
    hi, lo = _weights(Cout, Cin, k, x3, len(case))
    bias = ops.pad_bias((torch.randn((Cout,), generator=g) * 0.1).cuda(), max(Cout, ld))
    oh, ow = ((Hc + 1) // 2, (Wc + 1) // 2) if pool else (Hc, Wc)
    y = None
    if out_bf16:
        yh = _poison_like(torch.empty((N, oh, ow, Cout), dtype=torch.bfloat16, device="cuda"))
        y = ops.Act(yh, yh.clone() if x3 else None)
    y32 = _poison_like(torch.empty((N * Hc * Wc, ld), device="cuda")) if ld else None
    ops.conv2d_batch(xa, hi, lo, bias, k, relu, out_act=out_bf16, ld_f32=ld, out=y, out_f32=y32, fuse_pool=pool,
                     extents=_ext(sizes), halvings=halv)
    plan = ops.conv_last_plan()
    torch.cuda.synchronize()
    saw_other_plan = False
    for n, (h, w) in enumerate(lsz):
        ph, pw = ((h + 1) // 2, (w + 1) // 2) if pool else (h, w)
        if y is not None:
            planes = [y.hi] + ([y.lo] if x3 else [])
            for t in planes:
                outside = t[n].clone()
                outside[:ph, :pw] = 0
                assert not _bits(outside).any().item(), (case, n)
        if y32 is not None:
            outside = y32.view(N, Hc, Wc, ld)[n].clone()
            outside[:h, :w] = 0
            assert not _bits(outside).any().item(), (case, n)
        if h == 0 or w == 0:
            continue
        xn = ops.Act(xa.hi[n, :h, :w].contiguous(), None if xa.lo is None else xa.lo[n, :h, :w].contiguous())
        ys, ys32 = ops.conv2d(xn, hi, lo, bias, k, relu, out_act=out_bf16, ld_f32=ld, fuse_pool=pool)
        plan1 = ops.conv_last_plan()
        saw_other_plan |= any(plan1[f] != plan[f] for f in PLAN_KEYS)
        if y is not None:
            assert torch.equal(_bits(y.hi[n, :ph, :pw]), _bits(ys.hi)), (case, n)
            if x3:
                assert torch.equal(_bits(y.lo[n, :ph, :pw]), _bits(ys.lo)), (case, n)
        if y32 is not None:
            assert torch.equal(_bits(y32.view(N, Hc, Wc, ld)[n, :h, :w]), _bits(ys32.view(h, w, ld))), (case, n)
    if differs:
        assert saw_other_plan, (case, plan)


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
def test_c8_first_layer_ext_equals_per_image(x3):
    """pack_image_c8_batch_ext + conv3x3_c8_batch_ext over a canvas whose pixels outside the images are poisoned = the
    one-image pack + conv1_1 on each image, bit for bit; packed planes and outputs are 0 outside every image."""
    ops = _ops()
    Hc, Wc, Cout = 40, 64, 64
    sizes = [(40, 64), (37, 61), (17, 5), (0, 0), (1, 64)]
    N = len(sizes)
    prec = "bf16x3" if x3 else "bf16"
    g = torch.Generator().manual_seed(5)
    x = _poison_like(torch.empty((N, 3, Hc, Wc)))
    for n, (h, w) in enumerate(sizes):
        x[n, :, :h, :w] = torch.randn((3, h, w), generator=g) * 50
    x = x.cuda()
    wt = (torch.randn((Cout, 3, 3, 3), generator=g) * 0.1).cuda()
    whi, wlo = ops.pack_conv_weights_c8(wt, precision=prec)
    bias = ops.pad_bias((torch.randn((Cout,), generator=g) * 0.1).cuda(), Cout)
    ext = _ext(sizes)
    packed = ops.pack_image_c8_batch(x, precision=prec, extents=ext)
    yh = _poison_like(torch.empty((N, Hc, Wc, Cout), dtype=torch.bfloat16, device="cuda"))
    y = ops.conv3x3_c8_batch(packed, N, Hc, Wc, whi, wlo, bias, True, out=ops.Act(yh, yh.clone() if x3 else None), extents=ext)
    torch.cuda.synchronize()
    rows = Hc * (Wc + 2) * 8
    for n, (h, w) in enumerate(sizes):
        for t in [packed.hi] + ([packed.lo] if x3 else []):
            plane = t[n, :rows].view(Hc, Wc + 2, 8).clone()
            plane[:h, 1:w + 1] = 0
            assert not _bits(plane).any().item() and not _bits(t[n, rows:]).any().item(), n
        for t in [y.hi] + ([y.lo] if x3 else []):
            outside = t[n].clone()
            outside[:h, :w] = 0
            assert not _bits(outside).any().item(), n
        if h == 0 or w == 0:
            continue
        p1 = ops.pack_image_c8(x[n, :, :h, :w].contiguous(), precision=prec)
        assert torch.equal(_bits(packed.hi[n, :rows].view(Hc, Wc + 2, 8)[:h, :w + 2]), _bits(p1.hi[:h * (w + 2) * 8].view(h, w + 2, 8)))
        y1 = ops.conv3x3_c8(p1, h, w, whi, wlo, bias, True)
        assert torch.equal(_bits(y.hi[n, :h, :w]), _bits(y1.hi)), n
        if x3:
            assert torch.equal(_bits(y.lo[n, :h, :w]), _bits(y1.lo)), n


# ------------------------------------------------------------------------------------------------ 2: post-processing
# feature-map sizes (fh, fw) of the images in a 24 x 40 canvas, their input extents (4 halvings) and clip bounds
POST_MAPS = [(24, 40), (9, 13), (1, 1), (17, 40), (0, 0)]
POST_EXT = [(24 * 16, 40 * 16), (9 * 16 - 15, 13 * 16), (5, 16), (17 * 16 - 1, 40 * 16 - 3), (0, 0)]
POST_CLIP = [(384, 640), (129, 129), (5, 16), (271, 637), (0, 0)]       # (129, 129): forward.py's (H, H), SURVEY Q7


def test_post_maps_match_extents():
    assert [(_layer_ext(h, 4), _layer_ext(w, 4)) for h, w in POST_EXT] == POST_MAPS


def test_proposals_batch_ext_equals_per_image():
    """frcnn_proposals_batch_ext = frcnn_proposals on each image's own map and clip bounds (rois, scores, count), with the
    canvas cells outside every map poisoned."""
    ops = _ops()
    Hc, Wc, A, ld = 24, 40, 9, 64
    N = len(POST_MAPS)
    g = torch.Generator().manual_seed(11)
    rpn = _poison_like(torch.empty((N, Hc, Wc, ld)))
    for n, (fh, fw) in enumerate(POST_MAPS):
        rpn[n, :fh, :fw, :2 * A] = torch.randn((fh, fw, 2 * A), generator=g) * 3
        rpn[n, :fh, :fw, 2 * A:6 * A] = torch.randn((fh, fw, 4 * A), generator=g) * 0.3
        rpn[n, :fh, :fw, 6 * A:] = 0
    rpn = rpn.cuda()
    anchors = torch.from_numpy(ANCHORS).cuda()
    pre_n, post_n = 6000, 300
    work = ops.proposals_batch(rpn.view(N, Hc * Wc, ld), None, anchors, A, Hc, Wc, 16, 0, 0, 16, pre_n, post_n, 0.7,
                               layout="nhwc", ld=ld, cls_is_logits=True, extents=_ext(POST_EXT), halvings=4, im_info=_ext(POST_CLIP))
    torch.cuda.synchronize()
    for n, (fh, fw) in enumerate(POST_MAPS):
        if fh == 0:
            assert work.count[n].item() == 0 and not work.rois[n].any().item()
            continue
        one = ops.proposals(rpn[n, :fh, :fw].contiguous().view(fh * fw, ld), None, anchors, A, fh, fw, 16, POST_CLIP[n][0],
                            POST_CLIP[n][1], 16, pre_n, post_n, 0.7, layout="nhwc", ld=ld, cls_is_logits=True)
        torch.cuda.synchronize()
        R = one.count.item()
        assert work.count[n].item() == R and (R > 0 or fh == 1), n
        assert torch.equal(_bits(work.rois[n]), _bits(one.rois)) and torch.equal(_bits(work.scores[n]), _bits(one.scores)), n


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
def test_roi_pool_batch_ext_clamps_to_each_image(x3):
    """frcnn_roi_pool_batch_ext = frcnn_roi_pool on each image's own map: RoIs that reach or cross the map's border are
    clamped to it, not to the canvas, whose other pixels hold huge values and NaN."""
    ops = _ops()
    Hc, Wc, C, R = 24, 40, 512, 64
    N = len(POST_MAPS)
    g = torch.Generator().manual_seed(12)
    feat = _poison_like(torch.empty((N, Hc, Wc, C)))
    rois = torch.zeros((N, R, 4))
    for n, (fh, fw) in enumerate(POST_MAPS):
        feat[n, :fh, :fw] = torch.relu(torch.randn((fh, fw, C), generator=g))
        H, W = fh * 16, fw * 16
        x1 = torch.rand((R,), generator=g) * W
        y1 = torch.rand((R,), generator=g) * H
        rois[n] = torch.stack([x1, y1, x1 + torch.rand((R,), generator=g) * 2 * W, y1 + torch.rand((R,), generator=g) * 2 * H], 1)
        rois[n, 0] = torch.tensor([0.0, 0.0, W - 1.0, H - 1.0])           # exactly the map
        rois[n, 1] = torch.tensor([W - 9.0, H - 9.0, W + 200.0, H + 300.0])
    feat, rois = feat.cuda(), rois.cuda()
    fa = _act(feat, x3)
    counts = torch.tensor([R, R - 3, 7, R, R], dtype=torch.int32, device="cuda")
    o32 = torch.empty((N, R, 49, C), device="cuda")
    out, _ = ops.roi_pool_batch(fa, rois, counts, 7, 7, 1.0 / 16, out_f32=o32, extents=_ext(POST_EXT), halvings=4)
    torch.cuda.synchronize()
    for n, (fh, fw) in enumerate(POST_MAPS):
        if fh == 0:
            assert not _bits(out.hi[n]).any().item()
            continue
        fn = ops.Act(fa.hi[n, :fh, :fw].contiguous(), None if fa.lo is None else fa.lo[n, :fh, :fw].contiguous())
        one, one32 = ops.roi_pool(fn, rois[n].contiguous(), counts[n:n + 1], 7, 7, 1.0 / 16, want_f32=True)
        torch.cuda.synchronize()
        assert torch.equal(_bits(out.hi[n]), _bits(one.hi[0])), n
        if x3:
            assert torch.equal(_bits(out.lo[n]), _bits(one.lo[0])), n
        assert torch.equal(_bits(o32[n]), _bits(one32)), n
        assert torch.isfinite(o32[n]).all().item() and o32[n].max().item() < 100, n


def test_head_decode_batch_ext_clips_per_image():
    """frcnn_head_decode_batch_ext = frcnn_head_decode with each image's own clip bounds."""
    ops = _ops()
    N, R, NC, ld = len(POST_CLIP), 300, 21, 128
    g = torch.Generator().manual_seed(13)
    sd = (torch.randn((N, R, ld), generator=g) * 2).cuda()
    rois = (torch.rand((N, R, 4), generator=g) * 700).sort(dim=2).values.cuda()
    counts = torch.tensor([300, 0, 17, 299, 300], dtype=torch.int32, device="cuda")
    prob, boxes = ops.head_decode_batch(sd, ld, rois, counts, NC, 0, 0, im_info=_ext(POST_CLIP))
    torch.cuda.synchronize()
    for n, (ih, iw) in enumerate(POST_CLIP):
        p1, b1 = ops.head_decode(sd[n].contiguous(), ld, rois[n].contiguous(), counts[n:n + 1], NC, ih, iw)
        torch.cuda.synchronize()
        assert torch.equal(_bits(prob[n]), _bits(p1)) and torch.equal(_bits(boxes[n]), _bits(b1)), n


# --------------------------------------------------------------------------------------------------- 3: the whole plan
def _images(sizes, seed):
    return [torch.from_numpy(orc.make_image(h, w, seed=seed + i)[0].astype(np.float32)).cuda() for i, (h, w) in enumerate(sizes)]


def _canvas_result(plan):
    torch.cuda.synchronize()
    return plan.unpack_result(plan.result.cpu().numpy())


def _want(eng, imgs, clips=None):
    out = []
    for i, x in enumerate(imgs):
        p = eng.plan(int(x.shape[1]), int(x.shape[2]))
        p.set_clip(*(clips[i] if clips else x.shape[1:]))
        out += _per_image(p, x[None])
    return out


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_canvas_plan_equals_forward_plan(params, precision):
    """CanvasBatchPlan, N = 3 on a 150 x 201 canvas = ForwardPlan per image on every result field (per-class NMS on); the
    same graph then serves another size mix -- a small image in the slot a large one held, a clip bound of (H, H), an
    empty slot -- without a re-capture and without stale pixels."""
    from frcnn_b200.engine import CanvasBatchPlan, Engine
    eng = Engine(params, precision=precision, anchors=ANCHORS, with_detect=True, det_conf=0.05)
    plan = eng.canvas_plan(3, 150, 201)
    assert isinstance(plan, CanvasBatchPlan) and eng.canvas_plan(3, 150, 201) is plan
    first = _images([(150, 201), (128, 96), (150, 150)], seed=30)
    want = _want(eng, first)
    for rep in range(2):
        plan.forward(first)
        for n, (g, w) in enumerate(zip(_canvas_result(plan), want)):
            assert w["count"] > 0
            _assert_same(g, w, ("first mix", rep, n))
    graph = plan.graph
    assert graph is not None
    second = _images([(128, 96), (149, 201)], seed=40)
    clips = [(128, 128), (149, 201)]
    want2 = _want(eng, second, clips)
    plan.forward(second, img_infos=clips)
    assert plan.graph is graph and plan.image_sizes == [(128, 96), (149, 201), (0, 0)]
    got = _canvas_result(plan)
    for n, w in enumerate(want2):
        _assert_same(got[n], w, ("second mix", n))
    assert got[2]["count"] == 0 and not got[2]["keep_count"].any()
    probs, boxes, counts = plan.forward(second, img_infos=clips)
    assert counts.cpu().tolist() == [w["count"] for w in want2] + [0]
    # Engine.forward_images: chunks of N, default canvas = the largest H and W rounded up to 64
    imgs = _images([(150, 201), (64, 64), (100, 30), (128, 96), (150, 150)], seed=50)
    want3 = _want(eng, imgs)
    res = eng.forward_images(imgs, N=2)
    assert any(k[:4] == ("canvas", 2, 192, 256) for k in eng.plans)
    for (p, b), w in zip(res, want3):
        assert p.shape[0] == w["count"] and np.array_equal(p.cpu().numpy(), w["prob"]) and np.array_equal(b.cpu().numpy(), w["boxes"])


def test_canvas_plan_headline_sizes(params):
    """VOC-style inputs, short side 600 and long side up to 1000 (600 x 800, 600 x 901, 600 x 1000) in one 600 x 1000
    canvas, bf16x3 with the per-class NMS = ForwardPlan on each."""
    from frcnn_b200.engine import CanvasBatchPlan, ForwardPlan, PackedWeights
    wts = PackedWeights(params, "bf16x3")
    imgs = _images([(600, 800), (600, 901), (600, 1000)], seed=60)
    plan = CanvasBatchPlan(wts, 3, 600, 1000, anchors=ANCHORS, with_detect=True, det_conf=0.05)
    plan.forward(imgs)
    got = _canvas_result(plan)
    for n, x in enumerate(imgs):
        p1 = ForwardPlan(wts, 600, int(x.shape[2]), anchors=ANCHORS, with_detect=True, det_conf=0.05)
        w = _per_image(p1, x[None])[0]
        assert w["count"] > 0
        _assert_same(got[n], w, n)
        del p1


# ----------------------------------------------------------------------------------------------------------- 4: errors
def test_canvas_errors(params):
    """Too many images, an image larger than the canvas, keep_rpn_debug, ResNet, and NULL extents / bad N at the C
    entries all raise or return FRCNN_ERR_ARG."""
    from frcnn_b200 import _lib
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.engine import CanvasBatchPlan, Engine
    from frcnn_b200.resnet_engine import ResNetEngine
    eng = Engine(params, precision="bf16", anchors=ANCHORS)
    plan = eng.canvas_plan(2, 64, 96)
    x = torch.zeros((3, 64, 96), device="cuda")
    with pytest.raises(FrcnnError):
        plan.forward([x, x, x])
    with pytest.raises(FrcnnError):
        plan.forward([torch.zeros((3, 65, 96), device="cuda")])
    with pytest.raises(FrcnnError):
        plan.forward([torch.zeros((3, 64, 97), device="cuda")])
    with pytest.raises(FrcnnError):
        plan.forward([x], img_infos=[(64, 96), (64, 96)])
    with pytest.raises(FrcnnError):
        CanvasBatchPlan(eng.weights, 2, 64, 96, anchors=ANCHORS, keep_rpn_debug=True)
    with pytest.raises(FrcnnError):
        eng.forward_images([x], canvas=(32, 96))
    with pytest.raises(FrcnnError):
        eng.forward_images([torch.zeros((64, 96), device="cuda")])
    reng = ResNetEngine(orc.make_resnet_params(50, seed=5), 50, precision="bf16", anchors=ANCHORS, post_n=50)
    with pytest.raises(FrcnnError):
        reng.forward_images([x])
    lib = _lib.load()
    buf = torch.zeros((1 << 20,), device="cuda")
    p = ctypes.c_void_p(buf.data_ptr())
    e = _ext([(8, 8)])
    pe = ctypes.c_void_p(e.data_ptr())
    assert lib.frcnn_conv2d_batch_ext(p, None, 1, 8, 8, 64, p, None, p, 64, 3, 1, 0, p, None, None, 0, None, 0, None) == _lib.ERR_ARG
    assert lib.frcnn_conv2d_batch_ext(p, None, 0, 8, 8, 64, p, None, p, 64, 3, 1, 0, p, None, None, 0, pe, 0, None) == _lib.ERR_ARG
    assert lib.frcnn_conv2d_batch_ext(p, None, 1, 8, 8, 64, p, None, p, 64, 3, 1, 0, p, None, None, 0, pe, 31, None) == _lib.ERR_ARG
    assert lib.frcnn_conv3x3_c8_batch_ext(p, None, 1, 8, 8, p, None, p, 64, 1, None, p, None, None) == _lib.ERR_ARG
    assert lib.frcnn_pack_image_c8_batch_ext(p, 1, 3, 8, 8, 192, 64, 8, 1, None, p, None, None) == _lib.ERR_ARG
    assert lib.frcnn_pack_image_c8_batch_ext(p, 0, 3, 8, 8, 192, 64, 8, 1, pe, p, None, None) == _lib.ERR_ARG
    assert lib.frcnn_roi_pool_batch_ext(p, None, 1, 8, 8, 64, p, 0, None, 0, 4, 7, 7, ctypes.c_float(1.0), None, 0, p, None, None, 0,
                                        None) == _lib.ERR_ARG
    assert lib.frcnn_roi_pool_batch_ext(p, None, 0, 8, 8, 64, p, 0, None, 0, 4, 7, 7, ctypes.c_float(1.0), pe, 0, p, None, None, 0,
                                        None) == _lib.ERR_ARG
    assert lib.frcnn_head_decode_batch_ext(1, p, p, 128, 0, p, 0, None, 0, 4, 21, None, p, 0, p, 0, None) == _lib.ERR_ARG
    assert lib.frcnn_head_decode_batch_ext(0, p, p, 128, 0, p, 0, None, 0, 4, 21, pe, p, 0, p, 0, None) == _lib.ERR_ARG
    ws = lib.frcnn_proposals_batch_workspace_bytes(1, 9, 8, 8, 6000)
    for n_, ext_, info_ in ((1, None, pe), (1, pe, None), (0, pe, pe)):
        assert lib.frcnn_proposals_batch_ext(n_, p, 1, 64, 0, 1, p, 1, 64, 0, p, 9, 8, 8, 16, ext_, 4, info_, 16, 6000, 300, 0.7,
                                             p, 1200, p, 300, p, 1, p, ws, None) == _lib.ERR_ARG
    torch.cuda.synchronize()
