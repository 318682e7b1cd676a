"""GPU tests of the ResNet trunk in batches and canvas batches: the batched ResNet kernels (first-layer im2col, 3x3/2 max-pool,
2x subsample, residual convolution), the per-level extent kernel, and resnet_engine.ResNetBatchPlan / ResNetCanvasBatchPlan
behind ResNetBatchEngine.  Every image's result must be bit-identical to the one-image entry (or ResNetForwardPlan) on that
image alone, every output pixel outside an image must be exactly 0, and whatever the canvas holds outside an image (huge
values, NaN, a previous larger image) must never reach its results."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_batch_gpu import ANCHORS, _act, _assert_same, _bits, _per_image, _weights
from test_canvas_batch_gpu import _ext, _poison_like

pytestmark = pytest.mark.gpu
# image sizes in a 40 x 53 canvas: odd and even, one pixel, an empty slot, an over-large extent (clamped to the slot)
SIZES = [(40, 53), (23, 30), (1, 1), (0, 0), (7, 2), (10 ** 6, 31)]
HC, WC = 40, 53


def _ops():
    from frcnn_b200 import ops
    return ops


def _clamp(sizes, Hc, Wc):
    return [(min(h, Hc), min(w, Wc)) for h, w in sizes]


def _conv1(e):
    return max((e - 1) // 2 + 1, 0)


def _pool1(c):
    return (c - 2) // 2 + 1 if c >= 2 else 0


def _outside_zero(t, n, h, w):
    o = t[n].clone()
    o[:h, :w] = 0
    return not _bits(o).any().item()


def _planes(a):
    return [a.hi] + ([a.lo] if a.lo is not None else [])


# ------------------------------------------------------------------------------------------------ 1: the batched kernels
@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
def test_im2col_batch_equals_per_image(x3):
    """frcnn_pack_image_im2col_batch[_ext] (7x7/2 pad 3, K = 147 -> 160) = the one-image im2col of each (cropped) image; with
    extents the canvas outside every image is poisoned and the output outside each image's conv1 extent is 0."""
    ops = _ops()
    from frcnn_b200.resnet_engine import CONV1_KPAD
    prec = "bf16x3" if x3 else "bf16"
    N = len(SIZES)
    g = torch.Generator().manual_seed(1)
    x = _poison_like(torch.empty((N, 3, HC, WC)))
    for n, (h, w) in enumerate(_clamp(SIZES, HC, WC)):
        x[n, :, :h, :w] = torch.randn((3, h, w), generator=g) * 50
    x = x.cuda()
    out = ops.pack_image_im2col_batch(x, 7, 2, 3, CONV1_KPAD, precision=prec, extents=_ext(SIZES))
    torch.cuda.synchronize()
    for n, (h, w) in enumerate(_clamp(SIZES, HC, WC)):
        oh, ow = _conv1(h), _conv1(w)
        assert all(_outside_zero(t, n, oh, ow) for t in _planes(out)), n
        if h == 0 or w == 0:
            continue
        one = ops.pack_image_im2col_general(x[n, :, :h, :w].contiguous(), 7, 2, 3, CONV1_KPAD, precision=prec)
        for a, b in zip(_planes(out), _planes(one)):
            assert torch.equal(_bits(a[n, :oh, :ow]), _bits(b)), n
    # a same-size batch (no extents) of finite images
    xs = (torch.randn((3, 3, 37, 50), generator=g) * 50).cuda()
    out = ops.pack_image_im2col_batch(xs, 7, 2, 3, CONV1_KPAD, precision=prec)
    torch.cuda.synchronize()
    for n in range(3):
        one = ops.pack_image_im2col_general(xs[n], 7, 2, 3, CONV1_KPAD, precision=prec)
        for a, b in zip(_planes(out), _planes(one)):
            assert torch.equal(_bits(a[n]), _bits(b)), n


def _neg_inf_padded(a, n, h, w):
    """Image n's top-left h x w of Act a, padded with -inf to at least 3 x 3 (so the one-image pool accepts it; -inf never
    wins a max)."""
    ops = _ops()
    H, W = max(h, 3), max(w, 3)
    planes = []
    for k, t in enumerate(_planes(a)):
        p = torch.full((H, W, t.shape[-1]), float("-inf") if k == 0 else 0.0, dtype=t.dtype, device=t.device)
        p[:h, :w] = t[n, :h, :w]
        planes.append(p)
    return ops.Act(planes[0], planes[1] if len(planes) > 1 else None)


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
def test_maxpool3x3s2_batch_equals_per_image(x3):
    """frcnn_maxpool3x3s2_ceil_batch[_ext] = the one-image pool of each image: windows clipped at the image's border (the
    canvas outside is poisoned; the images hold negative values, -0.0 and a NaN, so a zero outside would change a max),
    outputs outside the pooled extent are 0."""
    ops = _ops()
    N, C = len(SIZES), 64
    g = torch.Generator().manual_seed(2)
    x = _poison_like(torch.empty((N, HC, WC, C)))
    for n, (h, w) in enumerate(_clamp(SIZES, HC, WC)):
        x[n, :h, :w] = torch.randn((h, w, C), generator=g) - 1.0
    x[0, 0, 0, :8] = -0.0
    x[1, 3, 4, 5] = float("nan")
    xa = _act(x.cuda(), x3)
    y = ops.maxpool3x3s2_ceil_batch(xa, extents=_ext(SIZES))
    torch.cuda.synchronize()
    for n, (h, w) in enumerate(_clamp(SIZES, HC, WC)):
        ph, pw = _pool1(h), _pool1(w)
        assert all(_outside_zero(t, n, ph, pw) for t in _planes(y)), n
        if ph == 0 or pw == 0:
            continue
        one = ops.maxpool3x3s2_ceil(_neg_inf_padded(xa, n, h, w))
        for a, b in zip(_planes(y), _planes(one)):
            assert torch.equal(_bits(a[n, :ph, :pw]), _bits(b[:ph, :pw])), n
    xs = _act(torch.randn((3, 31, 44, C), generator=g).cuda(), x3)
    y = ops.maxpool3x3s2_ceil_batch(xs)
    torch.cuda.synchronize()
    for n in range(3):
        one = ops.maxpool3x3s2_ceil(ops.Act(xs.hi[n], None if xs.lo is None else xs.lo[n]))
        for a, b in zip(_planes(y), _planes(one)):
            assert torch.equal(_bits(a[n]), _bits(b)), n


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
def test_subsample2x_batch_equals_per_image(x3):
    """frcnn_subsample2x_batch over a canvas whose input is 0 outside every image (as the layers before it leave it) = the
    one-image subsample of each image, and 0 outside ceil(extent / 2)."""
    ops = _ops()
    N, C = len(SIZES), 64
    g = torch.Generator().manual_seed(3)
    x = torch.zeros((N, HC, WC, C))
    for n, (h, w) in enumerate(_clamp(SIZES, HC, WC)):
        x[n, :h, :w] = torch.randn((h, w, C), generator=g)
    xa = _act(x.cuda(), x3)
    y = ops.subsample2x_batch(xa)
    torch.cuda.synchronize()
    for n, (h, w) in enumerate(_clamp(SIZES, HC, WC)):
        sh, sw = (h + 1) // 2, (w + 1) // 2
        assert all(_outside_zero(t, n, sh, sw) for t in _planes(y)), n
        if h == 0 or w == 0:
            continue
        xn = ops.Act(xa.hi[n, :h, :w].contiguous(), None if xa.lo is None else xa.lo[n, :h, :w].contiguous())
        one = ops.subsample2x(xn)
        for a, b in zip(_planes(y), _planes(one)):
            assert torch.equal(_bits(a[n, :sh, :sw]), _bits(b)), n


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
@pytest.mark.parametrize("ksize", [1, 3])
def test_conv2d_res_batch_equals_per_image(ksize, relu, x3):
    """frcnn_conv2d_res_batch[_ext] = frcnn_conv2d_res on each image: the canvas input is 0 outside every image (as the
    layers before it leave it), the residual and the output buffers are poisoned there, and every output pixel outside an
    image is 0 -- whatever the residual holds at it."""
    ops = _ops()
    Hc, Wc, Cin, Cout = 19, 32, 128, 256
    sizes = [(19, 32), (10, 13), (1, 1), (0, 0), (6, 31)]
    N = len(sizes)
    g = torch.Generator().manual_seed(10 * ksize + 2 * relu + x3)
    x = torch.zeros((N, Hc, Wc, Cin))
    r = _poison_like(torch.empty((N, Hc, Wc, Cout)))
    for n, (h, w) in enumerate(sizes):
        x[n, :h, :w] = torch.relu(torch.randn((h, w, Cin), generator=g))
        r[n, :h, :w] = torch.randn((h, w, Cout), generator=g)
    xa, ra = _act(x.cuda(), x3), _act(r.cuda(), x3)
    hi, lo = _weights(Cout, Cin, ksize, x3, 7 + ksize)
    bias = ops.pad_bias((torch.randn((Cout,), generator=g) * 0.1).cuda(), Cout)
    yh = _poison_like(torch.empty((N, Hc, Wc, Cout), dtype=torch.bfloat16, device="cuda"))
    y = ops.conv2d_res_batch(xa, hi, lo, bias, ksize, relu, ra, out=ops.Act(yh, yh.clone() if x3 else None), extents=_ext(sizes))
    yb = ops.conv2d_res_batch(xa, hi, lo, bias, ksize, relu, ra)          # same-size batch: every slot is a whole image
    torch.cuda.synchronize()
    for n, (h, w) in enumerate(sizes):
        assert all(_outside_zero(t, n, h, w) for t in _planes(y)), n
        whole = ops.conv2d_res(ops.Act(xa.hi[n], None if xa.lo is None else xa.lo[n]), hi, lo, bias, ksize, relu,
                               ops.Act(ra.hi[n], None if ra.lo is None else ra.lo[n]))
        for a, b in zip(_planes(yb), _planes(whole)):
            assert torch.equal(_bits(a[n]), _bits(b)), n
        if h == 0 or w == 0:
            continue
        crop = lambda a: ops.Act(a.hi[n, :h, :w].contiguous(), None if a.lo is None else a.lo[n, :h, :w].contiguous())  # noqa: E731
        one = ops.conv2d_res(crop(xa), hi, lo, bias, ksize, relu, crop(ra))
        for a, b in zip(_planes(y), _planes(one)):
            assert torch.equal(_bits(a[n, :h, :w]), _bits(b)), n


def test_level_extents_rule_and_clamp():
    """frcnn_resnet_level_extents for every h, w in 1..200 on a 200 x 200 canvas = the level rule; extents larger than the
    canvas are clamped to it, negative ones read as 0."""
    ops = _ops()
    from test_resnet_batch_abi_cpu import _levels
    hs, ws = np.meshgrid(np.arange(1, 201), np.arange(1, 201), indexing="ij")
    sizes = np.stack([hs.ravel(), ws.ravel()], 1).astype(np.int32)
    lv = ops.resnet_level_extents(torch.from_numpy(sizes).cuda(), 200, 200).cpu().numpy()
    rule = np.array([_levels(e) for e in range(201)])                     # [e, level]
    assert np.array_equal(lv[:, :, 0], rule[sizes[:, 0]].T) and np.array_equal(lv[:, :, 1], rule[sizes[:, 1]].T)
    lv = ops.resnet_level_extents(_ext([(10 ** 9, -5), (150, 201), (0, 0)]), 150, 201).cpu().numpy()
    canvas = list(zip(_levels(150), _levels(201)))
    assert [tuple(v) for v in lv[:, 0]] == [(c[0], 0) for c in canvas]
    assert [tuple(v) for v in lv[:, 1]] == canvas and not lv[:, 2].any()


# --------------------------------------------------------------------------------------------------- 2: the whole plans
def _images(sizes, seed):
    return [torch.from_numpy(orc.make_image(h, w, seed=seed + i)[0].astype(np.float32)).cuda() for i, (h, w) in enumerate(sizes)]


def _result(plan):
    torch.cuda.synchronize()
    return plan.unpack_result(plan.result.cpu().numpy())


def _want(eng, imgs, check_levels=None):
    """ResNetForwardPlan per image; check_levels: a canvas plan whose level extents must be those plans' map sizes."""
    out = []
    for i, x in enumerate(imgs):
        p = eng.plan(int(x.shape[1]), int(x.shape[2]))
        out += _per_image(p, x[None])
        if check_levels is not None:
            stage_out = {B["name"].split("/")[0]: B["out"] for B in p.blocks}
            maps = [p.x_col, p.p1, stage_out["res3"], stage_out["res4"], stage_out["res5"]]
            assert [tuple(v) for v in check_levels.level_ext[:, i].cpu().tolist()] == [tuple(m.hi.shape[:2]) for m in maps], i
    return out


@pytest.fixture(scope="module")
def r50():
    from frcnn_b200.resnet_engine import ResNetBatchEngine
    return ResNetBatchEngine(orc.make_resnet_params(50, seed=11), 50, precision="bf16x3", anchors=ANCHORS, with_detect=True,
                             det_conf=0.05, post_n=100)


def test_resnet50_canvas_plan_equals_forward_plan(r50):
    """ResNetCanvasBatchPlan, N = 4 on a 192 x 256 canvas poisoned outside the images = ResNetForwardPlan per image on every
    result field (per-class NMS lists included); the same graph then serves another size mix with no re-capture."""
    from frcnn_b200.resnet_engine import ResNetCanvasBatchPlan
    plan = r50.canvas_plan(4, 192, 256)
    assert isinstance(plan, ResNetCanvasBatchPlan) and r50.canvas_plan(4, 192, 256) is plan
    plan.x_in.copy_(_poison_like(plan.x_in))
    first = _images([(160, 224), (150, 201), (97, 129)], seed=30)
    plan.forward(first)
    want = _want(r50, first, check_levels=plan)
    for rep in range(2):
        got = _result(plan)
        for n, w in enumerate(want):
            assert w["count"] > 0
            _assert_same(got[n], w, ("first mix", rep, n))
        assert got[3]["count"] == 0 and not got[3]["keep_count"].any()
        plan.forward(None)
    graph = plan.graph
    assert graph is not None
    second = _images([(64, 96), (192, 256), (33, 250), (150, 201)], seed=40)
    clips = [(64, 64), (192, 256), (33, 250), (150, 201)]
    plan.forward(second, img_infos=clips)
    assert plan.graph is graph and plan.image_sizes == [(64, 96), (192, 256), (33, 250), (150, 201)]
    got = _result(plan)
    for n, x in enumerate(second):
        p = r50.plan(int(x.shape[1]), int(x.shape[2]))
        p.set_clip(*clips[n])
        _assert_same(got[n], _per_image(p, x[None])[0], ("second mix", n))


def test_resnet50_batch_plan_equals_forward_plan(r50):
    """ResNetBatchPlan, N = 2 images of one shape = ResNetForwardPlan per image; Engine.forward_batch returns the same."""
    from frcnn_b200.resnet_engine import ResNetBatchPlan
    H, W = 150, 201
    imgs = _images([(H, W), (H, W)], seed=50)
    x = torch.stack(imgs)
    bplan = r50.batch_plan(2, H, W)
    assert isinstance(bplan, ResNetBatchPlan) and bplan.level_ext is None
    bplan.forward(x)
    want = _want(r50, imgs)
    for n, (g, w) in enumerate(zip(_result(bplan), want)):
        assert w["count"] > 0
        _assert_same(g, w, n)
    res = r50.forward_batch(x)
    for (p, b), w in zip(res, want):
        assert np.array_equal(p.cpu().numpy(), w["prob"]) and np.array_equal(b.cpu().numpy(), w["boxes"])


def test_resnet_engine_forward_images_and_raw_photos(r50):
    """Engine.forward_images on a ResNetBatchEngine (chunks of N on the default canvas) = ResNetForwardPlan per image;
    detect_images (raw photos) raises FrcnnError before anything is queued."""
    from frcnn_b200._lib import FrcnnError
    imgs = _images([(150, 201), (64, 64), (100, 37)], seed=60)
    want = _want(r50, imgs)
    res = r50.forward_images(imgs, N=2)
    assert any(k[:4] == ("canvas", 2, 192, 256) for k in r50.plans)
    for (p, b), w in zip(res, want):
        assert p.shape[0] == w["count"] and np.array_equal(p.cpu().numpy(), w["prob"]) and np.array_equal(b.cpu().numpy(), w["boxes"])
    photos = [np.zeros((120, 160, 3), np.uint8)]
    with pytest.raises(FrcnnError, match="raw_input"):
        r50.detect_images(photos)
    with pytest.raises(FrcnnError, match="raw_input"):
        r50.raw_canvas_plan(photos)


def test_resnet101_canvas_headline_sizes():
    """ResNet-101 at the VOC-style sizes 600 x 800 and 600 x 1000 in one 600 x 1000 canvas (bf16x3, per-class NMS) =
    ResNetForwardPlan on each."""
    from frcnn_b200.resnet_engine import ResNetCanvasBatchPlan, ResNetForwardPlan, ResNetPackedWeights
    wts = ResNetPackedWeights(orc.make_resnet_params(101, seed=12), 101, "bf16x3")
    kw = dict(anchors=ANCHORS, feat_stride=32, with_detect=True, det_conf=0.05)
    imgs = _images([(600, 800), (600, 1000)], seed=70)
    plan = ResNetCanvasBatchPlan(wts, 2, 600, 1000, **kw)
    plan.forward(imgs)
    got = _result(plan)
    del plan
    for n, x in enumerate(imgs):
        p1 = ResNetForwardPlan(wts, 600, int(x.shape[2]), **kw)
        w = _per_image(p1, x[None])[0]
        assert w["count"] > 0
        _assert_same(got[n], w, n)
        del p1
