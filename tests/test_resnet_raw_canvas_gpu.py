"""GPU tests of the ResNet detector on raw photos: frcnn_preprocess_bgr8_canvas_im2col (ops.preprocess_im2col_canvas) resizes,
mean-subtracts and writes the first-layer im2col planes of N uint8 photos of different sizes in one launch, and
ResNetRawCanvasBatchPlan, ResNetPhotoEngine.detect_images and CanvasStreamRunner run the ResNet detector from those photos.
Everything is compared bit for bit: the planes against the resize followed by a copy into a zeroed canvas and the existing
float im2col, each image's results against a ResNetForwardPlan on that image alone, and no descriptor value may move an
access outside the arena or the planes."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_batch_gpu import ANCHORS, _assert_same, _bits
from test_canvas_batch_gpu import _canvas_result, _ext, _poison_like
from test_raw_canvas_gpu import CANVASES, MEANS, SOURCES, STREAM_SHAPES, _descriptors, _photo, _photos, _raw_want

pytestmark = pytest.mark.gpu
CONV1 = (7, 2, 3, 160)                 # ksize, stride, pad, K_pad of the ResNet trunk's conv1


def _ops():
    from frcnn_b200 import ops
    return ops


def _conv_out(e, ks, stride, pad):
    t = e + 2 * pad - ks
    return 0 if t < 0 else t // stride + 1


def _fused(arena_t, src_off, src_hw, inv, ext, Hc, Wc, prec, means=MEANS, geom=CONV1):
    """ops.preprocess_im2col_canvas into poisoned planes followed by 4096 poisoned guard elements, which must stay as they were."""
    ops = _ops()
    ks, st, pd, kp = geom
    shape = (len(src_off), _conv_out(Hc, ks, st, pd), _conv_out(Wc, ks, st, pd), kp)
    n = int(np.prod(shape))
    bufs = [_poison_like(torch.empty((n + 4096,), dtype=torch.bfloat16, device="cuda")) for _ in range(2 if prec == "bf16x3" else 1)]
    planes = [b[:n].view(shape) for b in bufs] + [None]
    tails = [b[n:].clone() for b in bufs]
    out = ops.preprocess_im2col_canvas(arena_t, torch.tensor(src_off, dtype=torch.int64, device="cuda"), _ext(src_hw),
                                       torch.tensor(inv, dtype=torch.float64, device="cuda"), _ext(ext), Hc, Wc, means, ks, st, pd,
                                       kp, precision=prec, out=ops.Act(planes[0], planes[1]))
    torch.cuda.synchronize()
    assert all(torch.equal(_bits(b[n:]), _bits(t)) for b, t in zip(bufs, tails))
    return out


def _im2col(floats, Hc, Wc, prec, geom=CONV1):
    """The existing path: float32 (3,H,W) images (None = empty) copied into a zeroed canvas (cropped to it), then
    ops.pack_image_im2col_batch with extents.  Returns (Act, [(H, W)])."""
    ks, st, pd, kp = geom
    x = torch.zeros((len(floats), 3, Hc, Wc), device="cuda")
    ext = []
    for n, f in enumerate(floats):
        f = None if f is None else torch.as_tensor(f)[:, :Hc, :Wc]
        ext.append((0, 0) if f is None else tuple(f.shape[1:]))
        if f is not None:
            x[n, :, :f.shape[1], :f.shape[2]] = f.cuda()
    return _ops().pack_image_im2col_batch(x, ks, st, pd, kp, precision=prec, extents=_ext(ext)), ext


def _assert_planes(got, want, ext, geom=CONV1):
    """Bit-identical planes, something nonzero inside every image and exactly 0 outside each image's output extent."""
    ks, st, pd, _ = geom
    assert (got.lo is None) == (want.lo is None)
    for g, w in ((got.hi, want.hi),) + (((got.lo, want.lo),) if want.lo is not None else ()):
        assert g.shape == w.shape and torch.equal(_bits(g), _bits(w))
        for n, (h, wd) in enumerate(ext):
            oh, ow = _conv_out(h, ks, st, pd), _conv_out(wd, ks, st, pd)
            plane = g[n].clone()
            assert oh == 0 or ow == 0 or _bits(plane[:oh, :ow]).any().item(), n
            plane[:oh, :ow] = 0
            assert not _bits(plane).any().item(), n


# ------------------------------------------------------------------------------------------------------- 1-4: the kernel
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
@pytest.mark.parametrize("canvas", list(CANVASES))
def test_fused_kernel_equals_oracle_resize_then_im2col(canvas, prec):
    """The VGG16 raw test's sources (600x800, 600x901, 562x1000, an empty slot, 600x600, 460x1000, 600x600 of one value) on
    a 608x1024 and the tight 600x1000 canvas = the oracle's img_preprocessing, a zeroed canvas and the float im2col."""
    Hc, Wc = CANVASES[canvas]
    imgs = _photos(SOURCES, seed=110)
    arena, src_off, src_hw, inv, ext = _descriptors(imgs)
    got = _fused(torch.from_numpy(arena).cuda(), src_off, src_hw, inv, ext, Hc, Wc, prec)
    want, ext2 = _im2col([None if im is None else orc.img_preprocessing(im)[0] for im in imgs], Hc, Wc, prec)
    assert ext2 == ext
    _assert_planes(got, want, ext)


def test_fused_kernel_equals_device_preprocess_then_im2col():
    from frcnn_b200 import preprocess
    Hc, Wc = CANVASES["608x1024"]
    imgs = _photos(SOURCES, seed=120)
    arena, src_off, src_hw, inv, ext = _descriptors(imgs)
    got = _fused(torch.from_numpy(arena).cuda(), src_off, src_hw, inv, ext, Hc, Wc, "bf16x3")
    want, _ = _im2col([None if im is None else preprocess.img_preprocessing(im)[0] for im in imgs], Hc, Wc, "bf16x3")
    _assert_planes(got, want, ext)


def test_fused_kernel_other_means_and_unaligned_shuffled_offsets():
    """Means other than the default, and the images at odd byte offsets in an order unrelated to their slots."""
    Hc, Wc = 600, 1000
    means = np.array([10.5, 200.25, 0.1])
    imgs = _photos([(333, 500), None, (97, 211), (375, 500)], seed=130)
    offsets = [700001, 0, 7, 61403 + 7]
    assert offsets[3] >= offsets[2] + imgs[2].size and offsets[0] >= offsets[3] + imgs[3].size
    arena, src_off, src_hw, inv, ext = _descriptors(imgs, offsets)
    got = _fused(torch.from_numpy(arena).cuda(), src_off, src_hw, inv, ext, Hc, Wc, "bf16x3", means=means)
    want, _ = _im2col([None if im is None else orc.img_preprocessing(im, pixel_means=means)[0] for im in imgs], Hc, Wc, "bf16x3")
    _assert_planes(got, want, ext)
    other, _ = _im2col([None if im is None else orc.img_preprocessing(im)[0] for im in imgs], Hc, Wc, "bf16x3")
    assert not torch.equal(_bits(got.hi), _bits(other.hi))


def test_bad_descriptors_give_empty_or_clamped_slots_and_touch_nothing_else():
    """The arena is the middle third of a larger allocation filled with 0xAB, so a source that overruns it would be read by
    value, and the planes are followed by poisoned guard elements.  A slot whose source is not inside the arena (by one
    byte, by a negative offset, past its end, by a size whose byte count wraps around in 32 bits) or has a non-positive size
    is all zero; an extent larger than the canvas is clamped; a 1 / im_scale of 0, -inf, +inf, 1e300 or NaN reads the first
    or the last source pixel only."""
    from frcnn_b200 import preprocess
    Hc, Wc = 96, 160
    a, b = _photo((40, 60), 1), _photo((30, 50), 2)              # resize to 600 x 900 and 600 x 1000: both clamped to the canvas
    A = 1 << 15
    big = torch.full((3 * A,), 0xAB, dtype=torch.uint8)
    big[A:A + a.size] = torch.from_numpy(a.reshape(-1))
    big[2 * A - b.size:2 * A] = torch.from_numpy(b.reshape(-1))
    big = big.cuda()
    before = big.clone()
    arena = big[A:2 * A]
    sa, sb = preprocess.plan_size(40, 60), preprocess.plan_size(30, 50)
    full = (600, 1000)
    inf = float("inf")
    slots = [                                          # (src_off, src_hw, inv_scale, extents)
        (0, (40, 60), 1.0 / sa[0], sa[1:]),                                   # 0: the first byte of the arena
        (A - b.size + 1, (30, 50), 1.0 / sb[0], sb[1:]),                      # 1: overruns by one byte
        (-64, (40, 60), 1.0 / sa[0], sa[1:]),                                 # 2: negative offset
        (0, (0, 60), 1.0, full), (0, (-3, 7), 1.0, full),                     # 3, 4: non-positive size
        (0, (1, 1431655766), 1.0, (1, 2)),                                    # 5: 3 * h0 * w0 = 2^32 + 2
        (A + 1, (1, 1), 1.0, full),                                           # 6: offset past the end
        (A - b.size, (30, 50), 1.0 / sb[0], (sb[1] + 50, sb[2] + 9)),         # 7: the last byte; extent beyond the canvas
        (0, (40, 60), 0.0, sa[1:]),                                           # 8: first pixel
        (0, (40, 60), -inf, sa[1:]),                                          # 9: first pixel
        (0, (40, 60), 1e300, sa[1:]),                                         # 10: last pixel
        (0, (40, 60), inf, (10 ** 9, 10 ** 9)),                               # 11: last pixel; a huge extent
        (0, (40, 60), float("nan"), (50, 70)),                                # 12: NaN: one end pixel
    ]
    got = _fused(arena, [s[0] for s in slots], [s[1] for s in slots], [s[2] for s in slots], [s[3] for s in slots], Hc, Wc, "bf16x3")
    assert torch.equal(big, before)
    fa, fb = orc.img_preprocessing(a)[0], orc.img_preprocessing(b)[0]
    pixel = lambda p: np.broadcast_to((p - MEANS.reshape(3)).astype(np.float32).reshape(3, 1, 1), (3, Hc, Wc)).copy()  # noqa: E731
    first, last = pixel(a[0, 0]), pixel(a[-1, -1])
    for end in (first, last):
        want, ext = _im2col([fa, None, None, None, None, None, None, fb, first, first, last, last, end[:, :50, :70]], Hc, Wc, "bf16x3")
        if torch.equal(_bits(got.hi[-1]), _bits(want.hi[-1])):
            break
    assert ext == [(Hc, Wc)] + [(0, 0)] * 6 + [(Hc, Wc)] * 5 + [(50, 70)]
    _assert_planes(got, want, ext)


@pytest.mark.parametrize("geom", [(3, 1, 1, 32), (1, 1, 0, 8), (5, 3, 0, 80), (11, 4, 2, 368), (45, 1, 0, 6080)],
                         ids=lambda g: "k%ds%dp%dK%d" % g)
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_other_geometries_equal_float_im2col(geom, prec):
    """Filters the entry accepts besides conv1's: a 3x3 / 1, a 1x1, a stride larger than half the filter, a strided 11x11
    and the largest filter (45x45, whose window leaves room for two output rows and one column per CTA), on a canvas
    smaller than the resized photos (their extents are clamped) and on one wider than many column tiles."""
    from frcnn_b200 import preprocess
    for Hc, Wc, shapes in ((70, 90, [(300, 500), (40, 40), None]), (48, 1200, [(20, 60), (33, 50)])):
        imgs = _photos(shapes, seed=140 + Hc)
        arena, src_off, src_hw, inv, ext = _descriptors(imgs)
        got = _fused(torch.from_numpy(arena).cuda(), src_off, src_hw, inv, ext, Hc, Wc, prec, geom=geom)
        want, ext2 = _im2col([None if im is None else preprocess.img_preprocessing(im)[0] for im in imgs], Hc, Wc, prec, geom=geom)
        assert ext2 == [(0, 0) if e == (0, 0) else (min(e[0], Hc), min(e[1], Wc)) for e in ext]
        _assert_planes(got, want, ext2, geom=geom)


# --------------------------------------------------------------------------------------------------------- 5: the plan
@pytest.fixture(scope="module")
def r50():
    from frcnn_b200.resnet_engine import ResNetPhotoEngine
    return ResNetPhotoEngine(orc.make_resnet_params(50, seed=21), 50, precision="bf16x3", anchors=ANCHORS, with_detect=True,
                             det_conf=0.02, post_n=100)


def test_resnet50_raw_canvas_plan_equals_forward_plan_per_image(r50):
    """ResNetRawCanvasBatchPlan, N = 4 on a 600 x 1000 canvas: every result field of every photo = ResNetForwardPlan on
    preprocess.img_preprocessing of that photo alone; the same graph then serves a second mix (two empty slots), also with
    forward.py's clip bounds (H, H); CUDA-tensor photos give the same; the plan survives clone() and has the float canvas
    plan's launch count."""
    from frcnn_b200 import preprocess
    from frcnn_b200.resnet_engine import ResNetRawCanvasBatchPlan
    plan = r50.canvas_plan(4, 600, 1000, raw_input=True, arena_bytes=5 << 20)
    assert isinstance(plan, ResNetRawCanvasBatchPlan) and plan.x_in is None and plan.extents.data_ptr() == plan.block.data_ptr()
    first = _photos([(300, 500), (375, 500), (333, 500), (720, 1280)], seed=150)
    want = _raw_want(r50, first)
    for rep in range(2):
        probs, boxes, counts, scales = plan.forward_raw(first)
        assert scales == [preprocess.plan_size(*im.shape[:2])[0] for im in first]
        for n, (g, w) in enumerate(zip(_canvas_result(plan), want)):
            assert w["count"] > 0
            _assert_same(g, w, ("first mix", rep, n))
    assert plan.image_sizes == [(600, 1000), (600, 800), (600, 901), (562, 1000)]
    graph = plan.graph
    assert graph is not None
    second = _photos([(97, 211), (375, 500)], seed=160)           # 460 x 1000 where 600 x 1000 was
    for clips in (None, [(460, 460), (600, 600)]):
        want2 = _raw_want(r50, second, clips)
        plan.forward_raw(second, img_infos=clips)
        assert plan.graph is graph and plan.image_sizes == [(460, 1000), (600, 800), (0, 0), (0, 0)]
        got = _canvas_result(plan)
        for n, w in enumerate(want2):
            _assert_same(got[n], w, ("second mix", clips, n))
        for n in (2, 3):
            assert got[n]["count"] == 0 and not got[n]["keep_count"].any()
    plan.forward_raw([torch.from_numpy(im).cuda() for im in second], img_infos=[(460, 460), (600, 600)])
    assert plan.graph is graph
    for n, (g, w) in enumerate(zip(_canvas_result(plan), want2)):
        _assert_same(g, w, ("device photos", n))
    twin = plan.clone()
    assert type(twin) is ResNetRawCanvasBatchPlan and twin.raw_input and twin.arena_bytes == plan.arena_bytes
    assert twin.pixel_means == plan.pixel_means
    twin.forward_raw(second, img_infos=[(460, 460), (600, 600)])
    for n, (g, w) in enumerate(zip(_canvas_result(twin), want2)):
        _assert_same(g, w, ("clone", n))
    del twin
    floats = r50.canvas_plan(4, 600, 1000)
    floats.forward([preprocess.img_preprocessing(second[1])[0]])
    assert plan.n_launches == floats.n_launches > 0


# ------------------------------------------------------------------------------------- 6: detections, host to host
@pytest.fixture(scope="module")
def stream_case(r50):
    """10 photos of three sizes and, per photo, what forward.py's loop gives on the one-image ResNet path."""
    from frcnn_b200 import preprocess
    imgs = [_photo(STREAM_SHAPES[(i * 7) % 3], 170 + i) for i in range(10)]
    want = []
    for im in imgs:
        x, s = preprocess.img_preprocessing(im)
        prob, boxes, _ = r50(x, img_info=tuple(x.shape[1:]))        # the per-shape plans are shared with the tests above
        want.append((preprocess.detections(prob, boxes, s, nms_thresh=0.3, conf=0.02), s))
    assert sum(len(d) for d, _ in want) > 0
    return imgs, want


def test_detect_images_equals_one_image_path(r50, stream_case):
    imgs, want = stream_case
    got = r50.detect_images(imgs[:6], N=4, conf=0.02)
    assert any(k[:4] == ("raw_canvas", 4, 640, 1024) for k in r50.plans)
    assert len(got) == 6 and all(g == w[0] for g, w in zip(got, want))
    assert r50.detect_images([]) == []


@pytest.mark.parametrize("lanes", [1, 2])
def test_canvas_stream_runner_equals_detect_images(r50, stream_case, lanes):
    from frcnn_b200.engine import CanvasStreamRunner
    imgs, want = stream_case
    plan = r50.raw_canvas_plan(imgs, N=4, conf=0.02)
    runner = CanvasStreamRunner(plan, depth=2, lanes=lanes)
    seen = []
    res = runner.run(imgs, on_result=lambda i, dets, s: seen.append((i, dets, s)))
    torch.cuda.synchronize()
    assert [i for i, _, _ in seen] == list(range(10)) and res == [d for _, d, _ in seen]
    assert all(d == w[0] and s == w[1] for (_, d, s), w in zip(seen, want))
    assert runner.h2d_copies == 3
    assert res == r50.detect_images(imgs, N=4, conf=0.02)


# ----------------------------------------------------------------------------------------------------- 7: ResNet-101
def test_resnet101_raw_canvas_stream_shapes():
    """ResNet-101: 300x500, 333x500 and 375x500 photos (600x1000, 600x901, 600x800) in one 600 x 1000 canvas = the
    per-image ResNetForwardPlan on each."""
    from frcnn_b200.resnet_engine import ResNetPhotoEngine
    eng = ResNetPhotoEngine(orc.make_resnet_params(101, seed=22), 101, precision="bf16x3", anchors=ANCHORS, with_detect=True,
                            det_conf=0.02)
    photos = _photos(STREAM_SHAPES, seed=180)
    plan = eng.canvas_plan(3, 600, 1000, raw_input=True)
    plan.forward_raw(photos)
    got = _canvas_result(plan)
    want = _raw_want(eng, photos)
    for n, w in enumerate(want):
        assert w["count"] > 0
        _assert_same(got[n], w, n)
