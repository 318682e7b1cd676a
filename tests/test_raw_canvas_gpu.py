"""GPU tests of the raw-photo front end of canvas batches: frcnn_preprocess_bgr8_canvas (ops.preprocess_pack_canvas) resizes,
mean-subtracts and packs N uint8 photos of different sizes straight into the first-layer planes of a canvas, and
CanvasBatchPlan(raw_input=True), Engine.detect_images and CanvasStreamRunner run detection from those photos.  Everything
is compared bit for bit: the planes against the oracle's resize followed by the existing pack, each image's results against
a ForwardPlan on that image alone, and no descriptor value may move an access outside the arena or the planes."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_batch_gpu import ANCHORS, _assert_same, _bits
from test_canvas_batch_gpu import _canvas_result, _ext, _poison_like, _want

pytestmark = pytest.mark.gpu
MEANS = orc.PIXEL_MEANS
# (375,500) -> 600x800, (333,500) -> 600x901, (720,1280) -> 562x1000, (600,600) unscaled, (97,211) -> 460x1000,
# (1,1) -> 600x600 of one value; None = an empty slot
SOURCES = [(375, 500), (333, 500), (720, 1280), None, (600, 600), (97, 211), (1, 1)]
CANVASES = {"608x1024": (608, 1024), "tight": (600, 1000)}


@pytest.fixture(scope="module")
def params():
    return orc.make_params(seed=1234)


def _ops():
    from frcnn_b200 import ops
    return ops


def _photo(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, (shape[0], shape[1], 3), dtype=np.uint8)


def _photos(shapes, seed=0):
    return [None if s is None else _photo(s, seed + i) for i, s in enumerate(shapes)]


def _descriptors(imgs, offsets=None):
    """(arena bytes as a uint8 array, src_off, src_hw, inv_scale, extents) with the images one after the other (64-byte
    aligned) or at the given offsets."""
    from frcnn_b200 import preprocess
    src_off, src_hw, inv, ext, end = [], [], [], [], 0
    for n, im in enumerate(imgs):
        if im is None:
            src_off.append(0), src_hw.append((0, 0)), inv.append(0.0), ext.append((0, 0))
            continue
        off = (end + 63) // 64 * 64 if offsets is None else offsets[n]
        s, H, W = preprocess.plan_size(im.shape[0], im.shape[1])
        src_off.append(off), src_hw.append(im.shape[:2]), inv.append(1.0 / s), ext.append((H, W))
        end = max(end, off + im.size)
    arena = np.full((end,), 0x5A, dtype=np.uint8)
    for im, off in zip(imgs, src_off):
        if im is not None:
            arena[off:off + im.size] = im.reshape(-1)
    return arena, src_off, src_hw, inv, ext


def _fused(arena_t, src_off, src_hw, inv, ext, Hc, Wc, prec, means=MEANS):
    """ops.preprocess_pack_canvas into poisoned planes."""
    ops = _ops()
    N = len(src_off)
    hi = _poison_like(torch.empty((N, ops._lib.load().frcnn_image_c8_elems(Hc, Wc)), dtype=torch.bfloat16, device="cuda"))
    out = ops.preprocess_pack_canvas(arena_t, torch.tensor(src_off, dtype=torch.int64, device="cuda"), _ext(src_hw),
                                     torch.tensor(inv, dtype=torch.float64, device="cuda"), _ext(ext), Hc, Wc, means,
                                     precision=prec, out=ops.Act(hi, hi.clone() if prec == "bf16x3" else None))
    torch.cuda.synchronize()
    return out


def _packed(floats, Hc, Wc, prec):
    """The existing pack of float32 (3,H,W) images (None = empty) copied into a zero canvas: (Act, [(H, W)])."""
    x = torch.zeros((len(floats), 3, Hc, Wc), device="cuda")
    ext = []
    for n, f in enumerate(floats):
        f = None if f is None else torch.as_tensor(f)[:, :Hc, :Wc]
        ext.append((0, 0) if f is None else tuple(f.shape[1:]))
        if f is not None:
            x[n, :, :f.shape[1], :f.shape[2]] = f.cuda()
    return _ops().pack_image_c8_batch(x, precision=prec, extents=_ext(ext)), ext


def _assert_planes(got, want, ext, Hc, Wc):
    """Bit-identical planes, and exactly 0 at every stored pixel outside each image (pad columns and slack included)."""
    rows = Hc * (Wc + 2) * 8
    for g, w in ((got.hi, want.hi),) + (((got.lo, want.lo),) if want.lo is not None else ()):
        assert torch.equal(_bits(g), _bits(w))
        for n, (h, wd) in enumerate(ext):
            plane = g[n, :rows].view(Hc, Wc + 2, 8).clone()
            assert h == 0 or _bits(plane[:h, 1:wd + 1, :3]).any().item(), n
            plane[:h, 1:wd + 1] = 0
            assert not _bits(plane).any().item() and not _bits(g[n, rows:]).any().item(), n
    assert (got.lo is None) == (want.lo is None)


# ------------------------------------------------------------------------------------------------------- 1-3: the kernel
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
@pytest.mark.parametrize("canvas", list(CANVASES))
def test_fused_kernel_equals_oracle_resize_then_pack(canvas, prec):
    Hc, Wc = CANVASES[canvas]
    imgs = _photos(SOURCES, seed=10)
    arena, src_off, src_hw, inv, ext = _descriptors(imgs)
    got = _fused(torch.from_numpy(arena).cuda(), src_off, src_hw, inv, ext, Hc, Wc, prec)
    want, ext2 = _packed([None if im is None else orc.img_preprocessing(im)[0] for im in imgs], Hc, Wc, prec)
    assert ext2 == ext
    _assert_planes(got, want, ext, Hc, Wc)


def test_fused_kernel_equals_device_preprocess_then_pack():
    from frcnn_b200 import preprocess
    Hc, Wc = CANVASES["608x1024"]
    imgs = _photos(SOURCES, seed=20)
    arena, src_off, src_hw, inv, ext = _descriptors(imgs)
    got = _fused(torch.from_numpy(arena).cuda(), src_off, src_hw, inv, ext, Hc, Wc, "bf16x3")
    want, _ = _packed([None if im is None else preprocess.img_preprocessing(im)[0] for im in imgs], Hc, Wc, "bf16x3")
    _assert_planes(got, want, ext, Hc, Wc)


def test_fused_kernel_other_means_and_unaligned_shuffled_offsets():
    """Means other than the default, and the images at odd byte offsets in an order unrelated to their slots."""
    Hc, Wc = 600, 1000
    means = np.array([10.5, 200.25, 0.1])
    imgs = _photos([(333, 500), None, (97, 211), (375, 500)], seed=30)
    offsets = [700001, 0, 7, 61403 + 7]              # slot 2's image first, then slot 3's, then slot 0's
    assert offsets[3] >= offsets[2] + imgs[2].size and offsets[0] >= offsets[3] + imgs[3].size
    arena, src_off, src_hw, inv, ext = _descriptors(imgs, offsets)
    got = _fused(torch.from_numpy(arena).cuda(), src_off, src_hw, inv, ext, Hc, Wc, "bf16x3", means=means)
    want, _ = _packed([None if im is None else orc.img_preprocessing(im, pixel_means=means)[0] for im in imgs], Hc, Wc, "bf16x3")
    _assert_planes(got, want, ext, Hc, Wc)
    other, _ = _packed([None if im is None else orc.img_preprocessing(im)[0] for im in imgs], Hc, Wc, "bf16x3")
    assert not torch.equal(_bits(got.hi), _bits(other.hi))


# ----------------------------------------------------------------------------------------------- 4: descriptor safety
def test_bad_descriptors_give_empty_slots_and_touch_nothing_else():
    """The arena is the middle third of a larger allocation filled with 0xAB, so a source that overruns it would be read by
    value.  A slot whose source is not inside the arena (by one byte, by a negative offset, by a size whose byte count
    wraps around in 32 bits) or has a non-positive size is all zero; its neighbours are unaffected, the first and the last
    byte of the arena are usable, and an extent larger than the canvas is clamped."""
    from frcnn_b200 import preprocess
    Hc, Wc = 96, 160
    a, b = _photo((40, 60), 1), _photo((30, 50), 2)              # resize to 600 x 900 and 600 x 1000: both clamped to the canvas
    A = 1 << 15
    big = torch.full((3 * A,), 0xAB, dtype=torch.uint8)
    big[A:A + a.size] = torch.from_numpy(a.reshape(-1))
    big[2 * A - b.size:2 * A] = torch.from_numpy(b.reshape(-1))
    arena = big.cuda()[A:2 * A]
    sa, sb = preprocess.plan_size(40, 60), preprocess.plan_size(30, 50)
    full = (600, 1000)
    slots = [                                          # (src_off, src_hw, inv_scale, extents)
        (0, (40, 60), 1.0 / sa[0], sa[1:]),                                   # 0: the first byte of the arena
        (A - b.size + 1, (30, 50), 1.0 / sb[0], sb[1:]),                      # 1: overruns by one byte
        (-64, (40, 60), 1.0 / sa[0], sa[1:]),                                 # 2: negative offset
        (0, (0, 60), 1.0, full), (0, (-3, 7), 1.0, full),                     # 3, 4: non-positive size
        (0, (1, 1431655766), 1.0, (1, 2)),                                    # 5: 3 * h0 * w0 = 2^32 + 2
        (A + 1, (1, 1), 1.0, full),                                           # 6: offset past the end
        (A - b.size, (30, 50), 1.0 / sb[0], (sb[1] + 50, sb[2] + 9)),         # 7: the last byte; extent beyond the canvas
        (0, (40, 60), 0.0, sa[1:]),                                           # 8: a zero 1 / im_scale reads pixel (0, 0) only,
        (0, (40, 60), 1e300, sa[1:]),                                         # 9: a huge one the last pixel only
    ]
    got = _fused(arena, [s[0] for s in slots], [s[1] for s in slots], [s[2] for s in slots], [s[3] for s in slots], Hc, Wc, "bf16x3")
    fa, fb = orc.img_preprocessing(a)[0], orc.img_preprocessing(b)[0]
    first = np.broadcast_to((a[0, 0] - MEANS.reshape(3)).astype(np.float32).reshape(3, 1, 1), (3, Hc, Wc)).copy()
    last = np.broadcast_to((a[-1, -1] - MEANS.reshape(3)).astype(np.float32).reshape(3, 1, 1), (3, Hc, Wc)).copy()
    want, ext = _packed([fa, None, None, None, None, None, None, fb, first, last], Hc, Wc, "bf16x3")
    assert ext == [(Hc, Wc)] + [(0, 0)] * 6 + [(Hc, Wc)] * 3
    _assert_planes(got, want, ext, Hc, Wc)


# --------------------------------------------------------------------------------------------------------- 5: the plan
def _raw_want(eng, imgs, clips=None):
    from frcnn_b200 import preprocess
    return _want(eng, [preprocess.img_preprocessing(im)[0] for im in imgs], clips)


def test_raw_canvas_plan_equals_forward_plan_per_image(params):
    """CanvasBatchPlan(raw_input=True), N = 4 on a 600 x 1000 canvas: every result field of every photo = ForwardPlan on
    preprocess.img_preprocessing of that photo alone; the same graph then serves a second mix (a smaller image where a
    larger one was, two empty slots), also with forward.py's clip bounds (H, H); CUDA-tensor photos give the same."""
    from frcnn_b200 import preprocess
    from frcnn_b200.engine import CanvasBatchPlan, Engine
    eng = Engine(params, precision="bf16x3", anchors=ANCHORS, with_detect=True, det_conf=0.05)
    plan = eng.canvas_plan(4, 600, 1000, raw_input=True, arena_bytes=5 << 20)
    assert isinstance(plan, CanvasBatchPlan) and plan.x_in is None and plan.extents.data_ptr() == plan.block.data_ptr()
    first = _photos([(300, 500), (375, 500), (333, 500), (720, 1280)], seed=40)
    want = _raw_want(eng, first)
    for rep in range(2):
        probs, boxes, counts, scales = plan.forward_raw(first)
        assert scales == [preprocess.plan_size(*im.shape[:2])[0] for im in first]
        for n, (g, w) in enumerate(zip(_canvas_result(plan), want)):
            assert w["count"] > 0 and w["conf_count"].sum() > 0
            _assert_same(g, w, ("first mix", rep, n))
    assert plan.image_sizes == [(600, 1000), (600, 800), (600, 901), (562, 1000)]
    graph = plan.graph
    assert graph is not None
    second = _photos([(97, 211), (375, 500)], seed=50)           # 460 x 1000 where 600 x 1000 was
    for clips in (None, [(460, 460), (600, 600)]):
        want2 = _raw_want(eng, second, clips)
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
    # the raw front end replaces the first launch: the float-input canvas plan has as many
    twin = plan.clone()
    assert twin.raw_input and twin.arena_bytes == plan.arena_bytes and twin.pixel_means == plan.pixel_means
    del twin
    floats = eng.canvas_plan(4, 600, 1000)
    floats.forward([preprocess.img_preprocessing(second[1])[0]])
    assert plan.n_launches == floats.n_launches > 0


def test_raw_plan_refuses_what_does_not_fit(params):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.engine import CanvasStreamRunner, Engine
    eng = Engine(params, precision="bf16", anchors=ANCHORS)
    plan = eng.canvas_plan(2, 600, 1000, raw_input=True, arena_bytes=1 << 20)
    ok = _photo((300, 500), 1)
    for bad in ([_photo((500, 300), 2)], [ok, ok, ok], [ok, _photo((400, 500), 3)], [ok.astype(np.float32)], [ok[:, :, 0]],
                [ok, torch.from_numpy(ok).cuda()]):
        with pytest.raises(FrcnnError):
            plan.forward_raw(bad)
    with pytest.raises(FrcnnError):
        plan.forward([torch.zeros((3, 600, 1000), device="cuda")])
    with pytest.raises(FrcnnError):
        eng.canvas_plan(2, 600, 1000).forward_raw([ok])
    with pytest.raises(FrcnnError):
        CanvasStreamRunner(plan)                    # no per-class NMS in this plan
    assert plan.graph is None                       # nothing was queued


# ------------------------------------------------------------------------------------- 6, 7: detections, host to host
STREAM_SHAPES = [(300, 500), (375, 500), (333, 500)]


@pytest.fixture(scope="module")
def stream_case(params):
    """10 photos of three sizes and, per photo, what forward.py's loop gives on the one-image path."""
    from frcnn_b200 import preprocess
    from frcnn_b200.engine import Engine
    eng = Engine(params, precision="bf16x3", anchors=ANCHORS)
    imgs = [_photo(STREAM_SHAPES[(i * 7) % 3], 60 + i) for i in range(10)]
    want = []
    for im in imgs:
        x, s = preprocess.img_preprocessing(im)
        prob, boxes, _ = eng(x)
        want.append((preprocess.detections(prob, boxes, s, nms_thresh=0.3, conf=0.05), s))
    assert all(len(d) > 0 for d, _ in want)
    return eng, imgs, want


def test_detect_images_equals_one_image_path(stream_case):
    eng, imgs, want = stream_case
    got = eng.detect_images(imgs[:6], N=4, conf=0.05)
    assert any(k[:4] == ("canvas", 4, 640, 1024) for k in eng.plans)
    assert len(got) == 6 and all(g == w[0] and len(g) > 0 for g, w in zip(got, want))
    assert eng.detect_images([]) == []


@pytest.mark.parametrize("lanes", [1, 2])
def test_canvas_stream_runner_delivers_in_order(stream_case, lanes):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.engine import CanvasStreamRunner
    eng, imgs, want = stream_case
    plan = eng.raw_canvas_plan(imgs, N=4, conf=0.05)
    runner = CanvasStreamRunner(plan, depth=2, lanes=lanes)
    seen = []
    res = runner.run(imgs, on_result=lambda i, dets, s: seen.append((i, dets, s)))
    torch.cuda.synchronize()
    assert [i for i, _, _ in seen] == list(range(10)) and res == [d for _, d, _ in seen]
    assert all(d == w[0] and s == w[1] for (_, d, s), w in zip(seen, want))
    assert runner.h2d_copies == 3 and runner.h2d_bytes < 3 * (plan.header_bytes + plan.arena_bytes)
    # a photo that does not fit the canvas (portrait: 800 x 600) or the arena, last in the list: nothing runs
    for bad in (_photo((500, 375), 1), _photo((1100, 1100), 2)):
        n = len(seen)
        with pytest.raises(FrcnnError):
            runner.run(imgs[:5] + [bad], on_result=lambda i, dets, s: seen.append((i, dets, s)))
        assert len(seen) == n and runner.h2d_copies == 3
    assert runner.run(imgs[8:], on_result=None) == [want[8][0], want[9][0]]
