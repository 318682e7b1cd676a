"""GPU tests of the canvas and raw-photo C entries: frcnn_forward_vgg16_canvas (engine.CCanvasForward) against
CanvasBatchPlan, frcnn_detect_vgg16_raw against Engine.detect_images, and frcnn_detection_lists_batch
(ops.detection_lists_batch) against preprocess.result_detections -- every value bit for bit or exactly equal, also from a
captured CUDA graph replayed for a second size mix, and nothing written past an image's list."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_batch_gpu import ANCHORS

pytestmark = pytest.mark.gpu
SENTINEL = -12345
OTHER_MEANS = (90.5, 121.25, 101.0)


@pytest.fixture(scope="module")
def params():
    return orc.make_params(seed=1234)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _images(sizes, seed):
    return [torch.from_numpy(orc.make_image(h, w, seed=seed + i)[0].astype(np.float32)).cuda() for i, (h, w) in enumerate(sizes)]


def _photo(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, (shape[0], shape[1], 3), dtype=np.uint8)


def _assert_equals_plan(cf, plan, what):
    torch.cuda.synchronize()
    for n in range(plan.N):
        assert int(cf.count[n]) == int(plan.result.view(plan.N, plan.block_words)[n, 0]), (what, n)
        assert _same(cf.prob[n], plan.prob[n]) and _same(cf.boxes[n], plan.boxes[n]), (what, n)


# ------------------------------------------------------------------------------------------------ frcnn_forward_vgg16_canvas
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_canvas_c_entry_equals_canvas_plan(params, precision):
    """N = 4 slots of 150 x 201, three images of different sizes (one slot empty, one clip bound forward.py's (H, H)):
    the C call = CanvasBatchPlan on every output; the call captured once into a CUDA graph then serves a second size mix."""
    from frcnn_b200.engine import CCanvasForward, Engine
    eng = Engine(params, precision=precision, anchors=ANCHORS)
    plan = eng.canvas_plan(4, 150, 201)
    cf = CCanvasForward(eng.weights, 4, 150, 201, ANCHORS)
    first, clips = _images([(150, 201), (128, 96), (150, 150)], seed=30), [(150, 201), (128, 128), (150, 150)]
    plan.forward(first, clips)
    cf.forward(first, clips)
    _assert_equals_plan(cf, plan, "eager")
    assert int(cf.count[3]) == 0 and all(int(cf.count[n]) > 0 for n in range(3))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="thread_local"):
        cf.launch()
    second = _images([(64, 80), (150, 201), (16, 16), (100, 33)], seed=50)
    for imgs, cl in ((second, None), (first, clips)):
        cf.prob.fill_(7.0)
        cf.count.fill_(-1)
        cf.set_images(imgs, cl)
        g.replay()
        plan.forward(imgs, cl)
        _assert_equals_plan(cf, plan, "replay")


def test_canvas_c_entry_600x1000(params):
    """The benchmarked canvas, N = 3 with photos' resized sizes."""
    from frcnn_b200.engine import CCanvasForward, Engine
    eng = Engine(params, precision="bf16x3", anchors=ANCHORS)
    plan = eng.canvas_plan(3, 600, 1000)
    cf = CCanvasForward(eng.weights, 3, 600, 1000, ANCHORS)
    imgs = _images([(600, 800), (600, 1000), (600, 901)], seed=7)
    plan.forward(imgs)
    cf.forward(imgs)
    _assert_equals_plan(cf, plan, "600x1000")


# ------------------------------------------------------------------------------------------------ frcnn_detect_vgg16_raw
@pytest.mark.parametrize("clips", ["resized", "forward_py"])
def test_raw_c_entry_equals_detect_images(params, clips):
    """Raw 300x500, 333x500 and 375x500 photos with non-default means: the C call's lists = Engine.detect_images exactly,
    its prob / boxes / count = the plan's; the captured call then serves a second set of photos."""
    from frcnn_b200.engine import CCanvasForward, Engine
    from frcnn_b200 import preprocess
    eng = Engine(params, precision="bf16x3", anchors=ANCHORS)
    shapes = [(300, 500), (333, 500), (375, 500)]
    photos = [_photo(s, 80 + i) for i, s in enumerate(shapes)]
    infos = None if clips == "resized" else [(preprocess.plan_size(*s)[1],) * 2 for s in shapes]
    want = eng.detect_images(photos, N=4, conf=0.05, img_infos=infos, pixel_means=OTHER_MEANS)
    assert all(len(w) > 0 for w in want)
    plan = [p for k, p in eng.plans.items() if k[0] == "canvas"][0]
    assert (plan.N, plan.H, plan.W) == (4, 640, 1024)
    cf = CCanvasForward(eng.weights, 4, 640, 1024, ANCHORS, raw_input=True, pixel_means=OTHER_MEANS, arena_bytes=plan.arena_bytes,
                        det_conf=0.05)
    assert cf.header_bytes == plan.header_bytes
    got = cf.detect_raw(photos, infos)
    assert got == want
    _assert_equals_plan(cf, plan, "raw")
    assert int(cf.det_count[3]) == 0 and [int(v) for v in cf.det_count[:3]] == [len(w) for w in want]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="thread_local"):
        cf.launch()
    second = [_photo(s, 90 + i) for i, s in enumerate([(375, 500), (300, 500)])]
    want2 = eng.detect_images(second, N=4, conf=0.05, pixel_means=OTHER_MEANS)
    cf.lists.fill_(SENTINEL)
    cf.stage_raw(second)
    g.replay()
    assert cf.fetch_detections(2) == want2
    assert int(cf.det_count[2]) == int(cf.det_count[3]) == 0


# ------------------------------------------------------------------------------------------------ frcnn_detection_lists_batch
def _embedded(shape, dtype, pad=96):
    """A dense tensor of `shape` inside a SENTINEL-filled allocation with `pad` guard elements on each side."""
    n = int(np.prod(shape))
    buf = torch.full((pad + n + pad,), SENTINEL, dtype=torch.int32, device="cuda")
    return buf, buf[pad:pad + n].view(dtype).view(shape)


def _run_lists(prob, boxes, keep_idx, conf_count, im_scale, stride_pad=0):
    """ops.detection_lists_batch on host arrays (inputs at image strides padded by stride_pad elements), outputs embedded in
    poisoned allocations.  Returns (per-image lists, dets, scores, det_count, guard buffers)."""
    from frcnn_b200 import ops
    N, R, NC = prob.shape
    cap = (NC - 1) * R

    def dev(a, dtype):
        flat = np.full((N, int(np.prod(a.shape[1:])) + stride_pad), SENTINEL, dtype=np.int32).view(dtype)
        flat[:, :flat.shape[1] - stride_pad] = a.reshape(N, -1)
        return torch.from_numpy(flat).cuda()[:, :flat.shape[1] - stride_pad].view(a.shape)

    bufs = [_embedded((N, cap, 5), torch.int32), _embedded((N, cap), torch.float32), _embedded((N,), torch.int32)]
    dets, scores, count = ops.detection_lists_batch(dev(prob, np.float32), dev(boxes, np.float32), dev(keep_idx, np.int32),
                                                    dev(conf_count, np.int32),
                                                    torch.tensor(im_scale, dtype=torch.float64, device="cuda"),
                                                    out=tuple(b[1] for b in bufs))
    torch.cuda.synchronize()
    d, s, c = dets.cpu().numpy(), scores.cpu().numpy(), count.cpu().numpy()
    for n in range(N):                                    # nothing past an image's list, nothing outside the outputs
        assert (d[n, c[n]:] == SENTINEL).all() and (s[n, c[n]:].view(np.int32) == SENTINEL).all(), n
    for buf, t in bufs:
        pad = (buf.numel() - t.numel()) // 2
        assert (buf[:pad] == SENTINEL).all() and (buf[pad + t.numel():] == SENTINEL).all()
    lists = [[(*(int(v) for v in d[n, k]), float(s[n, k])) for k in range(c[n])] for n in range(N)]
    return lists, d, s, c


def _want_lists(prob, boxes, keep_idx, conf_count, im_scale):
    from frcnn_b200 import preprocess
    return [preprocess.result_detections(dict(prob=prob[n], boxes=boxes[n], keep_idx=keep_idx[n], conf_count=conf_count[n]),
                                         float(im_scale[n])) for n in range(prob.shape[0])]


def _block(N, R, NC, seed, lo=-50.0, hi=1100.0):
    """Synthetic prob / boxes and per-class keep lists: permutations of the rows, the listed counts random in [0, R]."""
    rng = np.random.default_rng(seed)
    prob = rng.random((N, R, NC)).astype(np.float32)
    boxes = (rng.random((N, R, 4 * NC)) * (hi - lo) + lo).astype(np.float32)
    keep_idx = np.stack([np.stack([rng.permutation(R) for _ in range(NC - 1)]) for _ in range(N)]).astype(np.int32)
    conf_count = rng.integers(0, R + 1, (N, NC - 1)).astype(np.int32)
    return prob, boxes, keep_idx, conf_count


def test_lists_equal_result_detections():
    """Five images of the graph's shape (R = 300, 21 classes): empty classes, an image with no detections, an image whose
    list is full (cap rows), negative and large coordinates, several im_scale values, inputs at padded image strides."""
    N, R, NC = 5, 300, 21
    prob, boxes, keep_idx, conf_count = _block(N, R, NC, seed=1, lo=-2000.0, hi=1100.0)
    boxes[3] *= np.float32(1e6)                           # up to +-2e9 / 1.2, still inside the int32 range
    conf_count[0, ::3] = 0
    conf_count[1] = 0                                     # no detections at all
    conf_count[2] = R                                     # the list is full: (NC-1) * R rows
    im_scale = [1.6, 1.8018018018018018, 0.78125, 1.2, 4.739336492890995]
    got, _, _, count = _run_lists(prob, boxes, keep_idx, conf_count, im_scale, stride_pad=40)
    assert count.tolist() == conf_count.sum(axis=1).tolist() and count[1] == 0 and count[2] == (NC - 1) * R
    assert got == _want_lists(prob, boxes, keep_idx, conf_count, im_scale)


def test_lists_divide_in_float32_not_float64():
    """im_scale = 1.2 and 600 / 449: coordinates whose float32 quotient truncates to another int than the float64 quotient
    (18 / 1.2: 14 against 15; 5943.875 / 1.3363...: 4448 against 4447)."""
    N, R, NC = 2, 8, 3
    prob, boxes, keep_idx, conf_count = _block(N, R, NC, seed=2)
    boxes[0, :, 4:8] = np.array([18.0, 30.0, 36.0, 54.0], np.float32)
    boxes[1, :, 4:8] = np.array([5943.875, 6543.875, 7143.875, 1.0], np.float32)
    conf_count[:] = R
    im_scale = [1.2, 600 / 449]
    got = _run_lists(prob, boxes, keep_idx, conf_count, im_scale)[0]
    assert got == _want_lists(prob, boxes, keep_idx, conf_count, im_scale)
    f64 = [int(float(v) / s) for v, s in ((18.0, 1.2), (5943.875, 600 / 449))]
    assert (got[0][0][1], got[1][0][1]) == (14, 4448) and f64 == [15, 4447]


def test_lists_many_classes_span_several_scan_chunks():
    """300 classes (the scan runs in chunks of 256 classes) with one to three rows each, some classes empty."""
    N, R, NC = 3, 3, 300
    prob, boxes, keep_idx, conf_count = _block(N, R, NC, seed=3)
    conf_count[1, 250:262] = 0
    conf_count[2] = 1
    im_scale = [1.6, 2.0, 0.5]
    got, _, _, count = _run_lists(prob, boxes, keep_idx, conf_count, im_scale)
    assert count.tolist() == conf_count.sum(axis=1).tolist()
    assert got == _want_lists(prob, boxes, keep_idx, conf_count, im_scale)


def _rzi(q):
    """cvt.rzi.s32.f32: NaN -> 0, truncation toward zero, saturation to the int32 range."""
    if np.isnan(q):
        return 0
    if np.isinf(q):
        return 2 ** 31 - 1 if q > 0 else -2 ** 31
    return int(min(max(int(q), -2 ** 31), 2 ** 31 - 1))


def test_lists_non_finite_and_out_of_range_convert_as_cvt_rzi():
    """The one deviation from Python's int(): NaN -> 0, +-inf and quotients past the int32 range saturate.  Scores (NaN
    included) are copied bit for bit; conf_count is clamped to [0, R]; a keep index outside [0, R) gives (c, 0, 0, 0, 0), 0."""
    f32 = np.float32
    N, R, NC = 1, 6, 2
    vals = np.array([np.nan, -np.nan, np.inf, -np.inf, 3.0e38, -3.0e38, 2147483648.0, -2147483648.0, 2147483520.0, -2147483904.0,
                     -0.0, -0.9999999, 0.9999999, 1.0e10, -1.0e10, 5.5, -5.5, 7.0, -7.0, 1.0, 2.0, 3.0, 4.0, 5.0], f32)
    boxes = np.zeros((N, R, 4 * NC), f32)
    boxes[0, :, 4:8] = vals.reshape(R, 4)
    prob = np.zeros((N, R, NC), f32)
    prob[0, :, 1] = np.array([np.nan, 0.5, np.inf, -0.0, 1e-45, 0.9], f32)
    keep_idx = np.array([[[5, 4, 3, 2, 1, 0]]], np.int32)
    for scale in (1.0, 0.5, 1.2):
        got, d, s, c = _run_lists(prob, boxes, keep_idx, np.array([[R]], np.int32), [scale])
        assert c[0] == R
        for k, r in enumerate(keep_idx[0, 0]):
            with np.errstate(over="ignore", invalid="ignore"):
                q = boxes[0, r, 4:8] / scale              # NumPy's float32 quotient
            assert q.dtype == f32
            assert d[0, k].tolist() == [1] + [_rzi(v) for v in q], (scale, r)
            assert s[0, k].view(np.int32) == prob[0, r, 1].view(np.int32), (scale, r)
    # finite, in-range rows still equal result_detections
    fin = np.array([[[5, 4, 0, 0, 0, 0]]], np.int32)
    assert _run_lists(prob, boxes, fin, np.array([[2]], np.int32), [1.2])[0] == _want_lists(prob, boxes, fin, [[2]], [1.2])
    # conf_count clamped to [0, R]; keep indices outside [0, R) read nothing
    got, d, s, c = _run_lists(prob, boxes, np.array([[[-1, R, 1 << 30, 2, 0, 0]]], np.int32), np.array([[R + 50]], np.int32), [1.0])
    assert c[0] == R and d[0, :3].tolist() == [[1, 0, 0, 0, 0]] * 3 and s[0, :3].tolist() == [0.0] * 3
    got, d, s, c = _run_lists(prob, boxes, keep_idx, np.array([[-4]], np.int32), [1.0])
    assert c[0] == 0 and got == [[]]
