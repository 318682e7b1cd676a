"""CPU tests of the raw-photo training input: the bicubic restatement (voc_ref.cubic_resize) against cv2.resize, the box
scaling rule against NumPy's `bbox *= im_scale`, the training block's ground-truth section and every error a bad batch
raises before anything is queued, and the declared signatures of frcnn_preprocess_voc_canvas_im2col and
frcnn_voc_scale_gt_batch."""
import ctypes

import numpy as np
import pytest

import voc_ref
from test_train_targets_abi_cpu import _params

# the stand-in dataset's sizes (datasets/pascal_voc_dataset.py) and the degenerate shapes
VOC_SIZES = [(375, 500), (333, 500), (500, 375), (500, 500), (281, 500), (500, 334), (442, 500), (375, 1000)]
EDGE_SIZES = [(1, 1), (1, 7), (7, 1), (2, 2), (3, 3), (4, 1000)]


def _photo(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _cv2_resize(img, s, ipp):
    cv2 = pytest.importorskip("cv2")
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(ipp)
    try:
        out = cv2.resize(img, None, None, fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
    finally:
        cv2.ipp.setUseIPP(was)
    return out.reshape(out.shape[0], out.shape[1], -1)


@pytest.mark.parametrize("shape", VOC_SIZES + EDGE_SIZES)
def test_cubic_restatement_equals_opencv(shape):
    """Bit for bit against OpenCV's own float INTER_CUBIC (IPP off); within IPP_BOUND of cv2's default IPP path."""
    h0, w0 = shape
    img = voc_ref.mean_subtract(_photo(h0, w0, h0 * 7 + w0))
    s, H, W = voc_ref.plan_size(h0, w0)
    want = voc_ref.cubic_resize(img, H, W, 1.0 / s)
    generic = _cv2_resize(img, s, False)
    assert generic.shape == want.shape
    assert np.array_equal(generic.view(np.uint32), want.view(np.uint32))
    ipp = _cv2_resize(img, s, True)
    assert float(np.abs(ipp - want).max()) <= voc_ref.IPP_BOUND


def test_cubic_restatement_keeps_overshoot():
    """No clamping: a step edge overshoots the source's range, as the float path does."""
    photo = np.zeros((20, 20, 3), dtype=np.uint8)
    photo[:, 10:] = 255
    img = voc_ref.mean_subtract(photo)
    out = voc_ref.cubic_resize(img, 600, 600, 20 / 600)
    assert out.max() > img.max() and out.min() < img.min()


def test_cubic_taps_stay_inside_for_any_scale():
    for inv in (0.0, -1.0, -1e30, 1e30, np.inf, -np.inf, np.nan):
        idx, w, _ = voc_ref.cubic_taps(50, 7, inv)
        assert idx.min() >= 0 and idx.max() <= 6
        assert all(np.isfinite(c).all() for c in w)


def test_box_scaling_rule_matches_numpy():
    """f32(box) * f32(im_scale) is what `bbox *= im_scale` leaves in a float32 array, on adversarial values."""
    from frcnn_b200 import preprocess
    rng = np.random.default_rng(5)
    vals = np.concatenate([rng.uniform(0, 1000, 4000), [0.0, -0.0, 1e-45, 3.4e38, np.inf, -np.inf, np.nan, 499.99997, 0.5]])
    bbox = vals.astype(np.float32).reshape(-1, 1)[: len(vals) // 4 * 4].reshape(-1, 4)
    for h0, w0 in VOC_SIZES + [(333, 499), (1, 3), (7, 1000), (600, 601)]:
        s = voc_ref.plan_size(h0, w0)[0]
        ref = bbox.copy()
        with np.errstate(over="ignore", invalid="ignore"):
            ref *= s
            got = preprocess.voc_scale_boxes(bbox, s)
        assert ref.dtype == np.float32 and got.dtype == np.float32
        assert np.array_equal(ref.view(np.uint32), got.view(np.uint32))


def test_gt_section_layout():
    from frcnn_b200 import preprocess
    layout, nbytes = preprocess.voc_gt_layout(3, 4)
    assert nbytes % 256 == 0
    spans = sorted((off, off + int(np.prod(shape)) * 4) for off, _, shape in layout.values())
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])) and spans[-1][1] <= nbytes
    boxes = [np.array([[1, 2, 3, 4]], np.float32), np.array([[5, 6, 7, 8], [9, 10, 11, 12]], np.float32)]
    sec = preprocess.voc_gt_section(boxes, [np.array([7]), np.array([1, 20])], [1.6, 1.8018018018018018], 3, 4)
    v = {k: sec[o:o + int(np.prod(sh)) * 4].view(dt).reshape(sh) for k, (o, dt, sh) in layout.items()}
    assert v["count"].tolist() == [1, 2, 0]
    assert v["scale"].tolist() == [np.float32(1.6), np.float32(1.8018018018018018), 0.0]
    assert v["raw_gt"][1, 1].tolist() == [9, 10, 11, 12, 20]
    assert not v["raw_gt"][2].any() and not v["raw_gt"][0, 1:].any()


def _input(N=2, Hc=600, Wc=1000, max_gt=3, arena_bytes=None):
    from frcnn_b200.engine import RawPhotoInput
    return RawPhotoInput(N, Hc, Wc, "cpu", arena_bytes=arena_bytes, max_gt=max_gt)


def test_training_block_layout():
    from frcnn_b200 import preprocess
    inp = _input(N=4, max_gt=256)
    hdr = preprocess.raw_header_layout(4)[1]
    assert inp.header_bytes == hdr + preprocess.voc_gt_layout(4, 256)[1]
    assert inp.pixel_means == preprocess.VOC_MEANS
    assert inp.arena.numel() == 4 * 3 * 600 * 1000
    scale, count, raw_gt = inp.gt_fields
    assert scale.data_ptr() == inp.block.data_ptr() + hdr
    assert tuple(raw_gt.shape) == (4, 256, 5) and raw_gt.data_ptr() + raw_gt.numel() * 4 <= inp.arena.data_ptr()


@pytest.mark.parametrize("case,words", [
    ("too_many", ["3 images for 2 slots"]),
    ("too_big", ["does not fit"]),
    ("no_boxes", ["G, 4", "1 <= G <= 3"]),
    ("too_many_boxes", ["1 <= G <= 3"]),
    ("label_count", ["labels of shape"]),
    ("list_count", ["2 photos, 1 box lists"]),
    ("arena", ["the arena holds"]),
    ("no_gt", ["boxes and labels"]),
])
def test_training_batch_errors(case, words):
    """Every bad batch raises FrcnnError in RawPhotoInput.upload before it touches a stream (the input lives on the CPU)."""
    from frcnn_b200._lib import FrcnnError
    p = [_photo(375, 500, 1), _photo(333, 500, 2)]
    b = [np.array([[1, 2, 30, 40]], np.float32)] * 2
    lab = [np.array([3])] * 2
    kw, inp = {}, _input()
    if case == "too_many":
        p, b, lab = p + p[:1], b + b[:1], lab + lab[:1]
    elif case == "too_big":
        inp = _input(Hc=599)
    elif case == "no_boxes":
        b, lab = [np.zeros((0, 4), np.float32), b[1]], [np.zeros((0,), np.int32), lab[1]]
    elif case == "too_many_boxes":
        b, lab = [np.ones((4, 4), np.float32), b[1]], [np.ones((4,), np.int32), lab[1]]
    elif case == "label_count":
        lab = [np.array([1, 2]), lab[1]]
    elif case == "list_count":
        b = b[:1]
    elif case == "arena":
        inp = _input(arena_bytes=375 * 500 * 3 + 100)
    elif case == "no_gt":
        b = None
    with pytest.raises(FrcnnError) as e:
        inp.upload(p, boxes=b, labels=lab, **kw)
    assert all(w in str(e.value) for w in words), str(e.value)


def test_declared_signatures():
    from frcnn_b200 import _lib
    lib = _lib.load()
    ctype = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "double": ctypes.c_double}
    for name in ("frcnn_preprocess_voc_canvas_im2col", "frcnn_voc_scale_gt_batch"):
        params = _params(name)
        res, args = _lib.SIGNATURES[name]
        assert res is ctypes.c_int and getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0].replace("const ", "")
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
    assert _params("frcnn_preprocess_voc_canvas_im2col")[1:] == _params("frcnn_preprocess_bgr8_canvas_im2col")[1:]


def test_scale_gt_rejects_bad_arguments():
    from frcnn_b200 import _lib
    lib = _lib.load()
    P = ctypes.c_void_p(16)
    for args in ((None, P, P, 1, 1, P, P), (P, P, P, 0, 1, P, P), (P, P, P, 65536, 1, P, P), (P, P, P, 1, 0, P, P),
                 (P, P, P, 1, (1 << 20) + 1, P, P), (P, P, P, 1, 1, None, P)):
        assert lib.frcnn_voc_scale_gt_batch(*args, None) == -1
        assert "frcnn_voc_scale_gt_batch" in _lib.last_error()


def test_voc_raw_example_matches_get_example():
    """get_raw_example is get_example's input: the same photo, boxes and labels before the transform."""
    from datasets.pascal_voc_dataset import VOC
    ds = VOC("train")
    for i in range(4):
        photo, bbox, label = ds.get_raw_example(i)
        img, im_info, gt = ds.get_example(i)
        assert photo.dtype == np.uint8 and photo.shape[2] == 3 and bbox.dtype == np.float32 and label.dtype == np.int32
        s, H, W = voc_ref.plan_size(*photo.shape[:2])
        assert tuple(im_info) == (H, W) == img.shape[1:]
        assert np.array_equal(gt[:, 4], label) and np.array_equal(gt[:, :4], voc_ref.voc_transform(photo, bbox, label)[2][:, :4])
