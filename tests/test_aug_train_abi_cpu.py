"""CPU tests of training-time augmentation on raw photos (flip and multi-scale): the declared signatures and argument errors
of frcnn_voc_augment_batch, frcnn_preprocess_voc_canvas_im2col_flip and frcnn_voc_flip_scale_gt_batch, the augmentation
section's layout and candidate table, every error a trainer or a batch raises before anything is queued, and the launch
sequence of an augmenting step (recorded, as tests/test_trainer_launches_cpu.py records it)."""
import ctypes

import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import voc_aug_ref
import voc_ref
from test_train_targets_abi_cpu import _params
from test_trainer_launches_cpu import ANCHORS, H, POST_N, W, _vgg_params, rec  # noqa: F401  (rec: the recorder fixture)

ENTRIES = ("frcnn_voc_augment_batch", "frcnn_preprocess_voc_canvas_im2col_flip", "frcnn_voc_flip_scale_gt_batch")
VOC_SIZES = [(375, 500), (333, 500), (500, 375), (500, 500), (281, 500), (500, 334), (442, 500), (375, 1000)]
SCALES = (480, 576, 600, 688, 864, 1000)


def test_declared_signatures():
    from frcnn_b200 import _lib
    lib = _lib.load()
    ctype = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "double": ctypes.c_double}
    for name in ENTRIES:
        params = _params(name)
        res, args = _lib.SIGNATURES[name]
        assert res is ctypes.c_int and getattr(lib, name).argtypes == args and len(args) == len(params), name
        for p, a in zip(params, args):
            typ = p.rsplit(" ", 1)[0].replace("const ", "")
            assert a is (ctypes.c_void_p if "*" in typ else ctype[typ]), (name, p)
    plain, flip = _params("frcnn_preprocess_voc_canvas_im2col"), _params("frcnn_preprocess_voc_canvas_im2col_flip")
    assert flip[:6] + flip[7:] == plain and flip[6] == "const int* flip"
    assert _params("frcnn_voc_flip_scale_gt_batch") == (_params("frcnn_voc_scale_gt_batch")[:3] + ["const int* src_hw", "const int* flip"]
                                                        + _params("frcnn_voc_scale_gt_batch")[3:])


def _rejects(call, name, *args):
    from frcnn_b200 import _lib
    assert call(*args) == -1, args
    assert name in _lib.last_error(), _lib.last_error()


def test_augment_rejects_bad_arguments():
    from frcnn_b200 import _lib
    call = _lib.load().frcnn_voc_augment_batch
    P = ctypes.c_void_p(16)
    good = [P, 4, 3, P, P, P, P, 1, P, P, P, P, P, P, None]
    fn = "frcnn_voc_augment_batch"
    for i in (3, 4, 5, 6, 8, 9, 10, 11, 12, 13):                        # every output and candidate array
        args = list(good)
        args[i] = None
        _rejects(call, fn, *args)
    _rejects(call, fn, None, *good[1:])                                   # a draw without seeds
    for k, v in ((1, 0), (1, 65536), (2, 0), (2, 9), (7, -1), (7, 3)):   # N, S, draw
        args = list(good)
        args[k] = v
        _rejects(call, fn, *args)


def test_flip_pack_and_gt_reject_bad_arguments():
    from frcnn_b200 import _lib
    lib = _lib.load()
    P = ctypes.c_void_p(16)
    fn = "frcnn_preprocess_voc_canvas_im2col_flip"
    pack = [P, 1 << 20, P, P, P, P, P, 2, 600, 1000, 1.0, 2.0, 3.0, 3, 1, 1, 32, P, P, None]
    for i, v in ((6, None), (0, None), (7, 0), (7, 65536), (13, 0), (16, 20), (8, 0)):
        args = list(pack)
        args[i] = v
        _rejects(lib.frcnn_preprocess_voc_canvas_im2col_flip, fn, *args)
    fn = "frcnn_voc_flip_scale_gt_batch"
    gt = [P, P, P, P, P, 2, 8, P, P, None]
    for i, v in ((3, None), (4, None), (0, None), (5, 0), (5, 65536), (6, 0), (6, (1 << 20) + 1), (8, None)):
        args = list(gt)
        args[i] = v
        _rejects(lib.frcnn_voc_flip_scale_gt_batch, fn, *args)


@pytest.mark.parametrize("N,S", [(1, 1), (3, 5), (4, 8), (65535, 8)])
def test_aug_layout(N, S):
    from frcnn_b200 import preprocess
    layout, nbytes = preprocess.voc_aug_layout(N, S)
    assert nbytes % 256 == 0
    want = {"cand_inv": (np.float64, (N, S)), "cand_hw": (np.int32, (N, S, 2)), "cand_scale": (np.float32, (N, S)),
            "choice": (np.int32, (N, 2)), "flip": (np.int32, (N,))}
    assert {k: (dt, sh) for k, (_, dt, sh) in layout.items()} == want
    spans = sorted((off, off + int(np.prod(sh)) * np.dtype(dt).itemsize) for off, dt, sh in layout.values())
    assert spans[0][0] == 0 and all(a[1] <= b[0] for a, b in zip(spans, spans[1:])) and spans[-1][1] <= nbytes
    assert all(off % 16 == 0 for off, _, _ in layout.values())


def test_candidate_table_is_plan_size():
    from frcnn_b200 import preprocess
    shapes = VOC_SIZES[:6]
    sec, cands = preprocess.voc_aug_section(shapes, 7, 1000, 1000, SCALES)
    v = preprocess.voc_aug_views(sec, 7, len(SCALES))
    for n, (h0, w0) in enumerate(shapes):
        for k, s in enumerate(SCALES):
            im_scale, Hs, Ws = voc_ref.plan_size(h0, w0, s)
            assert cands[n][k] == im_scale and tuple(v["cand_hw"][n, k]) == (Hs, Ws)
            assert v["cand_inv"][n, k] == 1.0 / im_scale and v["cand_scale"][n, k] == np.float32(im_scale)
    assert not v["cand_hw"][6:].any() and not v["choice"].any() and not v["flip"].any()
    sec2, _ = preprocess.voc_aug_section(VOC_SIZES[6:], 2, 1000, 1000, SCALES)
    v2 = preprocess.voc_aug_views(sec2, 2, len(SCALES))
    assert [tuple(v2["cand_hw"][n, 2]) for n in range(2)] == [voc_ref.plan_size(*s)[1:] for s in VOC_SIZES[6:]]


@pytest.mark.parametrize("shape", [(375, 500), (333, 500), (7, 5)])
def test_restatement_defaults_are_the_plain_transform(shape):
    """voc_aug_ref.voc_transform(flip=False, scale=600) is voc_ref.voc_transform bit for bit; with flip it is the plain
    transform of the mirrored photo and boxes."""
    h0, w0 = shape
    photo = _photo(h0, w0, h0 + w0)
    boxes = np.array([[0, 1, w0 - 1, h0 - 1], [1.5, 0, 3.25, 2]], np.float32)
    labels = np.array([4, 9])
    plain, aug = voc_ref.voc_transform(photo, boxes, labels), voc_aug_ref.voc_transform(photo, boxes, labels)
    assert plain[1] == aug[1]
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in ((plain[0], aug[0]), (plain[2], aug[2])))
    flipped = voc_aug_ref.voc_transform(photo, boxes, labels, flip=True, scale=480)
    mirror = voc_aug_ref.voc_transform(np.ascontiguousarray(photo[:, ::-1]), voc_aug_ref.flip_boxes(boxes, w0), labels,
                                       scale=480)
    assert np.array_equal(flipped[0].view(np.uint32), mirror[0].view(np.uint32)) and np.array_equal(flipped[2], mirror[2])
    fb = voc_aug_ref.flip_boxes(boxes, w0)
    assert fb[0].tolist() == [0, 1, w0 - 1, h0 - 1]                                  # a full-width box maps onto itself
    assert np.array_equal(voc_aug_ref.flip_boxes(fb, w0), boxes)                     # exact on these values


def test_candidate_that_does_not_fit_is_named():
    from frcnn_b200 import preprocess
    from frcnn_b200._lib import FrcnnError
    with pytest.raises(FrcnnError, match=r"image 1 \(375 x 500\) at scale 864 resizes to 750 x 1000"):
        preprocess.voc_aug_section([(333, 500), (375, 500)], 2, 700, 1000, (600, 864))


def _photo(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _canvas(kind="rpn", **kw):
    from frcnn_b200.train_engine import CanvasRcnnTrainer, CanvasRpnTrainer
    if kind == "rpn":
        return CanvasRpnTrainer(_vgg_params(), 2, H, W, ANCHORS, device="cpu", **kw)
    return CanvasRcnnTrainer(_vgg_params(), 2, H, W, ANCHORS, post_n=POST_N, device="cpu", **kw)


@pytest.mark.parametrize("kw,words", [
    (dict(augment="device"), "needs raw_input=True"),
    (dict(augment="list", raw_input=False), "needs raw_input=True"),
    (dict(augment="both", raw_input=True), "augment must be"),
    (dict(augment="device", raw_input=True, scales=()), "scales must be"),
    (dict(augment="device", raw_input=True, scales=tuple(range(100, 1000, 100))), "scales must be"),
    (dict(augment="device", raw_input=True, scales=(0, 600)), "scales must be"),
    (dict(raw_input=True, scales=(480, 600)), "need augment"),
    (dict(raw_input=True, flip=False), "need augment"),
])
@pytest.mark.parametrize("kind", ["rpn", "rcnn"])
def test_constructor_rejects(monkeypatch, kind, kw, words):
    from frcnn_b200 import train_engine
    from frcnn_b200._lib import FrcnnError

    def alloc(*a, **k):
        raise AssertionError("the trainer allocated its buffers before it rejected the options")
    monkeypatch.setattr(train_engine._ConvTrainer, "_init_params", alloc)
    with pytest.raises(FrcnnError, match=words):
        _canvas(kind, **kw)


@pytest.mark.parametrize("case,words", [
    ("not_list", "need augment='list'"),
    ("plain", "need augment='list'"),
    ("flip_len", "flips needs one value"),
    ("index_len", "scale_index needs one value"),
    ("index_range", "scale_index needs one value in [0, 2)"),
    ("negative", "scale_index needs one value"),
    ("flip_off", "flip=False"),
    ("no_fit", "at scale 96"),
])
def test_put_raw_rejects(rec, case, words):  # noqa: F811
    """Every bad augmented batch raises FrcnnError before anything is queued (the trainer lives on the CPU)."""
    from frcnn_b200._lib import FrcnnError
    photos = [_photo(12, 16, 1), _photo(16, 12, 2)]
    boxes = [np.array([[1, 2, 8, 9]], np.float32)] * 2
    labels = [np.array([3])] * 2
    kw, tr = dict(flips=[True, False], scale_index=[1, 0]), None
    if case == "not_list":
        tr = _canvas(raw_input=True, augment="device", scales=(32, 48))
    elif case == "plain":
        tr, kw = _canvas(raw_input=True), dict(scale_index=[0, 0])
    else:
        tr = _canvas("rcnn" if case in ("index_range", "no_fit") else "rpn", raw_input=True, augment="list",
                     scales=(32, 96) if case == "no_fit" else (32, 48), flip=case != "flip_off")
        if case == "flip_len":
            kw["flips"] = [True]
        elif case == "index_len":
            kw["scale_index"] = [0, 1, 1]
        elif case == "index_range":
            kw["scale_index"] = [0, 2]
        elif case == "negative":
            kw["scale_index"] = [-1, 0]
    with pytest.raises(FrcnnError) as e:
        tr.put_raw(photos, boxes, labels, **kw)
    assert words in str(e.value), str(e.value)


def _trunk_kinds():
    return ("vgg16_rpn", "vgg16_rcnn", "resnet50_rpn", "resnet50_rcnn")


def _make(kind, **kw):
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer
    if kind.startswith("vgg16"):
        return _canvas(kind.split("_")[1], **kw)
    r50 = orc.make_resnet_params(50, seed=3)
    if kind == "resnet50_rpn":
        return CanvasResNetRpnTrainer(r50, 2, H, W, ANCHORS, n_layers=50, device="cpu", **kw)
    return CanvasResNetRcnnTrainer(r50, 2, H, W, ANCHORS, n_layers=50, post_n=POST_N, device="cpu", **kw)


def _forward_trace(rec, tr):
    tr.forward()
    tr.backward()                 # cached buffers first, as test_trainer_launches_cpu._warm
    rec.reset()
    tr.forward()
    return list(rec.calls)


@pytest.mark.parametrize("kind", _trunk_kinds())
@pytest.mark.parametrize("mode", ["device", "list"])
def test_augmenting_step_launches(rec, kind, mode):  # noqa: F811
    """The augmenting step starts with frcnn_voc_augment_batch (before the ResNet level extents) and packs through the
    _flip entries; the rest of its forward is the plain raw step's, launch for launch."""
    plain = _forward_trace(rec, _make(kind, raw_input=True))
    aug = _forward_trace(rec, _make(kind, raw_input=True, augment=mode, scales=(32, 48)))
    names = [c[0] for c in aug]
    assert names[0] == "frcnn_voc_augment_batch"
    assert aug[0][8] == (0 if mode == "list" else 1) and aug[0][3] == 2          # draw, S
    pack = 2 if kind.startswith("resnet") else 1
    if pack == 2:
        assert names[1] == "frcnn_resnet_level_extents"
    assert names[pack] == "frcnn_preprocess_voc_canvas_im2col_flip" and names[pack + 1] == "frcnn_voc_flip_scale_gt_batch"
    assert "frcnn_preprocess_voc_canvas_im2col" not in names and "frcnn_voc_scale_gt_batch" not in names
    twin = {"frcnn_preprocess_voc_canvas_im2col_flip": "frcnn_preprocess_voc_canvas_im2col",
            "frcnn_voc_flip_scale_gt_batch": "frcnn_voc_scale_gt_batch"}
    assert [twin.get(n, n) for n in names[1:]] == [c[0] for c in plain]
    # scalar arguments beyond the inserted pointers are the plain step's
    assert [a for a in aug[pack][8:] if not isinstance(a, str)] == [a for a in plain[pack - 1][7:] if not isinstance(a, str)]
    # without augment the raw step packs as before
    assert plain[pack - 1][0] == "frcnn_preprocess_voc_canvas_im2col" and plain[pack][0] == "frcnn_voc_scale_gt_batch"


@pytest.mark.parametrize("kind", ["vgg16_rpn", "vgg16_rcnn"])
def test_flip_false_draws_scale_only(rec, kind):  # noqa: F811
    aug = _forward_trace(rec, _make(kind, raw_input=True, augment="device", scales=(32, 48, 64), flip=False))
    assert aug[0][0] == "frcnn_voc_augment_batch" and aug[0][8] == 2 and aug[0][3] == 3


@pytest.mark.parametrize("mode,advance", [("device", True), ("list", False)])
def test_seed_advance(rec, mode, advance):  # noqa: F811
    """A device draw advances the seeds by N once per step, also when nothing else in the step draws; a list step does not."""
    for kind, kw in (("vgg16_rpn", dict(subsample="none")), ("vgg16_rcnn", dict(sample="list", dropout="explicit"))):
        tr = _make(kind, raw_input=True, augment=mode, scales=(32,), **kw)
        before = tr.seeds.clone()
        tr.forward()
        assert torch.equal(tr.seeds, before + (tr.N if advance else 0)), kind
    tr = _make("vgg16_rpn", raw_input=True, augment=mode, scales=(32,))          # device subsampling: still one advance
    before = tr.seeds.clone()
    tr.forward()
    assert torch.equal(tr.seeds, before + tr.N)
