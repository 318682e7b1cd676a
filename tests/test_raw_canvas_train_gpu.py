"""GPU tests of training on raw photos: frcnn_preprocess_voc_canvas_im2col (the VOC dataset's mean subtraction + bicubic
resize + the first layer's im2col in one launch), frcnn_voc_scale_gt_batch, and CanvasRpnTrainer / CanvasRcnnTrainer with
raw_input=True.  The bar is bit-identity everywhere: the planes against voc_ref's transform put through ImageInput.put +
pack_image_im2col_batch, and each raw step against step() on voc_ref's preprocessed images and scaled boxes."""
import numpy as np
import pytest
import torch

import voc_ref
from test_canvas_rcnn_train_gpu import _rcnn_params
from test_canvas_train_gpu import ANCHORS, _flat_equal
from test_train_gpu import _train_case

pytestmark = pytest.mark.gpu
HC, WC = 1000, 1000            # holds both orientations: 500x375 resizes to 800x600, 375x500 to 600x800
VOC = [(375, 500), (333, 500), (500, 375), (375, 1000), (500, 334), (442, 500), (281, 500)]


def _photos(sizes, seed):
    rng = np.random.default_rng(seed)
    photos, boxes, labels = [], [], []
    for h, w in sizes:
        photos.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        G = int(rng.integers(1, 5))
        x1, y1 = rng.uniform(0, max(w - 60, 1), G), rng.uniform(0, max(h - 60, 1), G)
        b = np.stack([x1, y1, np.minimum(x1 + rng.uniform(30, w / 2 + 30, G), w - 1),
                      np.minimum(y1 + rng.uniform(30, h / 2 + 30, G), h - 1)], 1)
        boxes.append(b.astype(np.float32))
        labels.append(rng.integers(1, 21, G).astype(np.int32))
    return photos, boxes, labels


def _float_batch(photos, boxes, labels):
    """voc_ref's transform: the float images and (G, 5) ground truth that step() takes."""
    xs, gts = [], []
    for p, b, l in zip(photos, boxes, labels):
        img, _, gt = voc_ref.voc_transform(p, b, l)
        xs.append(torch.from_numpy(img).cuda())
        gts.append(torch.from_numpy(gt).cuda())
    return xs, gts


def _bits(act):
    return [t.view(torch.int16) for t in (act.hi, act.lo) if t is not None]


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("N", [1, 2, 4])
def test_fused_launch_equals_oracle(N, precision):
    from frcnn_b200 import ops
    from frcnn_b200.engine import ImageInput, RawPhotoInput
    for mix in range(2):
        sizes = [VOC[(mix * 3 + k) % len(VOC)] for k in range(N - (1 if N > 1 and mix else 0))]   # mix 1: an empty slot
        photos, boxes, labels = _photos(sizes, 10 * N + mix)
        raw = RawPhotoInput(N, HC, WC, "cuda", max_gt=8)
        raw.upload(photos, boxes=boxes, labels=labels)
        got = ops.Act(torch.full((N, HC, WC, 32), 7.0, dtype=torch.bfloat16, device="cuda"),
                      torch.full((N, HC, WC, 32), 7.0, dtype=torch.bfloat16, device="cuda") if precision == "bf16x3" else None)
        ops.preprocess_voc_im2col_canvas(*raw.descriptors, HC, WC, raw.pixel_means, 3, 1, 1, 32, out=got)
        xs, gts = _float_batch(photos, boxes, labels)
        ref_in = ImageInput(N, HC, WC, "cuda", canvas=True)
        ref_in.put(xs)
        want = ops.pack_image_im2col_batch(ref_in.x_in, 3, 1, 1, 32, precision=precision, extents=ref_in.extents)
        gt = torch.full((N, 8, 5), 9.0, device="cuda")
        cnt = torch.full((N,), 9, dtype=torch.int32, device="cuda")
        raw.scale_gt(gt, cnt)
        torch.cuda.synchronize()
        for g, w in zip(_bits(got), _bits(want)):
            assert torch.equal(g, w), (N, mix)
        assert torch.equal(raw.extents, ref_in.extents) and torch.equal(raw.im_info, ref_in.extents)
        for n in range(N):
            G = gts[n].shape[0] if n < len(gts) else 0
            assert int(cnt[n]) == G
            if G:
                assert _flat_equal(gt[n, :G], gts[n]), n
            assert not gt[n, G:].any()


def test_fused_launch_bad_descriptors():
    """inv_scale 0, negative, inf, NaN: nothing is read outside the arena or written outside the planes, and the values are
    finite and the same on every launch."""
    from frcnn_b200 import ops
    from frcnn_b200.engine import RawPhotoInput
    photos, boxes, labels = _photos([(375, 500), (333, 500), (1, 1), (500, 375)], 3)
    raw = RawPhotoInput(4, HC, WC, "cuda", max_gt=8)
    raw.upload(photos, boxes=boxes, labels=labels)
    inv = raw.descriptors[3]
    for bad in ([0.0, -1.0, float("inf"), float("nan")], [float("-inf"), 1e300, -1e-300, float("nan")]):
        inv.copy_(torch.tensor(bad, dtype=torch.float64))
        outs = []
        for _ in range(2):
            buf = torch.full((5, HC, WC, 32), 3.0, dtype=torch.bfloat16, device="cuda")
            act = ops.Act(buf[:4], torch.empty((4, HC, WC, 32), dtype=torch.bfloat16, device="cuda"))
            raw.pack_im2col(act, 3, 1, 1, 32)
            torch.cuda.synchronize()
            assert bool((buf[4] == 3.0).all())                  # nothing past the planes
            assert bool(torch.isfinite(act.hi.float()).all()) and bool(torch.isfinite(act.lo.float()).all())
            outs.append([t.clone() for t in _bits(act)])
        assert all(torch.equal(a, b) for a, b in zip(*outs))


def _mixes(N):
    """Three replays with a different size mix each; from N = 2 on, the second leaves a slot empty."""
    return [[VOC[(3 * t + k) % len(VOC)] for k in range(N - (1 if N > 1 and t == 1 else 0))] for t in range(3)]


@pytest.mark.parametrize("N", [1, 2, 4])
def test_rpn_raw_step_equals_float_step(N):
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.train_engine import CanvasRpnTrainer
    params = _train_case(HC, WC, 3)[0]
    raw = CanvasRpnTrainer(params, N, HC, WC, ANCHORS, seed=5, raw_input=True)
    flt = CanvasRpnTrainer(params, N, HC, WC, ANCHORS, seed=5)
    captured = None
    for t, sizes in enumerate(_mixes(N)):
        photos, boxes, labels = _photos(sizes, 100 * N + t)
        xs, gts = _float_batch(photos, boxes, labels)
        lr_ = raw.step_raw(photos, boxes, labels)
        lf = flt.step(xs, gts)
        torch.cuda.synchronize()
        captured = captured or raw.graph
        assert raw.graph is captured and raw.n_updates == t + 1
        assert _flat_equal(lr_, lf), t
        assert _flat_equal(raw.g_flat, flt.g_flat), t
        assert _flat_equal(raw.w_flat, flt.w_flat) and _flat_equal(raw.v_flat, flt.v_flat), t
    with pytest.raises(FrcnnError, match="raw_input=True"):
        raw.put(xs, gts)
    with pytest.raises(FrcnnError, match="raw_input=False"):
        flt.put_raw(photos, boxes, labels)
    with pytest.raises(FrcnnError, match="disable lists need"):
        raw.put_raw(photos, boxes, labels, disable_pos=[torch.zeros(1, dtype=torch.int32)] * len(photos))


@pytest.mark.parametrize("mode", ["device", "list"])
def test_rcnn_raw_step_equals_float_step(mode):
    from frcnn_b200.train_engine import CanvasRcnnTrainer
    N, post_n = 2, 300
    params = _rcnn_params(HC, WC, 7)
    kw = dict(post_n=post_n, seed=11, sample=mode, dropout="device" if mode == "device" else "explicit")
    raw = CanvasRcnnTrainer(params, N, HC, WC, ANCHORS, raw_input=True, **kw)
    flt = CanvasRcnnTrainer(params, N, HC, WC, ANCHORS, **kw)
    rng = np.random.default_rng(2)
    captured = None
    for t, sizes in enumerate(_mixes(N)):
        photos, boxes, labels = _photos(sizes, 300 + t)
        xs, gts = _float_batch(photos, boxes, labels)
        extra = {}
        if mode == "list":
            extra = dict(keep_inds=[torch.from_numpy(rng.choice(64, 24, replace=False).astype(np.int32)) for _ in sizes],
                         masks=[[torch.from_numpy(rng.integers(0, 2, (post_n, 4096), dtype=np.uint8)).cuda() for _ in range(2)]
                                for _ in sizes])
        lr_ = raw.step_raw(photos, boxes, labels, **extra)
        lf = flt.step(xs, gts, **extra)
        torch.cuda.synchronize()
        captured = captured or raw.graph
        assert raw.graph is captured and raw.n_updates == t + 1
        assert _flat_equal(lr_, lf), t
        assert _flat_equal(raw.g_flat, flt.g_flat), t
        assert _flat_equal(raw.w_flat, flt.w_flat) and _flat_equal(raw.v_flat, flt.v_flat), t
