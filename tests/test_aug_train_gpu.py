"""GPU tests of training-time augmentation on raw photos: frcnn_preprocess_voc_canvas_im2col_flip and
frcnn_voc_flip_scale_gt_batch against voc_aug_ref.voc_transform(flip=, scale=), frcnn_voc_augment_batch's draws against their
NumPy restatement, and the canvas trainers with augment="device" / "list" against their float-input twins fed the host
transform of the same draws.  The bar is bit-identity everywhere."""
import numpy as np
import pytest
import torch

import voc_aug_ref
import voc_ref
from test_canvas_rcnn_train_gpu import _rcnn_params
from test_canvas_train_gpu import ANCHORS, _flat_equal
from test_raw_canvas_train_gpu import HC, VOC, WC, _bits, _photos
from test_train_gpu import _train_case
from test_train_targets_edges_gpu import _mix64

pytestmark = pytest.mark.gpu
SCALES = (480, 600, 800)
_KEY = np.uint64(0xD6E8FEB86659FD93)
_HI = np.uint64(0xFFFFFFFF00000000)


def _draws(seeds, S, flip=True):
    """frcnn_voc_augment_batch's draw (include/frcnn_b200.h) in NumPy: (flip [n], scale index [n]) for int64 seeds."""
    s = np.asarray(seeds, np.int64).view(np.uint64) ^ _mix64(np.array([3], np.uint64))[0]
    with np.errstate(over="ignore"):
        k0 = (_mix64(s ^ (np.uint64(0) * _KEY)) & _HI) | np.uint64(0)
        k1 = (_mix64(s ^ (np.uint64(1) * _KEY)) & _HI) | np.uint64(1)
    f = (k0 >> np.uint64(63)).astype(np.int64) if flip else np.zeros(len(s), np.int64)
    return f, ((k1 >> np.uint64(32)) * np.uint64(S) >> np.uint64(32)).astype(np.int64)


def _edge_boxes(boxes, sizes):
    """The photos' boxes with a first box touching x = 0 and x = w0 - 1."""
    out = []
    for b, (h, w) in zip(boxes, sizes):
        b = b.copy()
        b[0, 0], b[0, 2] = 0.0, w - 1
        out.append(b)
    return out


def _float_batch(photos, boxes, labels, flips, scales):
    xs, gts = [], []
    for p, b, l, f, s in zip(photos, boxes, labels, flips, scales):
        img, _, gt = voc_aug_ref.voc_transform(p, b, l, flip=bool(f), scale=s)
        xs.append(torch.from_numpy(img).cuda())
        gts.append(torch.from_numpy(gt).cuda())
    return xs, gts


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("N", [1, 2, 4])
def test_flip_pack_and_boxes_equal_oracle(N, precision):
    from frcnn_b200 import ops
    from frcnn_b200.engine import ImageInput, RawPhotoInput
    for mix in range(2):
        sizes = [VOC[(mix * 3 + k) % len(VOC)] for k in range(N - (1 if N > 1 and mix else 0))]   # mix 1: an empty slot
        photos, boxes, labels = _photos(sizes, 20 * N + mix)
        boxes = _edge_boxes(boxes, sizes)
        flips = [(n + mix) % 2 for n in range(len(sizes))]
        index = [(n + mix) % len(SCALES) for n in range(len(sizes))]
        raw = RawPhotoInput(N, HC, WC, "cuda", max_gt=8, scales=SCALES)
        raw.upload(photos, boxes=boxes, labels=labels, flips=flips, scale_index=index)
        raw.augment(None, 0)
        planes = lambda: ops.Act(torch.full((N, HC, WC, 32), 7.0, dtype=torch.bfloat16, device="cuda"),  # noqa: E731
                                 torch.full((N, HC, WC, 32), 7.0, dtype=torch.bfloat16, device="cuda") if precision == "bf16x3" else None)
        got = ops.preprocess_voc_im2col_canvas_flip(*raw.descriptors, raw.aug["flip"], HC, WC, raw.pixel_means, 3, 1, 1, 32,
                                                    out=planes())
        gt = torch.full((N, 8, 5), 9.0, device="cuda")
        cnt = torch.full((N,), 9, dtype=torch.int32, device="cuda")
        ops.voc_flip_scale_gt(*raw.gt_fields, raw.descriptors[2], raw.aug["flip"], gt, cnt)
        xs, gts = _float_batch(photos, boxes, labels, flips, [SCALES[k] for k in index])
        ref_in = ImageInput(N, HC, WC, "cuda", canvas=True)
        ref_in.put(xs)
        want = ops.pack_image_im2col_batch(ref_in.x_in, 3, 1, 1, 32, precision=precision, extents=ref_in.extents)
        # every flip at 0: the _flip entries are the plain entries bit for bit
        raw.aug["flip"].zero_()
        plain, flat = planes(), planes()
        ops.preprocess_voc_im2col_canvas(*raw.descriptors, HC, WC, raw.pixel_means, 3, 1, 1, 32, out=plain)
        ops.preprocess_voc_im2col_canvas_flip(*raw.descriptors, raw.aug["flip"], HC, WC, raw.pixel_means, 3, 1, 1, 32, out=flat)
        gt0, gt1 = torch.full_like(gt, 5.0), torch.full_like(gt, 6.0)
        ops.voc_scale_gt(*raw.gt_fields, gt0, cnt.clone())
        ops.voc_flip_scale_gt(*raw.gt_fields, raw.descriptors[2], raw.aug["flip"], gt1, cnt.clone())
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
        for g, w in zip(_bits(flat), _bits(plain)):
            assert torch.equal(g, w), (N, mix)
        assert _flat_equal(gt0, gt1)


@pytest.mark.parametrize("S", [1, 3, 5])
def test_draws_equal_restatement(S):
    from frcnn_b200 import ops
    n = 4096
    rng = np.random.default_rng(S)
    seeds = rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    cand_hw = rng.integers(1, 1000, (n, S, 2)).astype(np.int32)
    cand_inv = rng.uniform(0.3, 3.0, (n, S))
    cand_scale = (1.0 / cand_inv).astype(np.float32)
    src_hw = rng.integers(1, 500, (n, 2)).astype(np.int32)
    src_hw[7] = (0, 0)                                                    # an empty slot
    for draw in (1, 2):
        choice = torch.full((n, 2), -5, dtype=torch.int32, device="cuda")
        out = dict(flip=torch.full((n,), 9, dtype=torch.int32, device="cuda"),
                   extents=torch.full((n, 2), -1, dtype=torch.int32, device="cuda"),
                   im_info=torch.full((n, 2), -1, dtype=torch.int32, device="cuda"),
                   inv_scale=torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
                   scale=torch.full((n,), -1.0, dtype=torch.float32, device="cuda"))
        ops.voc_augment(dev(seeds), dev(cand_hw), dev(cand_inv), dev(cand_scale), dev(src_hw), choice, out["flip"], out["extents"],
                        out["im_info"], out["inv_scale"], out["scale"], draw)
        torch.cuda.synchronize()
        f, k = _draws(seeds, S, flip=draw == 1)
        c = choice.cpu().numpy()
        assert np.array_equal(c[:, 0], f) and np.array_equal(c[:, 1], k)
        if draw == 1:
            assert 0.45 <= f.mean() <= 0.55
        counts = np.bincount(k, minlength=S)
        assert len(counts) == S and np.all(np.abs(counts - n / S) <= 0.15 * n / S), counts
        live = np.ones(n, bool)
        live[7] = False
        r = np.arange(n)
        assert np.array_equal(out["extents"].cpu().numpy()[live], cand_hw[r, k][live])
        assert np.array_equal(out["im_info"].cpu().numpy(), out["extents"].cpu().numpy())
        assert np.array_equal(out["inv_scale"].cpu().numpy()[live], cand_inv[r, k][live])
        assert np.array_equal(out["scale"].cpu().numpy()[live].view(np.uint32), cand_scale[r, k][live].view(np.uint32))
        assert np.array_equal(out["flip"].cpu().numpy()[live], f[live])
        assert not out["extents"][7].any() and float(out["inv_scale"][7]) == 0 and int(out["flip"][7]) == 0
    # draw 0 reads the staged choice, clamping the index
    choice = dev(np.stack([np.arange(n) % 2, np.arange(n) % (S + 3) - 1], 1).astype(np.int32))
    ops.voc_augment(None, dev(cand_hw), dev(cand_inv), dev(cand_scale), dev(src_hw), choice, out["flip"], out["extents"],
                    out["im_info"], out["inv_scale"], out["scale"], 0)
    torch.cuda.synchronize()
    k = np.clip(np.arange(n) % (S + 3) - 1, 0, S - 1)
    assert np.array_equal(out["extents"].cpu().numpy()[live], cand_hw[np.arange(n), k][live])
    assert np.array_equal(out["flip"].cpu().numpy()[live], (np.arange(n) % 2)[live])


def _mixes(N):
    return [[VOC[(3 * t + k) % len(VOC)] for k in range(N - (1 if N > 1 and t == 1 else 0))] for t in range(3)]


def _run_pair(raw, flt, N, photo_seed, extra=None, list_mode=False):
    """Three steps of the augmenting raw trainer and its float twin on the host transform of the raw trainer's choices;
    bit-identical losses, gradient, weights and optimizer state after each.  Returns the per-step choices."""
    rng = np.random.default_rng(photo_seed)
    captured, seen = None, []
    for t, sizes in enumerate(_mixes(N)):
        photos, boxes, labels = _photos(sizes, photo_seed + t)
        boxes = _edge_boxes(boxes, sizes)
        kw = dict(extra(sizes) if extra else {})
        if list_mode:
            kw.update(flips=[bool(v) for v in rng.integers(0, 2, len(sizes))],
                      scale_index=[int(v) for v in rng.integers(0, len(SCALES), len(sizes))])
        cands = raw.put_raw(photos, boxes, labels, **kw)
        assert [len(c) for c in cands] == [len(SCALES)] * len(sizes)
        lr_ = raw._step()
        aug = raw.augmentation()
        assert raw.image_sizes == [a[2] for a in aug]
        flips = [a[0] for a in aug[:len(sizes)]]
        index = [int(v) for v in raw.input.aug["choice"][:len(sizes), 1].cpu()]
        assert [aug[n][1] for n in range(len(sizes))] == [cands[n][index[n]] for n in range(len(sizes))]
        if list_mode:
            assert flips == kw["flips"] and index == kw["scale_index"]
        for n, (h0, w0) in enumerate(sizes):
            assert aug[n][2] == voc_ref.plan_size(h0, w0, SCALES[index[n]])[1:]
        assert all(a == (False, 0.0, (0, 0)) for a in aug[len(sizes):])
        xs, gts = _float_batch(photos, boxes, labels, flips, [SCALES[k] for k in index])
        fkw = {k: v for k, v in kw.items() if k not in ("flips", "scale_index")}
        lf = flt.step(xs, gts, **fkw)
        torch.cuda.synchronize()
        captured = captured or raw.graph
        assert raw.graph is captured and raw.n_updates == t + 1
        assert _flat_equal(lr_, lf), t
        assert _flat_equal(raw.g_flat, flt.g_flat), t
        assert _flat_equal(raw.w_flat, flt.w_flat) and _flat_equal(raw.v_flat, flt.v_flat), t
        seen.append(tuple(zip(flips, index)))
    return seen


@pytest.mark.parametrize("mode", ["device", "list"])
@pytest.mark.parametrize("N", [1, 4])
def test_rpn_augmented_step_equals_float_step(N, mode):
    from frcnn_b200.train_engine import CanvasRpnTrainer
    params = _train_case(HC, WC, 3)[0]
    raw = CanvasRpnTrainer(params, N, HC, WC, ANCHORS, seed=5, raw_input=True, augment=mode, scales=SCALES)
    flt = CanvasRpnTrainer(params, N, HC, WC, ANCHORS, seed=5)
    seen = _run_pair(raw, flt, N, 500 + N, list_mode=mode == "list")
    assert len(set(seen)) > 1, seen                       # the draws change between replays of the one graph
    if mode == "device":                                  # slot n of step t draws with seed + t*N + n
        f, k = _draws(np.arange(3 * N) + 5, len(SCALES))
        assert seen == [tuple((bool(f[t * N + n]), int(k[t * N + n])) for n in range(len(sizes))) for t, sizes in enumerate(_mixes(N))]


def test_rcnn_augmented_step_equals_float_step():
    """Augmentation shares the step's seed advance: the device sampling and dropout still draw what the float trainer's do."""
    from frcnn_b200.train_engine import CanvasRcnnTrainer
    N = 2
    params = _rcnn_params(HC, WC, 7)
    kw = dict(post_n=300, seed=11, sample="device", dropout="device")
    raw = CanvasRcnnTrainer(params, N, HC, WC, ANCHORS, raw_input=True, augment="device", scales=SCALES, **kw)
    flt = CanvasRcnnTrainer(params, N, HC, WC, ANCHORS, **kw)
    seen = _run_pair(raw, flt, N, 700)
    assert len(set(seen)) > 1, seen
    assert torch.equal(raw.masks, flt.masks) and torch.equal(raw.seeds, flt.seeds)


def test_resnet_augmented_step_equals_float_step():
    """The level extents are derived after the selection."""
    from test_resnet_train_gpu import _case
    from frcnn_b200.resnet_train import CanvasResNetRpnTrainer
    N = 2
    params = _case(50, HC, WC, 3)[0]
    raw = CanvasResNetRpnTrainer(params, N, HC, WC, ANCHORS, n_layers=50, seed=5, raw_input=True, augment="device",
                                 scales=SCALES)
    flt = CanvasResNetRpnTrainer(params, N, HC, WC, ANCHORS, n_layers=50, seed=5)
    seen = _run_pair(raw, flt, N, 900)
    assert len(set(seen)) > 1, seen
