"""GPU tests of the RCNN training step on a canvas of images of different sizes (CanvasRcnnTrainer) and of its four batched
entries: frcnn_proposal_targets_batch, frcnn_rcnn_loss_batch, frcnn_roi_pool_backward_batch_ext and
frcnn_dropout_masks_batch.

The reference for every per-slot number is the one-image path on that slot alone (frcnn_roi_overlaps + frcnn_roi_targets,
frcnn_rcnn_loss, frcnn_roi_pool_backward, RcnnTrainer with the slot's kept list and masks), and the bar is bit-identity.
Device-mode sampling is checked against the oracle's ProposalTargetLayer with a `choice` that restates the key rule in
NumPy.  Only the summed weight gradients are compared within 5e-5 of max-norm against the float64 sum of the per-image
gradients."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_canvas_train_gpu import _flat_equal, _gt_boxes, _images
from test_train_gpu import _rel, _train_case
from test_train_targets_edges_gpu import _mix64, _sample_key

pytestmark = pytest.mark.gpu
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
BG_XOR = 0xA5A5A5A5DEADBEEF


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------------------------------------ proposal targets
R_CAP, MAX_GT, NC = 300, 6, 21
# (R_n, G_n) per slot: ragged counts, a slot without ground truth, one without RoIs, one at R_cap
PT_SLOTS = [(211, 3), (300, 6), (57, 0), (0, 2), (140, 1)]


def _pt_case(seed=0):
    rng = np.random.default_rng(seed)
    N = len(PT_SLOTS)
    rois = np.full((N, R_CAP, 4), 7e3, f32)                 # poison past each count
    gt = np.full((N, MAX_GT, 5), 5e3, f32)
    for n, (R, G) in enumerate(PT_SLOTS):
        g = _gt_boxes(rng, 480, 640, max(G, 1))
        if n == 0:
            g[0] = [0, 0, 99, 99, 4]                        # exact IoU boundaries against this row
        gt[n, :G] = g[:G]
        c = g[rng.integers(0, len(g), R)]
        jit = rng.normal(0, 1, (R, 4)) * np.array([[0.15, 0.15, 0.15, 0.15]]) * (c[:, 2:3] - c[:, 0:1] + 1)
        r = np.floor(c[:, :4] + jit * rng.uniform(0, 3, (R, 1)))
        r[:, 2:] = np.maximum(r[:, 2:], r[:, :2] + 1)
        rois[n, :R] = r
    rois[0, :4] = [[0, 0, 99, 49], [0, 0, 99, 9], [0, 0, 99, 10], [0, 0, 99, 48]]     # IoU 0.5, 0.1, just above / below
    rois[0, 4] = [np.nan, 0, 10, 10]                        # a NaN coordinate: overlap 0 (bbox.pyx's iw > 0 test), in neither set
    rois[1, 5:8] = rois[1, 4]                               # equal boxes: equal overlaps, distinct keys
    counts = np.array([[1, R] for R, _ in PT_SLOTS], np.int32)
    return rois, gt, counts


def _key_choice(seed, max_ov):
    def choice(inds, size):
        s = seed if max_ov[inds[0]] >= 0.5 else seed ^ BG_XOR
        k = _sample_key(s, np.asarray(inds))
        return np.sort(np.asarray(inds)[np.argsort(k, kind="stable")[:size]])
    return choice


def test_key_restatement():
    assert int(_mix64(np.array([0], np.uint64))[0]) == 0xE220A8397B1DCDAF


@pytest.mark.parametrize("mode", [1, 2])
def test_proposal_targets_batch(mode):
    from frcnn_b200 import train_ops
    rois, gt, counts = _pt_case()
    N = len(PT_SLOTS)
    work = train_ops.ProposalTargetsBatch(N, R_CAP, NC, "cuda")
    for t in (work.keep, work.labels, work.argmax, work.counts):
        t.fill_(-7)
    for t in (work.use_gt, work.bbox_reg_targets, work.max_overlaps):
        t.fill_(float("nan"))
    seeds = np.array([3, 2 ** 50 + 1, 9, 10, 123456789], np.uint64)
    rng = np.random.default_rng(3)
    lists = []
    for R, _ in PT_SLOTS:
        k = rng.permutation(np.arange(-2, max(R, 1) + 3))[:min(128, max(R, 1) + 5)].astype(np.int32)
        lists.append(k)
    offs = np.concatenate([[0], np.cumsum([len(v) for v in lists])]).astype(np.int32)
    cnt = _dev(counts)
    train_ops.proposal_targets_batch(_dev(rois), cnt[:, 1], _dev(gt), _dev(np.array([g for _, g in PT_SLOTS], np.int32)), work,
                                     mode=mode, seeds=_dev(seeds.view(np.int64)), keep_list=_dev(np.concatenate(lists)),
                                     list_offsets=_dev(offs))
    torch.cuda.synchronize()
    c = work.counts.cpu().numpy()
    for n, (R, G) in enumerate(PT_SLOTS):
        if R == 0 or G == 0:
            assert c[n].tolist() == [0] * 8, n
            assert (work.keep[n] == -1).all()
            continue
        rd, gd = _dev(rois[n]), _dev(gt[n, :G])
        mo, am = train_ops.roi_overlaps(rd, _dev(np.array([R], np.int32)), gd)
        assert _flat_equal(work.max_overlaps[n].view(torch.int32), mo.view(torch.int32)), n
        assert torch.equal(work.argmax[n], am), n
        if mode == 2:
            valid = [int(r) for r in lists[n] if 0 <= r < R]
            assert c[n][0] == len(valid) and c[n][4] == len(lists[n]) - len(valid), n
            keep = _dev(np.array(valid, np.int32))
        else:
            mo_np = mo.cpu().numpy()[:R]
            ref = orc.proposal_target_layer(rois[n, :R], gt[None, n, :G], NC, choice=_key_choice(int(seeds[n]), mo_np))
            keep_np = ref["keep_inds"]
            assert work.keep[n, :c[n][0]].cpu().numpy().tolist() == keep_np.tolist(), n
            fg, bg = (mo_np >= 0.5).sum(), ((mo_np >= 0.1) & (mo_np < 0.5)).sum()
            assert c[n][1:6].tolist() == [ref["n_fg"], fg, bg, 0, R], n
            keep = _dev(keep_np)
        k = int(c[n][0])
        assert torch.equal(work.keep[n, :k], keep) and bool((work.keep[n, k:] == -1).all()), n
        use_gt, ext, labels = train_ops.roi_targets(rd, gd, am, keep, NC)
        assert _flat_equal(work.use_gt[n, :k], use_gt) and _flat_equal(work.bbox_reg_targets[n, :k], ext), n
        assert torch.equal(work.labels[n, :k], labels), n
        if mode == 1:
            np.testing.assert_array_equal(work.use_gt[n, :k].cpu().numpy(), ref["use_gt_boxes"])
            # the oracle's NumPy log may differ from the device's logf in the last bit (bit-equality with frcnn_roi_targets
            # is checked above)
            np.testing.assert_allclose(work.bbox_reg_targets[n, :k].cpu().numpy(), ref["bbox_reg_targets"], rtol=1e-6, atol=0)
    if mode == 1:                                            # the boundary rows of slot 0
        mo0 = work.max_overlaps[0, :5].cpu().numpy()
        assert mo0[0] == 0.5 and mo0[1] == 0.1 and mo0[4] == 0.0


# a seed whose fg keys of rows 25 and 131 share their top 32 bits (found by a host search over seeds)
TIE_SEED, TIE_LO, TIE_HI = 284096, 25, 131


def _tie_and_nan_case():
    inf = np.inf
    keys = _sample_key(TIE_SEED, np.arange(300))
    assert keys[TIE_LO] >> np.uint64(32) == keys[TIE_HI] >> np.uint64(32)
    below = [int(r) for r in np.argsort(keys, kind="stable") if keys[r] < keys[TIE_LO]][:31]
    rois = np.zeros((2, 300, 4), f32)
    gt = np.zeros((2, 2, 5), f32)
    # slot 0: 33 fg rows, the tied pair ranked 32nd / 33rd by key: the quota of 32 keeps the lower index of the pair only
    gt[0, 0] = [0, 0, 99, 99, 5]
    rois[0] = [300, 300, 350, 350]
    rois[0, below + [TIE_LO, TIE_HI]] = [0, 0, 99, 99]
    # slot 1: an infinite gt box; every infinite RoI has a NaN IoU with it (inf / NaN arithmetic), 0 with the finite box
    gt[1] = [[0, 0, 99, 99, 2], [-inf, -inf, inf, inf, 3]]
    rng = np.random.default_rng(4)
    rois[1, :60] = np.floor([0, 0, 99, 99] + rng.normal(0, 15, (60, 4)))
    rois[1, 60:100] = [-inf, -inf, inf, inf]
    counts = np.array([[1, 300], [1, 100]], np.int32)
    return rois, gt, counts, np.array([1, 2], np.int32), sorted(below + [TIE_LO])


def test_proposal_targets_device_hash_tie_and_nan_overlaps():
    from frcnn_b200 import train_ops
    rois, gt, counts, gtc, want0 = _tie_and_nan_case()
    work = train_ops.ProposalTargetsBatch(2, R_CAP, NC, "cuda")
    seeds = np.array([TIE_SEED, 77], np.uint64)
    train_ops.proposal_targets_batch(_dev(rois), _dev(counts)[:, 1], _dev(gt), _dev(gtc), work, mode=1,
                                     seeds=_dev(seeds.view(np.int64)))
    torch.cuda.synchronize()
    c = work.counts.cpu().numpy()
    assert c[0].tolist() == [32, 32, 33, 0, 0, 300, 0, 0]
    assert work.keep[0, :32].cpu().numpy().tolist() == want0 and TIE_HI not in want0
    for n in range(2):
        R, G = int(counts[n, 1]), int(gtc[n])
        mo = work.max_overlaps[n, :R].cpu().numpy()
        ref = orc.proposal_target_layer(rois[n, :R], gt[None, n, :G], NC, choice=_key_choice(int(seeds[n]), mo))
        assert work.keep[n, :c[n][0]].cpu().numpy().tolist() == ref["keep_inds"].tolist(), n
        assert c[n][1] == ref["n_fg"], n
        if n == 1:
            assert np.isnan(ref["max_overlaps"][60:]).all()        # NaN: in neither set, on the device as in the oracle
            assert (work.keep[1, :c[1][0]].cpu().numpy() < 60).all()


# ------------------------------------------------------------------------------------------------ loss
def test_rcnn_loss_batch_equals_per_slot():
    from frcnn_b200 import train_ops
    rois, gt, counts = _pt_case(1)
    N = len(PT_SLOTS)
    work = train_ops.ProposalTargetsBatch(N, R_CAP, NC, "cuda")
    train_ops.proposal_targets_batch(_dev(rois), _dev(counts)[:, 1], _dev(gt), _dev(np.array([g for _, g in PT_SLOTS], np.int32)),
                                     work, mode=1, seeds=_dev(np.arange(N, dtype=np.int64) + 40))
    ld = 128
    head = _dev(np.random.default_rng(2).standard_normal((N * R_CAP, ld)).astype(f32))
    dhead = torch.full_like(head, float("nan"))
    losses = train_ops.rcnn_loss_batch(head, work, delta=1.0, dhead=dhead).clone()
    torch.cuda.synchronize()
    c = work.counts.cpu().numpy()
    assert (c[:, 0] == 0).sum() >= 2
    for n in range(N):
        rows = slice(n * R_CAP, (n + 1) * R_CAP)
        k = int(c[n][0])
        if k == 0:
            assert losses[n].cpu().numpy().tolist() == [0.0] * 4 and bool((dhead[rows] == 0).all()), n
            continue
        lo, dh = train_ops.rcnn_loss(head[rows], work.keep[n, :k], work.labels[n, :k], work.bbox_reg_targets[n, :k], NC, 1.0)
        assert _flat_equal(losses[n], lo) and _flat_equal(dhead[rows].contiguous(), dh), n


# ------------------------------------------------------------------------------------------------ RoI pooling backward
def test_roi_pool_backward_batch_equals_per_slot():
    from frcnn_b200 import ops, train_ops
    N, fhc, fwc, C, R = 4, 38, 63, 64, 50
    ext_px = np.array([[600, 1000], [333, 500], [0, 0], [187, 613]], np.int32)
    gen = torch.Generator(device="cuda").manual_seed(5)
    hi = torch.randn((N, fhc, fwc, C), device="cuda", generator=gen).to(torch.bfloat16)
    lo = (torch.randn((N, fhc, fwc, C), device="cuda", generator=gen) * 1e-3).to(torch.bfloat16)
    for n, (h, w) in enumerate(ext_px):                       # the canvas is 0 outside each image
        hi[n, -(-h // 16):] = 0
        hi[n, :, -(-w // 16):] = 0
        lo[n, -(-h // 16):] = 0
        lo[n, :, -(-w // 16):] = 0
    rng = np.random.default_rng(7)
    rois = np.zeros((N, R, 4), f32)
    for n, (h, w) in enumerate(ext_px):
        x1, y1 = rng.uniform(-50, max(w, 1), R), rng.uniform(-50, max(h, 1), R)
        rois[n] = np.stack([x1, y1, x1 + rng.uniform(0, 400, R), y1 + rng.uniform(0, 300, R)], 1)   # some past the image
    cnt = np.array([[1, 50], [1, 31], [1, 0], [1, 44]], np.int32)
    g = ops.Act(torch.randn((N, R, 49 * C), device="cuda", generator=gen).to(torch.bfloat16),
                (torch.randn((N, R, 49 * C), device="cuda", generator=gen) * 1e-3).to(torch.bfloat16))
    feat, rd, cd = ops.Act(hi, lo), _dev(rois), _dev(cnt)
    out = train_ops.roi_pool_backward_batch(feat, rd, cd[:, 1], g, _dev(ext_px), 4, 7, 7, 1.0 / 16)
    out = out.view(N, fhc, fwc, C)
    torch.cuda.synchronize()
    for n, (h, w) in enumerate(ext_px):
        fh, fw = -(-h // 16), -(-w // 16)
        if fh == 0:
            assert bool((out[n] == 0).all())
            continue
        one = train_ops.roi_pool_backward(ops.Act(hi[n, :fh, :fw].contiguous(), lo[n, :fh, :fw].contiguous()), rd[n],
                                          cd[n, 1:2].contiguous(), ops.Act(g.hi[n][None], g.lo[n][None]), 7, 7, 1.0 / 16)
        assert _flat_equal(out[n, :fh, :fw].contiguous(), one.view(fh, fw, C)), n
        rest = out[n].clone()
        rest[:fh, :fw] = 0
        assert bool((rest == 0).all()), n


# ------------------------------------------------------------------------------------------------ dropout masks
def _masks_ref(seed, salt, rows, cols):
    with np.errstate(over="ignore"):
        s = np.uint64(seed) ^ _mix64(np.array([salt], np.uint64))[0]
    return (_sample_key(int(s), np.arange(rows * cols)) >> np.uint64(63)).astype(np.uint8).reshape(rows, cols)


def test_dropout_masks_batch():
    from frcnn_b200 import train_ops
    seeds = np.array([0, 1, 2 ** 63 + 5], np.uint64)
    out = torch.full((3, 37, 4096), 9, dtype=torch.uint8, device="cuda")
    train_ops.dropout_masks_batch(_dev(seeds.view(np.int64)), 1, out)
    got = out.cpu().numpy()
    for n, s in enumerate(seeds):
        np.testing.assert_array_equal(got[n], _masks_ref(int(s), 1, 37, 4096))
    assert 0.48 < got.mean() < 0.52
    other = torch.empty_like(out)
    train_ops.dropout_masks_batch(_dev(seeds.view(np.int64)), 2, other)       # another layer's salt
    assert not torch.equal(other, out)


# ------------------------------------------------------------------------------------------------ the step
def _rcnn_params(H, W, seed):
    params = _train_case(H, W, seed)[0]
    rng = np.random.default_rng(seed + 1)
    for k in ("cls_score/W", "bbox_pred/W"):
        params[k] = (rng.standard_normal(params[k].shape) * 0.02).astype(f32)
    return params


def _keep_and_masks(rt, x, gt, post_n, seed):
    """A kept list the reference would draw for this image (NumPy sampling on its proposals) and explicit masks."""
    np.random.seed(seed)
    rt.forward(x, gt)
    torch.cuda.synchronize()
    keep = rt.keep.clone()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    masks = [(torch.rand((post_n, 4096), device="cuda", generator=gen) >= 0.5).to(torch.uint8) for _ in range(2)]
    return keep, masks


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_full_size_step_is_rcnn_trainer_bit_for_bit(precision):
    from frcnn_b200.train_engine import CanvasRcnnTrainer, RcnnTrainer
    H, W, post_n = 296, 392, 120
    params = _rcnn_params(H, W, 3)
    xs, gts = _images([(H, W)] * 2, 4)
    rt = RcnnTrainer(params, H, W, ANCHORS, precision=precision, post_n=post_n)
    ct = CanvasRcnnTrainer(params, 1, H, W, ANCHORS, precision=precision, post_n=post_n, sample="list", dropout="explicit")
    for k in range(2):
        keep, masks = _keep_and_masks(rt, xs[k], gts[k], post_n, 10 + k)
        lr_ = rt.forward(xs[k], gts[k], keep_inds=keep, masks=masks)
        rt.backward()
        ct.put([xs[k]], [gts[k]], keep_inds=[keep], masks=[masks])
        lc = ct.forward().clone()
        ct.backward()
        torch.cuda.synchronize()
        assert _flat_equal(lc[0], lr_), k
        R = int(rt.prop.count.item())
        assert int(ct.head_ext[0, 1]) == R
        assert _flat_equal(ct.prop.rois[0, :R].contiguous(), rt.prop.rois[:R].contiguous()), k
        assert _flat_equal(ct.head_grad, rt.head_grad), k
        assert _flat_equal(ct.dfeat, rt.dfeat), k
        assert _flat_equal(ct.g_flat, rt.g_flat), k
        rt.update()
        ct.update()
        torch.cuda.synchronize()
        assert _flat_equal(ct.w_flat, rt.w_flat) and _flat_equal(ct.v_flat, rt.v_flat), k


MIX = [(296, 392), (250, 300), (161, 377)]          # plus one empty slot


def test_mixed_sizes_equal_per_image_trainers():
    from frcnn_b200.train_engine import CanvasRcnnTrainer, RcnnTrainer
    Hc, Wc, post_n = 296, 392, 100
    params = _rcnn_params(Hc, Wc, 5)
    xs, gts = _images(MIX, 6)
    refs, keeps, masks = [], [], []
    for n, (h, w) in enumerate(MIX):
        rt = RcnnTrainer(params, h, w, ANCHORS, post_n=post_n)
        k, m = _keep_and_masks(rt, xs[n], gts[n], post_n, 20 + n)
        refs.append(rt)
        keeps.append(k)
        masks.append(m)
    ct = CanvasRcnnTrainer(params, 4, Hc, Wc, ANCHORS, post_n=post_n, sample="list", dropout="explicit")
    ct.put(xs, gts, keep_inds=keeps, masks=masks)
    losses = ct.forward().clone()
    dbg = {}
    ct.backward(debug=dbg)
    torch.cuda.synchronize()
    assert losses[3].cpu().numpy().tolist() == [0.0] * 4                       # the empty slot
    gsum = {k: np.zeros(ct.index[k][2], np.float64) for k in ct.index}
    dfeat = ct.dfeat.view(4, ct.fh, ct.fw, 512)
    for n, rt in enumerate(refs):
        lo = rt.forward(xs[n], gts[n], keep_inds=keeps[n], masks=masks[n])
        rd = {}
        rt.backward(debug=rd)
        torch.cuda.synchronize()
        assert _flat_equal(losses[n], lo), n
        R = int(rt.prop.count.item())
        assert int(ct.head_ext[n, 1]) == R, n
        assert _flat_equal(ct.prop.rois[n, :R].contiguous(), rt.prop.rois[:R].contiguous()), n
        for a, b in ((ct.fc6, rt.fc6), (ct.fc7, rt.fc7), (ct.pool5, rt.pool5)):
            assert torch.equal(a.hi[n, 0, :R], b.hi[0, :R]) and torch.equal(a.lo[n, 0, :R], b.lo[0, :R]), n
        rows = slice(n * post_n, (n + 1) * post_n)
        assert _flat_equal(ct.head_grad[rows].contiguous(), rt.head_grad), n
        assert _flat_equal(dbg["roi"]["dpool5"][n][:, :, :R].contiguous(), rd["roi"]["dpool5"][:, :, :R].contiguous()), n
        fh, fw = rt.fh, rt.fw
        assert _flat_equal(dfeat[n, :fh, :fw].contiguous(), rt.dfeat.view(fh, fw, 512)), n
        rest = dfeat[n].clone()
        rest[:fh, :fw] = 0
        assert bool((rest == 0).all()), n
        for key, d in rd.items():
            if not key.startswith("trunk/"):
                continue
            for f, v in d.items():
                c = dbg[key][f][n]
                _, hh, ww = v.shape
                assert _flat_equal(c[:, :hh, :ww].contiguous(), v), (key, f, n)
                out = c.clone()
                out[:, :hh, :ww] = 0
                assert bool((out == 0).all()), (key, f, n)
        for k in ct.index:
            gsum[k] += rt.grads(k).cpu().numpy()
    worst = max(_rel(ct.grads(k).cpu().numpy(), gsum[k]) for k in ct.index)
    print("summed-gradient worst error (of max-norm): %.2e" % worst)
    assert worst <= 5e-5


def test_graph_replay_equals_eager_run():
    from frcnn_b200.train_engine import CanvasRcnnTrainer
    Hc, Wc, N, post_n = 296, 392, 3, 100
    params = _rcnn_params(Hc, Wc, 7)
    xs, gts = _images(MIX, 8)
    kw = dict(post_n=post_n, sample="device", dropout="device", seed=31)
    a = CanvasRcnnTrainer(params, N, Hc, Wc, ANCHORS, **kw)
    b = CanvasRcnnTrainer(params, N, Hc, Wc, ANCHORS, **kw)
    masks = []
    for it in range(3):
        la = a.step(xs, gts)                                 # eager, then capture, then replays
        masks.append(a.masks.clone())
        b.put(xs, gts)
        b.run()
        torch.cuda.synchronize()
        assert _flat_equal(la, b.ptargets.losses), it
        assert torch.equal(a.masks, b.masks) and torch.equal(a.ptargets.keep, b.ptargets.keep), it
        assert _flat_equal(a.w_flat, b.w_flat), it
    assert a.graph is not None and a.n_updates == 3
    assert not torch.equal(masks[1], masks[2])              # replays draw fresh masks
    ref = _masks_ref(31 + 2 * N + 1, 1, post_n, 4096)         # step 2, slot 1, fc6
    np.testing.assert_array_equal(masks[2][0, 1].cpu().numpy(), ref)


def test_headline_size_float64_check():
    """test_train_gpu.test_rcnn_train_step_layerwise_and_end_to_end on the canvas trainer at 600x1000 with the default 300
    proposals (N = 1, the reference's kept set in list mode, explicit masks): fc weight / data gradients vs float64
    products of the step's own tensors, exact ReLU + dropout masking, RoI-pool backward vs autograd on its feature map,
    end to end against the autograd oracle (losses 2e-4, gradients 3e-2 of max-norm), and one update lowers the loss."""
    import torchvision
    from frcnn_b200.train_engine import CanvasRcnnTrainer
    from test_train_gpu import _ulp_diff_f32
    H, W, post_n = 600, 1000, 300
    params, x, gt, info = _train_case(H, W, 5)
    rng = np.random.default_rng(12)
    for k in ("fc6/W", "fc7/W", "cls_score/W", "bbox_pred/W"):
        params[k] = (rng.standard_normal(params[k].shape) * (0.002 if k == "fc6/W" else 0.01)).astype(f32)
    gt[0, :, 4] = [3, 7, 1]
    xd, gd = _dev(x[0]), _dev(gt[0])
    ct = CanvasRcnnTrainer(params, 1, H, W, ANCHORS, post_n=post_n, sample="list", dropout="explicit")
    ct.put([xd], [gd], keep_inds=[torch.zeros((0,), dtype=torch.int32)])
    ct.forward()                                             # the proposals, to draw the kept set from
    torch.cuda.synchronize()
    R = int(ct.head_ext[0, 1])
    rois = ct.prop.rois[0, :R].cpu().numpy()
    np.random.seed(5)
    ro = orc.proposal_target_layer(rois, gt)                 # the reference's draw on these proposals
    keep = ro["keep_inds"]
    gen = torch.Generator(device="cuda").manual_seed(3)
    mk = [(torch.rand((post_n, 4096), device="cuda", generator=gen) >= 0.5).to(torch.uint8) for _ in range(2)]
    ct.put([xd], [gd], keep_inds=[torch.from_numpy(keep)], masks=[mk])
    losses = ct.forward().clone()[0]
    dbg = {}
    ct.backward(debug=dbg)
    torch.cuda.synchronize()
    pt = ct.ptargets
    n_keep = int(pt.counts[0, 0])
    assert n_keep == len(keep) and np.array_equal(pt.keep[0, :n_keep].cpu().numpy(), keep)
    labels, ext = pt.labels[0, :n_keep].cpu().numpy(), pt.bbox_reg_targets[0, :n_keep].cpu().numpy()
    assert np.array_equal(pt.use_gt[0, :n_keep].cpu().numpy(), ro["use_gt_boxes"])
    assert _ulp_diff_f32(ext, ro["bbox_reg_targets"]).max() <= 2
    masks = [m.cpu().numpy()[:R] for m in mk]
    print("R=%d kept=%d" % (R, n_keep))
    # ---- local checks on the step's own tensors (float64 references)
    f64 = lambda a: np.asarray(a, np.float64)                                     # noqa: E731
    val = lambda a: (a.hi.float() + a.lo.float()).cpu().numpy()[0, 0]          # noqa: E731  [R_cap, C]
    flat = lambda t: f64(t[0].cpu().numpy().reshape(t.shape[1], -1).T)          # noqa: E731  [N, C, 1, R_cap] -> [R_cap, C]
    dyh = f64(ct.head_grad.cpu().numpy())
    fc7, fc6, pool5 = f64(val(ct.fc7)), f64(val(ct.fc6)), f64(val(ct.pool5))
    Wh = f64(np.concatenate([params["cls_score/W"], params["bbox_pred/W"]], 0))
    got_wh = np.concatenate([ct.grads("cls_score/W").cpu().numpy(), ct.grads("bbox_pred/W").cpu().numpy()], 0)
    e = [_rel(got_wh, dyh[:, :105].T @ fc7)]
    e.append(_rel(np.concatenate([ct.grads("cls_score/b").cpu().numpy(), ct.grads("bbox_pred/b").cpu().numpy()]), dyh[:, :105].sum(0)))
    g7 = flat(dbg["fc7"]["g_in"])
    e.append(_rel(g7, dyh[:, :105] @ Wh))
    dy7 = flat(dbg["fc7"]["dy"])
    assert np.array_equal(dy7, np.where(fc7 > 0, 2.0 * g7, 0.0))
    e.append(_rel(ct.grads("fc7/W").cpu().numpy(), dy7.T @ fc6))
    e.append(_rel(ct.grads("fc7/b").cpu().numpy(), dy7.sum(0)))
    g6 = flat(dbg["fc6"]["g_in"])
    e.append(_rel(g6, dy7 @ f64(params["fc7/W"])))
    dy6 = flat(dbg["fc6"]["dy"])
    assert np.array_equal(dy6, np.where(fc6 > 0, 2.0 * g6, 0.0))
    W6_hwc = f64(params["fc6/W"]).reshape(4096, 512, 49).transpose(0, 2, 1).reshape(4096, -1)
    e.append(_rel(ct.grads("fc6/W").cpu().numpy(), dy6.T @ pool5))
    e.append(_rel(ct.grads("fc6/b").cpu().numpy(), dy6.sum(0)))
    dp5 = flat(dbg["roi"]["dpool5"])
    e.append(_rel(dp5, dy6 @ W6_hwc))
    print("head local errors (dWh, dbh, dX7, dW7, db7, dX6, dW6, db6, dpool5):", ["%.1e" % v for v in e])
    assert max(e) <= 5e-5
    # RoI-pool backward on the step's feature map
    feat = ct._chw(ct.feat)[0].cpu().numpy()
    xf = torch.from_numpy(feat).double()[None].requires_grad_(True)
    br = torch.cat([torch.zeros((R, 1), dtype=torch.float64), torch.from_numpy(rois).double()], 1)
    yp = torchvision.ops.roi_pool(xf, br, (7, 7), 1.0 / 16)
    yp.backward(torch.from_numpy(dp5[:R].reshape(R, 7, 7, 512).transpose(0, 3, 1, 2)))
    want_df = xf.grad[0].numpy().transpose(1, 2, 0).reshape(-1, 512)
    assert np.abs(dbg["roi"]["dfeat"].cpu().numpy() - want_df).max() <= 1e-6 * np.abs(want_df).max()
    # ---- end to end
    want = orc.rcnn_train_step(params, x, rois, keep, labels, ext, masks)
    Lv = losses.cpu().numpy()
    print("losses", Lv, "oracle", want["losses"])
    for i in (0, 1, 3):
        assert abs(Lv[i] - want["losses"][i]) <= 2e-4 * max(1.0, want["losses"][i])
    assert abs(Lv[2] - want["losses"][2]) <= 1.0 / len(keep) + 1e-6
    worst = 0.0
    for name in ct.index:
        gdev = ct.grads(name).cpu().numpy()
        if name == "fc6/W":
            gdev = gdev.reshape(4096, 49, 512).transpose(0, 2, 1).reshape(4096, -1)
        worst = max(worst, _rel(gdev, want["grads"][name]))
        assert np.abs(want["grads"][name]).max() > 0, name
    print("end-to-end worst gradient error (of max-norm): %.2e" % worst)
    assert worst <= 3e-2
    ct.update()
    l2 = ct.forward().clone()[0].cpu().numpy()
    print("loss_rcnn %.5f -> %.5f" % (Lv[3], l2[3]))
    assert l2[3] < Lv[3]
