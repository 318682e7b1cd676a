"""GPU tests of the ResNet training steps on a canvas of images of different sizes (CanvasResNetRpnTrainer,
CanvasResNetRcnnTrainer) and of their two batch re-layouts, frcnn_maxpool3x3s2_backward_batch and
frcnn_grad_prepare_stride2_batch.

The reference for every per-image number is the one-image path on that image alone (the one-image entries,
ResNetRpnTrainer, ResNetRcnnTrainer with the same kept rows and masks), and the bar is bit-identity.  Only the weight and
bias gradients, which sum N images in one GEMM / one reduction, are compared within 5e-5 of max-norm against the float64
sum of the per-image gradients; at the headline 600x1000 canvas every convolution's dW / db / dX is checked against
float64 conv gradients of the step's own tensors, with the bounds of test_resnet_train_gpu's 600x1000 check."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import resnet_train_ref as rtr
from resnet_ref import maxpool_cover_all, pool3s2_out, split_rne
from test_canvas_train_gpu import _flat_equal
from test_raw_canvas_train_gpu import HC, VOC, WC, _bits, _float_batch, _photos
from test_resnet_rcnn_train_gpu import _rcnn_case
from test_resnet_train_gpu import _adversarial, _bits_equal, _case, _dev, _rel

pytestmark = pytest.mark.gpu
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


# ------------------------------------------------------------------------------------------------ (1) the batch entries
def _act(hi, lo, x3):
    from frcnn_b200 import ops
    return ops.Act(hi.contiguous().cuda(), lo.contiguous().cuda() if x3 else None)


def _empty_like(a, shape=None):
    from frcnn_b200 import ops
    sh = tuple(shape or a.hi.shape)
    return ops.Act(torch.full(sh, 7, dtype=torch.bfloat16, device="cuda"),
                   None if a.lo is None else torch.full(sh, 7, dtype=torch.bfloat16, device="cuda"))


def _slot(a, n, h=None, w=None):
    """Slot n of an [N, H, W, C] Act, cropped to h x w (a dense copy)."""
    from frcnn_b200 import ops
    crop = lambda t: None if t is None else t[n, :h, :w].contiguous()          # noqa: E731
    return ops.Act(crop(a.hi), crop(a.lo))


def _pooled(y_hi, y_lo, x3):
    """The 3x3/2 cover_all pool of [N, H, W, C] host planes (y_lo read only for bf16x3): the forward kernel's (H, W >= 3),
    else the restatement per image (below the forward's minimum)."""
    from frcnn_b200 import ops
    N, H, W, _ = y_hi.shape
    if H >= 3 and W >= 3:
        return ops.maxpool3x3s2_ceil_batch(_act(y_hi, y_lo, x3))
    his, los = zip(*[split_rne(maxpool_cover_all(rtr.pair_f32(y_hi[n], y_lo[n] if x3 else None)).float()) for n in range(N)])
    return _act(torch.stack(his), torch.stack(los), x3)


def _pool_inputs(N, H, W, C, x3, seed):
    y_hi, y_lo = split_rne(_adversarial((N, H, W, C), seed))
    gen = torch.Generator().manual_seed(seed + 1)
    gv = torch.randn((N, pool3s2_out(H), pool3s2_out(W), C), generator=gen)
    g_hi, g_lo = split_rne(gv)
    return _act(g_hi, g_lo, x3), _act(y_hi, y_lo, x3), _pooled(y_hi, y_lo, x3)


def _check_pool(N, H, W, C, x3, seed):
    from frcnn_b200 import train_ops
    g, y, p = _pool_inputs(N, H, W, C, x3, seed)
    out = _empty_like(y)
    tb = train_ops.TBuf(1, C, H, W, "cuda", x3, N=N)
    train_ops.maxpool3x3s2_backward_batch(N, g, y, p, out=out, tbuf=tb)
    for n in range(N):
        o1 = _empty_like(y, (H, W, C))
        t1 = train_ops.TBuf(1, C, H, W, "cuda", x3)
        train_ops.maxpool3x3s2_backward(_slot(g, n), _slot(y, n), _slot(p, n), out=o1, tbuf=t1)
        torch.cuda.synchronize()
        assert _bits_equal(out.hi[n], o1.hi) and _bits_equal(None if out.lo is None else out.lo[n], o1.lo), (N, H, W, n)
        blk = slice(n * tb.Kp, (n + 1) * tb.Kp)
        assert _bits_equal(tb.hi[:, :, blk], t1.hi), (N, H, W, n)
        if x3:
            assert _bits_equal(tb.lo[:, :, blk], t1.lo), (N, H, W, n)


def _check_stride2(N, H, W, C, x3, planes, seed):
    from frcnn_b200 import train_ops
    gen = torch.Generator().manual_seed(seed)
    g = _act(*split_rne(torch.randn((N, (H + 1) // 2, (W + 1) // 2, C), generator=gen)), x3)
    y = _act(*split_rne(_adversarial((N, H, W, C), seed + 2)), x3)
    out = _empty_like(y)
    tb = train_ops.TBuf(planes, C, H, W, "cuda", x3, N=N)
    train_ops.grad_prepare_stride2_batch(N, H, W, C, g, y=y, out=out, tbuf=tb)
    for n in range(N):
        o1 = _empty_like(y, (H, W, C))
        t1 = train_ops.TBuf(planes, C, H, W, "cuda", x3)
        train_ops.grad_prepare_stride2(H, W, C, _slot(g, n), y=_slot(y, n), out=o1, tbuf=t1)
        torch.cuda.synchronize()
        assert _bits_equal(out.hi[n], o1.hi) and _bits_equal(None if out.lo is None else out.lo[n], o1.lo), (N, H, W, n)
        blk = slice(n * tb.Kp, (n + 1) * tb.Kp)
        assert _bits_equal(tb.hi[:, :, blk], t1.hi) and (not x3 or _bits_equal(tb.lo[:, :, blk], t1.lo)), (N, H, W, n)


SIZES = [(H, W) for H in range(2, 10) for W in range(2, 10)] + [(37, 63), (150, 251)]


@pytest.mark.parametrize("x3", [True, False])
@pytest.mark.parametrize("N", [1, 3])
def test_batch_relayouts_equal_per_image(N, x3):
    """Every H, W in 2..9 and two ragged sizes, odd and even: each image of the batch entries equals the one-image entry
    bit for bit (NHWC and transposed planes).  With N = 3 every image after the first reads its g / p at the route's own
    image stride, which differs from the 2x2 pool's ceil(H/2) x ceil(W/2) for every odd H (pool) and for every size
    (stride-2 scatter, which has no p)."""
    for H, W in SIZES:
        C = 64 if H * W > 100 else 16
        _check_pool(N, H, W, C, x3, 100 * H + W)
        _check_stride2(N, H, W, C, x3, 1 + 2 * ((H + W) % 2), 7 * H + W)


def _canvas_slots(N, Hc, Wc, C, ext, seed):
    """y [N, Hc, Wc, C] post-ReLU-like values with ties at 0, zero outside each slot's extent, and zero stripes along the
    image's last two rows and columns in slot 1, so that the border windows there have maximum 0."""
    gen = torch.Generator().manual_seed(seed)
    vals = torch.tensor([0.0, 0.0, 0.5, 1.25, 1.25, 3.0, 0.75, 2.5], dtype=torch.float32)
    y = vals[torch.randint(0, len(vals), (N, Hc, Wc, C), generator=gen)]
    for n, (h, w) in enumerate(ext):
        y[n, h:] = 0
        y[n, :, w:] = 0
        if n == 1:
            y[n, max(h - 2, 0):h] = 0
            y[n, :, max(w - 2, 0):w] = 0
    return y


@pytest.mark.parametrize("x3", [True, False])
def test_batch_relayouts_on_a_canvas(x3):
    """Images zero outside odd and even extents in 37 x 63 slots, the pooled map from the _ext forward pool and the incoming
    gradient zero outside the pooled (subsampled) extent, as the canvas step leaves them: inside each image the batch
    entries equal the one-image entry on the cropped image, bit for bit, and they write 0 outside it."""
    from frcnn_b200 import ops, train_ops
    Hc, Wc, C = 37, 63, 64
    ext = [(37, 63), (24, 41), (19, 30), (2, 2), (36, 7)]
    N = len(ext)
    ext_d = _dev(np.array(ext, np.int32))
    y = _act(*split_rne(_canvas_slots(N, Hc, Wc, C, ext, 3)), x3)
    p = ops.maxpool3x3s2_ceil_batch(y, extents=ext_d)
    gen = torch.Generator().manual_seed(4)
    ph, pw = pool3s2_out(Hc), pool3s2_out(Wc)
    gv = torch.randn((N, ph, pw, C), generator=gen)
    sv = torch.randn((N, (Hc + 1) // 2, (Wc + 1) // 2, C), generator=gen)
    for n, (h, w) in enumerate(ext):
        gv[n, pool3s2_out(h):] = 0
        gv[n, :, pool3s2_out(w):] = 0
        sv[n, (h + 1) // 2:] = 0
        sv[n, :, (w + 1) // 2:] = 0
    g, s = _act(*split_rne(gv), x3), _act(*split_rne(sv), x3)
    out_p, out_s = _empty_like(y), _empty_like(y)
    train_ops.maxpool3x3s2_backward_batch(N, g, y, p, out=out_p)
    train_ops.grad_prepare_stride2_batch(N, Hc, Wc, C, s, y=y, out=out_s)
    torch.cuda.synchronize()
    hit = 0
    for n, (h, w) in enumerate(ext):
        o1 = _empty_like(y, (h, w, C))
        q, r = pool3s2_out(h), pool3s2_out(w)
        train_ops.maxpool3x3s2_backward(_slot(g, n, q, r), _slot(y, n, h, w), _slot(p, n, q, r), out=o1)
        o2 = _empty_like(y, (h, w, C))
        train_ops.grad_prepare_stride2(h, w, C, _slot(s, n, (h + 1) // 2, (w + 1) // 2), y=_slot(y, n, h, w), out=o2)
        torch.cuda.synchronize()
        for got, want in ((out_p, o1), (out_s, o2)):
            for a, b in ((got.hi, want.hi), (got.lo, want.lo)):
                if a is None:
                    continue
                assert _bits_equal(a[n, :h, :w], b), (n, h, w)
                rest = a[n].clone()
                rest[:h, :w] = 0
                assert not bool(rest.view(torch.int16).any()), (n, h, w)
        hit += int(torch.count_nonzero(o1.hi))
    assert hit > 0


# ------------------------------------------------------------------------------------------------ the trainers
def _gt_for(rng, h, w, G):
    """G boxes covering large parts of an h x w image (so that RPN proposals overlap them), in (x1, y1, x2, y2, label)."""
    x1, y1 = rng.uniform(0, 0.3 * w, G), rng.uniform(0, 0.3 * h, G)
    x2, y2 = x1 + rng.uniform(0.4 * w, 0.7 * w, G), y1 + rng.uniform(0.4 * h, 0.7 * h, G)
    g = np.stack([x1, y1, np.minimum(x2, w - 1), np.minimum(y2, h - 1), rng.integers(1, 21, G)], 1)
    return np.floor(g).astype(f32)


def _images(sizes, seed):
    rng = np.random.default_rng(seed)
    xs, gts = [], []
    for k, (h, w) in enumerate(sizes):
        xs.append(_dev(orc.make_image(h, w, seed=seed * 10 + k)[0]))
        gts.append(_dev(_gt_for(rng, h, w, 2 + k % 2)))
    return xs, gts


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
def test_full_size_rpn_step_is_resnet_rpn_trainer_bit_for_bit(precision):
    from frcnn_b200.resnet_train import CanvasResNetRpnTrainer, ResNetRpnTrainer
    H, W = 200, 264
    params = _case(50, H, W, 2)[0]
    xs, gts = _images([(H, W)] * 2, 4)
    rt = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50, precision=precision, seed=9)
    ct = CanvasResNetRpnTrainer(params, 1, H, W, ANCHORS, n_layers=50, precision=precision, seed=9)
    for k in range(2):
        lr_ = rt.forward(xs[k], gts[k])
        rt.backward()
        ct.put([xs[k]], [gts[k]])
        lc = ct.forward().clone()
        ct.backward()
        torch.cuda.synchronize()
        assert _flat_equal(lc[0], lr_), k
        assert torch.equal(ct.targets.labels_full[0], rt.targets.labels_full), k
        assert _flat_equal(ct.g_flat, rt.g_flat), k
        rt.update()
        ct.update()
        torch.cuda.synchronize()
        assert _flat_equal(ct.w_flat, rt.w_flat) and _flat_equal(ct.v_flat, rt.v_flat), k
    f1, f2 = ct.folded_params(), rt.folded_params()
    assert all(np.array_equal(f1[n][0].view(np.int32), f2[n][0].view(np.int32)) for n in f2)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_full_size_rcnn_step_is_resnet_rcnn_trainer_bit_for_bit(precision):
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, ResNetRcnnTrainer
    H, W, post_n = 296, 392, 120
    params, x, gt, _ = _rcnn_case(50, H, W, 3)
    xd, gd = _dev(x[0]), _dev(gt[0])
    rt = ResNetRcnnTrainer(params, H, W, ANCHORS, n_layers=50, precision=precision, post_n=post_n)
    ct = CanvasResNetRcnnTrainer(params, 1, H, W, ANCHORS, n_layers=50, precision=precision, post_n=post_n, sample="list",
                                 dropout="explicit")
    for k in range(2):
        keep, masks = _keep_and_masks(rt, xd, gd, post_n, 10 + k)
        lr_ = rt.forward(xd, gd, keep_inds=keep, masks=masks)
        rt.backward()
        ct.put([xd], [gd], keep_inds=[keep], masks=[masks])
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


# conv1, pool1, res3, res4 all odd for 197 x 229 (99 x 115, 49 x 57, 25 x 29, 13 x 15); even ones for 166 x 131
HC_MIX, WC_MIX = 224, 288
MIX = [(197, 229), (166, 131), (224, 288)]            # plus one empty slot


def _compare_debug(dbg, rd, n, keys):
    for key, d in rd.items():
        if not keys(key):
            continue
        for f, v in d.items():
            c = dbg[key][f][n]
            _, hh, ww = v.shape
            assert _flat_equal(c[:, :hh, :ww].contiguous(), v), (key, f, n)        # inside the image: bit for bit
            out = c.clone()
            out[:, :hh, :ww] = 0
            assert bool((out == 0).all()), (key, f, n)                              # outside: 0


# The mixed-size RPN step updates with this learning rate: at the default 0.001 the summed gradient of three images of this
# random-init trunk can overshoot, which says nothing about the canvas (the gradient itself is checked against the
# per-image sum first).
RPN_MIX_LR = 1e-5


def _update_and_loss(ct, losses, check_loss=True):
    """Two updates on the device gradient follow WeightDecay + MomentumSGD; with check_loss, the summed loss goes down."""
    lr, mom, wd = f32(ct.lr), f32(0.9), f32(0.0005)
    for it in range(2):
        if it:
            ct.forward()
            ct.backward()
        w0 = {k: ct.weights(k).cpu().numpy().copy() for k in ct.index}
        v0 = {k: ct.view(ct.v_flat, k).cpu().numpy().copy() for k in ct.index}
        g0 = {k: ct.grads(k).cpu().numpy().copy() for k in ct.index}
        ct.update()
        for k in ct.index:
            v = (mom * v0[k] - lr * (wd * w0[k] + g0[k]).astype(f32)).astype(f32)
            np.testing.assert_allclose(ct.weights(k).cpu().numpy(), (w0[k] + v).astype(f32), rtol=3e-7, atol=1e-10)
    after = ct.forward().clone()
    print("summed loss %.5f -> %.5f" % (float(losses[:, 3].sum()), float(after[:, 3].sum())))
    if check_loss:
        assert float(after[:, 3].sum()) < float(losses[:, 3].sum())


def test_mixed_sizes_rpn_equal_per_image_trainers():
    from frcnn_b200.resnet_train import CanvasResNetRpnTrainer, ResNetRpnTrainer
    params = _case(50, HC_MIX, WC_MIX, 5)[0]
    xs, gts = _images(MIX, 6)
    ct = CanvasResNetRpnTrainer(params, 4, HC_MIX, WC_MIX, ANCHORS, n_layers=50, subsample="none", lr=RPN_MIX_LR)
    ct.put(xs, gts)
    losses = ct.forward().clone()
    dbg = {}
    ct.backward(debug=dbg)
    torch.cuda.synchronize()
    assert losses[3].cpu().numpy().tolist() == [0.0] * 4                       # the empty slot
    gsum = {k: np.zeros(ct.index[k][2], np.float64) for k in ct.index}
    for n, (h, w) in enumerate(MIX):
        rt = ResNetRpnTrainer(params, h, w, ANCHORS, n_layers=50, subsample="none")
        lo = rt.forward(xs[n], gts[n])
        rd = {}
        rt.backward(debug=rd)
        torch.cuda.synchronize()
        assert _flat_equal(losses[n], lo), n
        assert [tuple(v) for v in ct.level_ext[:, n].cpu().numpy()] == [rt.c1_hw, tuple(rt.p1.hi.shape[:2])] + [
            (B["H"], B["W"]) for B in rt.blocks if B["stride"] == 2], n
        _compare_debug(dbg, rd, n, lambda key: True)
        for k in ct.index:
            gsum[k] += rt.grads(k).cpu().numpy()
        del rt
    worst = max(_rel(ct.grads(k).cpu().numpy(), gsum[k]) for k in ct.index)
    print("summed-gradient worst error (of max-norm): %.2e" % worst)
    assert worst <= 5e-5
    _update_and_loss(ct, losses)


def test_mixed_sizes_rcnn_equal_per_image_trainers():
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, ResNetRcnnTrainer
    post_n = 100
    params = _rcnn_case(50, HC_MIX, WC_MIX, 5)[0]
    xs, gts = _images(MIX, 7)
    refs, keeps, masks = [], [], []
    for n, (h, w) in enumerate(MIX):
        rt = ResNetRcnnTrainer(params, h, w, ANCHORS, n_layers=50, post_n=post_n)
        k, m = _keep_and_masks(rt, xs[n], gts[n], post_n, 20 + n)
        refs.append(rt)
        keeps.append(k)
        masks.append(m)
    ct = CanvasResNetRcnnTrainer(params, 4, HC_MIX, WC_MIX, ANCHORS, n_layers=50, post_n=post_n, sample="list",
                                 dropout="explicit")
    ct.put(xs, gts, keep_inds=keeps, masks=masks)
    losses = ct.forward().clone()
    dbg = {}
    ct.backward(debug=dbg)
    torch.cuda.synchronize()
    assert losses[3].cpu().numpy().tolist() == [0.0] * 4                       # the empty slot
    gsum = {k: np.zeros(ct.index[k][2], np.float64) for k in ct.index}
    dfeat = ct.dfeat.view(4, ct.fh, ct.fw, 2048)
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
            assert _bits_equal(a.hi[n, 0, :R], b.hi[0, :R]) and _bits_equal(a.lo[n, 0, :R], b.lo[0, :R]), n
        rows = slice(n * post_n, (n + 1) * post_n)
        assert _flat_equal(ct.head_grad[rows].contiguous(), rt.head_grad), n
        fh, fw = rt.fh, rt.fw
        assert _flat_equal(dfeat[n, :fh, :fw].contiguous(), rt.dfeat.view(fh, fw, 2048)), n
        rest = dfeat[n].clone()
        rest[:fh, :fw] = 0
        assert bool((rest == 0).all()), n
        _compare_debug(dbg, rd, n, lambda key: key.startswith("trunk/"))
        for k in ct.index:
            gsum[k] += rt.grads(k).cpu().numpy()
    del refs
    worst = max(_rel(ct.grads(k).cpu().numpy(), gsum[k]) for k in ct.index)
    print("summed-gradient worst error (of max-norm): %.2e" % worst)
    assert worst <= 5e-5
    # the loss after an update is not compared: the forward recomputes the proposals from the updated trunk, so the same
    # kept indices name other RoIs, and the loss jumps whatever the step (on an H100 it rose at lr 1e-3, 1e-5 and 1e-7)
    _update_and_loss(ct, losses, check_loss=False)


def test_graph_replay_equals_eager_run():
    """Three mixes through step() (eager, captured, replayed) against put() + run() every time, for both trainers; with
    device subsampling, slot n of step t gets the labels ResNetRpnTrainer-style anchor targets draw with seed + t*N + n."""
    from frcnn_b200 import train_ops
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer
    N, seed = 3, 21
    mixes = [_images([(224, 288), (197, 229), (166, 131)], 7), _images([(200, 200), (224, 100)], 8),
             _images([(100, 288), (224, 288), (61, 77)], 9)]
    params = _rcnn_case(50, HC_MIX, WC_MIX, 5)[0]
    graph = CanvasResNetRpnTrainer(params, N, HC_MIX, WC_MIX, ANCHORS, n_layers=50, seed=seed)
    eager = CanvasResNetRpnTrainer(params, N, HC_MIX, WC_MIX, ANCHORS, n_layers=50, seed=seed)
    anchors = _dev(ANCHORS.astype(np.float64))
    for t, (xs, gts) in enumerate(mixes):
        lg = graph.step(xs, gts)
        eager.put(xs, gts)
        eager.run()
        le = eager.targets.losses.clone()
        torch.cuda.synchronize()
        assert graph.graph is not None and graph.n_updates == eager.n_updates == t + 1
        assert _flat_equal(lg, le), t
        assert _flat_equal(graph.w_flat, eager.w_flat) and _flat_equal(graph.v_flat, eager.v_flat), t
        for n, x in enumerate(xs):
            fh, fw = (int(v) for v in graph.level_ext[4, n].cpu())
            one = train_ops.anchor_targets(anchors, 9, fh, fw, 32, gts[n], x.shape[1], x.shape[2],
                                           mode=train_ops.SUBSAMPLE_DEVICE, seed=seed + t * N + n)
            torch.cuda.synchronize()
            assert torch.equal(graph.targets.labels_full[n, :9 * fh * fw], one.labels_full), (t, n)
            assert torch.equal(graph.targets.counts[n], one.counts), (t, n)
        if len(xs) < N:
            assert graph.targets.counts[N - 1].cpu().numpy().tolist() == [0] * 8
    del graph, eager
    kw = dict(n_layers=50, post_n=100, sample="device", dropout="device", seed=31)
    a = CanvasResNetRcnnTrainer(params, N, HC_MIX, WC_MIX, ANCHORS, **kw)
    b = CanvasResNetRcnnTrainer(params, N, HC_MIX, WC_MIX, ANCHORS, **kw)
    for t, (xs, gts) in enumerate(mixes):
        la = a.step(xs, gts)
        b.put(xs, gts)
        b.run()
        torch.cuda.synchronize()
        assert _flat_equal(la, b.ptargets.losses), t
        assert torch.equal(a.masks, b.masks) and torch.equal(a.ptargets.keep, b.ptargets.keep), t
        assert _flat_equal(a.w_flat, b.w_flat) and _flat_equal(a.v_flat, b.v_flat), t
    assert a.graph is not None and a.n_updates == 3


# ------------------------------------------------------------------------------------------------ raw photos
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("N", [1, 2, 4])
def test_fused_conv1_launch_equals_oracle(N, precision):
    """frcnn_preprocess_voc_canvas_im2col at conv1's ksize 7 / stride 2 / pad 3 / K_pad 160 against voc_ref's transform
    put through ImageInput.put + pack_image_im2col_batch, bit for bit."""
    from frcnn_b200 import ops
    from frcnn_b200.engine import ImageInput, RawPhotoInput
    Ho, Wo = (HC - 1) // 2 + 1, (WC - 1) // 2 + 1
    for mix in range(2):
        sizes = [VOC[(mix * 3 + k) % len(VOC)] for k in range(N - (1 if N > 1 and mix else 0))]   # mix 1: an empty slot
        photos, boxes, labels = _photos(sizes, 10 * N + mix)
        raw = RawPhotoInput(N, HC, WC, "cuda", max_gt=8)
        raw.upload(photos, boxes=boxes, labels=labels)
        got = ops.Act(torch.full((N, Ho, Wo, 160), 7.0, dtype=torch.bfloat16, device="cuda"),
                      torch.full((N, Ho, Wo, 160), 7.0, dtype=torch.bfloat16, device="cuda") if precision == "bf16x3" else None)
        ops.preprocess_voc_im2col_canvas(*raw.descriptors, HC, WC, raw.pixel_means, 7, 2, 3, 160, out=got)
        xs, _ = _float_batch(photos, boxes, labels)
        ref_in = ImageInput(N, HC, WC, "cuda", canvas=True)
        ref_in.put(xs)
        want = ops.pack_image_im2col_batch(ref_in.x_in, 7, 2, 3, 160, precision=precision, extents=ref_in.extents)
        torch.cuda.synchronize()
        for g, w in zip(_bits(got), _bits(want)):
            assert torch.equal(g, w), (N, mix)


def _mixes(N):
    """Three steps with a different size mix each; from N = 2 on, the second leaves a slot empty."""
    return [[VOC[(3 * t + k) % len(VOC)] for k in range(N - (1 if N > 1 and t == 1 else 0))] for t in range(3)]


@pytest.mark.parametrize("N", [1, 2, 4])
def test_rpn_raw_step_equals_float_step(N):
    from frcnn_b200.resnet_train import CanvasResNetRpnTrainer
    params = _case(50, HC, WC, 3)[0]
    raw = CanvasResNetRpnTrainer(params, N, HC, WC, ANCHORS, n_layers=50, seed=5, raw_input=True)
    flt = CanvasResNetRpnTrainer(params, N, HC, WC, ANCHORS, n_layers=50, seed=5)
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


@pytest.mark.parametrize("mode", ["device", "list"])
def test_rcnn_raw_step_equals_float_step(mode):
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer
    N, post_n = 2, 300
    params = _rcnn_case(50, HC, WC, 7)[0]
    kw = dict(n_layers=50, post_n=post_n, seed=11, sample=mode, dropout="device" if mode == "device" else "explicit")
    raw = CanvasResNetRcnnTrainer(params, N, HC, WC, ANCHORS, raw_input=True, **kw)
    flt = CanvasResNetRcnnTrainer(params, N, HC, WC, ANCHORS, **kw)
    rng = np.random.default_rng(2)
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
        assert raw.graph is not None and raw.n_updates == t + 1
        assert _flat_equal(lr_, lf), t
        assert _flat_equal(raw.g_flat, flt.g_flat), t
        assert _flat_equal(raw.w_flat, flt.w_flat) and _flat_equal(raw.v_flat, flt.v_flat), t


# ------------------------------------------------------------------------------------------------ (7) the headline shape
def _canvas_layerwise(ct, params, x_canvas, dbg, dev="cuda"):
    """test_resnet_train_gpu._layerwise on the canvas trainer's own [N] tensors: every routed / masked dy exactly the
    restated rule per slot, dW / db (BN-scaled) against float64 conv gradients summed over the slots, dX against the
    float64 data gradient inside each image (the trainer writes 0 outside it).  Returns the worst errors."""
    import torch.nn.grad as tg
    f64 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64, device=dev)        # noqa: E731
    chw = lambda a: ct._chw(a).cpu().numpy()                                              # noqa: E731
    host = lambda t: t.cpu().numpy()                                                      # noqa: E731
    lv = ct.level_ext.cpu().numpy()
    worst = dict(w=0.0, x=0.0)

    def inside(a, level):
        a = np.array(a)
        for n in range(ct.N):
            h, w = lv[level, n]
            a[n, :, h:] = 0
            a[n, :, :, w:] = 0
        return a

    def route(g_in, y, half):
        v = g_in
        if half:
            v = np.zeros_like(y)
            v[:, :, 0::2, 0::2] = g_in
        return np.where(y > 0, v, 0).astype(f32)

    def record(e_w, e_b, e_x):
        worst["w"], worst["x"] = max(worst["w"], e_w, e_b), max(worst["x"], e_x)

    R = ct.rpn_layer
    mid = f64(chw(R["y"]))
    dyh = f64(host(dbg["heads"]["dy"]))[:, :6 * ct.A]
    Wh = f64(np.concatenate([params["RPN/rpn_cls_score/W"], params["RPN/rpn_bbox_pred/W"]], 0))
    got_wh = np.concatenate([host(ct.grads("RPN/rpn_cls_score/W")), host(ct.grads("RPN/rpn_bbox_pred/W"))], 0)
    got_bh = np.concatenate([host(ct.grads("RPN/rpn_cls_score/b")), host(ct.grads("RPN/rpn_bbox_pred/b"))], 0)
    record(_rel(got_wh, host(tg.conv2d_weight(mid, Wh.shape, dyh))), _rel(got_bh, host(dyh.sum((0, 2, 3)))),
           _rel(host(dbg["heads"]["g_out"]), inside(host(tg.conv2d_input(mid.shape, Wh, dyh)), 4)))
    d = dbg[R["name"]]
    assert np.array_equal(host(d["dy"]), route(host(d["g_in"]), chw(R["y"]), False)), R["name"]
    feat, dy, Wr = f64(chw(ct.feat)), f64(host(d["dy"])), f64(params[R["name"] + "/W"])
    record(_rel(host(ct.grads(R["name"] + "/W")), host(tg.conv2d_weight(feat, Wr.shape, dy, padding=1))),
           _rel(host(ct.grads(R["name"] + "/b")), host(dy.sum((0, 2, 3)))),
           _rel(host(d["g_out"]), inside(host(tg.conv2d_input(feat.shape, Wr, dy, padding=1)), 4)))
    half = False
    for B in reversed(ct.blocks):
        base, level = B["name"], B["level"]
        xin = f64(chw(ct.input_of(B)))
        ins = {1: xin, 2: f64(chw(B["y1"])), 3: f64(chw(B["y2"])), 4: xin}
        outs = {1: chw(B["y1"]), 2: chw(B["y2"]), 3: chw(B["out"]), 4: chw(B["out"])}
        dys = {}
        for i in ((3, 4, 2, 1) if B["proj"] else (3, 2, 1)):
            n = "%s/conv%d" % (base, i)
            d, L = dbg[n], ct.conv[n]
            assert np.array_equal(host(d["dy"]), route(host(d["g_in"]), outs[i], half and i in (3, 4))), n
            dys[i] = f64(host(d["dy"]))
            s = host(L["s"])
            pad = 1 if i == 2 else 0
            Wf = f64(host(L["wf"]))
            dw_ref = host(tg.conv2d_weight(ins[i], Wf.shape, dys[i], padding=pad)) * s[:, None, None, None]
            dx_ref = tg.conv2d_input(ins[i].shape, Wf, dys[i], padding=pad)
            if i == 1:
                dx_ref = dx_ref + (tg.conv2d_input(xin.shape, f64(host(ct.conv[base + "/conv4"]["wf"])), dys[4])
                                   if B["proj"] else dys[3])
            record(_rel(host(ct.grads(n + "/W")), dw_ref), 0.0, _rel(host(d["g_out"]), inside(host(dx_ref), level)))
        half = B["stride"] == 2
    d, L = dbg["trunk/conv1"], ct.conv["trunk/conv1"]
    g_p1 = ct._acts[(ct.p1.hi.shape[1], ct.p1.hi.shape[2], 64, 3)]
    for n in range(ct.N):
        want_hi, want_lo = rtr.maxpool3x3s2_backward(g_p1.hi[n], None if g_p1.lo is None else g_p1.lo[n], ct.c1.hi[n],
                                                     None if ct.c1.lo is None else ct.c1.lo[n], ct.p1.hi[n],
                                                     None if ct.p1.lo is None else ct.p1.lo[n])
        dz = ct._acts[(ct.c1_hw[0], ct.c1_hw[1], 64, 0)]
        assert _bits_equal(dz.hi[n], want_hi) and _bits_equal(None if dz.lo is None else dz.lo[n], want_lo), n
    dzd = f64(host(d["dy"]))
    s = host(L["s"])
    dw_ref = host(tg.conv2d_weight(f64(x_canvas), (64, 3, 7, 7), dzd, stride=2, padding=3)) * s[:, None, None, None]
    record(_rel(host(ct.grads("trunk/conv1/W")), dw_ref), _rel(host(ct.grads("trunk/conv1/b")), host(dzd.sum((0, 2, 3))) * s), 0.0)
    print("canvas layer-wise worst: dW/db %.2e, dX %.2e" % (worst["w"], worst["x"]))
    return worst["w"], worst["x"]


def test_headline_size_layerwise_600x1000():
    """ResNet-101 on a 600 x 1000 canvas with a 600 x 800 and a 600 x 901 image: the layer-wise float64 check of
    test_resnet_train_gpu.test_resnet101_step_layerwise_600x1000 on the canvas step, within the same 5e-5."""
    from frcnn_b200.resnet_train import CanvasResNetRpnTrainer
    Hc, Wc = 600, 1000
    params = _case(101, Hc, Wc, 4)[0]
    xs, gts = _images([(600, 800), (600, 901)], 11)
    ct = CanvasResNetRpnTrainer(params, 2, Hc, Wc, ANCHORS, n_layers=101, subsample="none")
    ct.put(xs, gts)
    ct.forward()
    dbg = {}
    ct.backward(debug=dbg)
    torch.cuda.synchronize()
    x = np.zeros((2, 3, Hc, Wc), np.float64)
    for n, t in enumerate(xs):
        x[n, :, :t.shape[1], :t.shape[2]] = t.cpu().numpy()
    worst_w, worst_x = _canvas_layerwise(ct, params, x, dbg)
    assert worst_w <= 5e-5 and worst_x <= 5e-5
