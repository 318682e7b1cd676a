"""GPU tests of the RPN training step on a canvas of images of different sizes (CanvasRpnTrainer) and of its three
batched entries: frcnn_anchor_targets_batch, frcnn_rpn_loss_batch and frcnn_grad_prepare_batch.

The reference for every per-image number is the one-image path on that image alone (frcnn_anchor_targets,
frcnn_rpn_loss, frcnn_grad_prepare, RpnTrainer), and the bar is bit-identity: the batched kernels are the one-image kernels
with the image as a grid dimension.  Only the weight and bias gradients, which sum N images in one GEMM / one reduction,
are compared within 5e-5 of max-norm against the float64 sum of the per-image gradients."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
from test_train_gpu import _rel, _route_reference, _train_case

pytestmark = pytest.mark.gpu
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _fmap(e, k=4):
    return -(-e // (1 << k))


def _gt_boxes(rng, h, w, G):
    x1, y1 = rng.uniform(0, w * 0.7, G), rng.uniform(0, h * 0.7, G)
    bw, bh = rng.uniform(16, w * 0.6, G), rng.uniform(16, h * 0.6, G)
    g = np.stack([x1, y1, np.minimum(x1 + bw, w - 1), np.minimum(y1 + bh, h - 1), rng.integers(1, 21, G)], 1)
    return np.floor(g).astype(f32)


# ------------------------------------------------------------------------------------------------ anchor targets
# (extent h, w), clip bounds, gt count: ragged pooled sizes, an empty slot, different G_n, one slot at max_gt
SLOTS = [((600, 1000), (600, 1000), 8), ((333, 500), (333, 333), 1), ((0, 0), (0, 0), 0), ((296, 392), (296, 392), 3),
         ((187, 613), (187, 613), 5)]
MAX_GT = 8


def _targets_case(seed=0):
    from frcnn_b200 import train_ops
    rng = np.random.default_rng(seed)
    N = len(SLOTS)
    ext = np.array([s[0] for s in SLOTS], np.int32)
    info = np.array([s[1] for s in SLOTS], np.int32)
    gt = np.zeros((N, MAX_GT, 5), f32)
    gts = []
    for n, ((h, w), _, G) in enumerate(SLOTS):
        g = _gt_boxes(rng, max(h, 32), max(w, 32), G)
        gt[n, :G] = g
        gts.append(g)
    gt[:, :, :4] += np.where(np.arange(MAX_GT)[None, :, None] >= np.array([s[2] for s in SLOTS])[:, None, None], 1e4, 0)
    work = train_ops.AnchorTargetsBatch(N, 9, _fmap(600), _fmap(1000), MAX_GT, "cuda")
    counts = np.array([s[2] for s in SLOTS], np.int32)
    return train_ops, work, _dev(ext), _dev(info), _dev(gt), _dev(counts), gts


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_anchor_targets_batch_equals_per_image(mode):
    tops, work, ext, info, gt, counts, gts = _targets_case()
    anchors = _dev(ANCHORS.astype(np.float64))
    N = len(SLOTS)
    seeds = torch.tensor([11, 2 ** 40 + 3, 5, 77, 123456789], dtype=torch.int64, device="cuda")
    rng = np.random.default_rng(1)
    lists = [rng.integers(-3, 3000, rng.integers(0, 400)).astype(np.int32) for _ in range(N)]
    flat = _dev(np.concatenate(lists))
    offs = _dev(np.concatenate([[0], np.cumsum([len(v) for v in lists])]).astype(np.int32))
    # poison: entries past each slot's anchors must not matter, and the outputs are rewritten
    for t in (work.labels_full, work.inds_inside, work.counts):
        t.fill_(-7)
    work.targets_full.fill_(float("nan"))
    tops.anchor_targets_batch(anchors, 9, 16, ext, info, gt, counts, work, mode=mode, seeds=seeds, disable_pos=flat,
                              disable_offsets=offs)
    torch.cuda.synchronize()
    for n, ((h, w), (ih, iw), G) in enumerate(SLOTS):
        if G == 0 or h == 0:
            assert work.counts[n].cpu().numpy().tolist() == [0] * 8
            continue
        fh, fw = _fmap(h), _fmap(w)
        kw = dict(seed=int(seeds[n].item())) if mode == 1 else dict(disable_pos=_dev(lists[n])) if mode == 2 else {}
        one = tops.anchor_targets(anchors, 9, fh, fw, 16, _dev(gts[n]), ih, iw, mode=mode, **kw)
        torch.cuda.synchronize()
        n_all = 9 * fh * fw
        c = one.counts.cpu().numpy()
        assert np.array_equal(work.counts[n].cpu().numpy(), c), n
        assert torch.equal(work.labels_full[n, :n_all], one.labels_full), n
        assert torch.equal(work.targets_full[n, :n_all].view(torch.int32), one.targets_full.view(torch.int32)), n
        assert torch.equal(work.inds_inside[n, :c[0]], one.inds_inside[:c[0]]), n
        if mode == 1:
            assert c[1] + c[2] <= 256


# ------------------------------------------------------------------------------------------------ RPN loss
def test_rpn_loss_batch_equals_per_image():
    tops, work, ext, info, gt, counts, gts = _targets_case(3)
    anchors = _dev(ANCHORS.astype(np.float64))
    N, (_, fhc, fwc) = work.N, work.shape
    ld = 64
    seeds = torch.arange(N, dtype=torch.int64, device="cuda") + 40
    tops.anchor_targets_batch(anchors, 9, 16, ext, info, gt, counts, work, mode=1, seeds=seeds)
    g = torch.Generator(device="cuda").manual_seed(5)
    head = torch.randn((N * fhc * fwc, ld), device="cuda", generator=g) * 2
    dhead = torch.full_like(head, float("nan"))
    losses = tops.rpn_loss_batch(head, ld, anchors, 9, 16, ext, info, work, delta=3.0, loss_lambda=1.0, dhead=dhead).clone()
    torch.cuda.synchronize()
    covered = torch.zeros((N, fhc, fwc), dtype=torch.bool, device="cuda")
    H4 = head.view(N, fhc, fwc, ld)
    D4 = dhead.view(N, fhc, fwc, ld)
    for n, ((h, w), (ih, iw), G) in enumerate(SLOTS):
        if G == 0 or h == 0:
            assert losses[n].cpu().numpy().tolist() == [0.0] * 4
            continue
        fh, fw = _fmap(h), _fmap(w)
        one = tops.anchor_targets(anchors, 9, fh, fw, 16, _dev(gts[n]), ih, iw, mode=1, seed=40 + n)
        lo, ds, _ = tops.rpn_loss(H4[n, :fh, :fw].reshape(-1, ld).contiguous(), None, anchors, 9, fh, fw, 16, ih, iw, one,
                                  delta=3.0, loss_lambda=1.0, layout="nhwc", ld=ld)
        torch.cuda.synchronize()
        assert torch.equal(losses[n].view(torch.int32), lo.view(torch.int32)), n
        assert torch.equal(D4[n, :fh, :fw].reshape(-1, ld).view(torch.int32), ds.view(torch.int32)), n
        covered[n, :fh, :fw] = True
    rest = D4[~covered]
    assert rest.numel() > 0 and bool((rest == 0).all())             # every other element written, as +-0 (not the poison)


# ------------------------------------------------------------------------------------------------ re-layout
def _rand_act(shape, x3, gen, relu=False):
    from frcnn_b200 import ops
    v = torch.randn(shape, device="cuda", generator=gen)
    if relu:
        v = torch.where(torch.rand(shape, device="cuda", generator=gen) < 0.3, torch.zeros_like(v), v.abs())
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16) if x3 else None
    return ops.Act(hi.contiguous(), lo)


def _slot(a, n):
    from frcnn_b200 import ops
    return None if a is None else ops.Act(a.hi[n], None if a.lo is None else a.lo[n])


@pytest.mark.parametrize("case", ["y", "y_pool", "f32", "plain3", "times2", "y_bf16"])
def test_grad_prepare_batch_equals_per_image(case):
    from frcnn_b200 import ops, train_ops as tops
    N, H, W, C = 3, 13, 37, 64
    x3 = case != "y_bf16"
    gen = torch.Generator(device="cuda").manual_seed(7)
    y = _rand_act((N, H, W, C), x3, gen, relu=True)
    p = ops.maxpool2x2_ceil_batch(y) if case == "y_pool" else None
    gshape = (N, (H + 1) // 2, (W + 1) // 2, C) if p is not None else (N, H, W, C)
    g = _rand_act(gshape, x3, gen)
    g32 = torch.randn((N * H * W, C), device="cuda", generator=gen) if case == "f32" else None
    planes = 3 if case == "plain3" else 1
    kw = dict(g=None if g32 is not None else g, g_f32=g32, y=None if case in ("f32", "plain3") else y, p=p,
              times2=case == "times2")
    out = ops.Act(torch.full((N, H, W, C), 7, dtype=torch.bfloat16, device="cuda"),
                  torch.full((N, H, W, C), 7, dtype=torch.bfloat16, device="cuda") if x3 else None)
    tb = tops.TBuf(planes, C, H, W, "cuda", x3, N=N)
    tops.grad_prepare_batch(N, H, W, C, out=out, tbuf=tb, **kw)
    Kp = tb.Kp
    for n in range(N):
        o1 = ops.Act(torch.empty((H, W, C), dtype=torch.bfloat16, device="cuda"),
                     torch.empty((H, W, C), dtype=torch.bfloat16, device="cuda") if x3 else None)
        t1 = tops.TBuf(planes, C, H, W, "cuda", x3)
        k1 = dict(kw, g=_slot(kw["g"], n), y=_slot(kw["y"], n), p=_slot(p, n),
                  g_f32=None if g32 is None else g32.view(N, H * W, C)[n])
        tops.grad_prepare(H, W, C, out=o1, tbuf=t1, **k1)
        torch.cuda.synchronize()
        assert torch.equal(out.hi[n].view(torch.int16), o1.hi.view(torch.int16)), n
        assert torch.equal(tb.hi[:, :, n * Kp:(n + 1) * Kp].view(torch.int16), t1.hi.view(torch.int16)), n
        if x3:
            assert torch.equal(out.lo[n].view(torch.int16), o1.lo.view(torch.int16)), n
            assert torch.equal(tb.lo[:, :, n * Kp:(n + 1) * Kp].view(torch.int16), t1.lo.view(torch.int16)), n


# ------------------------------------------------------------------------------------------------ the trainer
def _images(sizes, seed):
    rng = np.random.default_rng(seed)
    xs, gts = [], []
    for k, (h, w) in enumerate(sizes):
        xs.append(_dev(orc.make_image(h, w, seed=seed * 10 + k)[0]))
        gts.append(_dev(_gt_boxes(rng, h, w, 2 + k % 3)))
    return xs, gts


def _flat_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_full_size_step_is_rpn_trainer_bit_for_bit(precision):
    from frcnn_b200.train_engine import CanvasRpnTrainer, RpnTrainer
    H, W = 296, 392
    params = _train_case(H, W, 3)[0]
    xs, gts = _images([(H, W)] * 2, 4)
    rt = RpnTrainer(params, H, W, ANCHORS, precision=precision, seed=9)
    ct = CanvasRpnTrainer(params, 1, H, W, ANCHORS, precision=precision, seed=9)
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


MIX = [(296, 392), (250, 300), (161, 377)]          # plus one empty slot


def _canvas_input(ct, xs):
    x = np.zeros((ct.N, 3, ct.H, ct.W), np.float64)
    for n, t in enumerate(xs):
        x[n, :, :t.shape[1], :t.shape[2]] = t.cpu().numpy()
    return x


def _canvas_layerwise_errors(ct, params, x_canvas, dbg, dev="cpu"):
    """The layer-wise float64 check of test_train_gpu._rpn_layerwise_errors on the canvas trainer's own [N] tensors: the
    routed / masked gradient exact per slot, dW / db against float64 conv gradients summed over the slots, dX against the
    float64 data gradient inside each image (the trainer writes 0 outside it)."""
    import torch.nn.grad as tg
    f64 = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(dev)
    host = lambda t: t.cpu().numpy()
    sizes = ct.image_sizes

    def mask(a, k):
        a = a.copy()
        for n, (h, w) in enumerate(sizes):
            a[n, :, _fmap(h, k):] = 0
            a[n, :, :, _fmap(w, k):] = 0
        return a

    worst_w = worst_x = 0.0
    for i, L in enumerate(ct.layers):
        name, d = L["name"], dbg[L["name"]]
        y = host(ct._chw(L["y"]))
        p = host(ct._chw(L["p"])) if L["pool"] else None
        g_in = host(d["g_in"])
        for n in range(ct.N):
            want = _route_reference(g_in[n], y[n], None if p is None else p[n])
            assert np.array_equal(host(d["dy"][n]), want), (name, n)
        dy = f64(host(d["dy"]))
        Wt = f64(params[name + "/W"])
        xin = f64(x_canvas) if i == 0 else f64(host(ct._chw(ct._input_of(L))))
        e_w = _rel(host(ct.grads(name + "/W")), host(tg.conv2d_weight(xin, Wt.shape, dy, padding=1)))
        e_b = _rel(host(ct.grads(name + "/b")), host(dy.sum((0, 2, 3))))
        e_x = 0.0
        if i > 0:
            dx = mask(host(tg.conv2d_input(xin.shape, Wt, dy, padding=1)), L["halvings"])
            e_x = _rel(host(d["g_out"]), dx)
        worst_w, worst_x = max(worst_w, e_w, e_b), max(worst_x, e_x)
    dyh = f64(host(dbg["heads"]["dy"]))[:, :54]
    mid = f64(host(ct._chw(ct.layers[13]["y"])))
    Wh = f64(np.concatenate([params["RPN/rpn_cls_score/W"], params["RPN/rpn_bbox_pred/W"]], 0))
    got_wh = np.concatenate([host(ct.grads("RPN/rpn_cls_score/W")), host(ct.grads("RPN/rpn_bbox_pred/W"))], 0)
    got_bh = np.concatenate([host(ct.grads("RPN/rpn_cls_score/b")), host(ct.grads("RPN/rpn_bbox_pred/b"))], 0)
    e_w = _rel(got_wh, host(tg.conv2d_weight(mid, Wh.shape, dyh)))
    e_b = _rel(got_bh, host(dyh.sum((0, 2, 3))))
    e_x = _rel(host(dbg["heads"]["g_out"]), mask(host(tg.conv2d_input(mid.shape, Wh, dyh)), 4))
    worst_w, worst_x = max(worst_w, e_w, e_b), max(worst_x, e_x)
    print("canvas layer-wise worst: dW/db %.2e, dX %.2e" % (worst_w, worst_x))
    return worst_w, worst_x


def test_mixed_sizes_equal_per_image_trainers():
    from frcnn_b200.train_engine import CanvasRpnTrainer, RpnTrainer
    Hc, Wc = 296, 392
    params = _train_case(Hc, Wc, 3)[0]
    xs, gts = _images(MIX, 6)
    ct = CanvasRpnTrainer(params, 4, Hc, Wc, ANCHORS, subsample="none")
    ct.put(xs, gts)
    losses = ct.forward().clone()
    dbg = {}
    ct.backward(debug=dbg)
    torch.cuda.synchronize()
    assert losses[3].cpu().numpy().tolist() == [0.0] * 4                       # the empty slot
    gsum = {k: np.zeros(ct.index[k][2], np.float64) for k in ct.index}
    for n, (h, w) in enumerate(MIX):
        rt = RpnTrainer(params, h, w, ANCHORS, subsample="none")
        lo = rt.forward(xs[n], gts[n])
        rd = {}
        rt.backward(debug=rd)
        torch.cuda.synchronize()
        assert _flat_equal(losses[n], lo), n
        for key, d in rd.items():
            for f, v in d.items():
                c = dbg[key][f][n]
                _, hh, ww = v.shape
                assert _flat_equal(c[:, :hh, :ww].contiguous(), v), (key, f, n)        # inside the image: bit for bit
                out = c.clone()
                out[:, :hh, :ww] = 0
                assert bool((out == 0).all()), (key, f, n)                              # outside: 0
        for k in ct.index:
            gsum[k] += rt.grads(k).cpu().numpy()
        del rt
    worst = max(_rel(ct.grads(k).cpu().numpy(), gsum[k]) for k in ct.index)
    print("summed-gradient worst error (of max-norm): %.2e" % worst)
    assert worst <= 5e-5
    worst_w, worst_x = _canvas_layerwise_errors(ct, params, _canvas_input(ct, xs), dbg)
    assert worst_w <= 5e-5 and worst_x <= 5e-5
    # two updates: WeightDecay + MomentumSGD on the device gradient, and the summed loss goes down
    lr, mom, wd = f32(0.001), f32(0.9), f32(0.0005)
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
    assert float(after[:, 3].sum()) < float(losses[:, 3].sum())


def test_graph_replay_equals_eager_run():
    from frcnn_b200 import train_ops
    from frcnn_b200.train_engine import CanvasRpnTrainer
    Hc, Wc, N, seed = 296, 392, 3, 21
    params = _train_case(Hc, Wc, 3)[0]
    mixes = [_images([(296, 392), (200, 300), (161, 377)], 7), _images([(250, 250), (296, 100)], 8),
             _images([(100, 392), (296, 392), (33, 47)], 9)]
    graph = CanvasRpnTrainer(params, N, Hc, Wc, ANCHORS, seed=seed)
    eager = CanvasRpnTrainer(params, N, Hc, Wc, ANCHORS, seed=seed)
    captured = None
    for t, (xs, gts) in enumerate(mixes):
        lg = graph.step(xs, gts)
        if t == 0:
            captured = graph.graph
        eager.put(xs, gts)
        eager.run()
        le = eager.targets.losses.clone()
        torch.cuda.synchronize()
        assert graph.graph is captured and graph.n_updates == eager.n_updates == t + 1
        assert _flat_equal(lg, le), t
        assert _flat_equal(graph.w_flat, eager.w_flat) and _flat_equal(graph.v_flat, eager.v_flat), t
        if t == 1:
            # the stream's images 3 and 4 get the labels RpnTrainer(seed=seed) draws for them: seed + 3, seed + 4
            anchors = _dev(ANCHORS.astype(np.float64))
            for n, x in enumerate(xs):
                fh, fw = _fmap(x.shape[1]), _fmap(x.shape[2])
                one = train_ops.anchor_targets(anchors, 9, fh, fw, 16, gts[n], x.shape[1], x.shape[2],
                                               mode=train_ops.SUBSAMPLE_DEVICE, seed=seed + t * N + n)
                torch.cuda.synchronize()
                assert torch.equal(graph.targets.labels_full[n, :9 * fh * fw], one.labels_full), n
                assert torch.equal(graph.targets.counts[n], one.counts), n
            assert graph.targets.counts[2].cpu().numpy().tolist() == [0] * 8


def test_headline_size_layerwise():
    from frcnn_b200.train_engine import CanvasRpnTrainer
    Hc, Wc = 600, 1000
    params = _train_case(Hc, Wc, 3)[0]
    xs, gts = _images([(600, 800), (600, 901)], 11)
    ct = CanvasRpnTrainer(params, 2, Hc, Wc, ANCHORS, subsample="none")
    ct.put(xs, gts)
    ct.forward()
    dbg = {}
    ct.backward(debug=dbg)
    torch.cuda.synchronize()
    worst_w, worst_x = _canvas_layerwise_errors(ct, params, _canvas_input(ct, xs), dbg, dev="cuda")
    assert worst_w <= 5e-5 and worst_x <= 5e-5


def test_list_mode_and_put_errors():
    from frcnn_b200 import FrcnnError
    from frcnn_b200.train_engine import CanvasRpnTrainer
    Hc, Wc = 192, 256                          # room for the smallest anchors inside both images
    params = _train_case(Hc, Wc, 3)[0]
    xs, gts = _images([(192, 256), (128, 160)], 12)
    ct = CanvasRpnTrainer(params, 2, Hc, Wc, ANCHORS, subsample="list", max_gt=4)
    big = _dev(np.zeros((5, 5), f32))
    bad = [
        lambda: ct.put(xs + xs[:1], gts + gts[:1]),                                    # too many images
        lambda: ct.put([_dev(orc.make_image(193, 256)[0])], gts[:1]),                   # does not fit the canvas
        lambda: ct.put(xs, gts[:1]),                                                   # list lengths differ
        lambda: ct.put(xs, [gts[0], big]),                                              # G_n above max_gt
        lambda: ct.put(xs, [gts[0], big[:0]]),                                          # G_n = 0
        lambda: ct.put(xs, gts, img_infos=[(192, 256)]),
        lambda: ct.put(xs, gts, disable_pos=[_dev(np.zeros(1, np.int32))]),
    ]
    ct.put(xs, gts, disable_pos=[_dev(np.arange(5, dtype=np.int32)), _dev(np.zeros(0, np.int32))])
    before = (ct.x_in.clone(), ct.gt.clone(), ct.gt_counts.clone(), ct.input.sizes.clone(), ct.disable_offsets.clone())
    for f in bad:
        with pytest.raises(FrcnnError):
            f()
    after = (ct.x_in, ct.gt, ct.gt_counts, ct.input.sizes, ct.disable_offsets)
    assert all(torch.equal(a, b) for a, b in zip(before, after))                       # nothing was queued
    assert ct.disable_offsets.cpu().numpy().tolist() == [0, 5, 5]
    ct.forward()
    c = ct.targets.counts.cpu().numpy()
    assert c[0, 3] + c[0, 4] - 5 <= c[0, 1] + c[0, 2] < c[0, 3] + c[0, 4]             # slot 0: up to 5 labels disabled
    assert c[1, 1] == c[1, 3] and c[1, 2] == c[1, 4]                                 # slot 1: an empty list
    with pytest.raises(FrcnnError):
        CanvasRpnTrainer(params, 1, Hc, Wc, ANCHORS, subsample="list").put(xs[:1], gts[:1], disable_pos=[xs[0]] * 2)
