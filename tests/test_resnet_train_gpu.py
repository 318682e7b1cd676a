"""GPU tests of the RPN training step with the ResNet trunk (frcnn_b200/resnet_train.py, frozen BatchNorm).

  (1) kernels, bit for bit against their restatements (tests/resnet_train_ref.py): the 3x3/2 cover_all max-pool backward,
      the stride-2 scatter, the per-channel scaled reduction and the BN fold -- and the trainer's packed planes equal
      ResNetPackedWeights' packing of its exported parameters and the BN constants;
  (2) layer by layer on the device's own tensors (ResNet-50 at a ragged 296x392, ResNet-101 at 600x1000): every routed or
      masked dy equals the restated rule exactly, every conv's dW (BN-scaled), db and dX (dgrad + residual where the
      block sums) lies within 5e-5 of max-norm of float64 conv gradients of the same inputs -- the bar of
      test_train_gpu.test_rpn_train_step_layerwise_and_end_to_end;
  (3) end to end against resnet_train_oracle.resnet_rpn_train_step (float64 autograd, BN unfolded): losses 1e-4, every
      gradient nonzero and within 5e-2 of max-norm per tensor and 2e-2 in L2 over the whole gradient (ReLU sign flips; the
      reason for the bound is in the test), the MomentumSGD + WeightDecay update over two steps, and the loss decreasing;
  (4) precision "bf16" against "bf16x3"; (5) bad calls raise FrcnnError before anything is queued."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import resnet_train_oracle as rto
import resnet_train_ref as rtr
from resnet_ref import maxpool_cover_all, pool3s2_out, split_rne

pytestmark = pytest.mark.gpu
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits_equal(a, b):
    if a is None or b is None:
        return a is None and b is None
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _adversarial(shape, seed):
    """Post-ReLU-like float32 values from a small set (ties in most windows) with NaN of both signs, +-inf and +-0."""
    g = torch.Generator().manual_seed(seed)
    vals = torch.tensor([0.0, -0.0, 0.5, 0.5, 1.25, 1.25, 3.0, float("inf"), float("-inf"), float("nan"), -float("nan"), -2.0,
                         0.75, 2.5, 1.0009765625], dtype=torch.float32)
    return vals[torch.randint(0, len(vals), shape, generator=g)]


# ------------------------------------------------------------------ (1) kernels
def _pool_case(H, W, C, x3, seed):
    from frcnn_b200 import ops, train_ops
    y_hi, y_lo = split_rne(_adversarial((H, W, C), seed))
    neg_nan = torch.rand((H, W, C), generator=torch.Generator().manual_seed(seed)) < 0.05
    y_hi.view(torch.int16)[neg_nan] = -63                          # 0xFFC1: a NaN with its sign bit set
    y_hi, y_lo = y_hi.cuda(), (y_lo.cuda() if x3 else None)
    ph, pw = pool3s2_out(H), pool3s2_out(W)
    y = ops.Act(y_hi, y_lo)
    if H >= 3 and W >= 3:
        p = ops.maxpool3x3s2_ceil(y)                                     # the forward's own pooled map
    else:                                                                # below the forward's minimum: the restated pool
        p_hi, p_lo = split_rne(maxpool_cover_all(rtr.pair_f32(y_hi, y_lo)).float())
        p = ops.Act(p_hi.contiguous(), p_lo.contiguous() if x3 else None)
    gen = torch.Generator().manual_seed(seed + 1)
    gv = torch.randn((ph, pw, C), generator=gen) * torch.tensor([1.0, 1e-3, 3e2])[torch.randint(0, 3, (ph, pw, C), generator=gen)]
    g_hi, g_lo = (t.cuda() for t in split_rne(gv))
    g = ops.Act(g_hi, g_lo if x3 else None)
    out = ops.Act(torch.empty_like(y_hi), torch.empty_like(y_hi) if x3 else None)
    tb = train_ops.TBuf(1, C, H, W, "cuda", x3)
    train_ops.maxpool3x3s2_backward(g, y, p, out=out, tbuf=tb)
    want_hi, want_lo = rtr.maxpool3x3s2_backward(g.hi, g.lo, y.hi, y.lo, p.hi, p.lo)
    assert _bits_equal(out.hi, want_hi) and _bits_equal(out.lo, want_lo), (H, W, x3)
    assert _bits_equal(tb.hi, rtr.transposed(want_hi, 1)), (H, W, x3)
    if x3:
        assert _bits_equal(tb.lo, rtr.transposed(want_lo, 1)), (H, W)
    return int(torch.count_nonzero(rtr.pair_f32(want_hi, want_lo)))


@pytest.mark.parametrize("x3", [True, False])
def test_pool_backward_every_small_size(x3):
    """The 3x3/2 pool backward at every conv1 output size from 2 to 9 (even sizes clip the last window) and ragged
    sizes, on windows full of ties, NaN of both signs, +-inf and +-0: NHWC planes and transposed planes bit for bit."""
    nonzero = 0
    for H in range(2, 10):
        for W in range(2, 10):
            nonzero += _pool_case(H, W, 16, x3, 100 * H + W)
    for H, W in ((37, 63), (150, 251), (300, 500)):
        nonzero += _pool_case(H, W, 64, x3, H + W)
    assert nonzero > 0


@pytest.mark.parametrize("x3", [True, False])
@pytest.mark.parametrize("planes", [1, 3])
@pytest.mark.parametrize("masked", [False, True])
def test_stride2_scatter(x3, planes, masked):
    from frcnn_b200 import ops, train_ops
    for H, W in ((1, 1), (2, 3), (5, 4), (8, 8), (19, 25), (38, 63), (75, 125)):
        C = 64
        gen = torch.Generator().manual_seed(H * 7 + W)
        g_hi, g_lo = (t.cuda() for t in split_rne(torch.randn(((H + 1) // 2, (W + 1) // 2, C), generator=gen)))
        g = ops.Act(g_hi, g_lo if x3 else None)
        y_hi, y_lo = (t.cuda() for t in split_rne(_adversarial((H, W, C), H + 3 * W)))
        y = ops.Act(y_hi, y_lo if x3 else None) if masked else None
        out = ops.Act(torch.empty((H, W, C), dtype=torch.bfloat16, device="cuda"),
                      torch.empty((H, W, C), dtype=torch.bfloat16, device="cuda") if x3 else None)
        tb = train_ops.TBuf(planes, C, H, W, "cuda", x3)
        train_ops.grad_prepare_stride2(H, W, C, g, y=y, out=out, tbuf=tb)
        want_hi, want_lo = rtr.grad_prepare_stride2(g.hi, g.lo, H, W, y.hi if masked else None)
        assert _bits_equal(out.hi, want_hi) and _bits_equal(out.lo, want_lo), (H, W)
        assert _bits_equal(tb.hi, rtr.transposed(want_hi, planes)), (H, W)
        if x3:
            assert _bits_equal(tb.lo, rtr.transposed(want_lo, planes)), (H, W)


@pytest.mark.parametrize("groups,splits,M,N,ld", [(1, 1, 64, 160, 160), (9, 4, 128, 64, 64), (1, 3, 96, 40, 64), (1, 1, 64, 1, 1)])
def test_scaled_reduction(groups, splits, M, N, ld):
    from frcnn_b200 import train_ops
    gen = torch.Generator().manual_seed(M + N)
    Mp = M + 8
    parts = (torch.randn((groups, splits, Mp, ld), generator=gen) * 10 ** torch.randint(-3, 4, (groups, splits, Mp, ld),
                                                                                        generator=gen).float()).float()
    s = torch.rand((Mp,), generator=gen, dtype=torch.float64) * 2 + 0.1
    dw = torch.full((M * N * groups,), float("nan"), dtype=torch.float32, device="cuda")
    train_ops.wgrad_reduce_scaled(parts.cuda(), M, N, s.cuda(), dw)
    acc = torch.zeros((groups, M, N), dtype=torch.float32)
    for k in range(splits):                                          # fp32, ascending split order
        acc = acc + parts[:, k, :M, :N]
    want = (s[:M].view(1, M, 1) * acc.double()).float().permute(1, 2, 0).reshape(-1)
    assert torch.equal(dw.cpu().view(torch.int32), want.view(torch.int32))


def test_fold_equals_fold_batchnorm():
    from frcnn_b200 import train_ops
    from frcnn_b200.resnet_engine import fold_batchnorm
    rng = np.random.default_rng(5)
    for shape in ((64, 3, 7, 7), (256, 64, 1, 1), (128, 128, 3, 3)):
        co = shape[0]
        W = rng.standard_normal(shape).astype(f32)
        gamma, beta = rng.uniform(0.2, 1.5, co).astype(f32), (rng.standard_normal(co) * 0.1).astype(f32)
        mean, var = (rng.standard_normal(co) * 0.1).astype(f32), rng.uniform(0.5, 2.0, co).astype(f32)
        b = (rng.standard_normal(co) * 0.05).astype(f32)
        s = np.asarray(gamma, np.float64) / np.sqrt(np.asarray(var, np.float64) + 2e-5)
        for bias in (b, None):
            Wf, bf = fold_batchnorm(W, gamma, beta, mean, var, bias)
            wf_d, bf_d = torch.empty(shape, dtype=torch.float32, device="cuda"), torch.empty((co,), dtype=torch.float32, device="cuda")
            train_ops.fold_batchnorm(_dev(W), _dev(s), wf_d, b=None if bias is None else _dev(bias), beta=_dev(beta), mean=_dev(mean),
                                     bf=bf_d)
            assert np.array_equal(wf_d.cpu().numpy().view(np.int32), Wf.view(np.int32))
            assert np.array_equal(bf_d.cpu().numpy().view(np.int32), bf.view(np.int32))


# ------------------------------------------------------------------ the trainer
def _case(n_layers, H, W, seed):
    rng = np.random.default_rng(seed)
    params = orc.make_resnet_params(n_layers=n_layers, seed=29)
    for k in ("RPN/rpn_cls_score/W", "RPN/rpn_bbox_pred/W"):        # livelier heads: every gradient path is exercised
        params[k] = (rng.standard_normal(params[k].shape) * 0.05).astype(f32)
    for k in ("RPN/rpn_conv_3x3/b", "RPN/rpn_cls_score/b", "RPN/rpn_bbox_pred/b", "trunk/conv1/b"):
        params[k] = (rng.standard_normal(params[k].shape) * 0.05).astype(f32)
    x = orc.make_image(H, W, seed=seed)
    gt = np.array([[[20, 30, 150, 170, 3], [100, 20, 330, 240, 7], [200, 150, 300, 280, 1]]], f32)
    gt[..., [0, 2]] = np.clip(gt[..., [0, 2]], 0, W - 1)
    gt[..., [1, 3]] = np.clip(gt[..., [1, 3]], 0, H - 1)
    return params, x, gt, np.array([[H, W]], np.int32)


def test_trainer_packs_what_resnet_packed_weights_packs():
    """The trainer's folded planes (at construction and after an update) equal ResNetPackedWeights' (TrunkOnly's) packing
    of export_params() together with the BN constants, bit for bit."""
    from frcnn_b200.resnet_engine import TrunkOnly
    from frcnn_b200.resnet_train import ResNetRpnTrainer
    H, W = 200, 264
    params, x, gt, _ = _case(50, H, W, 2)
    for prec in ("bf16x3", "bf16"):
        tr = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50, precision=prec, subsample="none")
        for step in range(2):
            if step:
                tr.step(_dev(x[0]), _dev(gt[0]))
            merged = dict(tr.export_params())
            merged.update(tr.bn_params)
            ref = TrunkOnly._W(merged, 50, prec, "cuda").convs
            torch.cuda.synchronize()
            for n in tr.conv:
                (hi, lo), b, _ = tr.packed[n]
                rh, rl, rb = ref[n[len("trunk/"):]]
                assert _bits_equal(hi, rh) and _bits_equal(lo, rl), (prec, step, n)
                assert torch.equal(b[:rb.numel()], rb) and not bool(b[rb.numel():].any()), (prec, step, n)


def _route_ref(g_in, y, half):
    """RPN / block masks on (C,H,W) float32 values: g_in (scattered to the even pixels when `half`) where y > 0, else 0."""
    if half:
        v = np.zeros_like(y)
        v[:, 0::2, 0::2] = g_in
    else:
        v = g_in
    return np.where(y > 0, v, 0).astype(f32)


def _layerwise(tr, params, x, dbg, dev="cuda"):
    """Part (2): exact masks / routing and float64 dW / db / dX of every conv.  Returns the worst errors."""
    import torch.nn.grad as tg
    f64 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64, device=dev)        # noqa: E731
    chw = lambda a: a.to_chw_f32().cpu().numpy()                                          # noqa: E731
    host = lambda t: t.cpu().numpy()                                                      # noqa: E731
    worst = dict(w=0.0, x=0.0)

    def record(name, e_w, e_b, e_x):
        print("  %-26s dW %.2e  db %.2e  dX %.2e" % (name, e_w, e_b, e_x))
        worst["w"], worst["x"] = max(worst["w"], e_w, e_b), max(worst["x"], e_x)

    # RPN heads and the RPN 3x3 conv (no BN)
    R = tr.rpn_layer
    mid = f64(chw(R["y"]))[None]
    dyh = f64(host(dbg["heads"]["dy"]))[None][:, :6 * tr.A]
    Wh = f64(np.concatenate([params["RPN/rpn_cls_score/W"], params["RPN/rpn_bbox_pred/W"]], 0))
    got_wh = np.concatenate([host(tr.grads("RPN/rpn_cls_score/W")), host(tr.grads("RPN/rpn_bbox_pred/W"))], 0)
    got_bh = np.concatenate([host(tr.grads("RPN/rpn_cls_score/b")), host(tr.grads("RPN/rpn_bbox_pred/b"))], 0)
    record("RPN heads", _rel(got_wh, host(tg.conv2d_weight(mid, Wh.shape, dyh))), _rel(got_bh, host(dyh.sum((0, 2, 3)))),
           _rel(host(dbg["heads"]["g_out"]), host(tg.conv2d_input(mid.shape, Wh, dyh))[0]))
    d = dbg[R["name"]]
    assert np.array_equal(host(d["dy"]), _route_ref(host(d["g_in"]), chw(R["y"]), False)), R["name"]
    feat = f64(chw(tr.feat))[None]
    dy = f64(host(d["dy"]))[None]
    Wr = f64(params[R["name"] + "/W"])
    record(R["name"], _rel(host(tr.grads(R["name"] + "/W")), host(tg.conv2d_weight(feat, Wr.shape, dy, padding=1))),
           _rel(host(tr.grads(R["name"] + "/b")), host(dy.sum((0, 2, 3)))),
           _rel(host(d["g_out"]), host(tg.conv2d_input(feat.shape, Wr, dy, padding=1))[0]))
    # the bottleneck blocks
    half = False
    for B in reversed(tr.blocks):
        base = B["name"]
        xin = f64(chw(tr.input_of(B)))[None]
        ins = {1: xin, 2: f64(chw(B["y1"]))[None], 3: f64(chw(B["y2"]))[None], 4: xin}
        outs = {1: chw(B["y1"]), 2: chw(B["y2"]), 3: chw(B["out"]), 4: chw(B["out"])}
        dys = {}
        for i in ((3, 4, 2, 1) if B["proj"] else (3, 2, 1)):
            n = "%s/conv%d" % (base, i)
            d, L = dbg[n], tr.conv[n]
            want = _route_ref(host(d["g_in"]), outs[i], half and i in (3, 4))
            assert np.array_equal(host(d["dy"]), want), n
            dys[i] = f64(host(d["dy"]))[None]
            s = host(L["s"])
            pad = 1 if i == 2 else 0
            Wf = f64(host(L["wf"]))
            dw_ref = host(tg.conv2d_weight(ins[i], Wf.shape, dys[i], padding=pad)) * s[:, None, None, None]
            dx_ref = tg.conv2d_input(ins[i].shape, Wf, dys[i], padding=pad)
            if i == 1:                                        # the block input's gradient: dgrad + the residual path
                dx_ref = dx_ref + (tg.conv2d_input(xin.shape, f64(host(tr.conv[base + "/conv4"]["wf"])), dys[4])
                                   if B["proj"] else dys[3])
            record(n, _rel(host(tr.grads(n + "/W")), dw_ref), 0.0, _rel(host(d["g_out"]), host(dx_ref)[0]))
        half = B["stride"] == 2
    # pool1 + conv1: the routed dy bit for bit, dW and db (BN-scaled) against float64
    d, L = dbg["trunk/conv1"], tr.conv["trunk/conv1"]
    Ho, Wo = tr.c1_hw
    g_p1 = tr._acts[(tr.p1.hi.shape[0], tr.p1.hi.shape[1], 64, 3)]
    want_hi, want_lo = rtr.maxpool3x3s2_backward(g_p1.hi, g_p1.lo, tr.c1.hi, tr.c1.lo, tr.p1.hi, tr.p1.lo)
    dz = tr._acts[(Ho, Wo, 64, 0)]
    assert _bits_equal(dz.hi, want_hi) and _bits_equal(dz.lo, want_lo), "trunk/conv1 routing"
    assert np.array_equal(host(d["g_in"]), chw(g_p1))
    dzd = f64(host(d["dy"]))[None]
    s = host(L["s"])
    dw_ref = host(tg.conv2d_weight(f64(x), (64, 3, 7, 7), dzd, stride=2, padding=3)) * s[:, None, None, None]
    record("trunk/conv1", _rel(host(tr.grads("trunk/conv1/W")), dw_ref),
           _rel(host(tr.grads("trunk/conv1/b")), host(dzd.sum((0, 2, 3))) * s), 0.0)
    print("layer-wise worst: dW/db %.2e, dX %.2e" % (worst["w"], worst["x"]))
    return worst["w"], worst["x"]


def test_resnet50_step_layerwise_and_end_to_end():
    """ResNet-50 at 296 x 392 (conv1 148x196, pool 74x98, then 37x49, 19x25, 10x13), subsample="none":
    (2) layer-wise on the device's tensors and (3) end to end against resnet_rpn_train_step.

    The end-to-end bound is 5e-2 of max-norm per tensor and 2e-2 for the whole flat gradient in L2, not VGG16's 1e-2 per
    tensor: ReLU sign flips compound over 53 convolutions.  Two float64 oracle runs at this case whose trunk weights
    differ by a relative 2^-17 (less than the bf16x3 rounding of the folded weights alone) already differ by 1.1e-2 of
    max-norm (trunk/conv1/W) and 4.7e-3 in L2; the device also rounds every stored activation to 16 bits."""
    from frcnn_b200.resnet_train import ResNetRpnTrainer
    H, W = 296, 392
    params, x, gt, info = _case(50, H, W, 3)
    tr = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50, precision="bf16x3", subsample="none")
    losses = tr.forward(_dev(x[0]), _dev(gt[0]))
    dbg = {}
    tr.backward(debug=dbg)
    torch.cuda.synchronize()
    worst_w, worst_x = _layerwise(tr, params, x, dbg)
    assert worst_w <= 5e-5 and worst_x <= 5e-5
    del dbg
    # ---- (3) end to end
    n_in = int(tr.targets.counts[0].item())
    inds = tr.targets.inds_inside[:n_in].cpu().numpy().astype(np.int64)
    labels = tr.targets.labels_full.cpu().numpy()[inds]
    targets = tr.targets.targets_full.cpu().numpy()[inds]
    r = orc.anchor_target_layer(tr.fh, tr.fw, gt, info, anchors=ANCHORS, feat_stride=32, choice=lambda a, n: a[:0])
    assert np.array_equal(labels, r["labels_before_subsample"]) and np.array_equal(inds, r["inds_inside"])
    want = rto.resnet_rpn_train_step(params, x, labels, targets, inds, n_layers=50)
    Lv = losses.cpu().numpy()
    print("losses", Lv, "oracle", want["losses"])
    assert abs(Lv[0] - want["losses"][0]) <= 1e-4 * max(1.0, want["losses"][0])
    assert abs(Lv[1] - want["losses"][1]) <= 1e-4 * max(1e-2, want["losses"][1])
    assert abs(Lv[3] - want["losses"][3]) <= 1e-4 * max(1.0, want["losses"][3])
    assert set(want["grads"]) == set(tr.index)
    worst = 0.0
    for name in tr.index:
        got = tr.grads(name).cpu().numpy()
        assert np.abs(want["grads"][name]).max() > 0 and np.abs(got).max() > 0, name
        worst = max(worst, _rel(got, want["grads"][name]))
    a = np.concatenate([tr.grads(k).cpu().numpy().ravel() for k in tr.index]).astype(np.float64)
    b = np.concatenate([want["grads"][k].ravel() for k in tr.index])
    l2 = float(np.linalg.norm(a - b) / np.linalg.norm(b))
    print("end-to-end worst gradient error (of max-norm): %.2e, flat gradient L2 %.2e" % (worst, l2))
    assert worst <= 5e-2 and l2 <= 2e-2
    # the optimizer on the device's gradient, over two steps (momentum in play on the second)
    lr, mom, wd = f32(0.001), f32(0.9), f32(0.0005)
    p0 = {k: tr.weights(k).cpu().numpy().copy() for k in tr.index}
    v0 = {k: np.zeros_like(p0[k]) for k in tr.index}
    for step in range(2):
        if step:
            tr.forward(_dev(x[0]), _dev(gt[0]))
            tr.backward()
        g = {k: tr.grads(k).cpu().numpy().copy() for k in tr.index}
        tr.update()
        for name in tr.index:
            gi = (wd * p0[name] + g[name]).astype(f32)
            v = (mom * v0[name] - lr * gi).astype(f32)
            np.testing.assert_allclose(tr.weights(name).cpu().numpy(), (p0[name] + v).astype(f32), rtol=3e-7, atol=1e-10)
            np.testing.assert_allclose(tr.view(tr.v_flat, name).cpu().numpy(), v, rtol=2e-6, atol=1e-12)
            p0[name], v0[name] = tr.weights(name).cpu().numpy().copy(), tr.view(tr.v_flat, name).cpu().numpy().copy()
    l3 = tr.forward(_dev(x[0]), _dev(gt[0])).cpu().numpy()
    print("loss after 0/2 updates: %.5f -> %.5f" % (Lv[3], l3[3]))
    assert l3[3] < Lv[3]


def test_resnet101_step_layerwise_600x1000():
    """Part (2) at the benchmarked 600 x 1000 image with ResNet-101 (float64 references on the GPU)."""
    from frcnn_b200.resnet_train import ResNetRpnTrainer
    H, W = 600, 1000
    params, x, gt, _ = _case(101, H, W, 4)
    tr = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=101, precision="bf16x3", subsample="none")
    tr.forward(_dev(x[0]), _dev(gt[0]))
    dbg = {}
    tr.backward(debug=dbg)
    torch.cuda.synchronize()
    worst_w, worst_x = _layerwise(tr, params, x, dbg)
    assert worst_w <= 5e-5 and worst_x <= 5e-5


def test_device_subsampling_step_and_bf16():
    """subsample="device" and "numpy" run a whole step; precision "bf16" gives finite gradients and a loss within 2e-2 of
    the bf16x3 ones.  Bound on the gradients: the whole flat gradient within 0.3 of the bf16x3 one in L2 norm (relative),
    each tensor within 0.5 of its max-norm (measured on an H100: 0.16 and 0.26).  Looser than VGG16's 0.1 per tensor:
    53 convolutions with 8-bit operands move more ReLU signs and pool maxima, and one moved sign shifts a whole tensor's
    gradient."""
    from frcnn_b200.resnet_train import ResNetRpnTrainer
    H, W = 200, 264
    params, x, gt, _ = _case(50, H, W, 7)
    xd, gd = _dev(x[0]), _dev(gt[0])
    res = {}
    for prec in ("bf16x3", "bf16"):
        tr = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50, precision=prec, subsample="none")
        l = tr.forward(xd, gd).cpu().numpy()
        tr.backward()
        assert bool(torch.isfinite(tr.g_flat).all())
        res[prec] = (l, {k: tr.grads(k).cpu().numpy().copy() for k in tr.index})
    assert abs(res["bf16"][0][3] - res["bf16x3"][0][3]) < 2e-2 * max(1.0, res["bf16x3"][0][3])
    errs = {k: _rel(res["bf16"][1][k], res["bf16x3"][1][k]) for k in res["bf16x3"][1]}
    name = max(errs, key=errs.get)
    a = np.concatenate([res["bf16"][1][k].ravel() for k in errs]).astype(np.float64)
    b = np.concatenate([res["bf16x3"][1][k].ravel() for k in errs]).astype(np.float64)
    l2 = float(np.linalg.norm(a - b) / np.linalg.norm(b))
    print("bf16 vs bf16x3: flat gradient L2 %.2e, worst tensor %s %.2e of max-norm" % (l2, name, errs[name]))
    assert l2 < 0.3 and errs[name] < 0.5
    for mode in ("device", "numpy"):
        tr = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50, subsample=mode)
        w0 = tr.w_flat.clone()
        np.random.seed(0)
        l = tr.step(xd, gd).cpu().numpy()
        assert np.isfinite(l).all() and bool(torch.isfinite(tr.w_flat).all()) and not torch.equal(tr.w_flat, w0)


def test_bad_calls_raise_before_queueing():
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.resnet_train import ResNetRpnTrainer
    H, W = 128, 160
    params, x, gt, _ = _case(50, H, W, 1)
    tr = ResNetRpnTrainer(params, H, W, ANCHORS, n_layers=50)
    seed = tr.seed
    for xx, gg in ((_dev(x[0][:, :-1]), _dev(gt[0])), (_dev(x[0]), _dev(gt[0][:, :4])), (_dev(x[0]), _dev(gt[0][:0])),
                   (torch.from_numpy(x[0]), _dev(gt[0])), (_dev(x[0][None]), _dev(gt[0]))):
        with pytest.raises(FrcnnError):
            tr.forward(xx, gg)
    assert tr.seed == seed and tr.last_losses is None
