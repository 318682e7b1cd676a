"""GPU parity tests of the RPN-training row (SURVEY.md 8f rank 1): frcnn_bbox_overlaps, frcnn_anchor_targets,
frcnn_rpn_loss through the C ABI, against the oracle (itself pinned to the reference's anchor_target_layer.py and compiled
bbox.pyx, tests/test_oracle_cpu.py) and against the committed golden vectors of the reference run.

Bar: labels / indices / counts bit-exact; float64 IoU bit-exact; regression targets: float64 arithmetic with CUDA's log()
instead of NumPy's, cast to float32 -> at most 1 float32 ulp apart (asserted, exact fraction printed); losses 1e-6 relative
(double accumulation on both sides, different summation order), gradients 1e-5 relative."""
import os

import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import golden_inputs as gi

pytestmark = pytest.mark.gpu
f32 = np.float32
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


@pytest.fixture(scope="module")
def tops():
    from frcnn_b200 import train_ops
    return train_ops


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _golden():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "anchor_target_layer.npz"))


def _ulp_diff_f32(a, b):
    ia = np.ascontiguousarray(a, f32).view(np.int32).astype(np.int64)
    ib = np.ascontiguousarray(b, f32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def test_bbox_overlaps_bit_exact(tops):
    g = _golden()
    boxes, _ = gi.box_transform_case(500, 1, 21)
    query, _ = gi.box_transform_case(17, 1, 22)
    got = tops.bbox_overlaps(_dev(boxes.astype(np.float64)), _dev(query.astype(np.float64))).cpu().numpy()
    assert np.array_equal(got, g["overlaps_500x17"])                       # the reference's compiled bbox.pyx output
    rng = np.random.default_rng(0)                                         # integer grid: exact ties, zero overlaps, identical boxes
    b = rng.integers(0, 30, (700, 2)).astype(np.float64)
    b = np.hstack([b, b + rng.integers(0, 25, (700, 2))])
    q = np.vstack([b[:40], b[100:110] + 0.5])
    assert np.array_equal(tops.bbox_overlaps(_dev(b), _dev(q)).cpu().numpy(), orc.bbox_overlaps(b, q))
    assert tops.bbox_overlaps(_dev(np.zeros((0, 4))), _dev(q)).shape == (0, 50)


def _run_targets(tops, name, mode, **kw):
    fh, fw, gt, info, seed = gi.anchor_target_case(name)
    w = tops.anchor_targets(_dev(ANCHORS.astype(np.float64)), 9, fh, fw, 16, _dev(gt[0]), int(info[0, 0]), int(info[0, 1]),
                            mode=mode, **kw)
    torch.cuda.synchronize()
    return w, (fh, fw, gt, info, seed)


@pytest.mark.parametrize("name", list(gi.ANCHOR_TARGET_CASES))
def test_anchor_targets_before_subsampling(tops, name):
    w, (fh, fw, gt, info, seed) = _run_targets(tops, name, tops.SUBSAMPLE_NONE)
    np.random.seed(seed)
    r = orc.anchor_target_layer(fh, fw, gt, info)
    counts = w.counts.cpu().numpy()
    n_in = int(counts[0])
    assert n_in == len(r["inds_inside"]) and int(counts[5]) == r["n_all"] == w.n_all
    inds = w.inds_inside[:n_in].cpu().numpy()
    assert np.array_equal(inds, r["inds_inside"])                                            # ascending np.where order
    lab_full = w.labels_full.cpu().numpy()
    before = r["labels_before_subsample"]
    assert np.array_equal(lab_full[inds], before)                                            # bit-exact labelling rules
    outside = np.ones(w.n_all, bool)
    outside[inds] = False
    assert (lab_full[outside] == -1).all()
    assert int(counts[1]) == int(counts[3]) == int((before == 1).sum())
    assert int(counts[2]) == int(counts[4]) == int((before == 0).sum())
    tg = w.targets_full.cpu().numpy()
    assert (tg[outside] == 0).all()
    ulp = _ulp_diff_f32(tg[inds], r["targets"])
    print("%s: targets exact %.4f%%, max ulp %d" % (name, 100.0 * (ulp == 0).mean(), ulp.max()))
    assert ulp.max() <= 1 and (ulp == 0).mean() > 0.999
    lab_c, tg_c, idx_c, n_all = w.compact()                                                  # the reference's return tuple
    assert n_all == r["n_all"] and np.array_equal(idx_c.cpu().numpy(), r["inds_inside"])
    assert np.array_equal(lab_c.cpu().numpy(), before) and np.array_equal(tg_c.cpu().numpy(), tg[inds])


@pytest.mark.parametrize("name", list(gi.ANCHOR_TARGET_CASES))
def test_anchor_targets_replay_reference_draws(tops, name):
    """Mode 2 with the index sets the reference's own np.random.choice calls returned (recorded in the golden file)
    reproduces the reference's final labels exactly."""
    g = _golden()
    ncall = int(g[name + "_n_choice_calls"])
    chosen = [g[name + "_choice%d_chosen" % i] for i in range(ncall)]
    dis = np.concatenate(chosen).astype(np.int32) if chosen else np.zeros((0,), np.int32)
    w, _ = _run_targets(tops, name, tops.SUBSAMPLE_LIST, disable_pos=_dev(dis) if dis.size else None)
    n_in = int(w.counts[0].item())
    inds = w.inds_inside[:n_in].cpu().numpy()
    assert np.array_equal(inds, g[name + "_inds_inside"])
    lab = w.labels_full.cpu().numpy()[inds]
    assert np.array_equal(lab, g[name + "_labels"])
    c = w.counts.cpu().numpy()
    assert int(c[1]) == int((lab == 1).sum()) and int(c[2]) == int((lab == 0).sum())
    ulp = _ulp_diff_f32(w.targets_full.cpu().numpy()[inds], g[name + "_targets"])
    assert ulp.max() <= 1


@pytest.mark.parametrize("name", ["c1_g8", "c1_g40_manyfg", "c1_g3_outside", "c1_g1", "t10_small"])
def test_anchor_targets_device_subsampling_properties(tops, name):
    """Mode 1 cannot match NumPy's Mersenne stream; it must satisfy what the reference's subsampling guarantees
    (anchor_target_layer.py:148-168) and be a deterministic function of the seed."""
    w0, _ = _run_targets(tops, name, tops.SUBSAMPLE_NONE)
    before = w0.labels_full.cpu().numpy().copy()
    w1, _ = _run_targets(tops, name, tops.SUBSAMPLE_DEVICE, seed=1234)
    a = w1.labels_full.cpu().numpy().copy()
    c = w1.counts.cpu().numpy().copy()
    fg_b, bg_b = int((before == 1).sum()), int((before == 0).sum())
    fg_a, bg_a = int((a == 1).sum()), int((a == 0).sum())
    assert (int(c[1]), int(c[2]), int(c[3]), int(c[4])) == (fg_a, bg_a, fg_b, bg_b)
    assert fg_a == min(fg_b, 128) and bg_a == min(bg_b, 256 - fg_a)
    changed = a != before
    assert (a[changed] == -1).all() and (before[changed] >= 0).all()                        # only disables, never relabels
    w2, _ = _run_targets(tops, name, tops.SUBSAMPLE_DEVICE, seed=1234)
    assert np.array_equal(w2.labels_full.cpu().numpy(), a)                                   # deterministic
    if changed.any():
        w3, _ = _run_targets(tops, name, tops.SUBSAMPLE_DEVICE, seed=99)
        assert not np.array_equal(w3.labels_full.cpu().numpy(), a)                           # seed matters


def test_anchor_targets_many_gt_boxes(tops):
    """n_gt beyond one shared-memory chunk (256) and a ResNet-sized map."""
    rng = np.random.default_rng(11)
    G, fh, fw, ih, iw = 300, 50, 84, 800, 1333
    w_ = rng.uniform(16, 500, G)
    h_ = rng.uniform(16, 400, G)
    x1 = np.floor(rng.uniform(0, iw - w_))
    y1 = np.floor(rng.uniform(0, ih - h_))
    gt = np.stack([x1, y1, np.floor(x1 + w_ - 1), np.floor(y1 + h_ - 1), rng.integers(0, 20, G)], 1).astype(f32)[None]
    info = np.array([[ih, iw]], np.int32)
    w = tops.anchor_targets(_dev(ANCHORS.astype(np.float64)), 9, fh, fw, 16, _dev(gt[0]), ih, iw, mode=tops.SUBSAMPLE_NONE)
    r = orc.anchor_target_layer(fh, fw, gt, info, choice=lambda inds, size: inds[:size])
    n_in = int(w.counts[0].item())
    inds = w.inds_inside[:n_in].cpu().numpy()
    assert np.array_equal(inds, r["inds_inside"])
    assert np.array_equal(w.labels_full.cpu().numpy()[inds], r["labels_before_subsample"])
    assert _ulp_diff_f32(w.targets_full.cpu().numpy()[inds], r["targets"]).max() <= 1


def test_anchor_targets_argument_errors(tops):
    from frcnn_b200._lib import FrcnnError
    with pytest.raises(FrcnnError):
        tops.anchor_targets(_dev(ANCHORS.astype(np.float64)), 9, 14, 14, 16, torch.zeros((0, 5), device="cuda"), 224, 224)
    with pytest.raises(FrcnnError):
        tops.anchor_targets(_dev(ANCHORS.astype(np.float64)), 9, 14, 14, 16, torch.zeros((3, 4), device="cuda"), 224, 224)


@pytest.mark.parametrize("name,layout", [("c1_g8", "nchw"), ("c1_g8", "nhwc"), ("t14_ref_test", "nchw"),
                                         ("c1_g3_outside", "nhwc"), ("t10_small", "nchw")])
def test_rpn_loss_and_gradients(tops, name, layout):
    g = _golden()
    ncall = int(g[name + "_n_choice_calls"])
    chosen = [g[name + "_choice%d_chosen" % i] for i in range(ncall)]
    dis = np.concatenate(chosen).astype(np.int32) if chosen else np.zeros((0,), np.int32)
    w, (fh, fw, gt, info, seed) = _run_targets(tops, name, tops.SUBSAMPLE_LIST, disable_pos=_dev(dis) if dis.size else None)
    labels, targets, inds = g[name + "_labels"], g[name + "_targets"], g[name + "_inds_inside"]
    A, n_all = 9, 9 * fh * fw
    rng = np.random.default_rng(5)
    score = (rng.standard_normal((1, 2 * A, fh, fw)) * 2).astype(f32)
    pred = (rng.standard_normal((1, 4 * A, fh, fw)) * 2.5).astype(f32)
    lam, delta = 1.5, 3.0
    lc, acc, dsc = orc.rpn_loss_cls(score, labels, inds, n_all, A)
    lb, dpr = orc.rpn_loss_bbox(pred, targets, inds, A, delta=delta)
    anchors = _dev(ANCHORS.astype(np.float64))
    if layout == "nchw":
        losses, ds, db = tops.rpn_loss(_dev(score[0]), _dev(pred[0]), anchors, A, fh, fw, 16, int(info[0, 0]), int(info[0, 1]), w,
                                       delta=delta, loss_lambda=lam)
        ds, db = ds.cpu().numpy()[None], db.cpu().numpy()[None]
    else:
        ld = 64
        m = np.zeros((fh * fw, ld), f32)
        m[:, :2 * A] = score[0].reshape(2 * A, -1).T
        m[:, 2 * A:6 * A] = pred[0].reshape(4 * A, -1).T
        losses, dm, _ = tops.rpn_loss(_dev(m), None, anchors, A, fh, fw, 16, int(info[0, 0]), int(info[0, 1]), w,
                                      delta=delta, loss_lambda=lam, layout="nhwc", ld=ld)
        dm = dm.cpu().numpy()
        assert (dm[:, 6 * A:] == 0).all()
        ds = dm[:, :2 * A].T.reshape(1, 2 * A, fh, fw)
        db = dm[:, 2 * A:6 * A].T.reshape(1, 4 * A, fh, fw)
    L = losses.cpu().numpy()
    want_total = float(lc) + lam * float(lb)
    print(name, layout, "losses", L, "oracle", float(lc), float(lb), float(acc), want_total)
    assert abs(L[0] - float(lc)) <= 1e-6 * max(1.0, abs(float(lc)))
    assert abs(L[1] - float(lb)) <= 1e-6 * max(1e-3, abs(float(lb)))
    assert abs(L[2] - float(acc)) <= 1e-6
    assert abs(L[3] - want_total) <= 2e-6 * max(1.0, abs(want_total))
    np.testing.assert_allclose(ds, dsc, rtol=1e-5, atol=1e-10)
    np.testing.assert_allclose(db, dpr * lam, rtol=1e-5, atol=1e-10)
    # the training step's gradient of the summed loss: grad_scale is a plain multiplier
    if layout == "nchw":
        _, ds2, db2 = tops.rpn_loss(_dev(score[0]), _dev(pred[0]), anchors, A, fh, fw, 16, int(info[0, 0]), int(info[0, 1]), w,
                                    delta=delta, loss_lambda=lam, grad_scale=0.5)
        np.testing.assert_allclose(ds2.cpu().numpy()[None], 0.5 * ds, rtol=1e-6, atol=1e-12)
        np.testing.assert_allclose(db2.cpu().numpy()[None], 0.5 * db, rtol=1e-6, atol=1e-12)


# ------------------------------------------------------------------ the drop-in classes (reference call statements)
@pytest.fixture(scope="module")
def dropin_installed():
    from frcnn_b200 import dropin
    dropin.install()


@pytest.mark.parametrize("name", list(gi.ANCHOR_TARGET_CASES))
def test_anchor_target_layer_class_same_numpy_seed_same_labels_as_reference(dropin_installed, name):
    """tests/test_anchor_target_layer.py:62-66 call statement.  In the default 'numpy' mode the drop-in draws from NumPy's
    global RNG exactly like the reference (same pools, same call order), so the SAME np.random.seed gives the reference's
    own labels -- compared with the golden vectors of the reference run, bit for bit."""
    from chainer import Variable
    from models.anchor_target_layer import AnchorTargetLayer
    g = _golden()
    fh, fw, gt, info, seed = gi.anchor_target_case(name)
    layer = AnchorTargetLayer(16, [0.5, 1, 2], [8, 16, 32])
    np.random.seed(seed)
    bbox_labels, bbox_reg_targets, inds_inside, n_all_bbox = layer(fh, fw, Variable(gt), Variable(info))
    assert isinstance(bbox_labels, np.ndarray) and bbox_labels.dtype == np.int32
    assert n_all_bbox == int(g[name + "_n_all"])
    assert np.array_equal(inds_inside, g[name + "_inds_inside"])
    assert np.array_equal(bbox_labels, g[name + "_labels"])
    assert bbox_reg_targets.dtype == np.float32 and _ulp_diff_f32(bbox_reg_targets, g[name + "_targets"]).max() <= 1
    assert len(bbox_labels) == len(inds_inside) == len(bbox_reg_targets)           # test_anchor_target_layer.py:76-77
    # device arrays in -> device arrays out (the reference's test_time GPU leg, :49-58)
    import chainer
    cp = chainer.cuda.cupy
    np.random.seed(seed)
    lab_d, tg_d, inds_d, _ = layer(fh, fw, Variable(cp.asarray(gt)), Variable(info))
    assert isinstance(lab_d, cp.ndarray) and np.array_equal(cp.asnumpy(lab_d), g[name + "_labels"])
    # "device" subsampling mode: same guarantees, no host RNG
    layer.subsample = "device"
    lab2, _, _, _ = layer(fh, fw, Variable(gt), Variable(info))
    assert (lab2 == 1).sum() <= 128 and (lab2 >= 0).sum() <= 256
    assert (lab2 == 1).sum() == (g[name + "_labels"] == 1).sum() and (lab2 == 0).sum() == (g[name + "_labels"] == 0).sum()


def test_bbox_overlaps_module_surface(dropin_installed):
    from models.bbox import bbox_overlaps
    boxes, _ = gi.box_transform_case(500, 1, 21)
    query, _ = gi.box_transform_case(17, 1, 22)
    got = bbox_overlaps(np.ascontiguousarray(boxes, dtype=np.float64), np.ascontiguousarray(query, dtype=np.float64))
    assert isinstance(got, np.ndarray) and np.array_equal(got, _golden()["overlaps_500x17"])


def test_rpn_training_branch_like_reference(dropin_installed):
    """RegionProposalNetwork.__call__ with train=True and gt_boxes (region_proposal_network.py:126-156): returns rpn_loss;
    compared with the oracle's losses on the device's own head outputs, with the reference-faithful NumPy subsampling."""
    from chainer import Variable
    from models.region_proposal_network import RegionProposalNetwork
    name = "c1_g8"
    fh, fw, gt, info, seed = gi.anchor_target_case(name)
    rng = np.random.default_rng(8)
    rpn = RegionProposalNetwork(loss_lambda=1., delta=3)
    for _, p in rpn.namedparams():                      # non-degenerate weights (the default N(0, 0.01) is fine too)
        if p.data.ndim == 4:
            p.data[...] = (rng.standard_normal(p.data.shape) * 0.02).astype(f32)
    rpn._params_changed()
    x = (np.maximum(rng.standard_normal((1, 512, fh, fw)), 0) * 1.0).astype(f32)
    rpn.train = True
    np.random.seed(seed)
    loss = rpn(Variable(x), Variable(info), Variable(gt))
    assert isinstance(loss, Variable) and loss.name == "rpn_loss" and loss.data.shape == ()
    y = rpn.head_out.cpu().numpy()                                          # [H*W, ld] fp32: the device's own logits/deltas
    score = y[:, :18].T.reshape(1, 18, fh, fw)
    pred = y[:, 18:54].T.reshape(1, 36, fh, fw)
    np.random.seed(seed)
    r = orc.anchor_target_layer(fh, fw, gt, info)
    lc, acc, dsc = orc.rpn_loss_cls(score, r["labels"], r["inds_inside"], r["n_all"], 9)
    lb, dpr = orc.rpn_loss_bbox(pred, r["targets"], r["inds_inside"], 9, delta=3.0)
    print("rpn_loss", float(loss.data), "cls", float(rpn.rpn_loss_cls.data), "bbox", float(rpn.rpn_loss_bbox.data),
          "acc", float(rpn.rpn_cls_accuracy.data), "| oracle", float(lc), float(lb), float(acc))
    assert abs(float(rpn.rpn_loss_cls.data) - float(lc)) <= 1e-6 * max(1.0, float(lc))
    assert abs(float(rpn.rpn_loss_bbox.data) - float(lb)) <= 1e-5 * max(1e-3, float(lb))
    assert abs(float(rpn.rpn_cls_accuracy.data) - float(acc)) <= 1e-6
    assert abs(float(loss.data) - (float(lc) + float(lb))) <= 2e-6 * max(1.0, float(lc) + float(lb))
    gmat = rpn.head_grad.cpu().numpy()
    np.testing.assert_allclose(gmat[:, :18].T.reshape(1, 18, fh, fw), dsc, rtol=1e-5, atol=1e-10)
    np.testing.assert_allclose(gmat[:, 18:54].T.reshape(1, 36, fh, fw), dpr, rtol=2e-5, atol=1e-10)
    # the head outputs themselves follow the fp32 oracle convs within the forward path's tolerance
    params = {"RPN/" + k.lstrip("/"): p.data for k, p in rpn.namedparams()}
    h = orc.relu(orc.conv2d(x, params["RPN/rpn_conv_3x3/W"], params["RPN/rpn_conv_3x3/b"], 1))
    want_score = orc.conv2d(h, params["RPN/rpn_cls_score/W"], params["RPN/rpn_cls_score/b"], 0)
    assert np.abs(score - want_score).max() <= 1e-4 * max(1.0, np.abs(want_score).max())


# ------------------------------------------------------------------ split-K NT GEMM (the weight-gradient engine)
def _ref_gemm_parts(A, B, groups, row_stride, S_eff, K):
    """float64 reference of parts[g][s] on the exact operand values (B: [N,K], or [3,N,K] when groups == 9)."""
    kb = K // 64
    per = -(-kb // S_eff)
    out = []
    for g in range(groups):
        off = (g // 3 - 1) * row_stride if groups == 9 else 0
        Bg = B[g % 3] if groups == 9 else B
        Bs = torch.zeros_like(Bg)
        lo, hi = max(0, -off), min(K, K - off)
        if hi > lo:
            Bs[:, lo:hi] = Bg[:, lo + off:hi + off]
        row = []
        for s in range(S_eff):
            k0, k1 = s * per * 64, min(K, (s + 1) * per * 64)
            row.append(A[:, k0:k1] @ Bs[:, k0:k1].T)
        out.append(torch.stack(row))
    return torch.stack(out)


@pytest.mark.parametrize("M,N,K,groups,splits,x3", [
    (64, 64, 64 * 37, 9, 5, True),        # conv1_2-like: half-empty M tile, single-CTA path, ragged last split
    (512, 512, 64 * 40, 9, 3, True),      # wide N (BN = 128), several pixel tiles
    (256, 128, 64 * 16, 1, 1, True),      # plain GEMM, no split
    (128, 64, 64 * 9, 9, 9, False),       # single-pass bf16
    (54, 512, 64 * 12, 1, 4, True),       # RPN heads: M not a multiple of anything
])
def test_gemm_nt_splitk_matches_float64(tops, M, N, K, groups, splits, x3):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    A = torch.randn((M, K), device="cuda", generator=g)
    B = torch.randn(((3, N, K) if groups == 9 else (N, K)), device="cuda", generator=g)
    row_stride = 40
    if x3:
        a_hi, a_lo = tops.split_bf16(A)
        b_hi, b_lo = tops.split_bf16(B)
        Ae, Be = a_hi.double() + a_lo.double(), b_hi.double() + b_lo.double()
    else:
        a_hi, b_hi, a_lo, b_lo = A.to(torch.bfloat16), B.to(torch.bfloat16), None, None
        Ae, Be = a_hi.double(), b_hi.double()
    parts = tops.gemm_nt_splitk(a_hi, a_lo, b_hi, b_lo, groups=groups, row_stride=row_stride, splits=splits)
    S_eff = parts.shape[1]
    assert parts.shape == (groups, S_eff, M, (N + 31) // 32 * 32) and S_eff <= splits
    want = _ref_gemm_parts(Ae, Be, groups, row_stride, S_eff, K)
    got = parts[..., :N].double()
    scale = want.abs().max().item()
    err = (got - want).abs().max().item()
    print("gemm M%d N%d K%d g%d s%d x3=%s: max err %.3g of scale %.3g" % (M, N, K, groups, S_eff, x3, err, scale))
    # bf16x3 drops the lo*lo term (2^-18 relative per product) and accumulates in the tensor core's truncating fp32
    assert err <= 2e-5 * scale
    # exactly representable operands -> exact sums (small integers, K short enough for fp32)
    Ai = torch.randint(-3, 4, (M, K), device="cuda", generator=g).float()
    Bi = torch.randint(-3, 4, tuple(B.shape), device="cuda", generator=g).float()
    pi = tops.gemm_nt_splitk(Ai.to(torch.bfloat16), None, Bi.to(torch.bfloat16), None, groups=groups, row_stride=row_stride,
                             splits=splits)
    assert torch.equal(pi[..., :N].double(), _ref_gemm_parts(Ai.double(), Bi.double(), groups, row_stride, pi.shape[1], K))


# ------------------------------------------------------------------ the whole train_rpn.py step
def _train_case(H, W, seed):
    rng = np.random.default_rng(seed)
    params = orc.make_params(seed=77)
    for k in ("RPN/rpn_cls_score/W", "RPN/rpn_bbox_pred/W"):       # livelier heads than N(0, 0.01): every gradient path is exercised
        params[k] = (rng.standard_normal(params[k].shape) * 0.05).astype(f32)
    for k in params:
        if k.endswith("/b") and (k.startswith("trunk/") or k.startswith("RPN/")):
            params[k] = (rng.standard_normal(params[k].shape) * 0.05).astype(f32)
    x = orc.make_image(H, W, seed=seed)
    fh, fw = -(-H // 16), -(-W // 16)
    gt = np.array([[[20, 30, 150, 170, 3], [100, 20, 330, 240, 7], [200, 150, 300, 280, 1]]], f32)
    gt[..., [0, 2]] = np.clip(gt[..., [0, 2]], 0, W - 1)
    gt[..., [1, 3]] = np.clip(gt[..., [1, 3]], 0, H - 1)
    info = np.array([[H, W]], np.int32)
    return params, x, gt, info


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _route_reference(g_in, y, p):
    """numpy restatement of frcnn_grad_prepare on the device's own tensors: max-pool routing to the first maximum of the
    2x2 ceil-mode window (when p is given) and the ReLU mask.  All (C,H,W) float32."""
    C, H, W = y.shape
    if p is None:
        v = g_in.copy()
    else:
        v = np.zeros_like(y)
        taken = np.zeros(p.shape, bool)
        for e in range(4):                                   # scan order (0,0),(0,1),(1,0),(1,1)
            dh, dw = e >> 1, e & 1
            ys = y[:, dh::2, dw::2]
            hh, ww = ys.shape[1:]
            hit = (ys == p[:, :hh, :ww]) & ~taken[:, :hh, :ww]
            v[:, dh::2, dw::2] = np.where(hit, g_in[:, :hh, :ww], 0)
            taken[:, :hh, :ww] |= hit
    return np.where(y > 0, v, 0).astype(f32)


def test_rpn_train_step_layerwise_and_end_to_end():
    """The whole train_rpn.py step: forward + AnchorTargetLayer + losses + backward (15 convs: weight gradient, data
    gradient, ReLU / max-pool backward) + WeightDecay + MomentumSGD.

    ReLU and max-pool make the end-to-end gradient DISCONTINUOUS in the forward activations: one pre-activation whose
    sign differs between two correct implementations changes every upstream gradient by ~1e-3 of its max-norm (the
    float32 and float64 runs of the oracle itself differ by 4e-4 from conv3_3 down for exactly this reason).  So:
      (1) layer by layer, on the DEVICE's own tensors: the masked/routed gradient is exactly the restated rule, and each
          layer's dW / db / dX match float64 conv gradients of the same inputs within 5e-5 of max-norm (continuous
          functions: bf16x3 precision only);
      (2) end to end against the float64 autograd oracle: losses 1e-4, every gradient within 1e-2 of max-norm (flips),
          and the optimizer update rule over two steps (momentum)."""
    from frcnn_b200.train_engine import RpnTrainer
    import torch.nn.grad as tg
    H, W = 296, 392                        # ragged pooled sizes: 296->148->74->37->19, 392->196->98->49->25
    params, x, gt, info = _train_case(H, W, 3)
    tr = RpnTrainer(params, H, W, ANCHORS, precision="bf16x3", subsample="none")
    losses = tr.forward(_dev(x[0]), _dev(gt[0]))
    dbg = {}
    tr.backward(debug=dbg)
    torch.cuda.synchronize()
    # ---- (1) layer-wise, float64 on the device's own activations / gradients
    f64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    worst_w = worst_x = 0.0
    for i, L in enumerate(tr.layers):
        name = L["name"]
        d = dbg[name]
        y = L["y"].to_chw_f32().cpu().numpy()
        p = L["p"].to_chw_f32().cpu().numpy() if L["pool"] else None
        want_dy = _route_reference(d["g_in"].cpu().numpy(), y, p)
        assert np.array_equal(d["dy"].cpu().numpy(), want_dy), name                       # exact: routing + mask
        dy = f64(d["dy"].cpu().numpy())[None]
        Wt = f64(params[name + "/W"])
        if i == 0:
            xin = f64(x)                                                                  # conv1_1 sees the image itself
        else:
            xin = f64(tr._input_of(L).to_chw_f32().cpu().numpy())[None]
        dw_ref = tg.conv2d_weight(xin, Wt.shape, dy, padding=1).numpy()
        e_w = _rel(tr.grads(name + "/W").cpu().numpy(), dw_ref)
        e_b = _rel(tr.grads(name + "/b").cpu().numpy(), dy.sum((0, 2, 3)).numpy())
        e_x = 0.0
        if i > 0:
            dx_ref = tg.conv2d_input(xin.shape, Wt, dy, padding=1).numpy()[0]
            e_x = _rel(d["g_out"].cpu().numpy(), dx_ref)
        print("  %-22s dW %.2e  db %.2e  dX %.2e" % (name, e_w, e_b, e_x))
        worst_w, worst_x = max(worst_w, e_w, e_b), max(worst_x, e_x)
    # twin heads (1x1): dY is the loss kernel's gradient itself
    dyh = f64(dbg["heads"]["dy"].cpu().numpy())[None][:, :54]
    mid = f64(tr.layers[13]["y"].to_chw_f32().cpu().numpy())[None]
    Wh = f64(np.concatenate([params["RPN/rpn_cls_score/W"], params["RPN/rpn_bbox_pred/W"]], 0))
    dwh = tg.conv2d_weight(mid, Wh.shape, dyh).numpy()
    got_wh = np.concatenate([tr.grads("RPN/rpn_cls_score/W").cpu().numpy(), tr.grads("RPN/rpn_bbox_pred/W").cpu().numpy()], 0)
    got_bh = np.concatenate([tr.grads("RPN/rpn_cls_score/b").cpu().numpy(), tr.grads("RPN/rpn_bbox_pred/b").cpu().numpy()], 0)
    e_w, e_b = _rel(got_wh, dwh), _rel(got_bh, dyh.sum((0, 2, 3)).numpy())
    e_x = _rel(dbg["heads"]["g_out"].cpu().numpy(), tg.conv2d_input(mid.shape, Wh, dyh).numpy()[0])
    print("  %-22s dW %.2e  db %.2e  dX %.2e" % ("RPN heads", e_w, e_b, e_x))
    worst_w, worst_x = max(worst_w, e_w, e_b), max(worst_x, e_x)
    print("layer-wise worst: dW/db %.2e, dX %.2e" % (worst_w, worst_x))
    assert worst_w <= 5e-5 and worst_x <= 5e-5
    # ---- (2) end to end
    n_in = int(tr.targets.counts[0].item())
    inds = tr.targets.inds_inside[:n_in].cpu().numpy().astype(np.int64)
    labels = tr.targets.labels_full.cpu().numpy()[inds]
    targets = tr.targets.targets_full.cpu().numpy()[inds]
    r = orc.anchor_target_layer(tr.fh, tr.fw, gt, info, choice=lambda a, n: a[:0])
    assert np.array_equal(labels, r["labels_before_subsample"]) and np.array_equal(inds, r["inds_inside"])
    want = orc.rpn_train_step(params, x, labels, targets, inds)
    Lv = losses.cpu().numpy()
    print("losses", Lv, "oracle", want["losses"])
    assert abs(Lv[0] - want["losses"][0]) <= 1e-4 * max(1.0, want["losses"][0])
    assert abs(Lv[1] - want["losses"][1]) <= 1e-4 * max(1e-2, want["losses"][1])
    assert abs(Lv[3] - want["losses"][3]) <= 1e-4 * max(1.0, want["losses"][3])
    worst = 0.0
    for name in tr.index:
        e = _rel(tr.grads(name).cpu().numpy(), want["grads"][name])
        worst = max(worst, e)
        assert np.abs(want["grads"][name]).max() > 0, name            # every trainable tensor receives a gradient
    print("end-to-end worst gradient error (of max-norm): %.2e" % worst)
    assert worst <= 1e-2
    # optimizer: the update applied to the DEVICE's gradient is the reference rule, exactly (fp32 ops in the same order)
    g_dev = {k: tr.grads(k).cpu().numpy().copy() for k in tr.index}
    tr.update()
    lr, mom, wd = f32(0.001), f32(0.9), f32(0.0005)
    v1 = {}
    for name in tr.index:
        w0 = params[name].astype(f32)
        gi = (wd * w0 + g_dev[name]).astype(f32)             # fma in the kernel: compare with a 1-ulp allowance below
        v = (mom * f32(0) - lr * gi).astype(f32)
        v1[name] = v
        np.testing.assert_allclose(tr.weights(name).cpu().numpy(), (w0 + v).astype(f32), rtol=3e-7, atol=1e-10)
        np.testing.assert_allclose(tr.view(tr.v_flat, name).cpu().numpy(), v, rtol=2e-6, atol=1e-12)
    # second step: momentum buffer in play
    p1 = {k: tr.weights(k).cpu().numpy().copy() for k in tr.index}
    vd = {k: tr.view(tr.v_flat, k).cpu().numpy().copy() for k in tr.index}
    tr.forward(_dev(x[0]), _dev(gt[0]))
    tr.backward()
    g2 = {k: tr.grads(k).cpu().numpy().copy() for k in tr.index}
    tr.update()
    for name in tr.index:
        gi = (wd * p1[name] + g2[name]).astype(f32)
        v = (mom * vd[name] - lr * gi).astype(f32)
        np.testing.assert_allclose(tr.weights(name).cpu().numpy(), (p1[name] + v).astype(f32), rtol=3e-7, atol=1e-10)
    # and the loss went down on the same image
    l3 = tr.forward(_dev(x[0]), _dev(gt[0])).cpu().numpy()
    print("loss after 0/2 updates: %.5f -> %.5f" % (Lv[3], l3[3]))
    assert l3[3] < Lv[3]


# ------------------------------------------------------------------ RCNN-head training (train_rcnn.py)
def _golden_ptl():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "proposal_target_layer.npz"))


@pytest.mark.parametrize("name", list(gi.PROPOSAL_TARGET_CASES))
def test_proposal_target_layer_device(tops, name):
    """frcnn_roi_overlaps + frcnn_roi_targets against the golden vectors of the reference's ProposalTargetLayer: best
    overlaps / arg-max bit-exact (float64), and -- with the reference run's own kept indices -- its matched gt rows exactly
    and its class-wise float32 targets (CUDA logf vs NumPy's float32 log: <= 2 ulp)."""
    g = _golden_ptl()
    props, gt, seed = gi.proposal_target_case(name)
    rois = _dev(props)
    mo, am = tops.roi_overlaps(rois, None, _dev(gt[0]))
    np.random.seed(seed)
    r = orc.proposal_target_layer(props, gt)
    assert np.array_equal(mo.cpu().numpy(), r["max_overlaps"]) and np.array_equal(am.cpu().numpy(), r["argmax"].astype(np.int32))
    keep = g[name + "_keep_inds"]
    use_gt, ext, labels = tops.roi_targets(rois, _dev(gt[0]), am, _dev(keep), 21)
    assert np.array_equal(use_gt.cpu().numpy(), g[name + "_use_gt_boxes"])
    assert np.array_equal(labels.cpu().numpy(), g[name + "_use_gt_boxes"][:, 4].astype(np.int32))
    want = g[name + "_bbox_reg_targets"]
    got = ext.cpu().numpy()
    assert np.array_equal(got == 0, want == 0)
    ulp = _ulp_diff_f32(got, want)
    print("%s: targets exact %.2f%%, max ulp %d" % (name, 100.0 * (ulp == 0).mean(), ulp.max()))
    assert ulp.max() <= 2


def test_rcnn_loss_and_gradient(tops):
    props, gt, seed = gi.proposal_target_case("few_fg")
    np.random.seed(seed)
    r = orc.proposal_target_layer(props, gt)
    rng = np.random.default_rng(4)
    R, ld = len(props), 128
    head = np.zeros((R, ld), f32)
    head[:, :21] = rng.standard_normal((R, 21)) * 2
    head[:, 21:105] = rng.standard_normal((R, 84)) * 0.8
    lc, lb, acc, tot, dcls, dbb = orc.rcnn_losses(head[:, :21], head[:, 21:105], r["use_gt_boxes"], r["bbox_reg_targets"], r["keep_inds"])
    losses, dh = tops.rcnn_loss(_dev(head), _dev(r["keep_inds"]), _dev(r["use_gt_boxes"][:, 4].astype(np.int32)),
                                _dev(r["bbox_reg_targets"]), 21, 1.0)
    L = losses.cpu().numpy()
    assert abs(L[0] - float(lc)) < 2e-6 * max(1, float(lc)) and abs(L[1] - float(lb)) < 2e-6 * max(1, float(lb))
    assert abs(L[2] - float(acc)) < 1e-6 and abs(L[3] - float(tot)) < 4e-6 * max(1, float(tot))
    d = dh.cpu().numpy()
    np.testing.assert_allclose(d[:, :21], dcls, rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(d[:, 21:105], dbb, rtol=1e-5, atol=1e-9)
    assert not d[:, 105:].any()


def test_roi_pool_backward_matches_autograd_and_is_reproducible(tops):
    import torchvision
    from frcnn_b200 import ops
    rng = np.random.default_rng(6)
    H, W, C, R = 19, 25, 64, 40
    feat = rng.standard_normal((C, H, W)).astype(f32)
    t = torch.from_numpy(np.ascontiguousarray(feat.transpose(1, 2, 0))).cuda()
    hi = t.to(torch.bfloat16)
    fa = ops.Act(hi.contiguous(), (t - hi.float()).to(torch.bfloat16).contiguous())
    fval = (fa.hi.float() + fa.lo.float()).cpu().numpy().transpose(2, 0, 1)
    xy = rng.uniform(-10, 300, (R, 2))
    wh = rng.uniform(5, 250, (R, 2))
    rois = np.hstack([xy, xy + wh]).astype(f32)
    g = rng.standard_normal((R, 49, C)).astype(f32)
    gt_ = torch.from_numpy(g.reshape(1, R, 49 * C)).cuda()
    ghi = gt_.to(torch.bfloat16)
    ga = ops.Act(ghi.contiguous(), (gt_ - ghi.float()).to(torch.bfloat16).contiguous())
    gval = (ga.hi.float() + ga.lo.float()).cpu().numpy().reshape(R, 7, 7, C)
    count = torch.tensor([R - 3], dtype=torch.int32, device="cuda")          # the last 3 rows are beyond the valid count
    d1 = tops.roi_pool_backward(fa, _dev(rois), count, ga).cpu().numpy()
    d2 = tops.roi_pool_backward(fa, _dev(rois), count, ga).cpu().numpy()
    assert np.array_equal(d1, d2)                                             # fixed-point accumulation: bit-reproducible
    x = torch.from_numpy(fval).double()[None].requires_grad_(True)
    br = torch.cat([torch.zeros((R - 3, 1), dtype=torch.float64), torch.from_numpy(rois[:R - 3]).double()], 1)
    y = torchvision.ops.roi_pool(x, br, (7, 7), 1.0 / 16)
    y.backward(torch.from_numpy(gval[:R - 3].transpose(0, 3, 1, 2)).double())
    want = x.grad[0].numpy().transpose(1, 2, 0).reshape(H * W, C)
    assert np.abs(d1 - want).max() <= 1e-6 * np.abs(want).max()


def test_rcnn_train_step_layerwise_and_end_to_end():
    """train_rcnn.py's update on the device (frcnn_b200.train_engine.RcnnTrainer) vs the autograd oracle, with the
    proposals / kept set / dropout masks of the device run fed to the oracle.  As for the RPN step the end-to-end
    gradient is discontinuous in the activations (ReLU, max-pool, RoI-pool arg-max), so the tight bars are local:
    fc weight / data gradients vs float64 products of the device's own tensors (5e-5), exact ReLU+dropout masking,
    RoI-pool backward vs autograd on the device's feature map; end to end: losses 2e-4, gradients 3e-2 of max-norm."""
    from frcnn_b200.train_engine import RcnnTrainer
    H, W = 296, 392
    params, x, gt, info = _train_case(H, W, 5)
    rng = np.random.default_rng(12)
    for k in ("fc6/W", "fc7/W", "cls_score/W", "bbox_pred/W"):
        params[k] = (rng.standard_normal(params[k].shape) * (0.002 if k == "fc6/W" else 0.01)).astype(f32)
    gt[0, :, 4] = [3, 7, 1]
    tr = RcnnTrainer(params, H, W, ANCHORS, post_n=100, sample="numpy")
    np.random.seed(5)
    losses = tr.forward(_dev(x[0]), _dev(gt[0]))
    dbg = {}
    tr.backward(debug=dbg)
    torch.cuda.synchronize()
    R = int(tr.prop.count.item())
    keep = tr.keep.cpu().numpy()
    rois = tr.prop.rois.cpu().numpy()[:R]
    labels, ext = tr.labels.cpu().numpy(), tr.ext.cpu().numpy()
    masks = [m.cpu().numpy()[:R] for m in tr.masks]
    print("R=%d kept=%d fg-labels=%s" % (R, len(keep), np.bincount(labels)[:8]))
    # the kept set is what the reference's ProposalTargetLayer draws from the same proposals under the same seed
    np.random.seed(5)
    ro = orc.proposal_target_layer(rois, gt)
    assert np.array_equal(ro["keep_inds"], keep) and np.array_equal(ro["use_gt_boxes"], tr.use_gt.cpu().numpy())
    assert _ulp_diff_f32(ext, ro["bbox_reg_targets"]).max() <= 2
    # ---- local checks on the device's own tensors (float64 references)
    f64 = lambda a: np.asarray(a, np.float64)
    val = lambda a: (a.hi.float() + a.lo.float()).cpu().numpy()[0]             # [R_cap, C]
    dyh = f64(tr.head_grad.cpu().numpy())                                      # [R_cap, ld]
    fc7, fc6, pool5 = f64(val(tr.fc7)), f64(val(tr.fc6)), f64(val(tr.pool5))
    Wh = f64(np.concatenate([params["cls_score/W"], params["bbox_pred/W"]], 0))
    got_wh = np.concatenate([tr.grads("cls_score/W").cpu().numpy(), tr.grads("bbox_pred/W").cpu().numpy()], 0)
    e = [_rel(got_wh, dyh[:, :105].T @ fc7)]
    e.append(_rel(np.concatenate([tr.grads("cls_score/b").cpu().numpy(), tr.grads("bbox_pred/b").cpu().numpy()]), dyh[:, :105].sum(0)))
    g7 = f64(dbg["fc7"]["g_in"].cpu().numpy().reshape(4096, -1).T)            # (C,1,R_cap) -> [R_cap, C]
    e.append(_rel(g7, dyh[:, :105] @ Wh))
    dy7 = f64(dbg["fc7"]["dy"].cpu().numpy().reshape(4096, -1).T)
    assert np.array_equal(dy7, np.where(fc7 > 0, 2.0 * g7, 0.0))                # ReLU + dropout backward: exact
    e.append(_rel(tr.grads("fc7/W").cpu().numpy(), dy7.T @ fc6))
    e.append(_rel(tr.grads("fc7/b").cpu().numpy(), dy7.sum(0)))
    g6 = f64(dbg["fc6"]["g_in"].cpu().numpy().reshape(4096, -1).T)
    e.append(_rel(g6, dy7 @ f64(params["fc7/W"])))
    dy6 = f64(dbg["fc6"]["dy"].cpu().numpy().reshape(4096, -1).T)
    assert np.array_equal(dy6, np.where(fc6 > 0, 2.0 * g6, 0.0))
    W6_hwc = f64(params["fc6/W"]).reshape(4096, 512, 49).transpose(0, 2, 1).reshape(4096, -1)
    e.append(_rel(tr.grads("fc6/W").cpu().numpy(), dy6.T @ pool5))
    e.append(_rel(tr.grads("fc6/b").cpu().numpy(), dy6.sum(0)))
    dp5 = f64(dbg["roi"]["dpool5"].cpu().numpy().reshape(49 * 512, -1).T)
    e.append(_rel(dp5, dy6 @ W6_hwc))
    print("head local errors (dWh, dbh, dX7, dW7, db7, dX6, dW6, db6, dpool5):", ["%.1e" % v for v in e])
    assert max(e) <= 5e-5
    # RoI-pool backward on the device's feature map
    import torchvision
    feat = tr.feat.to_chw_f32().cpu().numpy()
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
    exported = tr.export_params()
    assert np.array_equal(exported["fc6/W"], params["fc6/W"])                   # (h,w,c) <-> (c,h,w) round trip
    worst = 0.0
    for name in tr.index:
        gdev = tr.grads(name).cpu().numpy()
        if name == "fc6/W":
            gdev = gdev.reshape(4096, 49, 512).transpose(0, 2, 1).reshape(4096, -1)
        e2e = _rel(gdev, want["grads"][name])
        print("  e2e grad %-20s %.2e" % (name, e2e))
        worst = max(worst, e2e)
        assert np.abs(want["grads"][name]).max() > 0, name
    print("end-to-end worst gradient error (of max-norm): %.2e" % worst)
    assert worst <= 3e-2
    # one update, then the loss on the same image / kept set / masks goes down
    tr.update()
    l2 = tr.forward(_dev(x[0]), _dev(gt[0]), keep_inds=tr.keep, masks=tr.masks).cpu().numpy()
    print("loss_rcnn %.5f -> %.5f" % (Lv[3], l2[3]))
    assert l2[3] < Lv[3]


@pytest.mark.parametrize("name", list(gi.PROPOSAL_TARGET_CASES))
def test_proposal_target_layer_class_same_seed_same_result_as_reference(dropin_installed, name):
    """tests/test_proposal_target_layer.py:35-36 call statement; same np.random.seed -> the reference run's kept indices,
    matched gt rows and (<= 2 ulp) class-wise targets, from the golden vectors of the reference itself."""
    from chainer import Variable
    from models.proposal_target_layer import ProposalTargetLayer
    g = _golden_ptl()
    props, gt, seed = gi.proposal_target_case(name)
    layer = ProposalTargetLayer()
    np.random.seed(seed)
    use_gt_boxes, bbox_reg_targets, keep_inds = layer(props, Variable(gt))
    assert isinstance(keep_inds, np.ndarray) and keep_inds.dtype == np.int32
    assert np.array_equal(keep_inds, g[name + "_keep_inds"]) and np.array_equal(use_gt_boxes, g[name + "_use_gt_boxes"])
    assert bbox_reg_targets.shape == (len(keep_inds), 84) and _ulp_diff_f32(bbox_reg_targets, g[name + "_bbox_reg_targets"]).max() <= 2


def test_faster_rcnn_class_rcnn_training_branch(dropin_installed):
    """FasterRCNN.__call__ with rcnn_train = True and gt_boxes (faster_rcnn.py:117-173): returns loss_rcnn; the
    kept trainer completes the step (backward + optimizer update)."""
    from chainer import Variable
    from models.faster_rcnn import FasterRCNN
    from models.vgg16 import VGG16Prev
    np.random.seed(11)
    model = FasterRCNN(trunk_class=VGG16Prev)
    rng = np.random.default_rng(2)
    for path, p in model.namedparams():
        if path == "/trunk/conv1_1/W":
            p.data[...] *= f32(1.0 / 64)
        if path in ("/RPN/rpn_cls_score/W", "/RPN/rpn_bbox_pred/W"):
            p.data[...] = (rng.standard_normal(p.data.shape) * 0.03).astype(f32)
    model._params_changed()
    model.rcnn_train = True
    assert model.rpn_train is False
    H, W = 296, 392
    x = orc.make_image(H, W, seed=5)
    gt = np.array([[[20, 30, 150, 170, 3], [100, 20, 330, 240, 7], [200, 150, 300, 280, 1]]], f32)
    info = np.array([[H, W]], np.int32)
    np.random.seed(3)
    loss = model(Variable(x), Variable(info), Variable(gt))
    assert isinstance(loss, Variable) and loss.data.shape == ()
    tr = model.rcnn_trainer
    assert abs(float(loss.data) - (float(model.loss_cls.data) + float(model.loss_bbox.data))) < 1e-5 * max(1.0, float(loss.data))
    tr.backward()
    w0 = tr.weights("fc7/W").clone()
    g = tr.grads("fc7/W").clone()
    assert float(g.abs().max()) > 0 and bool(torch.isfinite(tr.g_flat).all())
    tr.update()                                      # the optimizer of train_rcnn.py on every trainable tensor
    want = w0 + (-tr.lr * (g + tr.weight_decay * w0))
    torch.testing.assert_close(tr.weights("fc7/W"), want, rtol=1e-6, atol=1e-9)
    print("FasterRCNN rcnn_train: loss_rcnn %.5f (cls %.5f, bbox %.5f, acc %.3f), kept %d of %d proposals" % (
        float(loss.data), float(model.loss_cls.data), float(model.loss_bbox.data), float(model.cls_accuracy.data),
        tr.keep.numel(), int(tr.prop.count.item())))
    # (that a step lowers the loss on a fixed kept set is asserted in test_rcnn_train_step_layerwise_and_end_to_end; here the
    #  proposals themselves move with the trunk, so the two losses are not comparable)
    # ---- the learnt weights flow back into the Link params (ADVICE r01): checkpoint / param_dict / inference see them
    w_fc7_dev = tr.weights("fc7/W").cpu().numpy()
    named = dict(model.namedparams())                         # namedparams() syncs from the trainer first
    assert np.array_equal(named["/fc7/W"].data, w_fc7_dev) and not np.array_equal(w_fc7_dev, w0.cpu().numpy())
    fc6_dev = tr.export_params()["fc6/W"]                     # back in the reference's (c, h, w) column order
    assert np.array_equal(named["/fc6/W"].data, fc6_dev)
    assert model.rcnn_trainer is tr and model._rcnn_trainer_key[1] == model.version_key()     # the trainer is kept, not rebuilt
    # ---- a new image shape: the new trainer starts from the CURRENT weights and inherits the momentum
    v_old = tr.v_flat.clone()
    H2, W2 = 200, 264
    np.random.seed(4)
    gt2 = np.array([[[20, 30, 150, 170, 3], [100, 20, 250, 190, 7]]], f32)
    model(Variable(orc.make_image(H2, W2, seed=6)), Variable(np.array([[H2, W2]], np.int32)), Variable(gt2))
    tr2 = model.rcnn_trainer
    assert tr2 is not tr and torch.equal(tr2.v_flat, v_old)
    assert np.array_equal(tr2.weights("fc7/W").cpu().numpy(), w_fc7_dev)
    # ---- a change made on a SUB-link is seen by the caches further up (version keys cover descendants)
    k0 = model.version_key()
    model.trunk.conv1_1.b.data = model.trunk.conv1_1.b.data + f32(0.5)          # assignment bumps the owning link
    assert model.version_key() != k0
    k1 = model.version_key()
    model.RPN._params_changed()
    assert model.version_key() != k1


def test_single_pass_bf16_mode_of_the_training_and_resnet_paths():
    """The `bf16` fast mode (lo planes absent) through every added kernel family: finite results close to the bf16x3 ones."""
    from frcnn_b200.resnet_engine import ResNetEngine
    from frcnn_b200.train_engine import RcnnTrainer, RpnTrainer
    H, W = 200, 264
    params, x, gt, info = _train_case(H, W, 7)
    gt[0, :, :4] = [[20, 30, 150, 170], [100, 20, 250, 190], [60, 80, 200, 180]]
    xd, gd = _dev(x[0]), _dev(gt[0])
    res = {}
    for prec in ("bf16x3", "bf16"):
        tr = RpnTrainer(params, H, W, ANCHORS, precision=prec, subsample="none")
        l = tr.forward(xd, gd).cpu().numpy()
        tr.backward()
        assert bool(torch.isfinite(tr.g_flat).all())
        res[prec] = (l, tr.grads("trunk/conv3_2/W").cpu().numpy().copy(), tr.grads("RPN/rpn_conv_3x3/b").cpu().numpy().copy())
        tr.update()
    assert abs(res["bf16"][0][3] - res["bf16x3"][0][3]) < 2e-2 * max(1.0, res["bf16x3"][0][3])
    assert _rel(res["bf16"][1], res["bf16x3"][1]) < 0.1 and _rel(res["bf16"][2], res["bf16x3"][2]) < 0.1
    keep = None
    for prec in ("bf16x3", "bf16"):
        rc = RcnnTrainer(params, H, W, ANCHORS, precision=prec, post_n=60, dropout=(prec == "bf16x3"))
        np.random.seed(1)
        l = rc.forward(xd, gd, keep_inds=keep).cpu().numpy()
        rc.backward()
        assert bool(torch.isfinite(rc.g_flat).all()) and np.isfinite(l).all()
        rc.update()
        assert bool(torch.isfinite(rc.w_flat).all())
    rp = orc.make_resnet_params(50, seed=3)
    feats = {}
    for prec in ("bf16x3", "bf16"):
        eng = ResNetEngine(rp, 50, precision=prec, anchors=ANCHORS, use_graph=False, post_n=50)
        p, b, plan = eng(torch.from_numpy(orc.make_image(128, 160, seed=2)[0]).cuda())
        feats[prec] = plan.acts[-1].to_chw_f32().cpu().numpy()
        assert np.isfinite(feats[prec]).all() and p.shape[1] == 21
    assert _rel(feats["bf16"], feats["bf16x3"]) < 5e-2


def test_bbox_transform_and_keep_inside_helpers(dropin_installed, tops):
    """models.bbox_transform.{bbox_transform, keep_inside} (reference :18-38, :112-130) through their kernels."""
    from models import bbox_transform as bt
    ex, _ = gi.box_transform_case(300, 1, 23)
    gt, _ = gi.box_transform_case(300, 1, 24)
    got = bt.bbox_transform(ex, np.hstack([gt, np.ones((300, 1), f32)]))          # gt rows carry a class column
    want = orc.bbox_transform(ex, gt)                                             # float32 in, float32 arithmetic
    assert isinstance(got, np.ndarray) and got.dtype == np.float32 and want.dtype == np.float32
    assert _ulp_diff_f32(got, want).max() <= 2
    allb = orc.all_anchor_boxes(38, 63, 16, ANCHORS)
    idx, rows = bt.keep_inside(allb, (600, 1000))
    widx, wrows = orc.keep_inside(allb, (600, 1000))
    assert np.array_equal(idx, widx) and np.array_equal(rows, wrows)
    flags = tops.keep_inside_flags(_dev(allb), 600, 1000).cpu().numpy()
    assert flags.sum() == len(widx) == 8151


def test_rpn_trainer_numpy_subsampling_reproduces_the_reference_labels():
    """RpnTrainer(subsample="numpy"): with np.random.seed(s) the labels the loss sees are the reference run's
    (oracle under the same seed, itself pinned to the reference's AnchorTargetLayer)."""
    from frcnn_b200.train_engine import RpnTrainer
    H, W = 600, 1000
    fh, fw, gt, info, seed = gi.anchor_target_case("c1_g8")
    params = orc.make_params(seed=77)
    x = orc.make_image(H, W, seed=1)
    tr = RpnTrainer(params, H, W, ANCHORS, subsample="numpy")
    np.random.seed(seed)
    tr.forward(_dev(x[0]), _dev(gt[0]))
    np.random.seed(seed)
    r = orc.anchor_target_layer(fh, fw, gt, info)
    n_in = int(tr.targets.counts[0].item())
    inds = tr.targets.inds_inside[:n_in].cpu().numpy()
    assert np.array_equal(tr.targets.labels_full.cpu().numpy()[inds], r["labels"])
    c = tr.targets.counts.cpu().numpy()
    assert (int(c[1]), int(c[2])) == (int((r["labels"] == 1).sum()), int((r["labels"] == 0).sum()))
