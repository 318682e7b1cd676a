"""GPU parity tests (run on an H100): every CUDA kernel, called through the C ABI, against the
CPU oracle on the same seeded inputs.  Integer / index / box results must be BIT-EXACT; dense
contractions must be within the stated tolerance of the oracle evaluated on identical inputs."""
import os

import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import golden_inputs as gi

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def ops():
    from frcnn_b200 import ops as _ops
    return _ops


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


# ------------------------------------------------------------------------------- NMS (bit-exact)
@pytest.mark.parametrize("name", list(gi.NMS_CASES))
def test_nms_device_vs_oracle_and_reference_golden(ops, golden_dir, name):
    g = np.load(os.path.join(golden_dir, "cpu_nms.npz"))
    dets, thr = gi.nms_case(name)
    want = orc.cpu_nms(dets, thr)
    assert want == g[name + "_keep"].tolist()
    keep, count = ops.nms(dev(dets) if len(dets) else torch.zeros((0, 5), device="cuda"), thr)
    n = int(count.item())
    assert keep[:n].cpu().tolist() == want
    # host-pointer drop-in used by models.cpu_nms.cpu_nms
    assert ops.cpu_nms_host(dets, thr) == want


def test_nms_max_keep_and_modes(ops):
    from frcnn_b200 import _lib
    dets, _ = gi.nms_case("n2000_t07")
    want = orc.cpu_nms(dets, 0.7)
    keep, count = ops.nms(dev(dets), 0.7, max_keep=300)
    assert int(count.item()) == 300 and keep[:300].cpu().tolist() == want[:300]
    # `>` float semantics of the reference's dead gpu_nms (nms_kernel.cu:71): IoU 0.5 == thresh is kept
    pair = np.array([[100, 100, 109, 109, 0.9], [100, 100, 109, 104, 0.8]], f32)
    k, c = ops.nms(dev(pair), 0.5, mode=_lib.NMS_GT_FLOAT)
    assert k[: int(c.item())].cpu().tolist() == [0, 1]
    k, c = ops.nms(dev(pair), 0.5, mode=_lib.NMS_GE_DOUBLE)
    assert k[: int(c.item())].cpu().tolist() == [0]
    # reference FFI `_nms`: pre-sorted host boxes
    order = np.argsort(-dets[:, 4], kind="stable")
    got = ops.gpu_nms_host(dets[order], 0.7)
    # `>` vs `>=` only differ at exact equality, absent from this random case
    assert order[got].tolist() == want


def test_nms_ties_use_the_pinned_rule(ops):
    rng = np.random.default_rng(3)
    dets = gi._clustered_dets(500, 77)
    dets[:, 4] = rng.integers(0, 8, size=500).astype(f32) / 8      # heavy ties
    want = orc.cpu_nms(dets, 0.7)
    keep, count = ops.nms(dev(dets), 0.7)
    assert keep[: int(count.item())].cpu().tolist() == want


# ------------------------------------------------------------------------------- ProposalLayer (bit-exact)
@pytest.mark.parametrize("name", list(gi.PROPOSAL_CASES))
def test_proposals_vs_oracle_and_reference_golden(ops, golden_dir, name):
    g = np.load(os.path.join(golden_dir, "proposal_layer.npz"))
    prob, pred, info, train = gi.proposal_case(name)
    pre, post = (orc.TRAIN_PRE, orc.TRAIN_POST) if train else (orc.TEST_PRE, orc.TEST_POST)
    dbg = {}
    want_rois, want_probs = orc.proposal_layer(prob, pred, info, pre_nms_top_n=pre, post_nms_top_n=post, debug=dbg)
    A, (H, W) = 9, prob.shape[2:]
    anchors = dev(orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32)))
    work = ops.proposals(dev(prob[0]), dev(pred[0]), anchors, A, H, W, 16, info[0, 0], info[0, 1], 16, pre, post,
                         0.7, layout="nchw", debug=True)
    R = int(work.count.item())
    assert R == len(want_rois)
    rois = work.rois.cpu().numpy()
    scores = work.scores.cpu().numpy()
    # bit-exact vs the oracle (same exp specification, same operation order)
    assert np.array_equal(rois[:R], want_rois)
    assert np.array_equal(scores[:R], want_probs.ravel())
    assert not rois[R:].any() and not scores[R:].any()
    ns = int(work.dbg_num.item())
    assert ns == len(dbg["dets"])
    assert np.array_equal(work.dbg_dets.cpu().numpy()[:ns], dbg["dets"])
    assert np.array_equal(work.dbg_idx.cpu().numpy()[:ns], dbg["anchor_index"])
    # and against the REFERENCE's own output: identical scores/order, boxes within 1e-6 of the image scale
    assert np.array_equal(scores[:R].reshape(-1, 1), g[name + "_probs"])
    np.testing.assert_allclose(rois[:R], g[name + "_rois"], rtol=2e-6, atol=1e-3)


def test_proposals_from_logits_nhwc(ops):
    """The fused entry used by the engine: NHWC [H*W, 64] fp32 logits+deltas, 18-way softmax inside."""
    rng = np.random.default_rng(9)
    H, W, A, ld = 19, 25, 9, 64
    logits = (rng.standard_normal((1, 18, H, W)) * 2).astype(f32)
    deltas = (rng.standard_normal((1, 36, H, W)) * 0.4).astype(f32)
    prob = orc.softmax_axis1(logits)
    want_rois, want_probs = orc.proposal_layer(prob, deltas, (300, 400))
    mat = np.zeros((H * W, ld), f32)
    mat[:, :18] = logits[0].reshape(18, -1).T
    mat[:, 18:54] = deltas[0].reshape(36, -1).T
    anchors = dev(orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32)))
    work = ops.proposals(dev(mat), None, anchors, A, H, W, 16, 300, 400, 16, 6000, 300, 0.7, layout="nhwc", ld=ld,
                         cls_is_logits=True)
    R = int(work.count.item())
    assert R == len(want_rois)
    assert np.array_equal(work.rois.cpu().numpy()[:R], want_rois)
    assert np.array_equal(work.scores.cpu().numpy()[:R], want_probs.ravel())


def test_proposals_all_filtered_and_tiny(ops):
    """Edge cases: every box below min_size -> R == 0; a 1x1 map."""
    A = 9
    anchors = dev(orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32)))
    prob = np.full((1, 18, 3, 3), 0.5, f32)
    pred = np.zeros((1, 36, 3, 3), f32)
    pred[0, 2::4] = -8.0
    pred[0, 3::4] = -8.0          # exp(-8): every box collapses below 16 px
    want_rois, _ = orc.proposal_layer(prob, pred, (48, 48))
    work = ops.proposals(dev(prob[0]), dev(pred[0]), anchors, A, 3, 3, 16, 48, 48, 16, 6000, 300, 0.7)
    assert len(want_rois) == 0 and int(work.count.item()) == 0 and not work.rois.any().item()
    rng = np.random.default_rng(1)
    prob = gi._unique_f32(rng, lambda m: rng.uniform(0, 1, size=m), 18).reshape(1, 18, 1, 1)
    pred = (rng.standard_normal((1, 36, 1, 1)) * 0.2).astype(f32)
    want_rois, want_probs = orc.proposal_layer(prob, pred, (200, 200))
    work = ops.proposals(dev(prob[0]), dev(pred[0]), anchors, A, 1, 1, 16, 200, 200, 16, 6000, 300, 0.7)
    R = int(work.count.item())
    assert R == len(want_rois) and np.array_equal(work.rois.cpu().numpy()[:R], want_rois)


# ------------------------------------------------------------------------------- dense: conv / GEMM on wgmma
def _quant16(a):
    """Value representable as bf16 hi + bf16 lo (what a bf16x3 operand holds)."""
    t = torch.from_numpy(np.ascontiguousarray(a, dtype=f32))
    hi = t.to(torch.bfloat16).float()
    lo = (t - hi).to(torch.bfloat16).float()
    return (hi + lo).numpy()


def _bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=f32)).to(torch.bfloat16).float().numpy()


def _conv_case(ops, H, W, Cin, Cout, ksize, precision, seed, relu=True, ld_f32=0, tile=None, check_act=True):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((Cin, H, W)).astype(f32)
    w = (rng.standard_normal((Cout, Cin, ksize, ksize)) * (2.0 / (Cin * ksize * ksize)) ** 0.5).astype(f32)
    b = (rng.standard_normal(Cout) * 0.1).astype(f32)
    q = _quant16 if precision == "bf16x3" else _bf16
    xq, wq = q(x), q(w)
    ref = torch.nn.functional.conv2d(torch.from_numpy(xq)[None].double(), torch.from_numpy(wq).double(),
                                     torch.from_numpy(b).double(), padding=(ksize - 1) // 2)[0]
    if relu:
        ref = ref.clamp_min(0)
    ref = ref.numpy()
    cpad = Cin if Cin % 8 == 0 else (Cin + 7) // 8 * 8
    act = ops.pack_image(dev(x), c_pad=cpad, precision=precision)
    wh, wl = ops.pack_conv_weights(dev(w), cin_pad=cpad, precision=precision)
    bias = ops.pad_bias(dev(b), max(Cout, ld_f32))
    if tile:
        ops.set_conv_tile(*tile)
    try:
        y, y32 = ops.conv2d(act, wh, wl, bias, ksize, relu, out_act=check_act, ld_f32=ld_f32)
        torch.cuda.synchronize()
    finally:
        ops.set_conv_tile(0, 0, 0)
    scale = np.abs(ref).max()
    if y32 is not None:
        got = y32.cpu().numpy().reshape(H, W, ld_f32)
        err = np.abs(got[:, :, :Cout].transpose(2, 0, 1) - ref).max() / scale
        # fp32 output: only the accumulation order (and, for bf16x3, the dropped lo*lo term) differs
        assert err < (3e-5 if precision == "bf16x3" else 1e-5), ("f32", err)
        assert not got[:, :, Cout:].any()
    if y is not None:
        got = y.to_chw_f32().cpu().numpy()
        err = np.abs(got - ref).max() / scale
        # stored activations are rounded to 16 (bf16x3) / 8 (bf16) significant bits
        assert err < (5e-5 if precision == "bf16x3" else 6e-3), ("act", err)
    return ref


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("shape", [
    (24, 40, 64, 64, 3),      # BK=64, BN=64, exact tiles
    (19, 33, 64, 128, 3),     # ragged H/W (TMA zero fill + store predicates)
    (13, 21, 128, 256, 3),    # wide Cout, few pixel tiles: plans BN=64 (BN=256: test_conv_gemm_coverage_gpu.py)
    (38, 63, 512, 512, 3),    # conv5 / RPN 3x3 real shape
    (11, 17, 16, 64, 3),      # BK=16 (SWIZZLE_32B) -- conv1_1 with the image padded to 16 channels
    (10, 12, 64, 96, 1),      # 1x1
])
def test_conv2d_vs_oracle(ops, precision, shape):
    H, W, Cin, Cout, k = shape
    _conv_case(ops, H, W, Cin, Cout, k, precision, seed=H * 1000 + W, ld_f32=(Cout + 31) // 32 * 32)


@pytest.mark.parametrize("tile", [(64, 8, 16), (128, 16, 8), (256, 4, 32), (128, 2, 64), (64, 1, 128), (128, 32, 4)])
def test_conv2d_tile_shapes(ops, tile):
    _conv_case(ops, 37, 45, 64, 256, 3, "bf16", seed=5, tile=tile, ld_f32=256)


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("shape", [(33, 41, 128, 256, 3),     # odd number of pixel tiles: the last pair has a dummy CTA
                                   (16, 8, 64, 128, 3),       # a single pixel tile (pairs not applicable)
                                   (1, 300, 512, 256, 1)])    # GEMM rows, 3 tiles
def test_conv2d_single_cta_and_cta_pair_agree_with_oracle(ops, precision, cta_group, shape):
    """Single CTAs and CTA pairs (a 2-CTA cluster, each CTA loading half of the weight tile and multicasting it to both)
    must both match the oracle."""
    H, W, Cin, Cout, k = shape
    ops.set_conv_cta_group(cta_group)
    try:
        _conv_case(ops, H, W, Cin, Cout, k, precision, seed=77, ld_f32=(Cout + 31) // 32 * 32)
    finally:
        ops.set_conv_cta_group(0)


def test_conv2d_first_layer_from_3_channels(ops):
    """conv1_1: C_in=3 padded to 16 channels (zeros), K-block = one tap x 16 channels."""
    rng = np.random.default_rng(11)
    x = (rng.uniform(0, 255, (3, 45, 70)) - 110).astype(f32)
    w = (rng.standard_normal((64, 3, 3, 3)) * 0.27).astype(f32)
    b = np.zeros(64, f32)
    ref = np.maximum(torch.nn.functional.conv2d(torch.from_numpy(_quant16(x))[None].double(),
                                                torch.from_numpy(_quant16(w)).double(), padding=1)[0].numpy(), 0)
    act = ops.pack_image(dev(x), c_pad=16)
    wh, wl = ops.pack_conv_weights(dev(w), cin_pad=16)
    y, _ = ops.conv2d(act, wh, wl, ops.pad_bias(dev(b), 64), 3, True)
    err = np.abs(y.to_chw_f32().cpu().numpy() - ref).max() / np.abs(ref).max()
    assert err < 5e-5, err


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_conv2d_first_layer_as_im2col_gemm(ops, precision):
    """conv1_1 the way the engine runs it: frcnn_pack_image_im2col3x3 + a K=32 (27 real) 1x1 GEMM with
    SWIZZLE_64B tiles.  Same oracle as the 16-channel-padded 3x3 path."""
    rng = np.random.default_rng(12)
    x = (rng.uniform(0, 255, (3, 45, 70)) - 110).astype(f32)
    w = (rng.standard_normal((64, 3, 3, 3)) * 0.27 / 64).astype(f32)
    b = (rng.standard_normal(64) * 0.1).astype(f32)
    q = _quant16 if precision == "bf16x3" else _bf16
    ref = torch.nn.functional.conv2d(torch.from_numpy(q(x))[None].double(), torch.from_numpy(q(w)).double(),
                                     torch.from_numpy(b).double(), padding=1)[0].clamp_min(0).numpy()
    act = ops.pack_image_im2col(dev(x), precision=precision)
    assert act.hi.shape == (45, 70, 32)
    # the packed image itself: centre tap == the pixel, zero padding at the border, zeros for k >= 27
    v = act.hi.float() + (act.lo.float() if act.lo is not None else 0)
    assert torch.equal(v[:, :, 12:15].permute(2, 0, 1).cpu(), torch.from_numpy(q(x)))
    assert not v[:, :, 27:].any() and not v[0, :, 0:9].any() and not v[:, 0, 0:27:9].any()
    wh, wl = ops.pack_conv_weights_im2col(dev(w), precision=precision)
    y, _ = ops.conv2d(act, wh, wl, ops.pad_bias(dev(b), 64), 1, True)
    err = np.abs(y.to_chw_f32().cpu().numpy() - ref).max() / np.abs(ref).max()
    assert err < (5e-5 if precision == "bf16x3" else 6e-3), err


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("shape", [(37, 45, 64, 64), (600 // 4, 1000 // 4 + 1, 64, 128), (19, 31, 128, 256)])
def test_conv2d_fused_maxpool_equals_conv_then_pool(ops, precision, shape):
    """The fused epilogue (conv + ReLU + 2x2 ceil-mode max-pool, odd H/W included) must give exactly the
    device's own un-fused conv followed by frcnn_maxpool2x2_ceil -- and match the oracle's pooled map."""
    H, W, Cin, Cout = shape
    rng = np.random.default_rng(H + W)
    x = rng.standard_normal((Cin, H, W)).astype(f32)
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * (2.0 / (9 * Cin)) ** 0.5).astype(f32)
    b = (rng.standard_normal(Cout) * 0.1).astype(f32)
    act = ops.pack_image(dev(x), c_pad=Cin, precision=precision)
    wh, wl = ops.pack_conv_weights(dev(w), precision=precision)
    bias = ops.pad_bias(dev(b), Cout)
    y_full, _ = ops.conv2d(act, wh, wl, bias, 3, True)
    want = ops.maxpool2x2_ceil(y_full)
    got, _ = ops.conv2d(act, wh, wl, bias, 3, True, fuse_pool=True)
    assert got.hi.shape == ((H + 1) // 2, (W + 1) // 2, Cout)
    if precision == "bf16x3":
        # the VALUE hi+lo must be identical; the (hi, lo) pair itself may differ at round-to-even ties
        # (the un-fused path re-splits an already 16-bit-rounded value)
        assert torch.equal(got.hi.float() + got.lo.float(), want.hi.float() + want.lo.float())
    else:
        assert torch.equal(got.hi, want.hi)
    q = _quant16 if precision == "bf16x3" else _bf16
    ref = torch.nn.functional.conv2d(torch.from_numpy(q(x))[None].double(), torch.from_numpy(q(w)).double(),
                                     torch.from_numpy(b).double(), padding=1).clamp_min(0)
    ref = torch.nn.functional.max_pool2d(ref, 2, 2, ceil_mode=True)[0].numpy()
    err = np.abs(got.to_chw_f32().cpu().numpy() - ref).max() / np.abs(ref).max()
    assert err < (5e-5 if precision == "bf16x3" else 6e-3), err


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_linear_as_1x1_with_row_count(ops, precision):
    """L.Linear over R RoIs == 1x1 conv with H=1, W=R; rows >= *m_valid come out as zeros."""
    rng = np.random.default_rng(21)
    R, K, N, valid = 300, 1024, 105, 171
    x = rng.standard_normal((R, K)).astype(f32)
    w = (rng.standard_normal((N, K)) * 0.03).astype(f32)
    b = (rng.standard_normal(N) * 0.1).astype(f32)
    q = _quant16 if precision == "bf16x3" else _bf16
    ref = q(x).astype(np.float64) @ q(w).astype(np.float64).T + b
    act = ops.pack_image(dev(x.T.reshape(K, 1, R).copy()), c_pad=K, precision=precision)   # [1,R,K]
    wh, wl = ops.pack_conv_weights(dev(w), precision=precision)
    m_valid = torch.tensor([valid], dtype=torch.int32, device="cuda")
    _, y32 = ops.conv2d(act, wh, wl, ops.pad_bias(dev(b), 128), 1, False, out_act=False, ld_f32=128, m_valid=m_valid)
    got = y32.cpu().numpy()
    err = np.abs(got[:valid, :N] - ref[:valid]).max() / np.abs(ref).max()
    assert err < 3e-5, err
    assert not got[valid:].any() and not got[:, N:].any()


def test_conv2d_real_layer_shapes_bf16x3(ops):
    """Two real VGG16 layers at the headline resolution against torch CPU fp32 on identical
    (16-bit-split) inputs: conv3_2 (150x250x256) and conv4_2 (75x125x512)."""
    for (H, W, C) in [(150, 250, 256), (75, 125, 512)]:
        rng = np.random.default_rng(H)
        x = np.maximum(rng.standard_normal((C, H, W)), 0).astype(f32)
        w = (rng.standard_normal((C, C, 3, 3)) * (2.0 / (9 * C)) ** 0.5).astype(f32)
        ref = torch.nn.functional.conv2d(torch.from_numpy(_quant16(x))[None], torch.from_numpy(_quant16(w)),
                                         padding=1)[0].clamp_min(0).numpy()
        act = ops.pack_image(dev(x), c_pad=C)
        wh, wl = ops.pack_conv_weights(dev(w))
        y, _ = ops.conv2d(act, wh, wl, ops.pad_bias(torch.zeros(C, device="cuda"), C), 3, True)
        err = np.abs(y.to_chw_f32().cpu().numpy() - ref).max() / np.abs(ref).max()
        assert err < 5e-5, (H, W, C, err)


# ------------------------------------------------------------------------------- pooling / head
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_maxpool_ceil(ops, precision):
    rng = np.random.default_rng(4)
    x = rng.standard_normal((64, 37, 63)).astype(f32)
    q = _quant16 if precision == "bf16x3" else _bf16
    want = orc.max_pool_2x2_ceil(q(x)[None])[0]
    got = ops.maxpool2x2_ceil(ops.pack_image(dev(x), c_pad=64, precision=precision)).to_chw_f32().cpu().numpy()
    assert got.shape == (64, 19, 32) and np.array_equal(got, want)


# (C, H, W): 64 = 8 channel groups per CTA, 192 = 24 groups (a slice of 16 + a partial one), 512 = the headline trunk (one CTA of
# 7 x 64 threads per RoI), W = 100 = a map wider than the headline one; "neg" = features that are NOT clipped at zero: the
# kernel takes the maximum on packed (hi, lo) bf16 pairs, which must order negative values and negative lo parts correctly
# (an all-negative window gives its negative maximum, an empty bin 0)
@pytest.mark.parametrize("shape", [(64, 38, 63, "relu"), (192, 21, 33, "neg"), (512, 38, 63, "relu"), (64, 30, 100, "neg")])
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_roi_pool_exact(ops, precision, shape):
    rng = np.random.default_rng(5)
    C, H, W, kind = shape
    R_cap, R = 300, 257
    feat = rng.standard_normal((C, H, W)).astype(f32)
    feat = np.maximum(feat, 0) if kind == "relu" else feat - 1.0
    q = _quant16 if precision == "bf16x3" else _bf16
    xy = rng.uniform(-20, [16 * W - 28, 16 * H - 28], size=(R_cap, 2))
    wh = rng.uniform(1, 500, size=(R_cap, 2))
    rois = np.hstack([xy, xy + wh]).astype(f32)
    rois[:6] = [[0, 0, 999, 599], [8, 8, 8, 8], [24, 40, 24, 40], [990, 590, 999, 599], [0, 0, 15, 15], [-30, -30, 5, 5]]
    want = orc.roi_pool(q(feat)[None], np.hstack([np.zeros((R_cap, 1), f32), rois]))      # (R,C,7,7)
    want[R:] = 0
    act = ops.pack_image(dev(feat), c_pad=C, precision=precision)
    count = torch.tensor([R], dtype=torch.int32, device="cuda")
    out, o32 = ops.roi_pool(act, dev(rois), count, want_f32=True)
    got = o32.cpu().numpy().reshape(R_cap, 7, 7, C).transpose(0, 3, 1, 2)
    assert np.array_equal(got, want)
    v = out.hi.float() + (out.lo.float() if out.lo is not None else 0)
    assert np.array_equal(v.cpu().numpy().reshape(R_cap, 7, 7, C).transpose(0, 3, 1, 2), want)


def test_head_decode_bit_exact(ops):
    rng = np.random.default_rng(6)
    R_cap, R, NC, ld = 300, 213, 21, 128
    mat = np.zeros((R_cap, ld), f32)
    mat[:, :NC] = rng.standard_normal((R_cap, NC)) * 2
    mat[:, NC:5 * NC] = rng.standard_normal((R_cap, 4 * NC)) * 0.5
    xy = rng.uniform(0, 800, size=(R_cap, 2))
    rois = np.hstack([xy, xy + rng.uniform(16, 300, size=(R_cap, 2))]).astype(f32)
    want_p = orc.softmax_axis1(mat[:, :NC])
    want_b = orc.clip_boxes(orc.bbox_transform_inv(rois, mat[:, NC:5 * NC]), (600, 1000))
    count = torch.tensor([R], dtype=torch.int32, device="cuda")
    p, b = ops.head_decode(dev(mat), ld, dev(rois), count, NC, 600, 1000)
    p, b = p.cpu().numpy(), b.cpu().numpy()
    assert np.array_equal(p[:R], want_p[:R]) and np.array_equal(b[:R], want_b[:R])
    assert not p[R:].any() and not b[R:].any()


def test_detect_per_class_nms(ops):
    rng = np.random.default_rng(8)
    R_cap, R, NC = 300, 288, 21
    logits = rng.standard_normal((R_cap, NC)) * 3
    prob = (np.exp(logits) / np.exp(logits).sum(1, keepdims=True)).astype(f32)
    base = gi._clustered_dets(R_cap, 55, ncl=12)[:, :4]
    boxes = np.tile(base, (1, NC)) + rng.standard_normal((R_cap, 4 * NC)).astype(f32) * 3
    boxes = boxes.astype(f32)
    count = torch.tensor([R], dtype=torch.int32, device="cuda")
    keep_idx, keep_count, conf_count = ops.detect(dev(prob), dev(boxes), count, nms_thresh=0.3, conf=0.3)
    keep_idx, keep_count, conf_count = keep_idx.cpu().numpy(), keep_count.cpu().numpy(), conf_count.cpu().numpy()
    for c in range(1, NC):
        dets = np.hstack([boxes[:R, 4 * c:4 * c + 4], prob[:R, c:c + 1]])
        want = orc.cpu_nms(dets, 0.3)
        assert keep_idx[c - 1, :keep_count[c - 1]].tolist() == want
        assert conf_count[c - 1] == int((dets[want, 4] >= 0.3).sum())


# ------------------------------------------------------------------------------- caller-side preprocessing ("next" row)
@pytest.mark.parametrize("shape", [(375, 500), (333, 500), (720, 1280), (600, 600), (97, 211)])
def test_preprocess_bgr8_bit_exact_vs_oracle(ops, shape):
    from frcnn_b200 import preprocess
    rng = np.random.default_rng(shape[0])
    img = rng.integers(0, 256, (shape[0], shape[1], 3), dtype=np.uint8)
    want, s = orc.img_preprocessing(img)
    got, s2 = preprocess.img_preprocessing(img)
    assert s2 == s and tuple(got.shape) == want.shape
    assert np.array_equal(got.cpu().numpy(), want)


def test_detections_assembly_matches_forward_py_loop(ops):
    from frcnn_b200 import preprocess
    rng = np.random.default_rng(31)
    R, NC = 120, 21
    logits = rng.standard_normal((R, NC)) * 4
    prob = (np.exp(logits) / np.exp(logits).sum(1, keepdims=True)).astype(f32)
    boxes = (np.tile(gi._clustered_dets(R, 9, ncl=6)[:, :4], (1, NC)) + rng.standard_normal((R, 4 * NC)) * 2).astype(f32)
    got = preprocess.detections(dev(prob), dev(boxes), 1.6, nms_thresh=0.3, conf=0.5)
    want = []
    for c, keep, dets in orc.detect(prob, boxes, 0.3, 0.5):                 # forward.py:50-57
        for d in dets:
            x1, y1, x2, y2 = map(int, d[:4] / 1.6)                           # forward.py:58
            want.append((c, x1, y1, x2, y2, float(d[4])))
    assert got == want and len(got) > 0


@pytest.mark.parametrize("x3", [True, False])
def test_long_k_gemm_rotating_accumulators_exact(ops, x3):
    """K = 25,088 (fc6) runs with its tensor-core partial sums promoted every 8 k-blocks: on small-integer operands every
    partial sum is exactly representable, so the result must equal the integer GEMM exactly -- in both precision modes --
    and a K just below the switch-over (one accumulator) must agree too."""
    g = torch.Generator(device="cuda").manual_seed(3)
    for K in (25088, 16320):                       # 392 k-blocks (rotation on) / 255 k-blocks (rotation off)
        M, N = 300, 128
        x = torch.randint(-2, 3, (1, M, K), device="cuda", generator=g).float()
        w = torch.randint(-2, 3, (N, K), device="cuda", generator=g).float()
        b = torch.randint(-5, 6, (N,), device="cuda", generator=g).float()
        xa = ops.Act(x.to(torch.bfloat16), torch.zeros_like(x, dtype=torch.bfloat16) if x3 else None)
        hi, lo = ops.pack_conv_weights(w, precision="bf16x3" if x3 else "bf16")
        y, y32 = ops.conv2d(xa, hi, lo, ops.pad_bias(b, N), 1, False, out_act=False, ld_f32=N)
        want = (x[0].double() @ w.double().T + b.double()).float()
        assert torch.equal(y32, want), (K, x3, float((y32 - want).abs().max()))


# ------------------------------------------------------------------------------- head linears, swapped operands + split-K
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("shape", [(300, 1024, 105, 171, False),      # cls_score|bbox_pred: one 128-row weight tile, fp32 out
                                   (300, 4096, 4096, 300, True),       # fc7
                                   (300, 25088, 4096, 233, True),      # fc6: 4 splits of 98 k-blocks, each promoting its sums
                                   (77, 192, 96, 50, True),            # ragged everything: R_cap < one N tile, 3 k-blocks
                                   (1000, 512, 256, 999, True)])       # config #4's RoI count (N tiles of 256)
def test_linear_swapab_vs_float64(ops, precision, shape):
    """frcnn_linear (weights on the M side, RoIs on the N side, K split over the SMs, fixed-order reduction) against the
    float64 product of the identical 16-bit-split operands; rows >= *m_valid are zero."""
    R, K, N, valid, relu = shape
    rng = np.random.default_rng(R + K + N)
    x = rng.standard_normal((R, K)).astype(f32)
    w = (rng.standard_normal((N, K)) * (1.0 / K) ** 0.5).astype(f32)
    b = (rng.standard_normal(N) * 0.1).astype(f32)
    q = _quant16 if precision == "bf16x3" else _bf16
    ref = (dev(q(x)).double() @ dev(q(w)).double().T).cpu().numpy() + b      # float64, on the GPU for fc6's size
    if relu:
        ref = np.maximum(ref, 0)
    xt = dev(x)[None]                                         # [1,R,K]
    hi = xt.to(torch.bfloat16)
    act = ops.Act(hi, (xt - hi.float()).to(torch.bfloat16) if precision == "bf16x3" else None)
    wh, wl = ops.pack_conv_weights(dev(w), precision=precision)
    m_valid = torch.tensor([valid], dtype=torch.int32, device="cuda")
    ld = (N + 31) // 32 * 32
    y, y32 = ops.linear(act, wh, wl, ops.pad_bias(dev(b), ld), relu, m_valid=m_valid, ld_f32=ld)
    y2, y32b = ops.linear(act, wh, wl, ops.pad_bias(dev(b), ld), relu, m_valid=m_valid, ld_f32=ld)
    torch.cuda.synchronize()
    got = y32.cpu().numpy()
    scale = np.abs(ref).max()
    err = np.abs(got[:valid, :N] - ref[:valid]).max() / scale
    assert err < 3e-5, err
    assert not got[valid:].any() and not got[:, N:].any()
    assert torch.equal(y32, y32b) and torch.equal(y.hi, y2.hi)                    # deterministic reduction
    val = y.hi[0].float() + (y.lo[0].float() if y.lo is not None else 0)
    err_act = np.abs(val.cpu().numpy()[:valid] - ref[:valid]).max() / scale
    assert err_act < (5e-5 if precision == "bf16x3" else 6e-3), err_act
    assert not val[valid:].any().item()


@pytest.mark.parametrize("x3", [True, False])
def test_linear_swapab_long_k_exact_on_integers(ops, x3):
    """Small-integer operands: every partial sum is exact in fp32, so split-K + promoted partial sums + the fixed-order
    reduction must reproduce the integer GEMM exactly (fc6: 4 splits of 98 promoted k-blocks; short K without promotion)."""
    g = torch.Generator(device="cuda").manual_seed(5)
    for K, N in ((25088, 4096), (4096, 256), (128, 256)):
        R = 300
        x = torch.randint(-2, 3, (1, R, K), device="cuda", generator=g).float()
        w = torch.randint(-2, 3, (N, K), device="cuda", generator=g).float()
        b = torch.randint(-5, 6, (N,), device="cuda", generator=g).float()
        xa = ops.Act(x.to(torch.bfloat16), torch.zeros_like(x, dtype=torch.bfloat16) if x3 else None)
        hi, lo = ops.pack_conv_weights(w, precision="bf16x3" if x3 else "bf16")
        _, y32 = ops.linear(xa, hi, lo, ops.pad_bias(b, N), False, ld_f32=N, want_act=False)
        want = (x[0].double() @ w.double().T + b.double()).float()
        assert torch.equal(y32, want), (K, x3, float((y32 - want).abs().max()))


# ------------------------------------------------------------------------------- compact first layer (sliding-window TMA)
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("shape", [(37, 45), (600 // 4, 1000 // 4 + 3), (16, 16), (9, 130)])
def test_conv1_1_compact_image_sliding_window(ops, precision, shape):
    """conv1_1 as frcnn_pack_image_c8 + frcnn_conv3x3_c8: the A operand of kernel row r is read through a tensor map whose
    pixel stride (16 B) is smaller than its 64-byte rows (stored pixels w..w+3 of row h+r-1; zero border columns in memory,
    rows -1 / H by TMA zero fill).  Against torch's conv2d on the identical 16-bit-split operands; the dense (C,H,W) source
    and the HWC-memory source (forward.py:45's strided view) must give the same bits."""
    H, W = shape
    rng = np.random.default_rng(H * 1000 + W)
    x = (rng.uniform(0, 255, size=(3, H, W)) - 110.0).astype(f32)
    w = (rng.standard_normal((64, 3, 3, 3)) * (2.0 / 27) ** 0.5).astype(f32)
    b = (rng.standard_normal(64) * 0.1).astype(f32)
    q = _quant16 if precision == "bf16x3" else _bf16
    ref = torch.nn.functional.conv2d(torch.from_numpy(q(x))[None].double(), torch.from_numpy(q(w)).double(),
                                     torch.from_numpy(b).double(), padding=1)[0].clamp_min(0).numpy()
    wh, wl = ops.pack_conv_weights_c8(dev(w), precision=precision)
    bias = ops.pad_bias(dev(b), 64)
    xc8 = ops.pack_image_c8(dev(x), precision=precision)
    y = ops.conv3x3_c8(xc8, H, W, wh, wl, bias, True)
    got = y.to_chw_f32().cpu().numpy()
    err = np.abs(got - ref).max() / np.abs(ref).max()
    assert err < (5e-5 if precision == "bf16x3" else 6e-3), err
    # HWC memory uploaded as it is: a (3,H,W)-shaped buffer whose bytes are the dense (H,W,3) image
    hwc_bytes = dev(np.ascontiguousarray(x.transpose(1, 2, 0))).reshape(3, H, W)
    y2 = ops.conv3x3_c8(ops.pack_image_c8(hwc_bytes, precision=precision, hwc_memory=True), H, W, wh, wl, bias, True)
    assert torch.equal(y2.hi, y.hi) and (y.lo is None or torch.equal(y2.lo, y.lo))
    # and the im2col formulation of the same layer agrees to rounding (different summation order inside the MMA)
    wih, wil = ops.pack_conv_weights_im2col(dev(w), precision=precision)
    y3, _ = ops.conv2d(ops.pack_image_im2col(dev(x), precision=precision), wih, wil, bias, 1, True)
    assert np.abs(y3.to_chw_f32().cpu().numpy() - got).max() / np.abs(ref).max() < (2e-5 if precision == "bf16x3" else 6e-3)
