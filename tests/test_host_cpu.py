"""CPU tests of host-side logic that needs no GPU: pure-host C-ABI helpers (called through the real library), the ResNet
graph description and BN folding, the oracle's training-step restatement against numerical differentiation."""
import ctypes

import numpy as np
import pytest

import frcnn_oracle as orc

f32 = np.float32


@pytest.fixture(scope="module")
def lib():
    from frcnn_b200 import _lib
    return _lib.load()


def test_padded_pixel_layout_helper(lib):
    """frcnn_padded_pixels: Wp = W+9 rounded up to 8, Kp = (H+2)*Wp rounded up to 64 (include/frcnn_b200.h)."""
    for H, W in [(600, 1000), (38, 63), (1, 1), (19, 25), (75, 125)]:
        wp = ctypes.c_int(0)
        kp = lib.frcnn_padded_pixels(H, W, ctypes.byref(wp))
        assert wp.value % 8 == 0 and W + 9 <= wp.value < W + 9 + 8
        assert kp % 64 == 0 and (H + 2) * wp.value <= kp < (H + 2) * wp.value + 64
        # every tap offset of every interior pixel stays inside [0, Kp): pixel (h, w) sits at (h+1)*Wp + 8 + w
        q_last = (H + 1) * wp.value + 8 + W                # pixel (H-1, W-1) shifted by (+1, +1)
        q_first = 8 - 1                                    # pixel (0, 0) shifted by (-1, -1) lands in row 0
        assert 0 <= q_first and q_last < kp


def test_splitk_effective_splits(lib):
    f = lib.frcnn_gemm_nt_splitk_splits
    assert f(64 * 37, 5) == 5 and f(64 * 37, 1) == 1 and f(64 * 4, 9) == 4 and f(64 * 40, 3) == 3
    for K, s in [(64 * 37, 5), (64 * 100, 7), (64 * 9, 9), (64 * 3, 2)]:
        eff = f(K, s)
        per = -(-(K // 64) // eff)
        assert (eff - 1) * per < K // 64 <= eff * per       # every split non-empty, all k-blocks covered


def test_resnet_graph_description_and_bn_folding():
    from frcnn_b200 import resnet_engine as re_
    for n, blocks in [(50, 16), (101, 33), (152, 50)]:
        bl = re_.block_list(n)
        assert len(bl) == blocks == len(orc.resnet_block_names(n)) and bl == orc.resnet_block_names(n)
        assert sum(3 + (1 if b[6] else 0) for b in bl) + 1 == {50: 53, 101: 104, 152: 155}[n]     # convolutions incl. conv1
        assert [b[5] for b in bl if b[1] == "a"] == [1, 2, 2, 2] and bl[-1][4] == 2048
    p = orc.make_resnet_params(50, seed=2)
    for conv, bn, bias in [("trunk/conv1", "trunk/bn1", p["trunk/conv1/b"]), ("trunk/res4/b3/conv2", "trunk/res4/b3/bn2", None)]:
        Wf, bf = re_.fold_batchnorm(p[conv + "/W"], p[bn + "/gamma"], p[bn + "/beta"], p[bn + "/avg_mean"], p[bn + "/avg_var"], bias)
        Wo, bo = orc.fold_bn(p[conv + "/W"], p, bn, bias)
        assert Wf.dtype == np.float32 and np.array_equal(Wf, Wo) and np.array_equal(bf, bo)
        # the folded convolution reproduces conv -> BN on random data
        import torch
        x = torch.randn(1, Wf.shape[1], 9, 11, dtype=torch.float64)
        y = torch.nn.functional.conv2d(x, torch.from_numpy(p[conv + "/W"]).double(), None if bias is None else torch.from_numpy(bias).double(),
                                       padding=Wf.shape[2] // 2)
        g, b_, m, v = (torch.from_numpy(p[bn + "/" + k]).double().view(1, -1, 1, 1) for k in ("gamma", "beta", "avg_mean", "avg_var"))
        want = g * (y - m) / torch.sqrt(v + orc.BN_EPS) + b_
        got = torch.nn.functional.conv2d(x, torch.from_numpy(Wf).double(), torch.from_numpy(bf).double(), padding=Wf.shape[2] // 2)
        assert float((got - want).abs().max()) < 1e-5 * float(want.abs().max())


def test_oracle_train_step_gradient_is_the_derivative_of_its_loss():
    """The autograd restatement (oracle.rpn_train_step) against central differences of its own loss, on a tiny image."""
    H, W = 64, 80
    rng = np.random.default_rng(0)
    params = orc.make_params(seed=5)
    for k in ("RPN/rpn_cls_score/W", "RPN/rpn_bbox_pred/W"):
        params[k] = (rng.standard_normal(params[k].shape) * 0.05).astype(f32)
    x = orc.make_image(H, W, seed=1)
    fh, fw = 4, 5
    n_all = 9 * fh * fw
    inds = np.arange(0, n_all, 3)
    labels = rng.integers(-1, 2, len(inds)).astype(np.int32)
    targets = rng.standard_normal((len(inds), 4)).astype(f32)
    out = orc.rpn_train_step(params, x, labels, targets, inds)
    for name, idx in [("RPN/rpn_bbox_pred/W", (3, 100, 0, 0)), ("RPN/rpn_conv_3x3/b", (7,)), ("trunk/conv5_3/W", (5, 9, 1, 2)),
                      ("trunk/conv1_1/W", (2, 1, 0, 1))]:
        eps = 1e-5 * max(float(params[name].std()), 1e-3)       # tiny against the tensor scale: stays between ReLU / max-pool kinks
        vals = []
        for sgn in (+1, -1):
            p2 = dict(params)
            w = params[name].astype(np.float64).copy()
            w[idx] += sgn * eps
            p2[name] = w
            vals.append(orc.rpn_train_step(p2, x, labels, targets, inds)["losses"][3])
        num = (vals[0] - vals[1]) / (2 * eps)
        ana = out["grads"][name][idx]
        assert abs(num - ana) <= 1e-3 * max(abs(ana), 1e-3) + 1e-7, (name, num, ana)
    # update rule: g += wd*w; v = m*v - lr*g; w += v
    k = "trunk/conv4_2/b"
    g = out["grads"][k] + 0.0005 * params[k]
    np.testing.assert_allclose(out["velocity"][k], -0.001 * g, rtol=1e-12, atol=0)
    np.testing.assert_allclose(out["params"][k], params[k] - 0.001 * g, rtol=1e-12, atol=0)


def test_preprocess_size_rule_matches_oracle_and_opencv():
    """frcnn_b200.preprocess.plan_size (host logic of forward.py:34-45): same scale and output size as the oracle's
    restatement for a sweep of image shapes, and the output size is what cv2.resize(fx=fy=scale) actually produces."""
    import cv2
    from frcnn_b200 import preprocess
    rng = np.random.default_rng(0)
    shapes = [(375, 500), (500, 375), (333, 500), (720, 1280), (600, 600), (97, 211), (1200, 400), (480, 640), (375, 625)]
    shapes += [tuple(int(v) for v in rng.integers(60, 1500, 2)) for _ in range(30)]
    for h0, w0 in shapes:
        s, H, W = preprocess.plan_size(h0, w0)
        so, Ho, Wo = orc.preprocess_plan(h0, w0)
        assert (H, W) == (Ho, Wo) and s == so, (h0, w0)
        out = cv2.resize(np.zeros((h0, w0, 3), np.float32), None, None, fx=s, fy=s, interpolation=cv2.INTER_LINEAR)
        assert out.shape[:2] == (H, W), (h0, w0, out.shape, (H, W))
        assert min(H, W) <= 600 + 1 and max(H, W) <= 1000 + 1


def test_host_copy_pool_is_a_memcpy():
    """frcnn_host_copy (the pageable -> pinned staging copy of the host-array front end) is pure host code: sleeping worker
    threads split the buffer; every byte count, including ragged tails and sizes below the threading threshold, must copy
    exactly and touch nothing behind the end."""
    import threading
    from frcnn_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(0)
    src = rng.integers(0, 256, size=9_000_001, dtype=np.uint8)
    for n in (0, 1, 4095, 4096, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, 7_200_000, 9_000_001):
        dst = np.full(src.size + 64, 0xAB, dtype=np.uint8)
        assert lib.frcnn_host_copy(dst.ctypes.data, src.ctypes.data, n) == 0
        assert np.array_equal(dst[:n], src[:n]) and (dst[n:] == 0xAB).all()
    # concurrent callers queue on the pool
    outs = [np.zeros(7_200_000, np.uint8) for _ in range(4)]
    ths = [threading.Thread(target=lambda o=o: [lib.frcnn_host_copy(o.ctypes.data, src.ctypes.data, o.size) for _ in range(5)]) for o in outs]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert all(np.array_equal(o, src[:o.size]) for o in outs)


def test_packed_pair_maximum_is_the_maximum_of_the_values():
    """What roi_pool_col_kernel relies on (csrc/head_ops.cu, 'RoI max pooling'): an activation is stored as v = hi + lo with
    hi = RN_bf16(v), lo = RN_bf16(v - hi), so |lo| <= ulp(hi)/2.  (1) hi + lo is exact in float32; (2) the order of the values is
    the lexicographic order of (hi, lo) -- equal values may have two different pairs (lo = +-ulp/2 exactly: v is a rounding
    midpoint, reachable from either neighbour), and only then; (3) the streaming fold the kernel uses (h' = max(h, b.h),
    l' = b.h > h ? b.l : b.h == h ? max(l, b.l) : l) returns a pair whose VALUE is the maximum, for any visiting order."""
    f32 = np.float32

    def rn_bf16(x):
        u = np.asarray(x, f32).view(np.uint32).astype(np.uint64)
        return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(f32)

    def split(x):
        hi = rn_bf16(x)
        return hi, rn_bf16(np.asarray(x, f32) - hi)

    rng = np.random.default_rng(11)
    x = np.concatenate([rng.standard_normal(200000).astype(f32) * f32(3), rng.uniform(-1e-3, 1e-3, 50000).astype(f32),
                        (rng.integers(-4096, 4096, 50000) / 8).astype(f32),          # many ties in hi, exact midpoints
                        np.array([0.0, -0.0, 257.0, 258.0, 255.0, -257.0, 1.0, 1.00390625, 0.99609375], f32)])
    hi, lo = split(x)
    v = hi + lo
    assert np.array_equal(v.astype(np.float64), hi.astype(np.float64) + lo.astype(np.float64))            # (1) exact sum
    ulp = np.ldexp(1.0, np.frexp(hi.astype(np.float64))[1] - 8)                                            # bf16: 8 significant bits
    assert np.all(np.abs(lo.astype(np.float64))[hi != 0] <= ulp[hi != 0] / 2)
    # a pair is not always the canonical split of its own value: when rounding lo lands on exactly half an ulp the value is a
    # midpoint and its re-split may pick the other neighbour -- same value, other pair; rare
    h2, l2 = split(v)
    other = (h2 != hi) | (l2 != lo)
    assert np.array_equal(h2 + l2, v) and 0 < other.sum() < 0.01 * len(x)
    # (2) sorting by (hi, lo) sorts by value (non-strictly: the equal-valued twin pairs are neighbours)
    order = np.lexsort((lo, hi))
    assert np.all(np.diff(v[order].astype(np.float64)) >= 0)
    # (3) the streaming fold over windows of random size and order, seeded with twin pairs where there are any
    twins = np.nonzero(other)[0]
    for k in range(300):
        idx = rng.integers(0, len(x), size=rng.integers(1, 70))
        if k % 3 == 0:
            idx = np.concatenate([idx, twins[rng.integers(0, len(twins), 3)]])
        h, l = f32(-np.inf), f32(-np.inf)
        for i in idx:
            bh, bl = hi[i], lo[i]
            l = bl if bh > h else (max(l, bl) if bh == h else l)
            h = max(h, bh)
        assert f32(h) + f32(l) == v[idx].max()
