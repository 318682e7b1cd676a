"""The ResNet detector against float64 at its benchmarked configuration, and its kernels at every size edge.

1. csrc/resnet_ops.cu against the explicit references of tests/resnet_ref.py, computed on the exact values the device
   holds: the 3x3/2 cover_all max-pool (one image and canvas, NaN / inf / signed-zero windows), the general im2col (one
   image and canvas), the im2col weight pack and the 2x subsample, bit for bit.
2. ResNet-101 at bench.py's 800x1333 / 1000 proposals, in bf16x3 and bf16, layer by layer: every convolution of the trunk,
   the RPN and the head, each fed the plan's own input and held PER ELEMENT to
   |dev - ref| <= TOL_ACT * (sum |x|*|w| + |b| + |residual|), the reference a float64 product of the packed planes.
   Each layer is re-launched on its own through ops (bit-identical) to read the kernel instantiation it ran.  The
   ProposalLayer (past its pre-NMS cut), RoI pooling, decode and per-class NMS on the device's own upstream tensors.
3. The whole device path against the fp32 oracle for the four images bench.py submits; ResNet-152's res4 blocks per
   element (its stage-wise check is test_resnet_gpu.py::test_resnet_faster_rcnn_forward_stagewise).
4. bench.py's LanePool(plan, lanes=4) over the graph plan: every lane bit-identical to the one-plan result."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc
import resnet_ref as rr
from test_conv_gemm_coverage_gpu import DISPATCH, TOL_ACT, conv_ref
from test_parity_hardening_gpu import _box_err_per_element, _match, _prob_err_per_element, _roi_bin_flips
from test_resnet_ref_cpu import IM2COL_GEOMETRIES, im2col_sizes

pytestmark = pytest.mark.gpu
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
H_BENCH, W_BENCH, POST_BENCH = 800, 1333, 1000       # bench.py --workload resnet101
BF16_NAN = (0x7FC0, 0xFFC0)                          # quiet NaN, both signs


@pytest.fixture(scope="module")
def ops():
    from frcnn_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def params101():
    return orc.make_resnet_params(101, seed=4321)


def bits(t):
    return t.view(torch.int16)


def planes_of(x32, precision):
    """float32 CUDA tensor -> (hi, lo or None) as the device stores it."""
    hi, lo = rr.split_rne(x32)
    return hi, (lo if precision == "bf16x3" else None)


def assert_planes(y, want, what):
    """Output planes y (ops.Act) bit for bit equal to the device's split of the float64 result `want` (split_rne of its
    float32 value; bf16 mode: hi alone).  A NaN result must be a NaN hi; a NaN lo (the split of +-inf) may have any payload.
    The split of -0.0 is (-0.0, +0.0): the sign of a zero result is carried by hi."""
    eh, el = rr.split_rne(want.float())
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(y.hi.float()), nan), (what, "NaN positions")
    assert torch.equal(bits(y.hi)[~nan], bits(eh)[~nan]), (what, "hi")
    if y.lo is not None:
        both_nan = torch.isnan(y.lo.float()) & torch.isnan(el.float())
        keep = ~nan & ~both_nan
        assert torch.equal(bits(y.lo)[keep], bits(el)[keep]), (what, "lo")


# ------------------------------------------------------------------------------- 1. the ResNet kernels at every size edge
def special_map(H, W, C, seed, precision):
    """[H,W,C] planes with NaN of both signs, +-inf and -0.0 / +0.0 pairs scattered over random data (every window of a
    3x3/2 pool meets some), and all-NaN / all-(-0.0) / all-(-inf) windows at fixed places."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((H, W, C), device="cuda", generator=g)
    r = torch.rand((H, W, C), device="cuda", generator=g)
    x = torch.where(r < 0.04, float("inf"), x)
    x = torch.where((r >= 0.04) & (r < 0.08), float("-inf"), x)
    x = torch.where((r >= 0.08) & (r < 0.16), 0.0, x)
    x = torch.where((r >= 0.16) & (r < 0.24), -0.0, x)
    hi, lo = planes_of(x, precision)
    nan_mask = (r >= 0.24) & (r < 0.34)
    sign = torch.rand((H, W, C), device="cuda", generator=g) < 0.5
    nan_bits = torch.where(sign, BF16_NAN[1] - 65536, BF16_NAN[0]).to(torch.int16)
    hi = torch.where(nan_mask, nan_bits.view(torch.bfloat16), hi)
    if C >= 8 and H >= 3 and W >= 3:
        hi[:3, :3, 0] = torch.tensor(BF16_NAN[0], dtype=torch.int16).view(torch.bfloat16)       # whole window NaN
        hi[:3, :3, 1] = -0.0                                                                     # whole window -0.0
        hi[:3, :3, 2] = float("-inf")
        hi[:3, :3, 3] = 0.0
        hi[0, 0, 3] = -0.0                                                                       # -0.0 first, +0.0 after
        hi[:3, :3, 4] = -0.0
        hi[2, 2, 4] = 0.0                                                                        # +0.0 last
        if lo is not None:
            lo[:3, :3, :5] = 0.0
            lo[:3, :3, 1] = -0.0                                                                 # (-0, -0) holds -0.0
            lo[0, 0, 3] = -0.0
            lo[:3, :3, 4] = -0.0
            lo[2, 2, 4] = 0.0
            lo[:3, :3, 2] = float("nan")                                                         # the split of -inf
    return hi, lo


def test_maxpool3x3s2_one_image_every_size(ops):
    """frcnn_maxpool3x3s2_ceil against Chainer's cover_all definition at every H, W in 3..24, C = 8 and 64, both
    precisions, on windows holding NaN (both signs), +-inf and signed zeros.  NaN is dropped unless the whole window is
    NaN and +0.0 ranks above -0.0 (DESIGN §2); an infinite value stored as its split (inf, NaN) is infinite."""
    seed = 0
    for precision in ("bf16x3", "bf16"):
        for C in (8, 64):
            for H in range(3, 25):
                for W in range(3, 25):
                    seed += 1
                    hi, lo = special_map(H, W, C, seed, precision)
                    y = ops.maxpool3x3s2_ceil(ops.Act(hi, lo))
                    want = rr.maxpool_cover_all(rr.pair_value(hi, lo))
                    assert y.hi.shape == want.shape, (H, W, C)
                    assert_planes(y, want, (precision, H, W, C))


def test_maxpool3x3s2_canvas_every_extent(ops):
    """frcnn_maxpool3x3s2_ceil_batch_ext on 24x24 slots with every extent pair in 0..24 (extents 0, 1 and 2 included,
    which the one-image entry refuses): windows clipped at the image's border, every other output exactly +0.0."""
    S, C = 24, 8
    ext = [(eh, ew) for eh in range(S + 1) for ew in range(S + 1)]
    N = len(ext)
    for precision in ("bf16x3", "bf16"):
        hs, ls = zip(*(special_map(S, S, C, 1000 + n, precision) for n in range(N)))
        hi = torch.stack(hs)
        lo = torch.stack(ls) if precision == "bf16x3" else None
        extents = torch.tensor(ext, dtype=torch.int32, device="cuda")
        y = ops.maxpool3x3s2_ceil_batch(ops.Act(hi, lo), extents=extents)
        So = rr.pool3s2_out(S)
        for n, (eh, ew) in enumerate(ext):
            want = rr.maxpool_cover_all(rr.pair_value(hi[n], None if lo is None else lo[n]), eh, ew, out_hw=(So, So))
            assert_planes(ops.Act(y.hi[n], None if y.lo is None else y.lo[n]), want, (precision, eh, ew))
        # the zero fill is +0.0 in both planes
        oh = torch.tensor([rr.pool3s2_out(e[0]) for e in ext], device="cuda")[:, None, None, None]
        ow = torch.tensor([rr.pool3s2_out(e[1]) for e in ext], device="cuda")[:, None, None, None]
        i = torch.arange(So, device="cuda")
        outside = (i[None, :, None, None] >= oh) | (i[None, None, :, None] >= ow)
        outside = outside.expand_as(y.hi)
        assert not bits(y.hi)[outside].any() and (y.lo is None or not bits(y.lo)[outside].any())


def im2col_expect(x, ks, stride, pad, k_pad, precision, eh=None, ew=None, out_hw=None):
    """The planes the im2col kernel must write: the RNE split of the float64 reference (exact float32 values)."""
    ref = rr.im2col(x, ks, stride, pad, k_pad, eh, ew, out_hw).float()
    return planes_of(ref, precision)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_pack_image_im2col_every_geometry(ops, precision):
    """frcnn_pack_image_im2col against F.unfold (float64, K reordered to (r*ks + s)*C + c) for ks in {1,3,5,7,11}, stride
    in {1,2,4}, pad 0..ks//2+1, on images from 1x1 up past both parities; the K columns [ks*ks*C, K_pad) are exactly 0."""
    g = torch.Generator(device="cuda").manual_seed(3)
    for ks, stride, pad in IM2COL_GEOMETRIES:
        C = 3 if stride != 2 else 5
        k_pad = -(-ks * ks * C // 8) * 8 + 8
        for H in im2col_sizes(ks, stride, pad):
            for W in im2col_sizes(ks, stride, pad):
                x = torch.randn((C, H, W), device="cuda", generator=g) * 50
                y = ops.pack_image_im2col_general(x, ks, stride, pad, k_pad, precision=precision)
                hi, lo = im2col_expect(x, ks, stride, pad, k_pad, precision)
                what = (ks, stride, pad, C, H, W)
                assert y.hi.shape == hi.shape, what
                assert torch.equal(bits(y.hi), bits(hi)), what
                assert lo is None or torch.equal(bits(y.lo), bits(lo)), what
                assert not bits(y.hi)[..., ks * ks * C:].any()


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_pack_image_im2col_canvas_every_geometry(ops, precision):
    """frcnn_pack_image_im2col_batch_ext: images of every side in one slot (nonzero data outside each image), each tap
    outside its image reads as the zero padding and every output pixel outside conv_out(extent) is 0."""
    g = torch.Generator(device="cuda").manual_seed(4)
    for ks, stride, pad in IM2COL_GEOMETRIES:
        C = 3
        k_pad = -(-ks * ks * C // 8) * 8 + 8
        sides = im2col_sizes(ks, stride, pad)
        S = sides[-1] + 1
        ext = [(eh, ew) for eh in [1] + sides + [S] for ew in ([1] + sides + [S])[::-1]]
        x = torch.randn((len(ext), C, S, S), device="cuda", generator=g) * 50
        extents = torch.tensor(ext, dtype=torch.int32, device="cuda")
        y = ops.pack_image_im2col_batch(x, ks, stride, pad, k_pad, precision=precision, extents=extents)
        Ho = rr.conv_out(S, ks, stride, pad)
        for n, (eh, ew) in enumerate(ext):
            hi, lo = im2col_expect(x[n], ks, stride, pad, k_pad, precision, eh, ew, out_hw=(Ho, Ho))
            what = (ks, stride, pad, eh, ew)
            assert torch.equal(bits(y.hi[n]), bits(hi)), what
            assert lo is None or torch.equal(bits(y.lo[n]), bits(lo)), what


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_pack_conv_weights_im2col_general_split(ops, precision):
    """frcnn_pack_conv_weights_im2col (through ops): hi = RNE-bf16(w), lo = RNE-bf16(w - hi), bit for bit in the im2col
    K order, zeros past ks*ks*Cin."""
    g = torch.Generator(device="cuda").manual_seed(5)
    for ks in (1, 3, 5, 7, 11):
        for Cin in (1, 3, 5):
            for Cout in (7, 64):
                w = torch.randn((Cout, Cin, ks, ks), device="cuda", generator=g) * 0.37
                k_pad = -(-ks * ks * Cin // 8) * 8 + 8
                hi, lo = ops.pack_conv_weights_im2col_general(w, k_pad, precision=precision)
                ref = torch.zeros((1, Cout, k_pad), device="cuda")
                ref[0, :, :ks * ks * Cin] = w.permute(0, 2, 3, 1).reshape(Cout, -1)
                eh, el = planes_of(ref, precision)
                assert torch.equal(bits(hi), bits(eh)), (ks, Cin, Cout)
                assert (lo is None) == (el is None) and (lo is None or torch.equal(bits(lo), bits(el))), (ks, Cin, Cout)


def test_subsample2x_every_size(ops):
    """frcnn_subsample2x == x[::2, ::2] bit for bit at every H, W in 1..9, both precisions."""
    g = torch.Generator(device="cuda").manual_seed(6)
    for precision in ("bf16x3", "bf16"):
        for H in range(1, 10):
            for W in range(1, 10):
                hi, lo = planes_of(torch.randn((H, W, 16), device="cuda", generator=g), precision)
                y = ops.subsample2x(ops.Act(hi, lo))
                assert torch.equal(bits(y.hi), bits(hi[::2, ::2])), (H, W)
                assert lo is None or torch.equal(bits(y.lo), bits(lo[::2, ::2])), (H, W)


# ------------------------------------------------------------------------------- 2. layer by layer at 800x1333
def act_value(a):
    return rr.pair_value(a.hi, a.lo)


def weight_value(hi, lo):
    return hi.double() + (lo.double() if lo is not None else 0)


def trunk_layers(plan, stage=None):
    """(name, kind, x, (w_hi, w_lo, bias), ksize, relu, residual, out) of every trunk convolution, in launch order."""
    cv = plan.w.convs
    L = [] if stage else [("conv1", "conv", plan.x_col, cv["conv1"], 1, True, None, plan.c1)]
    for B in plan.blocks:
        n = B["name"]
        if stage and not n.startswith(stage + "/"):
            continue
        x = B["xs"] if B["stride"] == 2 else B["x"]
        L.append((n + "/conv1", "conv", x, cv[n + "/conv1"], 1, True, None, B["y1"]))
        L.append((n + "/conv2", "conv", B["y1"], cv[n + "/conv2"], 3, True, None, B["y2"]))
        if B["proj"]:
            L.append((n + "/conv4", "conv", x, cv[n + "/conv4"], 1, False, None, B["sc"]))
        L.append((n + "/conv3", "res", B["y2"], cv[n + "/conv3"], 1, True, B["sc"] if B["proj"] else B["x"], B["out"]))
    return L


def head_layers(plan):
    w = plan.w
    return [("rpn 3x3", "conv", plan.feat, w.rpn3, 3, True, None, plan.rpn_mid),
            ("rpn cls|bbox", "conv_f32", plan.rpn_mid, w.rpn_heads, 1, False, None, plan.rpn_out),
            ("fc6", "linear", plan.pool5, w.fc6, 1, True, None, plan.fc6),
            ("fc7", "linear", plan.fc6, w.fc7, 1, True, None, plan.fc7),
            ("cls|bbox", "linear_f32", plan.fc7, w.head, 1, False, None, plan.head_out)]


def layer_error(plan, layer):
    """(worst |dev - ref| / (sum |x||w| + |b| + |res|), max-norm error) of one layer, float64 on the device."""
    name, kind, x, (whi, wlo, bias), k, relu, res, out = layer
    Cout = whi.shape[1]
    b = bias[:Cout].double()
    if kind.startswith("linear"):
        R = int(plan.prop.count.item())
        xv = act_value(x)[0, :R]
        xa = xv.abs()
        dev = act_value(out)[0, :R] if kind == "linear" else out[:R, :Cout].double()
        worst, dmax, rmax = 0.0, 0.0, 0.0
        step = 512                                               # output rows per float64 product (fc6: 2 x 411 MB of W)
        for c0 in range(0, Cout, step):
            wc = weight_value(whi[0, c0:c0 + step], None if wlo is None else wlo[0, c0:c0 + step])
            ref = xv @ wc.T + b[c0:c0 + step]
            bound = xa @ wc.abs().T + b[c0:c0 + step].abs()
            if relu:
                ref = ref.clamp_min(0)
            d = dev[:, c0:c0 + step]
            worst = max(worst, rr.elementwise_error(d, ref, bound))
            dmax, rmax = max(dmax, float((d - ref).abs().max())), max(rmax, float(ref.abs().max()))
            del wc, ref, bound
        return worst, dmax / rmax
    wv = weight_value(whi, wlo)                                  # [taps, Cout, Cin]
    xv = act_value(x)
    ref = conv_ref(xv, wv, b, k)
    bound = conv_ref(xv.abs(), wv.abs(), b.abs(), k)
    if res is not None:
        rv = act_value(res)
        ref += rv
        bound += rv.abs()
    if relu:
        ref = ref.clamp_min(0)
    if kind == "conv_f32":
        dev = out.view(ref.shape[0], ref.shape[1], -1)[:, :, :Cout].double()
    else:
        dev = act_value(out)
    return rr.elementwise_error(dev, ref, bound), rr.maxnorm_error(dev, ref)


def relaunch(ops, plan, layer):
    """The layer alone through ops on the plan's own input: asserts a bit-identical output, returns the instantiation."""
    name, kind, x, (whi, wlo, bias), k, relu, res, out = layer
    if kind == "conv":
        y, _ = ops.conv2d(x, whi, wlo, bias, k, relu)
        same = torch.equal(bits(y.hi), bits(out.hi)) and (y.lo is None or torch.equal(bits(y.lo), bits(out.lo)))
    elif kind == "res":
        y = ops.conv2d_res(x, whi, wlo, bias, k, relu, res)
        same = torch.equal(bits(y.hi), bits(out.hi)) and (y.lo is None or torch.equal(bits(y.lo), bits(out.lo)))
    elif kind == "conv_f32":
        _, y32 = ops.conv2d(x, whi, wlo, bias, k, relu, out_act=False, ld_f32=out.shape[1])
        same = torch.equal(y32, out)
    else:
        R = int(plan.prop.count.item())
        if kind == "linear":
            y, _ = ops.linear(x, whi, wlo, bias, relu, m_valid=plan.prop.count, work=plan.fc_work)
            same = torch.equal(bits(y.hi[0, :R]), bits(out.hi[0, :R])) and \
                (y.lo is None or torch.equal(bits(y.lo[0, :R]), bits(out.lo[0, :R])))
        else:
            _, y32 = ops.linear(x, whi, wlo, bias, relu, m_valid=plan.prop.count, ld_f32=out.shape[1], work=plan.fc_work,
                                want_act=False)
            same = torch.equal(y32[:R], out[:R])
    p = ops.conv_last_plan()
    torch.cuda.synchronize()
    assert same, (name, "re-launched alone it is not bit-identical to the plan's output")
    return (p["BN"], p["BK"], bool(p["x3"]), bool(p["promote"]), p["CG"])


def check_layers(ops, plan, layers, precision, title):
    """Every layer per element under TOL_ACT[precision]; prints the table, returns its rows."""
    tol = TOL_ACT[precision]
    rows = []
    for layer in layers:
        inst = relaunch(ops, plan, layer)
        worst, mn = layer_error(plan, layer)
        rows.append((layer[0], inst, worst, mn))
    print("\n%s (%s): layer, instantiation (BN, BK, x3, promote, CG), worst per-element error / bound, max-norm error"
          % (title, precision))
    for name, inst, worst, mn in rows:
        print("  %-16s %-28s %.3e  %.3e" % (name, inst, worst, mn))
    top = sorted(rows, key=lambda r: -r[2])[:3]
    print("  worst: " + ", ".join("%s %.3e (%.1fx under %.0e)" % (n, w, tol / max(w, 1e-300), tol) for n, _, w, _ in top))
    for name, inst, worst, mn in rows:
        assert inst in DISPATCH, (name, inst, "an instantiation test_conv_gemm_coverage_gpu.DISPATCH does not list")
        assert worst <= tol, (name, worst, tol)
    return rows


def check_pack(plan, params, n_layers):
    """Every packed trunk plane is the fold_batchnorm float32 weight split into RNE hi / lo, bit for bit, and every
    packed bias is the folded bias."""
    from frcnn_b200.resnet_engine import block_list, fold_batchnorm
    w = plan.w

    def fold(conv, bn, bias=None):
        return fold_batchnorm(params[conv + "/W"], params[bn + "/gamma"], params[bn + "/beta"], params[bn + "/avg_mean"],
                              params[bn + "/avg_var"], bias)

    def same(name, packed, Wf, bf, kmajor):
        hi, lo, b = packed
        W32 = torch.from_numpy(Wf).cuda()
        Cout = W32.shape[0]
        if kmajor:                                   # conv1: [1, Cout, K_pad], K = (r*7 + s)*3 + c
            want = torch.zeros(hi.shape, device="cuda")
            want[0, :, :W32[0].numel()] = W32.permute(0, 2, 3, 1).reshape(Cout, -1)
        else:                                        # [taps, Cout, Cin]
            want = W32.permute(2, 3, 0, 1).reshape(-1, Cout, W32.shape[1])
        eh, el = planes_of(want, w.precision)
        assert torch.equal(bits(hi), bits(eh)) and (el is None or torch.equal(bits(lo), bits(el))), name
        assert torch.equal(b[:Cout], torch.from_numpy(bf).cuda()) and not b[Cout:].any(), name
    same("conv1", w.convs["conv1"], *fold("trunk/conv1", "trunk/bn1", params["trunk/conv1/b"]), kmajor=True)
    for stage, blk, cin, mid, cout, stride, proj in block_list(n_layers):
        for ci in ((1, 2, 3, 4) if proj else (1, 2, 3)):
            base = "trunk/%s/%s" % (stage, blk)
            n = "%s/%s/conv%d" % (stage, blk, ci)
            same(n, w.convs[n], *fold(base + "/conv%d" % ci, base + "/bn%d" % ci), kmajor=False)


def run_plan(params, n_layers, precision, H, W, seed, post_n):
    from frcnn_b200.resnet_engine import ResNetEngine
    eng = ResNetEngine(params, n_layers, precision=precision, anchors=ANCHORS, use_graph=False, post_n=post_n,
                       with_detect=True, det_conf=0.05)
    x = orc.make_image(H, W, seed=seed)
    prob, boxes, plan = eng(torch.from_numpy(x[0]).cuda())
    torch.cuda.synchronize()
    return x, prob, boxes, plan


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_resnet101_800x1333_layer_by_layer(ops, params101, precision):
    """bench.py's ResNet-101 configuration, one layer at a time on the plan's own activations (see the module docstring),
    then the pool, the subsamples and the tail bit for bit on the device's own upstream tensors."""
    H, W = H_BENCH, W_BENCH
    x, prob, boxes, plan = run_plan(params101, 101, precision, H, W, 0, POST_BENCH)
    check_pack(plan, params101, 101)
    # conv1's im2col, the pool and every subsample: selections and copies, bit for bit
    hi, lo = im2col_expect(torch.from_numpy(x[0]).cuda(), 7, 2, 3, plan.x_col.hi.shape[2], precision)
    assert torch.equal(bits(plan.x_col.hi), bits(hi)) and (lo is None or torch.equal(bits(plan.x_col.lo), bits(lo)))
    assert_planes(plan.p1, rr.maxpool_cover_all(act_value(plan.c1)), "pool1")
    for B in plan.blocks:
        if B["stride"] == 2:
            assert torch.equal(bits(B["xs"].hi), bits(B["x"].hi[::2, ::2])), B["name"]
            assert B["xs"].lo is None or torch.equal(bits(B["xs"].lo), bits(B["x"].lo[::2, ::2])), B["name"]
    check_layers(ops, plan, trunk_layers(plan) + head_layers(plan), precision, "ResNet-101 %dx%d" % (H, W))
    # the tail on the device's own tensors: 25 x 42 x 9 = 9450 anchors against the pre-NMS cut of 6000
    R = prob.shape[0]
    info = np.array([[H, W]], np.int32)
    fh, fw = plan.fh, plan.fw
    assert fh * fw * 9 > plan.pre_n
    rpn = plan.rpn_out.cpu().numpy()
    logits = rpn[:, :18].T.reshape(1, 18, fh, fw)
    deltas = rpn[:, 18:54].T.reshape(1, 36, fh, fw)
    want_rois, want_fg = orc.proposal_layer(orc.softmax_axis1(logits), deltas, info, feat_stride=32,
                                            post_nms_top_n=POST_BENCH)
    rois = plan.prop.rois.cpu().numpy()[:R]
    assert R == len(want_rois) > 0
    assert np.array_equal(rois, want_rois) and np.array_equal(plan.prop.scores.cpu().numpy()[:R], want_fg.ravel())
    feat = plan.feat.to_chw_f32().cpu().numpy()[None]
    brois = np.concatenate((np.zeros((R, 1), np.float32), rois), axis=1)
    pool = act_value(plan.pool5)[0, :R].float().cpu().numpy().reshape(R, 7, 7, -1).transpose(0, 3, 1, 2)
    assert np.array_equal(pool, orc.roi_pool(feat, brois, 7, 7, 1.0 / 32))
    ho = plan.head_out.cpu().numpy()[:R]
    p, b = prob.cpu().numpy(), boxes.cpu().numpy()
    assert np.array_equal(p, orc.softmax_axis1(ho[:, :21]))
    assert np.array_equal(b, orc.clip_boxes(orc.bbox_transform_inv(rois, ho[:, 21:105]), (H, W)))
    keep_idx, keep_count, conf_count = [t.cpu().numpy() for t in plan.det]
    for c, keep, _ in orc.detect(p, b, 0.3, 0.05):
        assert keep_idx[c - 1, :conf_count[c - 1]].tolist() == keep.tolist(), c
    print("R = %d of %d anchors (pre-NMS cut %d); per-class NMS lists: %d detections" % (R, fh * fw * 9, plan.pre_n,
                                                                                          int(conf_count.sum())))


# ------------------------------------------------------------------------------- 3. pure end to end, and ResNet-152
@pytest.fixture(scope="module")
def engine101(params101):
    from frcnn_b200.resnet_engine import ResNetEngine
    return ResNetEngine(params101, 101, precision="bf16x3", anchors=ANCHORS, use_graph=False, post_n=POST_BENCH)


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_resnet101_800x1333_pure_end_to_end(params101, engine101, seed):
    """The whole device path against the whole fp32 oracle for bench.py's image `seed`, with
    test_headline_600x1000_pure_end_to_end_seeds's method and bounds; res5 within 1e-4 of the oracle's max-norm."""
    H, W = H_BENCH, W_BENCH
    x = orc.make_image(H, W, seed=seed)
    prob, boxes, plan = engine101(torch.from_numpy(x[0]).cuda())
    R = prob.shape[0]
    cls_ref, box_ref, aux = orc.faster_rcnn_resnet_forward(x, params101, np.array([[H, W]], np.int32), 101,
                                                           post_nms_top_n=POST_BENCH)
    e_feat = rr.maxnorm_error(torch.from_numpy(plan.feat.to_chw_f32().cpu().numpy()[None]).double(),
                              torch.from_numpy(aux["feature_map"]).double())
    rois = plan.prop.rois.cpu().numpy()[:R]
    ok, j = _match(rois, aux["proposals"], max(H, W))
    flips = ok & _roi_bin_flips(rois, aux["proposals"][j], scale=1.0 / 32)
    good = ok & ~flips
    p, b = prob.cpu().numpy(), boxes.cpu().numpy()
    e_p_abs = float(np.abs(p[good] - cls_ref[j[good]]).max())
    e_p_el, n_el = _prob_err_per_element(p[good], cls_ref[j[good]])
    e_b_max = float(np.abs(b[good] - box_ref[j[good]]).max() / max(H, W))
    e_b_el = _box_err_per_element(b[good], box_ref[j[good]], rois[good])
    print("seed %d ResNet-101 800x1333 pure e2e: res5 %.2e | R dev/oracle %d/%d matched %.4f RoI-bin flips %d | probs abs "
          "%.2e per-element(p>=1e-3, n=%d) %.2e | boxes /image-scale %.2e per-element(/RoI size) %.2e" %
          (seed, e_feat, R, len(aux["proposals"]), ok.mean(), int(flips.sum()), e_p_abs, n_el, e_p_el, e_b_max, e_b_el))
    assert e_feat < 1e-4
    assert ok.mean() >= 0.97 and good.mean() >= 0.97
    assert e_p_abs < 1e-4 * cls_ref.max()
    assert e_b_max < 3e-4


@pytest.fixture(scope="module")
def params152():
    return orc.make_resnet_params(152, seed=11)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_resnet152_res4_layer_by_layer(ops, params152, precision):
    """ResNet-152's 36 res4 blocks (all that differs from ResNet-101) per element at 600x1000, as above."""
    _, _, _, plan = run_plan(params152, 152, precision, 600, 1000, 4, 300)
    layers = trunk_layers(plan, stage="res4")
    assert len(layers) == 36 * 3 + 1
    check_layers(ops, plan, layers, precision, "ResNet-152 res4 600x1000")


# ------------------------------------------------------------------------------- 4. the benchmark's lane pool
def test_resnet101_lane_pool_bit_identical(params101):
    """LanePool(plan, lanes=4) over the graph plan bench.py times: the four bench images submitted twice (the second
    round in reverse order, so every lane runs another image), each result bit-identical to the one-plan result."""
    from frcnn_b200.engine import LanePool
    from frcnn_b200.resnet_engine import ResNetEngine
    eng = ResNetEngine(params101, 101, precision="bf16x3", anchors=ANCHORS, use_graph=True, post_n=POST_BENCH)
    plan = eng.plan(H_BENCH, W_BENCH)
    imgs = [torch.from_numpy(orc.make_image(H_BENCH, W_BENCH, seed=i)[0]).cuda() for i in range(4)]

    def result(p):
        R = int(p.prop.count.item())
        return R, [t[:R].clone() for t in (p.prob, p.boxes, p.prop.rois, p.prop.scores)]
    want = []
    for im in imgs:
        plan.forward(im)
        want.append(result(plan))
    pool = LanePool(plan, lanes=4)
    for order in (range(4), range(3, -1, -1)):
        pool.fork()
        lanes = [(pool.submit(i, imgs[k]), k) for i, k in enumerate(order)]
        pool.join()
        torch.cuda.synchronize()
        for p, k in lanes:
            R, got = result(p)
            assert R == want[k][0], k
            for g, w_ in zip(got, want[k][1]):
                assert torch.equal(g.view(torch.int32), w_.view(torch.int32)), k
