"""GPU tests of the batched forward path: N images of one shape through frcnn_conv2d_batch, frcnn_conv3x3_c8_batch,
frcnn_linear_batch and engine.BatchPlan.  Every image's result must be bit-identical to the one-image entry point (or
ForwardPlan) on that image, no image may read or write another image's data, and the batched launches keep the
one-image plan (only the tile count grows)."""
import numpy as np
import pytest
import torch

import frcnn_oracle as orc

pytestmark = pytest.mark.gpu
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
SENTINEL = -12345
PLAN_KEYS = ("BN", "BK", "x3", "promote", "CG", "TH", "TW", "n_parts", "splits")


@pytest.fixture(scope="module")
def params():
    return orc.make_params(seed=1234)


def _ops():
    from frcnn_b200 import ops
    return ops


def _act(t, x3):
    """bf16 hi/lo planes of a float32 tensor (lo = the rounding residual)."""
    ops = _ops()
    hi = t.to(torch.bfloat16)
    return ops.Act(hi.contiguous(), (t - hi.float()).to(torch.bfloat16).contiguous() if x3 else None)


def _canaried(shape, dtype, dev="cuda"):
    """A buffer of `shape` followed by 4096 sentinel elements: (view, whole buffer)."""
    n = int(np.prod(shape))
    buf = torch.full((n + 4096,), SENTINEL, dtype=torch.int32 if dtype == torch.float32 else torch.int16, device=dev)
    buf = buf.view(dtype)
    return buf[:n].view(shape), buf


def _tail_intact(buf, n):
    t = buf[n:].view(torch.int32 if buf.dtype == torch.float32 else torch.int16)
    return bool((t == SENTINEL).all().item())


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _weights(Cout, Cin, k, x3, seed):
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn((Cout, Cin, k, k), generator=g) * (2.0 / (Cin * k * k)) ** 0.5).cuda()
    hi, lo = ops.pack_conv_weights(w, precision="bf16x3" if x3 else "bf16")
    return hi, lo


# ------------------------------------------------------------------------------------------------ 1-3: convolutions
# (H, W, Cin, Cout, ksize, fused pool, bf16 out, ld_f32): trunk-like ragged sizes -- odd, not multiples of the 8x16 /
# 16x8 tiles, a ceil-mode pool remainder of one
CONV_CASES = {
    "conv3_3x3_pool": (75, 125, 128, 256, 3, True, True, 0),
    "conv4_3x3": (37, 63, 256, 512, 3, False, True, 0),
    "conv5_3x3_pool": (19, 33, 512, 512, 3, True, True, 0),
    "rpn_1x1_f32": (19, 31, 512, 54, 1, False, False, 64),
    "3x3_bf16_and_f32": (13, 21, 64, 64, 3, False, True, 64),
}


def _conv_io(case, N, x3, seed):
    H, W, Cin, Cout, k, pool, out_bf16, ld = CONV_CASES[case]
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn((N, H, W, Cin), generator=g)).cuda()
    hi, lo = _weights(Cout, Cin, k, x3, seed + 1)
    bias = _ops().pad_bias((torch.randn((Cout,), generator=g) * 0.1).cuda(), max(Cout, ld))
    return x, hi, lo, bias


def _conv_batch(case, xa, hi, lo, bias, N):
    """Batched launch into canaried outputs; returns (Act or None, f32 or None, list of (buffer, used elements), plan)."""
    ops = _ops()
    H, W, Cin, Cout, k, pool, out_bf16, ld = CONV_CASES[case]
    oh, ow = ((H + 1) // 2, (W + 1) // 2) if pool else (H, W)
    bufs, y, y32 = [], None, None
    if out_bf16:
        yh, bh = _canaried((N, oh, ow, Cout), torch.bfloat16)
        bufs.append((bh, yh.numel()))
        yl = None
        if xa.lo is not None:
            yl, bl = _canaried((N, oh, ow, Cout), torch.bfloat16)
            bufs.append((bl, yl.numel()))
        y = ops.Act(yh, yl)
    if ld:
        y32, b32 = _canaried((N * H * W, ld), torch.float32)
        bufs.append((b32, y32.numel()))
    ops.conv2d_batch(xa, hi, lo, bias, k, True if out_bf16 else False, out_act=out_bf16, ld_f32=ld, out=y, out_f32=y32,
                     fuse_pool=pool)
    plan = ops.conv_last_plan()
    return y, y32, bufs, plan


def _conv_single(case, xa_n, hi, lo, bias):
    ops = _ops()
    H, W, Cin, Cout, k, pool, out_bf16, ld = CONV_CASES[case]
    y, y32 = ops.conv2d(xa_n, hi, lo, bias, k, True if out_bf16 else False, out_act=out_bf16, ld_f32=ld, fuse_pool=pool)
    return y, y32, ops.conv_last_plan()


def _check_conv_images(case, N, xa, y, y32, hi, lo, bias, only=None):
    H, W = CONV_CASES[case][:2]
    plan1 = None
    for n in range(N) if only is None else only:
        xn = _ops().Act(xa.hi[n], None if xa.lo is None else xa.lo[n])
        ys, ys32, plan1 = _conv_single(case, xn, hi, lo, bias)
        if y is not None:
            assert torch.equal(_bits(y.hi[n]), _bits(ys.hi)), (case, n)
            if y.lo is not None:
                assert torch.equal(_bits(y.lo[n]), _bits(ys.lo)), (case, n)
        if y32 is not None:
            assert torch.equal(_bits(y32[n * H * W:(n + 1) * H * W]), _bits(ys32)), (case, n)
    return plan1


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
@pytest.mark.parametrize("N", [1, 2, 3, 5])
@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv2d_batch_equals_per_image_conv(case, N, x3):
    """Each image of a batched launch is bit-identical to frcnn_conv2d on that image; the plan is the one-image plan with N
    times the tiles; nothing is written past the last image."""
    x, hi, lo, bias = _conv_io(case, N, x3, seed=N * 7 + len(case))
    xa = _act(x, x3)
    y, y32, bufs, plan = _conv_batch(case, xa, hi, lo, bias, N)
    torch.cuda.synchronize()
    plan1 = _check_conv_images(case, N, xa, y, y32, hi, lo, bias)
    assert {k: plan[k] for k in PLAN_KEYS} == {k: plan1[k] for k in PLAN_KEYS}
    assert plan["num_tiles"] == N * plan1["num_tiles"]
    for buf, n in bufs:
        assert _tail_intact(buf, n), case


@pytest.mark.parametrize("case", ["conv4_3x3", "conv5_3x3_pool", "rpn_1x1_f32"])
def test_conv2d_batch_image_isolation(case):
    """Changing image j's input changes image j's output only: no image's halo reads its neighbour's rows."""
    N, x3 = 3, True
    x, hi, lo, bias = _conv_io(case, N, x3, seed=99)
    y0, y320, _, _ = _conv_batch(case, _act(x, x3), hi, lo, bias, N)
    before = [t.clone() for t in (y0.hi if y0 else None, y320) if t is not None]
    for j in range(N):
        x2 = x.clone()
        x2[j] = torch.relu(torch.randn_like(x2[j])) * 3 + 1
        xa2 = _act(x2, x3)
        y, y32, _, _ = _conv_batch(case, xa2, hi, lo, bias, N)
        H, W = CONV_CASES[case][:2]
        after = [t for t in (y.hi if y else None, y32) if t is not None]
        for b, a in zip(before, after):
            if b.dim() == 2:            # fp32 [N*H*W, ld]
                b, a = b.view(N, H * W, -1), a.view(N, H * W, -1)
            for n in range(N):
                same = torch.equal(_bits(b[n]), _bits(a[n]))
                assert same == (n != j), (case, j, n)
        _check_conv_images(case, N, xa2, y, y32, hi, lo, bias, only=[j])


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
@pytest.mark.parametrize("N", [1, 2, 3, 5])
def test_c8_first_layer_batch_equals_per_image(N, x3):
    """pack_image_c8_batch + conv3x3_c8_batch (conv1_1) = pack_image_c8 + conv3x3_c8 on every image, bit for bit, with
    canaries after the last image; changing one image changes only its own output."""
    ops = _ops()
    H, W, Cout = 37, 61, 64
    prec = "bf16x3" if x3 else "bf16"
    g = torch.Generator().manual_seed(N)
    x = (torch.randn((N, 3, H, W), generator=g) * 50).cuda()
    w = (torch.randn((Cout, 3, 3, 3), generator=g) * 0.1).cuda()
    whi, wlo = ops.pack_conv_weights_c8(w, precision=prec)
    bias = ops.pad_bias((torch.randn((Cout,), generator=g) * 0.1).cuda(), Cout)
    n8 = ops._lib.load().frcnn_image_c8_elems(H, W)

    def run(xb):
        ph, bph = _canaried((N, n8), torch.bfloat16)
        pl, bpl = _canaried((N, n8), torch.bfloat16) if x3 else (None, None)
        packed = ops.pack_image_c8_batch(xb, precision=prec, out=ops.Act(ph, pl))
        yh, byh = _canaried((N, H, W, Cout), torch.bfloat16)
        yl, byl = _canaried((N, H, W, Cout), torch.bfloat16) if x3 else (None, None)
        y = ops.conv3x3_c8_batch(packed, N, H, W, whi, wlo, bias, True, out=ops.Act(yh, yl))
        plan = ops.conv_last_plan()
        torch.cuda.synchronize()
        for b, n_ in ((bph, ph.numel()), (bpl, n8 * N), (byh, yh.numel()), (byl, yh.numel())):
            if b is not None:
                assert _tail_intact(b, n_)
        return packed, y, plan

    packed, y, plan = run(x)
    for n in range(N):
        p1 = ops.pack_image_c8(x[n], precision=prec)
        assert torch.equal(_bits(packed.hi[n]), _bits(p1.hi))
        y1 = ops.conv3x3_c8(p1, H, W, whi, wlo, bias, True)
        plan1 = ops.conv_last_plan()
        assert torch.equal(_bits(y.hi[n]), _bits(y1.hi))
        if x3:
            assert torch.equal(_bits(packed.lo[n]), _bits(p1.lo)) and torch.equal(_bits(y.lo[n]), _bits(y1.lo))
    assert {k: plan[k] for k in PLAN_KEYS} == {k: plan1[k] for k in PLAN_KEYS}
    assert plan["num_tiles"] == N * plan1["num_tiles"]
    if N > 1:
        before = y.hi.clone()
        x2 = x.clone()
        x2[N - 1] = -x2[N - 1]
        _, y2, _ = run(x2)
        for n in range(N):
            assert torch.equal(_bits(before[n]), _bits(y2.hi[n])) == (n != N - 1)


def test_pack_image_c8_batch_hwc_memory():
    """hwc_memory: the buffer holds dense (N,H,W,3) images; same planes as packing the (N,3,H,W) copy."""
    ops = _ops()
    x = torch.randn((2, 9, 14, 3), device="cuda")
    a = ops.pack_image_c8_batch(x.permute(0, 3, 1, 2).contiguous())
    b = ops.pack_image_c8_batch(x.view(2, 3, 9, 14), hwc_memory=True)          # same bytes, shaped (N,3,H,W)
    assert torch.equal(_bits(a.hi), _bits(b.hi)) and torch.equal(_bits(a.lo), _bits(b.lo))


# --------------------------------------------------------------------------------------------------- 4: head GEMMs
# (K, Cout, relu, ld_f32): fc6, fc7, cls_score|bbox_pred
LINEAR_CASES = {"fc6": (25088, 4096, True, 0), "fc7": (4096, 4096, True, 0), "head": (4096, 105, False, 128)}


@pytest.mark.parametrize("x3", [True, False], ids=["bf16x3", "bf16"])
@pytest.mark.parametrize("R_cap,counts", [(300, [0, 1, 299, 300]), (80, [80, 3])])
@pytest.mark.parametrize("layer", list(LINEAR_CASES))
def test_linear_batch_equals_per_image_linear(layer, R_cap, counts, x3):
    """frcnn_linear_batch = frcnn_linear per image, bit for bit (the one-image N tile and split count); rows past each
    image's count (up to the segment's round_up(R_cap, 32) rows) are zero.  R_cap 80: 96-row segments under a 128-wide
    N tile, so one tile spans two images' rows."""
    ops = _ops()
    K, Cout, relu, ld = LINEAR_CASES[layer]
    N, ld1 = len(counts), ops.round_up(R_cap, 32)
    g = torch.Generator().manual_seed(K + Cout + R_cap)
    x = torch.zeros((N, ld1, K))
    x[:, :R_cap] = torch.relu(torch.randn((N, R_cap, K), generator=g))
    x = x.cuda()
    xa = _act(x, x3)
    w = (torch.randn((Cout, K), generator=g) * (2.0 / K) ** 0.5).cuda()
    whi, wlo = ops.pack_conv_weights(w, precision="bf16x3" if x3 else "bf16")
    bias = ops.pad_bias((torch.randn((Cout,), generator=g) * 0.1).cuda(), max(Cout, ld))
    # counts strided as in a BatchPlan result buffer: count n at word n * 7
    cnt = torch.full((7 * N,), 999, dtype=torch.int32, device="cuda")
    cnt[::7] = torch.tensor(counts, dtype=torch.int32)
    y, y32 = ops.linear_batch(xa, whi, wlo, bias, relu, R_cap, counts=cnt, count_stride=7, ld_f32=ld, want_act=not ld)
    plan = ops.conv_last_plan()
    torch.cuda.synchronize()
    for n, c in enumerate(counts):
        xn = ops.Act(xa.hi[n:n + 1, :R_cap], None if xa.lo is None else xa.lo[n:n + 1, :R_cap])
        ys, ys32 = ops.linear(xn, whi, wlo, bias, relu, m_valid=cnt[7 * n:7 * n + 1], ld_f32=ld, want_act=not ld)
        plan1 = ops.conv_last_plan()
        if ld:
            assert torch.equal(_bits(y32[n, :R_cap]), _bits(ys32)), (layer, n)
            assert not y32[n, c:].any().item()
        else:
            assert torch.equal(_bits(y.hi[n, :R_cap]), _bits(ys.hi[0])), (layer, n)
            assert not y.hi[n, c:].float().any().item()
            if x3:
                assert torch.equal(_bits(y.lo[n, :R_cap]), _bits(ys.lo[0])), (layer, n)
    assert {k: plan[k] for k in PLAN_KEYS} == {k: plan1[k] for k in PLAN_KEYS}
    # the N tile walks all images' rows: N times the one-image tiles when the tile divides the segment (R_cap 300)
    bn = plan1["BN"]
    per_ntile = plan1["num_tiles"] // -(-ld1 // bn)
    assert plan["num_tiles"] == per_ntile * -(-N * ld1 // bn)
    if ld1 % plan1["BN"] == 0:
        assert plan["num_tiles"] == N * plan1["num_tiles"]


# --------------------------------------------------------------------------------------------- 5-7: the whole graph
FIELDS = ("prob", "boxes", "rois", "scores", "keep_count", "conf_count", "keep_idx")


def _images(N, H, W, seed, nan_at=None):
    x = np.stack([orc.make_image(H, W, seed=seed + n)[0] for n in range(N)]).astype(np.float32)
    if nan_at is not None:
        x[nan_at] = np.nan
    return torch.from_numpy(x).cuda()


def _assert_same(got, want, what):
    assert got["count"] == want["count"], what
    for f in FIELDS:
        a, b = np.asarray(got[f]), np.asarray(want[f])
        assert a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32)), (what, f)


def _per_image(plan1, x):
    out = []
    for n in range(x.shape[0]):
        plan1.forward(x[n])
        torch.cuda.synchronize()
        out.append({k: (v.copy() if isinstance(v, np.ndarray) else v)
                    for k, v in plan1.unpack_result(plan1.result.cpu().numpy()).items()})
    return out


def _batch_result(bplan):
    torch.cuda.synchronize()
    return bplan.unpack_result(bplan.result.cpu().numpy())


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("N", [1, 2, 3])
def test_batch_plan_equals_forward_plan_150x201(params, N, precision):
    """BatchPlan = ForwardPlan per image on every result field, with the per-class NMS on; an all-NaN image has no
    proposals; the graph replays twice and then takes a second input set."""
    from frcnn_b200.engine import BatchPlan, Engine
    H, W = 150, 201
    eng = Engine(params, precision=precision, anchors=ANCHORS, with_detect=True, det_conf=0.05)
    plan1 = eng.plan(H, W)
    bplan = eng.batch_plan(N, H, W)
    assert isinstance(bplan, BatchPlan) and eng.batch_plan(N, H, W) is bplan
    first = _images(N, H, W, seed=10, nan_at=1 if N > 1 else None)
    second = _images(N, H, W, seed=20)
    want1, want2 = _per_image(plan1, first), _per_image(plan1, second)
    assert all(w["count"] > 0 for w in want2)
    for rep in range(2):
        bplan.forward(first)
        for n, (g, w) in enumerate(zip(_batch_result(bplan), want1)):
            _assert_same(g, w, ("replay", rep, n))
    bplan.forward(second)
    for n, (g, w) in enumerate(zip(_batch_result(bplan), want2)):
        _assert_same(g, w, ("second input", n))
    # the host front end: one upload, one D2H of every block
    host = np.ascontiguousarray(second.cpu().numpy().copy())
    assert host.flags.c_contiguous and host.nbytes == bplan.x_in.numel() * 4, (host.flags, host.nbytes, bplan.x_in.shape)
    got = bplan.forward_host(host)
    for n, (g, w) in enumerate(zip(got, want2)):
        _assert_same(g, w, ("forward_host", n))
    # Engine.forward_batch: per-image (prob[:R], boxes[:R])
    for (p, b), w in zip(eng.forward_batch(second), want2):
        assert p.shape[0] == w["count"] and np.array_equal(p.cpu().numpy(), w["prob"]) and np.array_equal(b.cpu().numpy(), w["boxes"])


def test_batch_plan_without_proposals(params):
    """min_size above the image size: no image keeps a proposal; every later stage copes with zero RoIs, and the result
    equals ForwardPlan's (zero counts, zero rows, empty keep lists)."""
    from frcnn_b200.engine import Engine
    H, W, N = 96, 128, 2
    eng = Engine(params, precision="bf16x3", anchors=ANCHORS, with_detect=True, min_size=10000)
    x = _images(N, H, W, seed=3, nan_at=0)
    want = _per_image(eng.plan(H, W), x)
    bplan = eng.batch_plan(N, H, W)
    bplan.forward(x)
    got = _batch_result(bplan)
    for n, (g, w) in enumerate(zip(got, want)):
        assert w["count"] == 0
        _assert_same(g, w, n)


def test_batch_plan_equals_forward_plan_600x1000(params):
    """The benchmarked size: N = 4 at 600x1000, bf16x3, per-class NMS in the graph."""
    from frcnn_b200.engine import BatchPlan, ForwardPlan, PackedWeights
    H, W, N = 600, 1000, 4
    wts = PackedWeights(params, "bf16x3")
    plan1 = ForwardPlan(wts, H, W, anchors=ANCHORS, with_detect=True, det_conf=0.05)
    bplan = BatchPlan(wts, N, H, W, anchors=ANCHORS, with_detect=True, det_conf=0.05)
    x = _images(N, H, W, seed=0)
    want = _per_image(plan1, x)
    bplan.forward(x)
    bplan.forward(x)
    for n, (g, w) in enumerate(zip(_batch_result(bplan), want)):
        assert w["count"] > 0
        _assert_same(g, w, n)


def test_lane_pool_over_batch_plans(params):
    """LanePool keeps two batches in flight on two streams; every image equals its ForwardPlan result."""
    from frcnn_b200.engine import Engine, LanePool
    H, W, N = 96, 128, 2
    eng = Engine(params, precision="bf16x3", anchors=ANCHORS, with_detect=True, det_conf=0.05)
    plan1 = eng.plan(H, W)
    batches = [_images(N, H, W, seed=50 + 10 * i) for i in range(4)]
    want = [_per_image(plan1, b) for b in batches]
    pool = LanePool(eng.batch_plan(N, H, W), lanes=2)
    for rnd in range(0, 4, 2):
        pool.fork()
        used = [(i, pool.submit(i, batches[i])) for i in range(rnd, rnd + 2)]
        pool.join()
        for i, pl in used:
            for n, (g, w) in enumerate(zip(_batch_result(pl), want[i])):
                _assert_same(g, w, (i, n))


def test_batch_errors(params):
    """N < 1, an input of another shape, and a ResNet engine raise FrcnnError; so do bad batch calls of the C entries."""
    from frcnn_b200._lib import FrcnnError
    from frcnn_b200.engine import BatchPlan, Engine
    from frcnn_b200.resnet_engine import ResNetEngine
    ops = _ops()
    eng = Engine(params, precision="bf16", anchors=ANCHORS)
    for bad in (0, -1):
        with pytest.raises(FrcnnError):
            BatchPlan(eng.weights, bad, 64, 96, anchors=ANCHORS)
    bplan = eng.batch_plan(2, 64, 96)
    with pytest.raises(FrcnnError):
        bplan.forward(torch.zeros((3, 3, 64, 96), device="cuda"))
    with pytest.raises(FrcnnError):
        bplan.forward(torch.zeros((2, 3, 64, 98), device="cuda"))
    with pytest.raises(FrcnnError):
        eng.forward_batch(torch.zeros((3, 64, 96), device="cuda"))
    reng = ResNetEngine(orc.make_resnet_params(50, seed=5), 50, precision="bf16", anchors=ANCHORS, post_n=50)
    with pytest.raises(FrcnnError):
        reng.batch_plan(2, 64, 96)
    with pytest.raises(FrcnnError):
        reng.forward_batch(torch.zeros((2, 3, 64, 96), device="cuda"))
    xa = _act(torch.zeros((1, 8, 8, 64), device="cuda"), False)
    hi, lo = _weights(64, 64, 3, False, 1)
    bias = ops.pad_bias(torch.zeros(64, device="cuda"), 64)
    with pytest.raises(FrcnnError):
        ops.conv2d_batch(ops.Act(xa.hi[:0], None), hi, lo, bias, 3, True)
    with pytest.raises(FrcnnError):
        ops.linear_batch(_act(torch.zeros((2, 300, 64), device="cuda"), False), hi[:1, :, :64].contiguous(), None,
                         bias, True, 300)
