"""The conv kernel's TMA-store epilogue (csrc/conv_gemm_sm90.cu) checked bit for bit against the kernel's own fp32 output.

When one launch writes an fp32 output and bf16 outputs, both come from the same fp32 register values v: the fp32 values
leave through direct stores, the bf16 planes through the staged TMA tensor stores, as the exact split
hi = rn_bf16(v), lo = rn_bf16(v - hi) (v - hi is exact in fp32).  So at every live pixel the stored planes must equal the
split of the fp32 output bit for bit, whatever the accumulation order: the split oracle, assert_split_exact.  A swizzle,
box-origin, clipping or staging-reuse error fails it in one run, with no tolerance to hide in.  The fp32 output itself is
anchored to a float64 convolution of the exact operand values, and every launch asserts, through ops.conv_last_plan(),
the plan it was meant to reach.

Inputs are finite: the NaN payloads of __floats2bfloat162_rn and of torch's conversion differ."""
import pytest
import torch

from test_canvas_batch_gpu import _poison_like
from test_conv_gemm_coverage_gpu import (SMEM_BYTES, SMEM_FIXED, TOL_F32, assert_canary_intact, canary_view, cdiv, check_f32,
                                         conv_ref, make_conv, planes, pool_ref, rel_err, settings, stages_for)

pytestmark = pytest.mark.gpu

S16, S32 = 0x5A5A, 0x5A5A5A5A


@pytest.fixture(scope="module")
def ops():
    from frcnn_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def split_bf16(v):
    """pack_bf16x2's split of fp32 values: hi = rn_bf16(v), lo = rn_bf16(v - hi)."""
    hi = v.to(torch.bfloat16)
    return hi, (v - hi.float()).to(torch.bfloat16)


def assert_split_exact(y, y32, valid):
    """The split oracle.  y: Act [..., H, W, Cout]; y32: fp32 holding [..., H, W, >= Cout] in any shape; valid: bool
    [..., H, W], False outside an image's extent or at and past m_valid.  At every valid pixel the hi plane (and the lo
    plane, when present) is the split of y32[..., :Cout], bit for bit; at every other pixel every plane and y32 are +0."""
    shape = tuple(y.hi.shape)
    assert tuple(valid.shape) == shape[:-1], (tuple(valid.shape), shape)
    v = y32.reshape(shape[:-1] + (-1,))[..., :shape[-1]]
    for name, got, want in zip(("hi", "lo"), (y.hi, y.lo), split_bf16(v)):
        if got is None:
            continue
        bad = (bits(got) != bits(want)) & valid[..., None]
        if bad.any():
            i = tuple(bad.nonzero()[0].tolist())
            raise AssertionError("%s plane: %d of %d live values are not the split of the fp32 output; first at %s: "
                                 "stored %#06x, split %#06x of %r" % (name, int(bad.sum()), int(valid.sum()) * shape[-1], i,
                                                                      int(bits(got)[i]) & 0xFFFF,
                                                                      int(bits(want)[i]) & 0xFFFF, float(v[i])))
        assert not bits(got)[~valid].any(), "%s plane: a pixel outside the extent is not +0" % name
    assert not bits(v)[~valid].any(), "fp32 output: a pixel outside the extent is not +0"


def plan_of(BN, BK, x3, TH, TW, num_tiles, units, CG=1, stages=None):
    return dict(BN=BN, BK=BK, x3=int(x3), promote=0, CG=CG, TH=TH, TW=TW,
                stages=stages_for(BN, BK, x3) if stages is None else stages, grid=CG * min(num_tiles, units),
                num_tiles=num_tiles, n_parts=1, splits=1)


def block_k(Cin):
    return 64 if Cin >= 64 else (32 if Cin >= 32 else 16)


# ------------------------------------------------------------------------------- 1. box geometry
# (TH, TW, H, W): H - 1 is a multiple of TH (the last tile row holds one image row) and W is ragged for TW, so warpgroup
# 1's store box is partly outside the image in one tile and wholly outside it in another.  At TW = 128 the warpgroups
# split a row into halves: W mod 128 < 64 puts warpgroup 1's last box wholly outside, W mod 128 > 64 partly outside.
TILE_CASES = [(8, 16, 17, 37), (16, 8, 33, 21), (4, 32, 9, 70), (32, 4, 33, 11), (2, 64, 5, 150), (1, 128, 3, 150),
              (1, 128, 3, 230)]
# every (precision, BN) with an instantiation at BK = 64; Cout is an odd multiple of 32 below the N tile and ld_f32 > Cout,
# so a tile holds bf16 chunks, fp32-only chunks and (BN = 256) chunks past the covered columns
N_TILES = [("bf16", 64), ("bf16", 128), ("bf16", 256), ("bf16x3", 64), ("bf16x3", 128)]
COUT_LD = {64: (32, 64), 128: (96, 128), 256: (160, 192)}
GEOM_MAX_CTAS = 3          # every CTA reuses its staging tiles across several pixel tiles


def store_boxes(H, W, TH, TW):
    """(warpgroup, image pixels inside the box) of every bf16 TMA store box of an H x W image under a TH x TW tile."""
    bw, bh = min(TW, 64), max(64 // TW, 1)
    boxes = []
    for h0 in range(0, cdiv(H, TH) * TH, TH):
        for w0 in range(0, cdiv(W, TW) * TW, TW):
            for c in (0, 1):
                x, y = w0 + 64 * c % TW, h0 + 64 * c // TW
                boxes.append((c, max(0, min(W, x + bw) - x) * max(0, min(H, y + bh) - y)))
    return boxes


@pytest.mark.parametrize("precision,BN", N_TILES, ids=["%s-BN%d" % v for v in N_TILES])
@pytest.mark.parametrize("geom", TILE_CASES, ids=["%dx%d-H%d-W%d" % g for g in TILE_CASES])
def test_box_geometry_split_exact(ops, precision, BN, geom):
    """Every forced pixel tile x {bf16, bf16x3} x BN on a ragged image: the stored planes are the exact split of the fp32
    output, no byte outside the three outputs changes (views inside sentinel buffers, margins as in
    test_epilogue_stores_stay_inside_their_outputs), and the fp32 output matches float64."""
    TH, TW, H, W = geom
    boxes = store_boxes(H, W, TH, TW)
    assert (H - 1) % TH == 0 and W % TW
    if TW < 128 or W % TW > 64:
        assert any(c == 1 and 0 < n < 64 for c, n in boxes), boxes
    if TW < 128 or W % TW < 64:
        assert any(c == 1 and n == 0 for c, n in boxes), boxes
    Cout, ld = COUT_LD[BN]
    x3 = precision == "bf16x3"
    act, wh, wl, bias, ref = make_conv(ops, H, W, 64, Cout, 3, precision, seed=TILE_CASES.index(geom) * 8 + BN // 64 + x3,
                                       bias_pad=ld)
    margin_f32, margin_act = 128 * W * ld, 128 * W * Cout
    b32, y32 = canary_view(H * W * ld, torch.float32, margin_f32, S32)
    bh, yh = canary_view(H * W * Cout, torch.bfloat16, margin_act, S16)
    bl, yl = canary_view(H * W * Cout, torch.bfloat16, margin_act, S16) if x3 else (None, None)
    out = ops.Act(yh.view(H, W, Cout), yl.view(H, W, Cout) if x3 else None)
    with settings(ops, bn=BN, th=TH, tw=TW, max_ctas=GEOM_MAX_CTAS):
        ops.conv2d(act, wh, wl, bias, 3, False, out=out, out_f32=y32.view(H * W, ld), ld_f32=ld)
        plan = ops.conv_last_plan()
    torch.cuda.synchronize()
    assert plan == plan_of(BN, 64, x3, TH, TW, cdiv(H, TH) * cdiv(W, TW), GEOM_MAX_CTAS), plan
    assert_canary_intact(b32, H * W * ld, margin_f32, S32)
    assert_canary_intact(bh, H * W * Cout, margin_act, S16)
    if x3:
        assert_canary_intact(bl, H * W * Cout, margin_act, S16)
    assert_split_exact(out, y32, torch.ones((H, W), dtype=torch.bool, device="cuda"))
    check_f32(y32, ref, precision, Cout)


# ------------------------------------------------------------------------------- 2. batches and canvases
def live_mask(N, H, W, sizes, halvings):
    """bool [N, H, W]: the pixels inside each image's extent at this layer (every pixel without a canvas)."""
    live = torch.zeros((N, H, W), dtype=torch.bool, device="cuda")
    for n in range(N):
        h, w = (H, W) if sizes is None else (min(-(-e // (1 << halvings)), lim) for e, lim in zip(sizes[n], (H, W)))
        live[n, :h, :w] = True
    return live


def make_batch(ops, live, Cin, Cout, ksize, precision, seed, bias_pad=0):
    """make_conv for N images: the input is 0 outside every extent (as the previous canvas layer leaves it), and the
    float64 reference is [N, H, W, Cout]."""
    N, H, W = live.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((N, H, W, Cin), device="cuda", generator=g).masked_fill(~live[..., None], 0.0)
    w = torch.randn((ksize * ksize, Cout, Cin), device="cuda", generator=g) * (1.0 / (ksize * ksize * Cin)) ** 0.5
    b = torch.randn((Cout,), device="cuda", generator=g) * 0.5
    xh, xl, xv = planes(x, precision)
    wh, wl, wv = planes(w, precision)
    ref = torch.stack([conv_ref(xv[n], wv, b.double(), ksize) for n in range(N)])
    return ops.Act(xh, xl), wh, wl, ops.pad_bias(b, max(Cout, bias_pad)), ref


def poisoned(N, shape, dtype):
    """A poisoned buffer of N + 1 images and the view of its first N: image N is the tail no store may reach."""
    buf = _poison_like(torch.empty((N + 1,) + tuple(shape), dtype=dtype, device="cuda"))
    return buf, buf[:N]


def assert_tails_intact(bufs, tails, N):
    for buf, tail in zip(bufs, tails):
        assert torch.equal(bits(buf[N]), bits(tail)), "a store reached past the last image"


def extents_of(sizes):
    return None if sizes is None else torch.tensor(sizes, dtype=torch.int32, device="cuda")


def check_f32_live(y32, ref, live, precision):
    N, H, W, Cout = ref.shape
    got = y32.reshape(N, H, W, -1)
    assert rel_err(got[..., :Cout][live], ref[live]) < TOL_F32[precision]
    assert not got[..., Cout:].any(), "columns [Cout, ld_f32) must be zero"


# (N, H, W, Cin, Cout, ld_f32, ksize, precision, relu, BN, (TH, TW), CG, halvings, image sizes in input pixels or None)
BATCH_CASES = {
    "n2-batch-bf16x3": (2, 19, 37, 64, 96, 128, 3, "bf16x3", False, 128, (8, 16), 1, 0, None),
    "n5-batch-1x1-bk16-bf16": (5, 9, 70, 16, 32, 64, 1, "bf16", False, 64, (4, 32), 1, 0, None),
    "n3-canvas-halvings-bf16": (3, 23, 41, 64, 160, 160, 3, "bf16", True, 256, (16, 8), 1, 2, [(92, 164), (50, 97), (3, 1)]),
    # 9 pixel tiles per image, 45 in all: the last CTA pair's second CTA gets tile_origin's clamped past-the-end tile
    "n5-canvas-cg2-odd-tiles-bf16x3": (5, 17, 37, 64, 64, 64, 3, "bf16x3", True, 64, (8, 16), 2, 0,
                                       [(17, 37), (9, 16), (0, 0), (17, 1), (1, 37)]),
    # half-row boxes: extents end inside warpgroup 0's box (40), inside warpgroup 1's (100) and in the second column block
    "n3-canvas-1x128-bf16": (3, 5, 200, 64, 96, 128, 3, "bf16", False, 128, (1, 128), 1, 0, [(5, 40), (4, 150), (3, 100)]),
}


@pytest.mark.parametrize("case", list(BATCH_CASES))
def test_batch_and_canvas_split_exact(ops, sms, case):
    """frcnn_conv2d_batch(_ext) into poisoned outputs: in every image the planes are the split of the fp32 output inside
    the extent and +0 outside it, no poison is left, the image after the last one is untouched, and the fp32 output
    matches float64."""
    N, H, W, Cin, Cout, ld, k, precision, relu, BN, (TH, TW), CG, halv, sizes = BATCH_CASES[case]
    x3 = precision == "bf16x3"
    live = live_mask(N, H, W, sizes, halv)
    act, wh, wl, bias, ref = make_batch(ops, live, Cin, Cout, k, precision, seed=101 + len(case), bias_pad=ld)
    bh, yh = poisoned(N, (H, W, Cout), torch.bfloat16)
    bl, yl = poisoned(N, (H, W, Cout), torch.bfloat16) if x3 else (None, None)
    b32, y32 = poisoned(N, (H * W, ld), torch.float32)
    bufs = [b for b in (bh, bl, b32) if b is not None]
    tails = [b[N].clone() for b in bufs]
    out = ops.Act(yh, yl)
    with settings(ops, bn=BN, th=TH, tw=TW, cg=CG):
        ops.conv2d_batch(act, wh, wl, bias, k, relu, out=out, out_f32=y32.reshape(N * H * W, ld), ld_f32=ld,
                         extents=extents_of(sizes), halvings=halv)
        plan = ops.conv_last_plan()
    torch.cuda.synchronize()
    m_tiles = N * cdiv(H, TH) * cdiv(W, TW)
    assert plan == plan_of(BN, block_k(Cin), x3, TH, TW, cdiv(m_tiles, CG) * cdiv(ld, BN), sms // CG, CG=CG), plan
    if CG == 2:
        assert m_tiles % 2 == 1
    assert_tails_intact(bufs, tails, N)
    assert_split_exact(out, y32, live)
    check_f32_live(y32, ref.clamp_min(0) if relu else ref, live, precision)


# (N, H, W, Cin, Cout, ksize, precision, relu, res_lo, BN, (TH, TW), halvings, image sizes in input pixels or None);
# relu off is the trainers' residual dgrad sum
RES_CASES = {
    "relu-canvas-bf16x3-res-hi-lo": (3, 15, 22, 64, 64, 3, "bf16x3", True, True, 64, (8, 16), 1, [(30, 44), (17, 9), (2, 44)]),
    "relu-off-batch-bf16-res-hi": (2, 13, 21, 64, 128, 1, "bf16", False, False, 128, (4, 32), 0, None),
}


@pytest.mark.parametrize("case", list(RES_CASES))
def test_residual_batch_split_exact(ops, sms, case):
    """frcnn_conv2d_res_batch(_ext) has no fp32 output, so the fp32 values come from frcnn_conv2d_batch(_ext) of the same
    layer under the same plan (relu off): the kernel then adds res_hi and res_lo with round-to-nearest fp32 adds, applies
    the ReLU and zeroes pixels outside the extent, which torch repeats exactly in fp32.  The stored planes are the split
    of that, bit for bit."""
    N, H, W, Cin, Cout, k, precision, relu, res_lo, BN, (TH, TW), halv, sizes = RES_CASES[case]
    x3 = precision == "bf16x3"
    live = live_mask(N, H, W, sizes, halv)
    act, wh, wl, bias, ref = make_batch(ops, live, Cin, Cout, k, precision, seed=201 + len(case))
    g = torch.Generator(device="cuda").manual_seed(202)
    rh, rl, _ = planes(torch.randn((N, H, W, Cout), device="cuda", generator=g), "bf16x3")
    res = ops.Act(rh, rl if res_lo else None)
    ext = extents_of(sizes)
    y32 = torch.empty((N * H * W, Cout), device="cuda")
    bh, yh = poisoned(N, (H, W, Cout), torch.bfloat16)
    bl, yl = poisoned(N, (H, W, Cout), torch.bfloat16) if x3 else (None, None)
    bufs = [b for b in (bh, bl) if b is not None]
    tails = [b[N].clone() for b in bufs]
    out = ops.Act(yh, yl)
    with settings(ops, bn=BN, th=TH, tw=TW):
        ops.conv2d_batch(act, wh, wl, bias, k, False, out_act=False, out_f32=y32, ld_f32=Cout, extents=ext, halvings=halv)
        plan32 = ops.conv_last_plan()
        ops.conv2d_res_batch(act, wh, wl, bias, k, relu, res, out=out, extents=ext, halvings=halv)
        plan = ops.conv_last_plan()
    torch.cuda.synchronize()
    want_plan = plan_of(BN, block_k(Cin), x3, TH, TW, N * cdiv(H, TH) * cdiv(W, TW) * cdiv(Cout, BN), sms)
    assert plan32 == want_plan and plan == want_plan, (plan32, plan)
    assert_tails_intact(bufs, tails, N)
    check_f32_live(y32, ref, live, precision)
    v = y32.view(N, H, W, Cout) + rh.float()
    if res_lo:
        v = v + rl.float()
    if relu:
        v = v.clamp_min(0.0)
    v = torch.where(live[..., None], v, torch.zeros_like(v))
    assert_split_exact(out, v, live)


# ------------------------------------------------------------------------------- 3. staging reuse under hard schedules
# Layers whose epilogue dominates: one k-block per tile (1x1, Cin = 16), a short 1x1 main loop (Cin = 64), eight 32-channel
# chunks per tile back to back (BN = 256), and both planes per chunk (bf16x3).  (H, W, Cin, Cout, ksize, precision, BN, tile)
STAGING_LAYERS = {
    "1x1-cin16-bf16x3-bn128": (48, 240, 16, 128, 1, "bf16x3", 128, (1, 128)),
    "1x1-cin64-bf16-bn256": (48, 240, 64, 256, 1, "bf16", 256, (8, 16)),
    "3x3-cin64-bf16-bn256": (48, 240, 64, 256, 3, "bf16", 256, (4, 32)),
    "3x3-cin64-bf16x3-bn128": (48, 240, 64, 128, 3, "bf16x3", 128, (16, 8)),
}
MAX_RESERVE = 96 * 1024                  # frcnn_conv2d_set_smem_reserve's cap


def two_stage_reserve(BN, BK, x3):
    """The largest shared-memory reserve (at most 96 KB) that leaves two stages, or 96 KB where no reserve can."""
    stage = (2 if x3 else 1) * (128 + BN) * BK * 2
    return min(SMEM_BYTES - SMEM_FIXED - 2 * stage, MAX_RESERVE)


@pytest.mark.parametrize("layer", list(STAGING_LAYERS))
def test_staging_reuse_schedules_split_exact(ops, sms, layer):
    """Each layer under the default schedule, one CTA walking every tile (max_ctas = 1: the staging tile is reused while
    earlier stores still drain), the reserve that leaves two stages, CTA pairs (BK = 64 only; also one pair walking every
    tile) and programmatic dependent launch: each launch once, into poisoned outputs.  Every run passes the split oracle,
    and every schedule is bit-identical to the default one, whose fp32 output matches float64.  The 1x1 Cin = 16 layer
    cannot get down to two stages under the 96 KB reserve cap; it runs at 96 KB."""
    H, W, Cin, Cout, k, precision, BN, (TH, TW) = STAGING_LAYERS[layer]
    x3 = precision == "bf16x3"
    BK = block_k(Cin)
    act, wh, wl, bias, ref = make_conv(ops, H, W, Cin, Cout, k, precision, seed=301 + len(layer))
    every = torch.ones((H, W), dtype=torch.bool, device="cuda")

    def run(**s):
        y = ops.Act(_poison_like(torch.empty((H, W, Cout), dtype=torch.bfloat16, device="cuda")),
                    _poison_like(torch.empty((H, W, Cout), dtype=torch.bfloat16, device="cuda")) if x3 else None)
        y32 = _poison_like(torch.empty((H * W, Cout), device="cuda"))
        with settings(ops, bn=BN, th=TH, tw=TW, **s):
            ops.conv2d(act, wh, wl, bias, k, False, out=y, out_f32=y32, ld_f32=Cout)
            plan = ops.conv_last_plan()
        torch.cuda.synchronize()
        assert_split_exact(y, y32, every)
        return [t for t in (y.hi, y.lo, y32) if t is not None], plan

    m_tiles = cdiv(H, TH) * cdiv(W, TW)
    n_tiles = cdiv(Cout, BN)
    want, base_plan = run()
    assert base_plan == plan_of(BN, BK, x3, TH, TW, m_tiles * n_tiles, sms), base_plan
    check_f32(want[-1], ref, precision, Cout)
    reserve = two_stage_reserve(BN, BK, x3)
    variants = [("max_ctas=1", dict(max_ctas=1), dict(grid=1)),
                ("reserve=%d" % reserve, dict(reserve=reserve), dict(stages=stages_for(BN, BK, x3, reserve))),
                ("pdl=1", dict(pdl=1), {})]
    if BK == 64:
        pairs = cdiv(m_tiles, 2) * n_tiles
        variants += [("CG=2", dict(cg=2), dict(CG=2, num_tiles=pairs, grid=2 * min(pairs, sms // 2))),
                     ("CG=2,max_ctas=2", dict(cg=2, max_ctas=2), dict(CG=2, num_tiles=pairs, grid=2))]
    if layer != "1x1-cin16-bf16x3-bn128":
        assert stages_for(BN, BK, x3, reserve) == 2
    for name, s, expect in variants:
        got, plan = run(**s)
        assert plan == dict(base_plan, **expect), (name, plan)
        for i, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(bits(a), bits(b)), (name, i)


# ------------------------------------------------------------------------------- 4. visibility to the next kernel
@pytest.mark.parametrize("mode", ["eager-pdl0", "eager-pdl1", "graph-pdl1"])
def test_tma_stores_visible_to_next_kernel(ops, sms, mode):
    """Convolution B reads convolution A's TMA-stored output straight after it on one stream: eagerly with programmatic
    dependent launch off and on, and replayed from a captured CUDA graph.  A runs on two CTAs, so its last tiles' stores
    are in flight when it exits; every output is poisoned before the run, so a read of A's output before its stores
    landed shows.  Both launches pass the split oracle and float64 (B's reference is the float64 convolution of A's
    stored value).  The one comparison with another launch of the same path: B's outputs equal, bit for bit, B run after a
    full synchronise on a clone of A's output."""
    H, W, C = 40, 64, 64
    act, wh, wl, bias, ref_a = make_conv(ops, H, W, C, C, 3, "bf16x3", seed=401, relu_input=True)
    g = torch.Generator(device="cuda").manual_seed(402)
    whb, wlb, wvb = planes(torch.randn((9, C, C), device="cuda", generator=g) * (1.0 / (9 * C)) ** 0.5, "bf16x3")
    bb = torch.randn((C,), device="cuda", generator=g) * 0.5
    bias_b = ops.pad_bias(bb, C)

    def new_act():
        return ops.Act(torch.empty((H, W, C), dtype=torch.bfloat16, device="cuda"),
                       torch.empty((H, W, C), dtype=torch.bfloat16, device="cuda"))
    ya, yb = new_act(), new_act()
    ya32, yb32 = torch.empty((H * W, C), device="cuda"), torch.empty((H * W, C), device="cuda")

    def poison():
        for t in (ya.hi, ya.lo, ya32, yb.hi, yb.lo, yb32):
            t.copy_(_poison_like(t))

    def chain(pdl):
        with settings(ops, max_ctas=2, pdl=pdl):
            ops.conv2d(act, wh, wl, bias, 3, True, out=ya, out_f32=ya32, ld_f32=C)
            plan_a = ops.conv_last_plan()
            ops.set_conv_max_ctas(0)
            ops.conv2d(ya, whb, wlb, bias_b, 3, True, out=yb, out_f32=yb32, ld_f32=C)
            plan_b = ops.conv_last_plan()
        return plan_a, plan_b

    # the reference: A, a full synchronise, then B on a copy of A's output
    poison()
    chain(0)
    torch.cuda.synchronize()
    a_copy = ops.Act(ya.hi.clone(), ya.lo.clone())
    ref_b = ops.conv2d(a_copy, whb, wlb, bias_b, 3, True, ld_f32=C)
    ref_b = [ref_b[0].hi, ref_b[0].lo, ref_b[1]]
    ref_plan_b = ops.conv_last_plan()
    torch.cuda.synchronize()

    pdl = int(mode.endswith("pdl1"))
    if mode.startswith("graph"):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            plan_a, plan_b = chain(pdl)
        poison()
        graph.replay()
    else:
        poison()
        plan_a, plan_b = chain(pdl)
    torch.cuda.synchronize()
    assert plan_a["grid"] == 2 and plan_a["num_tiles"] >= 8, plan_a
    assert plan_b == ref_plan_b and plan_b["grid"] == min(plan_b["num_tiles"], sms), (plan_b, ref_plan_b)
    every = torch.ones((H, W), dtype=torch.bool, device="cuda")
    assert_split_exact(ya, ya32, every)
    assert_split_exact(yb, yb32, every)
    check_f32(ya32, ref_a.clamp_min(0), "bf16x3", C)
    ref_b64 = conv_ref(ya.hi.double() + ya.lo.double(), wvb, bb.double(), 3).clamp_min(0)
    check_f32(yb32, ref_b64, "bf16x3", C)
    for i, (a, b) in enumerate(zip((yb.hi, yb.lo, yb32), ref_b)):
        assert torch.equal(bits(a), bits(b)), (mode, i)


# ------------------------------------------------------------------------------- 5. the direct-store outputs
@pytest.mark.parametrize("precision,BN,Cout", [("bf16", 256, 160), ("bf16x3", 128, 96)])
def test_direct_store_outputs_split_exact(ops, sms, precision, BN, Cout):
    """The two outputs that still leave through direct stores.  The fused-pool launch cannot write fp32, so an fp32-only
    launch and an unpooled fp32 + bf16 launch of the same layer run beside it, all three forced to the same N tile and the
    8 x 16 pixel tile (the same arithmetic).  The pooled planes are the split of the ceil-mode 2 x 2 max of the fp32
    output (the kernel takes the max in fp32, then splits it); the fp32-only output matches float64 and is bit-identical
    to the fp32 output written beside the bf16 planes, which pass the split oracle; no byte around the fp32-only and the
    pooled outputs changes.  H = 8*4 + 1 and W = 16*3 + 1: the last pool windows hold one pixel."""
    H, W = 33, 49
    x3 = precision == "bf16x3"
    act, wh, wl, bias, ref = make_conv(ops, H, W, 64, Cout, 3, precision, seed=501 + BN, relu_input=True)
    oh, ow = cdiv(H, 2), cdiv(W, 2)
    margin = 128 * W * Cout
    b32, y32 = canary_view(H * W * Cout, torch.float32, margin, S32)
    bh, yh = canary_view(oh * ow * Cout, torch.bfloat16, margin, S16)
    bl, yl = canary_view(oh * ow * Cout, torch.bfloat16, margin, S16) if x3 else (None, None)
    pooled = ops.Act(yh.view(oh, ow, Cout), yl.view(oh, ow, Cout) if x3 else None)
    plans = []
    with settings(ops, bn=BN, th=8, tw=16):
        ops.conv2d(act, wh, wl, bias, 3, True, out_act=False, out_f32=y32.view(H * W, Cout), ld_f32=Cout)
        plans.append(ops.conv_last_plan())
        yu, yu32 = ops.conv2d(act, wh, wl, bias, 3, True, ld_f32=Cout)
        plans.append(ops.conv_last_plan())
        ops.conv2d(act, wh, wl, bias, 3, True, out=pooled, fuse_pool=True)
        plans.append(ops.conv_last_plan())
    torch.cuda.synchronize()
    want_plan = plan_of(BN, 64, x3, 8, 16, cdiv(H, 8) * cdiv(W, 16), sms)
    assert all(p == want_plan for p in plans), plans
    assert_canary_intact(b32, H * W * Cout, margin, S32)
    assert_canary_intact(bh, oh * ow * Cout, margin, S16)
    if x3:
        assert_canary_intact(bl, oh * ow * Cout, margin, S16)
    check_f32(y32, ref.clamp_min(0), precision, Cout)
    assert torch.equal(bits(y32.view(H * W, Cout)), bits(yu32))
    assert_split_exact(yu, yu32, torch.ones((H, W), dtype=torch.bool, device="cuda"))
    assert_split_exact(pooled, pool_ref(y32.view(H, W, Cout)), torch.ones((oh, ow), dtype=torch.bool, device="cuda"))
