"""The Hopper conv/GEMM kernel (csrc/conv_gemm_sm90.cu) across its whole dispatch table, its persistent schedule and the
head's production plans.

Every dense result is compared with a float64 product of the exact operand values (bf16 hi + lo for bf16x3, bf16 for
single pass), computed with torch on the GPU.  Every launch asserts, through ops.conv_last_plan(), the instantiation,
pixel tile, pipeline depth, grid and split plan it was meant to reach: a planner that silently narrowed a forced setting
would make the test fail instead of quietly testing something else."""
import contextlib
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONV_SRC = os.path.join(ROOT, "chainer-faster-rcnn_b200", "csrc", "conv_gemm_sm90.cu")

SMEM_BYTES = 227 * 1024                   # dynamic shared memory of one H100 CTA
SMEM_FIXED = 1024 + 512 + 2 * 64 * 36 * 4  # alignment slack + barriers + the epilogue's transpose tiles
TOL_F32 = {"bf16x3": 3e-5, "bf16": 1e-5}  # fp32 output, relative to the max-norm of the reference
TOL_ACT = {"bf16x3": 5e-5, "bf16": 6e-3}  # stored bf16 hi (+ lo) activations


def cdiv(a, b):
    return -(-a // b)


def stages_for(BN, BK, x3, reserve=0):
    """Pipeline stages launch_conv gives an instantiation (no resident weights)."""
    stage = (2 if x3 else 1) * (128 + BN) * BK * 2
    return min(20, (SMEM_BYTES - reserve - SMEM_FIXED) // stage)


@pytest.fixture(scope="module")
def ops():
    from frcnn_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def settings(ops, bn=0, th=0, tw=0, cg=0, max_ctas=0, reserve=0, pdl=None):
    """The per-thread launch overrides of the conv kernel, restored to their defaults on exit."""
    ops.set_conv_tile(bn, th, tw)
    ops.set_conv_cta_group(cg)
    ops.set_conv_max_ctas(max_ctas)
    ops.set_conv_smem_reserve(reserve)
    if pdl is not None:
        ops.set_programmatic_launch(pdl)
    try:
        yield
    finally:
        ops.set_conv_tile(0, 0, 0)
        ops.set_conv_cta_group(0)
        ops.set_conv_max_ctas(0)
        ops.set_conv_smem_reserve(0)
        ops.set_programmatic_launch(-1)


def planes(x, precision):
    """float32 CUDA tensor -> (hi, lo or None) bf16 operand planes and the exact float64 value they hold."""
    hi = x.to(torch.bfloat16)
    if precision == "bf16":
        return hi, None, hi.double()
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo, hi.double() + lo.double()


def conv_ref(xv, wv, bias, ksize):
    """float64 stride-1 'same' convolution: xv [H,W,Cin], wv [taps,Cout,Cin] (tap = r*ksize+s), bias [Cout] -> [H,W,Cout]."""
    H, W, Cin = xv.shape
    if ksize == 1:
        return (xv.reshape(H * W, Cin) @ wv[0].T).reshape(H, W, -1) + bias
    xp = torch.nn.functional.pad(xv, (0, 0, 1, 1, 1, 1))
    out = bias.expand(H, W, wv.shape[1]).clone()
    for r in range(3):
        for s in range(3):
            out += (xp[r:r + H, s:s + W].reshape(H * W, Cin) @ wv[3 * r + s].T).reshape(H, W, -1)
    return out


def pool_ref(ref):
    """F.MaxPooling2D(2, 2) ceil mode of an [H,W,C] map."""
    return torch.nn.functional.max_pool2d(ref.permute(2, 0, 1)[None], 2, 2, ceil_mode=True)[0].permute(1, 2, 0)


def rel_err(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


def act_value(y):
    return y.hi.double() + (y.lo.double() if y.lo is not None else 0)


def make_conv(ops, H, W, Cin, Cout, ksize, precision, seed, relu_input=False, bias_pad=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((H, W, Cin), device="cuda", generator=g)
    if relu_input:
        x = x.clamp_min(0)
    w = torch.randn((ksize * ksize, Cout, Cin), device="cuda", generator=g) * (1.0 / (ksize * ksize * Cin)) ** 0.5
    b = torch.randn((Cout,), device="cuda", generator=g) * 0.5
    xh, xl, xv = planes(x, precision)
    wh, wl, wv = planes(w, precision)
    return ops.Act(xh, xl), wh, wl, ops.pad_bias(b, max(Cout, bias_pad)), conv_ref(xv, wv, b.double(), ksize)


def check_f32(y32, ref, precision, Cout):
    H, W, _ = ref.shape
    got = y32.view(H, W, -1)
    err = rel_err(got[:, :, :Cout], ref)
    assert err < TOL_F32[precision], ("f32", err)
    assert not got[:, :, Cout:].any(), "columns [Cout, ld_f32) must be zero"
    return err


def check_act(y, ref, precision):
    err = rel_err(act_value(y), ref)
    assert err < TOL_ACT[precision], ("act", err)
    return err


# ------------------------------------------------------------------------------- a. the dispatch table
# (BN, BK, x3, promote, CG): one line per FRCNN_DISPATCH(...) of conv2d_impl, in source order
DISPATCH = [
    (256, 64, False, False, 1), (256, 64, False, False, 2), (128, 64, False, False, 1), (128, 64, False, False, 2),
    (64, 64, False, False, 1), (64, 64, False, False, 2), (128, 64, True, False, 1), (128, 64, True, False, 2),
    (64, 64, True, False, 1), (64, 64, True, False, 2), (128, 64, False, True, 1), (128, 64, False, True, 2),
    (64, 64, False, True, 1), (64, 64, False, True, 2), (64, 64, True, True, 1), (64, 64, True, True, 2),
    (128, 32, False, False, 1), (64, 32, False, False, 1), (128, 32, True, False, 1), (64, 32, True, False, 1),
    (256, 16, False, False, 1), (128, 16, False, False, 1), (64, 16, False, False, 1), (128, 16, True, False, 1),
    (64, 16, True, False, 1),
]
# (H, W, Cin, ksize, TH, TW) per instantiation.  H and W are ragged for the pixel tile.  Cin picks BK (16 / 32 / >= 64);
# the long-K (promote) lines are a 1x1 layer of 259 k-blocks, so the last 8-k-block chunk has 3.  The k-blocks per
# tile are never a multiple of the stage count, so the ring's stage and phase carry into the next tile at an offset.
# CTA-pair lines have an odd number of pixel tiles (the last pair has a CTA past the last tile).
K_PROMOTE = 64 * 259
MATRIX_SHAPE = {
    (256, 64, False, False, 1): (19, 37, 64, 3, 8, 16), (256, 64, False, False, 2): (19, 37, 64, 3, 8, 16),
    (128, 64, False, False, 1): (35, 19, 64, 3, 16, 8), (128, 64, False, False, 2): (35, 19, 64, 3, 16, 8),
    (64, 64, False, False, 1): (9, 70, 64, 3, 4, 32), (64, 64, False, False, 2): (9, 70, 64, 3, 4, 32),
    (128, 64, True, False, 1): (5, 150, 320, 1, 2, 64), (128, 64, True, False, 2): (5, 150, 320, 1, 2, 64),
    (64, 64, True, False, 1): (11, 19, 64, 3, 32, 4), (64, 64, True, False, 2): (11, 19, 64, 3, 32, 4),
    (128, 64, False, True, 1): (13, 21, K_PROMOTE, 1, 16, 8), (128, 64, False, True, 2): (13, 21, K_PROMOTE, 1, 16, 8),
    (64, 64, False, True, 1): (5, 150, K_PROMOTE, 1, 2, 64), (64, 64, False, True, 2): (5, 150, K_PROMOTE, 1, 2, 64),
    (64, 64, True, True, 1): (7, 40, K_PROMOTE, 1, 8, 16), (64, 64, True, True, 2): (7, 40, K_PROMOTE, 1, 8, 16),
    (128, 32, False, False, 1): (19, 37, 32, 3, 8, 16), (64, 32, False, False, 1): (35, 19, 32, 3, 16, 8),
    (128, 32, True, False, 1): (13, 70, 32, 3, 4, 32), (64, 32, True, False, 1): (5, 150, 32, 3, 2, 64),
    (256, 16, False, False, 1): (19, 37, 16, 3, 8, 16), (128, 16, False, False, 1): (11, 19, 16, 3, 32, 4),
    (64, 16, False, False, 1): (13, 21, 16, 3, 16, 8), (128, 16, True, False, 1): (35, 19, 16, 3, 16, 8),
    (64, 16, True, False, 1): (13, 70, 16, 3, 4, 32),
}
# Cout is not a multiple of BN (a partial N tile: the weight TMA zero-fills rows >= Cout) and ld_f32 > Cout is not a
# multiple of BN either (the epilogue stops at the last covered 32-column chunk)
MATRIX_COUT_LD = {256: (288, 320), 128: (160, 192), 64: (96, 160)}
MATRIX_MAX_CTAS = 3


def dispatch_id(inst):
    BN, BK, x3, promote, CG = inst
    return "BN%d-BK%d-%s%s-CG%d" % (BN, BK, "bf16x3" if x3 else "bf16", "-promote" if promote else "", CG)


def parse_dispatch_table(path=CONV_SRC):
    """The (BN, BK, x3, promote, CG) of every FRCNN_DISPATCH(...) line of conv2d_impl."""
    txt = open(path).read()
    rows = re.findall(r"^\s*FRCNN_DISPATCH\((\d+),\s*(\d+),\s*(true|false),\s*(true|false),\s*(\d+)\)", txt, flags=re.M)
    return [(int(a), int(b), c == "true", d == "true", int(e)) for a, b, c, d, e in rows]


@pytest.mark.gpu
@pytest.mark.parametrize("inst", DISPATCH, ids=dispatch_id)
def test_dispatch_instantiation_vs_float64(ops, inst):
    BN, BK, x3, promote, CG = inst
    H, W, Cin, k, TH, TW = MATRIX_SHAPE[inst]
    Cout, ld = MATRIX_COUT_LD[BN]
    precision = "bf16x3" if x3 else "bf16"
    act, wh, wl, bias, ref = make_conv(ops, H, W, Cin, Cout, k, precision, seed=DISPATCH.index(inst), bias_pad=ld)
    with settings(ops, bn=BN, th=TH, tw=TW, cg=CG, max_ctas=MATRIX_MAX_CTAS):
        y, y32 = ops.conv2d(act, wh, wl, bias, k, False, ld_f32=ld)
        plan = ops.conv_last_plan()
    torch.cuda.synchronize()
    num_tiles = cdiv(cdiv(H, TH) * cdiv(W, TW), CG) * cdiv(ld, BN)
    units = max(MATRIX_MAX_CTAS // CG, 1)
    assert plan == dict(BN=BN, BK=BK, x3=int(x3), promote=int(promote), CG=CG, TH=TH, TW=TW, stages=stages_for(BN, BK, x3),
                        grid=CG * min(num_tiles, units), num_tiles=num_tiles, n_parts=1, splits=1)
    kb = k * k * cdiv(Cin, BK)
    assert kb % plan["stages"] != 0 and num_tiles >= 2 * units and H % TH and W % TW and Cout % BN and ld % BN
    e32 = check_f32(y32, ref, precision, Cout)
    ea = check_act(y, ref, precision)
    print("%s: f32 err %.3g, act err %.3g" % (dispatch_id(inst), e32, ea))


# ------------------------------------------------------------------------------- b. schedule invariance (bit-exact)
def schedule_variants(cg2_allowed, reserve2):
    """(name, settings, expectation) of launch settings that must not change a tile's arithmetic."""
    v = [("max_ctas=%d" % m, dict(max_ctas=m), {}) for m in (1, 5, 67)]
    v.append(("reserve=%d" % reserve2, dict(reserve=reserve2), {"stages": 2}))
    if cg2_allowed:
        v.append(("CG=2", dict(cg=2), {"CG": 2}))
        v.append(("CG=2,max_ctas=5", dict(cg=2, max_ctas=5), {"CG": 2, "grid": 4}))
    v.append(("pdl=1", dict(pdl=1), {}))
    v.append(("pdl=0", dict(pdl=0), {}))
    return v


def assert_schedule_invariant(ops, run, base_settings, cg2_allowed, reserve2):
    with settings(ops, **base_settings):
        want = run()
        base_plan = ops.conv_last_plan()
        again = run()                               # a repeated launch
    assert all(torch.equal(a, b) for a, b in zip(want, again))
    assert base_plan["stages"] > 2 and base_plan["CG"] == 1
    for name, s, expect in schedule_variants(cg2_allowed, reserve2):
        with settings(ops, **dict(base_settings, **s)):
            got = run()
            plan = ops.conv_last_plan()
        torch.cuda.synchronize()
        for key in ("BN", "BK", "x3", "promote", "TH", "TW", "n_parts", "splits"):
            assert plan[key] == base_plan[key], (name, key, plan, base_plan)
        units = s.get("max_ctas", 0) or base_plan["grid"]
        if "max_ctas" in s and "cg" not in s:
            assert plan["grid"] == min(units, base_plan["num_tiles"]), (name, plan)
        for key, val in expect.items():
            assert plan[key] == val, (name, key, plan)
        for i, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), (name, i, (a.float() - b.float()).abs().max().item())


@pytest.mark.gpu
def test_schedule_invariance_bf16_bn256_fused_pool(ops):
    """conv3_3-like: bf16, BN = 256, fused 2x2 pool."""
    act, wh, wl, bias, ref = make_conv(ops, 37, 45, 256, 256, 3, "bf16", seed=31, relu_input=True)

    def run():
        y, _ = ops.conv2d(act, wh, wl, bias, 3, True, fuse_pool=True)
        return [y.hi]
    assert_schedule_invariant(ops, run, dict(bn=256), True, 80 * 1024)
    with settings(ops, bn=256):
        y = run()
        assert ops.conv_last_plan()["BN"] == 256
    assert rel_err(y[0], pool_ref(ref.clamp_min(0))) < TOL_ACT["bf16"]


@pytest.mark.gpu
def test_schedule_invariance_bf16x3_bn128_conv5(ops):
    """conv5-like: bf16x3 at BN = 128 (conv5's plan at the 600 x 1000 input; this smaller map alone would plan 64),
    bf16 hi / lo and fp32 outputs."""
    act, wh, wl, bias, ref = make_conv(ops, 19, 25, 512, 512, 3, "bf16x3", seed=32, relu_input=True)

    def run():
        y, y32 = ops.conv2d(act, wh, wl, bias, 3, False, ld_f32=512)
        return [y.hi, y.lo, y32]
    assert_schedule_invariant(ops, run, dict(bn=128), True, 48 * 1024)
    with settings(ops, bn=128):
        y = run()
        assert ops.conv_last_plan()["BN"] == 128
    check_f32(y[2], ref, "bf16x3", 512)


@pytest.mark.gpu
def test_schedule_invariance_bf16x3_promote_gemm(ops):
    """A long-K 1x1 GEMM in bf16x3: (64, 64, bf16x3, promote)."""
    act, wh, wl, bias, ref = make_conv(ops, 1, 300, K_PROMOTE, 192, 1, "bf16x3", seed=33)

    def run():
        y, y32 = ops.conv2d(act, wh, wl, bias, 1, False, ld_f32=192)
        return [y.hi, y.lo, y32]
    assert_schedule_invariant(ops, run, {}, True, 80 * 1024)
    y = run()
    p = ops.conv_last_plan()
    assert (p["BN"], p["x3"], p["promote"]) == (64, 1, 1)
    check_f32(y[2], ref, "bf16x3", 192)


@pytest.mark.gpu
@pytest.mark.parametrize("groups", [1, 9])
def test_schedule_invariance_gemm_nt_splitk(ops, groups):
    """Split-K GEMM mode (the training weight gradients), bf16x3: several parts per launch, CTA pairs included."""
    from frcnn_b200 import train_ops as tops
    M, N, K, splits = (300, 256, 64 * 40, 3) if groups == 1 else (256, 128, 64 * 12, 2)
    g = torch.Generator(device="cuda").manual_seed(34 + groups)
    a_hi, a_lo = tops.split_bf16(torch.randn((M, K), device="cuda", generator=g))
    b_hi, b_lo = tops.split_bf16(torch.randn(((3, N, K) if groups == 9 else (N, K)), device="cuda", generator=g))

    def run():
        return [tops.gemm_nt_splitk(a_hi, a_lo, b_hi, b_lo, groups=groups, row_stride=40, splits=splits)]
    assert_schedule_invariant(ops, run, {}, True, 48 * 1024)
    run()
    p = ops.conv_last_plan()
    assert p["n_parts"] == groups * splits and p["splits"] == splits


# ------------------------------------------------------------------------------- c. the head's production plans
def plan_linear(R, K, N, sms):
    """frcnn_linear's plan (linear_swapab.cu plan_linear) followed by conv2d_impl's register cap on the N tile."""
    ld = cdiv(R, 32) * 32
    bn, best = 128, -1
    for c in (256, 128, 64):
        padded = cdiv(ld, c) * c
        if best < 0 or padded < best:
            best, bn = padded, c
    kb = K // 64
    base = cdiv(N, 128) * cdiv(ld, bn)
    red_cost = cdiv(N, 128) * 128 * ld * 8.0 / 5e6 / 0.75
    splits, best_cost = 1, 0.0
    s = 1
    while s <= 16 and s * 2 <= (kb if kb > 1 else 2):
        per = cdiv(kb, s)
        if cdiv(kb, per) == s:
            cost = cdiv(base * s, sms) * per + red_cost * s
            if s == 1 or cost < best_cost:
                best_cost, splits = cost, s
        s += 1
    return ld, bn, splits, cdiv(kb, splits) >= 64


def expected_linear_plan(R, K, N, x3, sms):
    ld, bn, splits, promote = plan_linear(R, K, N, sms)
    cap = (64 if x3 else 128) if promote else (128 if x3 else 256)
    while bn > cap:
        bn //= 2
    num_tiles = cdiv(N, 128) * cdiv(ld, bn) * splits
    return dict(BN=bn, BK=64, x3=int(x3), promote=int(promote), CG=1, TH=1, TW=128, stages=stages_for(bn, 64, x3),
                grid=min(num_tiles, sms), num_tiles=num_tiles, n_parts=splits, splits=splits)


HEAD_PLANS = [(300, 25088, 4096), (300, 4096, 4096), (1000, 100352, 4096), (1000, 4096, 4096), (1000, 4096, 105)]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("shape", HEAD_PLANS, ids=lambda s: "R%d-K%d-N%d" % s)
def test_linear_production_plan_vs_float64(ops, sms, precision, shape):
    """fc6 / fc7 / cls_score|bbox_pred at 300 RoIs, and config #4's head (1000 RoIs of a 2048-channel trunk) through
    frcnn_linear: the split-K plan, the promotion of long splits and the instantiation, checked against the plan hook."""
    R, K, N = shape
    x3 = precision == "bf16x3"
    valid = R - 67
    g = torch.Generator(device="cuda").manual_seed(R + K + N)
    xh, xl, xv = planes(torch.randn((1, R, K), device="cuda", generator=g).clamp_min(0), precision)
    wh, wl, wv = planes(torch.randn((1, N, K), device="cuda", generator=g) * (1.0 / K) ** 0.5, precision)
    b = torch.randn((N,), device="cuda", generator=g) * 0.5
    ref = xv[0] @ wv[0].T + b.double()
    del xv, wv
    act = ops.Act(xh, xl)
    ld = cdiv(N, 32) * 32
    m_valid = torch.tensor([valid], dtype=torch.int32, device="cuda")
    bias = ops.pad_bias(b, ld)
    y, y32 = ops.linear(act, wh, wl, bias, False, m_valid=m_valid, ld_f32=ld)
    plan = ops.conv_last_plan()
    assert plan == expected_linear_plan(R, K, N, x3, sms), plan
    if (R, K, N) == (300, 25088, 4096) and sms == 132:
        assert plan["splits"] == 4 and plan["promote"] == 1          # 4 splits of 98 k-blocks (12 chunks of 8 + 2)
    if (R, K) == (1000, 100352):
        assert plan["splits"] == 1 and plan["promote"] == 1 and plan["BN"] == (64 if x3 else 128)   # one 1568-k-block run
    y2, y32b = ops.linear(act, wh, wl, bias, False, m_valid=m_valid, ld_f32=ld)
    torch.cuda.synchronize()
    err = rel_err(y32[:valid, :N], ref[:valid])
    assert err < 3e-5, err
    assert not y32[valid:].any() and not y32[:, N:].any()
    assert torch.equal(y32, y32b) and torch.equal(y.hi, y2.hi)
    val = act_value(y)[0]
    err_act = rel_err(val[:valid], ref[:valid])
    assert err_act < TOL_ACT[precision], err_act
    assert not val[valid:].any()
    print("linear R%d K%d N%d %s: plan %s, f32 err %.3g, act err %.3g" % (R, K, N, precision, plan, err, err_act))


@pytest.mark.gpu
@pytest.mark.parametrize("x3", [True, False])
@pytest.mark.parametrize("shape", [(300, 25088, 4096), (1000, 100352, 4096)], ids=lambda s: "R%d-K%d-N%d" % s)
def test_linear_production_plan_exact_on_integers(ops, sms, x3, shape):
    """Small-integer operands at fc6's plan (4 promoted splits) and config #4's (one promoted 1568-k-block run): every
    partial sum is exact in fp32, so the result must be the integer GEMM exactly."""
    R, K, N = shape
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randint(-2, 3, (1, R, K), device="cuda", generator=g).float()
    w = torch.randint(-2, 3, (1, N, K), device="cuda", generator=g).float()
    b = torch.randint(-5, 6, (N,), device="cuda", generator=g).float()
    xa = ops.Act(x.to(torch.bfloat16), torch.zeros_like(x, dtype=torch.bfloat16) if x3 else None)
    wh = w.to(torch.bfloat16)
    wl = torch.zeros_like(wh) if x3 else None
    _, y32 = ops.linear(xa, wh, wl, ops.pad_bias(b, N), False, ld_f32=N, want_act=False)
    plan = ops.conv_last_plan()
    assert plan == expected_linear_plan(R, K, N, x3, sms) and plan["promote"] == 1, plan
    want = (x[0].double() @ w[0].double().T + b.double()).float()
    assert torch.equal(y32, want), float((y32 - want).abs().max())


# ------------------------------------------------------------------------------- d. epilogue edges
@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_m_valid_edges(ops, precision):
    """Rows (pixels) >= *m_valid are exact zeros in every output: counts inside warpgroup 0, between the two warpgroups
    and at tile edges of a 3-tile GEMM."""
    M, K, N = 300, 256, 96
    act, wh, wl, bias, ref = make_conv(ops, 1, M, K, N, 1, precision, seed=41, bias_pad=128)
    ref = ref[0]
    for valid in (0, 1, 63, 64, 65, 127, 128, 129, M):
        m_valid = torch.tensor([valid], dtype=torch.int32, device="cuda")
        y, y32 = ops.conv2d(act, wh, wl, bias, 1, False, ld_f32=128, m_valid=m_valid)
        torch.cuda.synchronize()
        val = act_value(y)[0]
        if valid:
            assert rel_err(y32[:valid, :N], ref[:valid]) < TOL_F32[precision], valid
            assert rel_err(val[:valid], ref[:valid]) < TOL_ACT[precision], valid
        assert not y32[valid:].any() and not y.hi[0, valid:].any(), valid
        assert y.lo is None or not y.lo[0, valid:].any(), valid


@pytest.mark.gpu
@pytest.mark.parametrize("precision,res_lo", [("bf16", False), ("bf16x3", False), ("bf16x3", True)])
def test_residual_epilogue_vs_float64(ops, precision, res_lo):
    """frcnn_conv2d_res: relu(conv(x) + bias + res_hi (+ res_lo)); res_lo = NULL adds the hi plane only."""
    H, W, C = 23, 37, 128
    act, wh, wl, bias, ref = make_conv(ops, H, W, C, C, 3, precision, seed=42)
    g = torch.Generator(device="cuda").manual_seed(43)
    rh, rl, _ = planes(torch.randn((H, W, C), device="cuda", generator=g), "bf16x3")
    res = ops.Act(rh, rl if res_lo else None)
    y = ops.conv2d_res(act, wh, wl, bias, 3, True, res)
    torch.cuda.synchronize()
    want = (ref + act_value(res)).clamp_min(0)
    check_act(y, want, precision)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_fused_pool_tile_remainder_one(ops, precision):
    """Fused 2x2 ceil-mode pool with H = 8*4 + 1 and W = 16*3 + 1: the last tile row and column hold one pixel, a window
    of one; bf16 at BN = 256, bf16x3 at its widest N tile (128)."""
    H, W, C = 33, 49, 256
    act, wh, wl, bias, ref = make_conv(ops, H, W, 128, C, 3, precision, seed=44, relu_input=True)
    with settings(ops, bn=256 if precision == "bf16" else 128):
        y, _ = ops.conv2d(act, wh, wl, bias, 3, True, fuse_pool=True)
        plan = ops.conv_last_plan()
    torch.cuda.synchronize()
    assert (plan["BN"], plan["TH"], plan["TW"]) == ((256 if precision == "bf16" else 128), 8, 16)
    assert y.hi.shape == (17, 25, C)
    check_act(y, pool_ref(ref.clamp_min(0)), precision)


def canary_view(n, dtype, margin, sentinel):
    """A view of n elements inside a buffer with `margin` sentinel elements on either side."""
    store = torch.int16 if dtype == torch.bfloat16 else torch.int32
    buf = torch.full((n + 2 * margin,), sentinel, dtype=store, device="cuda")
    return buf, buf[margin:margin + n].view(dtype)


def assert_canary_intact(buf, n, margin, sentinel):
    assert bool((buf[:margin] == sentinel).all()), "store before the output"
    assert bool((buf[margin + n:] == sentinel).all()), "store past the output"


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_epilogue_stores_stay_inside_their_outputs(ops, precision):
    """Outputs passed as views into larger sentinel-filled buffers: no byte outside the view changes.  A pixel tile reaches
    at most TH - 1 rows and TW - 1 columns past the image, i.e. fewer than 32 * W + 128 pixels past the end of an unpooled
    output, so a margin of 128 * W pixels catches every stray store and keeps it inside the allocation."""
    H, W, Cin, Cout, ld = 37, 45, 64, 96, 128
    S16, S32 = 0x5A5A, 0x5A5A5A5A
    act, wh, wl, bias, ref = make_conv(ops, H, W, Cin, Cout, 3, precision, seed=45, relu_input=True, bias_pad=ld)
    for tile in ((8, 16), (32, 4), (1, 128)):
        TH, TW = tile
        assert (cdiv(H, TH) * TH - H) * W + cdiv(W, TW) * TW <= 128 * W
        margin_f32, margin_act = 128 * W * ld, 128 * W * Cout
        b32, y32 = canary_view(H * W * ld, torch.float32, margin_f32, S32)
        bh, yh = canary_view(H * W * Cout, torch.bfloat16, margin_act, S16)
        bl, yl = canary_view(H * W * Cout, torch.bfloat16, margin_act, S16)
        out = ops.Act(yh.view(H, W, Cout), yl.view(H, W, Cout) if precision == "bf16x3" else None)
        with settings(ops, th=TH, tw=TW, bn=64):
            ops.conv2d(act, wh, wl, bias, 3, False, out=out, out_f32=y32.view(H * W, ld), ld_f32=ld)
            assert (ops.conv_last_plan()["TH"], ops.conv_last_plan()["TW"]) == tile
        torch.cuda.synchronize()
        assert_canary_intact(b32, H * W * ld, margin_f32, S32)
        assert_canary_intact(bh, H * W * Cout, margin_act, S16)
        if precision == "bf16x3":
            assert_canary_intact(bl, H * W * Cout, margin_act, S16)
        check_f32(y32.view(H * W, ld), ref, precision, Cout)
        check_act(out, ref, precision)
    # fused pool: [ceil(H/2), ceil(W/2), Cout] inside sentinels
    oh, ow = cdiv(H, 2), cdiv(W, 2)
    margin = 128 * W * Cout
    bh, yh = canary_view(oh * ow * Cout, torch.bfloat16, margin, S16)
    bl, yl = canary_view(oh * ow * Cout, torch.bfloat16, margin, S16)
    out = ops.Act(yh.view(oh, ow, Cout), yl.view(oh, ow, Cout) if precision == "bf16x3" else None)
    ops.conv2d(act, wh, wl, bias, 3, True, out=out, fuse_pool=True)
    torch.cuda.synchronize()
    assert_canary_intact(bh, oh * ow * Cout, margin, S16)
    if precision == "bf16x3":
        assert_canary_intact(bl, oh * ow * Cout, margin, S16)
    check_act(out, pool_ref(ref.clamp_min(0)), precision)


# ------------------------------------------------------------------------------- e. shared-memory reserve
# The VGG16 trunk at the 600 x 1000 input (conv1_1 runs on the compact first-layer path, conv5_2, conv5_3 and the RPN's
# 3x3 conv have conv5_1's plan): (name, H, W, Cin, Cout, fused pool)
VGG16_LAYERS = [("conv1_2", 600, 1000, 64, 64, True), ("conv2_1", 300, 500, 64, 128, False),
                ("conv2_2", 300, 500, 128, 128, True), ("conv3_1", 150, 250, 128, 256, False),
                ("conv3_2", 150, 250, 256, 256, False), ("conv3_3", 150, 250, 256, 256, True),
                ("conv4_1", 75, 125, 256, 512, False), ("conv4_2", 75, 125, 512, 512, False),
                ("conv4_3", 75, 125, 512, 512, True), ("conv5_1", 38, 63, 512, 512, False)]
RESERVES = [0, 48 * 1024, 81408, 81920, 96 * 1024]


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("layer", VGG16_LAYERS, ids=lambda l: l[0])
def test_smem_reserve_sweep_on_production_plans(ops, precision, layer):
    """Every documented reserve (0..96 KB) launches every production conv plan.  Where two stages of the planned N tile
    do not fit (bf16x3 BN = 128 above 81,408 B) the planner narrows the tile; the result then matches the oracle, and
    otherwise it is bit-identical to the full pipeline depth."""
    name, H, W, Cin, Cout, pool = layer
    x3 = precision == "bf16x3"
    act, wh, wl, bias, ref = make_conv(ops, H, W, Cin, Cout, 3, precision, seed=H + Cin, relu_input=True)
    want = ref.clamp_min(0)
    if pool:
        want = pool_ref(want)
    del ref
    base, base_bn = None, None
    for reserve in RESERVES:
        with settings(ops, reserve=reserve):
            y, _ = ops.conv2d(act, wh, wl, bias, 3, True, fuse_pool=pool)
            plan = ops.conv_last_plan()
        torch.cuda.synchronize()
        if base is None:
            base, base_bn = y, plan["BN"]
            if x3 and name != "conv1_2":
                assert base_bn == 128, plan
        bn = base_bn
        while bn > 64 and stages_for(bn, 64, x3, reserve) < 2:
            bn //= 2
        assert plan["BN"] == bn and plan["stages"] == stages_for(bn, 64, x3, reserve) >= 2, (reserve, plan)
        check_act(y, want, precision)
        if bn == base_bn:
            assert torch.equal(y.hi, base.hi) and (y.lo is None or torch.equal(y.lo, base.lo)), reserve


# ------------------------------------------------------------------------------- f. programmatic dependent launch
@pytest.mark.gpu
def test_programmatic_launch_graph_is_bit_identical():
    """The 150 x 201 bf16x3 forward graph captured with programmatic dependent launch on and off gives the same bits."""
    import frcnn_oracle as orc
    from frcnn_b200 import ops
    from frcnn_b200.engine import Engine
    params = orc.make_params(seed=1234)
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    x = torch.from_numpy(orc.make_image(150, 201, seed=1)[0]).cuda()
    outs = []
    for pdl in (1, 0):
        ops.set_programmatic_launch(pdl)
        try:
            eng = Engine(params, precision="bf16x3", anchors=anchors, use_graph=True)
            prob, boxes, plan = eng(x)
            torch.cuda.synchronize()
            outs.append([prob.clone(), boxes.clone(), plan.acts[-1].hi.clone(), plan.acts[-1].lo.clone()])
        finally:
            ops.set_programmatic_launch(-1)
    for a, b in zip(*outs):
        assert a.shape == b.shape and torch.equal(a, b)
