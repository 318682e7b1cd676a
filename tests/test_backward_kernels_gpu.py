"""The conv-backward and optimizer entry points one by one (train_backward.cu, rcnn_train.cu), against bit-level or float64
restatements of the same operation on the exact operand values (tests/backward_ref.py), at the benchmarked 600x1000
layer shapes, at the block edges of each kernel and on special values.

Bars: grad_prepare, pack_conv_weights_dgrad, wgrad_reduce, sgd_momentum(_bf16g), cast_f32_bf16 and dropout bit-exact (NaN
compared as NaN-ness only); products of the bf16x3 GEMM 5e-5 of max-norm (the bar the training step states), 3e-5 / 1e-5 on
the fp32 output of the data-gradient conv; integer-valued variants exact; RoI-pool backward 1e-6 of max-norm (its 2^-44
fixed point) and bit-identical across calls."""
import numpy as np
import pytest
import torch
import torch.nn.grad as tg

import backward_ref as br

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = 0x5A5A                     # bf16 sentinel (a finite number) where a kernel must not store
GUARD = 64                        # sentinel elements past the end of an NHWC output


@pytest.fixture(scope="module")
def tops():
    from frcnn_b200 import train_ops
    return train_ops


@pytest.fixture(scope="module")
def ops():
    from frcnn_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _sentinel(n):
    return torch.full((n,), SENT, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def _rel(got, want):
    got, want = got.double(), want.double()
    return float((got - want).abs().max() / max(float(want.abs().max()), 1e-300))


def assert_bits(got, want, what):
    """bf16 tensors equal bit for bit; where `want` is NaN, `got` must be NaN (any payload)."""
    nan = torch.isnan(want.float())
    assert torch.equal(torch.isnan(got.float()), nan), "%s: NaN positions differ" % what
    gb, wb = br.bits(got)[~nan], br.bits(want)[~nan]
    bad = int((gb != wb).sum())
    assert bad == 0, "%s: %d of %d elements differ" % (what, bad, gb.numel())


def _pair(shape, gen, scale=1.0, lo=True):
    v = torch.randn(shape, device=DEV, generator=gen) * scale
    hi, l = br.split(v)
    return hi, (l if lo else None)


def _relu_ties(shape, gen, resplit=True):
    """Post-ReLU activation with many exact ties and zeros: values k/2, k in 0..3; a random half of the positive elements
    stored as the other (hi, lo) pair of the same value (v - 1/16, 1/16)."""
    v = torch.randint(-3, 4, shape, device=DEV, generator=gen).clamp_min(0).float() * 0.5
    hi, lo = v.to(torch.bfloat16), torch.zeros(shape, dtype=torch.bfloat16, device=DEV)
    if resplit:
        alt = (torch.rand(shape, device=DEV, generator=gen) < 0.5) & (v > 0)
        hi = torch.where(alt, (v - 0.0625).to(torch.bfloat16), hi)
        lo = torch.where(alt, torch.full_like(lo, 0.0625), lo)
    return hi, lo


def _pool_of(y, gen):
    """2x2 ceil-mode max of y's values, each pooled value stored in a random one of its two (hi, lo) forms."""
    H, W, C = y[0].shape
    v = br.value(*y)
    pad = torch.full((H + H % 2, W + W % 2, C), -float("inf"), device=DEV)
    pad[:H, :W] = v
    pv = pad.view((H + 1) // 2, 2, (W + 1) // 2, 2, C).amax((1, 3))
    hi, lo = pv.to(torch.bfloat16), torch.zeros_like(pv, dtype=torch.bfloat16)
    alt = (torch.rand(pv.shape, device=DEV, generator=gen) < 0.5) & (pv > 0)
    hi = torch.where(alt, (pv - 0.0625).to(torch.bfloat16), hi)
    lo = torch.where(alt, torch.full_like(lo, 0.0625), lo)
    return hi, lo


def run_prepare(tops, ops, H, W, C, g=None, g_f32=None, y=None, p=None, planes=1, times2=False, outputs="both", lo_out=True):
    """frcnn_grad_prepare into sentinel-filled buffers, compared byte for byte with backward_ref.grad_prepare: the NHWC
    planes (plus a guard past their end) and the whole transposed buffers, padding included."""
    n = H * W * C
    act = lambda pr: None if pr is None else ops.Act(pr[0], pr[1])
    o = tb = None
    if outputs in ("both", "o"):
        bufs = [_sentinel(n + GUARD) for _ in range(2 if lo_out else 1)]
        o = ops.Act(bufs[0][:n].view(H, W, C), bufs[1][:n].view(H, W, C) if lo_out else None)
    if outputs in ("both", "t"):
        tb = tops.TBuf(planes, C, H, W, DEV, x3=lo_out)
        for t in (tb.hi, tb.lo):
            if t is not None:
                br.bits(t).fill_(SENT)
    tops.grad_prepare(H, W, C, g=act(g), g_f32=g_f32, y=act(y), p=act(p), out=o, tbuf=tb, times2=times2)
    torch.cuda.synchronize()
    w_hi, w_lo, t_hi, t_lo, written = br.grad_prepare(H, W, C, g=g, g_f32=g_f32, y=y, p=p, planes=planes, times2_=times2)
    if o is not None:
        for buf, got, want, name in zip(bufs, (o.hi, o.lo), (w_hi, w_lo), ("o_hi", "o_lo")):
            assert_bits(got, want, name)
            assert (br.bits(buf[n:]) == SENT).all(), name + ": store past the end"
    if tb is not None:
        sent = _sentinel(1).view(())
        for got, want, name in zip((tb.hi, tb.lo), (t_hi, t_lo), ("t_hi", "t_lo")):
            if got is not None:
                assert_bits(got, torch.where(written, want, sent), name)
    return o.hi if o is not None else w_hi


# ------------------------------------------------------------------ A. grad_prepare
# (H, W, C, mode, planes, outputs): H 1/2/3/37, W 1..1000 across the 256-pixel blocks, C 8..520 (part-full 64-channel
# blocks), the RCNN pool5 call (H = 1, C = 25,088), every source / mask / routing mode and output selection
PREP_CASES = [
    (1, 1, 8, "relu", 3, "both"),
    (2, 7, 32, "pool", 3, "both"),
    (3, 8, 64, "pool", 1, "both"),
    (3, 9, 72, "relu", 3, "both"),
    (37, 255, 64, "pool", 3, "both"),
    (2, 256, 32, "plain", 3, "both"),
    (3, 257, 72, "pool", 3, "both"),
    (2, 511, 8, "relu", 1, "both"),
    (1, 512, 520, "relu", 3, "both"),
    (3, 513, 64, "pool", 3, "t"),
    (2, 1000, 64, "relu", 3, "o"),
    (37, 9, 520, "nolo", 3, "both"),
    (37, 1000, 32, "pool", 1, "both"),
    (3, 513, 72, "nolo_out", 3, "both"),
    (1, 300, 25088, "plain", 1, "t"),
    (1, 300, 4096, "relu_x2", 1, "both"),
    (5, 9, 64, "f32_wide", 1, "both"),
    (5, 9, 64, "f32_narrow", 3, "both"),
    (38, 63, 64, "f32", 1, "both"),
]


def _prep_inputs(H, W, C, mode, gen):
    kw = {}
    if mode.startswith("f32"):
        ld = {"f32_wide": C + 32, "f32_narrow": C - 24, "f32": C}[mode]
        kw["g_f32"] = torch.randn((H * W, ld), device=DEV, generator=gen)
        if mode != "f32":
            kw["y"] = _relu_ties((H, W, C), gen)
        return kw
    if mode == "pool":
        y = _relu_ties((H, W, C), gen)
        kw["y"], kw["p"] = y, _pool_of(y, gen)
        kw["g"] = _pair(((H + 1) // 2, (W + 1) // 2, C), gen)
        return kw
    kw["g"] = _pair((H, W, C), gen, lo=(mode != "nolo"))
    if mode in ("relu", "relu_x2", "nolo", "nolo_out"):
        kw["y"] = _relu_ties((H, W, C), gen)
    kw["times2"] = mode == "relu_x2"
    return kw


@pytest.mark.parametrize("H,W,C,mode,planes,outputs", PREP_CASES)
def test_grad_prepare_bit_exact(tops, ops, H, W, C, mode, planes, outputs):
    kw = _prep_inputs(H, W, C, mode, _gen(H * 7919 + W * 31 + C))
    run_prepare(tops, ops, H, W, C, planes=planes, outputs=outputs, lo_out=(mode != "nolo_out"), **kw)


# the grad_prepare calls of the RPN step at 600x1000: (H, W, Cout, pooled) of every layer shape, the layer's incoming gradient
# routed / masked into one plane, and its input re-laid out into three shifted planes (one for conv1_1's 32-channel im2col)
RPN_600 = [(600, 1000, 64, 32, False), (600, 1000, 64, 64, True), (300, 500, 128, 64, False), (300, 500, 128, 128, True),
           (150, 250, 256, 128, False), (150, 250, 256, 256, True), (75, 125, 512, 256, False), (75, 125, 512, 512, True),
           (38, 63, 512, 512, False)]


@pytest.mark.parametrize("H,W,co,ci,pooled", RPN_600)
def test_grad_prepare_rpn_layers_600x1000(tops, ops, H, W, co, ci, pooled):
    gen = _gen(H + co + ci)
    kw = _prep_inputs(H, W, co, "pool" if pooled else "relu", gen)
    run_prepare(tops, ops, H, W, co, planes=1, **kw)
    x = _relu_ties((H, W, ci), gen)
    run_prepare(tops, ops, H, W, ci, g=x, planes=1 if ci == 32 else 3, outputs="t")


def test_grad_prepare_times2_exhaustive(tops, ops):
    """Every bf16 pattern, in both halves of a 32-bit word, in g_hi and g_lo: bf16(2x) -- inf stays inf, NaN stays NaN,
    overflow gives inf, subnormals are doubled, signs kept."""
    pat = br.all_bf16_patterns()
    g_hi = br.from_bits(pat, DEV).view(2, 1024, 64)
    g_lo = br.from_bits(pat[::-1].copy(), DEV).view(2, 1024, 64)
    got = run_prepare(tops, ops, 2, 1024, 64, g=(g_hi, g_lo), times2=True, planes=3)
    x = g_hi.float()
    assert torch.isinf(got.float()[torch.isinf(x)]).all()
    assert (br.bits(got)[(x == 0) & ~torch.signbit(x)] == 0).all()


def test_grad_prepare_relu_mask_exhaustive(tops, ops):
    """Every bf16 pattern as y_hi (y_lo = 0, the split of that value): the gradient passes where y > 0, so +0, -0, every
    negative value and every NaN block it, +inf and positive subnormals pass."""
    pat = br.all_bf16_patterns()
    y_hi = br.from_bits(pat, DEV).view(2, 1024, 64)
    g = _pair((2, 1024, 64), _gen(3))
    got = run_prepare(tops, ops, 2, 1024, 64, g=g, y=(y_hi, torch.zeros_like(y_hi)), planes=1)
    blocked = torch.isnan(y_hi.float()) | (y_hi.float() <= 0)
    assert (br.bits(got)[blocked] == 0).all() and torch.equal(got[~blocked], g[0][~blocked])
    # the fp32 source honours the same mask
    g32 = torch.randn((2 * 1024, 64), device=DEV, generator=_gen(4))
    run_prepare(tops, ops, 2, 1024, 64, g_f32=g32, y=(y_hi, torch.zeros_like(y_hi)), planes=3)


def test_grad_prepare_routing_ties(tops, ops):
    """One 2x2 window per channel with a tie of equal positive maxima at each pair of scan positions, the pooled value
    stored as the other (hi, lo) split: the gradient goes to the first position in (0,0), (0,1), (1,0), (1,1) order."""
    import itertools
    combos = [c for r in (1, 2, 3, 4) for c in itertools.combinations(range(4), r)]     # 15 tie sets
    C = 16
    y = torch.zeros((2, 2, C), device=DEV)
    for ch, cset in enumerate(combos):
        for e in cset:
            y[e >> 1, e & 1, ch] = 1.5
    y[0, 0, 15] = 0.0                                          # channel 15: a window whose maximum is 0
    yh = y.to(torch.bfloat16)
    ph = torch.full((1, 1, C), 1.5 - 0.0625, device=DEV).to(torch.bfloat16)
    pl = torch.full((1, 1, C), 0.0625, device=DEV).to(torch.bfloat16)
    ph[..., 15], pl[..., 15] = 0, 0
    g = (torch.arange(1, C + 1, device=DEV).float().view(1, 1, C).to(torch.bfloat16), None)
    got = run_prepare(tops, ops, 2, 2, C, g=g, y=(yh, torch.zeros_like(yh)), p=(ph, pl), planes=3)
    for ch, cset in enumerate(combos):
        first = min(cset)
        want = torch.zeros((2, 2), device=DEV)
        want[first >> 1, first & 1] = ch + 1
        assert torch.equal(got[..., ch].float(), want), (ch, cset)
    assert not got[..., 15].float().any()


def test_grad_prepare_argument_errors(tops, ops):
    from frcnn_b200._lib import FrcnnError
    g = _pair((3, 5, 16), _gen(1))
    a = ops.Act(*g)
    tb = tops.TBuf(1, 16, 3, 5, DEV)
    with pytest.raises(FrcnnError):
        tops.grad_prepare(3, 5, 12, g=a, tbuf=tb)                                   # C % 8 != 0
    with pytest.raises(FrcnnError):
        tops.grad_prepare(3, 5, 16, g=a, tbuf=tops.TBuf(2, 16, 3, 5, DEV))          # planes == 2
    with pytest.raises(FrcnnError):
        tops.grad_prepare(3, 5, 16, g=a)                                            # no output
    g32 = torch.zeros((15, 16), device=DEV)
    with pytest.raises(FrcnnError):
        tops.grad_prepare(3, 5, 16, g_f32=g32, y=a, p=ops.Act(*_pair((2, 3, 16), _gen(2))), tbuf=tb)   # fp32 + pooling
    with pytest.raises(FrcnnError):
        tops.grad_prepare(3, 5, 16, g_f32=g32, tbuf=tb, times2=True)               # fp32 + times2
    torch.cuda.synchronize()


# ------------------------------------------------------------------ B. pack_conv_weights_dgrad
@pytest.mark.parametrize("Cout,Cin,kh,kw,cout_pad,x3", [
    (64, 32, 3, 3, 64, True), (40, 24, 3, 3, 48, True), (16, 8, 1, 1, 16, True), (24, 16, 1, 3, 32, False),
    (54, 512, 1, 1, 64, True)])
def test_pack_conv_weights_dgrad_bit_exact(tops, Cout, Cin, kh, kw, cout_pad, x3):
    w = torch.randn((Cout, Cin, kh, kw), device=DEV, generator=_gen(Cout * Cin)) * 0.05
    arg = w[:, :, 0, 0] if (kh, kw) == (1, 1) and Cin == 512 else w             # the RPN heads pass a [54, 512] matrix
    hi, lo = tops.pack_conv_weights_dgrad(arg, cout_pad=cout_pad, x3=x3)
    torch.cuda.synchronize()
    want_hi, want_lo = br.pack_dgrad(w, cout_pad)
    assert hi.shape == (kh * kw, Cin, cout_pad)
    assert_bits(hi, want_hi, "hi")
    if x3:
        assert_bits(lo, want_lo, "lo")
    else:
        assert lo is None


# ------------------------------------------------------------------ C. data gradient through the conv kernel
def _unpack_dgrad(hi, lo, Cout, kh, kw):
    """The OIHW float64 filter whose dgrad pack the kernel read (inverse of backward_ref.pack_dgrad)."""
    v = hi.double() + (lo.double() if lo is not None else 0)
    taps, Cin, _ = v.shape
    return torch.flip(v[:, :, :Cout].reshape(kh, kw, Cin, Cout).permute(3, 2, 0, 1), (2, 3))


TOL_F32 = {"bf16x3": 3e-5, "bf16": 1e-5}


@pytest.mark.parametrize("H,W,Cout,Cin,k,cout_pad,precision", [
    (37, 45, 64, 32, 3, 64, "bf16x3"), (13, 70, 128, 64, 3, 128, "bf16"), (19, 25, 54, 512, 1, 64, "bf16x3"),
    (19, 25, 54, 512, 1, 64, "bf16"), (5, 3, 72, 96, 3, 72, "bf16x3"), (37, 45, 64, 32, 3, 64, "integer")])
def test_dgrad_conv_matches_float64(tops, ops, H, W, Cout, Cin, k, cout_pad, precision):
    """dX = conv(dY, rot180 swapped W) on frcnn_conv2d vs float64 conv2d_input; Cin = 54 padded to 64 is the RPN heads'."""
    gen = _gen(H * W + Cin)
    x3 = precision == "bf16x3"
    if precision == "integer":
        w = torch.randint(-3, 4, (Cout, Cin, k, k), device=DEV, generator=gen).float()
        dy = torch.randint(-3, 4, (H, W, cout_pad), device=DEV, generator=gen).float()
    else:
        w = torch.randn((Cout, Cin, k, k), device=DEV, generator=gen) * 0.05
        dy = torch.randn((H, W, cout_pad), device=DEV, generator=gen)
    dy[..., Cout:] = 0
    dhi, dlo = tops.pack_conv_weights_dgrad(w if k == 3 else w[:, :, 0, 0], cout_pad=cout_pad, x3=x3)
    d_hi, d_lo = br.split(dy) if x3 else (dy.to(torch.bfloat16), None)
    bias = ops.pad_bias(torch.zeros(Cin, device=DEV), Cin)
    y, y32 = ops.conv2d(ops.Act(d_hi, d_lo), dhi, dlo, bias, k, False, ld_f32=Cin)
    plan = ops.conv_last_plan()
    torch.cuda.synchronize()
    assert plan["x3"] == (1 if x3 else 0) and plan["grid"] > 0, plan
    We = _unpack_dgrad(dhi, dlo, Cout, k, k)
    dye = br.value(d_hi, d_lo).double()[..., :Cout].permute(2, 0, 1)[None]
    want = tg.conv2d_input((1, Cin, H, W), We, dye, padding=k // 2)[0].permute(1, 2, 0).reshape(H * W, Cin)
    if precision == "integer":
        assert torch.equal(y32.double(), want)
        return
    err = _rel(y32, want)
    err_act = _rel(br.value(y.hi, y.lo).reshape(H * W, Cin), want)
    print("dgrad %dx%d %d->%d k%d %s: f32 %.2e, act %.2e" % (H, W, Cout, Cin, k, precision, err, err_act))
    assert err < TOL_F32[precision] and (precision != "bf16x3" or err_act < 5e-5)


# ------------------------------------------------------------------ D. wgrad_reduce alone
@pytest.mark.parametrize("groups,S,M,Mp,N,ld,scale", [
    (1, 1, 64, 64, 32, 32, 1.0), (9, 7, 40, 64, 72, 96, 0.5), (9, 1, 64, 128, 64, 64, 1.0 / 3), (1, 7, 54, 64, 512, 512, 1.0),
    (9, 7, 512, 512, 512, 512, 0.1)])
def test_wgrad_reduce_bit_exact(tops, groups, S, M, Mp, N, ld, scale):
    parts = torch.randn((groups, S, Mp, ld), device=DEV, generator=_gen(groups * S + M))
    parts[:, :, :, :N] *= torch.logspace(-3, 3, N, device=DEV)                     # mixed magnitudes: rounding matters
    dw = torch.full((M * N * groups + GUARD,), 7.0, device=DEV)
    tops.wgrad_reduce(parts, M, N, dw[:M * N * groups], scale=scale)
    torch.cuda.synchronize()
    assert torch.equal(dw[:M * N * groups], br.wgrad_reduce(parts, M, N, scale))
    assert (dw[M * N * groups:] == 7.0).all()


# ------------------------------------------------------------------ D/E. dW, db, dX of every RPN-step layer at 600x1000
LAYERS_600 = {  # name: (H, W, Cin, Cout, kind)
    "conv1_1": (600, 1000, 32, 64, "im2col"), "conv1_2": (600, 1000, 64, 64, "3x3"), "conv2_1": (300, 500, 64, 128, "3x3"),
    "conv2_2": (300, 500, 128, 128, "3x3"), "conv3_1": (150, 250, 128, 256, "3x3"), "conv3_x": (150, 250, 256, 256, "3x3"),
    "conv4_1": (75, 125, 256, 512, "3x3"), "conv4_x": (75, 125, 512, 512, "3x3"), "conv5_x/rpn_conv_3x3": (38, 63, 512, 512, "3x3"),
    "rpn heads": (38, 63, 512, 54, "heads")}


@pytest.mark.parametrize("values", ["random", "zero_mean", "integer"])
@pytest.mark.parametrize("name", list(LAYERS_600))
def test_layer_gradients_600x1000(tops, ops, name, values):
    """grad_prepare -> gemm_nt_splitk (RpnTrainer._splits) -> wgrad_reduce, bias_grad and the dgrad conv at the RPN step's
    600x1000 layer shapes, against float64 conv2d_weight / sum / conv2d_input of the operand values the kernels read.
    "random": dY with a mean, so db is a large sum; "zero_mean": dY without one, so db is a small sum of cancelling terms
    (the hard case for bias_grad's per-thread fp32 sums); "integer": small integers in single-pass bf16, every sum below
    2^24 -- exact."""
    from frcnn_b200.train_engine import RpnTrainer
    H, W, ci, co, kind = LAYERS_600[name]
    gen = _gen(H * ci + co)
    integer = values == "integer"
    x3 = not integer
    ld = 64 if kind == "heads" else co

    def pair(v):
        return br.split(v) if x3 else (v.to(torch.bfloat16), None)

    if integer:
        xv = torch.randint(0, 4, (H, W, ci), device=DEV, generator=gen).float()
        gv = torch.randint(-3, 4, (H, W, ld), device=DEV, generator=gen).float()
        wv = torch.randint(-3, 4, (co, ci, 3, 3), device=DEV, generator=gen).float()
    else:
        xv = torch.randn((H, W, ci), device=DEV, generator=gen).clamp_min(0)
        gv = torch.randn((H, W, ld), device=DEV, generator=gen) * 1e-3 + (2e-4 if values == "random" else 0.0)
        wv = torch.randn((co, ci, 3, 3), device=DEV, generator=gen) * 0.02
    if kind == "im2col":
        xv[..., 27:] = 0
    gv[..., co:] = 0
    x = ops.Act(*pair(xv))
    dyT = tops.TBuf(1, ld, H, W, DEV, x3=x3)
    dy_hi = torch.empty((H, W, ld), dtype=torch.bfloat16, device=DEV)
    dy = ops.Act(dy_hi, torch.empty_like(dy_hi) if x3 else None)
    if kind == "heads":
        tops.grad_prepare(H, W, ld, g_f32=gv.view(H * W, ld), out=dy, tbuf=dyT)
    else:
        yv = torch.randn((H, W, co), device=DEV, generator=gen).clamp_min(0) if not integer else \
            torch.randint(-1, 3, (H, W, co), device=DEV, generator=gen).clamp_min(0).float()
        tops.grad_prepare(H, W, co, g=ops.Act(*pair(gv)), y=ops.Act(*pair(yv)), out=dy, tbuf=dyT)
    groups = 9 if kind == "3x3" else 1
    xT = tops.TBuf(3 if kind != "im2col" else 1, ci, H, W, DEV, x3=x3)
    tops.grad_prepare(H, W, ci, g=x, tbuf=xT)
    K = dyT.Kp
    pl = 1 if xT.planes == 3 and groups == 1 else 0
    b_hi = xT.hi if groups == 9 else xT.hi[pl]
    b_lo = None if not x3 else (xT.lo if groups == 9 else xT.lo[pl])
    splits = RpnTrainer._splits(None, groups, ld, ci, K // 64)
    parts = tops.gemm_nt_splitk(dyT.hi[0], dyT.lo[0] if x3 else None, b_hi, b_lo, groups=groups, row_stride=dyT.Wp, splits=splits)
    plan = ops.conv_last_plan()
    dw = torch.empty((co * ci * groups,), device=DEV)
    tops.wgrad_reduce(parts, co, ci, dw)
    db = torch.empty((co,), device=DEV)
    tops.bias_grad(dyT, co, db)
    torch.cuda.synchronize()
    assert plan["n_parts"] == groups * parts.shape[1] and plan["x3"] == (1 if x3 else 0), plan
    dye = br.value(dy.hi, dy.lo).double()[..., :co].permute(2, 0, 1)[None]
    xe = br.value(x.hi, x.lo).double().permute(2, 0, 1)[None]
    if groups == 9:
        dw_ref = tg.conv2d_weight(xe, (co, ci, 3, 3), dye, padding=1).reshape(-1)
    else:
        dw_ref = (dye[0].reshape(co, -1) @ xe[0].reshape(ci, -1).T).reshape(-1)
    db_ref = dye.sum((0, 2, 3))
    e_w, e_b = _rel(dw, dw_ref), _rel(db, db_ref)
    e_x = 0.0
    if kind != "im2col":
        wk = wv if kind == "3x3" else wv[:, :, 1, 1]
        dhi, dlo = tops.pack_conv_weights_dgrad(wk, cout_pad=ld, x3=x3)
        gx, gx32 = ops.conv2d(dy, dhi, dlo, ops.pad_bias(torch.zeros(ci, device=DEV), ci), 3 if kind == "3x3" else 1, False,
                              ld_f32=ci)
        torch.cuda.synchronize()
        k = 3 if kind == "3x3" else 1
        dx_ref = tg.conv2d_input((1, ci, H, W), _unpack_dgrad(dhi, dlo, co, k, k), dye, padding=k // 2)[0].permute(1, 2, 0)
        if integer:
            assert torch.equal(gx32.double(), dx_ref.reshape(H * W, ci)), name
        e_x = _rel(br.value(gx.hi, gx.lo), dx_ref)
    print("%-22s %s %dx%d splits %d: dW %.2e  db %.2e  dX %.2e" % (name, values, H, W, parts.shape[1], e_w, e_b, e_x))
    if integer:
        assert torch.equal(dw.double(), dw_ref) and torch.equal(db.double(), db_ref), name
    else:
        assert e_w <= 5e-5 and e_b <= 5e-5 and e_x <= 5e-5, (e_w, e_b, e_x)


# ------------------------------------------------------------------ D. the RCNN head's weight gradients over 300 RoIs
@pytest.mark.parametrize("values", ["random", "integer"])
@pytest.mark.parametrize("name,M,N,m_out", [("fc6", 4096, 49 * 512, None), ("fc7", 4096, 4096, None),
                                            ("cls_score|bbox_pred", 128, 4096, 105)])
def test_rcnn_fc_weight_gradients_300_rois(tops, ops, name, M, N, m_out, values):
    """RcnnTrainer._fc_wgrad as the step runs it: grad_prepare (ReLU + ratio-0.5 dropout backward) of dY and the transposed
    input over R_cap = 300 RoI rows (the last 40 invalid, zero as the forward's m_valid leaves them), then one un-split
    gemm_nt_splitk straight into dW (fc6, fc7) or through wgrad_reduce (the heads' 105 of 128 rows); and bias_grad.
    Against float64 dY^T X on the operand values the kernels read."""
    from frcnn_b200.train_engine import RcnnTrainer
    R_cap, valid = 300, 260
    gen = _gen(M + N)
    integer = values == "integer"
    x3 = not integer

    def pair(v):
        return br.split(v) if x3 else (v.to(torch.bfloat16), None)

    if integer:
        gv = torch.randint(-3, 4, (1, R_cap, M), device=DEV, generator=gen).float()
        xv = torch.randint(0, 4, (1, R_cap, N), device=DEV, generator=gen).float()
    else:
        gv = torch.randn((1, R_cap, M), device=DEV, generator=gen) * 1e-3
        xv = torch.randn((1, R_cap, N), device=DEV, generator=gen).clamp_min(0)
    yv = torch.randint(-1, 3, (1, R_cap, M), device=DEV, generator=gen).clamp_min(0).float()
    gv[:, valid:], xv[:, valid:], yv[:, valid:] = 0, 0, 0
    if m_out is not None:
        gv[..., m_out:] = 0
    dy_hi = torch.empty((1, R_cap, M), dtype=torch.bfloat16, device=DEV)
    dy = ops.Act(dy_hi, torch.empty_like(dy_hi) if x3 else None)
    dyT = tops.TBuf(1, M, 1, R_cap, DEV, x3=x3)
    if m_out is not None:        # the heads' gradient is the loss kernel's fp32 matrix, no mask
        tops.grad_prepare(1, R_cap, M, g_f32=gv.view(R_cap, M), out=dy, tbuf=dyT)
    else:
        tops.grad_prepare(1, R_cap, M, g=ops.Act(*pair(gv)), y=ops.Act(*pair(yv)), out=dy, tbuf=dyT, times2=True)
    x = ops.Act(*pair(xv))
    xT = tops.TBuf(1, N, 1, R_cap, DEV, x3=x3)
    tops.grad_prepare(1, R_cap, N, g=x, tbuf=xT)
    rows = m_out or M
    dw = torch.full((rows * N,), 7.0, device=DEV)
    RcnnTrainer._fc_wgrad(None, dyT, xT, M, N, dw, m_out=m_out)
    db = torch.empty((rows,), device=DEV)
    tops.bias_grad(dyT, rows, db)
    torch.cuda.synchronize()
    dye = br.value(dy.hi, dy.lo).double()[0, :, :rows]
    xe = br.value(x.hi, x.lo).double()[0]
    dw_ref = (dye.T @ xe).reshape(-1)
    db_ref = dye.sum(0)
    e_w, e_b = _rel(dw, dw_ref), _rel(db, db_ref)
    print("%-20s %s R_cap %d: dW %.2e  db %.2e" % (name, values, R_cap, e_w, e_b))
    if integer:
        assert torch.equal(dw.double(), dw_ref) and torch.equal(db.double(), db_ref)
    else:
        assert e_w <= 5e-5 and e_b <= 5e-5, (e_w, e_b)


# ------------------------------------------------------------------ E. bias_grad exactness
@pytest.mark.parametrize("H,W,C,lo,scale", [(37, 64, 64, True, 1.0), (37, 64, 520, True, 0.5), (5, 255, 8, False, 1.0),
                                            (1, 300, 4096, True, 2.0)])
def test_bias_grad_exact(tops, H, W, C, lo, scale):
    """hi integers, lo multiples of 2^-10 over the whole [C, Kp] plane (every partial sum is exact in fp32): a dropped lo
    plane, a skipped stride or a lost block changes the result."""
    gen = _gen(C + W)
    tb = tops.TBuf(1, C, H, W, DEV, x3=lo)
    hi = torch.randint(-4, 5, tb.hi.shape, device=DEV, generator=gen).float()
    tb.hi.copy_(hi)
    want = hi.double()
    if lo:
        lv = torch.randint(-60, 61, tb.hi.shape, device=DEV, generator=gen).float() / 1024
        tb.lo.copy_(lv)
        want = want + lv.double()
    assert float(want.abs().sum(-1).max()) < 2 ** 14
    db = torch.empty((C + GUARD,), device=DEV).fill_(7.0)
    tops.bias_grad(tb, C, db[:C], scale=scale)
    torch.cuda.synchronize()
    assert torch.equal(db[:C].double(), want[0].sum(-1) * scale)
    assert (db[C:] == 7.0).all()


# ------------------------------------------------------------------ F. optimizer and the bf16 gradient bucket
LR, MOM, WD = 0.001, 0.9, 0.0005


def _opt_data(n, seed):
    rng = np.random.default_rng(seed)
    f = np.float32
    w = (rng.standard_normal(n) * 0.05).astype(f)
    v = (rng.standard_normal(n) * 1e-4).astype(f)
    g = (rng.standard_normal(n) * 1e-3).astype(f)
    if n >= 8:                 # pairs where fma(wd, w, g) differs from wd*w + g: g cancels most of wd*w
        k = n // 4
        g[:k] = -(f(WD) * w[:k]).astype(f) * f(1 + 2 ** -20)
    return w, v, g


def _mul_add(w, g):
    f = np.float32
    return ((f(WD) * w).astype(f) + g).astype(f)


def test_optimizer_and_cast_with_no_elements(tops):
    """n = 0 with valid pointers is a no-op (torch hands out NULL for empty tensors, so the C entry points are called
    directly)."""
    from frcnn_b200.ops import _p, _stream
    lib = tops._lib.load()
    w, v, g = (torch.full((4,), x, device=DEV) for x in (1.0, 2.0, 3.0))
    dst = _sentinel(4)
    for st in (lib.frcnn_sgd_momentum(_p(w), _p(v), _p(g), 0, LR, MOM, WD, _stream()),
               lib.frcnn_sgd_momentum_bf16g(_p(w), _p(v), _p(dst), 0, LR, MOM, WD, _stream()),
               lib.frcnn_cast_f32_bf16(_p(g), _p(dst), 0, _stream())):
        assert st == 0
    torch.cuda.synchronize()
    assert (w == 1).all() and (v == 2).all() and (br.bits(dst) == SENT).all()


@pytest.mark.parametrize("n", list(range(1, 10)) + [2 ** 20 + 3])
def test_sgd_momentum_bit_exact(tops, n):
    w, v, g = _opt_data(n, n)
    wt, vt, gt = (torch.from_numpy(a.copy()).to(DEV) for a in (w, v, g))
    tops.sgd_momentum(wt, vt, gt, LR, MOM, WD)
    want_w, want_v = br.sgd_momentum(w, v, g, LR, MOM, WD)
    torch.cuda.synchronize()
    assert np.array_equal(wt.cpu().numpy().view(np.int32), want_w.view(np.int32))
    assert np.array_equal(vt.cpu().numpy().view(np.int32), want_v.view(np.int32))
    if n >= 8:                 # the data tells fma from multiply-then-add
        assert (br.fmaf(np.full_like(w, np.float32(WD)), w, g) != _mul_add(w, g)).any()
    # bf16 gradient: the same rule on the reduced bf16 values
    gb = torch.from_numpy(g).to(DEV).to(torch.bfloat16)
    wt2, vt2 = (torch.from_numpy(a.copy()).to(DEV) for a in (w, v))
    tops.sgd_momentum_bf16g(wt2, vt2, gb, LR, MOM, WD)
    want_w2, want_v2 = br.sgd_momentum(w, v, gb.float().cpu().numpy(), LR, MOM, WD)
    torch.cuda.synchronize()
    assert np.array_equal(wt2.cpu().numpy().view(np.int32), want_w2.view(np.int32))
    assert np.array_equal(vt2.cpu().numpy().view(np.int32), want_v2.view(np.int32))


def _cast_patterns(n_random, seed):
    special = np.array([
        0x3F808000, 0x3F818000, 0x3F807FFF, 0xBF808000, 0xBF818000,        # ties to even, below a tie
        0x7F7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0xFF7FFFFF,                    # overflow to inf, largest finite
        0x00000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x80018000,        # subnormals
        0x00000000, 0x80000000, 0x7F800000, 0xFF800000,                    # zeros, infinities
        0x7FC00000, 0xFFC00001, 0x7F800001, 0x7FFFFFFF], np.uint32)        # NaNs (quiet, signalling)
    rng = np.random.default_rng(seed)
    rnd = rng.integers(0, 2 ** 32, n_random, dtype=np.uint64).astype(np.uint32)
    return np.concatenate([special, rnd]).view(np.float32)


@pytest.mark.parametrize("n,off", [(n, 0) for n in range(1, 10)] + [(7, 4), (9, 8), (1000003, 4), (4096, 12)])
def test_cast_f32_bf16_matches_torch_rne(tops, n, off):
    src_all = _cast_patterns(max(n + off, 32), n)
    src_t = torch.from_numpy(src_all.copy()).to(DEV)
    dst = _sentinel(len(src_all))
    tops.cast_f32_bf16(src_t[off:off + n], dst[off:off + n])
    torch.cuda.synchronize()
    want = torch.from_numpy(src_all[off:off + n].copy()).to(torch.bfloat16)     # torch's CPU RNE
    assert_bits(dst[off:off + n].cpu(), want, "cast")
    assert (br.bits(dst[:off]) == SENT).all() and (br.bits(dst[off + n:]) == SENT).all()


def test_cast_f32_bf16_alignment_errors(tops):
    from frcnn_b200._lib import FrcnnError
    src = torch.zeros((64,), device=DEV)
    dst = torch.zeros((64,), dtype=torch.bfloat16, device=DEV)
    with pytest.raises(FrcnnError):
        tops.cast_f32_bf16(src[1:9], dst[0:8])          # src 4 bytes off 16-byte alignment
    with pytest.raises(FrcnnError):
        tops.cast_f32_bf16(src[0:8], dst[2:10])         # dst 4 bytes off 8-byte alignment


# ------------------------------------------------------------------ G. dropout
@pytest.mark.parametrize("invert", [False, True])
def test_dropout_exhaustive(tops, ops, invert):
    """All 65,536 hi (and lo) patterns under mask on and off: bf16(x * 2) kept, x * 0 dropped (sign of zero kept,
    inf * 0 and NaN give NaN)."""
    pat = br.all_bf16_patterns()
    hi = br.from_bits(pat, DEV)
    lo = br.from_bits(pat[::-1].copy(), DEV)
    mask = (torch.arange(hi.numel(), device=DEV) % 2 == (1 if invert else 0)).to(torch.uint8)
    want = [(t.float() * torch.where(mask.bool(), 2.0, 0.0)).to(torch.bfloat16) for t in (hi, lo)]
    a = ops.Act(hi.clone(), lo.clone())
    tops.dropout_(a, mask)
    torch.cuda.synchronize()
    assert_bits(a.hi, want[0], "hi")
    assert_bits(a.lo, want[1], "lo")
    x = hi.float()
    dropped = ~mask.bool()
    assert torch.isnan(a.hi.float()[dropped & torch.isinf(x)]).all()
    assert torch.equal(torch.signbit(a.hi.float()[dropped & torch.isfinite(x)]), torch.signbit(x[dropped & torch.isfinite(x)]))
    b = ops.Act(hi.clone(), None)                        # lo absent
    tops.dropout_(b, mask)
    torch.cuda.synchronize()
    assert_bits(b.hi, want[0], "hi only")


# ------------------------------------------------------------------ H. roi_pool_backward
def _rois(R, H, W, inv_scale, gen_np):
    """RoIs in image coordinates: random ones plus partly / fully outside the map, degenerate (x2 < x1), single-pixel and
    larger than the map."""
    Wi, Hi = W * inv_scale, H * inv_scale
    xy = gen_np.uniform(-0.2 * Wi, Wi, (R, 2)) * [1, Hi / Wi]
    wh = gen_np.uniform(0, 0.6 * Wi, (R, 2)) * [1, Hi / Wi]
    r = np.hstack([xy, xy + wh])
    special = [[-50, -50, Wi + 50, Hi + 50], [Wi + 10, Hi + 10, Wi + 100, Hi + 90], [40, 40, 20, 10], [3, 3, 3, 3],
               [-30, 5, 10, 40], [Wi - 5, Hi - 5, Wi + 200, Hi + 200], [0, 0, inv_scale * 0.5, inv_scale * 0.5]]
    r[:len(special)] = special
    return r.astype(np.float32)


@pytest.mark.parametrize("H,W,C,R_cap,count,outh,outw,scale,feat_kind,lo", [
    (19, 25, 8, 40, None, 7, 7, 1.0 / 16, "relu", True),
    (19, 25, 520, 40, 33, 7, 7, 1.0 / 16, "integer", True),
    (19, 25, 64, 40, 60, 14, 14, 1.0 / 16, "relu", False),
    (30, 41, 8, 25, 25, 3, 5, 1.0 / 8, "integer", False),
    (38, 63, 512, 300, 300, 7, 7, 1.0 / 16, "relu", True)])
def test_roi_pool_backward_matches_float64(tops, ops, H, W, C, R_cap, count, outh, outw, scale, feat_kind, lo):
    gen_np = np.random.default_rng(H * C + R_cap)
    gen = _gen(H * C + R_cap)
    if feat_kind == "relu":
        fv = torch.randn((H, W, C), device=DEV, generator=gen).clamp_min(0)            # many zero ties
    else:
        fv = torch.randint(0, 4, (H, W, C), device=DEV, generator=gen).float()         # positive ties
    f_hi, f_lo = br.split(fv)
    if not lo:
        f_lo = None
    feat = ops.Act(f_hi, f_lo)
    rois = _rois(R_cap, H, W, round(1 / scale), gen_np)
    g_hi, g_lo = _pair((1, R_cap, outh * outw * C), gen, lo=lo)
    cnt = None if count is None else torch.tensor([count], dtype=torch.int32, device=DEV)
    rt = torch.from_numpy(rois).to(DEV)
    d1 = tops.roi_pool_backward(feat, rt, cnt, ops.Act(g_hi, g_lo), outh=outh, outw=outw, scale=scale)
    d2 = tops.roi_pool_backward(feat, rt, cnt, ops.Act(g_hi, g_lo), outh=outh, outw=outw, scale=scale)
    torch.cuda.synchronize()
    assert torch.equal(d1, d2)
    R = R_cap if count is None else min(count, R_cap)
    fval = br.value(f_hi, f_lo).cpu().numpy()
    gval = br.value(g_hi, g_lo).double().cpu().numpy().reshape(R_cap, outh, outw, C)[:R]
    _, am = br.roi_pool_argmax(fval, rois[:R], outh, outw, scale)
    want = br.roi_pool_backward(am, gval, H, W)
    err = float(np.abs(d1.cpu().numpy() - want).max())
    print("roi_pool_backward %dx%dx%d R=%d %dx%d: max err %.2e of %.2e" % (H, W, C, R, outh, outw, err, np.abs(want).max()))
    assert err <= 1e-6 * np.abs(want).max()


def test_roi_pool_backward_workspace_too_small(tops, ops):
    from frcnn_b200._lib import FrcnnError
    f = ops.Act(*_pair((5, 6, 8), _gen(1)))
    g = ops.Act(*_pair((1, 2, 49 * 8), _gen(2)))
    rois = torch.tensor([[0, 0, 40, 40], [8, 8, 60, 70]], dtype=torch.float32, device=DEV)
    need = tops._lib.load().frcnn_roi_pool_backward_workspace_bytes(5, 6, 8)
    with pytest.raises(FrcnnError):
        tops.roi_pool_backward(f, rois, None, g, ws=torch.empty((need - 8,), dtype=torch.uint8, device=DEV))
    torch.cuda.synchronize()


def test_stream_synchronize_waits_for_the_stream(ops):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.full((1 << 22,), 3.0, device=DEV) * 2
    ops.stream_synchronize(s)
    assert s.query() and float(x[-1]) == 6.0


def test_pack_image_im2col3x3_dense_entry_equals_strided(tops, ops):
    """frcnn_pack_image_im2col3x3 (dense (C,H,W) source) writes what the strided entry behind ops.pack_image_im2col
    writes, bit for bit, hi and lo."""
    from frcnn_b200.ops import _p, _stream
    x = torch.randn((3, 37, 45), device=DEV, generator=_gen(9)) * 50
    want = ops.pack_image_im2col(x)
    hi, lo = _sentinel(37 * 45 * 32).view(37, 45, 32), _sentinel(37 * 45 * 32).view(37, 45, 32)
    assert tops._lib.load().frcnn_pack_image_im2col3x3(_p(x), 3, 37, 45, _p(hi), _p(lo), _stream()) == 0
    torch.cuda.synchronize()
    assert_bits(hi, want.hi, "hi")
    assert_bits(lo, want.lo, "lo")
