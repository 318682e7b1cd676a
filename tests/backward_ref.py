"""Bit-level and float64 restatements of the conv-backward and optimizer entry points (train_backward.cu, rcnn_train.cu),
the references of tests/test_backward_kernels_gpu.py.  They take the exact operand values the kernels read -- bf16 (hi, lo)
planes as torch.bfloat16 tensors, fp32 as float32 -- and run on whichever device the tensors live on: the large shapes are
restated on the GPU, the CPU tests (test_backward_ref_cpu.py) check the restatements themselves on small hand-worked cases.

Rounding primitive: torch's float32 -> bfloat16 conversion (round to nearest, ties to even, subnormals kept, overflow to
inf, NaN stays NaN); test_backward_ref_cpu.py pins that on hand-picked bit patterns."""
import math

import numpy as np
import torch

PAD_LEFT = 8


def padded_pixels(H, W):
    """(Kp, Wp) of the transposed padded layout (include/frcnn_b200.h, frcnn_padded_pixels)."""
    Wp = (W + PAD_LEFT + 1 + 7) // 8 * 8
    Kp = ((H + 2) * Wp + 63) // 64 * 64
    return Kp, Wp


def bits(t):
    """bf16 tensor -> int16 bit patterns (same device)."""
    return t.view(torch.int16)


def from_bits(u16, device="cpu"):
    """uint16 / int16 NumPy array of bf16 bit patterns -> bfloat16 tensor."""
    return torch.from_numpy(np.ascontiguousarray(u16).view(np.int16)).to(device).view(torch.bfloat16)


def all_bf16_patterns():
    """The 65,536 bf16 bit patterns in two orders, interleaved: element 2i = pattern i, element 2i + 1 = pattern i + 1, so
    every pattern sits once in the low and once in the high half of a 32-bit word (131,072 elements)."""
    p = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    return np.stack([p, np.roll(p, -1)], 1).reshape(-1)


def split(v):
    """float32 -> (hi, lo) bf16 with hi = RN(v), lo = RN(v - hi): the kernels' split_bf16."""
    hi = v.to(torch.bfloat16)
    return hi, (v - hi.float()).to(torch.bfloat16)


def value(hi, lo):
    """float32 value of a (hi, lo) pair as the kernels form it: one correctly rounded fp32 add."""
    return hi.float() if lo is None else hi.float() + lo.float()


def times2(x):
    """bf16(2 x), correctly rounded (float32 2x is exact or already inf)."""
    return (x.float() * 2).to(torch.bfloat16)


def positive(y_hi):
    """Chainer's y > 0 on the hi plane (y > 0 iff hi > 0 for a split value); False for NaN."""
    return y_hi.float() > 0


def route_keep(y_hi, y_lo, p_hi, p_lo):
    """F.max_pooling_2d backward routing (2x2, stride 2, ceil mode): True at the FIRST element, in (0,0), (0,1), (1,0), (1,1)
    order, of each window whose value equals the pooled value -- values compared, not bit patterns.  y [H,W,C], p pooled."""
    H, W, _ = y_hi.shape
    yv, pv = value(y_hi, y_lo), value(p_hi, p_lo)
    pv_full = pv.repeat_interleave(2, 0).repeat_interleave(2, 1)[:H, :W]
    hit = yv == pv_full
    keep = torch.zeros_like(hit)
    taken = torch.zeros_like(pv, dtype=torch.bool)
    for dh, dw in ((0, 0), (0, 1), (1, 0), (1, 1)):
        h_sub = hit[dh::2, dw::2]
        hh, ww = h_sub.shape[:2]
        first = h_sub & ~taken[:hh, :ww]
        keep[dh::2, dw::2] = first
        taken[:hh, :ww] |= first
    return keep


def grad_prepare(H, W, C, g=None, g_f32=None, y=None, p=None, planes=1, times2_=False):
    """frcnn_grad_prepare restated.  g: (hi, lo|None) [Hs,Ws,C]; g_f32: float32 [H*W, ld]; y / p: (hi, lo|None) pairs.
    Returns (o_hi, o_lo, t_hi, t_lo, written): the NHWC planes [H,W,C] and the transposed planes [planes,C,Kp], with the
    bool mask [Kp] of the columns the kernel stores (elsewhere the caller's buffer must be left as it was)."""
    if g_f32 is not None:
        ld = g_f32.shape[1]
        v = torch.zeros((H * W, C), dtype=torch.float32, device=g_f32.device)
        n = min(ld, C)
        v[:, :n] = g_f32[:, :n]
        hi, lo = split(v.view(H, W, C))
    elif p is not None:
        rep = lambda t: t.repeat_interleave(2, 0).repeat_interleave(2, 1)[:H, :W]
        hi = rep(g[0])
        lo = rep(g[1]) if g[1] is not None else torch.zeros_like(hi)
    else:
        hi = g[0]
        lo = g[1] if g[1] is not None else torch.zeros_like(hi)
    keep = torch.ones((H, W, C), dtype=torch.bool, device=hi.device)
    if y is not None:
        keep &= positive(y[0])
    if p is not None:
        keep &= route_keep(y[0], y[1], p[0], p[1])
    zero = torch.zeros((), dtype=torch.bfloat16, device=hi.device)
    hi, lo = torch.where(keep, hi, zero), torch.where(keep, lo, zero)
    if times2_:
        hi, lo = times2(hi), times2(lo)
    Kp, Wp = padded_pixels(H, W)
    W8 = (W + 7) // 8 * 8
    t = []
    for plane in (hi, lo):
        tp = torch.zeros((planes, C, Kp), dtype=torch.bfloat16, device=hi.device)
        # row h of the map sits at k = (h + 1) * Wp + PAD_LEFT + w; the kernel stores the 8-pixel groups w < W8
        grid = tp[:, :, Wp:Wp + H * Wp].view(planes, C, H, Wp)
        chw = plane.permute(2, 0, 1)
        for pl in range(planes):
            shift = pl - 1 if planes == 3 else 0                     # plane pl at k holds pixel k + pl - 1
            lo_w, hi_w = max(0, -shift), min(W8, W - shift)
            if hi_w > lo_w:
                grid[pl, :, :, PAD_LEFT + lo_w:PAD_LEFT + hi_w] = chw[:, :, lo_w + shift:hi_w + shift]
        t.append(tp)
    written = torch.zeros((Kp,), dtype=torch.bool, device=hi.device)
    written[Wp:Wp + H * Wp].view(H, Wp)[:, PAD_LEFT:PAD_LEFT + W8] = True
    return hi, lo, t[0], t[1], written


def pack_dgrad(w, cout_pad):
    """frcnn_pack_conv_weights_dgrad restated: OIHW float32 -> [taps, Cin, cout_pad] (hi, lo), out[t][ci][co] =
    W[co][ci][kh-1-r][kw-1-s] with t = r*kw + s, zero for co >= Cout."""
    Cout, Cin, kh, kw = w.shape
    rot = torch.flip(w, (2, 3)).permute(2, 3, 1, 0).reshape(kh * kw, Cin, Cout)
    full = torch.zeros((kh * kw, Cin, cout_pad), dtype=torch.float32, device=w.device)
    full[:, :, :Cout] = rot
    return split(full)


def wgrad_reduce(parts, M, N, scale):
    """frcnn_wgrad_reduce restated in its fixed order: acc = 0; acc += parts[g][s] for s = 0..S-1; dw = acc * scale (all
    float32 roundings), laid out OIHW: dw[m][n][g]."""
    groups, S = parts.shape[:2]
    acc = torch.zeros((groups, M, N), dtype=torch.float32, device=parts.device)
    for s in range(S):
        acc = acc + parts[:, s, :M, :N]
    acc = acc * torch.tensor(scale, dtype=torch.float32)
    return acc.permute(1, 2, 0).reshape(-1)


# ---------------------------------------------------------------------------------------------- optimizer (NumPy)
def fmaf(a, b, c):
    """Correctly rounded float32 fma(a, b, c) of float32 arrays: a*b is exact in float64, TwoSum gives p + c = s + e exactly,
    s is rounded to odd with e's sign (53 >= 24 + 2 bits: the final round to float32 is then correct -- no double rounding)."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bp = s - c64
    e = (p - bp) + (c64 - (s - bp))
    even = (s.view(np.int64) & 1) == 0
    nudge = (e != 0) & even & np.isfinite(s)
    s = np.where(nudge, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    with np.errstate(over="ignore"):
        return s.astype(np.float32)


def sgd_momentum(w, v, g, lr, momentum, weight_decay):
    """WeightDecay + MomentumSGD as frcnn_sgd_momentum computes it (float32): g' = fma(rate, w, g); v = mom*v - lr*g';
    w = w + v.  Returns (w, v)."""
    f = np.float32
    gi = fmaf(np.full_like(w, f(weight_decay)), w, g)
    vi = (f(momentum) * v).astype(f) - (f(lr) * gi).astype(f)
    return (w + vi).astype(f), vi.astype(f)


# ---------------------------------------------------------------------------------------------- RoI pooling (NumPy)
def pool_value(hi, lo):
    """float32 value of a (hi, lo) pair in RoI pooling (common.cuh pool_pair_value): hi + lo, or hi itself when hi is
    +-inf or NaN (the split of +-inf has lo = NaN).  A missing lo plane is zero, as in the kernels: -0.0 becomes +0.0."""
    h = hi.float()
    return torch.where(torch.isfinite(h), h + (0.0 if lo is None else lo.float()), h)


def roi_coord(coord, scale):
    """int32 of roundf(float32(coord * scale)) as the kernels convert it (common.cuh roi_coord): half away from zero,
    NaN -> 0, saturated to the int32 range."""
    with np.errstate(over="ignore", invalid="ignore"):
        x = float(np.float32(coord) * np.float32(scale))
    if x != x:
        return 0
    r = x if math.isinf(x) else math.copysign(math.floor(abs(x) + 0.5), x)    # float64 holds |x| + 0.5 exactly
    return int(min(max(r, -2 ** 31), 2 ** 31 - 1))


def roi_bin(s, e, P, i, L):
    """[lo, hi) of bin i of P over the scaled extent [s, e], clamped to [0, L] (common.cuh roi_bin; Python ints do not
    overflow, float32 for the bin size and the products)."""
    f32 = np.float32
    b = f32(max(e - s + 1, 1)) / f32(P)
    lo = int(np.floor(f32(i) * b)) + s
    hi = int(np.ceil(f32(i + 1) * b)) + s
    return min(max(lo, 0), L), min(max(hi, 0), L)


def roi_pool_argmax(feat, rois, outh, outw, scale):
    """F.roi_pooling_2d forward with arg-max under the rule of orc_roi_pool / roi_pool_backward_kernel (DESIGN §2).
    feat [H,W,C] float32, rois [R,4] float32 (x1,y1,x2,y2).  Returns (max [R,outh,outw,C] float32: 0 for an empty bin,
    -inf for a window with no number above -inf (NaN is ignored); argmax [R,outh,outw,C] int64 = y*W + x of the first
    maximum in (y, x) order, -1 for an empty bin and where the maximum is -inf)."""
    H, W, C = feat.shape
    R = rois.shape[0]
    mx = np.zeros((R, outh, outw, C), np.float32)
    am = np.full((R, outh, outw, C), -1, np.int64)
    for r in range(R):
        sw, sh, ew, eh = (roi_coord(rois[r, j], scale) for j in range(4))
        for ph in range(outh):
            hs, he = roi_bin(sh, eh, outh, ph, H)
            for pw in range(outw):
                ws, we = roi_bin(sw, ew, outw, pw, W)
                if he <= hs or we <= ws:
                    continue
                win = feat[hs:he, ws:we].reshape(-1, C)
                win = np.where(np.isnan(win), np.float32(-np.inf), win)
                k = np.argmax(win, 0)                                   # first maximum in (y, x) order
                m = win[k, np.arange(C)]
                mx[r, ph, pw] = m
                ww = we - ws
                am[r, ph, pw] = np.where(m > -np.inf, (hs + k // ww) * W + ws + k % ww, -1)
    return mx, am


def roi_pool_backward(am, g, H, W):
    """float64 scatter of the bins' gradient g [R,outh,outw,C] to their arg-max positions -> dfeat [H*W, C]."""
    C = g.shape[-1]
    out = np.zeros((H * W * C,), np.float64)
    idx = am.reshape(-1, C)
    gg = g.reshape(-1, C).astype(np.float64)
    ok = idx >= 0
    flat = idx * C + np.arange(C)[None, :]
    np.add.at(out, flat[ok], gg[ok])
    return out.reshape(H * W, C)
