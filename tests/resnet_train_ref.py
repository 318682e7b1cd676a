"""Bit-exact restatements of the re-layouts the ResNet trunk's backward adds (include/frcnn_b200.h:
frcnn_maxpool3x3s2_backward, frcnn_grad_prepare_stride2) on bf16 hi/lo planes, and of the transposed padded layout they
write.  torch on any device; the CPU tests check them against torch autograd, the GPU tests against the kernels."""
import torch

from resnet_ref import pool3s2_out, split_rne

PAD_LEFT = 8


def pair_f32(hi, lo):
    """The float32 value of a split pair as the kernels read it: hi + lo (fp32 add), hi alone where hi is +-inf or NaN;
    a missing lo plane reads as +0."""
    h = hi.float()
    lo_f = torch.zeros_like(h) if lo is None else lo.float()
    return torch.where(torch.isfinite(h), h + lo_f, h)


def positive(hi):
    """y > 0 as the kernels test it: the bf16 bits read as int16 lie in (0, +inf] (NaN, +-0 and negatives excluded)."""
    b = hi.view(torch.int16).int()
    return (b > 0) & (b <= 0x7F80)


def _masked(acc_hi, acc_lo, keep):
    z = torch.zeros_like(acc_hi)
    return torch.where(keep, acc_hi, z), (None if acc_lo is None else torch.where(keep, acc_lo, z))


def maxpool3x3s2_backward(g_hi, g_lo, y_hi, y_lo, p_hi, p_lo):
    """frcnn_maxpool3x3s2_backward on [.., .., C] planes: window (i, j) sends g[i][j] to the first element of rows
    [2i, min(2i+3, H)) x columns [2j, min(2j+3, W)) in scan order whose value equals p[i][j]; each pixel sums what it
    receives in float32 in ascending (i, j) order from +0; the sum is kept where y > 0 and re-split.  Returns (hi, lo)."""
    H, W, C = y_hi.shape
    ph, pw = pool3s2_out(H), pool3s2_out(W)
    dev = y_hi.device
    yv, pv, gv = pair_f32(y_hi, y_lo), pair_f32(p_hi, p_lo), pair_f32(g_hi, g_lo)
    taken = torch.zeros((ph, pw, C), dtype=torch.bool, device=dev)
    hits = {}
    for dy in range(3):                                     # window element (dy, dx), scan order
        rows = 2 * torch.arange(ph, device=dev) + dy
        for dx in range(3):
            cols = 2 * torch.arange(pw, device=dev) + dx
            inside = (rows < H)[:, None, None] & (cols < W)[None, :, None]
            v = yv[rows.clamp(max=H - 1)][:, cols.clamp(max=W - 1)]
            hits[dy, dx] = inside & (v == pv) & ~taken
            taken |= hits[dy, dx]
    # a pixel (r, c) is element (dy, dx) of window ((r - dy) / 2, (c - dx) / 2): descending dy, dx is ascending (i, j)
    acc = torch.zeros((H, W, C), dtype=torch.float32, device=dev)
    for dy in (2, 1, 0):
        for dx in (2, 1, 0):
            sub = acc[dy::2, dx::2]
            nr, nc = min(ph, sub.shape[0]), min(pw, sub.shape[1])
            s = sub[:nr, :nc]
            s.copy_(torch.where(hits[dy, dx][:nr, :nc], s + gv[:nr, :nc], s))
    hi, lo = split_rne(acc)
    return _masked(hi, lo if g_lo is not None else None, positive(y_hi))


def grad_prepare_stride2(g_hi, g_lo, H, W, y_hi=None):
    """frcnn_grad_prepare_stride2: g's words at pixels (2i, 2j) of an H x W map, +0 elsewhere, then y > 0 when y is given."""
    C = g_hi.shape[-1]
    hi = torch.zeros((H, W, C), dtype=torch.bfloat16, device=g_hi.device)
    lo = None if g_lo is None else torch.zeros_like(hi)
    hi[0::2, 0::2] = g_hi
    if lo is not None:
        lo[0::2, 0::2] = g_lo
    if y_hi is None:
        return hi, lo
    return _masked(hi, lo, positive(y_hi))


def padded_pixels(H, W):
    """(Kp, Wp) of the transposed padded layout (frcnn_padded_pixels)."""
    Wp = (W + PAD_LEFT + 1 + 7) // 8 * 8
    return ((H + 2) * Wp + 63) // 64 * 64, Wp


def transposed(a, planes):
    """[H, W, C] plane -> the transposed padded planes [planes, C, Kp] the kernels write: pixel (h, w) at
    k = (h+1)*Wp + 8 + w.  The kernels store whole 8-pixel groups, columns w < W8 = W rounded up to 8; column w of plane j
    holds pixel w + j - 1 when planes = 3 (pixel w when planes = 1), 0 where that pixel is outside the map.  Every other
    column is 0."""
    H, W, C = a.shape
    Kp, Wp = padded_pixels(H, W)
    W8 = (W + 7) // 8 * 8
    out = torch.zeros((planes, C, Kp), dtype=a.dtype, device=a.device)
    src = torch.zeros((H, W8 + 2, C), dtype=a.dtype, device=a.device)
    src[:, 1:W + 1] = a                                                       # src column 1 + w = pixel w
    for pl in range(planes):
        shift = pl - 1 if planes == 3 else 0
        view = out[pl].view(C, -1)[:, :(H + 2) * Wp].view(C, H + 2, Wp)
        view[:, 1:H + 1, PAD_LEFT:PAD_LEFT + W8] = src[:, 1 + shift:1 + shift + W8].permute(2, 0, 1)
    return out
