"""Plain float64 references of the ResNet trunk's memory-bound kernels (csrc/resnet_ops.cu) and the per-element error
bound the trunk's convolutions are held to.  torch on any device: the CPU tests check them against torch's own operators
and explicit loops, the GPU tests run them on the device next to the kernels."""
import torch
import torch.nn.functional as F


def conv_out(e, ks, stride, pad):
    """Output size of a ks / stride / pad convolution over e pixels; 0 when not even one window fits."""
    t = e + 2 * pad - ks
    return t // stride + 1 if t >= 0 else 0


def pool3s2_out(c):
    """Output size of Chainer's max_pooling_2d(3, stride=2, pad=0, cover_all=True) over c pixels; 0 for c < 2."""
    return (c - 2) // 2 + 1 if c >= 2 else 0


def split_rne(x):
    """float32 tensor -> (hi, lo) bf16 planes as the device splits a value: hi = RNE-bf16(x), lo = RNE-bf16(x - hi)."""
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def pair_value(hi, lo):
    """The float64 value bf16 planes stand for (DESIGN §2): hi + lo, or hi alone where hi is +-inf or NaN (the split of
    +-inf has lo = NaN) or where there is no lo plane (bf16 mode)."""
    h = hi.double()
    if lo is None:
        return h
    return torch.where(torch.isfinite(h), h + lo.double(), h)


def maxpool_cover_all(x, eh=None, ew=None, out_hw=None):
    """Chainer max_pooling_2d(x, 3, stride=2) (pad 0, cover_all) of an [H, W, C] map, restated from its definition.

    Output pixel (i, j) is the maximum over rows [2i, 2i + 3) and columns [2j, 2j + 3), clipped to the image's eh x ew
    top-left pixels (a canvas slot holds a smaller image; default the whole map), for i < pool3s2_out(eh) and
    j < pool3s2_out(ew).  out_hw pads the result with +0.0 to the slot's output size.  The maximum follows DESIGN §2: NaN
    is dropped unless every value in the window is NaN, and +0.0 ranks above -0.0."""
    H, W, C = x.shape
    eh = H if eh is None else eh
    ew = W if ew is None else ew
    oh, ow = pool3s2_out(eh), pool3s2_out(ew)
    Ho, Wo = out_hw if out_hw is not None else (oh, ow)
    out = torch.zeros((Ho, Wo, C), dtype=torch.float64, device=x.device)
    if oh == 0 or ow == 0:
        return out
    x = x.double()
    best = torch.full((oh, ow, C), float("-inf"), dtype=torch.float64, device=x.device)
    any_num = torch.zeros((oh, ow, C), dtype=torch.bool, device=x.device)
    pos_zero = torch.zeros_like(any_num)
    for dy in range(3):
        rows = 2 * torch.arange(oh, device=x.device) + dy
        for dx in range(3):
            cols = 2 * torch.arange(ow, device=x.device) + dx
            v = x[rows.clamp(max=eh - 1)][:, cols.clamp(max=ew - 1)]
            inside = (rows < eh)[:, None, None] & (cols < ew)[None, :, None]
            num = inside & ~torch.isnan(v)
            best = torch.where(num, torch.maximum(best, v), best)
            any_num |= num
            pos_zero |= num & (v == 0) & ~torch.signbit(v)
    res = torch.where(any_num, best, torch.full_like(best, float("nan")))
    zero = res == 0
    res = torch.where(zero & pos_zero, torch.zeros_like(res), res)
    res = torch.where(zero & ~pos_zero, torch.full_like(res, -0.0), res)
    out[:oh, :ow] = res
    return out


def im2col(x, ks, stride, pad, k_pad, eh=None, ew=None, out_hw=None):
    """The first-layer im2col of a (C, H, W) image: [Ho, Wo, k_pad] float64, K index (r*ks + s)*C + c, from F.unfold.

    Taps outside the image's eh x ew top-left pixels (default the whole image) read as the zero padding; output pixels
    past conv_out(extent) (up to out_hw, the slot's output size) and columns [ks*ks*C, k_pad) are 0."""
    C, H, W = x.shape
    eh = H if eh is None else eh
    ew = W if ew is None else ew
    oh, ow = conv_out(eh, ks, stride, pad), conv_out(ew, ks, stride, pad)
    Ho, Wo = out_hw if out_hw is not None else (oh, ow)
    out = torch.zeros((Ho, Wo, k_pad), dtype=torch.float64, device=x.device)
    if oh == 0 or ow == 0:
        return out
    u = F.unfold(x[None, :, :eh, :ew].double(), ks, padding=pad, stride=stride)[0]      # [(c, r, s), oh*ow]
    out[:oh, :ow, :ks * ks * C] = u.view(C, ks * ks, oh, ow).permute(2, 3, 1, 0).reshape(oh, ow, ks * ks * C)
    return out


def elementwise_error(dev, ref, bound):
    """max over elements of |dev - ref| / bound, all float64.  bound is the same computation on absolute values
    (sum |x|*|w| + |b| + |residual|), so an error in a small-magnitude region (a border pixel, the last partial tile)
    counts as much as one in the largest.  Where the bound is 0 the result must be exact; a NaN, or a miss where the
    bound is 0, gives inf."""
    d = (dev - ref).abs()
    r = torch.where(bound > 0, d / bound, torch.where(d > 0, float("inf"), 0.0))
    r = torch.where(torch.isnan(d), float("inf"), r)
    return float(r.max()) if r.numel() else 0.0


def maxnorm_error(dev, ref):
    """max |dev - ref| / max |ref|: the figure the older tests print."""
    return float((dev - ref).abs().max() / ref.abs().max().clamp_min(1e-300))
