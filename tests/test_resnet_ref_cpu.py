"""CPU checks of the float64 references in tests/resnet_ref.py, which the ResNet GPU tests hold the kernels to."""
import numpy as np
import pytest
import torch

import resnet_ref as rr
from test_conv_gemm_coverage_gpu import TOL_ACT, conv_ref

# the im2col geometries of the GPU tests: ks, stride, pad in 0 .. ks//2 + 1
IM2COL_GEOMETRIES = [(ks, st, pad) for ks in (1, 3, 5, 7, 11) for st in (1, 2, 4) for pad in range(ks // 2 + 2)]


def im2col_sizes(ks, stride, pad):
    """Image sides for a geometry: 1 upward, smaller than the filter, and both parities past it; only sides with an output."""
    cand = {1, 2, 3, ks - 1, ks, ks + 1, 2 * ks + 1, 2 * ks + 2}
    return sorted(e for e in cand if e > 0 and rr.conv_out(e, ks, stride, pad) > 0)


def test_cover_all_pool_equals_torch_ceil_mode_on_finite_data():
    """On finite data Chainer's cover_all pool and torch's ceil_mode pool are the same operation, at every H and W in
    1..24; a side of 1 has no output (torch refuses it)."""
    g = torch.Generator().manual_seed(0)
    for H in range(1, 25):
        for W in range(1, 25):
            x = torch.randn((H, W, 5), generator=g, dtype=torch.float64)
            got = rr.maxpool_cover_all(x)
            if H == 1 or W == 1:
                assert got.numel() == 0
                continue
            want = F_pool(x)
            assert got.shape == want.shape and torch.equal(got, want), (H, W)


def F_pool(x):
    return torch.nn.functional.max_pool2d(x.permute(2, 0, 1)[None], 3, 2, ceil_mode=True)[0].permute(1, 2, 0)


def test_cover_all_pool_special_values_and_extents():
    """NaN is dropped unless the whole window is NaN, +0.0 ranks above -0.0 in either order, +-inf are ordinary
    values, and a canvas extent clips the windows and zero-fills the slot."""
    nan, inf = float("nan"), float("inf")
    x = torch.tensor([[nan, 1.0, -2.0], [-nan, nan, 0.5], [3.0, nan, -inf]], dtype=torch.float64)[:, :, None]
    assert rr.maxpool_cover_all(x).item() == 3.0
    assert torch.isnan(rr.maxpool_cover_all(torch.full((3, 3, 1), nan, dtype=torch.float64))).all()
    for a, b in ((-0.0, 0.0), (0.0, -0.0)):
        z = torch.tensor([[a, b], [-inf, -inf]], dtype=torch.float64)[:, :, None]
        r = rr.maxpool_cover_all(z).item()
        assert r == 0 and not np.signbit(r)
    z = torch.tensor([[-0.0, -0.0], [nan, -inf]], dtype=torch.float64)[:, :, None]
    assert np.signbit(rr.maxpool_cover_all(z).item())
    assert rr.maxpool_cover_all(torch.full((4, 4, 1), -inf, dtype=torch.float64)).eq(-inf).all()
    # a 5x5 image in an 8x8 slot: windows clipped at the image's border, the slot's other outputs +0.0
    g = torch.Generator().manual_seed(1)
    x = torch.randn((8, 8, 3), generator=g, dtype=torch.float64)
    got = rr.maxpool_cover_all(x, 5, 5, out_hw=(4, 4))
    assert torch.equal(got[:2, :2], F_pool(x[:5, :5]))
    assert not got[2:].any() and not got[:, 2:].any()


def im2col_loops(x, ks, stride, pad, k_pad):
    """im2col by explicit loops (numpy float64), the definition the unfold-based reference restates."""
    C, H, W = x.shape
    Ho, Wo = rr.conv_out(H, ks, stride, pad), rr.conv_out(W, ks, stride, pad)
    out = np.zeros((Ho, Wo, k_pad))
    for i in range(Ho):
        for j in range(Wo):
            for r in range(ks):
                for s in range(ks):
                    h, w = i * stride - pad + r, j * stride - pad + s
                    if 0 <= h < H and 0 <= w < W:
                        out[i, j, (r * ks + s) * C:(r * ks + s + 1) * C] = x[:, h, w]
    return out


@pytest.mark.parametrize("ks,stride,pad", IM2COL_GEOMETRIES, ids=lambda v: str(v))
def test_im2col_reference_equals_loops(ks, stride, pad):
    rng = np.random.default_rng(ks * 100 + stride * 10 + pad)
    C = 3
    k_pad = -(-ks * ks * C // 8) * 8 + 8
    sizes = im2col_sizes(ks, stride, pad)
    for H in sizes:
        for W in sizes[::2] + [sizes[-1]]:
            x = rng.standard_normal((C, H, W))
            got = rr.im2col(torch.from_numpy(x), ks, stride, pad, k_pad).numpy()
            assert np.array_equal(got, im2col_loops(x, ks, stride, pad, k_pad)), (H, W)
    # an extent inside a larger slot equals the cropped image, zero-padded to the slot's output size
    H = W = sizes[-1] + 3
    x = rng.standard_normal((C, H, W))
    eh, ew = sizes[0], sizes[-1]
    Ho, Wo = rr.conv_out(H, ks, stride, pad), rr.conv_out(W, ks, stride, pad)
    got = rr.im2col(torch.from_numpy(x), ks, stride, pad, k_pad, eh, ew, out_hw=(Ho, Wo)).numpy()
    want = np.zeros_like(got)
    sub = im2col_loops(x[:, :eh, :ew], ks, stride, pad, k_pad)
    want[:sub.shape[0], :sub.shape[1]] = sub
    assert np.array_equal(got, want)


def test_elementwise_bound_zero_on_exact_and_flags_a_border_pixel():
    """The per-element bound is 0 on an exact result, and it flags one perturbed border pixel of a small-magnitude
    border that the max-norm check lets through."""
    g = torch.Generator().manual_seed(2)
    H, W, Cin, Cout = 9, 13, 16, 8
    x = torch.randn((H, W, Cin), generator=g, dtype=torch.float64)
    x[:, -2:] *= 1e-3                                  # small-magnitude last columns, as at an image border
    w = torch.randn((9, Cout, Cin), generator=g, dtype=torch.float64) / 12
    b = torch.randn((Cout,), generator=g, dtype=torch.float64) * 1e-3
    ref = conv_ref(x, w, b, 3)
    bound = conv_ref(x.abs(), w.abs(), b.abs(), 3)
    assert rr.elementwise_error(ref.clone(), ref, bound) == 0.0
    tol = TOL_ACT["bf16x3"]
    dev = ref.clone()
    dev[H - 1, W - 1, 3] += 10 * tol * bound[H - 1, W - 1, 3]
    assert rr.maxnorm_error(dev, ref) < tol
    assert rr.elementwise_error(dev, ref, bound) > tol
    dev[0, 0, 0] = float("nan")
    assert rr.elementwise_error(dev, ref, bound) == float("inf")
    # where the bound is 0 (an all-zero window without bias) only the exact value passes
    zb = torch.zeros(3, dtype=torch.float64)
    assert rr.elementwise_error(zb, zb, zb) == 0.0
    assert rr.elementwise_error(zb + 1e-300, zb, zb) == float("inf")


def test_pair_value_and_split():
    x = torch.tensor([1.0 + 2 ** -10, float("inf"), float("-inf"), -0.0], dtype=torch.float32)
    hi, lo = rr.split_rne(x)
    v = rr.pair_value(hi, lo)
    assert v[0] == 1.0 + 2 ** -10 and v[1] == float("inf") and v[2] == float("-inf")
    assert torch.isnan(lo[1].float()) and v[3] == 0
    assert torch.equal(rr.pair_value(hi, None), hi.double())
