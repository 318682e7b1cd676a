"""GPU tests of RoI pooling against the CPU oracle at every bin geometry and on non-finite RoIs and features.

Kernels: roi_pool_col_kernel (frcnn_roi_pool, frcnn_roi_pool_batch) and roi_pool_backward_kernel (frcnn_roi_pool_backward).
The forward is compared with frcnn_oracle.roi_pool bit for bit, on its fp32 output and on the value of its packed (hi, lo)
planes, for the rule of DESIGN §2: the bins of roi_coord / roi_bin (common.cuh), NaN ignored, -inf for a window with no
number above -inf, 0 for an empty bin.  The edge matrix is tests/roi_pool_cases.py.  Memory safety is checked with guard
words after every output, never by reading or writing out of bounds.
"""
import ctypes

import numpy as np
import pytest
import torch

import backward_ref as br
import roi_pool_cases as rpc

pytestmark = pytest.mark.gpu
f32 = np.float32
GUARD = 4096                                 # elements of guard after every output
GUARD_BF16, GUARD_F32 = -12288.0, -2.0 ** 100   # exact in bf16 / fp32; no pooling of these inputs produces them


@pytest.fixture(scope="module")
def ops():
    from frcnn_b200 import ops as _ops
    return _ops


def assert_bits(got, want, what):
    g = np.ascontiguousarray(got, f32)
    w = np.ascontiguousarray(want, f32)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = g.view(np.uint32) != w.view(np.uint32)
    if bad.any():
        at = np.argwhere(bad)[:6]
        show = ["%s: got %08x want %08x" % (tuple(int(i) for i in ix), g.view(np.uint32)[tuple(ix)],
                                            w.view(np.uint32)[tuple(ix)]) for ix in at]
        raise AssertionError("%s: %d of %d values differ; %s" % (what, int(bad.sum()), bad.size, "; ".join(show)))


def _bf16_buf(n):
    return torch.full((n + GUARD,), GUARD_BF16, dtype=torch.bfloat16, device="cuda")


def _f32_buf(n):
    return torch.full((n + GUARD,), GUARD_F32, dtype=torch.float32, device="cuda")


def run_roi_pool(feat_hi, feat_lo, rois, count, outh, outw, scale, outputs):
    """frcnn_roi_pool through the C ABI.  outputs: a subset of {"hi", "lo", "f32"}; count: None (NULL) or an int.
    Returns {name: float32 [R_cap, outh, outw, C] CPU array}, after checking that every guard word is untouched."""
    from frcnn_b200 import _lib, ops as _ops
    H, W, C = feat_hi.shape
    R_cap = rois.shape[0]
    n = R_cap * outh * outw * C
    bufs = {"hi": _bf16_buf(n) if "hi" in outputs else None, "lo": _bf16_buf(n) if "lo" in outputs else None,
            "f32": _f32_buf(n) if "f32" in outputs else None}
    cnt = None if count is None else torch.tensor([count], dtype=torch.int32, device="cuda")
    fh = feat_hi.cuda()
    fl = None if feat_lo is None else feat_lo.cuda()
    rt = torch.from_numpy(np.ascontiguousarray(rois, f32)).cuda()
    _lib.check(_lib.load().frcnn_roi_pool(_ops._p(fh), _ops._p(fl), H, W, C, _ops._p(rt), _ops._p(cnt), R_cap, outh, outw,
                                          ctypes.c_float(scale), _ops._p(bufs["hi"]), _ops._p(bufs["lo"]),
                                          _ops._p(bufs["f32"]), _ops._stream()), "frcnn_roi_pool")
    torch.cuda.synchronize()
    res = {}
    for k, b in bufs.items():
        if b is None:
            continue
        guard = GUARD_BF16 if k != "f32" else GUARD_F32
        assert (b[n:].float() == guard).all(), "%s: a guard word after the output was written" % k
        res[k] = b[:n].float().cpu().numpy().reshape(R_cap, outh, outw, C)
    return res


def want_pool(hi, lo, rois, count, outh, outw, scale):
    """The oracle's output for the split planes (their pool_pair_value), rows at or past the count zero."""
    R_cap = rois.shape[0]
    R = R_cap if count is None else max(0, min(count, R_cap))
    want = np.zeros((R_cap, outh, outw, hi.shape[2]), f32)
    if R:
        want[:R] = rpc.oracle(rpc.pooled_input(hi, lo), rois[:R], outh, outw, scale)
    return want


def check_forward(hi, lo, rois, count, outh, outw, scale, outputs=("hi", "lo", "f32")):
    got = run_roi_pool(hi, lo, rois, count, outh, outw, scale, outputs)
    want = want_pool(hi, lo, rois, count, outh, outw, scale)
    if "f32" in got:
        assert_bits(got["f32"], want, "f32 output")
    if "lo" in got:                                  # the planes hold bf16 values: the float32 copies convert exactly
        ph, pl = (torch.from_numpy(got[k]).to(torch.bfloat16) for k in ("hi", "lo"))
        assert_bits(br.pool_value(ph, pl).numpy(), want, "value of the (hi, lo) planes")
        if lo is None:
            assert (got["lo"] == 0).all(), "the lo output of a bf16 input must be zero"
    elif "hi" in got and lo is None:
        assert_bits(br.pool_value(torch.from_numpy(got["hi"]).to(torch.bfloat16), None).numpy(), want,
                    "hi plane of a bf16 input")
    return got, want


# ------------------------------------------------------------------------------------------------ geometry
@pytest.mark.parametrize("scale", rpc.SCALES)
@pytest.mark.parametrize("outh,outw", rpc.OUT_SIZES)
def test_geometry_matrix(outh, outw, scale):
    """Every output size x scale on the edge RoIs (half-way ties of both signs, signed zeros, subnormal coordinates, x2 <
    x1, last row / column, larger than / partly / fully outside the map, bands sharing rows, heights k*outh and k*outh +- 1)
    and non-finite RoIs; C = 24 has a partial last channel slice at every outw."""
    rng = np.random.default_rng(outh * 1000 + outw)
    rois = np.vstack([rpc.geometry_rois(rpc.H, rpc.W, scale, outh, outw, rng), rpc.nonfinite_rois(rpc.H, rpc.W, scale)])
    hi, lo = rpc.split_planes(rpc.features("signed", rpc.H, rpc.W, 24, 11))
    check_forward(hi, lo, rois, None, outh, outw, scale)


# ------------------------------------------------------------------------------------------------ channels and outputs
OUTPUT_SETS = {"hi": ("hi",), "hi_lo": ("hi", "lo"), "f32": ("f32",), "all": ("hi", "lo", "f32")}


@pytest.mark.parametrize("outputs", list(OUTPUT_SETS))
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("C", [8, 16, 24, 56, 64, 200, 512, 520, 1024, 2048])
def test_channels_precisions_outputs(C, precision, outputs):
    """Every c8_per_cta (1 .. 64 channel groups per CTA at outw 7) and partial last slices, bf16 and bf16x3 inputs, and
    the output sets hi, hi + lo, f32 and all three."""
    H, W = 9, 13
    rng = np.random.default_rng(C)
    rois = rpc.geometry_rois(H, W, 1.0 / 16, 7, 7, rng, n_random=6)[::2]
    hi, lo = rpc.split_planes(rpc.features("signed", H, W, C, C), lo=precision == "bf16x3")
    got, want = check_forward(hi, lo, rois, len(rois) - 2, 7, 7, 1.0 / 16, OUTPUT_SETS[outputs])
    if outputs == "hi" and lo is not None:             # the hi plane alone is the hi of the same pairs
        full = run_roi_pool(hi, lo, rois, len(rois) - 2, 7, 7, 1.0 / 16, ("hi", "lo"))
        assert_bits(got["hi"], full["hi"], "hi plane with and without lo")


# ------------------------------------------------------------------------------------------------ launch shape, counts
@pytest.mark.parametrize("count", [None, 0, 1, "cap", "cap+5", -3])
@pytest.mark.parametrize("shape", [(64, 2, 2, 9000), (520, 1, 31, 1000)])     # 9000 CTAs of 1 slice; 1000 x 9 slices
def test_grid_stride_and_counts(shape, count):
    """R_cap * slices above the grid cap (132 * 64 CTAs), so that a CTA walks several RoIs, and counts NULL, 0, 1, R_cap,
    R_cap + 5 and negative: rows at or past the count are zero, the guard words after the output untouched."""
    C, outh, outw, R_cap = shape
    H, W = 6, 7
    rng = np.random.default_rng(R_cap)
    base = np.vstack([rpc.geometry_rois(H, W, 1.0 / 16, outh, outw, rng), rpc.nonfinite_rois(H, W, 1.0 / 16)])
    rois = base[rng.integers(0, len(base), R_cap)]
    cnt = {"cap": R_cap, "cap+5": R_cap + 5}.get(count, count)
    hi, lo = rpc.split_planes(rpc.features("relu", H, W, C, 5))
    got, _ = check_forward(hi, lo, rois, cnt, outh, outw, 1.0 / 16)
    R = R_cap if cnt is None else max(0, min(cnt, R_cap))
    for k in got:
        assert (got[k][R:] == 0).all() and not np.signbit(got[k][R:]).any(), k


# ------------------------------------------------------------------------------------------------ features
@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("kind", rpc.FEATURE_KINDS)
def test_feature_values(kind, precision):
    """Canonical split pairs of post-ReLU values (zero ties), values <= -1e37, all -inf and all NaN windows, +inf,
    magnitudes near FLT_MIN (subnormal lo parts) and lo parts of exactly +-ulp(hi)/2, pooled over the edge RoIs."""
    rng = np.random.default_rng(len(kind))
    rois = np.vstack([rpc.geometry_rois(rpc.H, rpc.W, 1.0 / 16, 7, 7, rng), rpc.nonfinite_rois(rpc.H, rpc.W, 1.0 / 16)])
    hi, lo = rpc.split_planes(rpc.features(kind, rpc.H, rpc.W, 40, 17), lo=precision == "bf16x3")
    for outh, outw in ((7, 7), (2, 3), (14, 14)):
        check_forward(hi, lo, rois, None, outh, outw, 1.0 / 16)


# ------------------------------------------------------------------------------------------------ batch
@pytest.mark.parametrize("N", [1, 2, 3])
def test_batch_equals_one_image_and_oracle(ops, N):
    """frcnn_roi_pool_batch: per-image counts, NaN RoIs in image 1 only, and outputs one gap of guard words apart per
    image.  Each image equals its one-image call and the oracle; the gaps are left untouched."""
    H, W, C, R_cap, outh, outw, scale = 11, 14, 72, 40, 7, 7, 1.0 / 16
    rng = np.random.default_rng(N)
    feats = [rpc.features(k, H, W, C, 30 + n) for n, k in zip(range(N), ("signed", "nan", "pos_inf"))]
    hi = torch.stack([rpc.split_planes(f)[0] for f in feats])
    lo = torch.stack([rpc.split_planes(f)[1] for f in feats])
    rois = np.stack([rpc.geometry_rois(H, W, scale, outh, outw, rng, n_random=R_cap)[:R_cap] for _ in range(N)])
    if N > 1:
        rois[1, ::3] = rpc.nonfinite_rois(H, W, scale)[: len(rois[1, ::3])]
    counts = [R_cap, R_cap - 7, 3][:N]
    K = outh * outw * C
    E, gap = R_cap * K, 136                                          # the image stride E + gap is a multiple of 8
    oh = torch.full((N, E + gap), GUARD_BF16, dtype=torch.bfloat16, device="cuda")
    ol = torch.full_like(oh, GUARD_BF16)
    o32 = torch.full((N, E + gap), GUARD_F32, dtype=torch.float32, device="cuda")
    ops.roi_pool_batch(ops.Act(hi.cuda(), lo.cuda()), torch.from_numpy(rois).cuda(),
                       torch.tensor(counts, dtype=torch.int32, device="cuda"), outh, outw, scale,
                       out=ops.Act(oh[:, :E].view(N, R_cap, K), ol[:, :E].view(N, R_cap, K)),
                       out_f32=o32[:, :E].view(N, R_cap, outh * outw, C))
    torch.cuda.synchronize()
    assert (oh[:, E:].float() == GUARD_BF16).all() and (ol[:, E:].float() == GUARD_BF16).all()
    assert (o32[:, E:] == GUARD_F32).all()
    for n in range(N):
        shape = (R_cap, outh, outw, C)
        one = run_roi_pool(hi[n], lo[n], rois[n], counts[n], outh, outw, scale, ("hi", "lo", "f32"))
        assert_bits(oh[n, :E].float().cpu().numpy().reshape(shape), one["hi"], "image %d hi" % n)
        assert_bits(ol[n, :E].float().cpu().numpy().reshape(shape), one["lo"], "image %d lo" % n)
        assert_bits(o32[n, :E].cpu().numpy().reshape(shape), one["f32"], "image %d f32" % n)
        assert_bits(one["f32"], want_pool(hi[n], lo[n], rois[n], counts[n], outh, outw, scale), "image %d vs oracle" % n)


# ------------------------------------------------------------------------------------------------ forward / backward
@pytest.mark.parametrize("kind,lo,outh,outw", [("relu", True, 7, 7), ("nan", True, 7, 7), ("pos_inf", True, 2, 3),
                                               ("neg_inf", False, 14, 14), ("huge_neg", True, 31, 1)])
def test_backward_routes_to_the_forward_maximum(ops, kind, lo, outh, outw):
    """On one RoI and feature matrix, frcnn_roi_pool_backward equals backward_ref.roi_pool_backward on
    backward_ref.roi_pool_argmax (the float64 tolerance of test_backward_kernels_gpu.py), and every arg-max pixel holds
    the forward's output: -inf windows and empty bins route nothing."""
    from frcnn_b200 import train_ops as tops
    H, W, C, scale = 19, 25, 32, 1.0 / 16
    rng = np.random.default_rng(outh * outw)
    rois = np.vstack([rpc.geometry_rois(H, W, scale, outh, outw, rng), rpc.nonfinite_rois(H, W, scale)])
    R_cap = len(rois)
    hi, l = rpc.split_planes(rpc.features(kind, H, W, C, 3), lo=lo)
    fwd = run_roi_pool(hi, l, rois, None, outh, outw, scale, ("f32",))["f32"]
    fval = rpc.pooled_input(hi, l)
    mx, am = br.roi_pool_argmax(fval, rois, outh, outw, scale)
    assert_bits(fwd, mx, "forward vs restatement")
    ok = am >= 0
    held = np.take_along_axis(fval.reshape(-1, C), np.where(ok, am, 0).reshape(-1, C), 0).reshape(am.shape)
    assert_bits(held[ok], fwd[ok], "arg-max pixel vs forward")
    assert ((fwd == 0) | (fwd == -np.inf))[~ok].all()
    g = torch.from_numpy(rng.standard_normal((1, R_cap, outh * outw * C)).astype(f32))
    g_hi, g_lo = br.split(g)
    d = tops.roi_pool_backward(ops.Act(hi.cuda(), None if l is None else l.cuda()), torch.from_numpy(rois).cuda(), None,
                               ops.Act(g_hi.cuda(), g_lo.cuda()), outh=outh, outw=outw, scale=scale)
    torch.cuda.synchronize()
    gval = br.value(g_hi, g_lo).double().numpy().reshape(R_cap, outh, outw, C)
    want = br.roi_pool_backward(am, gval, H, W)
    err = float(np.abs(d.cpu().numpy() - want).max())
    assert np.isfinite(d.cpu().numpy()).all()
    assert err <= 1e-6 * max(np.abs(want).max(), 1.0), err
