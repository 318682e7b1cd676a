"""CPU checks of the references in tests/backward_ref.py (the ones test_backward_kernels_gpu.py holds the kernels to), and a
guard that every C entry point of include/frcnn_b200.h is exercised by some test."""
import glob
import itertools
import os
import re
from fractions import Fraction

import numpy as np
import pytest
import torch

import backward_ref as br
import frcnn_oracle as orc
import roi_pool_cases as rpc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _b(u16):
    return br.from_bits(np.array(u16, np.uint16))


def _u16(t):
    return br.bits(t).numpy().view(np.uint16)


def test_bf16_rounding_primitive_is_rne():
    """torch's float32 -> bfloat16 conversion, the references' only rounding step: ties to even, subnormals kept, overflow
    to inf, NaN stays NaN."""
    cases = {0x3F808000: 0x3F80, 0x3F818000: 0x3F82, 0x3F808001: 0x3F81, 0xBF818000: 0xBF82, 0x7F7F7FFF: 0x7F7F,
             0x7F7F8000: 0x7F80, 0xFF7FFFFF: 0xFF80, 0x00008000: 0x0000, 0x00018000: 0x0002, 0x00007FFF: 0x0000,
             0x80000000: 0x8000, 0x7F800000: 0x7F80}
    x = torch.from_numpy(np.array(list(cases), np.uint32).view(np.float32))
    assert list(_u16(x.to(torch.bfloat16))) == list(cases.values())
    assert torch.isnan(torch.tensor([float("nan")]).to(torch.bfloat16).float()).all()


def test_times2_reference_on_special_values():
    x = _b([0x3F80, 0x0001, 0x0040, 0x807F, 0x7F00, 0x7F7F, 0xFF7F, 0x7F80, 0xFF80, 0x0000, 0x8000, 0x7FC0])
    got = br.times2(x)
    want = [0x4000, 0x0002, 0x0080, 0x80FE, 0x7F80, 0x7F80, 0xFF80, 0x7F80, 0xFF80, 0x0000, 0x8000]
    assert list(_u16(got)[:11]) == want and torch.isnan(got[11].float())


def test_positive_mask_reference():
    pat = br.all_bf16_patterns()
    keep = br.positive(br.from_bits(pat)).numpy()
    want = (pat >= 0x0001) & (pat <= 0x7F80)                   # (0, +inf]: positive numbers, NaN excluded
    assert np.array_equal(keep, want)


def _loop_grad_prepare(H, W, C, g, y, p, planes):
    """Element-by-element statement of frcnn_grad_prepare on float32 values (no lo planes) -> (NHWC [H,W,C], T [planes,C,Kp])."""
    Kp, Wp = br.padded_pixels(H, W)
    o = np.zeros((H, W, C), f32)
    for h, w, c in itertools.product(range(H), range(W), range(C)):
        if p is None:
            v = g[h, w, c]
        else:
            h0, w0 = h // 2 * 2, w // 2 * 2
            win = [(h0 + e // 2, w0 + e % 2) for e in range(4) if h0 + e // 2 < H and w0 + e % 2 < W]
            first = next((q for q in win if y[q[0], q[1], c] == p[h // 2, w // 2, c]), None)
            v = g[h // 2, w // 2, c] if first == (h, w) else 0
        if y is not None and not y[h, w, c] > 0:
            v = 0
        o[h, w, c] = v
    t = np.zeros((planes, C, Kp), f32)
    for pl, h, w in itertools.product(range(planes), range(H), range((W + 7) // 8 * 8)):
        src = w + pl - 1 if planes == 3 else w
        if 0 <= src < W:
            t[pl, :, (h + 1) * Wp + 8 + w] = o[h, src]
    return o, t


@pytest.mark.parametrize("H,W,C,pool,planes", [(3, 5, 8, True, 3), (4, 9, 16, True, 1), (2, 3, 8, False, 3), (1, 1, 8, False, 3)])
def test_grad_prepare_reference_matches_loop(H, W, C, pool, planes):
    rng = np.random.default_rng(H * W)
    y = np.maximum(rng.integers(-2, 3, (H, W, C)), 0).astype(f32)
    g_full = rng.integers(1, 9, (H, W, C)).astype(f32)
    p = None
    if pool:
        pad = np.full((H + H % 2, W + W % 2, C), -np.inf, f32)
        pad[:H, :W] = y
        p = pad.reshape((H + 1) // 2, 2, (W + 1) // 2, 2, C).max((1, 3))
        g_full = g_full[:(H + 1) // 2, :(W + 1) // 2]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(torch.bfloat16)
    o_hi, o_lo, t_hi, t_lo, written = br.grad_prepare(H, W, C, g=(t(g_full), None), y=(t(y), None),
                                                      p=(t(p), None) if pool else None, planes=planes)
    want_o, want_t = _loop_grad_prepare(H, W, C, g_full, y, p, planes)
    assert np.array_equal(o_hi.float().numpy(), want_o) and not o_lo.float().any()
    assert np.array_equal(t_hi.float().numpy(), want_t) and not t_lo.float().any()
    Kp, Wp = br.padded_pixels(H, W)
    assert Kp % 64 == 0 and Wp % 8 == 0 and Wp >= W + 9
    assert int(written.sum()) == H * ((W + 7) // 8 * 8)


def test_route_keep_first_of_tied_values_not_bits():
    """A 2x2 window with the maximum at (0,1) and (1,1); the pooled value is the other (hi, lo) split of the same value."""
    y_hi = torch.tensor([[1.0, 1.5], [0.5, 1.4375]]).to(torch.bfloat16)[..., None]
    y_lo = torch.tensor([[0.0, 0.0], [0.0, 0.0625]]).to(torch.bfloat16)[..., None]
    p_hi = torch.tensor([[1.4375]]).to(torch.bfloat16)[..., None]
    p_lo = torch.tensor([[0.0625]]).to(torch.bfloat16)[..., None]
    keep = br.route_keep(y_hi, y_lo, p_hi, p_lo)[..., 0]
    assert keep.tolist() == [[False, True], [False, False]]


def test_pack_dgrad_reference_matches_loop():
    rng = np.random.default_rng(0)
    w = rng.standard_normal((5, 3, 2, 3)).astype(f32)
    hi, lo = br.pack_dgrad(torch.from_numpy(w), 8)
    v = (hi.double() + lo.double()).numpy()
    for t, ci, co in itertools.product(range(6), range(3), range(8)):
        r, s = divmod(t, 3)
        want = w[co, ci, 1 - r, 2 - s] if co < 5 else 0.0
        assert abs(v[t, ci, co] - want) <= 2.0 ** -16 * abs(want)
    assert not hi[:, :, 5:].float().any()


def test_wgrad_reduce_reference_order():
    """acc += parts[s] in order s = 0..S-1, then * scale, each step rounded to float32."""
    parts = torch.tensor([1.0, 2.0 ** -24, 2.0 ** -24, -1.0], dtype=torch.float32).view(1, 4, 1, 1)
    assert br.wgrad_reduce(parts, 1, 1, 1.0).item() == 0.0              # (1 + e) + e rounds back to 1 twice
    parts = torch.arange(2 * 3 * 2 * 4, dtype=torch.float32).view(2, 3, 2, 4)
    got = br.wgrad_reduce(parts, 2, 3, 0.5).view(2, 3, 2)
    assert got[1, 2, 1].item() == 0.5 * float(parts[1, :, 1, 2].sum())


def _fma_exact(a, b, c):
    """Correctly rounded float32 a*b + c from exact rationals: nearest of the float32 neighbours, ties to even."""
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    r = f32(float(x))
    cands = [np.nextafter(r, f32(-np.inf)), r, np.nextafter(r, f32(np.inf))]
    best = min(cands, key=lambda q: (abs(Fraction(float(q)) - x), int(np.array(q).view(np.int32)) & 1))
    return f32(best)


def test_fmaf_is_correctly_rounded():
    # the double-rounding trap: a*b + c = 2^24 + 3 - 2^-46 rounds to the midpoint 2^24 + 3 in float64, whose float32
    # rounding (ties to even) is 2^24 + 4; the correct float32 result is 2^24 + 2
    a, b, c = (np.array([v], np.uint32).view(f32) for v in (0x3F800001, 0x3F7FFFFE, 0x4B800001))
    assert c[0] == 2 ** 24 + 2
    assert (a.astype(np.float64) * b + c).astype(f32)[0] == 2 ** 24 + 4
    assert br.fmaf(a, b, c)[0] == 2 ** 24 + 2
    rng = np.random.default_rng(1)
    n = 3000
    a = rng.standard_normal(n).astype(f32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(f32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(n) * 2.0 ** -rng.integers(5, 40, n))).astype(f32)
    got = br.fmaf(a, b, c)
    want = np.array([_fma_exact(*t) for t in zip(a, b, c)], f32)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_sgd_momentum_reference_rule():
    w, v, g = (np.array([x], f32) for x in (0.5, -0.25, 0.125))
    nw, nv = br.sgd_momentum(w, v, g, 0.001, 0.9, 0.0005)
    gi = f32(0.125) + f32(0.0005) * f32(0.5)                       # wd * 0.5 is exact: fma equals multiply-then-add here
    assert nv[0] == f32(f32(0.9) * f32(-0.25)) - f32(f32(0.001) * f32(gi)) and nw[0] == f32(0.5) + nv[0]


@pytest.mark.parametrize("outh,outw,scale", [(7, 7, 1.0 / 16), (3, 5, 1.0 / 8), (14, 14, 1.0 / 16)])
def test_roi_pool_argmax_max_equals_oracle(outh, outw, scale):
    """The restatement's maxima equal frcnn_oracle.roi_pool exactly (ReLU'd features: zero ties; RoIs outside the map,
    degenerate and rounding-tie RoIs); the arg-max points at a position holding that maximum, the first in (y, x) order."""
    rng = np.random.default_rng(outh * outw)
    H, W, C = 11, 17, 8
    feat = np.maximum(rng.standard_normal((H, W, C)), 0).astype(f32)
    feat[:, :, 3] = rng.integers(0, 3, (H, W))
    inv = round(1 / scale)
    xy = rng.uniform(-40, W * inv, (30, 2))
    rois = np.hstack([xy, xy + rng.uniform(0, 120, (30, 2))]).astype(f32)
    rois[:5] = [[-50, -50, W * inv + 50, H * inv + 50], [40, 40, 20, 10], [3, 3, 3, 3],
                [W * inv + 10, H * inv + 10, W * inv + 90, H * inv + 90], [0.5 * inv, 0.5 * inv, 1.5 * inv, 2.5 * inv]]
    mx, am = br.roi_pool_argmax(feat, rois, outh, outw, scale)
    brois = np.hstack([np.zeros((30, 1), f32), rois])
    want = orc.roi_pool(feat.transpose(2, 0, 1)[None], brois, outh, outw, scale).transpose(0, 2, 3, 1)
    assert np.array_equal(mx, want)
    flat = feat.reshape(H * W, C)
    ok = am >= 0
    assert np.array_equal(np.take_along_axis(flat, np.where(ok, am, 0).reshape(-1, C), 0).reshape(am.shape)[ok], mx[ok])
    assert (am[3] == -1).all() and (mx[3] == 0).all()                  # fully outside: every bin empty
    # the first maximum: a zero-tie window picks its first element in (y, x) order
    r, ph, pw, c = np.argwhere(ok & (mx == 0))[0]
    y0, x0 = divmod(int(am[r, ph, pw, c]), W)
    assert feat[y0, x0, c] == 0


@pytest.mark.parametrize("scale", rpc.SCALES)
@pytest.mark.parametrize("outh,outw", rpc.OUT_SIZES)
def test_roi_pool_argmax_equals_oracle_on_the_edge_matrix(outh, outw, scale):
    """The restatement equals frcnn_oracle.roi_pool bit for bit on every edge geometry, non-finite and out-of-range RoIs
    included, over features holding NaN, +-inf and values <= -1e37; its arg-max holds the maximum, and it is -1 exactly
    where the maximum is 0 of an empty bin or -inf."""
    rng = np.random.default_rng(outh * 64 + outw)
    rois = np.vstack([rpc.geometry_rois(rpc.H, rpc.W, scale, outh, outw, rng, n_random=4),
                      rpc.nonfinite_rois(rpc.H, rpc.W, scale)])
    feat = np.concatenate([rpc.features(k, rpc.H, rpc.W, 1, outh + outw) for k in ("nan", "pos_inf", "huge_neg", "relu")], 2)
    mx, am = br.roi_pool_argmax(feat, rois, outh, outw, scale)
    want = rpc.oracle(feat, rois, outh, outw, scale)
    assert np.array_equal(mx.view(np.uint32), want.view(np.uint32))
    ok = am >= 0
    C = feat.shape[2]
    held = np.take_along_axis(feat.reshape(-1, C), np.where(ok, am, 0).reshape(-1, C), 0).reshape(am.shape)
    assert np.array_equal(held[ok], mx[ok])
    assert ((mx == 0) | (mx == -np.inf))[~ok].all() and (mx > -np.inf)[ok].all()


def test_roi_pool_restatement_rule_known_answers():
    """roi_coord: half away from zero, NaN -> 0, saturation; roi_bin: no overflow past the int32 range."""
    assert [br.roi_coord(v, 1.0) for v in (2.5, -2.5, 0.49999997, -0.0, rpc.QNAN, rpc.NQNAN)] == [3, -3, 0, 0, 0, 0]
    assert [br.roi_coord(v, 1.0) for v in (np.inf, -np.inf, 1e12, -1e12, 2147483520.0)] == \
        [2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1, -2 ** 31, 2147483520]
    assert br.roi_bin(0, 2 ** 31 - 1, 2, 0, 5) == (0, 5) and br.roi_bin(0, 2 ** 31 - 1, 2, 1, 5) == (5, 5)
    assert br.roi_bin(-2 ** 31, 2 ** 31 - 1, 7, 3, 9) == (0, 9)        # bin 3 of 2^32 pixels: about [-3.1e8, 3.1e8)
    mx, am = br.roi_pool_argmax(np.array([[[np.nan]], [[-np.inf]]], f32), np.array([[0, 0, 0, 1]], f32), 1, 1, 1.0)
    assert mx[0, 0, 0, 0] == -np.inf and am[0, 0, 0, 0] == -1


def test_roi_pool_backward_scatter():
    am = np.array([[[[0, 3]], [[0, -1]]]])                             # R=1, 2x1 bins, C=2
    g = np.array([[[[1.5, 2.0]], [[0.25, 9.0]]]])
    d = br.roi_pool_backward(am, g, 2, 2)
    assert d[0, 0] == 1.75 and d[3, 1] == 2.0 and d.sum() == 3.75


# ---------------------------------------------------------------------------------------------- entry-point guard
# Entry points no test_*.py needs to reach: diagnostics and build metadata (each is exported and checked for presence by
# test_abi_cpu.py; none computes a result another entry point depends on).
UNTESTED_BY_DESIGN = {
    "frcnn_version",                 # build stamp, asserted by build()
    "frcnn_last_error",              # read by every failing call's FrcnnError message
    "frcnn_debug_sort_clocks",       # profiling hook of the top-k sort (tests/gpu_sort_profile.py)
    "frcnn_host_nms_phase_cycles",   # per-phase clock stamps of the host NMS (tests/gpu_host_api_profile.py)
}


# Entry points whose only front end lies outside ops / train_ops (the drop-in modules, the engine): the test file and the call
# in it that runs them.  Each is checked to be present, so a deleted test shows up here.
REACHED_THROUGH = {
    "frcnn_bbox_decode": ("test_dropin_gpu.py", "bt.bbox_transform_inv("),              # models.bbox_transform -> ops.bbox_decode
    "frcnn_bbox_transform": ("test_train_gpu.py", "bt.bbox_transform("),                # models.bbox_transform -> train_ops
    "frcnn_forward_vgg16": ("test_e2e_gpu.py", "CForward("),                            # engine.CForward, the one-call forward
    "frcnn_match_class_dets": ("test_dropin_gpu.py", "from models.cpu_nms import cpu_nms"),  # cpu_nms on a published result
    "frcnn_preprocess_bgr8": ("test_kernels_gpu.py", "preprocess.img_preprocessing("),  # frcnn_b200.preprocess
}


def _header_entry_points():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "frcnn_b200.h")).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(_nms|frcnn_[a-z0-9_]+)\s*\(", txt)))


def _front_end():
    """C entry point -> the ops / train_ops functions and classes that use it, directly or through one other ops / train_ops
    function or class (e.g. frcnn_linear_workspace_bytes -> linear_workspace -> linear)."""
    import ast
    uses = {}                                            # top-level ops / train_ops name -> names its body refers to
    for mod in ("ops", "train_ops"):
        tree = ast.parse(open(os.path.join(ROOT, "chainer-faster-rcnn_b200", "frcnn_b200", mod + ".py")).read())
        for top in tree.body:
            if isinstance(top, (ast.FunctionDef, ast.ClassDef)):
                uses[top.name] = {n.attr if isinstance(n, ast.Attribute) else n.id for n in ast.walk(top)
                                  if isinstance(n, (ast.Attribute, ast.Name))} - {top.name}
    out = {}
    for ep in _header_entry_points():
        first = {f for f, u in uses.items() if ep in u}
        # ops.Act is the activation container that nearly every front-end function builds; using it says nothing about
        # the one entry point its to_chw_f32 calls (frcnn_unpack_nhwc)
        out[ep] = first | {f for f, u in uses.items() if u & (first - {"Act"})}
    return out


def _unreached(test_files):
    """Header entry points (minus UNTESTED_BY_DESIGN) that none of `test_files` calls: neither by the C name on the loaded
    library (`lib.frcnn_x`) nor through its front-end function (`ops.f`, `train_ops.f`, `tops.f`) -- qualified names
    only, so a method or dict call of the same name does not count."""
    text = "\n".join(open(p).read() for p in test_files)
    wrappers = _front_end()
    missing = []
    for ep in _header_entry_points():
        if ep in UNTESTED_BY_DESIGN:
            continue
        if ep in REACHED_THROUGH:
            fname, call = REACHED_THROUGH[ep]
            if not any(os.path.basename(p) == fname and call in open(p).read() for p in test_files):
                missing.append(ep)
            continue
        pats = [r"\.%s\b" % re.escape(ep)] + [r"\b_?(?:ops|train_ops|tops)\.%s\b" % re.escape(w) for w in sorted(wrappers.get(ep, ()))]
        if not any(re.search(pt, text) for pt in pats):
            missing.append(ep)
    return missing


def _suite_files(exclude=()):
    skip = {"test_backward_ref_cpu.py", "test_abi_cpu.py"} | set(exclude)      # test_abi_cpu.py only checks symbols exist
    return sorted(p for p in glob.glob(os.path.join(ROOT, "tests", "test_*.py")) if os.path.basename(p) not in skip)


def test_every_entry_point_is_exercised_by_a_test():
    """Each C entry point is called in some tests/test_*.py, on the library or through its own ops / train_ops function."""
    missing = _unreached(_suite_files())
    assert not missing, "entry points no test reaches: %s" % missing
    assert (UNTESTED_BY_DESIGN | set(REACHED_THROUGH)) <= set(_header_entry_points())


def test_entry_point_guard_flags_an_unreached_entry_point():
    """Without the backward-kernel tests, the bf16 gradient-bucket entry points are reached by no test: the guard says so."""
    missing = _unreached(_suite_files(exclude=("test_backward_kernels_gpu.py",)))
    assert {"frcnn_cast_f32_bf16", "frcnn_sgd_momentum_bf16g"} <= set(missing), missing
