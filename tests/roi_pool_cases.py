"""The RoI-pooling edge matrix shared by the CPU tests (oracle vs restatement, torchvision, the UBSan build) and the GPU
tests (test_roi_pool_edges_gpu.py): bin geometries, RoIs at rounding ties and past the int32 range, non-finite RoIs, and
feature maps whose windows hold ties, huge negatives, -inf, NaN, +inf, subnormal lo parts and half-ulp lo parts."""
import numpy as np
import torch

import backward_ref as br

f32 = np.float32
OUT_SIZES = [(1, 1), (1, 31), (31, 1), (31, 31), (2, 3), (7, 7), (14, 14)]
SCALES = [1.0 / 16, 1.0 / 32, 1.0 / 8, 1.0, 0.3]
POW2_SCALES = SCALES[:4]
QNAN, NQNAN = np.array([0x7FC00000, 0xFFC00000], np.uint32).view(f32)
NONFINITE_COORDS = [QNAN, NQNAN, f32(np.inf), f32(-np.inf), f32(1e12), f32(-1e12)]
H, W = 37, 41                            # odd both ways; tall enough for heights of 2 * 14 + 1 rows


def geometry_rois(H, W, scale, outh, outw, rng, n_random=12):
    """RoIs in image coordinates (x1, y1, x2, y2) for a map of H x W at `scale`: half-way ties of coord * scale on both
    signs, signed zeros and subnormals, x2 < x1, single pixels on the last row and column, RoIs larger than the map,
    partly and fully outside it, heights below the bin count and heights of k*outh and k*outh +- 1, and random ones."""
    s = 1.0 / scale
    r = [[(k + 0.5) * s, (j + 0.5) * s, (k + 3.5) * s, (j + 4.5) * s] for k, j in ((0, 1), (2, 0), (5, 6))]
    r += [[-(k + 0.5) * s, -(j + 0.5) * s, (k + 1.5) * s, (j + 2.5) * s] for k, j in ((0, 0), (1, 2))]
    r += [[-0.0, -0.0, 4 * s, 3 * s], [1e-45, 1e-40, -1e-45, -1e-38], [-1e-45, 2e-45, 6 * s, 5 * s],
          [9 * s, 8 * s, 2 * s, 1 * s],                                  # x2 < x1, y2 < y1
          [(W - 1) * s, (H - 1) * s, (W - 1) * s, (H - 1) * s],           # the last pixel
          [(W - 1) * s, 2 * s, (W - 1) * s, 6 * s], [3 * s, (H - 1) * s, 9 * s, (H - 1) * s],
          [-5 * s, -7 * s, (W + 6) * s, (H + 3) * s],                     # larger than the map
          [-4 * s, (H - 3) * s, 3 * s, (H + 4) * s], [(W - 2) * s, -6 * s, (W + 9) * s, 2 * s],   # partly outside
          [(W + 2) * s, (H + 1) * s, (W + 9) * s, (H + 9) * s], [-20 * s, -15 * s, -5 * s, -1 * s],  # fully outside
          [0, 0, 2e9 * s, 2e9 * s], [-3e9 * s, -3e9 * s, 3e9 * s, 3e9 * s]]     # past the int32 range once scaled
    for k in (1, 2):
        for d in (-1, 0, 1):
            rh, rw = k * outh + d, k * outw + d
            if 1 <= rh <= H - 2:
                r.append([1 * s, 1 * s, (1 + max(min(rw, W - 2), 1) - 1) * s, (1 + rh - 1) * s])
            if 1 <= rw <= W - 2:
                r.append([2 * s, 0, (2 + rw - 1) * s, (max(min(rh, H - 1), 1) - 1) * s])
    if outh > 1:
        r.append([0, 3 * s, 6 * s, (3 + min(outh - 1, 3)) * s])          # fewer rows than bands: bands share rows
    xy = rng.uniform(-3, [W, H], (n_random, 2))
    wh = rng.uniform(0, [W, H], (n_random, 2))
    r += (np.hstack([xy, xy + wh]) * s).tolist()
    return np.array(r, f32)


def nonfinite_rois(H, W, scale):
    """NaN of both signs, +-inf and +-1e12 in each coordinate position of an ordinary RoI, and [0, 0, 1e12, 1e12]."""
    s = 1.0 / scale
    base = [2 * s, 3 * s, (W - 4) * s, (H - 5) * s]
    r = []
    for v in NONFINITE_COORDS:
        for j in range(4):
            roi = list(base)
            roi[j] = v
            r.append(roi)
    r += [[QNAN] * 4, [0, 0, 1e12, 1e12], [-1e12, -1e12, 1e12, 1e12], [np.inf, np.inf, -np.inf, -np.inf]]
    return np.array(r, f32)


FEATURE_KINDS = ["relu", "signed", "huge_neg", "neg_inf", "nan", "pos_inf", "tiny", "half_ulp"]


def features(kind, H, W, C, seed):
    """float32 [H,W,C] feature values of one kind; windows of all -inf / all NaN come from whole blocks of the map."""
    g = np.random.default_rng(seed)
    x = g.standard_normal((H, W, C)).astype(f32)
    if kind == "relu":
        x = np.maximum(x, 0)                                            # zero ties
    elif kind == "huge_neg":
        x = (f32(-1e37) * (1 + np.abs(x))).astype(f32)                  # every value <= -1e37
        x[:, ::5, ::3] = f32(-3.4e38)
    elif kind == "neg_inf":
        x[: H // 2] = -np.inf                                           # all -inf windows in the top half
        x[H // 2:, ::3] = -np.inf
    elif kind == "nan":
        x[: H // 2, : W // 2] = QNAN                                    # all-NaN windows in the top-left quarter
        x[H // 2:, ::2] = NQNAN
        x[:, :, ::7] = QNAN                                             # whole channels of NaN
    elif kind == "pos_inf":
        x[g.random((H, W, C)) < 0.03] = np.inf
        x[: H // 3, : W // 3, ::2] = -np.inf
    elif kind == "tiny":
        x = (x * f32(1.1754944e-38)).astype(f32)                        # near FLT_MIN: lo parts are subnormal
    elif kind == "half_ulp":
        hi = torch.from_numpy(x).to(torch.bfloat16).float().numpy()
        e = np.floor(np.log2(np.maximum(np.abs(hi), 1e-30)))
        half = np.exp2(e - 8).astype(f32)                               # ulp(hi) / 2 for a normal bf16 hi
        x = (hi + np.where(g.random(x.shape) < 0.5, half, -half)).astype(f32)
    return x


def split_planes(x, lo=True):
    """float32 [..] -> (hi, lo | None) bf16 CPU tensors: the canonical split of the conv epilogue."""
    hi, l = br.split(torch.from_numpy(np.ascontiguousarray(x)))
    return hi, (l if lo else None)


def pooled_input(hi, lo):
    """The float32 map the oracle pools for a split pair: common.cuh pool_pair_value."""
    return br.pool_value(hi, lo).numpy()


def oracle(feat_hwc, rois, outh, outw, scale):
    """frcnn_oracle.roi_pool on an [H,W,C] map and [R,4] RoIs -> [R, outh, outw, C]."""
    import frcnn_oracle as orc
    R = rois.shape[0]
    brois = np.hstack([np.zeros((R, 1), f32), rois]).astype(f32)
    out = orc.roi_pool(np.ascontiguousarray(feat_hwc.transpose(2, 0, 1))[None], brois, outh, outw, scale)
    return out.transpose(0, 2, 3, 1)
