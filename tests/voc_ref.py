"""The VOC training dataset's per-example transform (datasets/pascal_voc_dataset.py VOC.get_example) restated in NumPy: the
specification that frcnn_preprocess_voc_canvas_im2col and frcnn_voc_scale_gt_batch match bit for bit.

cubic_resize is OpenCV's generic float INTER_CUBIC (imgproc resize.cpp: resizeGeneric_ with HResizeCubic and VResizeCubic),
which cv2.resize runs on a float32 image when IPP is off (cv2.ipp.setUseIPP(False)); it equals that bit for bit.  With IPP
on (the default), cv2 4.13 hands float cubic to Intel IPP, whose arithmetic is not published.  Two differences are visible:
IPP keeps the source coordinate in double where OpenCV rounds it to float, which moves a tap by up to 2^-24 * 1000 =
6e-5 pixel and the result by that times the local slope (up to about 2 * 255 per pixel for the cubic), and it sums the taps
in another order (a few float ulps).  Measured over the test photos: 4.6e-5 where the coordinates are exact (scales 1.6 and
2.0), up to 7.1e-3 at 600/334; IPP_BOUND holds the bound the slope argument gives.
"""
import numpy as np

VOC_MEANS = np.array([103.939, 116.779, 123.68])       # BGR
IPP_BOUND = 6e-5 * 2 * 255                            # 3.1e-2; measured 7.1e-3
f32 = np.float32


def cubic_taps(n_out, n_in, inv_scale):
    """Per output index: the four clamped source indices [n_out, 4], the four float32 weights [4][n_out] and the border
    flag [n_out] of one axis (OpenCV's xofs / alpha / xmin-xmax)."""
    with np.errstate(invalid="ignore", over="ignore"):
        f = ((np.arange(n_out, dtype=np.float64) + 0.5) * inv_scale - 0.5).astype(np.float32)
        fl = np.floor(f)
        t = (f - fl).astype(np.float32)
    t[~((t >= 0) & (t < 1))] = 0                          # f = +-inf or NaN
    fl = np.where(np.isnan(fl), f32(-2), np.clip(fl, -2, n_in + 1))
    s = fl.astype(np.int64)
    border = (s < 1) | (s + 2 >= n_in)
    idx = np.clip(s[:, None] + np.arange(-1, 3)[None], 0, n_in - 1)
    A, one = f32(-0.75), f32(1)
    x1, y = t + one, one - t
    c0 = ((A * x1 - f32(5) * A) * x1 + f32(8) * A) * x1 - f32(4) * A
    c1 = ((A + f32(2)) * t - (A + f32(3))) * t * t + one
    c2 = ((A + f32(2)) * y - (A + f32(3))) * y * y + one
    c3 = one - c0 - c1 - c2
    return idx, [c0, c1, c2, c3], border


def cubic_resize(img, H, W, inv_scale):
    """float32 (h0, w0, C) -> float32 (H, W, C), OpenCV's float INTER_CUBIC with the scale 1 / inv_scale on both axes."""
    h0, w0, C = img.shape
    xi, xc, xb = cubic_taps(W, w0, inv_scale)
    yi, yc, _ = cubic_taps(H, h0, inv_scale)
    p = [img[:, xi[:, k]] * xc[k][None, :, None] for k in range(4)]
    h = np.where(xb[None, :, None], f32(0) + p[0], p[0])           # a border column's sum starts from 0.0f
    h = ((h + p[1]) + p[2]) + p[3]
    q = [h[yi[:, k]] * yc[k][:, None, None] for k in range(4)]
    vec = (((q[3] + q[2]) + q[1]) + q[0]).reshape(H, W * C)        # the 4-lane vector loop of VResizeCubicVec_32f
    tail = (((q[0] + q[1]) + q[2]) + q[3]).reshape(H, W * C)       # its scalar remainder
    end = (W * C) // 4 * 4
    return np.concatenate([vec[:, :end], tail[:, end:]], axis=1).reshape(H, W, C)


def plan_size(h0, w0, scale=600, max_size=1000):
    """VOC.get_example's im_scale and cv.resize's output size (round half to even)."""
    im_scale = float(scale) / float(min(h0, w0))
    if np.round(im_scale * max(h0, w0)) > max_size:
        im_scale = float(max_size) / float(max(h0, w0))
    return im_scale, int(np.rint(h0 * im_scale)), int(np.rint(w0 * im_scale))


def mean_subtract(photo, means=VOC_MEANS):
    """The reference's `img -= self.mean` on a float32 image: float32(double(u8) - mean_c)."""
    return (photo.astype(np.float64) - np.asarray(means, dtype=np.float64)).astype(np.float32)


def voc_transform(photo, boxes, labels):
    """uint8 (h0, w0, 3) BGR photo, (G, 4) boxes, (G,) labels -> (float32 (3, H, W) image, (H, W), float32 (G, 5) ground
    truth), as VOC.get_example computes them."""
    h0, w0, _ = photo.shape
    im_scale, H, W = plan_size(h0, w0)
    img = cubic_resize(mean_subtract(photo), H, W, 1.0 / im_scale)
    bbox = np.asarray(boxes, dtype=np.float32) * np.float32(im_scale)
    gt = np.concatenate((bbox, np.asarray(labels)[:, None]), axis=1).astype(np.float32)
    return np.ascontiguousarray(img.transpose(2, 0, 1)), (H, W), gt
