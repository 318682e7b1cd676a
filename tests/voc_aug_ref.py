"""The VOC training transform with py-faster-rcnn's augmentation (TRAIN.USE_FLIPPED, TRAIN.SCALES) restated in NumPy: the
specification that frcnn_preprocess_voc_canvas_im2col_flip, frcnn_voc_flip_scale_gt_batch and the augmenting canvas
trainers match bit for bit.  Built on voc_ref's plain transform, which it equals with flip=False, scale=600."""
import numpy as np

from voc_ref import cubic_resize, f32, mean_subtract, plan_size


def flip_boxes(boxes, w0):
    """py-faster-rcnn's horizontal flip in the inclusive pixel convention, float32: x1' = (w0 - x2) - 1, x2' = (w0 - x1) - 1;
    y1 and y2 unchanged."""
    b = np.array(boxes, dtype=np.float32)
    x1, x2 = b[:, 0].copy(), b[:, 2].copy()
    b[:, 0] = (f32(w0) - x2) - f32(1)
    b[:, 2] = (f32(w0) - x1) - f32(1)
    return b


def voc_transform(photo, boxes, labels, flip=False, scale=600):
    """uint8 (h0, w0, 3) BGR photo, (G, 4) boxes, (G,) labels -> (float32 (3, H, W) image, (H, W), float32 (G, 5) ground
    truth): the photo p[:, ::-1] and the boxes flip_boxes' when `flip`, then VOC.get_example's transform at the short-side
    target `scale` (plan_size, max_size 1000)."""
    h0, w0, _ = photo.shape
    im_scale, H, W = plan_size(h0, w0, scale)
    img = cubic_resize(mean_subtract(photo[:, ::-1] if flip else photo), H, W, 1.0 / im_scale)
    bbox = (flip_boxes(boxes, w0) if flip else np.asarray(boxes, dtype=np.float32)) * np.float32(im_scale)
    gt = np.concatenate((bbox, np.asarray(labels)[:, None]), axis=1).astype(np.float32)
    return np.ascontiguousarray(img.transpose(2, 0, 1)), (H, W), gt
