"""datasets.pascal_voc_dataset.VOC -- synthetic stand-in with the interface of /root/reference
datasets/pascal_voc_dataset.py:14-51 (LABELS, IMG_TARGET_SIZE, IMG_MAX_SIZE, VOC(mode, use_difficult), len(),
dataset[i] -> (img float32 (3,H,W), im_info int array (H, W), gt_boxes float32 (n,5) = x1,y1,x2,y2,label)).

The reference class subclasses chainercv.datasets.VOCDetectionDataset, which reads PASCAL VOC from disk (downloading it
on first use); neither ChainerCV nor the dataset exists offline.  This stand-in produces, deterministically per index,
a random uint8 BGR image of a VOC-like size and 1-6 random ground-truth boxes, and then applies the SAME per-example
transform as the reference (:33-51): mean subtraction, scale the short side to 600 capped at 1000 on the long side,
bicubic resize (cv2 when importable, else a nearest-neighbour resample), CHW float32, boxes scaled by im_scale.
It exists so that the reference's tests/test_faster_rcnn.py (setUp: `VOC('train')[1]`) runs unchanged; it is test
data, not part of the detection path.
"""
import numpy as np

try:                                   # the reference resizes with OpenCV (:46-47)
    import cv2 as cv
except ImportError:                    # pragma: no cover
    cv = None

_SIZES = ((375, 500), (333, 500), (500, 375), (500, 500), (281, 500), (500, 334), (442, 500), (375, 1000))


class VOC(object):

    LABELS = ('__background__',  # always index 0
              'aeroplane', 'bicycle', 'bird', 'boat',
              'bottle', 'bus', 'car', 'cat', 'chair',
              'cow', 'diningtable', 'dog', 'horse',
              'motorbike', 'person', 'pottedplant',
              'sheep', 'sofa', 'train', 'tvmonitor')
    IMG_TARGET_SIZE = 600
    IMG_MAX_SIZE = 1000

    def __init__(self, mode='train', use_difficult=False, n_examples=16):
        if mode not in ('train', 'val', 'trainval', 'test'):
            raise ValueError("mode must be one of train / val / trainval / test")
        self.mode, self.use_difficult = mode, use_difficult
        self._n = int(n_examples)
        self._seed0 = {'train': 1000, 'val': 2000, 'trainval': 3000, 'test': 4000}[mode]
        self.mean = np.array([[[103.939, 116.779, 123.68]]])  # BGR (:31)

    def __len__(self):
        return self._n

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self.get_example(j) for j in range(*i.indices(self._n))]
        if i < 0:
            i += self._n
        if not 0 <= i < self._n:
            raise IndexError(i)
        return self.get_example(i)

    def _raw_example(self, i):
        """What VOCDetectionDataset.get_example returns: (img float32 CHW 0..255, bbox float32 (n,4), label int32 (n,))."""
        rng = np.random.RandomState(self._seed0 + i)
        h, w = _SIZES[rng.randint(len(_SIZES))]
        img = rng.randint(0, 256, size=(3, h, w)).astype(np.float32)
        n = rng.randint(1, 7)
        x1 = rng.uniform(0, w - 60, size=n)
        y1 = rng.uniform(0, h - 60, size=n)
        x2 = np.minimum(x1 + rng.uniform(40, w / 2.0, size=n), w - 1)
        y2 = np.minimum(y1 + rng.uniform(40, h / 2.0, size=n), h - 1)
        bbox = np.stack([x1, y1, x2, y2], axis=1).astype(np.float32)
        label = rng.randint(1, len(self.LABELS), size=n).astype(np.int32)
        return img, bbox, label

    def get_raw_example(self, i):
        """Example i before the transform: (uint8 (h, w, 3) BGR photo, float32 (n, 4) boxes in photo coordinates, int32 (n,)
        labels) -- what CanvasRpnTrainer / CanvasRcnnTrainer(raw_input=True).put_raw take.  Their device transform follows
        the reference (float32 mean subtraction, then the bicubic resize); get_example below subtracts the means in float64."""
        img, bbox, label = self._raw_example(i)
        return np.ascontiguousarray(img.transpose(1, 2, 0).astype(np.uint8)), bbox, label

    def get_example(self, i):
        img, bbox, label = self._raw_example(i)
        img = img.transpose(1, 2, 0)
        img = img - self.mean
        im_size_min = np.min(img.shape[:2])
        im_size_max = np.max(img.shape[:2])
        im_scale = float(self.IMG_TARGET_SIZE) / float(im_size_min)
        if np.round(im_scale * im_size_max) > self.IMG_MAX_SIZE:
            im_scale = float(self.IMG_MAX_SIZE) / float(im_size_max)
        if cv is not None:
            img = cv.resize(img, None, None, fx=im_scale, fy=im_scale, interpolation=cv.INTER_CUBIC)
        else:                                       # pragma: no cover
            H, W = int(round(img.shape[0] * im_scale)), int(round(img.shape[1] * im_scale))
            ys = np.minimum((np.arange(H) / im_scale).astype(int), img.shape[0] - 1)
            xs = np.minimum((np.arange(W) / im_scale).astype(int), img.shape[1] - 1)
            img = img[ys][:, xs]
        img = img.transpose(2, 0, 1).astype(np.float32)
        bbox = bbox * im_scale
        bbox = np.concatenate((bbox, label[:, None]), axis=1).astype(np.float32)
        return img, np.asarray(img.shape[1:]), bbox
