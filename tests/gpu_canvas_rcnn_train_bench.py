"""Measurement (not a pytest): the RCNN training step on a stream of images of different sizes.

The stream is 600x{800, 901, 1000} images in turn (the shapes VOC photos take after the reference's resize to a short side
of 600), with synthetic ground truth, random-init VGG16 and bf16x3.  Modes:
  (a) per-shape  one RcnnTrainer per shape with its NumPy sampling (a host round trip per step); on every change of shape
                 the fp32 masters and momentum are copied into the next trainer (what a user can do without a canvas)
  (b) canvas N   CanvasRcnnTrainer on a 600x1000 canvas, N images per update (N = 1, 2, 4), device sampling and dropout
                 masks, graph replay
  (c) full size  every image 600x1000: RcnnTrainer against CanvasRcnnTrainer N = 1
Every mode is warmed up first; then the modes alternate round by round.  A round is ROUND_IMAGES images; its device time
comes from CUDA events around it (ending in a synchronise).  Reports the median and min-max device ms per image over the
rounds, images/s at the median and the device memory each mode holds (allocated after its warm-up, over the baseline).
Prints the card's name and power limit with the numbers, a markdown table and one JSON line."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
from frcnn_b200.train_engine import CanvasRcnnTrainer, RcnnTrainer  # noqa: E402

ROUNDS, ROUND_IMAGES = 7, 12
SHAPES = [(600, 800), (600, 901), (600, 1000)]
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stream(shapes, n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        h, w = shapes[k % len(shapes)]
        x = torch.from_numpy(orc.make_image(h, w, seed=k % 6)[0]).cuda()
        G = int(rng.integers(2, 8))
        x1, y1 = rng.uniform(0, w * 0.3, G), rng.uniform(0, h * 0.3, G)
        # large boxes: with random-init weights the proposals are arbitrary, and NumPy sampling must keep at least one RoI
        g = np.stack([x1, y1, np.minimum(x1 + rng.uniform(300, 700, G), w - 1), np.minimum(y1 + rng.uniform(250, 500, G), h - 1),
                      rng.integers(1, 21, G)], 1).astype(np.float32)
        out.append((x, torch.from_numpy(g).cuda()))
    return out


class PerShape(object):
    """(a): one RcnnTrainer per shape, masters and momentum handed on at every change of shape."""

    def __init__(self, params, shapes):
        self.tr = {s: RcnnTrainer(params, s[0], s[1], ANCHORS) for s in shapes}
        self.cur = None

    def run(self, images):
        for x, g in images:
            t = self.tr[tuple(x.shape[1:])]
            if self.cur is not None and self.cur is not t:
                t.w_flat.copy_(self.cur.w_flat)
                t.v_flat.copy_(self.cur.v_flat)
                t.repack()
            self.cur = t
            t.step(x, g)


class Canvas(object):
    """(b) / (c): CanvasRcnnTrainer.step on N images at a time."""

    def __init__(self, params, N):
        self.N, self.tr = N, CanvasRcnnTrainer(params, N, 600, 1000, ANCHORS)

    def run(self, images):
        for k in range(0, len(images), self.N):
            chunk = images[k:k + self.N]
            self.tr.step([x for x, _ in chunk], [g for _, g in chunk])


def main():
    params = orc.make_params(seed=1234)
    mixed = stream(SHAPES, ROUND_IMAGES)
    full = stream([(600, 1000)], ROUND_IMAGES, seed=1)
    modes = []
    base = torch.cuda.memory_allocated()
    np.random.seed(0)
    for name, build, images in [("(a) per-shape RcnnTrainer", lambda: PerShape(params, SHAPES), mixed),
                                ("(b) canvas N=1", lambda: Canvas(params, 1), mixed),
                                ("(b) canvas N=2", lambda: Canvas(params, 2), mixed),
                                ("(b) canvas N=4", lambda: Canvas(params, 4), mixed),
                                ("(c) 600x1000 RcnnTrainer", lambda: PerShape(params, [(600, 1000)]), full),
                                ("(c) 600x1000 canvas N=1", lambda: Canvas(params, 1), full)]:
        m = build()
        m.run(images)                                            # warm-up: every shape, the graph capture
        torch.cuda.synchronize()
        held = torch.cuda.memory_allocated() - base
        base = torch.cuda.memory_allocated()
        modes.append(dict(name=name, m=m, images=images, held_gb=held / 2 ** 30, ms=[]))
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(ROUNDS):
        for md in modes:
            ev0.record()
            md["m"].run(md["images"])
            ev1.record()
            torch.cuda.synchronize()
            md["ms"].append(ev0.elapsed_time(ev1) / len(md["images"]))
    gpu = card()
    rows = []
    print("card: %s; %d rounds of %d images per mode" % (gpu, ROUNDS, ROUND_IMAGES))
    print("| mode | ms / image (median) | min-max | images/s | memory held (GB) |")
    print("|---|---|---|---|---|")
    for md in modes:
        ms = np.array(md["ms"])
        med = float(np.median(ms))
        rows.append(dict(mode=md["name"], ms_median=med, ms_min=float(ms.min()), ms_max=float(ms.max()), images_per_s=1e3 / med,
                         memory_gb=md["held_gb"]))
        print("| %s | %.2f | %.2f-%.2f | %.1f | %.1f |" % (md["name"], med, ms.min(), ms.max(), 1e3 / med, md["held_gb"]))
    print(json.dumps(dict(card=gpu, rounds=ROUNDS, round_images=ROUND_IMAGES, rows=rows)))


if __name__ == "__main__":
    main()
