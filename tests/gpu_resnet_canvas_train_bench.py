"""Measurement (not a pytest): the ResNet training steps on a stream of images of different sizes, on one GPU.

Workloads, random-init ResNet-50 and ResNet-101 (frozen BN), bf16x3, synthetic ground truth:
  stream      600x{800, 901, 1000} images in turn (the shapes VOC photos take after the dataset's resize), for the RPN and
              the RCNN step:
                (a) per-shape  one ResNetRpnTrainer / ResNetRcnnTrainer per shape (RCNN: NumPy sampling, a host round trip
                               per step); on every change of shape the fp32 masters and momentum are copied into the next
                               trainer (what a user can do without a canvas)
                (b) canvas N   CanvasResNetRpnTrainer / CanvasResNetRcnnTrainer on a 600x1000 canvas, N images per update
                               (N = 1, 2, 4), device subsampling / sampling and dropout, graph replay
  raw         raw 375x500, 333x500 and 500x375 uint8 photos, ResNet-101, N = 2 on an 800x901 canvas:
                (c) host       the VOC transform on the host (voc_ref: mean subtraction, bicubic resize, boxes * im_scale),
                               upload of the float images, step()
                (d) raw        step_raw(): the transform inside the step's first launch
The modes of a workload run one after another, each built, warmed up on every shape (and captured) and then timed, and
freed before the next: the ResNet-101 RCNN trainers of all modes would not fit the card together.  A round is
ROUND_IMAGES images; its time is host wall time ending in a synchronise.  Reports images/s at the median round (and the
min-max) and each mode's peak device memory over the baseline.  Prints the card's name and power limit read in the same
run, a markdown table and one JSON line.

    python tests/gpu_resnet_canvas_train_bench.py [--rounds 3] [--out results/resnet_canvas_train_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
import voc_ref  # noqa: E402
from frcnn_b200.resnet_train import (CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer, ResNetRcnnTrainer,  # noqa: E402
                                     ResNetRpnTrainer)

ROUND_IMAGES = 12
SHAPES = [(600, 800), (600, 901), (600, 1000)]
PHOTOS = [(375, 500), (333, 500), (500, 375)]
RAW_N, RAW_HC, RAW_WC = 2, 800, 901
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def params_for(n_layers):
    """Random-init parameters with a head scaled for K = 2048*49 and livelier RPN heads (proposals that overlap the boxes,
    so that the RCNN step's NumPy sampling keeps RoIs)."""
    p = orc.make_resnet_params(n_layers=n_layers, seed=29)
    rng = np.random.default_rng(1)
    for k, s in (("RPN/rpn_cls_score/W", 0.05), ("RPN/rpn_bbox_pred/W", 0.05), ("fc6/W", 0.001), ("fc7/W", 0.01),
                 ("cls_score/W", 0.01), ("bbox_pred/W", 0.01)):
        p[k] = (rng.standard_normal(p[k].shape) * s).astype(np.float32)
    return p


def stream(shapes, n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        h, w = shapes[k % len(shapes)]
        x = torch.from_numpy(orc.make_image(h, w, seed=k % 6)[0]).cuda()
        G = int(rng.integers(2, 6))
        x1, y1 = rng.uniform(0, w * 0.3, G), rng.uniform(0, h * 0.3, G)
        g = np.stack([x1, y1, np.minimum(x1 + rng.uniform(300, 700, G), w - 1), np.minimum(y1 + rng.uniform(250, 500, G), h - 1),
                      rng.integers(1, 21, G)], 1).astype(np.float32)
        g[0, :4] = [4, 4, w - 5, h - 5]          # one box over most of the image: NumPy sampling always keeps RoIs
        out.append((x, torch.from_numpy(g).cuda()))
    return out


def photos(n, seed=0):
    rng = np.random.default_rng(seed)
    ph, bx, lb = [], [], []
    for k in range(n):
        h, w = PHOTOS[k % len(PHOTOS)]
        ph.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        G = int(rng.integers(1, 5))
        x1, y1 = rng.uniform(0, w * 0.4, G), rng.uniform(0, h * 0.4, G)
        bx.append(np.stack([x1, y1, np.minimum(x1 + rng.uniform(100, w / 2 + 100, G), w - 1),
                            np.minimum(y1 + rng.uniform(100, h / 2 + 100, G), h - 1)], 1).astype(np.float32))
        lb.append(rng.integers(1, 21, G).astype(np.int32))
    return ph, bx, lb


class PerShape(object):
    """(a): one trainer per shape, masters and momentum handed on at every change of shape."""

    def __init__(self, make, shapes):
        self.tr = {s: make(s) for s in shapes}
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
    """(b): step() on N images at a time."""

    def __init__(self, tr):
        self.tr, self.N = tr, tr.N

    def run(self, images):
        for k in range(0, len(images), self.N):
            chunk = images[k:k + self.N]
            self.tr.step([x for x, _ in chunk], [g for _, g in chunk])


class HostTransform(object):
    """(c): the VOC transform on the host, then step()."""

    def __init__(self, tr):
        self.tr, self.N = tr, tr.N

    def run(self, batch):
        ph, bx, lb = batch
        for k in range(0, len(ph), self.N):
            xs, gts = [], []
            for p, b, l in zip(ph[k:k + self.N], bx[k:k + self.N], lb[k:k + self.N]):
                img, _, gt = voc_ref.voc_transform(p, b, l)
                xs.append(torch.from_numpy(img).cuda())
                gts.append(torch.from_numpy(gt).cuda())
            self.tr.step(xs, gts)


class Raw(object):
    """(d): step_raw()."""

    def __init__(self, tr):
        self.tr, self.N = tr, tr.N

    def run(self, batch):
        ph, bx, lb = batch
        for k in range(0, len(ph), self.N):
            self.tr.step_raw(ph[k:k + self.N], bx[k:k + self.N], lb[k:k + self.N])


def measure(name, build, work, rounds):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    np.random.seed(0)
    m = build()
    m.run(work)                                                  # warm-up: every shape, the graph capture
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    ips = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        m.run(work)
        torch.cuda.synchronize()
        ips.append(ROUND_IMAGES / (time.perf_counter() - t0))
    del m
    ips = np.array(ips)
    row = dict(mode=name, images_per_s=float(np.median(ips)), ips_min=float(ips.min()), ips_max=float(ips.max()), peak_gb=peak)
    print("| %s | %.1f | %.1f-%.1f | %.1f |" % (name, row["images_per_s"], row["ips_min"], row["ips_max"], peak), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = card()
    print("card: %s; %d rounds of %d images per mode" % (gpu, args.rounds, ROUND_IMAGES))
    print("| mode | images/s (median) | min-max | peak memory (GB) |")
    print("|---|---|---|---|")
    mixed = stream(SHAPES, ROUND_IMAGES)
    raw_batch = photos(ROUND_IMAGES)
    rows = []
    for n_layers in (50, 101):
        params = params_for(n_layers)
        kw = dict(n_layers=n_layers)
        rows.append(measure("R%d RPN (a) per-shape" % n_layers,
                            lambda: PerShape(lambda s: ResNetRpnTrainer(params, s[0], s[1], ANCHORS, **kw), SHAPES), mixed,
                            args.rounds))
        for N in (1, 2, 4):
            rows.append(measure("R%d RPN (b) canvas N=%d" % (n_layers, N),
                                lambda: Canvas(CanvasResNetRpnTrainer(params, N, 600, 1000, ANCHORS, **kw)), mixed, args.rounds))
        rows.append(measure("R%d RCNN (a) per-shape" % n_layers,
                            lambda: PerShape(lambda s: ResNetRcnnTrainer(params, s[0], s[1], ANCHORS, **kw), SHAPES), mixed,
                            args.rounds))
        for N in (1, 2, 4):
            rows.append(measure("R%d RCNN (b) canvas N=%d" % (n_layers, N),
                                lambda: Canvas(CanvasResNetRcnnTrainer(params, N, 600, 1000, ANCHORS, **kw)), mixed, args.rounds))
        if n_layers == 101:
            for step, cls in (("RPN", CanvasResNetRpnTrainer), ("RCNN", CanvasResNetRcnnTrainer)):
                rows.append(measure("R101 %s raw photos (c) host transform + step, N=%d" % (step, RAW_N),
                                    lambda: HostTransform(cls(params, RAW_N, RAW_HC, RAW_WC, ANCHORS, **kw)), raw_batch,
                                    args.rounds))
                rows.append(measure("R101 %s raw photos (d) step_raw, N=%d" % (step, RAW_N),
                                    lambda: Raw(cls(params, RAW_N, RAW_HC, RAW_WC, ANCHORS, raw_input=True, **kw)), raw_batch,
                                    args.rounds))
        del params
    result = dict(card=gpu, rounds=args.rounds, round_images=ROUND_IMAGES, precision="bf16x3", rows=rows)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
