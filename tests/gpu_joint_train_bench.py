"""Measurement (not a pytest): the joint training step against the alternating RPN / RCNN schedule.

The workload of gpu_canvas_rcnn_train_bench.py: a stream of 600x{800, 901, 1000} images in turn on a 600x1000 canvas, with
synthetic ground truth, random-init VGG16 and bf16x3, device draws, graph replay.  For each N in (1, 2, 4) three trainers
are built side by side -- CanvasJointTrainer, CanvasRpnTrainer and CanvasRcnnTrainer -- warmed up, and then run in
alternating rounds.  The alternating schedule trains each image once per step kind, so its cost per image is the sum of the
RPN and RCNN steps' times.  Two more lines: the joint step with py-faster-rcnn's training proposal counts (pre_n=12000,
post_n=2000) at N = 4, and CanvasResNetJointTrainer (ResNet-101) at N = 4.

A round is ROUND_IMAGES images; its device time comes from CUDA events around it (ending in a synchronise).  Reports the
median and min-max device ms per image over the rounds, images/s at the median, and each trainer's peak device memory over
what was allocated before it was built.  Prints the card's name and power limit with the numbers, a markdown table and one
JSON line."""
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
from gpu_canvas_rcnn_train_bench import ANCHORS, ROUND_IMAGES, ROUNDS, SHAPES, card, stream  # noqa: E402
from frcnn_b200.resnet_train import CanvasResNetJointTrainer  # noqa: E402
from frcnn_b200.train_engine import CanvasJointTrainer, CanvasRcnnTrainer, CanvasRpnTrainer  # noqa: E402


class Canvas(object):
    """A canvas trainer's step on N images at a time."""

    def __init__(self, make, N):
        self.N, self.tr = N, make(N)

    def run(self, images):
        for k in range(0, len(images), self.N):
            chunk = images[k:k + self.N]
            self.tr.step([x for x, _ in chunk], [g for _, g in chunk])


def _measure(group, images):
    """Builds and warms up each (name, make, N) of `group`, then times them in alternating rounds."""
    modes = []
    for name, make, N in group:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        m = Canvas(make, N)
        m.run(images)                                            # warm-up: every shape, the graph capture
        torch.cuda.synchronize()
        modes.append(dict(name=name, m=m, peak_gb=(torch.cuda.max_memory_allocated() - base) / 2 ** 30, ms=[]))
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(ROUNDS):
        for md in modes:
            ev0.record()
            md["m"].run(images)
            ev1.record()
            torch.cuda.synchronize()
            md["ms"].append(ev0.elapsed_time(ev1) / len(images))
    rows = []
    for md in modes:
        ms = np.array(md["ms"])
        rows.append(dict(mode=md["name"], ms_median=float(np.median(ms)), ms_min=float(ms.min()), ms_max=float(ms.max()),
                         images_per_s=1e3 / float(np.median(ms)), peak_gb=md["peak_gb"]))
    del modes
    gc.collect()
    torch.cuda.empty_cache()
    return rows


def main():
    params = orc.make_params(seed=1234)
    images = stream(SHAPES, ROUND_IMAGES)
    kw = dict(subsample="device", sample="device", dropout="device")
    rows = []
    for N in (1, 2, 4):
        rows_n = _measure([
            ("joint N=%d" % N, lambda n: CanvasJointTrainer(params, n, 600, 1000, ANCHORS, **kw), N),
            ("rpn N=%d" % N, lambda n: CanvasRpnTrainer(params, n, 600, 1000, ANCHORS), N),
            ("rcnn N=%d" % N, lambda n: CanvasRcnnTrainer(params, n, 600, 1000, ANCHORS), N)], images)
        alt = rows_n[1]["ms_median"] + rows_n[2]["ms_median"]
        rows += rows_n + [dict(mode="alternating rpn + rcnn N=%d" % N, ms_median=alt, ms_min=rows_n[1]["ms_min"] + rows_n[2]["ms_min"],
                              ms_max=rows_n[1]["ms_max"] + rows_n[2]["ms_max"], images_per_s=1e3 / alt, peak_gb=None)]
    rows += _measure([("joint N=4 pre_n=12000 post_n=2000",
                       lambda n: CanvasJointTrainer(params, n, 600, 1000, ANCHORS, pre_n=12000, post_n=2000, **kw), 4)], images)
    del params
    gc.collect()
    r101 = orc.make_resnet_params(101, seed=1234)
    rows += _measure([("ResNet-101 joint N=4", lambda n: CanvasResNetJointTrainer(r101, n, 600, 1000, ANCHORS, n_layers=101,
                                                                                 **kw), 4)], images)
    gpu = card()
    print("card: %s; %d rounds of %d images per mode" % (gpu, ROUNDS, ROUND_IMAGES))
    print("| mode | ms / image (median) | min-max | images/s | peak memory (GB) |")
    print("|---|---|---|---|---|")
    for r in rows:
        print("| %s | %.2f | %.2f-%.2f | %.1f | %s |" % (r["mode"], r["ms_median"], r["ms_min"], r["ms_max"], r["images_per_s"],
                                                     "-" if r["peak_gb"] is None else "%.1f" % r["peak_gb"]))
    print(json.dumps(dict(card=gpu, rounds=ROUNDS, round_images=ROUND_IMAGES, rows=rows)))


if __name__ == "__main__":
    main()
