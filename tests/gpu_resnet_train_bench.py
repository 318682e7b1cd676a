"""Measurement (not a pytest): the RPN training step at 600x1000 with the ResNet-50 and ResNet-101 trunks
(ResNetRpnTrainer, frozen BatchNorm) beside the VGG16 step (RpnTrainer), bf16x3, device subsampling, random-init weights,
one synthetic image with three ground-truth boxes.

Every trainer is warmed up first; then the trainers alternate round by round.  A round is ROUND_STEPS steps; its device
time comes from CUDA events around it (ending in a synchronise).  Within the round, events after forward and after backward
split each step into forward, backward and update (the update includes the weight repack).  Reports the median and
min-max device ms per image over the rounds, images/s at the median, the share of forward / backward / update, and the
device memory each trainer holds (allocated after its warm-up, over the baseline; the gradient activations and transposed
buffers included).  Prints the card's name and power limit with the numbers, a markdown table and one JSON line."""
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
from frcnn_b200.resnet_train import ResNetRpnTrainer  # noqa: E402
from frcnn_b200.train_engine import RpnTrainer  # noqa: E402

ROUNDS, ROUND_STEPS, WARMUP = 7, 6, 3
H, W = 600, 1000
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed_round(tr, x, gt, n):
    """n steps; returns (total ms, forward ms, backward ms, update ms) from events around each phase."""
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(n)]
    for k in range(n):
        ev[k][0].record()
        tr.forward(x, gt)
        ev[k][1].record()
        tr.backward()
        ev[k][2].record()
        tr.update()
        ev[k][3].record()
    torch.cuda.synchronize()
    parts = np.array([[e[i].elapsed_time(e[i + 1]) for i in range(3)] for e in ev])
    return ev[0][0].elapsed_time(ev[-1][3]), parts.sum(0)


def main():
    x = torch.from_numpy(orc.make_image(H, W, seed=0)[0]).cuda()
    gt = torch.tensor([[40, 60, 400, 380, 3], [300, 100, 900, 560, 7], [600, 250, 850, 500, 1]], dtype=torch.float32).cuda()
    trainers = []
    base = torch.cuda.memory_allocated()
    for name, build in [("VGG16 RpnTrainer", lambda: RpnTrainer(orc.make_params(seed=1234), H, W, ANCHORS)),
                        ("ResNet-50 ResNetRpnTrainer", lambda: ResNetRpnTrainer(orc.make_resnet_params(50, seed=3), H, W, ANCHORS,
                                                                                n_layers=50)),
                        ("ResNet-101 ResNetRpnTrainer", lambda: ResNetRpnTrainer(orc.make_resnet_params(101, seed=3), H, W, ANCHORS,
                                                                                 n_layers=101))]:
        tr = build()
        for _ in range(WARMUP):
            tr.step(x, gt)
        torch.cuda.synchronize()
        held = torch.cuda.memory_allocated() - base
        base = torch.cuda.memory_allocated()
        trainers.append(dict(name=name, tr=tr, held_gb=held / 2 ** 30, ms=[], phases=np.zeros(3)))
    for _ in range(ROUNDS):
        for t in trainers:
            total, phases = timed_round(t["tr"], x, gt, ROUND_STEPS)
            t["ms"].append(total / ROUND_STEPS)
            t["phases"] += phases
    gpu = card()
    rows = []
    print("card: %s; %dx%d, bf16x3, %d rounds of %d steps per trainer" % (gpu, H, W, ROUNDS, ROUND_STEPS))
    print("| trainer | ms / image (median) | min-max | images/s | forward / backward / update | memory held (GB) |")
    print("|---|---|---|---|---|---|")
    for t in trainers:
        ms = np.array(t["ms"])
        med = float(np.median(ms))
        share = t["phases"] / t["phases"].sum()
        rows.append(dict(trainer=t["name"], ms_median=med, ms_min=float(ms.min()), ms_max=float(ms.max()), images_per_s=1e3 / med,
                         forward=float(share[0]), backward=float(share[1]), update=float(share[2]), memory_gb=t["held_gb"]))
        print("| %s | %.2f | %.2f-%.2f | %.1f | %.0f%% / %.0f%% / %.0f%% | %.2f |" % (
            t["name"], med, ms.min(), ms.max(), 1e3 / med, 100 * share[0], 100 * share[1], 100 * share[2], t["held_gb"]))
    print(json.dumps(dict(card=gpu, shape=[H, W], rounds=ROUNDS, round_steps=ROUND_STEPS, rows=rows)))


if __name__ == "__main__":
    main()
