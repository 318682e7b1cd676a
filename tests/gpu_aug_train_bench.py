"""Training on raw photos with and without device-side augmentation, on one GPU.

Workload: a stream of raw 375x500, 333x500 and 500x375 uint8 photos with 1-4 synthetic boxes each, N = 4 slots on a
1000x1000 canvas, random-init VGG16, bf16x3.  For CanvasRpnTrainer and CanvasRcnnTrainer, in one process, alternating
round by round after a warm-up:
  (a) plain  step_raw() with augment=None: the VOC transform at short side 600
  (b) flip   augment="device", scales=(600,): a per-slot horizontal flip drawn inside the step, same image sizes as (a)
  (c) multi  augment="device", scales=(480, 576, 688, 864, 1000): flip and multi-scale.  Its images are smaller on
             average, so its rate is not comparable to (a) and (b).
Prints one JSON line: host-wall images/s per mode (median, min, max over rounds, each round ending in a synchronise), the
first launches from CUDA events (frcnn_voc_augment_batch + the _flip pack + the flipped box scaling against the plain pack
+ box scaling, on the same block), and the card's name, power limit and max SM clock read in the same run.

    python tests/gpu_aug_train_bench.py [--rounds 6] [--steps 8] [--out results/aug_train_bench.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
from gpu_raw_canvas_train_bench import HC, N, WC, _card, _stream  # noqa: E402

MODES = {"plain": {}, "flip": dict(augment="device", scales=(600,)),
         "multi": dict(augment="device", scales=(480, 576, 688, 864, 1000))}


def _run(trainer, batches):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for batch in batches:
        trainer.step_raw([p for p, _, _ in batch], [b for _, b, _ in batch], [l for _, _, l in batch])
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _first_launches(plain, flip, reps=50):
    """The first launches of each step on its trainer's current block: plain pack + box scaling, against the augment draw +
    the _flip pack + the flipped box scaling."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def head(tr):
        if tr.augment is not None:
            tr.input.augment(tr.seeds, 1)
        tr.input.pack_im2col(tr.x_col, 3, 1, 1, 32)
        tr.input.scale_gt(tr.gt, tr.gt_counts)
    head(plain)
    head(flip)
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(reps):
        head(plain)
    ev[1].record()
    for _ in range(reps):
        head(flip)
    ev[2].record()
    torch.cuda.synchronize()
    return dict(plain_ms=round(ev[0].elapsed_time(ev[1]) / reps, 4), augment_ms=round(ev[1].elapsed_time(ev[2]) / reps, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from frcnn_b200 import _lib
    from frcnn_b200.train_engine import CanvasRcnnTrainer, CanvasRpnTrainer
    _lib.load()
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    params = orc.make_params(seed=1)
    stream = _stream(0, N * a.steps)
    batches = [stream[i:i + N] for i in range(0, len(stream), N)]
    res = dict(card=_card(), N=N, canvas=[HC, WC], precision="bf16x3", steps_per_round=a.steps, rounds=a.rounds)
    for name, cls in (("rpn", CanvasRpnTrainer), ("rcnn", CanvasRcnnTrainer)):
        tr = {m: cls(params, N, HC, WC, anchors, seed=3, raw_input=True, **kw) for m, kw in MODES.items()}
        for m in MODES:
            _run(tr[m], batches[:2])                           # eager step + capture, warm caches
        rates = {m: [] for m in MODES}
        for r in range(a.rounds):
            for m in (("plain", "flip", "multi") if r % 2 == 0 else ("flip", "plain", "multi")):
                rates[m].append(N * len(batches) / _run(tr[m], batches))
        out = {}
        for m in MODES:
            v = sorted(rates[m])
            out[m] = dict(img_per_s_median=round(float(np.median(v)), 2), img_per_s_min=round(v[0], 2),
                          img_per_s_max=round(v[-1], 2))
        out["flip_over_plain"] = round(out["flip"]["img_per_s_median"] / out["plain"]["img_per_s_median"], 4)
        if name == "rpn":
            out["first_launches"] = _first_launches(tr["plain"], tr["flip"])
        res[name] = out
        del tr
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
