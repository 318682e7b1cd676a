"""Measurement (not a pytest): PASCAL VOC evaluation on the device against scoring on the host, in ONE process.

    python tests/gpu_voc_eval_bench.py [--densities 60,240,480] [--photos 48] [--rounds 5] [--out FILE.json]

Part 1, a VOC07-test-sized set (4,952 images, 20 classes, up to 300 keep-list entries per class and image) fabricated at
several mean detection densities per image (test_voc_eval_gpu.fabricate, on the device as frcnn_detect_batch leaves its
outputs): CUDA events around the appends (64 images per call, as batch plans would hand them over) and around the evaluation
launches (ops.voc_eval, GT already on the device), medians over the rounds; the whole VocEvaluator.evaluate call on the host
clock (GT packing, one upload, launches, one download); and the NumPy oracle (tests/voc_eval_ref.py) on the same detections
on the host, once.  The oracle is written for clarity (Python loops over detections), so it is an upper bound on what a
tuned host scorer would take.  Part 2, raw photos of VOC sizes to mAP with random VGG16 weights, N = 4, det_conf = 0.05:
Engine.evaluate_images against Engine.detect_images followed by the oracle's scoring on the downloaded lists, alternated
round by round after a warm-up, host seconds (ending in a synchronise) and images/s.  The card's name and power limit are
read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
import voc_eval_ref as ref  # noqa: E402
from frcnn_b200 import ops  # noqa: E402
from frcnn_b200.engine import Engine  # noqa: E402
from frcnn_b200.evaluate import VocEvaluator, pack_gt  # noqa: E402
from test_voc_eval_gpu import VOC_SHAPES, _gt_from_first_pass, fabricate  # noqa: E402

NC, R, M, BATCH = 21, 300, 4952, 64


def events_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def part1(density, rounds):
    data = fabricate(2007, M, R, NC, density)
    dev = {k: torch.from_numpy(data[k]).cuda() for k in ("prob", "boxes", "keep", "conf")}
    t0 = time.perf_counter()
    want = ref.voc_eval(ref.detections_from_lists(data["prob"], data["boxes"], data["keep"], data["conf"], data["scale"]),
                        *data["gt"], NC)
    host_s = time.perf_counter() - t0
    D = int(want["n_det"].sum())
    ev = VocEvaluator(NC, max_images=M, capacity=D + 1024)
    blob, G, (ob, ol, od) = pack_gt(*data["gt"], M, NC, ev.max_gt)
    b = torch.from_numpy(blob).cuda()
    gt = (b[:4 * (M + 1)].view(torch.int32), b[ob:ob + 16 * G].view(torch.float32).view(G, 4), b[ol:ol + 4 * G].view(torch.int32),
          b[od:od + G])

    def appends():
        ev.reset()
        ev.put_scales(data["scale"], 0)
        for s in range(0, M, BATCH):
            ev._append(dev["prob"][s:s + BATCH], dev["boxes"][s:s + BATCH], dev["keep"][s:s + BATCH], dev["conf"][s:s + BATCH])

    def launches():
        ops.voc_eval(NC, ev.capacity, M, ev.max_gt, *gt, 0.5, ev.ws, out=ev.out)

    appends()
    launches()
    app, evl, call = [], [], []
    for _ in range(rounds):
        app.append(events_ms(appends))
        evl.append(events_ms(launches))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = ev.evaluate(*data["gt"])
        call.append(1e3 * (time.perf_counter() - t0))
    ok = np.array_equal(res.tp, want["tp"]) and np.array_equal(res.ap07.view(np.int64), want["ap07"].view(np.int64))
    return dict(density=density, detections=D, append_ms=statistics.median(app), evaluate_launches_ms=statistics.median(evl),
                evaluate_call_ms=statistics.median(call), host_oracle_s=host_s, map07=res.map07, map=res.map, equal_to_oracle=ok)


def host_scoring(lists, gt):
    rows = [(d[0], n, j, d[5], d[1:5]) for n, dets in enumerate(lists) for j, d in enumerate(dets)]
    dets = dict(cls=np.array([r[0] for r in rows], np.int64), img=np.array([r[1] for r in rows], np.int64),
                pos=np.array([r[2] for r in rows], np.int64), score=np.array([r[3] for r in rows], np.float32),
                box=np.array([r[4] for r in rows], np.float32).reshape(-1, 4))
    return ref.voc_eval(dets, *gt, NC)


def part2(n_photos, rounds):
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    eng = Engine(orc.make_params(seed=1234), precision="bf16x3", anchors=anchors, with_detect=True)
    rng = np.random.default_rng(9)
    photos = [rng.integers(0, 256, VOC_SHAPES[i % len(VOC_SHAPES)] + (3,), dtype=np.uint8) for i in range(n_photos)]
    gt = _gt_from_first_pass(eng.detect_images(photos, N=4, conf=0.05), 10)

    def device():
        return eng.evaluate_images(photos, *gt, N=4, conf=0.05).map07

    def host():
        return host_scoring(eng.detect_images(photos, N=4, conf=0.05), gt)["map07"]

    device()
    host()
    t = {"device": [], "host": []}
    for _ in range(rounds):
        for name, fn in (("device", device), ("host", host)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            v = fn()
            torch.cuda.synchronize()
            t[name].append(time.perf_counter() - t0)
            t[name + "_map07"] = v
    out = dict(photos=n_photos, N=4)
    for name in ("device", "host"):
        s = statistics.median(t[name])
        out[name] = dict(seconds=s, images_per_s=n_photos / s, map07=t[name + "_map07"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--densities", default="60,240,480")
    ap.add_argument("--photos", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_voc_eval_bench needs a CUDA device")
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode().strip()
    res = dict(card=card, voc07_sized=[part1(int(d), args.rounds) for d in args.densities.split(",")],
               photos_to_map=part2(args.photos, max(1, args.rounds // 2)))
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
