"""Training on raw photos against the host transform, on one GPU.

Workload: a stream of raw 375x500, 333x500 and 500x375 uint8 photos with 1-4 synthetic boxes each, N = 4 slots on a
1000x1000 canvas, random-init VGG16, bf16x3.  For CanvasRpnTrainer and CanvasRcnnTrainer, in one process, alternating
round by round after a warm-up:
  (a) host   the reference's per-photo transform on the host (float32 mean subtraction, cv2.resize INTER_CUBIC, CHW,
             boxes * im_scale), upload of the float images and boxes, step()
  (b) raw    step_raw(): one upload of the photos and boxes, the transform inside the step's first launch
Prints one JSON line: host-wall images/s per mode (median, min, max over rounds, each round ending in a synchronise), device
ms per image (graph replay), host-to-device bytes per image, the fused first launch against the unfused sequence (float
images already on the device copied into the canvas + pack_image_im2col_batch_ext) with its achieved bandwidth, and the
card's name, power limit and max SM clock read in the same run.

    python tests/gpu_raw_canvas_train_bench.py [--rounds 6] [--steps 8] [--out results/raw_train_bench.json]
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

N, HC, WC = 4, 1000, 1000     # the smallest square canvas that holds both orientations (500x375 -> 800x600)
SIZES = [(375, 500), (333, 500), (500, 375)]
HBM_TBS = 3.35          # H100 SXM data sheet


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def _stream(seed, count):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(count):
        h, w = SIZES[i % len(SIZES)]
        G = int(rng.integers(1, 5))
        x1, y1 = rng.uniform(0, w - 60, G), rng.uniform(0, h - 60, G)
        b = np.stack([x1, y1, x1 + rng.uniform(30, 50, G), y1 + rng.uniform(30, 50, G)], 1).astype(np.float32)
        out.append((rng.integers(0, 256, (h, w, 3), dtype=np.uint8), b, rng.integers(1, 21, G).astype(np.int32)))
    return out


def _host_transform(photo, bbox, label):
    """datasets/pascal_voc_dataset.py VOC.get_example, with cv2 as the reference runs it."""
    import cv2
    img = photo.astype(np.float32)
    img -= voc_ref.VOC_MEANS
    s, _, _ = voc_ref.plan_size(*photo.shape[:2])
    img = cv2.resize(img, None, None, fx=s, fy=s, interpolation=cv2.INTER_CUBIC)
    img = img.transpose(2, 0, 1).astype(np.float32)
    bbox = bbox.copy()
    bbox *= s
    return img, np.concatenate((bbox, label[:, None]), axis=1).astype(np.float32)


def _run(trainer, mode, batches):
    h2d = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for batch in batches:
        if mode == "host":
            xs, gts = [], []
            for p, b, l in batch:
                img, gt = _host_transform(p, b, l)
                xs.append(torch.from_numpy(img).cuda(non_blocking=True))
                gts.append(torch.from_numpy(gt).cuda(non_blocking=True))
                h2d += img.nbytes + gt.nbytes
            trainer.step(xs, gts)
        else:
            trainer.step_raw([p for p, _, _ in batch], [b for _, b, _ in batch], [l for _, _, l in batch])
            h2d += trainer.input.header_bytes + sum(p.nbytes for p, _, _ in batch)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, h2d


def _device_ms(trainer, reps=10):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        trainer.graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps / N


def _first_launch(trainer, batch, reps=50):
    """The fused launch against the unfused device sequence, on the trainer's current raw block."""
    from frcnn_b200.engine import ImageInput
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    out = trainer.x_col
    trainer.input.pack_im2col(out, 3, 1, 1, 32)
    xs = [torch.from_numpy(_host_transform(p, b, l)[0]).cuda() for p, b, l in batch]
    ref = ImageInput(N, HC, WC, trainer.device, canvas=True)
    ref.put(xs)
    ref.pack_im2col(out, 3, 1, 1, 32)
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(reps):
        trainer.input.pack_im2col(out, 3, 1, 1, 32)
    ev[1].record()
    for _ in range(reps):
        ref.put(xs)
        ref.pack_im2col(out, 3, 1, 1, 32)
    ev[2].record()
    torch.cuda.synchronize()
    fused = ev[0].elapsed_time(ev[1]) / reps
    unfused = ev[1].elapsed_time(ev[2]) / reps
    written = N * HC * WC * 32 * 2 * 2                   # hi + lo bf16 planes
    return dict(fused_ms=round(fused, 4), unfused_device_ms=round(unfused, 4), planes_MB=round(written / 1e6, 1),
                fused_TBps=round(written / fused / 1e9, 3), share_of_3_35=round(written / fused / 1e9 / HBM_TBS, 3))


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
        tr = {"host": cls(params, N, HC, WC, anchors, seed=3), "raw": cls(params, N, HC, WC, anchors, seed=3, raw_input=True)}
        for mode in ("host", "raw"):
            _run(tr[mode], mode, batches[:2])                     # eager step + capture, warm caches
        rates = {"host": [], "raw": []}
        h2d = {}
        for r in range(a.rounds):
            for mode in (("host", "raw") if r % 2 == 0 else ("raw", "host")):
                dt, h2d[mode] = _run(tr[mode], mode, batches)
                rates[mode].append(N * len(batches) / dt)
        out = {}
        for mode in ("host", "raw"):
            v = sorted(rates[mode])
            out[mode] = dict(img_per_s_median=round(float(np.median(v)), 2), img_per_s_min=round(v[0], 2),
                             img_per_s_max=round(v[-1], 2), device_ms_per_img=round(_device_ms(tr[mode]), 3),
                             h2d_bytes_per_img=int(h2d[mode] / (N * len(batches))))
        out["raw_over_host"] = round(out["raw"]["img_per_s_median"] / out["host"]["img_per_s_median"], 3)
        if name == "rpn":
            out["first_launch"] = _first_launch(tr["raw"], batches[0])
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
