"""Measurement (not a pytest): raw uint8 photos of mixed sizes to detections on the host, three ways, in ONE process.

    python tests/gpu_raw_canvas_bench.py [--images 96] [--rounds 7] [--out FILE.json]

The stream is raw BGR photos of 300x500, 333x500 and 375x500 (they resize to 600x1000, 600x901 and 600x800), bf16x3,
per-class NMS on, and every mode ends with the forward.py detection lists on the host:
  a  one StreamRunner(src_hw=...) per source shape (one ForwardPlan graph per shape, the stream sorted by shape)
  b  the float-input canvas path: per image an upload + preprocess.img_preprocessing, then CanvasBatchPlan.forward(images)
     and one download per batch (N = 4)
  c  CanvasStreamRunner on CanvasBatchPlan(raw_input=True), N = 4 and N = 8
Modes alternate round by round after a warm-up of every plan; the medians over the rounds are reported: host wall images/s
(the clock stops after a device synchronise), device ms per image (CUDA events on the submitting stream around the whole
round) and host-to-device copies and bytes per image (counted from what each mode enqueues).  (b) and (c) must return
identical detections.  The second part times, with CUDA events over many launches, the fused first launch
(frcnn_preprocess_bgr8_canvas) against preprocess + copy into the canvas + pack at N = 4 on a 600 x 1000 canvas, with the
bytes each moves computed from the shapes.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
from frcnn_b200 import ops, preprocess  # noqa: E402
from frcnn_b200.engine import CanvasStreamRunner, Engine, StreamRunner  # noqa: E402

SHAPES = [(300, 500), (333, 500), (375, 500)]
HC, WC = 600, 1000


def timed(fn):
    """(result, host seconds ending in a synchronise, device ms between events on the current stream)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=96)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    assert args.images % 24 == 0 and args.rounds >= 5
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode().strip()
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    eng = Engine(orc.make_params(seed=1234), precision="bf16x3", anchors=anchors, with_detect=True, det_conf=0.05)
    rng = np.random.default_rng(7)
    imgs = [rng.integers(0, 256, SHAPES[i % 3] + (3,), dtype=np.uint8) for i in range(args.images)]
    n = len(imgs)

    # a: one StreamRunner per source shape
    runners = []
    for k, shp in enumerate(SHAPES):
        s, H, W = preprocess.plan_size(*shp)
        runners.append((StreamRunner(eng.plan(H, W), src_hw=shp, depth=8, lanes=1), s, [i for i in range(n) if i % 3 == k]))

    def mode_a():
        out = [None] * n
        for r, s, idx in runners:
            r.run([imgs[i] for i in idx], on_result=lambda j, res, s=s, idx=idx: out.__setitem__(idx[j], preprocess.result_detections(res, s)))
        return out

    # b: upload + preprocess per image, float-input canvas plan
    fplan = eng.canvas_plan(4, HC, WC)

    def mode_b():
        out = []
        for s0 in range(0, n, 4):
            xs, scales = zip(*[preprocess.img_preprocessing(im) for im in imgs[s0:s0 + 4]])
            fplan.forward(list(xs))
            res = fplan.fetch_result()
            out += [preprocess.result_detections(res[k], scales[k]) for k in range(4)]
        return out

    # c: the raw canvas runner
    crun = {N: CanvasStreamRunner(eng.canvas_plan(N, HC, WC, raw_input=True, arena_bytes=N * 3 * 375 * 500 + 64 * N), depth=2)
            for N in (4, 8)}
    modes = [("a_stream_runner_per_shape", mode_a), ("b_preprocess_then_canvas_n4", mode_b),
             ("c_canvas_stream_runner_n4", lambda: crun[4].run(imgs)), ("c_canvas_stream_runner_n8", lambda: crun[8].run(imgs))]
    outs = {name: fn() for name, fn in modes}                    # warm-up of every plan and shape
    torch.cuda.synchronize()
    assert outs["b_preprocess_then_canvas_n4"] == outs["c_canvas_stream_runner_n4"] == outs["c_canvas_stream_runner_n8"]
    assert outs["a_stream_runner_per_shape"] == outs["c_canvas_stream_runner_n4"] and all(len(d) > 0 for d in outs[modes[0][0]])
    src_bytes = sum(im.size for im in imgs)
    h2d = {"a_stream_runner_per_shape": (n, src_bytes), "b_preprocess_then_canvas_n4": (n + n // 4, src_bytes + (n // 4) * 16 * 4)}
    for N in (4, 8):
        c0, b0 = crun[N].h2d_copies, crun[N].h2d_bytes
        crun[N].run(imgs)
        h2d["c_canvas_stream_runner_n%d" % N] = (crun[N].h2d_copies - c0, crun[N].h2d_bytes - b0)
    wall, dev = {m: [] for m, _ in modes}, {m: [] for m, _ in modes}
    for _ in range(args.rounds):
        for name, fn in modes:
            got, sec, ms = timed(fn)
            assert got == outs[name]
            wall[name].append(n / sec)
            dev[name].append(ms / n)
    result = dict(card=card, images=n, rounds=args.rounds, shapes=SHAPES, modes={})
    for name, _ in modes:
        result["modes"][name] = dict(host_wall_images_per_s=round(statistics.median(wall[name]), 1),
                                     host_wall_min_max=[round(min(wall[name]), 1), round(max(wall[name]), 1)],
                                     device_ms_per_image=round(statistics.median(dev[name]), 3),
                                     h2d_copies_per_image=round(h2d[name][0] / n, 3), h2d_bytes_per_image=round(h2d[name][1] / n))

    # the first launch alone: fused kernel against preprocess + copy + pack, N = 4 on the 600 x 1000 canvas
    four = [imgs[0], imgs[1], imgs[2], imgs[3]]
    plan = crun[4].plan
    plan.forward_raw(four)
    dimg = [torch.from_numpy(im).cuda() for im in four]
    sizes = [preprocess.plan_size(*im.shape[:2])[1:] for im in four]
    x_in = torch.zeros((4, 3, HC, WC), device="cuda")
    ext = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    fl = [torch.empty((3, H, W), device="cuda") for H, W in sizes]
    planes = ops.Act(torch.empty_like(plan.acts[0].hi), torch.empty_like(plan.acts[0].lo))

    def fused():
        plan.input.pack_c8(plan.acts[0])

    def chain():
        for k in range(4):
            preprocess.img_preprocessing(dimg[k], out=fl[k])
            x_in[k, :, :sizes[k][0], :sizes[k][1]].copy_(fl[k], non_blocking=True)
        ops.pack_image_c8_batch(x_in, out=planes, extents=ext)

    reps, kern = 200, {"fused": [], "preprocess_copy_pack": []}
    for fn in (fused, chain):
        for _ in range(10):
            fn()
    assert torch.equal(planes.hi.view(torch.int16), plan.acts[0].hi.view(torch.int16))
    assert torch.equal(planes.lo.view(torch.int16), plan.acts[0].lo.view(torch.int16))
    for _ in range(args.rounds):
        for name, fn in (("fused", fused), ("preprocess_copy_pack", chain)):
            _, _, ms = timed(lambda: [fn() for _ in range(reps)])
            kern[name].append(1e3 * ms / reps)
    plane_bytes = 4 * int(plan.acts[0].hi.shape[1]) * 2 * 2                   # N slots, bf16, hi + lo
    raw = sum(im.size for im in four)
    f32 = sum(12 * H * W for H, W in sizes)
    moved = {"fused": raw + plane_bytes, "preprocess_copy_pack": (raw + f32) + 2 * f32 + (f32 + plane_bytes)}
    result["first_launch_n4_600x1000"] = {
        name: dict(us_per_batch=round(statistics.median(v), 1), launches=1 if name == "fused" else 9, bytes_moved=moved[name],
                   gb_per_s=round(moved[name] / statistics.median(v) / 1e3, 1)) for name, v in kern.items()}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
