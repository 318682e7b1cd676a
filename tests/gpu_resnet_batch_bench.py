"""Diagnostic (not a pytest): the ResNet-101 detector (random-init weights, bf16x3) one image at a time against batches and
canvas batches, everything in one process, the modes alternating round by round.

(a) BASELINE config #4: 800 x 1333, 1000 proposals -- one ResNetForwardPlan with one image in flight, a LanePool of 4 lanes
    (4 images in flight on 4 streams), and ResNetBatchPlan with N = 2 and N = 4.
(b) A stream of VOC-style images, short side 600 and long side 800, 901 or 1000, 300 proposals -- one ResNetForwardPlan per
    shape (one image in flight) against ResNetCanvasBatchPlan N = 4 and N = 8 on a 600 x 1000 canvas.

Prints the card, its power limit and max SM clock; per mode the device time per image (median over the rounds) and the
device memory its plans hold; and whether every batched image equals its ResNetForwardPlan result, bit for bit.

    python tests/gpu_resnet_batch_bench.py [--rounds 5] [--images 24]
"""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
from frcnn_b200.engine import LanePool  # noqa: E402
from frcnn_b200.resnet_engine import ResNetBatchPlan, ResNetCanvasBatchPlan, ResNetForwardPlan, ResNetPackedWeights  # noqa: E402

FIELDS = ("prob", "boxes", "rois", "scores")
SIZES = [(600, 800), (600, 901), (600, 1000)]


def device_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(reps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def built(make):
    """(object, bytes its construction and first run left allocated)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    obj = make()
    torch.cuda.synchronize()
    return obj, torch.cuda.memory_allocated() - base


def result(plan):
    torch.cuda.synchronize()
    return plan.unpack_result(plan.result.cpu().numpy())


def same(a, b):
    return a["count"] == b["count"] and all(np.array_equal(np.asarray(a[f]).view(np.int32), np.asarray(b[f]).view(np.int32))
                                            for f in FIELDS)


def timed(configs, rounds):
    for _, f in configs:          # warm-up: captures, module loads
        f()
    res = {name: [] for name, _ in configs}
    for _ in range(rounds):
        for name, f in configs:
            res[name].append(f())
    for name, _ in configs:
        m = statistics.median(res[name])
        print("  %-34s %7.3f ms  %6.1f img/s   (rounds: %s)" % (name, m, 1e3 / m, " ".join("%.3f" % v for v in res[name])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--images", type=int, default=24, help="images per timed window (a multiple of 24)")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("card (name, power limit, max SM clock): %s" % (q.stdout.strip().splitlines()[0] if q.stdout else "(nvidia-smi unavailable)"))
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    wts = ResNetPackedWeights(orc.make_resnet_params(101, seed=4321), 101, "bf16x3")
    n_img = args.images
    ok = total = 0

    # ---- (a) config #4
    H, W = 800, 1333
    kw = dict(anchors=anchors, feat_stride=32, post_n=1000)
    imgs = [torch.from_numpy(orc.make_image(H, W, seed=i)[0]).cuda() for i in range(4)]
    x4 = torch.stack(imgs)
    plan1, mem1 = built(lambda: ResNetForwardPlan(wts, H, W, **kw))
    pool, mem_pool = built(lambda: LanePool(plan1.clone(), lanes=4))
    bplans, bmem = {}, {}
    for N in (2, 4):
        bplans[N], bmem[N] = built(lambda N=N: ResNetBatchPlan(wts, N, H, W, **kw))

    def run_pool():
        pool.fork()
        for i in range(n_img):
            pool.submit(i, imgs[i % 4])
        pool.join()
    configs = [("ResNetForwardPlan, 1 in flight", lambda: device_ms(lambda i: plan1.forward(imgs[i % 4]), n_img) / n_img),
               ("LanePool, 4 lanes", lambda: device_ms(lambda i: run_pool(), 1) / n_img)]
    for N in (2, 4):
        configs.append(("ResNetBatchPlan N=%d" % N, lambda N=N: device_ms(lambda i: bplans[N].forward(x4[(i * N) % 4:(i * N) % 4 + N]),
                                                                          n_img // N) / n_img))
    print("(a) ResNet-101, 800x1333, 1000 proposals, bf16x3: device time per image, median of %d rounds of %d images:"
          % (args.rounds, n_img))
    timed(configs, args.rounds)
    print("  plan memory: ResNetForwardPlan %.0f MB, LanePool(4) %.0f MB, ResNetBatchPlan N=2 %.0f MB, N=4 %.0f MB"
          % (mem1 / 2**20, mem_pool / 2**20, bmem[2] / 2**20, bmem[4] / 2**20))
    want = []
    for x in imgs:
        plan1.forward(x)
        want.append(result(plan1))
    bplans[4].forward(x4)
    got = result(bplans[4])
    for k in range(4):
        pool.submit(k, imgs[k])
        pool.join()
        got_lane = result(pool.plans[k % len(pool)])
        ok += same(got[k], want[k]) + same(got_lane, want[k])
        total += 2
    print("  R per image: %s" % [w["count"] for w in want])
    del pool, bplans, plan1
    torch.cuda.empty_cache()

    # ---- (b) a stream of 600 x {800, 901, 1000}
    kw = dict(anchors=anchors, feat_stride=32, post_n=300)
    stream = [torch.from_numpy(orc.make_image(*SIZES[i % 3], seed=10 + i)[0]).cuda() for i in range(24)]

    def per_shape():
        plans = {}
        for x in stream[:3]:
            p = plans.setdefault(tuple(x.shape[1:]), ResNetForwardPlan(wts, int(x.shape[1]), int(x.shape[2]), **kw))
            p.forward(x)
        return plans
    shape_plans, shape_bytes = built(per_shape)
    cplans, cmem = {}, {}
    for N in (4, 8):
        def canvas(N=N):
            p = ResNetCanvasBatchPlan(wts, N, 600, 1000, **kw)
            p.forward(stream[:N])
            return p
        cplans[N], cmem[N] = built(canvas)
    graphs = {N: cplans[N].graph for N in cplans}

    def run_shapes(i):
        x = stream[i % 24]
        shape_plans[tuple(x.shape[1:])].forward(x)

    def run_canvas(N):
        def f(i):
            s = (i * N) % 24
            cplans[N].forward(stream[s:s + N])
        return f
    configs = [("ResNetForwardPlan per shape", lambda: device_ms(run_shapes, n_img) / n_img)]
    for N in (4, 8):
        configs.append(("ResNetCanvasBatchPlan N=%d" % N, lambda N=N: device_ms(run_canvas(N), n_img // N) / n_img))
    print("(b) ResNet-101, stream of 600x{800,901,1000}, 300 proposals, bf16x3: device time per image, median of %d rounds of "
          "%d images:" % (args.rounds, n_img))
    timed(configs, args.rounds)
    print("  plan memory: %d ResNetForwardPlans %.0f MB, ResNetCanvasBatchPlan N=4 %.0f MB, N=8 %.0f MB; re-capture: %s"
          % (len(shape_plans), shape_bytes / 2**20, cmem[4] / 2**20, cmem[8] / 2**20,
             "YES" if any(cplans[N].graph is not graphs[N] for N in cplans) else "none"))
    cplans[8].forward(stream[:8])
    got = result(cplans[8])
    for n in range(8):
        p = shape_plans[tuple(stream[n].shape[1:])]
        p.forward(stream[n])
        w = result(p)
        ok += same(got[n], w)
        total += 1
    print("bit-identical images (every batched / lane result vs ResNetForwardPlan): %d of %d" % (ok, total))


if __name__ == "__main__":
    main()
