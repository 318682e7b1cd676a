"""Diagnostic (not a pytest): a stream of VOC-style images of DIFFERENT sizes -- short side 600, long side 800, 901 or
1000, as the reference's data path scales photos -- through one ForwardPlan per shape (one image in flight) against
engine.CanvasBatchPlan on a 600 x 1000 canvas with N = 4 and N = 8.  bf16x3, per-class NMS in the graph, random-init
weights; everything in one process, the modes alternating round by round.

Prints the card and its power limit; per mode the device time per image (median over the rounds), the plans and graph
captures it needed, the device memory its plans hold and the peak during a run; the extent-path overhead (all-600x1000
inputs through CanvasBatchPlan against BatchPlan, N = 4); and whether every canvas image equals its ForwardPlan result.

    python tests/gpu_canvas_batch_bench.py [--rounds 5] [--images 48]
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
from frcnn_b200.engine import BatchPlan, CanvasBatchPlan, ForwardPlan, PackedWeights  # noqa: E402

SIZES = [(600, 800), (600, 901), (600, 1000)]
HC, WC = 600, 1000
FIELDS = ("prob", "boxes", "rois", "scores", "keep_count", "conf_count", "keep_idx")


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
    """(object, bytes its construction and first run left allocated, peak bytes above the start during that run)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    obj = make()
    torch.cuda.synchronize()
    return obj, torch.cuda.memory_allocated() - base, torch.cuda.max_memory_allocated() - base


def same(a, b):
    return a["count"] == b["count"] and all(np.array_equal(np.asarray(a[f]).view(np.int32), np.asarray(b[f]).view(np.int32))
                                            for f in FIELDS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--images", type=int, default=48, help="images per timed window (a multiple of 24)")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("card: %s" % q.stdout.strip().splitlines()[0] if q.stdout else "card: (nvidia-smi unavailable)")
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    kw = dict(anchors=anchors, with_detect=True, det_nms_thresh=0.3, det_conf=0.8)
    wts = PackedWeights(orc.make_params(seed=1234), "bf16x3")
    n_img = args.images
    stream = [torch.from_numpy(orc.make_image(*SIZES[i % 3], seed=i)[0]).cuda() for i in range(24)]
    full = [torch.from_numpy(orc.make_image(HC, WC, seed=100 + i)[0]).cuda() for i in range(4)]
    full4 = torch.stack(full)

    # per-shape plans: one ForwardPlan (buffers + graph) per distinct shape, as Engine.plan builds them
    def per_shape():
        plans = {}
        for x in stream[:3]:
            p = plans.setdefault(tuple(x.shape[1:]), ForwardPlan(wts, int(x.shape[1]), int(x.shape[2]), **kw))
            p.forward(x)
        return plans
    shape_plans, shape_bytes, shape_peak = built(per_shape)

    def canvas(N):
        p = CanvasBatchPlan(wts, N, HC, WC, **kw)
        p.forward(stream[:N])
        return p
    cplans, cmem = {}, {}
    for N in (4, 8):
        cplans[N], b, pk = built(lambda N=N: canvas(N))
        cmem[N] = (b, pk)
    bplan4, _, _ = built(lambda: BatchPlan(wts, 4, HC, WC, **kw))
    cplan4_full = CanvasBatchPlan(wts, 4, HC, WC, **kw)
    graphs = {N: cplans[N].graph for N in cplans}

    def run_shapes(i):
        x = stream[i % 24]
        shape_plans[tuple(x.shape[1:])].forward(x)

    def run_canvas(N):
        def f(i):
            s = (i * N) % 24
            cplans[N].forward(stream[s:s + N])
        return f

    configs = [("ForwardPlan per shape, 1 in flight", lambda: device_ms(run_shapes, n_img) / n_img)]
    for N in (4, 8):
        configs.append(("CanvasBatchPlan N=%d" % N, lambda N=N: device_ms(run_canvas(N), n_img // N) / n_img))
    configs.append(("BatchPlan N=4, all 600x1000", lambda: device_ms(lambda i: bplan4.forward(full4), n_img // 4) / n_img))
    configs.append(("CanvasBatchPlan N=4, all 600x1000", lambda: device_ms(lambda i: cplan4_full.forward(full), n_img // 4) / n_img))
    for _, f in configs:          # warm-up: captures, module loads
        f()
    res = {name: [] for name, _ in configs}
    for _ in range(args.rounds):
        for name, f in configs:
            res[name].append(f())
    recaptured = any(cplans[N].graph is not graphs[N] for N in cplans)
    print("device time per image, stream of 600x{800,901,1000} (last two rows: all 600x1000), bf16x3, per-class NMS in the "
          "graph, median of %d rounds of %d images:" % (args.rounds, n_img))
    for name, _ in configs:
        m = statistics.median(res[name])
        print("  %-36s %7.3f ms  %6.1f img/s   (rounds: %s)" % (name, m, 1e3 / m, " ".join("%.3f" % v for v in res[name])))
    print("plans / graph captures / memory held by the plans / peak above it during the first run:")
    print("  %-36s %d / %d / %.0f MB / %.0f MB" % ("ForwardPlan per shape", len(shape_plans),
                                                   sum(p.graph is not None for p in shape_plans.values()), shape_bytes / 2**20,
                                                   shape_peak / 2**20))
    for N in (4, 8):
        print("  %-36s 1 / 1 / %.0f MB / %.0f MB" % ("CanvasBatchPlan N=%d" % N, cmem[N][0] / 2**20, cmem[N][1] / 2**20))
    print("re-capture after the first mix: %s" % ("YES" if recaptured else "none"))
    # outputs: every image of one canvas replay against its ForwardPlan
    ok = 0
    cplans[8].forward(stream[:8])
    torch.cuda.synchronize()
    got = cplans[8].unpack_result(cplans[8].result.cpu().numpy())
    for n in range(8):
        p = shape_plans[tuple(stream[n].shape[1:])]
        p.forward(stream[n])
        torch.cuda.synchronize()
        want = p.unpack_result(p.result.cpu().numpy())
        ok += same(got[n], want)
        print("image %d (%dx%d): R=%d, canvas %s ForwardPlan" % (n, stream[n].shape[1], stream[n].shape[2], want["count"],
                                                                 "==" if same(got[n], want) else "!="))
    print("bit-identical images: %d of 8" % ok)


if __name__ == "__main__":
    main()
