"""Diagnostic (not a pytest): images per second of the batched forward (engine.BatchPlan) against one image at a time
(ForwardPlan) and against LanePool, at the benchmarked configuration: 600x1000, bf16x3, per-class NMS in the graph,
random-init weights.  Everything in one process, the configurations alternating round by round.

Prints the card and its power limit, device time per image of every configuration (median over the rounds), per-layer
times of conv4_x, conv5_x, the RPN 3x3 and fc6 at N = 1 and N = 4, and whether BatchPlan's outputs equal ForwardPlan's.

    python tests/gpu_batch_bench.py [--rounds 5] [--images 48]
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
from frcnn_b200 import ops  # noqa: E402
from frcnn_b200.engine import Engine, LanePool  # noqa: E402

H, W = 600, 1000
LAYERS = ("conv4_1", "conv4_2", "conv4_3", "conv5_1", "conv5_2", "conv5_3")


def device_ms(fn, reps, pool=None):
    """Device ms of reps calls of fn(i) on the current stream (pool: a LanePool whose lanes fork from and join into it)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    if pool is not None:
        pool.fork()
    for i in range(reps):
        fn(i)
    if pool is not None:
        pool.join()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def layer_times(plan, batch, reps=20):
    """ms per launch of conv4_x, conv5_x, the RPN 3x3 and fc6 on the plan's own buffers (launches back to back)."""
    w, out = plan.w, {}
    conv = ops.conv2d_batch if batch else ops.conv2d
    for i, (name, fused, _) in enumerate(plan.trunk_steps):
        if name in LAYERS:
            hi, lo, b = w.convs[name]
            out[name] = device_ms(lambda _: conv(plan.acts[i], hi, lo, b, 3, True, out=plan.acts[i + 1], fuse_pool=fused), reps) / reps
    hi, lo, b = w.rpn3
    out["rpn_3x3"] = device_ms(lambda _: conv(plan.feat, hi, lo, b, 3, True, out=plan.rpn_mid), reps) / reps
    hi, lo, b = w.fc6
    if batch:
        f = lambda _: ops.linear_batch(plan.pool5, hi, lo, b, True, plan.post_n, counts=plan.counts,   # noqa: E731
                                       count_stride=plan.block_words, out=plan.fc6, work=plan.fc_work)
    else:
        f = lambda _: ops.linear(plan.pool5, hi, lo, b, True, m_valid=plan.prop.count, out=plan.fc6, work=plan.fc_work)   # noqa: E731
    out["fc6"] = device_ms(f, reps) / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--images", type=int, default=48, help="images per timed window (a multiple of 8)")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card: %s" % q.stdout.strip().splitlines()[0] if q.stdout else "card: (nvidia-smi unavailable)")
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    eng = Engine(orc.make_params(seed=1234), precision="bf16x3", anchors=anchors, use_graph=True, with_detect=True,
                 det_nms_thresh=0.3, det_conf=0.8)
    imgs = [torch.from_numpy(orc.make_image(H, W, seed=i)[0]).cuda() for i in range(8)]
    batch = {N: torch.stack(imgs[:N]) for N in (1, 2, 4, 8)}
    plan = eng.plan(H, W)
    lanes4 = LanePool(plan, lanes=4)
    bplans = {N: eng.batch_plan(N, H, W) for N in (1, 2, 4, 8)}
    blanes = {N: LanePool(bplans[N].clone(), lanes=2) for N in (1, 2, 4, 8)}
    n_img = args.images

    def one(i):
        plan.forward(imgs[i % 8])

    def pooled(pool, src):
        def run(i):
            pool.submit(i, src(i))
        return run

    configs = [("ForwardPlan, 1 in flight", lambda: device_ms(one, n_img) / n_img)]

    configs.append(("LanePool, 4 lanes", lambda: device_ms(pooled(lanes4, lambda i: imgs[i % 8]), n_img, lanes4) / n_img))
    for N in (1, 2, 4, 8):
        bp, bl = bplans[N], blanes[N]
        configs.append(("BatchPlan N=%d, 1 in flight" % N,
                        lambda bp=bp, N=N: device_ms(lambda i: bp.forward(batch[N]), n_img // N) / n_img))
        configs.append(("BatchPlan N=%d, 2 lanes" % N,
                        lambda bl=bl, N=N: device_ms(pooled(bl, lambda i: batch[N]), n_img // N, bl) / n_img))
    for _, f in configs:          # warm-up: captures, module loads
        f()
    res = {name: [] for name, _ in configs}
    for _ in range(args.rounds):
        for name, f in configs:
            res[name].append(f())
    base = statistics.median(res["ForwardPlan, 1 in flight"])
    print("device time per image, 600x1000 bf16x3, per-class NMS in the graph, median of %d rounds of %d images:"
          % (args.rounds, n_img))
    for name, _ in configs:
        m = statistics.median(res[name])
        print("  %-30s %7.3f ms  %6.1f img/s  x%.2f vs one in flight   (rounds: %s)"
              % (name, m, 1e3 / m, base / m, " ".join("%.3f" % v for v in res[name])))
    # per-layer: ForwardPlan (N = 1) and BatchPlan N = 4, eager launches on the plans' own buffers
    plan.forward(imgs[0])
    bplans[4].forward(batch[4])
    torch.cuda.synchronize()
    t1, t4 = layer_times(plan, False), layer_times(bplans[4], True)
    t1b, t4b = layer_times(plan, False), layer_times(bplans[4], True)      # second pass, alternating
    print("per launch (ms), N=1 -> N=4 (per image):")
    for k in t1:
        a, b = statistics.mean((t1[k], t1b[k])), statistics.mean((t4[k], t4b[k]))
        print("  %-8s %7.4f -> %7.4f  (%6.4f per image, x%.2f)" % (k, a, b, b / 4, a / (b / 4)))
    # outputs: BatchPlan N = 4 against ForwardPlan on each image
    bplans[4].forward(batch[4])
    got = bplans[4].unpack_result(bplans[4].result.cpu().numpy())
    same = 0
    for n in range(4):
        plan.forward(imgs[n])
        want = plan.unpack_result(plan.result.cpu().numpy())
        ok = got[n]["count"] == want["count"] and all(
            np.array_equal(np.asarray(got[n][f]).view(np.int32), np.asarray(want[f]).view(np.int32))
            for f in ("prob", "boxes", "rois", "scores", "keep_count", "conf_count", "keep_idx"))
        same += ok
        print("image %d: R=%d, BatchPlan N=4 %s ForwardPlan" % (n, want["count"], "==" if ok else "!="))
    print("bit-identical images: %d of 4" % same)


if __name__ == "__main__":
    main()
