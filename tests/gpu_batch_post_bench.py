"""Diagnostic (not a pytest): device time of the post-processing stages of the 600x1000 forward -- ProposalLayer, RoI
pooling, head decode and the per-class NMS -- over N images, run once per image (the one-image entry points at pointer
offsets) against once per batch (the _batch entry points: one launch per kernel).  Inputs are the RPN output, feature map
and head output of a real BatchPlan forward (bf16x3, random-init weights).  CUDA events over many launches, the two
modes alternating round by round; prints the card and its power limit, and whether both modes wrote the same results.

    python tests/gpu_batch_post_bench.py [--rounds 5] [--reps 50]
"""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
from frcnn_b200 import ops  # noqa: E402
from frcnn_b200.engine import BatchPlan, PackedWeights  # noqa: E402

H, W = 600, 1000


def device_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def stages(bp):
    """{stage: (per-image fn, batched fn)} on the plan's own inputs; per-image outputs go to private buffers."""
    N, post, w = bp.N, bp.post_n, bp.w
    NC, hw = w.num_classes, bp.fh * bp.fw
    feat, rpn = bp.feat, bp.rpn_out.view(N, hw, w.rpn_ld)
    works = [ops.ProposalWorkspace(w.n_anchors, bp.fh, bp.fw, bp.pre_n, post, "cuda") for _ in range(N)]
    bwork = ops.ProposalBatchWorkspace(N, w.n_anchors, bp.fh, bp.fw, bp.pre_n, post, "cuda")
    pool1 = ops.Act(torch.empty((N, 1, post, 49 * 512), dtype=torch.bfloat16, device="cuda"),
                    torch.empty((N, 1, post, 49 * 512), dtype=torch.bfloat16, device="cuda"))
    poolb = ops.Act(pool1.hi[:, 0].clone(), pool1.lo[:, 0].clone())
    prob1 = torch.empty((N, post, NC), device="cuda")
    boxes1 = torch.empty((N, post, 4 * NC), device="cuda")
    probb, boxesb = torch.empty_like(prob1), torch.empty_like(boxes1)
    det1 = [ops.detect(bp.prob[k], bp.boxes[k], bp.prop.count[k:k + 1]) for k in range(N)]
    detb = ops.detect_batch(bp.prob, bp.boxes, bp.prop.count)
    cnt = bp.prop.count
    args = (w.n_anchors, bp.fh, bp.fw, bp.feat_stride, H, W, bp.min_size, bp.pre_n, post, bp.nms_thresh)
    img = lambda k: ops.Act(feat.hi[k], feat.lo[k])         # noqa: E731

    def prop1():
        for k in range(N):
            ops.proposals(rpn[k], None, bp.anchors, *args, layout="nhwc", ld=w.rpn_ld, cls_is_logits=True, work=works[k])

    def roi1():
        for k in range(N):
            ops.roi_pool(img(k), bp.prop.rois[k], cnt[k:k + 1], 7, 7, 1.0 / 16, out=ops.Act(pool1.hi[k], pool1.lo[k]))

    def dec1():
        for k in range(N):
            ops.head_decode(bp.head_out[k, :post], w.head_ld, bp.prop.rois[k], cnt[k:k + 1], NC, H, W, out_prob=prob1[k],
                            out_boxes=boxes1[k])

    def det1_():
        for k in range(N):
            ops.detect(bp.prob[k], bp.boxes[k], cnt[k:k + 1], out=det1[k])

    return {
        "proposals": (prop1, lambda: ops.proposals_batch(rpn, None, bp.anchors, *args, layout="nhwc", ld=w.rpn_ld,
                                                         cls_is_logits=True, work=bwork)),
        "roi_pool": (roi1, lambda: ops.roi_pool_batch(feat, bp.prop.rois, cnt, 7, 7, 1.0 / 16, out=poolb)),
        "head_decode": (dec1, lambda: ops.head_decode_batch(bp.head_out[:, :post], w.head_ld, bp.prop.rois, cnt, NC, H, W,
                                                            out_prob=probb, out_boxes=boxesb)),
        "detect": (det1_, lambda: ops.detect_batch(bp.prob, bp.boxes, cnt, out=detb)),
    }, (works, bwork, pool1, poolb, prob1, boxes1, probb, boxesb, det1, detb)


def outputs_agree(bufs):
    works, bwork, pool1, poolb, prob1, boxes1, probb, boxesb, det1, detb = bufs
    eq = lambda a, b: torch.equal(a.contiguous().view(torch.int32) if a.dtype == torch.float32 else a,      # noqa: E731
                                  b.contiguous().view(torch.int32) if b.dtype == torch.float32 else b)
    ok = all(eq(works[k].rois, bwork.rois[k]) and int(works[k].count.item()) == int(bwork.count[k]) for k in range(len(works)))
    ok = ok and torch.equal(pool1.hi[:, 0], poolb.hi) and torch.equal(pool1.lo[:, 0], poolb.lo)
    ok = ok and eq(prob1, probb) and eq(boxes1, boxesb)
    ok = ok and all(eq(det1[k][i], detb[i][k]) for k in range(len(det1)) for i in range(3))
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card: %s" % (q.stdout.strip().splitlines()[0] if q.stdout else "(nvidia-smi unavailable)"))
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    wts = PackedWeights(orc.make_params(seed=1234), "bf16x3")
    x = torch.stack([torch.from_numpy(orc.make_image(H, W, seed=i)[0]) for i in range(8)]).cuda()
    print("post-processing at 600x1000 (proposals 6000 -> 300, RoI pool 7x7x512, decode, 20-class NMS), device ms per batch")
    print("  %-3s %-12s %10s %10s %8s" % ("N", "stage", "per-image", "batched", "speedup"))
    for N in (1, 2, 4, 8):
        bp = BatchPlan(wts, N, H, W, anchors=anchors, with_detect=True, use_graph=False)
        bp.forward(x[:N])
        torch.cuda.synchronize()
        st, bufs = stages(bp)
        for one, bat in st.values():
            one(), bat()
        torch.cuda.synchronize()
        agree = outputs_agree(bufs)
        res = {k: ([], []) for k in st}
        for _ in range(args.rounds):
            for k, (one, bat) in st.items():
                res[k][0].append(device_ms(one, args.reps))
                res[k][1].append(device_ms(bat, args.reps))
        tot1 = tot2 = 0.0
        for k in st:
            a, b = statistics.median(res[k][0]), statistics.median(res[k][1])
            tot1, tot2 = tot1 + a, tot2 + b
            print("  %-3d %-12s %10.4f %10.4f %7.2fx" % (N, k, a, b, a / b))
        print("  %-3d %-12s %10.4f %10.4f %7.2fx   (outputs equal: %s)" % (N, "all", tot1, tot2, tot1 / tot2, agree))
        del bp, st, bufs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
