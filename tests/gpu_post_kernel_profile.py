"""Diagnostic (not a pytest): torch.profiler device time of the one-image post-processing kernels (rpn_decode_kernel,
topk_sort_kernel, rank_scatter_kernel, nms_mask_kernel, nms_scan_kernel, roi_pool_col_kernel, head_decode_kernel,
detect_kernel) in an eager ForwardPlan at 600x1000 (bf16x3, per-class NMS on), averaged over the profiled images.

    python tests/gpu_post_kernel_profile.py [--root TREE] [--images 20]

--root imports the package from another checkout of this project (e.g. an older build), so that two builds can be
compared in one session, alternating processes.
"""
import argparse
import collections
import os
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--images", type=int, default=20)
args = ap.parse_args()
for p in (args.root, os.path.join(args.root, "chainer-faster-rcnn_b200"), os.path.join(args.root, "oracle")):
    sys.path.insert(0, p)
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
from frcnn_b200.engine import ForwardPlan, PackedWeights  # noqa: E402

KERNELS = ("rpn_decode_kernel", "topk_sort_kernel", "rank_scatter_kernel", "nms_mask_kernel", "nms_scan_kernel",
           "roi_pool_col_kernel", "head_decode_kernel", "detect_kernel")


def main():
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    wts = PackedWeights(orc.make_params(seed=1234), "bf16x3")
    plan = ForwardPlan(wts, 600, 1000, anchors=anchors, with_detect=True, use_graph=False)
    imgs = [torch.from_numpy(orc.make_image(600, 1000, seed=i)[0]).cuda() for i in range(4)]
    for i in range(3):
        plan.forward(imgs[i % 4])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.images):
            plan.forward(imgs[i % 4])
        torch.cuda.synchronize()
    tot, cnt = collections.defaultdict(float), collections.defaultdict(int)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            for k in KERNELS:
                if k in ev.name:
                    tot[k] += ev.device_time_total
                    cnt[k] += 1
    print("root %s: device us per launch (%d images)" % (args.root, args.images))
    for k in KERNELS:
        print("  %-22s %9.2f us  (%d launches)" % (k, tot[k] / max(cnt[k], 1), cnt[k]))


if __name__ == "__main__":
    main()
