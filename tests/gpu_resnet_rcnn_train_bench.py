"""Measurement (not a pytest): the RCNN training step at 600x1000 with the ResNet-50 and ResNet-101 trunks
(ResNetRcnnTrainer, frozen BatchNorm) beside the VGG16 step (RcnnTrainer), bf16x3, 300 proposals, NumPy sampling (the
reference's ProposalTargetLayer draw, one host round trip per step), dropout on, random-init weights with livelier RPN
heads, one synthetic image with three ground-truth boxes.

Every trainer is warmed up first; then the trainers alternate round by round.  A round is ROUND_STEPS steps; its device
time comes from CUDA events around it (ending in a synchronise).  Within the round, events after forward and after backward
split each step into forward, backward and update (the update includes the weight repack).  Reports the median and
min-max device ms per image over the rounds, images/s at the median, the share of forward / backward / update, the device
memory each trainer holds (allocated after its warm-up, over the baseline), and CUDA-event times of fc6 alone: its
forward GEMM, data gradient, weight gradient and the repack of its planes from the fp32 master (median of FC_REPS runs
each, on the buffers the last step left).  Prints the card's name and power limit with the numbers, a markdown table and
one JSON line."""
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
from frcnn_b200.resnet_train import ResNetRcnnTrainer  # noqa: E402
from frcnn_b200.train_engine import RcnnTrainer  # noqa: E402

ROUNDS, ROUND_STEPS, WARMUP, FC_REPS = 7, 6, 3, 10
H, W, POST_N = 600, 1000, 300
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def lively(params):
    rng = np.random.default_rng(0)
    for k in ("RPN/rpn_cls_score/W", "RPN/rpn_bbox_pred/W"):
        params[k] = (rng.standard_normal(params[k].shape) * 0.05).astype(np.float32)
    return params


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


def fc6_times(tr):
    """Median CUDA-event ms of fc6's forward, data gradient, weight gradient and repack, each launched as the step does."""
    C, R_cap = tr.feat_ch, tr.post_n
    fwd, b, dg = tr.packed["fc6"]
    dy6, gp = tr._gact(1, R_cap, 4096), tr._gact(1, R_cap, 49 * C, tag=1)
    dy6T, p5T = tr._tbuf(1, 4096, 1, R_cap, tag=1), tr._tbuf(1, 49 * C, 1, R_cap)
    ops = dict(forward=lambda: tr._conv(tr.pool5, fwd, b, 1, True, "rois", out=tr.fc6),
               dgrad=lambda: tr._conv(dy6, dg, tr.zero_bias, 1, False, "roi_grads", out=gp),
               wgrad=lambda: tr._fc_wgrad(dy6T, p5T, 4096, 49 * C, tr.grads("fc6/W")),
               repack=lambda: tr._repack("fc6", tr.weights("fc6/W"), tr.weights("fc6/b"), 4096))
    out = {}
    for name, fn in ops.items():
        ms = []
        for _ in range(FC_REPS):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        out[name] = float(np.median(ms))
    return out


def main():
    x = torch.from_numpy(orc.make_image(H, W, seed=0)[0]).cuda()
    gt = torch.tensor([[40, 60, 400, 380, 3], [300, 100, 900, 560, 7], [600, 250, 850, 500, 1]], dtype=torch.float32).cuda()
    np.random.seed(0)
    trainers = []
    base = torch.cuda.memory_allocated()
    for name, build in [("VGG16 RcnnTrainer", lambda: RcnnTrainer(lively(orc.make_params(seed=1234)), H, W, ANCHORS, post_n=POST_N)),
                        ("ResNet-50 ResNetRcnnTrainer", lambda: ResNetRcnnTrainer(lively(orc.make_resnet_params(50, seed=3)), H, W,
                                                                                  ANCHORS, n_layers=50, post_n=POST_N)),
                        ("ResNet-101 ResNetRcnnTrainer", lambda: ResNetRcnnTrainer(lively(orc.make_resnet_params(101, seed=3)), H, W,
                                                                                   ANCHORS, n_layers=101, post_n=POST_N))]:
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
    for t in trainers:
        t["fc6"] = fc6_times(t["tr"])
    gpu = card()
    rows = []
    print("card: %s; %dx%d, bf16x3, %d proposals, NumPy sampling, dropout; %d rounds of %d steps per trainer"
          % (gpu, H, W, POST_N, ROUNDS, ROUND_STEPS))
    print("| trainer | ms / image (median) | min-max | images/s | forward / backward / update | memory held (GB) "
          "| fc6 forward / dgrad / wgrad / repack (ms) |")
    print("|---|---|---|---|---|---|---|")
    for t in trainers:
        ms = np.array(t["ms"])
        med = float(np.median(ms))
        share = t["phases"] / t["phases"].sum()
        f = t["fc6"]
        rows.append(dict(trainer=t["name"], ms_median=med, ms_min=float(ms.min()), ms_max=float(ms.max()), images_per_s=1e3 / med,
                         forward=float(share[0]), backward=float(share[1]), update=float(share[2]), memory_gb=t["held_gb"],
                         fc6_ms=f))
        print("| %s | %.2f | %.2f-%.2f | %.1f | %.0f%% / %.0f%% / %.0f%% | %.2f | %.3f / %.3f / %.3f / %.3f |" % (
            t["name"], med, ms.min(), ms.max(), 1e3 / med, 100 * share[0], 100 * share[1], 100 * share[2], t["held_gb"],
            f["forward"], f["dgrad"], f["wgrad"], f["repack"]))
    print(json.dumps(dict(card=gpu, shape=[H, W], post_n=POST_N, rounds=ROUNDS, round_steps=ROUND_STEPS, rows=rows)))


if __name__ == "__main__":
    main()
