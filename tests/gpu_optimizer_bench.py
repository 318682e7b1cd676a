"""Measurement (not a pytest): the optimizer update and the canvas RPN step under each rule.

(a) frcnn_optimizer_update per rule (fp32 gradient) at the parameter counts of the VGG16 RPN step (trunk + RPN) and RCNN
    step (trunk + fc6/fc7/cls_score/bbox_pred), and frcnn_sgd_momentum beside them: device time from CUDA events over
    ITERS launches, and the bytes the rule must move (20 per parameter, Adam 28) over that time against the data sheet's
    3.35 TB/s.
(b) CanvasRpnTrainer N = 4 on a 600x1000 canvas, with MomentumSGD and with Adam, alternated round by round: images/s
    at the median round.
Prints the card's name and power limit with the numbers, and one JSON line."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "chainer-faster-rcnn_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import frcnn_oracle as orc  # noqa: E402
from frcnn_b200 import optimizers, train_ops  # noqa: E402
from frcnn_b200.train_engine import TRUNK, CanvasRpnTrainer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
ITERS, ROUNDS, ROUND_STEPS = 50, 7, 10
ANCHORS = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def param_counts():
    trunk = sum(co * ci * 9 + co for _, ci, co in TRUNK)
    rpn = 512 * 512 * 9 + 512 + 54 * 512 + 54
    head = 25088 * 4096 + 4096 + 4096 * 4096 + 4096 + 105 * 4096 + 105
    return {"rpn_step": trunk + rpn, "rcnn_step": trunk + head}


def time_update(rule, n):
    w, g = torch.randn(n, device="cuda") * 0.01, torch.randn(n, device="cuda") * 1e-3
    s = [torch.zeros(n, device="cuda") for _ in range(2 if rule == optimizers.ADAM else 1)]
    if rule == "sgd_momentum":
        launch = lambda: train_ops.sgd_momentum(w, s[0], g, 0.001, 0.9, 0.0005)             # noqa: E731
        per = 20
    else:
        hyper = torch.from_numpy(optimizers.RULES[rule]().hyper(0.0005, 1)).cuda()
        launch = lambda: train_ops.optimizer_update(rule, w, s[0], s[1] if len(s) > 1 else None, g, hyper)   # noqa: E731
        per = 28 if rule == optimizers.ADAM else 20
    for _ in range(5):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(ITERS):
        launch()
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b) / ITERS
    del w, g, s
    torch.cuda.empty_cache()
    return ms, per * n / (ms * 1e-3)


def canvas_rates():
    from test_canvas_train_gpu import _images
    params = orc.make_params(seed=3)
    xs, gts = _images([(600, 1000), (600, 800), (600, 901), (500, 1000)], 5)
    trainers = {"MomentumSGD": CanvasRpnTrainer(params, 4, 600, 1000, ANCHORS, subsample="none"),
                "Adam": CanvasRpnTrainer(params, 4, 600, 1000, ANCHORS, subsample="none", optimizer=optimizers.Adam())}
    for tr in trainers.values():
        for _ in range(3):
            tr.step(xs, gts)
    torch.cuda.synchronize()
    ms = {k: [] for k in trainers}
    for _ in range(ROUNDS):
        for k, tr in trainers.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(ROUND_STEPS):
                tr.step(xs, gts)
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b) / ROUND_STEPS)
    return {k: dict(ms_per_step_median=float(np.median(v)), ms_min=min(v), ms_max=max(v),
                    images_per_s=4 * 1000.0 / float(np.median(v))) for k, v in ms.items()}


def main():
    torch.cuda.set_device(0)
    gpu = card()
    out = {"gpu": gpu, "update": {}}
    print("card:", gpu)
    for step, n in param_counts().items():
        for rule, name in [("sgd_momentum", "frcnn_sgd_momentum")] + [(r.rule, r.__name__) for r in optimizers.RULES]:
            ms, bps = time_update(rule, n)
            out["update"]["%s/%s" % (step, name)] = dict(params=n, ms=ms, bytes_per_s=bps, share_of_3_35TBps=bps / HBM_BYTES_PER_S)
            print("%-10s %-20s n=%11d  %.3f ms  %.2f TB/s  (%.0f %% of 3.35 TB/s)" % (step, name, n, ms, bps / 1e12,
                                                                                     100 * bps / HBM_BYTES_PER_S))
    out["canvas_rpn_N4"] = canvas_rates()
    for k, v in out["canvas_rpn_N4"].items():
        print("CanvasRpnTrainer N=4 %-12s %.2f ms/step (%.2f-%.2f)  %.1f images/s" % (
            k, v["ms_per_step_median"], v["ms_min"], v["ms_max"], v["images_per_s"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
