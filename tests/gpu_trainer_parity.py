"""Three training steps of every trainer kind with fixed seeds, saved to npz, to compare two builds of the trainers bit for
bit: losses, g_flat, w_flat and v_flat after the last step.  The kinds are the eight trainers (VGG16 and ResNet-50, one
image and canvas, RPN and RCNN) and the one-image VGG16 RPN step with NumPy subsampling.  The flat buffers are saved as
SHA-256 digests of their bytes: the ResNet RCNN trainers' are 1.6 GB each.

    python tests/gpu_trainer_parity.py --out a.npz [--pkg DIR]     # DIR: the chainer-faster-rcnn_b200 tree to import
    python tests/gpu_trainer_parity.py --compare a.npz b.npz
"""
import argparse
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W, STEPS = 296, 392, 3


def _inputs(torch, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    xs = [torch.randn((3, H, W), device="cuda", generator=g) * 50.0 for _ in range(n)]
    gts = [torch.tensor([[20.0 + 7 * k, 30.0, 160.0 + 5 * k, 200.0, 3.0], [150.0, 60.0, 370.0, 280.0, 11.0]],
                        device="cuda") for k in range(n)]
    return xs, gts


def run(out):
    import torch
    import frcnn_oracle as orc
    from frcnn_b200.resnet_train import CanvasResNetRcnnTrainer, CanvasResNetRpnTrainer, ResNetRcnnTrainer, ResNetRpnTrainer
    from frcnn_b200.train_engine import CanvasRcnnTrainer, CanvasRpnTrainer, RcnnTrainer, RpnTrainer
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    vgg = orc.make_params(seed=77)
    rng = np.random.default_rng(78)
    for k in ("cls_score/W", "bbox_pred/W"):
        vgg[k] = (rng.standard_normal(vgg[k].shape) * 0.02).astype(np.float32)
    r50 = orc.make_resnet_params(50, seed=3)
    for k, s in (("RPN/rpn_cls_score/W", 0.05), ("RPN/rpn_bbox_pred/W", 0.05), ("fc6/W", 0.001), ("fc7/W", 0.01),
                 ("cls_score/W", 0.01), ("bbox_pred/W", 0.01)):     # proposals that overlap the boxes, a live head
        r50[k] = (rng.standard_normal(r50[k].shape) * s).astype(np.float32)
    res = {}
    kinds = [("rpn", lambda: RpnTrainer(vgg, H, W, anchors)),
             ("rpn_numpy", lambda: RpnTrainer(vgg, H, W, anchors, subsample="numpy")),
             ("rcnn", lambda: RcnnTrainer(vgg, H, W, anchors, post_n=120)),
             ("canvas_rpn", lambda: CanvasRpnTrainer(vgg, 2, H, W, anchors)),
             ("canvas_rcnn", lambda: CanvasRcnnTrainer(vgg, 2, H, W, anchors, post_n=120)),
             ("resnet50", lambda: ResNetRpnTrainer(orc.make_resnet_params(50, seed=3), H, W, anchors, n_layers=50)),
             ("resnet50_rcnn", lambda: ResNetRcnnTrainer(r50, H, W, anchors, n_layers=50, post_n=120)),
             ("canvas_resnet50_rpn", lambda: CanvasResNetRpnTrainer(r50, 2, H, W, anchors, n_layers=50)),
             ("canvas_resnet50_rcnn", lambda: CanvasResNetRcnnTrainer(r50, 2, H, W, anchors, n_layers=50, post_n=120))]
    for name, make in kinds:
        torch.manual_seed(0)
        np.random.seed(0)
        tr = make()
        losses = []
        for s in range(STEPS):
            canvas = name.startswith("canvas")
            xs, gts = _inputs(torch, 2 if canvas else 1, 100 + s)
            np.random.seed(10 + s)
            losses.append(tr.step(xs, gts).clone() if canvas else tr.step(xs[0], gts[0]).clone())
        torch.cuda.synchronize()
        res[name + "/losses"] = torch.stack(losses).cpu().numpy()
        for f in ("g_flat", "w_flat", "v_flat"):
            res[name + "/" + f] = np.array(hashlib.sha256(getattr(tr, f).cpu().numpy().tobytes()).hexdigest())
        print(name, res[name + "/losses"][-1].ravel().tolist(), flush=True)
        del tr
        torch.cuda.empty_cache()
    np.savez(out, **res)


def compare(a, b):
    a, b = np.load(a), np.load(b)
    bad = [k for k in a.files if a[k].shape != b[k].shape or a[k].tobytes() != b[k].tobytes()]
    print("keys", len(a.files), "bit-identical" if not bad and a.files == b.files else "DIFFER: %s" % bad)
    return 1 if bad or a.files != b.files else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--pkg", default=os.path.join(ROOT, "chainer-faster-rcnn_b200"))
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    sys.path[:0] = [os.path.abspath(args.pkg), os.path.join(ROOT, "oracle")]
    run(args.out)
