"""Tuning sweep (not a pytest file): time every conv/GEMM layer of the headline config for each
N-tile / pixel-tile choice.  Prints a table; the winners go into the heuristic in conv_gemm_sm90.cu."""
import sys
import torch
sys.path[:0] = ["chainer-faster-rcnn_b200"]
from frcnn_b200 import ops

LAYERS = [  # H, W, Cin, Cout, k
    (600, 1000, 16, 64, 3), (600, 1000, 64, 64, 3), (300, 500, 64, 128, 3), (300, 500, 128, 128, 3),
    (150, 250, 128, 256, 3), (150, 250, 256, 256, 3), (75, 125, 256, 512, 3), (75, 125, 512, 512, 3),
    (38, 63, 512, 512, 3), (1, 300, 25088, 4096, 1), (1, 300, 4096, 4096, 1),
]
TILES = [(8, 16), (16, 8), (4, 32), (2, 64), (1, 128)]
precisions = sys.argv[1:] or ["bf16x3", "bf16"]
for prec in precisions:
    for (H, W, Cin, Cout, k) in LAYERS:
        x3 = prec == "bf16x3"
        hi = torch.randn(H, W, Cin, device="cuda").to(torch.bfloat16)
        act = ops.Act(hi, (torch.randn_like(hi.float()) * 0.01).to(torch.bfloat16) if x3 else None)
        wh = (torch.randn(k * k, Cout, Cin, device="cuda") * 0.02).to(torch.bfloat16)
        wl = (torch.randn(k * k, Cout, Cin, device="cuda") * 1e-4).to(torch.bfloat16) if x3 else None
        bias = torch.zeros(Cout, device="cuda")
        yh = torch.empty(H, W, Cout, device="cuda", dtype=torch.bfloat16)
        out = ops.Act(yh, torch.empty_like(yh) if x3 else None)
        gflop = 2.0 * H * W * Cout * k * k * Cin / 1e9
        res = []
        tiles = TILES if H > 1 else [(1, 128)]
        for cg in (1, 2):
            for bn in (64, 128, 256):
                if bn > Cout:
                    continue
                for (th, tw) in tiles:
                    ops.set_conv_tile(bn, th, tw)
                    ops.set_conv_cta_group(cg)
                    for _ in range(2):
                        ops.conv2d(act, wh, wl, bias, k, True, out=out)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(5):
                        ops.conv2d(act, wh, wl, bias, k, True, out=out)
                    e1.record()
                    torch.cuda.synchronize()
                    res.append((e0.elapsed_time(e1) / 5, bn, th, tw, cg))
        ops.set_conv_tile(0, 0, 0)
        ops.set_conv_cta_group(0)
        for _ in range(2):
            ops.conv2d(act, wh, wl, bias, k, True, out=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            ops.conv2d(act, wh, wl, bias, k, True, out=out)
        e1.record()
        torch.cuda.synchronize()
        auto = e0.elapsed_time(e1) / 5
        res.sort()
        best = res[0]
        print("%s %4dx%4dx%5d->%4d k%d  auto %.4f ms (%.0f TF) | best %.4f ms bn%d %dx%d (%.0f TF) | %s" % (
            prec, H, W, Cin, Cout, k, auto, gflop / auto, best[0], best[1], best[2], best[3], gflop / best[0],
            " ".join("cg%d/bn%d/%dx%d:%.3f" % (r[4], r[1], r[2], r[3], r[0]) for r in res[:8])), flush=True)
