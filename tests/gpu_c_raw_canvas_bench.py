"""Measurement (not a pytest): raw uint8 photos of mixed sizes to detections on the host through the one C call
frcnn_detect_vgg16_raw, against CanvasStreamRunner, in ONE process.

    python tests/gpu_c_raw_canvas_bench.py [--images 96] [--rounds 7] [--out FILE.json]

The stream is raw BGR photos of 300x500, 333x500 and 375x500 (they resize to 600x1000, 600x901 and 600x800), bf16x3,
N = 4 per batch on a 600 x 1000 canvas, per-class NMS at conf 0.05, and both modes end with forward.py's detection lists on
the host:
  c_api   what a C caller does: frcnn_detect_vgg16_raw captured ONCE into a CUDA graph (engine.CCanvasForward.launch); per
          batch the host writes the header and the photos into a pinned mirror of the [header | pixels] block, then one
          H2D of the block, one 8N-byte H2D of im_scale, one graph replay and ONE D2H of the lists buffer [det_count | dets |
          scores] -- the detection lists themselves, nothing to assemble on the host.  Two pinned slots: the host prepares
          batch b while the GPU runs batch b-1.
  runner  CanvasStreamRunner on CanvasBatchPlan(raw_input=True) (depth 2, one lane): one H2D, one graph, one D2H of the N
          result blocks, then preprocess.result_detections on the host.
Modes alternate round by round after a warm-up; the medians over the rounds are reported: host wall images/s (the clock stops
after a device synchronise), device ms per image (CUDA events on the submitting stream around the whole round) and the bytes
copied device-to-host per image.  Both modes must return identical detections.  The card's name and power limit are read in
the same run."""
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
from frcnn_b200.engine import CanvasStreamRunner, CCanvasForward, Engine  # noqa: E402

SHAPES = [(300, 500), (333, 500), (375, 500)]
HC, WC, N, CONF = 600, 1000, 4, 0.05


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


class CRawStream(object):
    """Host photos -> host detection lists through one captured frcnn_detect_vgg16_raw graph, two pinned slots deep."""

    def __init__(self, cf, depth=2):
        self.cf, self.D = cf, depth
        self.stage = [ops.PinnedBlock((cf.block.numel(),), np.uint8) for _ in range(depth)]
        self.scale = [ops.PinnedBlock((cf.N,), np.float64) for _ in range(depth)]
        self.res = [ops.PinnedBlock((cf.lists.numel(),), np.int32) for _ in range(depth)]
        self.done = [torch.cuda.Event() for _ in range(depth)]
        cf.launch()                                   # warm-up launch outside the capture
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, capture_error_mode="thread_local"):
            cf.launch()
        self.d2h_bytes = 0

    def run(self, imgs):
        cf, D, out, batches = self.cf, self.D, [], []
        cur = torch.cuda.current_stream()

        def deliver(b):
            s = b % D
            self.done[s].synchronize()
            out.extend(cf.unpack_lists(self.res[s].np, batches[b]))

        for b, s0 in enumerate(range(0, len(imgs), cf.N)):
            chunk, s = imgs[s0:s0 + cf.N], b % D
            if b >= D:
                deliver(b - D)                        # slot reuse: batch b-D is finished
            hdr, scales, _ = preprocess.raw_batch_header(preprocess.raw_photo_shapes(chunk), cf.N, cf.H, cf.W, cf.arena_bytes)
            batches.append(len(chunk))
            nbytes = preprocess.fill_raw_block(self.stage[s].np, hdr, chunk, cf.N)
            self.scale[s].np[:] = 0.0
            self.scale[s].np[:len(scales)] = scales
            self.stage[s].h2d(cf.block, cur, nbytes=nbytes)
            self.scale[s].h2d(cf.im_scale, cur)
            self.graph.replay()
            self.res[s].d2h(cf.lists, cur)
            self.d2h_bytes += self.res[s].nbytes
            self.done[s].record(cur)
        for b in range(max(0, len(batches) - D), len(batches)):
            deliver(b)
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=96)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    assert args.images % (3 * N) == 0 and args.rounds >= 5
    card = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]).decode().strip()
    anchors = orc.generate_anchors(ratios=(0.5, 1, 2), scales=(8, 16, 32))
    eng = Engine(orc.make_params(seed=1234), precision="bf16x3", anchors=anchors, with_detect=True, det_conf=CONF)
    rng = np.random.default_rng(7)
    imgs = [rng.integers(0, 256, SHAPES[i % 3] + (3,), dtype=np.uint8) for i in range(args.images)]
    n = len(imgs)
    arena = N * 3 * 375 * 500 + 64 * N
    runner = CanvasStreamRunner(eng.canvas_plan(N, HC, WC, raw_input=True, arena_bytes=arena), depth=2)
    cstream = CRawStream(CCanvasForward(eng.weights, N, HC, WC, anchors, raw_input=True, arena_bytes=arena, det_conf=CONF))

    def runner_d2h():
        return runner.n_words * 4 * (n // N)

    modes = [("c_api_detect_vgg16_raw_graph", lambda: cstream.run(imgs)), ("canvas_stream_runner", lambda: runner.run(imgs))]
    outs = {name: fn() for name, fn in modes}                   # warm-up
    torch.cuda.synchronize()
    assert outs["c_api_detect_vgg16_raw_graph"] == outs["canvas_stream_runner"] and all(len(d) > 0 for d in outs["canvas_stream_runner"])
    d0 = cstream.d2h_bytes
    cstream.run(imgs)
    d2h = {"c_api_detect_vgg16_raw_graph": (cstream.d2h_bytes - d0) / n, "canvas_stream_runner": runner_d2h() / n}
    wall, dev = {m: [] for m, _ in modes}, {m: [] for m, _ in modes}
    for _ in range(args.rounds):
        for name, fn in modes:
            got, sec, ms = timed(fn)
            assert got == outs[name]
            wall[name].append(n / sec)
            dev[name].append(ms / n)
    result = dict(card=card, images=n, rounds=args.rounds, shapes=SHAPES, N=N, canvas=[HC, WC], modes={})
    for name, _ in modes:
        result["modes"][name] = dict(host_wall_images_per_s=round(statistics.median(wall[name]), 1),
                                     host_wall_min_max=[round(min(wall[name]), 1), round(max(wall[name]), 1)],
                                     device_ms_per_image=round(statistics.median(dev[name]), 3),
                                     d2h_bytes_per_image=round(d2h[name]))
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
