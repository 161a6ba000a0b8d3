#!/usr/bin/env python
"""Canny annotator timing on one GPU, against cv2.Canny on the same host:

- CannyDetector.__call__ from a host image to a host map (the copies included) at 512^2, 512 x 768 and 1024^2: a host
  clock around `iters` calls, each of which ends in a synchronising copy back;
- cv2.Canny on the same images, at OpenCV's default thread count and at one thread;
- CannyDetector.detect on the device (CUDA events) at 1 x 512^2, 16 x 512^2 and 128 x 512^2, and on the spiral of
  tests/canny_golden.py (one 87 000-pixel candidate component);
- with --profile, a separate run: torch.profiler's device time per kernel over `iters` detect calls at 16 x 512^2.

    python tools/canny_bench.py [--iters 20] [--repeats 5] [--profile] [--out FILE]

Thresholds (100, 200) throughout, on tests/canny_golden.py's textured images.  Every figure is the median of `repeats`
windows of `iters` calls, and the JSON line also holds each figure's min and max ("<name>_spread").  Prints the card's
name and power limit read in the same run, and one JSON line."""
import argparse
import json
import os
import statistics
import sys
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.text_encoder_bench import card  # noqa: E402
import canny_golden as cg  # noqa: E402

HOST_SIZES = ((512, 512), (512, 768), (1024, 1024))
DEVICE_BATCHES = (1, 16, 128)
LOW, HIGH = 100, 200


def host_ms(fn, iters, repeats):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        ts.append((time.perf_counter() - t0) * 1e3 / iters)
    return ts


def device_ms(fn, iters, repeats):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / iters)
    return ts


def profile(det, iters):
    from torch.profiler import ProfilerActivity, profile as tprofile
    x = torch.from_numpy(np.stack([cg.image("textured", 512, 512, tag=f".bench{i}") for i in range(16)])).cuda()
    det.detect(x, LOW, HIGH)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            det.detect(x, LOW, HIGH)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        if "canny" in ev.key:
            per[ev.key] = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1e3 / iters
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from ctrlora_b200.annotator.canny import CannyDetector
    det = CannyDetector()
    c = card()
    print(f"card: {c['name']}, power limit {c['power_limit']}; cv2 {cv2.__version__}, {cv2.getNumThreads()} threads")
    res = {"card": c, "cv2_threads": cv2.getNumThreads()}
    if args.profile:
        res["profile_ms_16x512"] = profile(det, args.iters)
        for k, v in res["profile_ms_16x512"].items():
            print(f"  {k}: {v:.4f} ms per detect")
    else:
        def put(name, ts):
            res[name] = statistics.median(ts)
            res[name + "_spread"] = [min(ts), max(ts)]
            print(f"{name:32s} {res[name]:8.3f} ms  ({min(ts):.3f} .. {max(ts):.3f})")

        threads = cv2.getNumThreads()
        for h, w in HOST_SIZES:
            img = cg.image("textured", h, w, tag=".bench")
            assert np.array_equal(det(img, LOW, HIGH), cv2.Canny(img, LOW, HIGH))
            put(f"call_{h}x{w}", host_ms(lambda: det(img, LOW, HIGH), args.iters, args.repeats))
            put(f"cv2_{h}x{w}", host_ms(lambda: cv2.Canny(img, LOW, HIGH), args.iters, args.repeats))
            cv2.setNumThreads(1)
            put(f"cv2_1thread_{h}x{w}", host_ms(lambda: cv2.Canny(img, LOW, HIGH), args.iters, args.repeats))
            cv2.setNumThreads(threads)
        for b in DEVICE_BATCHES:
            x = torch.from_numpy(np.stack([cg.image("textured", 512, 512, tag=f".bench{i}") for i in range(b)])).cuda()
            put(f"detect_{b}x512", device_ms(lambda: det.detect(x, LOW, HIGH), args.iters, args.repeats))
            res[f"detect_{b}x512_per_image"] = res[f"detect_{b}x512"] / b
        x = torch.from_numpy(cg.spiral()).cuda()[None]
        put("detect_spiral_512", device_ms(lambda: det.detect(x, LOW, HIGH), args.iters, args.repeats))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
