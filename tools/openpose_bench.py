#!/usr/bin/env python
"""OpenPose body annotator timing on one GPU: bodypose_model.forward (synthetic weights) at the network inputs of
1 x 512^2, 1 x 1024^2 and 16 x 512^2 images, against the same network in torch eager (its nn modules, as the
reference's forward runs them) in fp32 with TF32 on and off and under fp16 autocast; and Body.__call__ (image in,
candidate and subset out, per image) against the eager fp32 forward followed by the reference's host post-process
(tests/openpose_golden.py's host_postprocess: numpy / cv2 / scipy, one channel at a time).

    python tools/openpose_bench.py [--iters 20] [--out FILE]

Times come from CUDA events around `iters` back-to-back forwards after warm-up (host launch overhead included), or a
host clock around calls that end on the host.  Body scales every image to height 184, so each case's network input is
184 x 184.  With synthetic weights the heatmaps are noisy and hold hundreds of peaks per image, so both detector
columns include host matching over many candidate pairs.  Prints the card's name and power limit read in the same run,
and one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.text_encoder_bench import card, timed_ms  # noqa: E402

CASES = ((1, 512), (1, 1024), (16, 512))


def eager_forward(net, x):
    """the reference bodypose_model.forward over net's own nn modules"""
    out1 = net.model0(x)
    l1, l2 = net.model1_1(out1), net.model1_2(out1)
    for s in range(2, 7):
        cat = torch.cat([l1, l2, out1], 1)
        l1, l2 = net.branch(s, 1)(cat), net.branch(s, 2)(cat)
    return l1, l2


def host_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("openpose_bench needs a CUDA device")
    import openpose_golden as og
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.openpose import Body, PostProcess, bodypose_model, network_input

    net = bodypose_model()
    net.load_state_dict(og.weights({k: tuple(v.shape) for k, v in net.state_dict().items()}))
    net = net.cuda()
    body = Body.__new__(Body)
    body.model, body.post = net, PostProcess()
    res = {"card": card(), "cases": {}}
    for b, s in CASES:
        imgs = [og.image((s, s), tag=f".bench{i}") for i in range(b)]
        x = torch.from_numpy(np.concatenate([network_input(im) for im in imgs])).cuda()
        r = {"input": list(x.shape), "ms": timed_ms(lambda: net(x), a.iters),
             "launches": ops.count_launches(lambda: net(x))}
        g = ops.profile_gemm(lambda: net(x))
        r["gemm_ms"], r["gflop"] = g["ms"], g["flops"] / 1e9
        r["detector_ms"] = host_ms(lambda: [body(im) for im in imgs], max(1, a.iters // b))
        with torch.no_grad():
            r["cudnn_allow_tf32"] = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = True
            r["eager_fp32_tf32_ms"] = timed_ms(lambda: eager_forward(net, x), a.iters)
            torch.backends.cudnn.allow_tf32 = False
            r["eager_fp32_strict_ms"] = timed_ms(lambda: eager_forward(net, x), a.iters)
            ref = eager_forward(net, x)
            torch.backends.cudnn.allow_tf32 = r["cudnn_allow_tf32"]
            with torch.autocast("cuda", dtype=torch.float16):
                r["eager_fp16_autocast_ms"] = timed_ms(lambda: eager_forward(net, x), a.iters)

            def eager_detector():
                for i, im in enumerate(imgs):
                    paf, heat = eager_forward(net, x[i:i + 1])
                    og.host_postprocess(paf[0].cpu().numpy(), heat[0].cpu().numpy(), s, s)
            r["eager_detector_ms"] = host_ms(eager_detector, max(1, a.iters // (4 * b)))
        r["rel_err_vs_eager_fp32_strict"] = [((o - e).norm() / e.norm()).item() for o, e in zip(net(x), ref)]
        res["cases"][f"{b}x{s}"] = r
        del x, ref
        torch.cuda.empty_cache()

    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit']}")
    for k, r in res["cases"].items():
        print(f"{k}^2 (network input {r['input']}): forward {r['ms']:.3f} ms ({r['launches']} launches, GEMMs "
              f"{r['gemm_ms']:.3f} ms for {r['gflop']:.0f} GFLOP); torch eager fp32 (TF32) {r['eager_fp32_tf32_ms']:.3f} "
              f"ms, fp32 (strict) {r['eager_fp32_strict_ms']:.3f} ms, fp16 autocast {r['eager_fp16_autocast_ms']:.3f} "
              f"ms; Body.__call__ {r['detector_ms']:.2f} ms vs eager fp32 + host post-process "
              f"{r['eager_detector_ms']:.2f} ms (all images); PAF / heatmap rel err vs strict eager fp32 " +
              ", ".join(f"{e:.1e}" for e in r["rel_err_vs_eager_fp32_strict"]))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
