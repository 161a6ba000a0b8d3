#!/usr/bin/env python
"""HED annotator timing on one GPU: ControlNetHED_Apache2.forward (synthetic weights) and the whole detector at
1 x 512^2, 1 x 1024^2 and 16 x 512^2, against the same network in torch eager (its nn modules, as the reference's
forward runs them) with fp32 weights and under fp16 autocast, and the reference's host post-process
(tests/hed_golden.py's host_post); plus the kernel launches of one forward and the time of its GEMMs.

    python tools/hed_bench.py [--iters 20] [--out FILE]

Times come from CUDA events around `iters` back-to-back calls after warm-up (host launch overhead included, as a
caller sees it); "graph ms" replays the same forward from a CUDA graph, which removes the host dispatch; "GEMM ms" is
ops.profile_gemm's summed per-launch device time of the forward's GEMMs.  "detector" is HEDdetector.__call__ from a
uint8 HWC host image to the uint8 host map (batch 1), or detect() over the batch of 16 with the maps copied to the host;
"eager detector" is the eager fp32 forward followed by the reference's post-process on the host, per image.  torch's
default lets cuDNN run fp32 convs in TF32 (torch.backends.cudnn.allow_tf32), which is how the reference's detector runs;
"eager fp32 (TF32)" is timed that way and "eager fp32 (strict)" with TF32 off.  Prints the card's name and power limit
read in the same run, and one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.image_encoder_bench import graphed_ms  # noqa: E402
from tools.text_encoder_bench import card, timed_ms  # noqa: E402

CASES = ((1, 512), (1, 1024), (16, 512))


def eager_forward(net, x):
    """the reference ControlNetHED_Apache2.__call__ over net's own nn modules"""
    h = x - net.norm
    out = []
    for i, blk in enumerate(net.blocks()):
        if i:
            h = F.max_pool2d(h, kernel_size=(2, 2), stride=(2, 2))
        for conv in blk.convs:
            h = F.relu(conv(h))
        out.append(blk.projection(h))
    return out


def host_ms(fn, iters):
    """wall time per call of a function that ends on the host (its own device-to-host copy synchronises)"""
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
        raise SystemExit("hed_bench needs a CUDA device")
    import hed_golden as hg
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.hed import ControlNetHED_Apache2, HEDdetector

    net = ControlNetHED_Apache2()
    net.load_state_dict(hg.weights({k: tuple(v.shape) for k, v in net.state_dict().items()}))
    net = net.cuda()
    det = HEDdetector.__new__(HEDdetector)
    det.netNetwork, det.device = net, "cuda"
    res = {"card": card(), "cases": {}}
    for b, s in CASES:
        imgs = [hg.image((s, s), tag=f".bench{i}") for i in range(b)]
        x = torch.from_numpy(np.stack(imgs)).float().permute(0, 3, 1, 2).contiguous().cuda()
        r = {"ms": timed_ms(lambda: net(x), a.iters), "graph_ms": graphed_ms(lambda: net(x), a.iters),
             "launches": ops.count_launches(lambda: net.detect(x))}
        g = ops.profile_gemm(lambda: net(x))
        r["gemm_ms"], r["gemm_tflops"], r["gflop"] = g["ms"], g["flops"] / g["ms"] / 1e9, g["flops"] / 1e9
        if b == 1:
            r["detector_ms"] = host_ms(lambda: det(imgs[0]), a.iters)
        else:
            r["detector_ms"] = host_ms(lambda: net.detect(x)[1].cpu(), a.iters)
        with torch.no_grad():
            r["cudnn_allow_tf32"] = torch.backends.cudnn.allow_tf32
            r["eager_fp32_ms"] = timed_ms(lambda: eager_forward(net, x), a.iters)
            torch.backends.cudnn.allow_tf32 = False
            r["eager_fp32_strict_ms"] = timed_ms(lambda: eager_forward(net, x), a.iters)
            ref = eager_forward(net, x)
            torch.backends.cudnn.allow_tf32 = r["cudnn_allow_tf32"]
            with torch.autocast("cuda", dtype=torch.float16):
                r["eager_fp16_autocast_ms"] = timed_ms(lambda: eager_forward(net, x), a.iters)
            r["eager_detector_ms"] = host_ms(
                lambda: [hg.host_post([e[0, 0].cpu().numpy() for e in eager_forward(net, x[i:i + 1])])
                         for i in range(b)], max(1, a.iters // 4))
        r["rel_err_vs_eager_fp32_strict"] = [((o - e).norm() / e.norm()).item() for o, e in zip(net(x), ref)]
        res["cases"][f"{b}x{s}"] = r
        del x, ref
        torch.cuda.empty_cache()

    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit']}")
    for k, r in res["cases"].items():
        print(f"{k}^2: forward {r['ms']:.3f} ms (graph replay {r['graph_ms']:.3f} ms, detect {r['launches']} launches, "
              f"GEMMs {r['gemm_ms']:.3f} ms for {r['gflop']:.0f} GFLOP at {r['gemm_tflops']:.0f} TFLOP/s); detector "
              f"{r['detector_ms']:.3f} ms; torch eager fp32 (TF32 {r['cudnn_allow_tf32']}) {r['eager_fp32_ms']:.3f} ms, "
              f"fp32 (strict) {r['eager_fp32_strict_ms']:.3f} ms, fp16 autocast "
              f"{r['eager_fp16_autocast_ms']:.3f} ms, eager fp32 + host post-process {r['eager_detector_ms']:.3f} ms; "
              f"side maps rel err vs strict eager fp32 " + ", ".join(f"{e:.1e}" for e in r["rel_err_vs_eager_fp32_strict"]))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
