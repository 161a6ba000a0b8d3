#!/usr/bin/env python
"""Anime line-art annotator timing on one GPU: UnetGenerator(3, 1, 8).forward (synthetic weights) at 1 x 512^2,
1 x 1024^2 and 16 x 512^2, against the same network in torch eager (its nn modules, as the reference's forward runs
them) in fp32 with TF32 off and on and under fp16 autocast, on the same weights and inputs; plus the kernel launches
of one call and the time of its GEMMs.

    python tools/lineart_anime_bench.py [--iters 20] [--out FILE]

Times come from CUDA events around `iters` back-to-back calls after warm-up (host launch overhead included, as a
caller sees it); "graph ms" replays the same forward from a CUDA graph, which removes the host dispatch; "GEMM ms" is
ops.replay_gemms' device time of the forward's GEMM launches alone.  Prints the card's name and power limit read in
the same run, and one JSON line."""
import argparse
import functools
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.image_encoder_bench import graphed_ms  # noqa: E402
from tools.text_encoder_bench import card, timed_ms  # noqa: E402

CASES = ((1, 512), (1, 1024), (16, 512))


def eager_block(blk, x):
    """the reference UnetSkipConnectionBlock.forward over blk's own nn modules (its LeakyReLU runs in place on x)"""
    from ctrlora_b200.annotator.lineart_anime import UnetSkipConnectionBlock
    y = x
    for m in blk.model:
        y = eager_block(m, y) if isinstance(m, UnetSkipConnectionBlock) else m(y)
    return y if blk.outermost else torch.cat([x, y], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lineart_anime_bench needs a CUDA device")
    import lineart_anime_golden as lg
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.lineart_anime import UnetGenerator

    norm = functools.partial(nn.InstanceNorm2d, affine=False, track_running_stats=False)
    gen = UnetGenerator(3, 1, lg.NUM_DOWNS, 64, norm_layer=norm)
    gen.load_state_dict(lg.weights({k: tuple(v.shape) for k, v in gen.state_dict().items()}))
    gen = gen.cuda()
    res = {"card": card(), "cases": {}}
    old_tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    for b, s in CASES:
        x = torch.rand(b, 3, s, s, device="cuda") * 2 - 1
        r = {"ms": timed_ms(lambda: gen(x), a.iters), "graph_ms": graphed_ms(lambda: gen(x), a.iters),
             "launches": ops.count_launches(lambda: gen(x))}
        g = ops.replay_gemms(lambda: gen(x), reps=a.iters)
        r["gemm_ms"], r["gemm_tflops"] = g["ms"], g["flops"] / g["ms"] / 1e9
        with torch.no_grad():
            for tf32 in (False, True):
                torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
                r[f"eager_fp32_{'tf32' if tf32 else 'notf32'}_ms"] = timed_ms(lambda: eager_block(gen.model, x),
                                                                              a.iters)
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
            with torch.autocast("cuda", dtype=torch.float16):
                r["eager_fp16_autocast_ms"] = timed_ms(lambda: eager_block(gen.model, x), a.iters)
            ref = eager_block(gen.model, x)
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old_tf32
        r["rel_err_vs_eager_fp32"] = ((gen(x) - ref).norm() / ref.norm()).item()
        res["cases"][f"{b}x{s}"] = r
        del x, ref
        torch.cuda.empty_cache()

    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit']}")
    for k, r in res["cases"].items():
        print(f"{k}^2: forward {r['ms']:.3f} ms (graph replay {r['graph_ms']:.3f} ms, {r['launches']} launches, GEMMs "
              f"{r['gemm_ms']:.3f} ms at {r['gemm_tflops']:.0f} TFLOP/s); torch eager fp32 {r['eager_fp32_notf32_ms']:.3f} "
              f"ms (TF32 {r['eager_fp32_tf32_ms']:.3f} ms), fp16 autocast {r['eager_fp16_autocast_ms']:.3f} ms; rel err vs "
              f"eager fp32 {r['rel_err_vs_eager_fp32']:.2e}")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
