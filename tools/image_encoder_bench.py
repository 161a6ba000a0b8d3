#!/usr/bin/env python
"""IP-Adapter image-encoder timing on one GPU: CLIPVisionModelWithProjection(pixel_values).image_embeds (CLIP ViT-H/14,
synthetic weights, 224 x 224) at batch 1 and 4 against transformers' CLIPVisionModelWithProjection in eager mode, fp16
(the reference app's setting) and fp32, on the same weights; the kernel launches of one call; and the attention kernel on
its own at the encoder's shape (16 heads, 257 x 257 tokens, d_head 80).

    python tools/image_encoder_bench.py [--iters 30] [--out FILE]

Every time comes from CUDA events around `iters` back-to-back calls after warm-up (host launch overhead included, as a
caller sees it); "device ms" replays the same call from a CUDA graph, which removes the host dispatch, so the two
together say whether a call is bound by the host.  Prints the card's name and power limit read in the same run, and one
JSON line."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.text_encoder_bench import card, timed_ms  # noqa: E402


def graphed_ms(fn, iters):
    """device time of fn replayed from one CUDA graph (no host dispatch)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    ms = timed_ms(graph.replay, iters)
    del graph
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_encoder_bench needs a CUDA device")
    import clip_vision_golden as cvg
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection as HFVision
    from ctrlora_b200 import ops
    from ctrlora_b200.image_encoder import CLIPVisionModelWithProjection

    enc = CLIPVisionModelWithProjection()  # built-in ViT-H/14
    sd = cvg.weights(enc, "vision")
    enc.load_state_dict(sd)
    enc = enc.cuda()
    hf32 = HFVision(CLIPVisionConfig(**cvg.VISION["sd15"], attn_implementation="eager")).eval()
    hf32.load_state_dict(sd)
    hf32 = hf32.cuda()
    hf16 = HFVision(CLIPVisionConfig(**cvg.VISION["sd15"], attn_implementation="eager")).eval()
    hf16.load_state_dict(sd)
    hf16 = hf16.half().cuda()
    del sd

    res = {"card": card(), "image_embeds_ms": {}, "image_embeds_device_ms": {}, "launches": {},
           "transformers_fp16_ms": {}, "transformers_fp32_ms": {}, "attention_us": {}}
    for b in (1, 4):
        px = cvg.pixels(b).cuda()
        px16 = px.half()
        res["image_embeds_ms"][b] = timed_ms(lambda: enc(px16), a.iters)
        res["image_embeds_device_ms"][b] = graphed_ms(lambda: enc(px16), a.iters)
        res["launches"][b] = ops.count_launches(lambda: enc(px16))
        with torch.no_grad():
            res["transformers_fp16_ms"][b] = timed_ms(lambda: hf16(px16), a.iters)
            res["transformers_fp32_ms"][b] = timed_ms(lambda: hf32(px), a.iters)
        q, k = (torch.randn((b * 257, 1280), device="cuda").half() for _ in range(2))
        vt = torch.randn((b, 16, 80, 264), device="cuda").half()
        out = torch.empty_like(q)
        res["attention_us"][b] = 1e3 * timed_ms(lambda: ops.attention(q, k, vt, b, 16, 257, 257, 80, out=out), 20 * a.iters)

    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit']}")
    for b in (1, 4):
        print(f"batch {b}: image_embeds {res['image_embeds_ms'][b]:.3f} ms (graph replay {res['image_embeds_device_ms'][b]:.3f} "
              f"ms, {res['launches'][b]} launches), transformers eager fp16 {res['transformers_fp16_ms'][b]:.3f} ms, fp32 "
              f"{res['transformers_fp32_ms'][b]:.3f} ms; attention 257x257 d80 {res['attention_us'][b]:.1f} us")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
