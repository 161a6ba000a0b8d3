#!/usr/bin/env python
"""CLIP text-encoder timing on one GPU: FrozenCLIPEmbedder.encode_tokens (CLIP ViT-L/14 text tower, synthetic weights,
77 tokens) at batch 1, 4 and 16 against transformers' CLIPTextModel in eager mode, fp32 and fp16, on the same weights;
and the causal attention kernel on its own at the encoder's shape (12 heads, 77 tokens).

    python tools/text_encoder_bench.py [--iters 50] [--out FILE]

Every time comes from CUDA events around `iters` back-to-back calls after warm-up (host launch overhead included, as a
caller sees it).  Prints the card's name and power limit read in the same run, and one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power}


def timed_ms(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("text_encoder_bench needs a CUDA device")
    import clip_golden
    from transformers import CLIPTextConfig, CLIPTextModel
    from ctrlora_b200 import ops
    from ctrlora_b200.text_encoder import CLIP_L_CONFIG, FrozenCLIPEmbedder

    enc = FrozenCLIPEmbedder()  # built-in CLIP ViT-L/14 architecture
    enc.load_state_dict(clip_golden.embedder_weights(enc))
    enc = enc.cuda()
    hf = CLIPTextModel(CLIPTextConfig(**CLIP_L_CONFIG, attn_implementation="eager")).eval()
    hf.load_state_dict({k[len("transformer."):]: v for k, v in enc.state_dict().items()})
    hf32 = hf.cuda()
    hf16 = CLIPTextModel(CLIPTextConfig(**CLIP_L_CONFIG, attn_implementation="eager")).eval()
    hf16.load_state_dict(hf32.state_dict())
    hf16 = hf16.half().cuda()

    res = {"card": card(), "encode_tokens_ms": {}, "transformers_fp32_ms": {}, "transformers_fp16_ms": {}}
    gen = torch.Generator().manual_seed(0)
    for b in (1, 4, 16):
        ids = torch.randint(0, 49406, (b, 77), generator=gen)
        ids[:, 0], ids[:, -1] = 49406, 49407
        ids_dev = ids.cuda()
        res["encode_tokens_ms"][b] = timed_ms(lambda: enc.encode_tokens(ids_dev), a.iters)
        with torch.no_grad():
            res["transformers_fp32_ms"][b] = timed_ms(lambda: hf32(input_ids=ids_dev), a.iters)
            res["transformers_fp16_ms"][b] = timed_ms(lambda: hf16(input_ids=ids_dev), a.iters)

    res["causal_attention_us"] = {}
    for b in (1, 4, 16):
        q, k = (torch.randn((b * 77, 768), device="cuda").half() for _ in range(2))
        vt = torch.randn((b, 12, 64, 80), device="cuda").half()
        out = torch.empty_like(q)
        res["causal_attention_us"][b] = 1e3 * timed_ms(lambda: ops.causal_attention(q, k, vt, b, 12, 77, out=out), 20 * a.iters)

    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit']}")
    for b in (1, 4, 16):
        print(f"batch {b:2d}: encode_tokens {res['encode_tokens_ms'][b]:.3f} ms, transformers eager fp32 "
              f"{res['transformers_fp32_ms'][b]:.3f} ms, fp16 {res['transformers_fp16_ms'][b]:.3f} ms, causal attention "
              f"{res['causal_attention_us'][b]:.1f} us")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
