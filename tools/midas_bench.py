#!/usr/bin/env python
"""MiDaS DPT-Large annotator timing on one GPU (synthetic weights of tests/midas_golden.py):

- MidasDetector.__call__ at 384^2, 512^2 and 512 x 768, eager (host conversion, the forward, the device post-process
  and the copy of the two uint8 maps) and the forward + post-process replayed from a CUDA graph;
- DPTDepthModel.forward at batch 8 x 384^2;
- the same forwards in plain torch (`torch_forward` below, written over the same nn parameters) in fp32 with TF32 off
  and on, and under fp16 autocast;
- the kernel launches of one call.

    python tools/midas_bench.py [--iters 10] [--repeats 5] [--out FILE]

Times come from CUDA events around `iters` back-to-back calls after warm-up; every figure is the median of `repeats`
such windows, and the JSON line also holds each figure's min and max over them ("<name>_spread").  Prints the card's
name and power limit read in the same run, and one JSON line."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.image_encoder_bench import graphed_ms  # noqa: E402
from tools.text_encoder_bench import card, timed_ms  # noqa: E402

DETECTOR_SIZES = ((384, 384), (512, 512), (512, 768))
BATCH = (8, 384, 384)


def _conv(m, x, **kw):
    return F.conv2d(x, m.weight, m.bias, stride=m.stride, padding=m.padding, **kw)


def torch_forward(model, x):
    """DPTDepthModel's forward in plain torch over the model's own parameters (reference: midas/vit.py forward_flex and
    forward_vit, blocks.py FeatureFusionBlock_custom, dpt_depth.py head)"""
    vit, pre, sc = model.pretrained.model, model.pretrained, model.scratch
    b, _, h, w = x.shape
    gh, gw = h // 16, w // 16
    t = _conv(vit.patch_embed.proj, x).flatten(2).transpose(1, 2)
    t = torch.cat([vit.cls_token.expand(b, -1, -1).to(t.dtype), t], 1) + model.pos_table(gh, gw)[None].to(t.dtype)
    hooks = []
    for i, blk in enumerate(vit.blocks[:24]):
        y = F.layer_norm(t, (t.shape[-1],), blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
        qkv = F.linear(y, blk.attn.qkv.weight, blk.attn.qkv.bias).view(b, -1, 3, 16, 64).permute(2, 0, 3, 1, 4)
        a = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2]).transpose(1, 2).reshape(b, -1, 1024)
        t = t + F.linear(a, blk.attn.proj.weight, blk.attn.proj.bias)
        y = F.layer_norm(t, (t.shape[-1],), blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
        t = t + F.linear(F.gelu(F.linear(y, blk.mlp.fc1.weight, blk.mlp.fc1.bias)), blk.mlp.fc2.weight, blk.mlp.fc2.bias)
        if i in (5, 11, 17, 23):
            hooks.append(t)
    layers = []
    for k, t in enumerate(hooks, 1):
        post = getattr(pre, f"act_postprocess{k}")
        lin = post[0].project[0]
        r = F.gelu(F.linear(torch.cat([t[:, 1:], t[:, :1].expand_as(t[:, 1:])], -1), lin.weight, lin.bias))
        r = _conv(post[3], r.transpose(1, 2).reshape(b, -1, gh, gw))
        if k in (1, 2):
            r = F.conv_transpose2d(r, post[4].weight, post[4].bias, stride=post[4].stride)
        elif k == 4:
            r = _conv(post[4], r)
        layers.append(r)
    rn = [_conv(getattr(sc, f"layer{k}_rn"), l) for k, l in enumerate(layers, 1)]

    def rcu(u, x):
        return _conv(u.conv2, F.relu(_conv(u.conv1, F.relu(x)))) + x

    def fuse(blk, x0, x1=None):
        y = x0 if x1 is None else x0 + rcu(blk.resConfUnit1, x1)
        y = F.interpolate(rcu(blk.resConfUnit2, y), scale_factor=2, mode="bilinear", align_corners=True)
        return _conv(blk.out_conv, y)

    p = fuse(sc.refinenet4, rn[3])
    for i in (3, 2, 1):
        p = fuse(getattr(sc, f"refinenet{i}"), p, rn[i - 1])
    oc = sc.output_conv
    y = F.interpolate(_conv(oc[0], p), scale_factor=2, mode="bilinear", align_corners=True)
    return F.relu(_conv(oc[4], F.relu(_conv(oc[2], y))))[:, 0]


REPEATS = 5


def med(res, key, fn):
    """res[key] = the median of REPEATS timings fn(), res[key + "_spread"] = [min, max]"""
    ts = sorted(fn() for _ in range(REPEATS))
    res[key], res[key + "_spread"] = ts[len(ts) // 2], [ts[0], ts[-1]]


def torch_times(model, x, iters):
    res = {}
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    with torch.no_grad():
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
            med(res, f"torch_fp32_{'tf32' if tf32 else 'notf32'}_ms", lambda: timed_ms(lambda: torch_forward(model, x), iters))
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        with torch.autocast("cuda", dtype=torch.float16):
            med(res, "torch_fp16_autocast_ms", lambda: timed_ms(lambda: torch_forward(model, x), iters))
        ref = torch_forward(model, x)
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    res["rel_err_vs_torch_fp32"] = ((model(x) - ref).norm() / ref.norm()).item()
    return res


def main():
    global REPEATS
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=REPEATS)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    REPEATS = a.repeats
    if not torch.cuda.is_available():
        raise SystemExit("midas_bench needs a CUDA device")
    import midas_golden as mg
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.midas import DPTDepthModel, MidasDetector

    shapes = {"model." + k: tuple(v.shape) for k, v in DPTDepthModel().state_dict().items()}
    sd = {k[len("model."):]: v for k, v in mg.weights(shapes).items()}
    res = {"card": card(), "detector": {}, "batch": {}}
    with tempfile.TemporaryDirectory() as d:
        torch.save(sd, os.path.join(d, "dpt_large_384.pt"))
        det = MidasDetector(ckpt_dir=d)
    model = det.model.model
    for h, w in DETECTOR_SIZES:
        img = mg.image((h, w))
        x = mg.image_tensor(img).cuda()

        def forward_maps():
            return ops.midas_maps(model(x), np.pi * 0.2, 0.02)

        def call_ms():
            for _ in range(3):
                det(img)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.iters):
                det(img)
            return (time.perf_counter() - t0) * 1e3 / a.iters

        forward_maps()  # the first call also builds the kernel-layout weights
        r = {"launches": ops.count_launches(forward_maps)}
        med(r, "call_ms", call_ms)
        med(r, "forward_maps_ms", lambda: timed_ms(forward_maps, a.iters))
        med(r, "graph_ms", lambda: graphed_ms(forward_maps, a.iters))
        r.update(torch_times(model, x, a.iters))
        res["detector"][f"{h}x{w}"] = r
    b, h, w = BATCH
    x = torch.cat([mg.image_tensor(mg.image((h, w), tag=str(i))) for i in range(b)]).cuda()
    r = {}
    med(r, "ms", lambda: timed_ms(lambda: model(x), a.iters))
    med(r, "graph_ms", lambda: graphed_ms(lambda: model(x), a.iters))
    r.update(torch_times(model, x, a.iters))
    res["batch"][f"{b}x{h}x{w}"] = r

    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit']}; medians of {REPEATS} windows")
    for k, r in res["detector"].items():
        print(f"detector {k}: call {r['call_ms']:.2f} ms (forward + maps {r['forward_maps_ms']:.2f} ms, graph replay "
              f"{r['graph_ms']:.2f} ms, {r['launches']} launches); torch fp32 {r['torch_fp32_notf32_ms']:.2f} ms, TF32 "
              f"{r['torch_fp32_tf32_ms']:.2f} ms, fp16 autocast {r['torch_fp16_autocast_ms']:.2f} ms; rel err vs torch "
              f"fp32 {r['rel_err_vs_torch_fp32']:.2e}; torch fp32 spread {r['torch_fp32_notf32_ms_spread']}")
    for k, r in res["batch"].items():
        print(f"forward {k}: {r['ms']:.2f} ms (graph replay {r['graph_ms']:.2f} ms); torch fp32 "
              f"{r['torch_fp32_notf32_ms']:.2f} ms, TF32 {r['torch_fp32_tf32_ms']:.2f} ms, fp16 autocast "
              f"{r['torch_fp16_autocast_ms']:.2f} ms; rel err vs torch fp32 {r['rel_err_vs_torch_fp32']:.2e}")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
