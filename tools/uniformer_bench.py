#!/usr/bin/env python
"""UniFormer segmentation annotator timing on one GPU (synthetic weights of tests/uniformer_golden.py):

- UniformerSegmentor.forward at 1 x 512^2, 1 x 512 x 853 and 16 x 512^2, eager and replayed from a CUDA graph;
- UniformerDetector.__call__ on a 384 x 640 image (host resize, the forward, the device output and the copy back);
- the same forwards in plain torch (`torch_forward` below, written over the same nn parameters, NCHW, with the
  Normalize the network folds in applied first) in fp32 with TF32 off and on, and under fp16 autocast;
- with --profile, a torch.profiler table of the kernels of one 16 x 512^2 forward (a run of its own).

    python tools/uniformer_bench.py [--iters 10] [--repeats 5] [--profile] [--out FILE]

Times come from CUDA events around `iters` back-to-back calls after warm-up; every figure is the median of `repeats`
such windows, and the JSON line also holds each figure's min and max ("<name>_spread").  Prints the card's name and
power limit read in the same run, and one JSON line."""
import argparse
import json
import os
import sys
import tempfile
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools.image_encoder_bench import graphed_ms  # noqa: E402
from tools.text_encoder_bench import card, timed_ms  # noqa: E402

FORWARDS = ((1, 512, 512), (1, 512, 853), (16, 512, 512))
DETECTOR_SIZE = (384, 640)
REPEATS = 5


def _conv(m, x, **kw):
    return F.conv2d(x, m.weight, m.bias, stride=m.stride, padding=m.padding, groups=m.groups, **kw)


def _bn(bn, x):
    return F.batch_norm(x, bn.running_mean, bn.running_var, bn.weight, bn.bias, False, 0.0, bn.eps)


def _ln_c(ln, x):
    """LayerNorm over the channels of an NCHW tensor"""
    return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), ln.weight, ln.bias, ln.eps).permute(0, 3, 1, 2)


def _cm(cm, x):
    return F.relu(_bn(cm.bn, _conv(cm.conv, x)))


def _up(x, size):
    return F.interpolate(x, size=size, mode="bilinear", align_corners=False)


def torch_forward(net, x):
    """UniformerSegmentor's forward in plain torch over the net's own parameters (reference: mmseg's UniFormer
    forward_features with CBlock / SABlock, and UPerHead.forward), from the un-normalised RGB input -> 1/4 logits NCHW"""
    from ctrlora_b200.annotator.uniformer import MEAN, STD
    bb, dh = net.backbone, net.decode_head
    mean = torch.tensor(MEAN, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(STD, device=x.device).view(1, 3, 1, 1)
    x = (x.flip(1) - mean) / std
    feats = []
    for i in (1, 2, 3, 4):
        pe = getattr(bb, f"patch_embed{i}")
        x = _ln_c(pe.norm, _conv(pe.proj, x))
        for blk in getattr(bb, f"blocks{i}"):
            x = x + _conv(blk.pos_embed, x)
            if i <= 2:
                x = x + _conv(blk.conv2, _conv(blk.attn, _conv(blk.conv1, _bn(blk.norm1, x))))
                x = x + _conv(blk.mlp.fc2, F.gelu(_conv(blk.mlp.fc1, _bn(blk.norm2, x))))
            else:
                b, c, h, w = x.shape
                t = x.flatten(2).transpose(1, 2)
                y = F.layer_norm(t, (c,), blk.norm1.weight, blk.norm1.bias, blk.norm1.eps)
                qkv = F.linear(y, blk.attn.qkv.weight, blk.attn.qkv.bias).view(b, -1, 3, c // 64, 64).permute(2, 0, 3, 1, 4)
                a = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2]).transpose(1, 2).reshape(b, -1, c)
                t = t + F.linear(a, blk.attn.proj.weight, blk.attn.proj.bias)
                y = F.layer_norm(t, (c,), blk.norm2.weight, blk.norm2.bias, blk.norm2.eps)
                t = t + F.linear(F.gelu(F.linear(y, blk.mlp.fc1.weight, blk.mlp.fc1.bias)), blk.mlp.fc2.weight,
                                 blk.mlp.fc2.bias)
                x = t.transpose(1, 2).reshape(b, c, h, w)
        feats.append(_ln_c(getattr(bb, f"norm{i}"), x))
    f4 = feats[3]
    psp = [f4] + [_up(_cm(m[1], F.adaptive_avg_pool2d(f4, m[0].output_size)), f4.shape[2:]) for m in dh.psp_modules]
    lats = [_cm(dh.lateral_convs[i], feats[i]) for i in range(3)] + [_cm(dh.bottleneck, torch.cat(psp, 1))]
    for i in (3, 2, 1):
        lats[i - 1] = lats[i - 1] + _up(lats[i], lats[i - 1].shape[2:])
    outs = [_cm(dh.fpn_convs[i], lats[i]) for i in range(3)] + [lats[3]]
    outs = [outs[0]] + [_up(o, outs[0].shape[2:]) for o in outs[1:]]
    return _conv(dh.conv_seg, _cm(dh.fpn_bottleneck, torch.cat(outs, 1)))


def med(res, key, fn):
    """res[key] = the median of REPEATS timings fn(), res[key + "_spread"] = [min, max]"""
    ts = sorted(fn() for _ in range(REPEATS))
    res[key], res[key + "_spread"] = ts[len(ts) // 2], [ts[0], ts[-1]]


def torch_times(net, x, iters):
    res = {}
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    with torch.no_grad():
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
            med(res, f"torch_fp32_{'tf32' if tf32 else 'notf32'}_ms", lambda: timed_ms(lambda: torch_forward(net, x), iters))
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        with torch.autocast("cuda", dtype=torch.float16):
            med(res, "torch_fp16_autocast_ms", lambda: timed_ms(lambda: torch_forward(net, x), iters))
        ref = torch_forward(net, x).permute(0, 2, 3, 1)
        ours = net(x)
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    res["rel_err_vs_torch_fp32"] = ((ours - ref).norm() / ref.norm()).item()
    return res


def profile(net, x, out_dir):
    from torch.profiler import ProfilerActivity, profile as prof
    with torch.no_grad():
        net(x)
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            net(x)
            torch.cuda.synchronize()
    table = p.key_averages().table(sort_by="cuda_time_total", row_limit=25)
    print(table)
    if out_dir:
        with open(os.path.join(out_dir, "uniformer_profile.txt"), "w") as f:
            f.write(table)


def main():
    global REPEATS
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=REPEATS)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    REPEATS = a.repeats
    if not torch.cuda.is_available():
        raise SystemExit("uniformer_bench needs a CUDA device")
    import uniformer_golden as ug
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.uniformer import UniformerDetector, UniformerSegmentor, network_input

    net = UniformerSegmentor()
    bn = [n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
    sd = ug.weights({k: tuple(v.shape) for k, v in net.state_dict().items()}, bn)
    palette = torch.randint(0, 256, (150, 3), generator=torch.Generator().manual_seed(0), dtype=torch.uint8)
    with tempfile.TemporaryDirectory() as d:
        torch.save({"state_dict": sd, "meta": {"PALETTE": palette.tolist()}}, os.path.join(d, "upernet_global_small.pth"))
        det = UniformerDetector(ckpt_dir=d)
    net = det.model
    res = {"card": card(), "forward": {}, "detector": {}}
    for b, h, w in FORWARDS:
        x = torch.cat([network_input(ug.image((h, w), tag=str(i))) for i in range(b)]).cuda()
        with torch.no_grad():
            net(x)
        r = {"launches": ops.count_launches(lambda: net(x))}
        med(r, "ms", lambda: timed_ms(lambda: net(x), a.iters))
        med(r, "graph_ms", lambda: graphed_ms(lambda: net(x), a.iters))
        r.update(torch_times(net, x, a.iters))
        res["forward"][f"{b}x{h}x{w}"] = r
    img = ug.image(DETECTOR_SIZE)

    def call_ms():
        for _ in range(3):
            det(img)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.iters):
            det(img)
        return (time.perf_counter() - t0) * 1e3 / a.iters

    r = {}
    med(r, "call_ms", call_ms)
    res["detector"][f"{DETECTOR_SIZE[0]}x{DETECTOR_SIZE[1]}"] = r

    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit']}; medians of {REPEATS} windows")
    for k, r in res["forward"].items():
        print(f"forward {k}: {r['ms']:.2f} ms (graph replay {r['graph_ms']:.2f} ms, {r['launches']} launches); torch "
              f"fp32 {r['torch_fp32_notf32_ms']:.2f} ms, TF32 {r['torch_fp32_tf32_ms']:.2f} ms, fp16 autocast "
              f"{r['torch_fp16_autocast_ms']:.2f} ms; rel err vs torch fp32 {r['rel_err_vs_torch_fp32']:.2e}")
    for k, r in res["detector"].items():
        print(f"detector {k}: call {r['call_ms']:.2f} ms")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if a.profile:
        b, h, w = FORWARDS[-1]
        x = torch.cat([network_input(ug.image((h, w), tag=str(i))) for i in range(b)]).cuda()
        profile(net, x, os.path.dirname(a.out) if a.out else None)


if __name__ == "__main__":
    main()
