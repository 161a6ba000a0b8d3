#!/usr/bin/env python
"""M-LSD line annotator timing on one GPU (synthetic weights of tests/mlsd_golden.py):

- MobileV2_MLSD_Large.forward at 1 x 512^2, 1 x 512 x 768 and 16 x 512^2, eager and replayed from a CUDA graph;
- MLSDdetector.__call__ on a 512 x 768 image (host input, the forward, the device decode, the copy back, the draw);
- ops.mlsd_decode alone against torch's sigmoid + max_pool2d + topk on the same 512 x 768 head map;
- the same forwards in plain torch (`torch_forward` below, written over the same nn parameters, NCHW, BatchNorm
  unfolded) in fp32 with TF32 off and on, and under fp16 autocast.

    python tools/mlsd_bench.py [--iters 10] [--repeats 5] [--out FILE]

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

FORWARDS = ((1, 512, 512), (1, 512, 768), (16, 512, 512))
DETECTOR_SIZE = (512, 768)
REPEATS = 5


def _cbn(seq, x, stride=1, padding=None, act=F.relu):
    """seq[0] (conv) and seq[1] (eval BatchNorm), then act"""
    c, bn = seq[0], seq[1]
    pad = c.padding if padding is None else padding
    y = F.conv2d(x, c.weight, c.bias, stride=stride, padding=pad, dilation=c.dilation, groups=c.groups)
    y = F.batch_norm(y, bn.running_mean, bn.running_var, bn.weight, bn.bias, False, 0.0, bn.eps)
    return act(y) if act is not None else y


def _relu6(x):
    return F.hardtanh(x, 0.0, 6.0)


def _conv_bn_relu6(seq, x, stride):
    """ConvBNReLU: stride 2 pads (0, 1, 0, 1) and convolves without padding (TFLite), stride 1 pads k // 2"""
    if stride == 2:
        return _cbn(seq, F.pad(x, (0, 1, 0, 1)), stride=2, padding=0, act=_relu6)
    k = seq[0].kernel_size[0]
    return _cbn(seq, x, padding=k // 2, act=_relu6)


def torch_forward(net, x, stages=False):
    """MobileV2_MLSD_Large's forward in plain torch over the net's own parameters (reference:
    models/mbv2_mlsd_large.py), fp32 [B, 4, H, W] -> [B, 9, H / 2, W / 2] (and c1 .. c5 with stages)"""
    f = net.backbone.features
    y = _conv_bn_relu6(f[0], x, 2)
    feats = []
    for i in range(1, 14):
        blk = f[i]
        layers = list(blk.conv)
        t = y
        if len(layers) == 4:
            t = _conv_bn_relu6(layers[0], t, 1)
        t = _conv_bn_relu6(layers[-3], t, blk.stride)
        t = _cbn([layers[-2], layers[-1]], t, act=None)
        y = y + t if blk.use_res_connect else t
        if i in (1, 3, 6, 10, 13):
            feats.append(y)
    c1, c2, c3, c4, c5 = feats

    def block_a(blk, a, b):
        b = _cbn(blk.conv1, b)
        a = _cbn(blk.conv2, a)
        if blk.upscale:
            b = F.interpolate(b, scale_factor=2.0, mode="bilinear", align_corners=True)
        return torch.cat((a, b), 1)

    def block_b(blk, x):
        return _cbn(blk.conv2, _cbn(blk.conv1, x) + x)

    y = block_b(net.block16, block_a(net.block15, c4, c5))
    y = block_b(net.block18, block_a(net.block17, c3, y))
    y = block_b(net.block20, block_a(net.block19, c2, y))
    y = block_b(net.block22, block_a(net.block21, c1, y))
    c = net.block23
    y = F.conv2d(_cbn(c.conv2, _cbn(c.conv1, y)), c.conv3.weight, c.conv3.bias)[:, 7:]
    return (y, feats) if stages else y


def torch_decode(tp):
    """the reference's decode on an NCHW [1, 9, h, w] map: sigmoid, the 3 x 3 peak mask, topk 200"""
    heat = torch.sigmoid(tp[:, 0])
    keep = (F.max_pool2d(heat, 3, stride=1, padding=1) == heat).float()
    return torch.topk((heat * keep).reshape(-1), 200)


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
        ref = torch_forward(net, x)
        ours = net(x)
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    res["rel_err_vs_torch_fp32"] = ((ours - ref).norm() / ref.norm()).item()
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
        raise SystemExit("mlsd_bench needs a CUDA device")
    import mlsd_golden as mg
    from ctrlora_b200 import ops
    from ctrlora_b200.annotator.mlsd import CENTER, DISP, MLSDdetector, MobileV2_MLSD_Large, network_input

    net = MobileV2_MLSD_Large()
    bn = [n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
    sd = mg.weights({k: tuple(v.shape) for k, v in net.state_dict().items()}, bn)
    with tempfile.TemporaryDirectory() as d:
        torch.save(sd, os.path.join(d, "mlsd_large_512_fp32.pth"))
        det = MLSDdetector(ckpt_dir=d)
    net = det.model
    res = {"card": card(), "forward": {}, "detector": {}, "decode": {}}
    for b, h, w in FORWARDS:
        x = torch.cat([network_input(mg.image((h, w), tag=str(i))) for i in range(b)]).cuda()
        with torch.no_grad():
            net(x)
        r = {"launches": ops.count_launches(lambda: net(x))}
        med(r, "ms", lambda: timed_ms(lambda: net(x), a.iters))
        med(r, "graph_ms", lambda: graphed_ms(lambda: net(x), a.iters))
        r.update(torch_times(net, x, a.iters))
        res["forward"][f"{b}x{h}x{w}"] = r
    img = mg.image(DETECTOR_SIZE)

    def call_ms():
        for _ in range(3):
            det(img, 0.1, 0.1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.iters):
            det(img, 0.1, 0.1)
        return (time.perf_counter() - t0) * 1e3 / a.iters

    r = {}
    med(r, "call_ms", call_ms)
    res["detector"][f"{DETECTOR_SIZE[0]}x{DETECTOR_SIZE[1]}"] = r
    with torch.no_grad():
        tp, _ = net._run(network_input(img).cuda())
        tp_nchw = tp[..., CENTER:].permute(0, 3, 1, 2).contiguous()
    r = {}
    med(r, "ours_ms", lambda: timed_ms(lambda: ops.mlsd_decode(tp, CENTER, DISP), a.iters * 10))
    med(r, "torch_ms", lambda: timed_ms(lambda: torch_decode(tp_nchw), a.iters * 10))
    res["decode"][f"{DETECTOR_SIZE[0] // 2}x{DETECTOR_SIZE[1] // 2}"] = r

    print(f"card: {res['card']['name']}, power limit {res['card']['power_limit']}; medians of {REPEATS} windows")
    for k, r in res["forward"].items():
        print(f"forward {k}: {r['ms']:.2f} ms (graph replay {r['graph_ms']:.2f} ms, {r['launches']} launches); torch "
              f"fp32 {r['torch_fp32_notf32_ms']:.2f} ms, TF32 {r['torch_fp32_tf32_ms']:.2f} ms, fp16 autocast "
              f"{r['torch_fp16_autocast_ms']:.2f} ms; rel err vs torch fp32 {r['rel_err_vs_torch_fp32']:.2e}")
    for k, r in res["detector"].items():
        print(f"detector {k}: call {r['call_ms']:.2f} ms")
    for k, r in res["decode"].items():
        print(f"decode {k}: ours {r['ours_ms']:.3f} ms, torch sigmoid + max_pool2d + topk {r['torch_ms']:.3f} ms")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
