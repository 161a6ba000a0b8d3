"""The M-LSD line annotator (annotator/mlsd/__init__.py MLSDdetector: MobileV2_MLSD_Large of
models/mbv2_mlsd_large.py and pred_lines of utils.py) on the sm_90a kernels.

Switching a caller over is an import swap: `from ctrlora_b200.annotator.mlsd import MLSDdetector`.  The modules keep
the reference's tree (`backbone.features.N.conv.*`, `block15` .. `block23`), so `state_dict()` equals the reference
network's and mlsd_large_512_fp32.pth loads with strict=True.  The nn modules hold the parameters only; every eval
BatchNorm is folded into its conv at prep time, and the network runs on fp16 pixel-major activations with fp32
accumulation:

- the stem ConvBNReLU(4, 32, stride 2): a stride-2 tap gather over taps (0..2, 0..2), zero outside (the TFLite padding
  F.pad(x, (0, 1, 0, 1)) followed by a padding-0 conv), from the fp32 NCHW input, then one GEMM with ReLU6;
- each InvertedResidual: the expand 1 x 1 as a GEMM with ReLU6, the depthwise 3 x 3 (stride 2 with the TFLite padding)
  with ReLU6 in one ctrlora_dwconv_act_f16, the project 1 x 1 as a GEMM with the block's residual fused;
- BlockTypeA: both 1 x 1 convs (+ ReLU) write their channel slice of the 128-channel concatenation; the deeper one is
  upsampled (bilinear x 2, align_corners=True) into its slice;
- BlockTypeB: relu(conv1(x)) + x as one 3 x 3 GEMM with the ReLU before the residual, then conv2 + ReLU;
- BlockTypeC: the dilation-5 conv as a 9-tap gather at offsets {-5, 0, 5}^2 and one GEMM (+ ReLU), the 3 x 3 conv
  (+ ReLU), then conv3 as a GEMM with fp32 output: the 16-column head map whose columns 7.. are the reference's output;
- MLSDdetector: the line decode (sigmoid, 3 x 3 peaks, the 200 best) on the device in ctrlora_mlsd_decode; the 200
  candidates come back and the host applies the two thresholds and draws the lines with cv2.line, as pred_lines and
  MLSDdetector.__call__ do.

Inference only, on the current stream.
"""
import cv2
import numpy as np
import torch
import torch.nn as nn

from .. import ops, prepare
from .common import checkpoint_path, device_input, freeze

CKPT_NAME = "mlsd_large_512_fp32.pth"
# MobileNetV2's inverted residual setting up to the 96-channel stage: (expansion t, channels c, blocks n, stride s)
SETTING = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1))
FPN = (1, 3, 6, 10, 13)        # features after which c1 .. c5 are taken
STEM_TAPS = [(ky, kx) for ky in range(3) for kx in range(3)]
DIL_TAPS = [(5 * (ky - 1), 5 * (kx - 1)) for ky in range(3) for kx in range(3)]
HEAD_LD = 16                   # block23.conv3's output columns; the reference keeps columns 7..15
CENTER, DISP = 7, 8            # the centre map and the first of the four displacement maps among them
TOPK = ops.MLSD_TOPK


# ------------------------------------------------------------------------------------------------ modules
class _ConvBNReLU(nn.Sequential):
    """Conv2d (no bias), BatchNorm2d, ReLU6: keys .0 and .1"""

    def __init__(self, cin, cout, k=3, groups=1):
        super().__init__(nn.Conv2d(cin, cout, k, bias=False, groups=groups), nn.BatchNorm2d(cout), nn.ReLU6())


class _InvertedResidual(nn.Module):
    def __init__(self, cin, cout, stride, t):
        super().__init__()
        hidden = int(round(cin * t))
        self.stride = stride
        self.use_res_connect = stride == 1 and cin == cout
        layers = [_ConvBNReLU(cin, hidden, 1)] if t != 1 else []
        layers += [_ConvBNReLU(hidden, hidden, 3, groups=hidden), nn.Conv2d(hidden, cout, 1, bias=False),
                   nn.BatchNorm2d(cout)]
        self.conv = nn.Sequential(*layers)


class _MobileNetV2(nn.Module):
    def __init__(self):
        super().__init__()
        features = [_ConvBNReLU(4, 32, 3)]
        cin = 32
        for t, c, n, s in SETTING:
            for i in range(n):
                features.append(_InvertedResidual(cin, c, s if i == 0 else 1, t))
                cin = c
        self.features = nn.Sequential(*features)


def _cbr(cin, cout, k, dilation=1):
    return nn.Sequential(nn.Conv2d(cin, cout, k, padding=dilation * (k // 2), dilation=dilation), nn.BatchNorm2d(cout),
                         nn.ReLU())


class _BlockTypeA(nn.Module):
    def __init__(self, in_c1, in_c2, out_c1, out_c2, upscale=True):
        super().__init__()
        self.conv1 = _cbr(in_c2, out_c2, 1)
        self.conv2 = _cbr(in_c1, out_c1, 1)
        self.upscale = upscale


class _BlockTypeB(nn.Module):
    def __init__(self, in_c, out_c):
        super().__init__()
        self.conv1 = _cbr(in_c, in_c, 3)
        self.conv2 = _cbr(in_c, out_c, 3)


class _BlockTypeC(nn.Module):
    def __init__(self, in_c, out_c):
        super().__init__()
        self.conv1 = _cbr(in_c, in_c, 3, dilation=5)
        self.conv2 = _cbr(in_c, in_c, 3)
        self.conv3 = nn.Conv2d(in_c, out_c, 1)


def fold_bn(conv, bn=None):
    """(weight, bias) fp32 of `conv` followed by the eval BatchNorm `bn`: w * s, (b - mean) * s + beta with
    s = gamma / sqrt(var + eps) per output channel; a missing conv bias is 0"""
    w = conv.weight.detach().float()
    b = conv.bias.detach().float() if conv.bias is not None else torch.zeros(w.shape[0], device=w.device)
    if bn is None:
        return w, b
    s = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
    return w * s.view(-1, 1, 1, 1), (b - bn.running_mean.detach().float()) * s + bn.bias.detach().float()


def _params(conv, bn=None):
    ps = [conv.weight] + ([conv.bias] if conv.bias is not None else [])
    return ps + ([bn.weight, bn.bias, bn.running_mean, bn.running_var] if bn is not None else [])


def check_size(h, w):
    """ValueError unless the decoder's concatenations fit: H and W are 0 or 1 mod 16 and at least 16"""
    if h % 16 > 1 or w % 16 > 1 or h < 16 or w < 16:
        raise ValueError(f"{h} x {w}: M-LSD needs H and W equal to 0 or 1 mod 16 and at least 16 (the reference's "
                         "decoder concatenates the x2-upsampled deeper level with the next one)")


class MobileV2_MLSD_Large(nn.Module):
    """models/mbv2_mlsd_large.py's MobileV2_MLSD_Large.  forward(x fp32 [B, 4, H, W]: the reference's input, the RGB
    values and the constant channel scaled by / 127.5 - 1) -> fp32 [B, 9, H // 2, W // 2], the reference's output.
    H and W must be 0 or 1 mod 16 and at least 16, as the reference's decoder needs.  split_k: see common.freeze."""

    def __init__(self):
        super().__init__()
        self.backbone = _MobileNetV2()
        self.block15 = _BlockTypeA(64, 96, 64, 64, upscale=False)
        self.block16 = _BlockTypeB(128, 64)
        self.block17 = _BlockTypeA(32, 64, 64, 64)
        self.block18 = _BlockTypeB(128, 64)
        self.block19 = _BlockTypeA(24, 64, 64, 64)
        self.block20 = _BlockTypeB(128, 64)
        self.block21 = _BlockTypeA(16, 64, 64, 64)
        self.block22 = _BlockTypeB(128, 64)
        self.block23 = _BlockTypeC(64, 16)
        freeze(self)

    # ---- kernel-layout weights
    def _stem(self):
        conv, bn = self.backbone.features[0][0], self.backbone.features[0][1]

        def build():
            w, b = fold_bn(conv, bn)
            return prepare.flat_conv_weight(w, 8), b.contiguous()  # K = 9 taps x 4 channels = 36 -> 40
        return self._prep.get("stem", _params(conv, bn), build)

    def _pw(self, key, conv, bn=None):
        """a 1 x 1 conv (+ BatchNorm) -> fp16 [N, 1, K], fp32 bias"""
        def build():
            w, b = fold_bn(conv, bn)
            return prepare.linear_weight(w.reshape(w.shape[0], -1).contiguous()), b.contiguous()
        return self._prep.get(key, _params(conv, bn), build)

    def _dw(self, key, conv, bn):
        """a depthwise 3 x 3 conv + BatchNorm -> fp32 [9, C] tap-major, fp32 bias"""
        def build():
            w, b = fold_bn(conv, bn)
            return w.reshape(w.shape[0], 9).t().contiguous(), b.contiguous()
        return self._prep.get(key, _params(conv, bn), build)

    def _c3(self, key, conv, bn, flat=False):
        """a 3 x 3 conv + BatchNorm -> fp16 [N, 9, C] for the implicit GEMM, or [N, 1, 9 C] for a tap gather (flat)"""
        def build():
            w, b = fold_bn(conv, bn)
            return (prepare.flat_conv_weight(w) if flat else prepare.conv_weight(w)), b.contiguous()
        return self._prep.get(key, _params(conv, bn), build)

    # ---- forward
    def _check(self, x):
        if x.dim() != 4 or x.shape[1] != 4:
            raise ValueError(f"input must be [B, 4, H, W], got {tuple(x.shape)}")
        check_size(x.shape[2], x.shape[3])
        return device_input(self, x, self.block23.conv3.weight)

    def _inverted_residual(self, i, blk, x):
        sk = self.split_k
        layers = list(blk.conv)
        t = x
        if len(layers) == 4:
            we, be = self._pw(("expand", i), layers[0][0], layers[0][1])
            t = ops.gemm_relu6(x, we, bias=be, split_k=sk)
        dw = layers[-3]
        wd, bd = self._dw(("dw", i), dw[0], dw[1])
        t = ops.dwconv_act(t, wd, bd, 3, stride=blk.stride, act="relu6")
        wp, bp = self._pw(("project", i), layers[-2], layers[-1])
        return ops.gemm(t, wp, bias=bp, residual=x if blk.use_res_connect else None, split_k=sk)

    def _backbone(self, x):
        """c1 .. c5: fp16 [B, h, w, C] at H / 2 (16), H / 4 (24), H / 8 (32), H / 16 (64, 96)"""
        ws, bs = self._stem()
        rows = ops.tap_gather_act(x, STEM_TAPS, reflect=False, k_pad=ws.shape[-1], stride=2)
        y = ops.gemm_relu6(rows, ws, bias=bs, split_k=self.split_k)
        feats = []
        for i in range(1, FPN[-1] + 1):
            y = self._inverted_residual(i, self.backbone.features[i], y)
            if i in FPN:
                feats.append(y)
        return feats

    def _block_a(self, name, blk, a, b):
        """cat(conv2(a), up?(conv1(b))): fp16 [B, h, w, 128], each half written in place"""
        sk = self.split_k
        n, h, w, _ = a.shape
        cat = torch.empty((n, h, w, 128), device=a.device, dtype=torch.float16)
        w2, b2 = self._pw((name, "conv2"), blk.conv2[0], blk.conv2[1])
        ops.gemm_relu(a, w2, bias=b2, out=cat[..., :64], split_k=sk)
        w1, b1 = self._pw((name, "conv1"), blk.conv1[0], blk.conv1[1])
        if blk.upscale:
            ops.upsample_bilinear2x_into(ops.gemm_relu(b, w1, bias=b1, split_k=sk), cat[..., 64:])
        else:
            ops.gemm_relu(b, w1, bias=b1, out=cat[..., 64:], split_k=sk)
        return cat

    def _block_b(self, name, blk, x):
        sk = self.split_k
        w1, b1 = self._c3((name, "conv1"), blk.conv1[0], blk.conv1[1])
        y = ops.gemm_relu_residual(x, w1, ksize=3, bias=b1, residual=x, split_k=sk)
        w2, b2 = self._c3((name, "conv2"), blk.conv2[0], blk.conv2[1])
        return ops.gemm_relu(y, w2, ksize=3, bias=b2, split_k=sk)

    def _block_c(self, blk, x):
        sk = self.split_k
        wd, bd = self._c3(("block23", "conv1"), blk.conv1[0], blk.conv1[1], flat=True)
        rows = ops.tap_gather(x, DIL_TAPS, reflect=False, k_pad=wd.shape[-1])
        y = ops.gemm_relu(rows, wd, bias=bd, split_k=sk)
        w2, b2 = self._c3(("block23", "conv2"), blk.conv2[0], blk.conv2[1])
        y = ops.gemm_relu(y, w2, ksize=3, bias=b2, split_k=sk)
        w3, b3 = self._pw(("block23", "conv3"), blk.conv3)
        return ops.gemm(y, w3, bias=b3, out_f32=True, split_k=sk)

    def _run(self, x):
        """(the head map fp32 [B, H // 2, W // 2, HEAD_LD], [c1 .. c5])"""
        feats = self._backbone(self._check(x))
        c1, c2, c3, c4, c5 = feats
        y = self._block_b("block16", self.block16, self._block_a("block15", self.block15, c4, c5))
        y = self._block_b("block18", self.block18, self._block_a("block17", self.block17, c3, y))
        y = self._block_b("block20", self.block20, self._block_a("block19", self.block19, c2, y))
        y = self._block_b("block22", self.block22, self._block_a("block21", self.block21, c1, y))
        return self._block_c(self.block23, y), feats

    @torch.no_grad()
    def forward(self, x):
        return self._run(x)[0][..., CENTER:].permute(0, 3, 1, 2).contiguous()

    @torch.no_grad()
    def forward_stages(self, x):
        """(forward's output, {"features": c1 .. c5 fp16 [B, h, w, C]})"""
        tp, feats = self._run(x)
        return tp[..., CENTER:].permute(0, 3, 1, 2).contiguous(), {"features": feats}


# ------------------------------------------------------------------------------------------------ detector
def network_input(img):
    """pred_lines' network input for an HWC uint8 image at its own size: [image, ones] as float32 NCHW, then
    / 127.5 - 1.0 in float32 (numpy's operations, so the values are the reference's bit for bit).  The reference's
    cv2.resize to the image's own size is a copy and is skipped."""
    h, w = img.shape[:2]
    x = np.concatenate([img, np.ones([h, w, 1])], axis=-1).transpose(2, 0, 1)[None].astype("float32")
    return torch.from_numpy(np.ascontiguousarray((x / 127.5) - 1.0))


def returns_zeros(h, w, thr_v):
    """True where the reference's __call__ returns an all-zero map whatever the image: its decoder cannot concatenate
    (H or W not 0 or 1 mod 16, or below 16), torch.topk has fewer than 200 scores, or no score can exceed thr_v (a
    sigmoid never exceeds 1)"""
    return h % 16 > 1 or w % 16 > 1 or h < 16 or w < 16 or (h // 2) * (w // 2) < TOPK or not thr_v < 1


def select_lines(idx, val, w2, thr_v, thr_d):
    """pred_lines' filter over the decoded candidates (idx int [TOPK] flat indices into the [h2, w2] map, val fp32
    [TOPK, 6] as ops.mlsd_decode returns them) -> [(x_start, y_start, x_end, y_end)] as ints, in candidate order.  A
    candidate is kept when score > thr_v and dist > thr_d, with the fp32 values widened to float64 (numpy 1.26's
    comparison); each endpoint is int(2 * (x + d)) with x + d in float64, as int64 + float32 promotes."""
    lines = []
    for i, v in zip(np.asarray(idx).tolist(), np.asarray(val, dtype=np.float32)):
        if float(v[0]) > thr_v and float(v[1]) > thr_d:
            y, x = divmod(int(i), w2)
            d = [float(t) for t in v[2:6]]
            lines.append((int(2 * (x + d[0])), int(2 * (y + d[1])), int(2 * (x + d[2])), int(2 * (y + d[3]))))
    return lines


def draw_lines(h, w, lines):
    """MLSDdetector.__call__'s map: every line drawn with cv2.line(..., [255, 255, 255], 1) on a zero 3-channel image,
    channel 0 of it -> uint8 [h, w]"""
    out = np.zeros((h, w, 3), dtype=np.uint8)
    for x0, y0, x1, y1 in lines:
        cv2.line(out, (x0, y0), (x1, y1), [255, 255, 255], 1)
    return np.ascontiguousarray(out[:, :, 0])


class MLSDdetector:
    """The reference's MLSDdetector: __call__(HWC uint8 RGB image, thr_v, thr_d) -> uint8 [H, W] line map, from
    mlsd_large_512_fp32.pth in `ckpt_dir` (default: the reference's checkpoint directory).  Nothing is downloaded.

    The reference swallows every exception of its body and returns the zeros drawn so far; this detector returns zeros
    in exactly the cases where that happens (see returns_zeros, and when no candidate passes the thresholds), without
    running the network when the size or thr_v already decides it.  The one deliberate difference: an image that is not
    3-D, not 3-channel or not uint8 raises ValueError instead of being turned into zeros."""

    def __init__(self, ckpt_dir=None, device="cuda"):
        self.device = device
        path = checkpoint_path(ckpt_dir, CKPT_NAME)
        self.model = MobileV2_MLSD_Large().to(device)
        self.model.load_state_dict(torch.load(path, map_location="cpu", weights_only=True), strict=True)

    def __call__(self, input_image, thr_v, thr_d):
        img = input_image
        if not isinstance(img, np.ndarray) or img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.uint8:
            raise ValueError("MLSDdetector takes an HWC uint8 RGB image, got "
                             f"{getattr(img, 'dtype', type(img))} {getattr(img, 'shape', '')}")
        h, w = img.shape[:2]
        if returns_zeros(h, w, thr_v):
            return np.zeros((h, w), dtype=np.uint8)
        tp, _ = self.model._run(network_input(img).to(self.device))
        idx, val = ops.mlsd_decode(tp, CENTER, DISP)
        return draw_lines(h, w, select_lines(idx[0].cpu().numpy(), val[0].cpu().numpy(), w // 2, thr_v, thr_d))
