"""The HED soft-edge annotator (annotator/hed/__init__.py: ControlNetHED_Apache2 and HEDdetector) on the sm_90a kernels.

Switching a caller over is an import swap: `from ctrlora_b200.annotator.hed import HEDdetector`.
`ControlNetHED_Apache2` keeps the reference's module tree (norm, block1 ... block5, each `convs` + `projection`), so
`state_dict()` equals the reference's and ControlNetHED.pth loads with strict=True.  The nn modules only hold the
parameters; forward runs:

- `x - norm` as one fp32 torch op on the NCHW input, exactly as the reference computes it;
- block1's first conv (K = 27): a zero-masked 3x3 tap gather from that fp32 tensor (padded to K = 32) and one 1x1
  ctrlora_gemm_f16 with the bias and the ReLU in its epilogue (ops.gemm_relu);
- every other 3x3 conv + ReLU: one implicit 3x3 ctrlora_gemm_f16 (zero padding 1 is the TMA out-of-bounds fill) with
  the bias and the ReLU in its epilogue;
- each block's projection (1x1 conv C -> 1) and the next block's max_pool2d(2, 2): ctrlora_hed_side_pool_f16, one read
  of the block's output;
- HEDdetector's host post-process (cv2.resize of the five maps to H x W, mean, float64 sigmoid, safe_step, uint8):
  ctrlora_hed_fuse, through resize tables built on the host by `resize_tables`.

Activations are fp16 pixel-major with fp32 accumulation.  Inference only, on the current stream.  H and W must be at
least 16: the fifth block sees H // 16 x W // 16 pixels.  Odd sizes work: the pools floor as max_pool2d does.
"""
import collections
import os

import numpy as np
import torch
import torch.nn as nn

from .. import ops, prepare
from .lineart import TAPS3, default_ckpt_dir

MIN_SIZE = 16
TABLE_CACHE_SIZES = 8  # output sizes whose device resize tables are kept (least recently used goes first)


def resize_tables(src, dst):
    """cv2.resize(INTER_LINEAR)'s coordinates along one axis of length src -> dst: (int32 [dst] source index, fp32 [dst]
    fraction), output position i = (1 - frac) * s[idx] + frac * s[idx + 1] (the neighbour clamped to the map).  A
    restatement of OpenCV's resizeGeneric rule: scale = 1 / (dst / src) in float64, fx = (float)((i + 0.5) * scale - 0.5),
    sx = floor(fx), fx -= sx in float32, then sx < 0 -> (0, 0) and sx >= src - 1 -> (src - 1, 0)."""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    lo, hi = s < 0, s >= src - 1
    f[lo | hi] = 0.0
    s[lo] = 0
    s[hi] = src - 1
    return s.astype(np.int32), f


def level_sizes(h, w):
    """(h, w) of the five blocks' outputs: each pool floors"""
    sizes = [(h, w)]
    for _ in range(4):
        h, w = h // 2, w // 2
        sizes.append((h, w))
    return sizes


class DoubleConvBlock(nn.Module):
    def __init__(self, input_channel, output_channel, layer_number):
        super().__init__()
        self.convs = nn.Sequential(*[nn.Conv2d(input_channel if i == 0 else output_channel, output_channel, 3, padding=1)
                                     for i in range(layer_number)])
        self.projection = nn.Conv2d(output_channel, 1, 1)


class ControlNetHED_Apache2(nn.Module):
    """The reference's HED network with its parameters; forward(x fp32 [B, 3, H, W], RGB in 0..255) -> the five fp32
    side maps [B, 1, H / 2^i, W / 2^i] (floor).

    split_k: passed to every GEMM (0 lets the tile model choose; 1 pins one plan per row, so a batch of B equals B
    batches of 1 bit for bit)."""

    def __init__(self):
        super().__init__()
        self.norm = nn.Parameter(torch.zeros(1, 3, 1, 1))
        self.block1 = DoubleConvBlock(3, 64, 2)
        self.block2 = DoubleConvBlock(64, 128, 2)
        self.block3 = DoubleConvBlock(128, 256, 3)
        self.block4 = DoubleConvBlock(256, 512, 3)
        self.block5 = DoubleConvBlock(512, 512, 3)
        self.split_k = 0
        self.eval()
        for p in self.parameters():
            p.requires_grad = False
        self.__dict__["_prep"] = prepare.PrepCache()
        self.__dict__["_tables"] = collections.OrderedDict()

    def blocks(self):
        return [self.block1, self.block2, self.block3, self.block4, self.block5]

    # ---- kernel-layout weights (rebuilt by the PrepCache whenever a parameter changes, e.g. after load_state_dict)
    def _conv_weights(self, key, conv, flat):
        """(fp16 weight, fp32 bias): [Cout, 9, Cin] for the implicit 3x3 GEMM, or flat [Cout, 1, 32] (tap-major,
        channel-minor, zero-padded from 27) for block1's first conv on the tap gather"""
        def build():
            w = prepare.conv_weight(conv.weight)
            if flat:
                co, taps, ci = w.shape
                full = torch.zeros((co, 1, 32), device=w.device, dtype=torch.float16)
                full[:, 0, :taps * ci] = w.reshape(co, taps * ci)
                w = full
            return w, prepare.bias_f32(conv.bias)
        return self._prep.get(key, [conv.weight, conv.bias], build)

    def _side_weights(self, key, proj):
        def build():
            return proj.weight.detach().float().reshape(-1).contiguous(), prepare.bias_f32(proj.bias)
        return self._prep.get(key, [proj.weight, proj.bias], build)

    def _resize_tables(self, h, w, device):
        """device (idx, frac) pairs of levels 1..4 for an h x w output, host-built; the last TABLE_CACHE_SIZES sizes are
        kept, so a caller that runs many image sizes holds a bounded set"""
        key = (h, w, str(device))
        tabs = self._tables.get(key)
        if tabs is None:
            tabs = []
            for lh, lw in level_sizes(h, w)[1:]:
                (ri, rf), (ci, cf) = resize_tables(lh, h), resize_tables(lw, w)
                tabs.append((torch.from_numpy(np.concatenate([ri, ci])).to(device),
                             torch.from_numpy(np.concatenate([rf, cf])).to(device)))
            self._tables[key] = tabs
            while len(self._tables) > TABLE_CACHE_SIZES:
                self._tables.popitem(last=False)
        self._tables.move_to_end(key)
        return tabs

    def _check(self, x):
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"input must be [B, 3, H, W], got {tuple(x.shape)}")
        h, w = x.shape[2], x.shape[3]
        if h < MIN_SIZE or w < MIN_SIZE:
            raise ValueError(f"{h} x {w}: H and W must be at least {MIN_SIZE} (the fifth block sees H // 16 x W // 16 "
                             "pixels)")
        dev = self.norm.device
        if dev.type != "cuda":
            raise RuntimeError("ControlNetHED_Apache2 runs on the sm_90a kernels only: move the model to a CUDA device")
        return x.to(dev, torch.float32).contiguous()

    def _run(self, x, stages=None):
        """the five fp32 side maps; with `stages` (a list) also the five blocks' fp16 outputs"""
        x = self._check(x)
        h = (x - self.norm).contiguous()  # the reference's `x - self.norm`, in fp32
        sides = []
        for i, blk in enumerate(self.blocks()):
            for j, conv in enumerate(blk.convs):
                w, b = self._conv_weights(f"b{i}.{j}", conv, flat=i == 0 and j == 0)
                if i == 0 and j == 0:
                    h = ops.gemm_relu(ops.tap_gather(h, TAPS3, reflect=False, k_pad=w.shape[-1]), w, bias=b,
                                      split_k=self.split_k)
                else:
                    h = ops.gemm_relu(h, w, ksize=3, bias=b, split_k=self.split_k)
            if stages is not None:
                stages.append(h)
            pw, pb = self._side_weights(f"p{i}", blk.projection)
            side, h = ops.hed_side_pool(h, pw, pb, pool=i < 4)
            sides.append(side)
        return sides

    @torch.no_grad()
    def forward(self, x):
        return tuple(self._run(x))

    @torch.no_grad()
    def detect(self, x, safe=False):
        """(fp32 [B, H, W] mean of the five resized side maps, uint8 [B, H, W] edge map), as HEDdetector computes them"""
        sides = self._run(x)
        _, _, h, w = sides[0].shape
        return ops.hed_fuse(sides, self._resize_tables(h, w, sides[0].device), safe)

    @torch.no_grad()
    def forward_stages(self, x):
        """(the five side maps, [the outputs of block1 ... block5 as fp32 NCHW])"""
        st = []
        sides = self._run(x, stages=st)
        return tuple(sides), [ops.nhwc_to_nchw_f32(s) for s in st]


class HEDdetector:
    """The reference's HEDdetector: ControlNetHED.pth from `ckpt_dir` (default: the reference's annotator_ckpts_path);
    __call__(HWC uint8 RGB image, safe=False) -> HW uint8 edge map.  Nothing is downloaded: a missing checkpoint raises
    FileNotFoundError with the path it was expected at."""

    def __init__(self, ckpt_dir=None, device="cuda"):
        ckpt_dir = ckpt_dir if ckpt_dir is not None else default_ckpt_dir()
        if ckpt_dir is None:
            raise FileNotFoundError("no checkpoint directory: the reference's annotator package is not importable, so "
                                    "pass ckpt_dir (the directory holding ControlNetHED.pth)")
        path = os.path.join(ckpt_dir, "ControlNetHED.pth")
        if not os.path.isfile(path):
            raise FileNotFoundError(f"ControlNetHED.pth not found at {path}: ctrlora_b200 never downloads checkpoints; "
                                    f"fetch lllyasviel/Annotators' ControlNetHED.pth into {ckpt_dir}")
        self.netNetwork = ControlNetHED_Apache2()
        self.netNetwork.load_state_dict(torch.load(path, map_location="cpu", weights_only=True), strict=True)
        self.netNetwork = self.netNetwork.to(device).eval()
        self.device = device

    def __call__(self, input_image, safe=False):
        assert input_image.ndim == 3
        image = torch.from_numpy(input_image.copy()).float().permute(2, 0, 1).unsqueeze(0).contiguous()
        _, u8 = self.netNetwork.detect(image.to(self.device), safe=safe)
        return u8[0].cpu().numpy()
