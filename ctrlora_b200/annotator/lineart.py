"""The line-art annotator (annotator/lineart/__init__.py: informative-drawings' Generator and LineartDetector) on the
sm_90a kernels.

Switching a caller over is an import swap: `from ctrlora_b200.annotator.lineart import LineartDetector`.  `Generator`
keeps the reference's module tree (model0 ... model4, same indices), so `state_dict()` equals the reference's and
sk_model.pth / sk_model2.pth load with strict=True.  The nn modules only hold the parameters; forward runs:

- model0, ReflectionPad2d(3) + Conv2d(7): a reflect tap gather straight from the fp32 NCHW input (K = 49 * 3 padded to
  160) and one ctrlora_gemm_f16;
- model1, Conv2d(3, stride 2, padding 1): ctrlora_im2col_s2_pad_f16 and one GEMM each;
- model2, ReflectionPad2d(1) + Conv2d(3): a reflect tap gather (K = 9 * 256) and one GEMM each;
- model3, ConvTranspose2d(3, stride 2, padding 1, output_padding 1): four sub-pixel phases with 1, 2, 2 and 4 taps,
  each a zero-masked tap gather and a GEMM whose weight is a slice of the transposed kernel;
- every InstanceNorm2d + ReLU (and ResidualBlock's `x + conv_block(x)`) as one ctrlora_instance_norm_f16, which also
  interleaves the transposed convs' phases;
- model4, ReflectionPad2d(3) + Conv2d(64 -> 1, 7) + Sigmoid, and the detector's uint8 quantisation: ctrlora_lineart_out_f16.

The convs in front of an InstanceNorm run without their bias: the norm subtracts each channel's mean, so a per-channel
constant cancels exactly.  Activations are fp16 pixel-major with fp32 accumulation and fp32 statistics.  Inference
only, on the current stream.  H and W must be multiples of 4 (the two stride-2 convs and the two transposed convs then
give back H x W) and at least 8 (the residual blocks' ReflectionPad2d(1) needs 2 x 2 pixels).
"""
import functools

import numpy as np
import torch
import torch.nn as nn

from .. import ops, prepare
from . import common
from .common import TAPS3, checkpoint_path, device_input, freeze, phase_weights

TAPS7 = [(ky - 3, kx - 3) for ky in range(7) for kx in range(7)]
# ConvTranspose2d(3, stride 2, padding 1, output_padding 1): output row 2m + py reads input rows m + dy through kernel
# row ky, for the (dy, ky) of PHASE_ROWS[py] (oy = 2 iy - 1 + ky); the same for columns.  Phase p = 2 py + px.
PHASE_ROWS = (((0, 1),), ((0, 2), (1, 0)))
phase_taps = functools.partial(common.phase_taps, PHASE_ROWS)  # (py, px) -> [(dy, dx, ky, kx)]


class ResidualBlock(nn.Module):
    def __init__(self, features):
        super().__init__()
        self.conv_block = nn.Sequential(
            nn.ReflectionPad2d(1), nn.Conv2d(features, features, 3), nn.InstanceNorm2d(features), nn.ReLU(inplace=True),
            nn.ReflectionPad2d(1), nn.Conv2d(features, features, 3), nn.InstanceNorm2d(features))


class Generator(nn.Module):
    """informative-drawings' Generator with the reference's parameters; forward(x fp32 [B, 3, H, W]) -> fp32 [B, 1, H, W].

    split_k: passed to every GEMM (0 lets the tile model choose; 1 pins one plan per row, so a batch of B equals B
    batches of 1 bit for bit)."""

    def __init__(self, input_nc, output_nc, n_residual_blocks=9, sigmoid=True):
        super().__init__()
        self.model0 = nn.Sequential(nn.ReflectionPad2d(3), nn.Conv2d(input_nc, 64, 7), nn.InstanceNorm2d(64),
                                    nn.ReLU(inplace=True))
        down = []
        for cin in (64, 128):
            down += [nn.Conv2d(cin, 2 * cin, 3, stride=2, padding=1), nn.InstanceNorm2d(2 * cin), nn.ReLU(inplace=True)]
        self.model1 = nn.Sequential(*down)
        self.model2 = nn.Sequential(*[ResidualBlock(256) for _ in range(n_residual_blocks)])
        up = []
        for cin in (256, 128):
            up += [nn.ConvTranspose2d(cin, cin // 2, 3, stride=2, padding=1, output_padding=1), nn.InstanceNorm2d(cin // 2),
                   nn.ReLU(inplace=True)]
        self.model3 = nn.Sequential(*up)
        out = [nn.ReflectionPad2d(3), nn.Conv2d(64, output_nc, 7)]
        if sigmoid:
            out.append(nn.Sigmoid())
        self.model4 = nn.Sequential(*out)
        freeze(self)

    # ---- kernel-layout weights
    def _conv_gemm_weight(self, key, conv):
        """Conv2d weight -> fp16 [Cout, 1, k_pad], K zero-padded to a multiple of 16"""
        return self._prep.get(key, [conv.weight], lambda: prepare.flat_conv_weight(conv.weight, 16))

    def _phase_weights(self, key, convt):
        """ConvTranspose2d weight [Cin, Cout, 3, 3] -> per phase 2 py + px: (gather taps, fp16 [Cout, 1, taps * Cin])"""
        return self._prep.get(key, [convt.weight], lambda: phase_weights(convt, PHASE_ROWS))

    def _out_weights(self):
        conv = self.model4[1]

        def build():
            w = conv.weight.detach().float()[0].permute(1, 2, 0).reshape(49, -1).contiguous()  # [taps, C]
            return w, prepare.bias_f32(conv.bias)
        return self._prep.get("out", [conv.weight, conv.bias], build)

    def _gemm(self, a, w, out=None):
        return ops.gemm(a, w, out=out, split_k=self.split_k)

    def _check(self, x):
        if self.model4[1].out_channels != 1 or not isinstance(self.model4[-1], nn.Sigmoid):
            raise NotImplementedError("the output kernel computes Conv2d(64 -> 1) + Sigmoid only (Generator(3, 1, ...))")
        if x.dim() != 4 or x.shape[1] != self.model0[1].in_channels:
            raise ValueError(f"input must be [B, {self.model0[1].in_channels}, H, W], got {tuple(x.shape)}")
        h, w = x.shape[2], x.shape[3]
        if h % 4 or w % 4:
            raise NotImplementedError(f"{h} x {w}: H and W must be multiples of 4 (the transposed convs otherwise change "
                                      "the output size)")
        if h < 8 or w < 8:
            raise ValueError(f"{h} x {w}: H and W must be at least 8 (ReflectionPad2d(1) of the residual blocks)")
        return device_input(self, x, self.model4[1].weight)

    def _run(self, x, want_u8=False, stages=None):
        x = self._check(x)
        b = x.shape[0]
        conv0 = self.model0[1]
        w0 = self._conv_gemm_weight("m0", conv0)
        a = ops.tap_gather(x, TAPS7, reflect=True, k_pad=w0.shape[-1])
        h = ops.instance_norm(self._gemm(a, w0), relu=True)
        if stages is not None:
            stages.append(h)
        for i in (0, 3):
            h = ops.instance_norm(self._gemm(ops.im2col_s2(h, pad_lo=1), self._conv_gemm_weight(f"m1.{i}", self.model1[i])),
                                  relu=True)
        if stages is not None:
            stages.append(h)
        for j, blk in enumerate(self.model2):
            wa = self._conv_gemm_weight(f"m2.{j}.a", blk.conv_block[1])
            wb = self._conv_gemm_weight(f"m2.{j}.b", blk.conv_block[5])
            t = ops.instance_norm(self._gemm(ops.tap_gather(h, TAPS3, reflect=True, k_pad=wa.shape[-1]), wa), relu=True)
            h = ops.instance_norm(self._gemm(ops.tap_gather(t, TAPS3, reflect=True, k_pad=wb.shape[-1]), wb), relu=False,
                                  residual=h)
        if stages is not None:
            stages.append(h)
        for i in (0, 3):
            convt = self.model3[i]
            _, hh, ww, cin = h.shape
            ph = torch.empty((4, b, hh, ww, convt.out_channels), device=h.device, dtype=torch.float16)
            for p, (taps, wp) in enumerate(self._phase_weights(f"m3.{i}", convt)):
                self._gemm(ops.tap_gather(h, taps, reflect=False, k_pad=len(taps) * cin), wp, out=ph[p])
            h = ops.instance_norm(ph, relu=True, phases=True)
        if stages is not None:
            stages.append(h)
        w4, b4 = self._out_weights()
        return ops.lineart_out(h, w4, b4, want_u8=want_u8)

    @torch.no_grad()
    def forward(self, x, cond=None):
        return self._run(x)

    @torch.no_grad()
    def detect(self, x):
        """(fp32 [B, 1, H, W] map, uint8 [B, H, W] map (uint8)clip(map * 255, 0, 255)), as LineartDetector quantises"""
        return self._run(x, want_u8=True)

    @torch.no_grad()
    def forward_stages(self, x):
        """(fp32 map, [the outputs of model0, model1, model2, model3 as fp32 NCHW])"""
        st = []
        y = self._run(x, stages=st)
        return y, [ops.nhwc_to_nchw_f32(s) for s in st]


class LineartDetector:
    """The reference's LineartDetector: sk_model.pth (fine) and sk_model2.pth (coarse) from `ckpt_dir` (default: the
    reference's checkpoint directory); __call__(HWC uint8 image, coarse) -> HW uint8 line map.  Nothing is downloaded:
    a missing checkpoint raises FileNotFoundError with the path it was expected at."""

    def __init__(self, ckpt_dir=None, device="cuda"):
        self.ckpt_dir, self.device = ckpt_dir, device
        self.model = self.load_model("sk_model.pth")
        self.model_coarse = self.load_model("sk_model2.pth")

    def load_model(self, name):
        path = checkpoint_path(self.ckpt_dir, name)
        model = Generator(3, 1, 3)
        model.load_state_dict(torch.load(path, map_location="cpu", weights_only=True), strict=True)
        return model.to(self.device).eval()

    def __call__(self, input_image, coarse):
        model = self.model_coarse if coarse else self.model
        assert input_image.ndim == 3
        # host side, as the reference computes it on the device: fp32 image / 255, HWC -> 1CHW
        image = torch.from_numpy(np.ascontiguousarray(input_image)).float() / 255.0
        image = image.permute(2, 0, 1).unsqueeze(0).contiguous()
        _, u8 = model.detect(image.to(self.device))
        return u8[0].cpu().numpy()
