"""The anime line-art annotator (annotator/lineart_anime/__init__.py: Anime2Sketch's UnetGenerator and
LineartAnimeDetector) on the sm_90a kernels.

Switching a caller over is an import swap: `from ctrlora_b200.annotator.lineart_anime import LineartAnimeDetector`.
`UnetGenerator` keeps the reference's module tree (the nested `model.model.N` Sequentials, same indices), so
`state_dict()` equals the reference's and netG.pth loads with strict=True.  The nn modules only hold the parameters;
forward runs, for the blocks from the outermost (0) to the innermost (num_downs - 1):

- every Conv2d(4, stride 2, padding 1): a stride-2, 16-tap zero-masked gather that applies the block's
  LeakyReLU(0.2) as it loads (block 0: none, straight from the fp32 NCHW input, K = 48 padded to 64) and one
  ctrlora_gemm_f16.  The convs in front of an InstanceNorm run without their bias (the norm subtracts each channel's
  mean, so a per-channel constant cancels exactly); block 0's conv keeps its bias, the innermost conv its bias and,
  in the GEMM's epilogue, the ReLU that follows it;
- every ConvTranspose2d(4, stride 2, padding 1) but the outermost: four sub-pixel phases of 2 x 2 taps each.  A middle
  block's input is the concatenation [x, up] of its submodule, which is never materialised: each phase is one GEMM
  with two operand pairs, gather(relu(x)) @ W_x + gather(relu(up)) @ W_up (the `a2` / `w2` operand), then one
  ctrlora_instance_norm_f16 interleaves the phases;
- block 0's ReLU + ConvTranspose2d(128 -> 1) + Tanh (and the detector's * 127.5 + 127.5): ctrlora_lineart_anime_out_f16.

The reference's LeakyReLU(0.2, True) runs in place on the tensor a block later concatenates, so the skip half of
every block's output is leaky(x), not x; downstream only the parent's ReLU reads it, and relu(leaky(x)) = relu(x).
Activations are fp16 pixel-major with fp32 accumulation and fp32 statistics.  Inference only, on the current stream.
H and W must be multiples of 2^num_downs (the reference's `cat` fails on any other size).
"""
import functools
import os

import cv2
import numpy as np
import torch
import torch.nn as nn

from .. import ops, prepare
from .lineart import default_ckpt_dir

TAPS4 = [(ky - 1, kx - 1) for ky in range(4) for kx in range(4)]  # Conv2d(4, stride 2, padding 1): iy = 2y - 1 + ky
# ConvTranspose2d(4, stride 2, padding 1): output row 2m + py reads input rows m + dy through kernel row ky, for the
# (dy, ky) of PHASE_ROWS[py] (oy = 2 iy - 1 + ky); the same for columns.  Phase p = 2 py + px.
PHASE_ROWS = (((0, 1), (-1, 3)), ((1, 0), (0, 2)))


def phase_taps(py, px):
    """[(dy, dx, ky, kx)] of the sub-pixel phase (py, px)"""
    return [(dy, dx, ky, kx) for dy, ky in PHASE_ROWS[py] for dx, kx in PHASE_ROWS[px]]


def _is_instance_norm(norm_layer):
    """nn.InstanceNorm2d, or a partial of it that keeps affine and track_running_stats off (the detector's)"""
    if norm_layer is nn.InstanceNorm2d:
        return True
    return (isinstance(norm_layer, functools.partial) and norm_layer.func is nn.InstanceNorm2d and not norm_layer.args
            and set(norm_layer.keywords) <= {"affine", "track_running_stats"} and not any(norm_layer.keywords.values()))


class UnetSkipConnectionBlock(nn.Module):
    """The reference's block, parameters only: UnetGenerator runs the blocks"""

    def __init__(self, outer_nc, inner_nc, input_nc=None, submodule=None, outermost=False, innermost=False,
                 norm_layer=nn.BatchNorm2d, use_dropout=False):
        super().__init__()
        self.outermost = outermost
        if isinstance(norm_layer, functools.partial):
            use_bias = norm_layer.func == nn.InstanceNorm2d
        else:
            use_bias = norm_layer == nn.InstanceNorm2d
        if input_nc is None:
            input_nc = outer_nc
        downconv = nn.Conv2d(input_nc, inner_nc, kernel_size=4, stride=2, padding=1, bias=use_bias)
        downrelu = nn.LeakyReLU(0.2, True)
        downnorm = norm_layer(inner_nc)
        uprelu = nn.ReLU(True)
        upnorm = norm_layer(outer_nc)
        if outermost:
            upconv = nn.ConvTranspose2d(inner_nc * 2, outer_nc, kernel_size=4, stride=2, padding=1)
            model = [downconv, submodule, uprelu, upconv, nn.Tanh()]
        elif innermost:
            upconv = nn.ConvTranspose2d(inner_nc, outer_nc, kernel_size=4, stride=2, padding=1, bias=use_bias)
            model = [downrelu, downconv, uprelu, upconv, upnorm]
        else:
            upconv = nn.ConvTranspose2d(inner_nc * 2, outer_nc, kernel_size=4, stride=2, padding=1, bias=use_bias)
            model = [downrelu, downconv, downnorm, submodule, uprelu, upconv, upnorm]
            if use_dropout:
                model.append(nn.Dropout(0.5))
        self.model = nn.Sequential(*model)

    def convs(self):
        """(down Conv2d, up ConvTranspose2d)"""
        down = [m for m in self.model if isinstance(m, nn.Conv2d)]
        up = [m for m in self.model if isinstance(m, nn.ConvTranspose2d)]
        return down[0], up[0]


class UnetGenerator(nn.Module):
    """Anime2Sketch's UnetGenerator with the reference's parameters; forward(x fp32 [B, 3, H, W]) -> fp32 [B, 1, H, W].

    Only what LineartAnimeDetector builds runs: input_nc = 3, output_nc = 1, ngf = 64, an InstanceNorm2d norm_layer
    without affine parameters or running statistics, num_downs >= 5, no dropout; anything else raises
    NotImplementedError.  split_k: passed to every GEMM (0 lets the tile model choose; 1 pins one plan per row, so a
    batch of B equals B batches of 1 bit for bit)."""

    def __init__(self, input_nc, output_nc, num_downs, ngf=64, norm_layer=nn.BatchNorm2d, use_dropout=False):
        super().__init__()
        if input_nc != 3 or output_nc != 1 or ngf != 64 or num_downs < 5 or use_dropout or \
                not _is_instance_norm(norm_layer):
            raise NotImplementedError(
                "the sm_90a UnetGenerator runs what LineartAnimeDetector builds: UnetGenerator(3, 1, num_downs >= 5, 64, "
                "norm_layer=partial(nn.InstanceNorm2d, affine=False, track_running_stats=False), use_dropout=False)")
        blk = UnetSkipConnectionBlock(ngf * 8, ngf * 8, submodule=None, norm_layer=norm_layer, innermost=True)
        for _ in range(num_downs - 5):
            blk = UnetSkipConnectionBlock(ngf * 8, ngf * 8, submodule=blk, norm_layer=norm_layer)
        blk = UnetSkipConnectionBlock(ngf * 4, ngf * 8, submodule=blk, norm_layer=norm_layer)
        blk = UnetSkipConnectionBlock(ngf * 2, ngf * 4, submodule=blk, norm_layer=norm_layer)
        blk = UnetSkipConnectionBlock(ngf, ngf * 2, submodule=blk, norm_layer=norm_layer)
        self.model = UnetSkipConnectionBlock(output_nc, ngf, input_nc=input_nc, submodule=blk, outermost=True,
                                             norm_layer=norm_layer)
        self.num_downs = num_downs
        self.split_k = 0
        self.eval()
        for p in self.parameters():
            p.requires_grad = False
        self.__dict__["_prep"] = prepare.PrepCache()

    def blocks(self):
        """the UnetSkipConnectionBlocks from the outermost (0) to the innermost (num_downs - 1)"""
        res, blk = [], self.model
        while blk is not None:
            res.append(blk)
            blk = next((m for m in blk.model if isinstance(m, UnetSkipConnectionBlock)), None)
        return res

    # ---- kernel-layout weights (rebuilt by the PrepCache whenever a parameter changes, e.g. after load_state_dict)
    def _down_weight(self, i, conv):
        """Conv2d weight -> fp16 [Cout, 1, k_pad]: tap-major, channel-minor columns (the gather's order), zero-padded to
        a multiple of 64 (block 0: K = 48)"""
        def build():
            co, ci, kh, kw = conv.weight.shape
            k = kh * kw * ci
            w = prepare.conv_weight(conv.weight).view(co, 1, k)
            k_pad = (k + 63) // 64 * 64
            if k_pad == k:
                return w
            full = torch.zeros((co, 1, k_pad), device=w.device, dtype=torch.float16)
            full[:, :, :k] = w
            return full
        return self._prep.get(f"down{i}", [conv.weight], build)

    def _phase_weights(self, i, convt, split):
        """ConvTranspose2d weight [Cin, Cout, 4, 4] -> per phase 2 py + px: (gather taps, fp16 [Cout, 1, 4 * Cin]) or,
        with split, (taps, fp16 [Cout, 1, 4 * Cin / 2] over the first half of the input channels, fp16 [Cout, 4 * Cin / 2]
        over the second) -- the skip and the submodule halves of the concatenation"""
        def build():
            wt = convt.weight.detach().float().permute(1, 2, 3, 0)  # [Cout, ky, kx, Cin]
            cin = wt.shape[-1]
            res = []
            for py in (0, 1):
                for px in (0, 1):
                    taps = phase_taps(py, px)
                    sel = torch.stack([wt[:, ky, kx] for _, _, ky, kx in taps], 1)  # [Cout, taps, Cin]
                    halves = (sel[..., :cin // 2], sel[..., cin // 2:]) if split else (sel,)
                    ws = [prepare.linear_weight(h.reshape(h.shape[0], -1).contiguous()) for h in halves]
                    if split:
                        ws[1] = ws[1].view(ws[1].shape[0], -1)
                    res.append(([(dy, dx) for dy, dx, _, _ in taps], *ws))
            return res
        return self._prep.get(f"up{i}", [convt.weight], build)

    def _out_weights(self, convt):
        def build():
            return convt.weight.detach().float().reshape(convt.in_channels, 16).contiguous(), prepare.bias_f32(convt.bias)
        return self._prep.get("out", [convt.weight, convt.bias], build)

    def _check(self, x):
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"input must be [B, 3, H, W], got {tuple(x.shape)}")
        h, w = x.shape[2], x.shape[3]
        m = 1 << self.num_downs
        if h % m or w % m:
            raise NotImplementedError(f"{h} x {w}: H and W must be multiples of {m} (2^num_downs: the U-Net's skip "
                                      "concatenations need every level to halve exactly)")
        dev = self.model.model[0].weight.device
        if dev.type != "cuda":
            raise RuntimeError("UnetGenerator runs on the sm_90a kernels only: move the model to a CUDA device")
        return x.to(dev, torch.float32).contiguous()

    def _gather(self, x, taps, act, stride=1):
        c = x.shape[1] if x.dtype == torch.float32 else x.shape[-1]
        k = len(taps) * c
        return ops.tap_gather_act(x, taps, reflect=False, k_pad=(k + 63) // 64 * 64, stride=stride, act=act)

    def _up(self, i, convt, skip, sub_up):
        """block i's ConvTranspose2d + InstanceNorm over [relu(skip) | relu(sub_up)] (sub_up None: the innermost block,
        whose input `skip` is the ReLU'd conv output) -> fp16 [B, 2h, 2w, Cout]"""
        b, h, w, _ = skip.shape
        ph = torch.empty((4, b, h, w, convt.out_channels), device=skip.device, dtype=torch.float16)
        for p, (taps, *ws) in enumerate(self._phase_weights(i, convt, split=sub_up is not None)):
            if sub_up is None:
                ops.gemm(self._gather(skip, taps, None), ws[0], out=ph[p], split_k=self.split_k)
            else:
                ops.gemm(self._gather(skip, taps, "relu"), ws[0], a2=self._gather(sub_up, taps, "relu"), w2=ws[1],
                         out=ph[p], split_k=self.split_k)
        return ops.instance_norm(ph, relu=False, phases=True)

    def _run(self, x, scale=1.0, shift=0.0, stages=None):
        x = self._check(x)
        blocks = self.blocks()
        n = len(blocks)
        sk = self.split_k
        down0, up0 = blocks[0].convs()
        # xs[i]: the input of block i >= 1 (before its in-place LeakyReLU), fp16 pixel-major
        xs = [None, ops.gemm(self._gather(x, TAPS4, None, stride=2), self._down_weight(0, down0),
                             bias=prepare.bias_f32(down0.bias), split_k=sk)]
        for i in range(1, n - 1):
            conv = blocks[i].convs()[0]
            xs.append(ops.instance_norm(ops.gemm(self._gather(xs[i], TAPS4, "leaky", stride=2),
                                                 self._down_weight(i, conv), split_k=sk), relu=False))
        conv, convt = blocks[n - 1].convs()
        inner = ops.gemm_relu(self._gather(xs[n - 1], TAPS4, "leaky", stride=2), self._down_weight(n - 1, conv),
                              bias=prepare.bias_f32(conv.bias), split_k=sk)
        up = self._up(n - 1, convt, inner, None)
        if stages is not None:
            stages.append((xs[n - 1], up))
        for i in range(n - 2, 0, -1):
            up = self._up(i, blocks[i].convs()[1], xs[i + 1], up)
            if stages is not None:
                stages.append((xs[i], up))
        wo, bo = self._out_weights(up0)
        return ops.lineart_anime_out(xs[1], up, wo, bo, scale=scale, shift=shift)

    @torch.no_grad()
    def forward(self, x):
        return self._run(x)

    @torch.no_grad()
    def detect(self, x):
        """forward(x) * 127.5 + 127.5 (fp32, a multiply then an add), as LineartAnimeDetector scales the map"""
        return self._run(x, scale=127.5, shift=127.5)

    @torch.no_grad()
    def forward_stages(self, x):
        """(fp32 map, [the outputs of blocks 1 ... num_downs - 1 as fp32 NCHW]): block i's output is the reference's
        cat([leaky(x), up], 1), its skip half overwritten by the in-place LeakyReLU"""
        st = []
        y = self._run(x, stages=st)
        outs = []
        for skip, up in reversed(st):
            leaky = ops.tap_gather_act(skip, [(0, 0)], reflect=False, k_pad=skip.shape[-1], act="leaky")
            outs.append(torch.cat([ops.nhwc_to_nchw_f32(leaky), ops.nhwc_to_nchw_f32(up)], 1))
        return y, outs


def load_netg(path):
    """netG.pth as the reference loads it: every key containing 'module.' has it removed"""
    ckpt = torch.load(path, map_location="cpu", weights_only=True)
    for key in list(ckpt.keys()):
        if "module." in key:
            ckpt[key.replace("module.", "")] = ckpt[key]
            del ckpt[key]
    return ckpt


class LineartAnimeDetector:
    """The reference's LineartAnimeDetector: netG.pth from `ckpt_dir` (default: the reference's annotator_ckpts_path);
    __call__(HWC uint8 image) -> HW uint8 line map.  Nothing is downloaded: a missing checkpoint raises
    FileNotFoundError with the path it was expected at."""

    def __init__(self, ckpt_dir=None, device="cuda"):
        ckpt_dir = ckpt_dir if ckpt_dir is not None else default_ckpt_dir()
        if ckpt_dir is None:
            raise FileNotFoundError("no checkpoint directory: the reference's annotator package is not importable, so "
                                    "pass ckpt_dir (the directory holding netG.pth)")
        path = os.path.join(ckpt_dir, "netG.pth")
        if not os.path.isfile(path):
            raise FileNotFoundError(f"netG.pth not found at {path}: ctrlora_b200 never downloads checkpoints; fetch "
                                    f"lllyasviel/Annotators' netG.pth into {ckpt_dir}")
        norm_layer = functools.partial(nn.InstanceNorm2d, affine=False, track_running_stats=False)
        net = UnetGenerator(3, 1, 8, 64, norm_layer=norm_layer, use_dropout=False)
        net.load_state_dict(load_netg(path), strict=True)
        self.device = device
        self.model = net.to(device).eval()

    def __call__(self, input_image):
        H, W, C = input_image.shape
        Hn = 256 * int(np.ceil(float(H) / 256.0))
        Wn = 256 * int(np.ceil(float(W) / 256.0))
        img = cv2.resize(input_image, (Wn, Hn), interpolation=cv2.INTER_CUBIC)
        # host side, as the reference computes it on the device: fp32 image / 127.5 - 1, 'h w c -> 1 c h w'
        image_feed = torch.from_numpy(img).float() / 127.5 - 1.0
        image_feed = image_feed.permute(2, 0, 1).unsqueeze(0).contiguous()
        line = self.model.detect(image_feed.to(self.device))[0, 0].cpu().numpy()
        line = cv2.resize(line, (W, H), interpolation=cv2.INTER_CUBIC)
        return line.clip(0, 255).astype(np.uint8)
