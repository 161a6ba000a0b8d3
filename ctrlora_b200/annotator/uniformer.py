"""The UniFormer segmentation annotator (annotator/uniformer/__init__.py UniformerDetector: mmseg's EncoderDecoder with
a UniFormer-S backbone and a UPerHead, exp/upernet_global_small/config.py) on the sm_90a kernels.

Switching a caller over is an import swap: `from ctrlora_b200.annotator.uniformer import UniformerDetector`.  The
modules keep mmseg's tree (`backbone.*`, `decode_head.*`, `auxiliary_head.*`), so `state_dict()` equals the
reference segmentor's and upernet_global_small.pth loads with strict=True.  The auxiliary FCNHead is loaded and never
run, as in the reference's inference.  The nn modules hold the parameters only; forward runs, on fp16 pixel-major
activations with fp32 accumulation:

- patch_embed1: ctrlora_patch_gather_hw (4 x 4, stride 4) + one GEMM whose weight and bias have mmseg's Normalize
  folded in (mean, std and the BGR order: mmseg reads the RGB input as BGR and reverses it), so the network takes the
  resized image's 0..255 RGB values; patch_embed2..4: a 2 x 2 stride-2 tap gather + one GEMM.  Both truncate odd
  sizes as the stride-k Conv2d does.  Each is followed by its LayerNorm (eps 1e-5);
- CBlock (stages 1-2): x + dw3x3(x) in one ctrlora_dwconv_f16; conv1 with norm1 (BatchNorm) folded in, dw5x5, conv2 +
  residual; mlp.fc1 with norm2 folded in, GELU, mlp.fc2 + residual;
- SABlock (stages 3-4): x + dw3x3(x), then text_encoder.run_layers over the one block (LayerNorm eps 1e-6, fused
  q | k | v, global attention at d_head 64, exact GELU) on the fp16 stream;
- norm1..4 (LayerNorm eps 1e-6) give the four features; norm4 writes into the PPM's concatenation buffer;
- UPerHead: every ConvModule's BatchNorm folded into its conv, ReLU in the GEMM's epilogue; the PPM's four
  AdaptiveAvgPool2d in one ctrlora_adaptive_avg_pool_f16, its 1 x 1 convs as GEMMs on the pooled rows, and every
  bilinear resize (align_corners=False) by ctrlora_resize_bilinear_f16, writing its channel slice of the
  concatenation in place or accumulating into the lateral it is added to; conv_seg writes fp32 logits at 1/4 size;
- UniformerDetector: the logits resized to the network size, then to the input size, the argmax and the palette
  lookup in one ctrlora_seg_output launch.  Softmax is monotonic and not computed.

Inference only, on the current stream.  The palette is read from the checkpoint's meta["PALETTE"].
"""
import cv2
import numpy as np
import torch
import torch.nn as nn

from .. import ops, prepare
from ..text_encoder import run_layers
from .common import checkpoint_path, device_input, freeze, vit_block_weights

CKPT_NAME = "upernet_global_small.pth"
EMBED = (64, 128, 320, 512)
LAYERS = (3, 4, 8, 3)
HEAD_DIM = 64
CHANNELS = 512                 # UPerHead channels
POOL_SCALES = (1, 2, 3, 6)
NUM_CLASSES = 150
LOGIT_LD = 152                 # conv_seg's output row: the classes padded to a multiple of 4 (fp32 vector loads)
IMG_SCALE = (2048, 512)        # the test pipeline's Resize(img_scale, keep_ratio=True)
MEAN = (123.675, 116.28, 103.53)
STD = (58.395, 57.12, 57.375)
TAPS2 = [(0, 0), (0, 1), (1, 0), (1, 1)]


def rescale_size(h, w):
    """mmcv.imrescale's output (height, width) for an h x w image at IMG_SCALE: scale = min(2048 / long side,
    512 / short side), each side int(side * scale + 0.5)"""
    scale = min(max(IMG_SCALE) / max(h, w), min(IMG_SCALE) / min(h, w))
    return int(h * float(scale) + 0.5), int(w * float(scale) + 0.5)


# ------------------------------------------------------------------------------------------------ backbone (UniFormer)
class _PatchEmbed(nn.Module):
    def __init__(self, cin, dim, patch):
        super().__init__()
        self.norm = nn.LayerNorm(dim)
        self.proj = nn.Conv2d(cin, dim, kernel_size=patch, stride=patch)


class _CMlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Conv2d(dim, hidden, 1)
        self.fc2 = nn.Conv2d(hidden, dim, 1)


class _CBlock(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.pos_embed = nn.Conv2d(dim, dim, 3, padding=1, groups=dim)
        self.norm1 = nn.BatchNorm2d(dim)
        self.conv1 = nn.Conv2d(dim, dim, 1)
        self.conv2 = nn.Conv2d(dim, dim, 1)
        self.attn = nn.Conv2d(dim, dim, 5, padding=2, groups=dim)
        self.norm2 = nn.BatchNorm2d(dim)
        self.mlp = _CMlp(dim, 4 * dim)


class _Attention(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.qkv = nn.Linear(dim, 3 * dim)
        self.proj = nn.Linear(dim, dim)


class _Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


class _SABlock(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.pos_embed = nn.Conv2d(dim, dim, 3, padding=1, groups=dim)
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = _Attention(dim)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = _Mlp(dim, 4 * dim)


class _UniFormer(nn.Module):
    def __init__(self):
        super().__init__()
        cins = (3,) + EMBED[:3]
        for i, (cin, dim, patch) in enumerate(zip(cins, EMBED, (4, 2, 2, 2)), 1):
            setattr(self, f"patch_embed{i}", _PatchEmbed(cin, dim, patch))
        for i, (dim, n) in enumerate(zip(EMBED, LAYERS), 1):
            block = _CBlock if i <= 2 else _SABlock
            setattr(self, f"blocks{i}", nn.ModuleList(block(dim) for _ in range(n)))
            setattr(self, f"norm{i}", nn.LayerNorm(dim, eps=1e-6))


# ------------------------------------------------------------------------------------------------ heads
class _ConvModule(nn.Module):
    """mmcv's ConvModule(conv_cfg=None, norm_cfg=BN, act_cfg=ReLU): conv without bias, BatchNorm, ReLU"""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, padding=k // 2, bias=False)
        self.bn = nn.BatchNorm2d(cout)


class _UPerHead(nn.Module):
    def __init__(self, num_classes):
        super().__init__()
        self.conv_seg = nn.Conv2d(CHANNELS, num_classes, 1)
        self.psp_modules = nn.ModuleList(
            nn.Sequential(nn.AdaptiveAvgPool2d(s), _ConvModule(EMBED[-1], CHANNELS, 1)) for s in POOL_SCALES)
        self.bottleneck = _ConvModule(EMBED[-1] + len(POOL_SCALES) * CHANNELS, CHANNELS, 3)
        self.lateral_convs = nn.ModuleList(_ConvModule(c, CHANNELS, 1) for c in EMBED[:-1])
        self.fpn_convs = nn.ModuleList(_ConvModule(CHANNELS, CHANNELS, 3) for _ in EMBED[:-1])
        self.fpn_bottleneck = _ConvModule(len(EMBED) * CHANNELS, CHANNELS, 3)


class _FCNHead(nn.Module):
    """the auxiliary head (in_channels 320, channels 256, one conv): loaded, never run"""

    def __init__(self, num_classes):
        super().__init__()
        self.conv_seg = nn.Conv2d(256, num_classes, 1)
        self.convs = nn.Sequential(_ConvModule(EMBED[2], 256, 3))


def load_checkpoint(path):
    """(state dict, palette uint8 [classes, 3]) of an mmcv checkpoint: the weights under "state_dict" (a "module."
    prefix stripped, as mmcv's load_checkpoint does), the palette from meta["PALETTE"]"""
    ckpt = torch.load(path, map_location="cpu", weights_only=True)
    sd = ckpt.get("state_dict", ckpt)
    sd = {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}
    palette = (ckpt.get("meta") or {}).get("PALETTE")
    if palette is None:
        raise ValueError(f"{path}: the checkpoint has no meta['PALETTE'] (the class colours of the segmentation map)")
    return sd, torch.tensor(np.asarray(palette), dtype=torch.uint8)


def _bn_affine(bn):
    """eval BatchNorm as y = x * s + t: (s, t) fp32"""
    s = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
    return s, bn.bias.detach().float() - bn.running_mean.detach().float() * s


def _bn_params(bn):
    return [bn.weight, bn.bias, bn.running_mean, bn.running_var]


class UniformerSegmentor(nn.Module):
    """mmseg's EncoderDecoder of exp/upernet_global_small/config.py (UniFormer-S: embed_dim [64, 128, 320, 512],
    layers [3, 4, 8, 3], head_dim 64, qkv_bias, global attention; UPerHead with 512 channels; 150 classes).
    forward(x fp32 [B, 3, H, W]: the resized image's RGB values in 0..255, un-normalised) -> fp32 logits
    [B, H4, W4, num_classes] at the 1/4 level (H4 = H // 4, W4 = W // 4).  Other configurations raise
    NotImplementedError.  split_k: passed to every GEMM (0 lets the tile model choose; 1 pins one plan per row, so a
    batch of B equals B batches of 1 bit for bit).  `palette` (uint8 [classes, 3], a buffer outside the state dict) is
    set by load()."""

    def __init__(self, num_classes=NUM_CLASSES, windows=False, hybrid=False):
        super().__init__()
        if windows or hybrid or num_classes != NUM_CLASSES:
            raise NotImplementedError("the sm_90a UniformerSegmentor runs upernet_global_small only: windows=False, "
                                      f"hybrid=False, num_classes={NUM_CLASSES}")
        self.backbone = _UniFormer()
        self.decode_head = _UPerHead(num_classes)
        self.auxiliary_head = _FCNHead(num_classes)
        self.register_buffer("palette", torch.zeros((num_classes, 3), dtype=torch.uint8), persistent=False)
        freeze(self)

    def load(self, path):
        sd, palette = load_checkpoint(path)
        self.load_state_dict(sd, strict=True)
        if palette.shape != self.palette.shape:
            raise ValueError(f"{path}: meta['PALETTE'] has shape {tuple(palette.shape)}, expected ({NUM_CLASSES}, 3)")
        self.palette.copy_(palette)

    # ---- kernel-layout weights
    def _patch1(self):
        """patch_embed1.proj with Normalize folded in: fp16 [64, 1, 48] over the RGB input's (c, ky, kx), fp32 bias"""
        pe = self.backbone.patch_embed1.proj

        def build():
            w = pe.weight.detach().float()
            mean = torch.tensor(MEAN, device=w.device).view(1, 3, 1, 1)
            std = torch.tensor(STD, device=w.device).view(1, 3, 1, 1)
            # the network's channel c reads the input's channel 2 - c, normalised by mean[c], std[c]
            wf = (w / std).flip(1)
            b = pe.bias.detach().float() - (w * (mean / std)).sum(dim=(1, 2, 3))
            return prepare.linear_weight(wf.reshape(w.shape[0], -1).contiguous()), b.contiguous()
        return self._prep.get("patch1", [pe.weight, pe.bias], build)

    def _patch(self, i):
        pe = getattr(self.backbone, f"patch_embed{i}").proj
        return self._prep.get(("patch", i), [pe.weight, pe.bias],
                              lambda: (prepare.flat_conv_weight(pe.weight), prepare.bias_f32(pe.bias)))

    def _ln(self, key, ln):
        return self._prep.get(key, [ln.weight, ln.bias],
                              lambda: (prepare.bias_f32(ln.weight), prepare.bias_f32(ln.bias), ln.eps))

    def _dw(self, key, conv):
        """depthwise Conv2d [C, 1, k, k] -> (fp32 [k * k, C], fp32 bias)"""
        def build():
            c, _, k, _ = conv.weight.shape
            return conv.weight.detach().float().reshape(c, k * k).t().contiguous(), prepare.bias_f32(conv.bias)
        return self._prep.get(key, [conv.weight, conv.bias], build)

    def _conv1x1(self, key, conv, bn_in=None):
        """a 1 x 1 Conv2d (bias) as fp16 [N, 1, K], with an eval BatchNorm on its input folded in"""
        def build():
            w = conv.weight.detach().float().reshape(conv.out_channels, -1)
            b = conv.bias.detach().float()
            if bn_in is not None:
                s, t = _bn_affine(bn_in)
                b = b + w @ t
                w = w * s[None, :]
            return prepare.linear_weight(w.contiguous()), b.contiguous()
        params = [conv.weight, conv.bias] + (_bn_params(bn_in) if bn_in is not None else [])
        return self._prep.get(key, params, build)

    def _cm(self, key, cm):
        """ConvModule: conv (no bias) with its BatchNorm folded in -> (fp16 weight for ops.gemm, fp32 bias)"""
        def build():
            s, t = _bn_affine(cm.bn)
            w = cm.conv.weight.detach().float() * s.view(-1, 1, 1, 1)
            wk = prepare.conv_weight(w) if cm.conv.kernel_size[0] == 3 else prepare.linear_weight(w.reshape(w.shape[0], -1))
            return wk, t.contiguous()
        return self._prep.get(key, [cm.conv.weight] + _bn_params(cm.bn), build)

    def _seg(self):
        conv = self.decode_head.conv_seg

        def build():
            w = torch.zeros((LOGIT_LD, CHANNELS), device=conv.weight.device)
            b = torch.zeros(LOGIT_LD, device=conv.weight.device)
            w[:NUM_CLASSES] = conv.weight.detach().float().reshape(NUM_CLASSES, CHANNELS)
            b[:NUM_CLASSES] = conv.bias.detach().float()
            return prepare.linear_weight(w), b
        return self._prep.get("conv_seg", [conv.weight, conv.bias], build)

    # ---- forward
    def _check(self, x):
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"input must be [B, 3, H, W], got {tuple(x.shape)}")
        if x.shape[2] < 32 or x.shape[3] < 32:
            raise ValueError(f"{x.shape[2]} x {x.shape[3]}: the 1/32 level needs H, W >= 32")
        return device_input(self, x, self.backbone.norm1.weight)

    def _cblock(self, i, j, blk, x):
        sk = self.split_k
        x = ops.dwconv(x, *self._dw(("pos", i, j), blk.pos_embed), 3, residual=x)
        w1, b1 = self._conv1x1(("conv1", i, j), blk.conv1, blk.norm1)
        w2, b2 = self._conv1x1(("conv2", i, j), blk.conv2)
        t = ops.dwconv(ops.gemm(x, w1, bias=b1, split_k=sk), *self._dw(("dw5", i, j), blk.attn), 5)
        x = ops.gemm(t, w2, bias=b2, residual=x, split_k=sk)
        wf1, bf1 = self._conv1x1(("fc1", i, j), blk.mlp.fc1, blk.norm2)
        wf2, bf2 = self._conv1x1(("fc2", i, j), blk.mlp.fc2)
        h = ops.gemm(x, wf1, bias=bf1, split_k=sk)
        ops.gelu_(h)
        return ops.gemm(h, wf2, bias=bf2, residual=x, split_k=sk)

    def _sablock(self, i, j, blk, x):
        b, h, w, c = x.shape
        x = ops.dwconv(x, *self._dw(("pos", i, j), blk.pos_embed), 3, residual=x)
        y = run_layers([blk], self._prep, x.view(b * h * w, c), b, h * w, c // HEAD_DIM, "gelu", causal=False, f32=False,
                       weights=lambda prep, layer, _: vit_block_weights(prep, layer, (i, j)), split_k=self.split_k)
        return y.view(b, h, w, c)

    def _embed(self, i, x):
        """patch_embed{i}: the stride-k conv (odd sizes truncated) and its LayerNorm -> fp16 [B, h, w, C]"""
        pe = getattr(self.backbone, f"patch_embed{i}")
        if i == 1:
            b, _, hh, ww = x.shape
            h, w = hh // 4, ww // 4
            wk, bk = self._patch1()
            rows = ops.patch_gather_hw(x, 4, wk.shape[-1])
        else:
            b, hh, ww, _ = x.shape
            h, w = hh // 2, ww // 2
            wk, bk = self._patch(i)
            rows = ops.tap_gather_act(x, TAPS2, reflect=False, k_pad=wk.shape[-1], stride=2).view(b * h * w, -1)
        y = ops.gemm(rows, wk, bias=bk, split_k=self.split_k)
        return ops.layernorm_rows(y, *self._ln(("pe_norm", i), pe.norm)).view(b, h, w, -1)

    def _backbone(self, x):
        """(the four features fp16 [B, h_i, w_i, C_i], the PPM's concatenation buffer fp16 [B, h32, w32, 512 + 4 * 512]
        whose first 512 channels are the last feature)"""
        feats = []
        for i in (1, 2, 3, 4):
            x = self._embed(i, x)
            blocks = getattr(self.backbone, f"blocks{i}")
            for j, blk in enumerate(blocks):
                x = self._cblock(i, j, blk, x) if i <= 2 else self._sablock(i, j, blk, x)
            b, h, w, c = x.shape
            norm = self._ln(("norm", i), getattr(self.backbone, f"norm{i}"))
            if i == 4:
                cat5 = torch.empty((b, h, w, c + len(POOL_SCALES) * CHANNELS), device=x.device, dtype=torch.float16)
                ops.layernorm_rows(x.view(-1, c), *norm, out=cat5.view(b * h * w, -1)[:, :c])
                feats.append(cat5[..., :c])
            else:
                feats.append(ops.layernorm_rows(x.view(-1, c), *norm).view(b, h, w, c))
        return feats, cat5

    def _head(self, feats, cat5):
        dh = self.decode_head
        sk = self.split_k
        f4 = feats[3]
        b = f4.shape[0]
        for j, (s, rows) in enumerate(zip(POOL_SCALES, ops.adaptive_avg_pool(f4, POOL_SCALES))):
            wp, bp = self._cm(("ppm", j), dh.psp_modules[j][1])
            y = ops.gemm_relu(rows, wp, bias=bp, split_k=sk)
            lo = EMBED[-1] + j * CHANNELS
            ops.resize_bilinear(y.view(b, s, s, CHANNELS), out=cat5[..., lo:lo + CHANNELS])
        wb, bb = self._cm("bottleneck", dh.bottleneck)
        lats = []
        for i in range(3):
            wl, bl = self._cm(("lateral", i), dh.lateral_convs[i])
            lats.append(ops.gemm_relu(feats[i], wl, bias=bl, split_k=sk))
        lats.append(ops.gemm_relu(cat5, wb, ksize=3, bias=bb, split_k=sk))
        for i in (3, 2, 1):
            ops.resize_bilinear(lats[i], out=lats[i - 1], accumulate=True)
        _, h4, w4, _ = lats[0].shape
        cat4 = torch.empty((b, h4, w4, len(EMBED) * CHANNELS), device=f4.device, dtype=torch.float16)
        for i in range(3):
            wf, bf = self._cm(("fpn", i), dh.fpn_convs[i])
            dst = cat4[..., i * CHANNELS:(i + 1) * CHANNELS]
            if i == 0:
                ops.gemm_relu(lats[0], wf, ksize=3, bias=bf, out=dst, split_k=sk)
            else:
                ops.resize_bilinear(ops.gemm_relu(lats[i], wf, ksize=3, bias=bf, split_k=sk), out=dst)
        ops.resize_bilinear(lats[3], out=cat4[..., 3 * CHANNELS:])
        wfb, bfb = self._cm("fpn_bottleneck", dh.fpn_bottleneck)
        y = ops.gemm_relu(cat4, wfb, ksize=3, bias=bfb, split_k=sk)
        ws, bs = self._seg()
        return ops.gemm(y, ws, bias=bs, out_f32=True, split_k=sk)

    def _run(self, x):
        """(fp32 logits [B, H4, W4, LOGIT_LD] whose channels beyond num_classes are zero, the four features)"""
        feats, cat5 = self._backbone(self._check(x))
        return self._head(feats, cat5), feats

    @torch.no_grad()
    def forward(self, x):
        return self._run(x)[0][..., :NUM_CLASSES]

    @torch.no_grad()
    def forward_stages(self, x):
        """(logits as forward returns them, {"features": the four backbone outputs after norm1..4, fp16 [B, h, w, C]})"""
        logits, feats = self._run(x)
        return logits[..., :NUM_CLASSES], {"features": feats}


def network_input(img):
    """UniformerDetector's network input for an HWC uint8 RGB image: cv2 INTER_LINEAR to rescale_size (mmcv.imrescale),
    as fp32 [1, 3, h, w] RGB values (Normalize is folded into patch_embed1)"""
    h, w = img.shape[:2]
    nh, nw = rescale_size(h, w)
    x = cv2.resize(np.ascontiguousarray(img), (nw, nh), interpolation=cv2.INTER_LINEAR)
    return torch.from_numpy(x).permute(2, 0, 1).unsqueeze(0).float().contiguous()


class UniformerDetector:
    """The reference's UniformerDetector: __call__(HWC uint8 RGB image) -> uint8 [H, W, 3] RGB segmentation map,
    palette[label] per pixel, from upernet_global_small.pth in `ckpt_dir` (default: the reference's checkpoint
    directory).  Nothing is downloaded."""

    def __init__(self, ckpt_dir=None, device="cuda"):
        self.device = device
        path = checkpoint_path(ckpt_dir, CKPT_NAME)
        self.model = UniformerSegmentor().to(device)
        self.model.load(path)

    def __call__(self, img):
        assert img.ndim == 3 and img.shape[2] == 3
        x = network_input(img)
        logits, _ = self.model._run(x.to(self.device))
        rgb = ops.seg_output(logits, NUM_CLASSES, tuple(x.shape[2:]), img.shape[:2], self.model.palette)
        return rgb[0].cpu().numpy()
