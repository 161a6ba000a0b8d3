"""The MiDaS depth annotator (annotator/midas/__init__.py MidasDetector, api.py MiDaSInference, midas/dpt_depth.py
DPTDepthModel with the ViT-L/16 of midas/vit.py and the fusion blocks of midas/blocks.py) on the sm_90a kernels.

Switching a caller over is an import swap: `from ctrlora_b200.annotator.midas import MidasDetector`.  The modules keep
the reference's tree (timm's VisionTransformer names under `pretrained.model`, `act_postprocess1..4`, `scratch.*`), so
`state_dict()` equals the reference's and dpt_large_384.pt loads with strict=True.  The nn modules hold the parameters
only; forward runs:

- the ViT: the 16 x 16 patch Conv2d as ctrlora_patch_gather_hw + one GEMM (K = 768), the cls token and the position
  table (the 24 x 24 grid resized to gh x gw with the reference's own F.interpolate, once per grid size) added by
  ctrlora_clip_vision_embed, then text_encoder.run_layers over the 24 blocks (pre-norm, eps 1e-6, fused q|k|v, full
  attention at d_head 64, exact GELU, fp32 residual stream), handing back the stream after blocks 5, 11, 17 and 23.
  The final `norm` is not run: forward_vit discards its output;
- the readout `GELU(Linear(cat(token, cls)))`: the cls half is a per-image row term (ctrlora_small_linear straight
  from the fp32 stream) added in the GEMM of the token half, then GELU in place;
- reassemble: 1x1 GEMMs; each ConvTranspose2d(kernel = stride = s) is one GEMM with N = s^2 C followed by
  ctrlora_depth_to_space_bias; the stride-2 Conv2d is im2col_s2 + GEMM;
- the fusion neck: every 3x3 conv is an implicit GEMM, RCU conv1 with the ReLU in its epilogue and conv2 with the skip
  as its residual; ctrlora_add_relu_f16 supplies relu(x) and the fusion sum with its ReLU.  Each block's 1x1 out_conv
  runs before the bilinear x2 upsample (ctrlora_upsample_bilinear2x_f16), not after: a 1x1 conv commutes with an
  interpolation whose weights sum to 1, and it then runs on a quarter of the pixels;
- the head: conv3x3, upsample, conv3x3 + ReLU on the GEMM, then ctrlora_midas_head_out_f16 (32 -> 1, bias, ReLU) into
  the fp32 depth [B, 16 gh, 16 gw].

Activations are fp16 pixel-major with fp32 accumulation.  Inference only, on the current stream.  The input's gh = H // 16
and gw = W // 16 must be even and >= 2 (otherwise the reference's stride-2 branch and x2 upsample disagree in size);
rows and columns beyond 16 gh, 16 gw are ignored, as the reference's patch conv ignores them.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops, prepare
from ..text_encoder import run_layers
from .common import SizeCache, checkpoint_path, device_input, freeze, vit_block_weights

HOOKS = (5, 11, 17, 23)             # vitl16_384's hooked blocks
FEATURES = (256, 512, 1024, 1024)   # reassemble widths
POS_CACHE_SIZES = 8                 # grid sizes whose resized position table is kept (least recently used goes first)
CKPT_NAME = "dpt_large_384.pt"


# ------------------------------------------------------------------------------------------------ the ViT (timm names)
class _PatchEmbed(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.proj = nn.Conv2d(3, dim, kernel_size=16, stride=16)


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


class _Block(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = _Attention(dim)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = _Mlp(dim, 4 * dim)


class _VisionTransformer(nn.Module):
    """timm's vit_large_patch16_384 parameters: 24 blocks of width 1024, 16 heads, a 24 x 24 position grid"""

    def __init__(self, dim=1024, depth=24, grid=24, num_classes=1000):
        super().__init__()
        self.patch_embed = _PatchEmbed(dim)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, grid * grid + 1, dim))
        self.blocks = nn.ModuleList(_Block(dim) for _ in range(depth))
        self.norm = nn.LayerNorm(dim, eps=1e-6)   # forward_flex's output is discarded by forward_vit: never run
        self.head = nn.Linear(dim, num_classes)   # timm's classifier: never run


class _ProjectReadout(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.project = nn.Sequential(nn.Linear(2 * dim, dim), nn.GELU())


def _postprocess(dim, feat, resize):
    """act_postprocessN: [readout, Transpose, Unflatten, Conv2d 1x1, resize]; the parameter-free slots are Identity"""
    mods = [_ProjectReadout(dim), nn.Identity(), nn.Identity(), nn.Conv2d(dim, feat, kernel_size=1)]
    if resize is not None:
        mods.append(resize)
    return nn.Sequential(*mods)


class _Pretrained(nn.Module):
    def __init__(self, dim=1024):
        super().__init__()
        self.model = _VisionTransformer(dim)
        f = FEATURES
        self.act_postprocess1 = _postprocess(dim, f[0], nn.ConvTranspose2d(f[0], f[0], kernel_size=4, stride=4))
        self.act_postprocess2 = _postprocess(dim, f[1], nn.ConvTranspose2d(f[1], f[1], kernel_size=2, stride=2))
        self.act_postprocess3 = _postprocess(dim, f[2], None)
        self.act_postprocess4 = _postprocess(dim, f[3], nn.Conv2d(f[3], f[3], kernel_size=3, stride=2, padding=1))


# ------------------------------------------------------------------------------------------------ scratch
class _RCU(nn.Module):
    def __init__(self, features):
        super().__init__()
        self.conv1 = nn.Conv2d(features, features, kernel_size=3, padding=1)
        self.conv2 = nn.Conv2d(features, features, kernel_size=3, padding=1)


class _Fusion(nn.Module):
    """FeatureFusionBlock_custom(features, ReLU(False), deconv=False, bn=False, expand=False, align_corners=True)"""

    def __init__(self, features):
        super().__init__()
        self.out_conv = nn.Conv2d(features, features, kernel_size=1)
        self.resConfUnit1 = _RCU(features)
        self.resConfUnit2 = _RCU(features)


class _Scratch(nn.Module):
    def __init__(self, features=256):
        super().__init__()
        for i, c in enumerate(FEATURES, 1):
            setattr(self, f"layer{i}_rn", nn.Conv2d(c, features, kernel_size=3, padding=1, bias=False))
        for i in range(1, 5):
            setattr(self, f"refinenet{i}", _Fusion(features))
        self.output_conv = nn.Sequential(
            nn.Conv2d(features, features // 2, kernel_size=3, padding=1), nn.Identity(),
            nn.Conv2d(features // 2, 32, kernel_size=3, padding=1), nn.ReLU(True),
            nn.Conv2d(32, 1, kernel_size=1), nn.ReLU(True), nn.Identity())


def load_checkpoint(path):
    """BaseModel.load's state dict: the file's dict, or its "model" entry when it also holds an "optimizer" """
    params = torch.load(path, map_location="cpu", weights_only=True)
    if "optimizer" in params:
        params = params["model"]
    return params


class DPTDepthModel(nn.Module):
    """The reference's DPTDepthModel(path, backbone="vitl16_384", non_negative=True) (readout "project", 256 features);
    forward(x fp32 [B, 3, H, W]) -> fp32 [B, 16 gh, 16 gw].  Other configurations raise NotImplementedError.
    split_k: passed to every GEMM (0 lets the tile model choose; 1 pins one plan per row, so a batch of B equals B
    batches of 1 bit for bit)."""

    def __init__(self, path=None, non_negative=True, backbone="vitl16_384", features=256, readout="project",
                 channels_last=False, use_bn=False):
        super().__init__()
        if backbone != "vitl16_384" or not non_negative or features != 256 or readout != "project" or use_bn:
            raise NotImplementedError("the sm_90a DPTDepthModel runs DPT-Large only: backbone='vitl16_384', "
                                      "non_negative=True, features=256, readout='project', use_bn=False")
        self.pretrained = _Pretrained()
        self.scratch = _Scratch(features)
        freeze(self)
        self.__dict__["_pos"] = SizeCache(POS_CACHE_SIZES)
        if path is not None:
            self.load(path)

    def load(self, path):
        self.load_state_dict(load_checkpoint(path), strict=True)

    # ---- kernel-layout weights
    def _lin(self, key, m):
        return self._prep.get(key, [m.weight, m.bias], lambda: (prepare.linear_weight(m.weight), prepare.bias_f32(m.bias)))

    def _conv(self, key, conv):
        """Conv2d -> (fp16 [Cout, 1, taps * Cin] tap-major, fp32 bias or None); 3x3 stride-1 convs keep [Cout, 9, Cin]"""
        def build():
            w = prepare.flat_conv_weight(conv.weight) if conv.stride != (1, 1) else prepare.conv_weight(conv.weight)
            return w, prepare.bias_f32(conv.bias)
        return self._prep.get(key, [conv.weight, conv.bias], build)

    def _patch(self):
        pe = self.pretrained.model.patch_embed.proj

        def build():
            return prepare.linear_weight(pe.weight.detach().reshape(pe.weight.shape[0], -1)), prepare.bias_f32(pe.bias)
        return self._prep.get("patch", [pe.weight, pe.bias], build)

    def _readout(self, k):
        """(fp16 [C, 1, C] token half, fp16 [C, C] cls half, fp32 bias) of act_postprocess{k}'s readout Linear"""
        lin = getattr(self.pretrained, f"act_postprocess{k}")[0].project[0]

        def build():
            c = lin.out_features
            w = lin.weight.detach()
            tok = prepare.linear_weight(w[:, :c].contiguous())
            cls = prepare.linear_weight(w[:, c:].contiguous()).view(c, c)
            return tok, cls, prepare.bias_f32(lin.bias)
        return self._prep.get(("readout", k), [lin.weight, lin.bias], build)

    def _convt(self, k):
        """ConvTranspose2d(C, C, s, stride s) [Cin, Cout, s, s] -> fp16 [s * s * Cout, 1, Cin], row (ky * s + kx) * Cout + co"""
        convt = getattr(self.pretrained, f"act_postprocess{k}")[4]

        def build():
            ci, co, s, _ = convt.weight.shape
            w = convt.weight.detach().float().permute(2, 3, 1, 0).reshape(s * s * co, ci).contiguous()
            return prepare.linear_weight(w), prepare.bias_f32(convt.bias)
        return self._prep.get(("convt", k), [convt.weight, convt.bias], build)

    def _head_out(self):
        conv = self.scratch.output_conv[4]
        return self._prep.get("head_out", [conv.weight, conv.bias],
                              lambda: (conv.weight.detach().float().reshape(-1).contiguous(), prepare.bias_f32(conv.bias)))

    def _f32(self, key, p):
        return self._prep.get(key, [p], lambda: prepare.bias_f32(p.detach().reshape(-1)))

    def pos_table(self, gh, gw):
        """fp32 [gh * gw + 1, C]: the reference's _resize_pos_embed (bilinear, align_corners=False) on the device; the last
        POS_CACHE_SIZES grid sizes are kept, and every entry is rebuilt when pos_embed changes"""
        pe = self.pretrained.model.pos_embed

        def build():
            posemb = pe.detach().float()
            tok, grid = posemb[:, :1], posemb[0, 1:]
            g = int(math.sqrt(len(grid)))
            grid = grid.reshape(1, g, g, -1).permute(0, 3, 1, 2)
            grid = F.interpolate(grid, size=(gh, gw), mode="bilinear")
            grid = grid.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)
            return torch.cat([tok, grid], dim=1)[0].contiguous()
        return self._pos.fetch((gh, gw), build, [pe])

    # ---- forward
    def grid(self, x):
        """(gh, gw) of input x, ValueError outside the reference's domain (before any launch)"""
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"input must be [B, 3, H, W], got {tuple(x.shape)}")
        gh, gw = x.shape[2] // 16, x.shape[3] // 16
        if gh < 2 or gw < 2 or gh % 2 or gw % 2:
            raise ValueError(f"{x.shape[2]} x {x.shape[3]}: H // 16 and W // 16 must be even and >= 2 (got {gh} x {gw}); "
                             "otherwise DPT's stride-2 reassemble branch and its x2 upsample disagree in size")
        return gh, gw

    def _check(self, x):
        gh, gw = self.grid(x)
        return device_input(self, x, self.pretrained.model.cls_token), gh, gw

    def _vit(self, x, gh, gw):
        """the residual stream after the hooked blocks: four fp32 [B * (P + 1), C]"""
        vit = self.pretrained.model
        b = x.shape[0]
        w_patch, b_patch = self._patch()
        rows = ops.patch_gather_hw(x, 16, w_patch.shape[-1])
        patch = ops.gemm(rows, w_patch, bias=b_patch, out_f32=True, split_k=self.split_k)
        h = ops.clip_vision_embed(patch, self._f32("cls", vit.cls_token), self.pos_table(gh, gw), b)
        _, kept = run_layers(vit.blocks[:HOOKS[-1] + 1], self._prep, h, b, gh * gw + 1, 16, "gelu", causal=False,
                             weights=vit_block_weights, keep=HOOKS, split_k=self.split_k)
        return kept

    def _reassemble(self, k, h, b, gh, gw):
        """act_postprocess{k} of one hooked stream -> fp16 [B, h_k, w_k, FEATURES[k - 1]]"""
        c = h.shape[1]
        p = gh * gw
        tok_w, cls_w, bias = self._readout(k)
        cls_term = ops.small_linear(h.view(b, (p + 1) * c)[:, :c], cls_w, bias)
        tok = ops.cast_rows(h.view(-1)[c:], b, p * c, (p + 1) * c).view(b * p, c)
        sk = self.split_k
        r = ops.gemm(tok, tok_w, rowbias=cls_term, rows_per_img=p, split_k=sk)
        ops.gelu_(r)
        post = getattr(self.pretrained, f"act_postprocess{k}")
        w1, b1 = self._conv(("post", k), post[3])
        y = ops.gemm(r.view(b, gh, gw, c), w1, bias=b1, split_k=sk)
        if k in (1, 2):
            wt, bt = self._convt(k)
            t = ops.gemm(y, wt, out_f32=True, split_k=sk)
            return ops.depth_to_space_bias(t, bt, post[4].stride[0])
        if k == 4:
            w4, b4 = self._conv(("post4s2", k), post[4])
            return ops.gemm(ops.im2col_s2(y, pad_lo=1), w4, bias=b4, split_k=sk)
        return y

    def _rcu_tail(self, key, unit, s, r):
        """conv2(relu(conv1(r))) + s, with r = relu(s)"""
        w1, b1 = self._conv(key + (1,), unit.conv1)
        w2, b2 = self._conv(key + (2,), unit.conv2)
        t = ops.gemm_relu(r, w1, ksize=3, bias=b1, split_k=self.split_k)
        return ops.gemm(t, w2, ksize=3, bias=b2, residual=s, split_k=self.split_k)

    def _fusion(self, i, x0, x1=None):
        """refinenet{i}(x0[, x1]) -> fp16 [B, 2h, 2w, 256]"""
        blk = getattr(self.scratch, f"refinenet{i}")
        if x1 is not None:
            u = self._rcu_tail(("rcu1", i), blk.resConfUnit1, x1, ops.add_relu(x1))
            s, r = ops.add_relu(x0, u)
        else:
            s, r = x0, ops.add_relu(x0)
        y = self._rcu_tail(("rcu2", i), blk.resConfUnit2, s, r)
        wo, bo = self._conv(("out_conv", i), blk.out_conv)
        return ops.upsample_bilinear2x(ops.gemm(y, wo, bias=bo, split_k=self.split_k))

    def _run(self, x, stages=None):
        x, gh, gw = self._check(x)
        b = x.shape[0]
        kept = self._vit(x, gh, gw)
        layers = [self._reassemble(k, h, b, gh, gw) for k, h in zip((1, 2, 3, 4), kept)]
        sk = self.split_k
        rn = [ops.gemm(layer, self._conv(("rn", k), getattr(self.scratch, f"layer{k}_rn"))[0], ksize=3, split_k=sk)
              for k, layer in zip((1, 2, 3, 4), layers)]
        path = self._fusion(4, rn[3])
        paths = [path]
        for i in (3, 2, 1):
            path = self._fusion(i, path, rn[i - 1])
            paths.append(path)
        oc = self.scratch.output_conv
        w0, b0 = self._conv("head0", oc[0])
        w2, b2 = self._conv("head2", oc[2])
        head = ops.gemm_relu(ops.upsample_bilinear2x(ops.gemm(path, w0, ksize=3, bias=b0, split_k=sk)), w2, ksize=3,
                             bias=b2, split_k=sk)
        wo, bo = self._head_out()
        depth = ops.midas_head_out(head, wo, bo)
        if stages is not None:
            stages.update(hooks=kept, layers=layers, rn=rn, paths=paths, head=head)
        return depth

    @torch.no_grad()
    def forward(self, x):
        return self._run(x)

    @torch.no_grad()
    def forward_stages(self, x):
        """(depth, {"hooks": the four hooked fp32 streams [B * (P + 1), C], "layers": the reassembled fp16 NHWC layer_1..4,
        "rn": layer1_rn..layer4_rn, "paths": refinenet4..1 outputs, "head": the head's last 32-channel activation})"""
        st = {}
        depth = self._run(x, stages=st)
        return depth, st


MODEL_TYPES = ("dpt_large", "dpt_hybrid", "midas_v21", "midas_v21_small")


class MiDaSInference(nn.Module):
    """The reference's MiDaSInference: `model` is the DPTDepthModel loaded from dpt_large_384.pt in `ckpt_dir` (default:
    the reference's checkpoint directory).  Only "dpt_large" is implemented; nothing is downloaded."""

    def __init__(self, model_type="dpt_large", ckpt_dir=None):
        super().__init__()
        if model_type not in MODEL_TYPES:
            raise ValueError(f"model_type {model_type!r} is not one of {MODEL_TYPES}")
        if model_type != "dpt_large":
            raise NotImplementedError(f"model_type {model_type!r}: only 'dpt_large' runs on the sm_90a kernels")
        path = checkpoint_path(ckpt_dir, CKPT_NAME)
        self.model = DPTDepthModel(path=path, backbone="vitl16_384", non_negative=True)

    def forward(self, x):
        return self.model(x)


class MidasDetector:
    """The reference's MidasDetector: __call__(HWC uint8 image, a=pi * 0.2, bg_th=0.02) -> (uint8 depth map, uint8
    normal map [.., 3]), both 16 gh x 16 gw.  The post-process runs on the device; only the two maps come back."""

    def __init__(self, ckpt_dir=None, device="cuda"):
        self.device = device
        self.model = MiDaSInference(model_type="dpt_large", ckpt_dir=ckpt_dir).to(device)

    def __call__(self, input_image, a=np.pi * 0.2, bg_th=0.02):
        assert input_image.ndim == 3
        # host side, as the reference computes it on the device: fp32 image / 127.5 - 1, 'h w c -> 1 c h w'
        x = (torch.from_numpy(np.ascontiguousarray(input_image)).float() / 127.5 - 1.0).permute(2, 0, 1).unsqueeze(0)
        self.model.model.grid(x)
        depth = self.model(x.contiguous().to(self.device))
        d8, n8 = ops.midas_maps(depth, np.float32(a), np.float32(bg_th))
        return d8[0].cpu().numpy(), n8[0].cpu().numpy()
