"""Drop-in for the reference's `ldm/modules/diffusionmodules/model.py`: the first-stage VAE's `Encoder` / `Decoder`
(and their `ResnetBlock`, `AttnBlock`, `Downsample`, `Upsample`) with the reference's constructor kwargs, attribute tree
and state-dict keys, evaluated on the same sm_90a kernels as the UNet (SURVEY.md §8 rows f1 / f3).

Why it is on the path: every CtrLoRA `apply_model` starts with `0.18215 * VAE.encode(hint).sample()`
(cldm/cldm_ctrlora_finetune.py:76-77) -- 1117 GFLOP per 512x512 image, more than the ControlNet + UNet pass it feeds.

Kernel sequence (all pixel-major fp16, fp32 accumulation / statistics):
    ResnetBlock   groupnorm(eps 1e-6)+swish -> conv3x3 implicit GEMM -> groupnorm+swish -> conv3x3 (+ identity residual, or the
                  1x1 nin_shortcut accumulated into the same accumulator tile)                        reference :129-149
    Downsample    F.pad(0,1,0,1) + conv3x3 stride 2 = right/bottom-padded stride-2 gather + plain GEMM      :80-84
    Upsample      nearest x2 + conv3x3                                                                       :61-65
    AttnBlock     groupnorm -> one [q|k|v] GEMM (V stored transposed) -> per image: fp32 logits GEMM (q k^T), row softmax,
                  P V GEMM -> proj_out (+ residual).  Single head with d = C = 512: the d <= 160 flash kernels do not apply;
                  the N x N matrix exists here (fp32 64 MiB per image at 64x64) exactly as in the reference   :179-203
"""
import numpy as np
import torch
import torch.nn as nn

from ctrlora_b200 import ops, prepare
from ctrlora_b200.runtime import nchw_view, pixel_major
from ldm.modules.diffusionmodules.openaimodel import _Conv

f32 = prepare.bias_f32


def nonlinearity(x):
    """swish (reference :41-43); the networks below apply it inside the GroupNorm kernel."""
    return x * torch.sigmoid(x)


def Normalize(in_channels, num_groups=32):
    return nn.GroupNorm(num_groups=num_groups, num_channels=in_channels, eps=1e-6, affine=True)


def _gn(norm, xp, silu):
    return ops.groupnorm(xp, f32(norm.weight), f32(norm.bias), norm.eps, silu, groups=norm.num_groups)


class Upsample(nn.Module):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if self.with_conv:
            self.conv = _Conv(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def forward(self, x):
        up = nchw_view(ops.upsample2x(pixel_major(x).contiguous()))
        return self.conv(up) if self.with_conv else up


class Downsample(nn.Module):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if not with_conv:
            raise NotImplementedError("avg-pool downsampling (resamp_with_conv=False) is not used by the SD VAE")
        self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)
        self._prep = prepare.PrepCache()

    def forward(self, x):
        xp = pixel_major(x).contiguous()
        c = xp.shape[-1]
        col = ops.im2col_s2(xp, pad_lo=0)  # zeros on the right / bottom only: F.pad(x, (0, 1, 0, 1))
        wk = self._prep.get("w", [self.conv.weight], lambda: prepare.conv_weight(self.conv.weight).view(-1, 1, 9 * c))
        return nchw_view(ops.gemm(col, wk, bias=f32(self.conv.bias)))


class ResnetBlock(nn.Module):
    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout, temb_channels=512):
        super().__init__()
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.use_conv_shortcut = conv_shortcut
        if dropout != 0.0:
            raise NotImplementedError("dropout > 0 is not used by the SD VAE")
        self.norm1 = Normalize(in_channels)
        self.conv1 = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if temb_channels > 0:
            self.temb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = Normalize(out_channels)
        self.dropout = nn.Dropout(dropout)
        self.conv2 = nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            if self.use_conv_shortcut:
                self.conv_shortcut = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
            else:
                self.nin_shortcut = nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)
        self._prep = prepare.PrepCache()

    def _w(self, key, conv):
        return self._prep.get(key, [conv.weight], lambda: prepare.conv_weight(conv.weight))

    def forward(self, x, temb=None):
        if temb is not None:
            raise NotImplementedError("timestep-conditioned ResnetBlocks belong to the (unused) `Model` class, not the VAE")
        xp = pixel_major(x)
        b, h, w, cin = xp.shape
        a = _gn(self.norm1, xp, True)
        hmid = ops.gemm(a, self._w("w1", self.conv1), ksize=3, bias=f32(self.conv1.bias))
        c = _gn(self.norm2, hmid, True)
        w2 = self._w("w2", self.conv2)
        if self.in_channels == self.out_channels:
            out = ops.gemm(c, w2, ksize=3, bias=f32(self.conv2.bias), residual=xp.reshape(b * h * w, cin))
        elif self.use_conv_shortcut:
            sk = ops.gemm(xp, self._w("wsk3", self.conv_shortcut), ksize=3, bias=f32(self.conv_shortcut.bias))
            out = ops.gemm(c, w2, ksize=3, bias=f32(self.conv2.bias), residual=sk.view(b * h * w, -1))
        else:
            sk = self.nin_shortcut
            wsk = self._prep.get("wsk", [sk.weight], lambda: prepare.conv_weight(sk.weight).view(self.out_channels, cin))
            bsum = self._prep.get("bsum", [self.conv2.bias, sk.bias],
                                  lambda: (self.conv2.bias.float() + sk.bias.float()).contiguous())
            out = ops.gemm(c, w2, ksize=3, bias=bsum, a2=xp, w2=wsk)
        return nchw_view(out)


class AttnBlock(nn.Module):
    """Single-head spatial self-attention with d = in_channels (reference :152-203)."""

    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.k = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.v = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.proj_out = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self._prep = prepare.PrepCache()

    def forward(self, x):
        xp = pixel_major(x)
        b, h, w, c = xp.shape
        n = h * w
        if n % 8:
            raise NotImplementedError("AttnBlock needs H*W to be a multiple of 8")
        dev = xp.device
        xn = _gn(self.norm, xp, False)
        convs = (self.q, self.k, self.v)
        wqkv, bqkv = self._prep.get("qkv", [m.weight for m in convs] + [m.bias for m in convs], lambda: (
            torch.cat([prepare.conv_weight(m.weight) for m in convs], 0).contiguous(),
            torch.cat([m.bias.detach().float() for m in convs], 0).contiguous()))
        q = torch.empty((b * n, c), device=dev, dtype=torch.float16)
        k = torch.empty_like(q)
        vt = torch.empty((b, 1, c, n), device=dev, dtype=torch.float16)  # V transposed per image: [C, tokens]
        ops.gemm(xn.view(b * n, c), wqkv, bias=bqkv, seg_outs=[q, k, vt], seg_width=c, transposed=(0, 0, 1), rows_per_img=n,
                 head_dim=c, tok_pad=n)
        o = torch.empty((b * n, c), device=dev, dtype=torch.float16)
        logits = torch.empty((n, n), device=dev, dtype=torch.float32)
        scale = float(int(c) ** (-0.5))
        for i in range(b):
            qi, ki = q[i * n:(i + 1) * n], k[i * n:(i + 1) * n]
            ops.gemm(qi, ki.view(n, 1, c), out=logits, out_f32=True)              # w_[i, j] = q_i . k_j   (fp32)
            p = ops.softmax_rows(logits, scale)                                    # softmax over keys j
            ops.gemm(p, vt[i].view(c, 1, n), out=o[i * n:(i + 1) * n])            # h_[i, :] = sum_j p[i, j] v_j
        wo = self._prep.get("o", [self.proj_out.weight], lambda: prepare.conv_weight(self.proj_out.weight))
        out = ops.gemm(o.view(b, h, w, c), wo, bias=f32(self.proj_out.bias), residual=xp.reshape(b * n, c))
        return nchw_view(out)


MemoryEfficientAttnBlock = AttnBlock  # the xformers variant (reference :205-268) computes the same function


def make_attn(in_channels, attn_type="vanilla", attn_kwargs=None):
    if attn_type in ("vanilla", "vanilla-xformers"):
        return AttnBlock(in_channels)
    if attn_type == "none":
        return nn.Identity(in_channels)
    raise NotImplementedError(f"attn_type {attn_type!r} is not used by the SD VAE")


class _Tail:
    """norm_out -> swish -> conv_out shared by Encoder / Decoder: fp32 NCHW result like the reference's.  `post` = an
    optional (weight [O, C_out], bias [O]) 1x1 map composed INTO conv_out in fp32 (AutoencoderKL.encode folds quant_conv in,
    so the 2z-channel moments never round to fp16 in between)."""

    @staticmethod
    def run(mod, h, post=None, key="tail"):
        hp = pixel_major(h)
        a = _gn(mod.norm_out, hp, True)
        conv = mod.conv_out
        params = [conv.weight, conv.bias] + ([post[0], post[1]] if post is not None else [])

        def build():
            wt, bs = conv.weight.detach().float(), conv.bias.detach().float()
            if post is not None:
                pw, pb = post[0].detach().float().view(post[0].shape[0], -1), post[1].detach().float()
                wt = torch.einsum("oj,jikl->oikl", pw, wt)
                bs = pw @ bs + pb
            n = wt.shape[0]
            n_pad = (n + 15) // 16 * 16
            wk = prepare.conv_weight(wt.contiguous(), pad_out=n_pad)
            bias = torch.cat([bs, torch.zeros(n_pad - n, device=bs.device)]).contiguous()
            return wk, bias, n

        wk, bias, n = mod._prep.get((key, post is not None), params, build)
        y = ops.gemm(a, wk, ksize=3, bias=bias, out_f32=True)
        return ops.nhwc_to_nchw_f32(y, n)


class Encoder(nn.Module):
    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="vanilla", **ignore_kwargs):
        super().__init__()
        if use_linear_attn:
            raise NotImplementedError("linear attention is not used by the SD VAE")
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.conv_in = _Conv(in_channels, self.ch, kernel_size=3, stride=1, padding=1)
        curr_res = resolution
        in_ch_mult = (1,) + tuple(ch_mult)
        self.in_ch_mult = in_ch_mult
        self.down = nn.ModuleList()
        block_in = ch
        for i_level in range(self.num_resolutions):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_in = ch * in_ch_mult[i_level]
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(make_attn(block_in, attn_type=attn_type))
            down = nn.Module()
            down.block = block
            down.attn = attn
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, resamp_with_conv)
                curr_res = curr_res // 2
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = make_attn(block_in, attn_type=attn_type)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, 2 * z_channels if double_z else z_channels, kernel_size=3, stride=1, padding=1)
        self._prep = prepare.PrepCache()

    def features(self, x):
        """everything before norm_out (reference :518-539)"""
        h = self.conv_in(x)
        for i_level in range(self.num_resolutions):
            for i_block in range(self.num_res_blocks):
                h = self.down[i_level].block[i_block](h, None)
                if len(self.down[i_level].attn) > 0:
                    h = self.down[i_level].attn[i_block](h)
            if i_level != self.num_resolutions - 1:
                h = self.down[i_level].downsample(h)
        h = self.mid.block_1(h, None)
        h = self.mid.attn_1(h)
        return self.mid.block_2(h, None)

    def forward(self, x, post=None):
        return _Tail.run(self, self.features(x), post)


class Decoder(nn.Module):
    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, give_pre_end=False, tanh_out=False,
                 use_linear_attn=False, attn_type="vanilla", **ignorekwargs):
        super().__init__()
        if use_linear_attn:
            raise NotImplementedError("linear attention is not used by the SD VAE")
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.give_pre_end = give_pre_end
        self.tanh_out = tanh_out
        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res)
        print("Working with z of shape {} = {} dimensions.".format(self.z_shape, np.prod(self.z_shape)))
        self.conv_in = _Conv(z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = make_attn(block_in, attn_type=attn_type)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=self.temb_ch, dropout=dropout)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks + 1):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(make_attn(block_in, attn_type=attn_type))
            up = nn.Module()
            up.block = block
            up.attn = attn
            if i_level != 0:
                up.upsample = Upsample(block_in, resamp_with_conv)
                curr_res = curr_res * 2
            self.up.insert(0, up)  # prepend to get consistent order
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)
        self._prep = prepare.PrepCache()

    def forward(self, z):
        self.last_z_shape = z.shape
        c_pad = (z.shape[1] + 7) // 8 * 8
        return self.run(pixel_major(z, c_pad if c_pad != z.shape[1] else None))

    def run(self, zp):
        """zp: pixel-major fp16 [B, h, w, Cp >= z_channels] (extra channels zero): what AutoencoderKL.decode's
        post_quant_conv GEMM leaves, so the latent never takes a detour through NCHW."""
        cp = zp.shape[-1]
        w_in = self.conv_in.kernel_weight(pad_in=cp if cp != self.conv_in.in_channels else None)
        h = nchw_view(ops.gemm(zp, w_in, ksize=3, bias=f32(self.conv_in.bias)))
        h = self.mid.block_1(h, None)
        h = self.mid.attn_1(h)
        h = self.mid.block_2(h, None)
        for i_level in reversed(range(self.num_resolutions)):
            for i_block in range(self.num_res_blocks + 1):
                h = self.up[i_level].block[i_block](h, None)
                if len(self.up[i_level].attn) > 0:
                    h = self.up[i_level].attn[i_block](h)
            if i_level != 0:
                h = self.up[i_level].upsample(h)
        if self.give_pre_end:
            return h
        out = _Tail.run(self, h)
        return torch.tanh(out) if self.tanh_out else out
