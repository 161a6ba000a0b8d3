"""Drop-in for the reference's `ldm/modules/diffusionmodules/openaimodel.py`: TimestepEmbedSequential, ResBlock,
Down/Upsample and UNetModel with the reference's constructor kwargs, attribute tree and state-dict keys.

Kernel sequence of one ResBlock (reference ResBlock._forward :254-274):
    groupnorm+SiLU -> conv3x3 implicit GEMM (+bias + time-embedding row term) -> groupnorm+SiLU ->
    conv3x3 implicit GEMM (+bias + skip: residual read, or the 1x1 skip conv accumulated into the same accumulator tile)
Decoder blocks take their `cat([h, hs.pop() + control.pop()], 1)` input as a CatSpec: the first GroupNorm reads the
pieces in place.
"""
from abc import abstractmethod

import torch
import torch.nn as nn

from ctrlora_b200 import ops, prepare
from ctrlora_b200.runtime import CatSpec, EmbPack, nchw_view, pixel_major, to_f16_rows
from ldm.modules.attention import SpatialTransformer
from ldm.modules.diffusionmodules.util import (checkpoint, conv_nd, linear, normalization,  # noqa: F401
                                               timestep_embedding, zero_module)
from ldm.util import exists  # noqa: F401


def convert_module_to_f16(x):
    pass


def convert_module_to_f32(x):
    pass


class TimestepBlock(nn.Module):
    """Any module where forward() takes timestep embeddings as a second argument."""

    @abstractmethod
    def forward(self, x, emb):
        """Apply the module to `x` given `emb` timestep embeddings."""


class TimestepEmbedSequential(nn.Sequential, TimestepBlock):
    """Sequential that routes (x, emb) to TimestepBlocks and (x, context) to SpatialTransformers (reference :73-87).
    `other` / `emb_other`: the same block of a second network and that network's time embedding; each layer then runs
    on the lower half of the batch and its partner in `other` on the upper half, in the same launches."""

    def forward(self, x, emb, context=None, other=None, emb_other=None):
        for i, layer in enumerate(self):
            pair = {} if other is None else {"other": other[i]}
            if isinstance(layer, TimestepBlock):
                x = layer(x, emb, emb_other=emb_other, **pair)
            elif isinstance(layer, SpatialTransformer):
                x = layer(x, context, **pair)
            else:
                x = layer(x, **pair)
        return x


class _Conv(nn.Conv2d):
    """nn.Conv2d parameter holder whose forward is the wgmma implicit GEMM (3x3 pad 1 / 1x1, stride 1)."""

    def _cache(self):
        c = self.__dict__.get("_prep")
        if c is None:
            c = self.__dict__["_prep"] = prepare.PrepCache()
        return c

    def kernel_weight(self, pad_in=None, pad_out=None):
        return self._cache().get(("w", pad_in, pad_out), [self.weight],
                                 lambda: prepare.conv_weight(self.weight, pad_in, pad_out))

    def forward(self, x):
        k = self.kernel_size[0]
        if self.stride != (1, 1) or self.padding != ((k - 1) // 2,) * 2 or k not in (1, 3):
            raise NotImplementedError("only 1x1 and 3x3 stride-1 'same' convolutions are on the CtrLoRA path")
        cin = self.in_channels
        c_pad = (cin + 7) // 8 * 8
        xp = pixel_major(x, c_pad if c_pad != cin else None)
        w = self.kernel_weight(pad_in=c_pad if c_pad != cin else None)
        return nchw_view(ops.gemm(xp, w, ksize=k, bias=prepare.bias_f32(self.bias)))


def _conv2d(*args, **kwargs):
    return _Conv(*args, **kwargs)


class Upsample(nn.Module):
    """nearest x2 then conv3x3 (reference :90-118)."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.dims = dims
        if dims != 2 or not use_conv:
            raise NotImplementedError("Upsample: dims=2 with conv only (conv_resample=True)")
        self.conv = _conv2d(self.channels, self.out_channels, 3, padding=padding)

    def forward(self, x):
        assert x.shape[1] == self.channels
        up = ops.upsample2x(pixel_major(x).contiguous())
        return self.conv(nchw_view(up))


class Downsample(nn.Module):
    """conv3x3 stride 2 pad 1 (reference :133-159): stride-2 gather kernel + plain GEMM over K = 9*C."""

    def __init__(self, channels, use_conv, dims=2, out_channels=None, padding=1):
        super().__init__()
        self.channels = channels
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.dims = dims
        if dims != 2 or not use_conv or padding != 1:
            raise NotImplementedError("Downsample: dims=2, conv, padding=1 only (conv_resample=True)")
        self.op = nn.Conv2d(self.channels, self.out_channels, 3, stride=2, padding=padding)
        self._prep = prepare.PrepCache()

    def _weight(self):
        return self._prep.get("w", [self.op.weight],
                              lambda: prepare.conv_weight(self.op.weight).view(self.out_channels, 1, 9 * self.channels))

    def run(self, xp, out=None, other=None):
        """pixel-major fp16 [B, H, W, C] -> [B, H/2, W/2, Cout] (into `out` if given); `other`: the same layer of a
        second network, applied to the upper half of the batch in the same launch."""
        col = ops.im2col_s2(xp.contiguous())  # [B, H/2, W/2, 9*C]
        hi = None if other is None else {"w": other._weight(), "bias": prepare.bias_f32(other.op.bias)}
        return ops.gemm(col, self._weight(), bias=prepare.bias_f32(self.op.bias), out=out, hi=hi)

    def forward(self, x, other=None):
        assert x.shape[1] == self.channels
        return nchw_view(self.run(pixel_major(x), other=other))


class ResBlock(TimestepBlock):
    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False, use_scale_shift_norm=False,
                 dims=2, use_checkpoint=False, up=False, down=False):
        super().__init__()
        if use_scale_shift_norm or up or down or dims != 2 or dropout != 0:
            raise NotImplementedError("ResBlock: scale-shift norm / resblock_updown / dropout are not on the CtrLoRA path")
        self.channels = channels
        self.emb_channels = emb_channels
        self.dropout = dropout
        self.out_channels = out_channels or channels
        self.use_conv = use_conv
        self.use_checkpoint = use_checkpoint
        self.use_scale_shift_norm = use_scale_shift_norm
        self.in_layers = nn.Sequential(normalization(channels), nn.SiLU(),
                                       nn.Conv2d(channels, self.out_channels, 3, padding=1))
        self.updown = False
        self.h_upd = self.x_upd = nn.Identity()
        self.emb_layers = nn.Sequential(nn.SiLU(), linear(emb_channels, self.out_channels))
        self.out_layers = nn.Sequential(normalization(self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
                                        zero_module(nn.Conv2d(self.out_channels, self.out_channels, 3, padding=1)))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        elif use_conv:
            raise NotImplementedError("ResBlock use_conv=True (3x3 skip) is not on the CtrLoRA path")
        else:
            self.skip_connection = nn.Conv2d(channels, self.out_channels, 1)
        self._prep = prepare.PrepCache()

    def _kernel_params(self):
        """the prepared operands of the block's kernels: GroupNorm affines, conv weights and biases"""
        f32 = prepare.bias_f32
        gn1, conv1 = self.in_layers[0], self.in_layers[2]
        gn2, conv2 = self.out_layers[0], self.out_layers[3]
        k = {"gn1": (f32(gn1.weight), f32(gn1.bias), gn1.eps), "gn2": (f32(gn2.weight), f32(gn2.bias), gn2.eps),
             "w1": self._prep.get("w1", [conv1.weight], lambda: prepare.conv_weight(conv1.weight)), "b1": f32(conv1.bias),
             "w2": self._prep.get("w2", [conv2.weight], lambda: prepare.conv_weight(conv2.weight)), "wsk": None,
             "b2": f32(conv2.bias)}
        if not isinstance(self.skip_connection, nn.Identity):
            sk = self.skip_connection
            k["wsk"] = self._prep.get("wsk", [sk.weight], lambda: prepare.conv_weight(sk.weight).view(self.out_channels, -1))
            k["b2"] = self._prep.get("bsum", [conv2.bias, sk.bias], lambda: (conv2.bias.float() + sk.bias.float()).contiguous())
        return k

    def _rowbias(self, emb):
        """time-embedding term: a slice of the network's batched GEMV, or this block's own small linear"""
        if isinstance(emb, EmbPack):
            rowbias = emb.slices.get(id(self))
            raw = emb.raw
        else:
            rowbias, raw = None, emb
        if rowbias is None:
            lin = self.emb_layers[1]
            rowbias = ops.small_linear(raw.float().contiguous(), self.emb_weight(), prepare.bias_f32(lin.bias), silu_in=True)
        return rowbias

    def emb_weight(self):
        lin = self.emb_layers[1]
        return self._prep.get("emb", prepare.linear_params(lin),
                              lambda: prepare.effective_linear_weight(lin).view(lin.out_features, lin.in_features))

    def forward(self, x, emb, other=None, emb_other=None):
        """`other` / `emb_other`: the same block of a second network and that network's time embedding, applied to the
        upper half of the batch in the same launches."""
        k = self._kernel_params()
        o = None if other is None else other._kernel_params()
        (g1, b1, eps1), (g2, b2, eps2) = k["gn1"], k["gn2"]
        hi1, hi2 = ({}, {}) if o is None else ({"gamma_hi": o["gn1"][0], "beta_hi": o["gn1"][1]},
                                               {"gamma_hi": o["gn2"][0], "beta_hi": o["gn2"][1]})
        if isinstance(x, CatSpec):  # the decoder's concatenated input, read in place
            x1 = pixel_major(x.x1)
            a, xp = ops.groupnorm(x1, g1, b1, eps1, True,
                                  add1=None if x.add1 is None else pixel_major(x.add1), add1_scale=x.s1,
                                  x2=None if x.x2 is None else pixel_major(x.x2),
                                  add2=None if x.add2 is None else pixel_major(x.add2), add2_scale=x.s2,
                                  want_raw=True, **hi1)
        else:
            xp = pixel_major(x)
            a = ops.groupnorm(xp, g1, b1, eps1, True, **hi1)
        b, h, w, cin = xp.shape
        assert cin == self.channels, (cin, self.channels)
        hmid = ops.gemm(a, k["w1"], ksize=3, bias=k["b1"], rowbias=self._rowbias(emb),
                        hi=None if o is None else {"w": o["w1"], "bias": o["b1"], "rowbias": other._rowbias(emb_other)})
        c = ops.groupnorm(hmid, g2, b2, eps2, True, **hi2)
        hi = None if o is None else {"w": o["w2"], "bias": o["b2"], "w2": o["wsk"]}
        if k["wsk"] is not None:
            out = ops.gemm(c, k["w2"], ksize=3, bias=k["b2"], a2=xp, w2=k["wsk"], hi=hi)
        else:
            out = ops.gemm(c, k["w2"], ksize=3, bias=k["b2"], residual=xp.view(b * h * w, cin), hi=hi)
        return nchw_view(out)


class AttentionBlock(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError("legacy AttentionBlock (use_spatial_transformer=False) is not on the CtrLoRA path")


def count_flops_attn(model, _x, y):
    raise NotImplementedError


class UNetModel(nn.Module):
    """The SD UNet (reference :412-786) restricted to the options the CtrLoRA configs use; unsupported options raise."""

    transformer_cls = SpatialTransformer  # openaimodel_ip.UNetModel swaps in the IP-Adapter variant

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, num_classes=None,
                 use_checkpoint=False, use_fp16=False, num_heads=-1, num_head_channels=-1, num_heads_upsample=-1,
                 use_scale_shift_norm=False, resblock_updown=False, use_new_attention_order=False,
                 use_spatial_transformer=False, transformer_depth=1, context_dim=None, n_embed=None, legacy=True,
                 disable_self_attentions=None, num_attention_blocks=None, disable_middle_self_attn=False,
                 use_linear_in_transformer=False):
        super().__init__()
        if not use_spatial_transformer or context_dim is None:
            raise NotImplementedError("UNetModel: use_spatial_transformer=True with a context_dim is required")
        if num_classes is not None or n_embed is not None or resblock_updown or use_scale_shift_norm or dims != 2:
            raise NotImplementedError("UNetModel: option outside the CtrLoRA configs")
        if isinstance(context_dim, (list, tuple)) or type(context_dim).__name__ == "ListConfig":
            context_dim = list(context_dim)
        if num_heads_upsample == -1:
            num_heads_upsample = num_heads
        if num_heads == -1 and num_head_channels == -1:
            raise ValueError("Either num_heads or num_head_channels has to be set")
        self.image_size = image_size
        self.in_channels = in_channels
        self.model_channels = model_channels
        self.out_channels = out_channels
        self.num_res_blocks = len(channel_mult) * [num_res_blocks] if isinstance(num_res_blocks, int) else list(num_res_blocks)
        self.attention_resolutions = list(attention_resolutions)
        self.dropout = dropout
        self.channel_mult = tuple(channel_mult)
        self.conv_resample = conv_resample
        self.num_classes = num_classes
        self.use_checkpoint = use_checkpoint
        self.dtype = torch.float32  # the module-boundary dtype of the reference (use_fp16 unset); kernels run fp16
        self.num_heads = num_heads
        self.num_head_channels = num_head_channels
        self.num_heads_upsample = num_heads_upsample
        self.predict_codebook_ids = False

        def heads_of(ch):
            if num_head_channels == -1:
                return num_heads, ch // num_heads
            return ch // num_head_channels, num_head_channels

        def transformer(ch, level_idx=None, disable_sa=False):
            nh, dh = heads_of(ch)
            if legacy:
                dh = ch // nh
            return type(self).transformer_cls(ch, nh, dh, depth=transformer_depth, context_dim=context_dim,
                                              disable_self_attn=disable_sa, use_linear=use_linear_in_transformer,
                                              use_checkpoint=use_checkpoint)

        def resblock(cin, cout):
            return ResBlock(cin, time_embed_dim, dropout, out_channels=cout, dims=dims, use_checkpoint=use_checkpoint,
                            use_scale_shift_norm=use_scale_shift_norm)

        time_embed_dim = model_channels * 4
        self.time_embed = nn.Sequential(linear(model_channels, time_embed_dim), nn.SiLU(),
                                        linear(time_embed_dim, time_embed_dim))
        self.input_blocks = nn.ModuleList([TimestepEmbedSequential(_conv2d(in_channels, model_channels, 3, padding=1))])
        self._feature_size = model_channels
        skip_chans = [model_channels]
        ch, ds = model_channels, 1
        for level, mult in enumerate(self.channel_mult):
            for nr in range(self.num_res_blocks[level]):
                layers = [resblock(ch, mult * model_channels)]
                ch = mult * model_channels
                if ds in self.attention_resolutions:
                    dsa = disable_self_attentions[level] if exists(disable_self_attentions) else False
                    if not exists(num_attention_blocks) or nr < num_attention_blocks[level]:
                        layers.append(transformer(ch, disable_sa=dsa))
                self.input_blocks.append(TimestepEmbedSequential(*layers))
                skip_chans.append(ch)
            if level != len(self.channel_mult) - 1:
                self.input_blocks.append(TimestepEmbedSequential(Downsample(ch, conv_resample, dims=dims, out_channels=ch)))
                skip_chans.append(ch)
                ds *= 2
        self.middle_block = TimestepEmbedSequential(resblock(ch, ch), transformer(ch, disable_sa=disable_middle_self_attn),
                                                    resblock(ch, ch))
        self.output_blocks = nn.ModuleList([])
        for level, mult in list(enumerate(self.channel_mult))[::-1]:
            for i in range(self.num_res_blocks[level] + 1):
                ich = skip_chans.pop()
                layers = [resblock(ch + ich, model_channels * mult)]
                ch = model_channels * mult
                if ds in self.attention_resolutions:
                    dsa = disable_self_attentions[level] if exists(disable_self_attentions) else False
                    if not exists(num_attention_blocks) or i < num_attention_blocks[level]:
                        layers.append(transformer(ch, disable_sa=dsa))
                if level and i == self.num_res_blocks[level]:
                    layers.append(Upsample(ch, conv_resample, dims=dims, out_channels=ch))
                    ds //= 2
                self.output_blocks.append(TimestepEmbedSequential(*layers))
        self.out = nn.Sequential(normalization(ch), nn.SiLU(), zero_module(_conv2d(model_channels, out_channels, 3, padding=1)))
        self._prep = prepare.PrepCache()

    def convert_to_fp16(self):
        pass

    def convert_to_fp32(self):
        pass

    # ---- fused helpers shared with ControlNet (cldm/cldm.py) -----------------------------------------------------
    def _resblocks(self):
        return [m for m in self.modules() if isinstance(m, ResBlock)]

    def embed(self, timesteps, out_raw=None, out_all=None):
        """timestep_embedding -> time_embed MLP -> every ResBlock's emb_layers, as three launches (reference: one
        Linear per ResBlock, openaimodel.py:263; the ControlNet's are LoRA-wrapped, cldm_ctrlora_finetune.py:21-38).
        out_raw / out_all: optional fp32 destination rows ([B, 1280] / [B, sum Cout], row strides free)."""
        f32 = prepare.bias_f32
        t_emb = timestep_embedding(timesteps, self.model_channels)
        l0, l2 = self.time_embed[0], self.time_embed[2]
        w0 = self._prep.get("te0", prepare.linear_params(l0), lambda: prepare.effective_linear_weight(l0).view(l0.out_features, -1))
        w2 = self._prep.get("te2", prepare.linear_params(l2), lambda: prepare.effective_linear_weight(l2).view(l2.out_features, -1))
        hid = ops.small_linear(t_emb, w0, f32(l0.bias), silu_out=True)
        emb = ops.small_linear(hid, w2, f32(l2.bias), out=out_raw)
        blocks = self._resblocks()
        lins = [b.emb_layers[1] for b in blocks]
        params = [p for lin in lins for p in prepare.linear_params(lin)] + [lin.bias for lin in lins]
        wcat, bcat = self._prep.get("emb_cat", params, lambda: (
            torch.cat([b.emb_weight() for b in blocks], 0).contiguous(),
            torch.cat([lin.bias.detach().float() for lin in lins], 0).contiguous()))
        allout = ops.small_linear(emb, wcat, bcat, silu_in=True, out=out_all)  # [B, sum Cout]
        slices, off = {}, 0
        for b in blocks:
            slices[id(b)] = allout[:, off:off + b.out_channels]
            off += b.out_channels
        return EmbPack(emb, slices)

    def final(self, h):
        """out = GroupNorm32 -> SiLU -> conv3x3 (reference :726-730, :786): fp32 NCHW result like the reference's."""
        gn, conv = self.out[0], self.out[2]
        hp = pixel_major(h)
        a = ops.groupnorm(hp, prepare.bias_f32(gn.weight), prepare.bias_f32(gn.bias), gn.eps, True)
        n_pad = (self.out_channels + 15) // 16 * 16
        w = conv.kernel_weight(pad_out=n_pad)
        bias = self._prep.get("out_bias", [conv.bias], lambda: torch.cat(
            [conv.bias.detach().float(), torch.zeros(n_pad - self.out_channels, device=conv.bias.device)]).contiguous())
        y = ops.gemm(a, w, ksize=3, bias=bias, out_f32=True)  # [B, H, W, n_pad] fp32
        return ops.nhwc_to_nchw_f32(y, self.out_channels)

    def forward(self, x, timesteps=None, context=None, y=None, **kwargs):
        assert y is None, "class-conditional UNets are not on the CtrLoRA path"
        hs = []
        emb = self.embed(timesteps)
        from ctrlora_b200.runtime import context_f16
        ctx = context_f16(context)
        h = x
        for module in self.input_blocks:
            h = module(h, emb, ctx)
            hs.append(h)
        h = self.middle_block(h, emb, ctx)
        for module in self.output_blocks:
            h = module(CatSpec(h, x2=hs.pop()), emb, ctx)
        return self.final(h)
