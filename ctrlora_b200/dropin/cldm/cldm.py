"""Drop-in for the reference's `cldm/cldm.py`: `ControlledUnetModel`, `ControlNet`, `ControlLDM`.

Data flow of one `apply_model` (reference :329-344 and cldm_ctrlora_finetune.py:67-82):
    ControlNet: 12 input blocks, each followed by its 1x1 zero-conv (a wgmma GEMM), middle block, middle_block_out
    -> 13 residuals (pixel-major fp16, returned as logical-NCHW views)
    UNet: encoder + middle, then for each decoder block the next ResBlock's GroupNorm kernel reads
    [h (+ s*c_mid) | hs_i + s_i*c_i] in place: the residual adds, the control_scales multiply and torch.cat of the
    reference (:34-42, finetune :79) are not separate passes over HBM.

Twin pass (ControlLDM._control_and_unet): the ControlNet and the UNet encoder have the same shapes layer for layer and
do not depend on each other, so sampling runs them as one batch-2B pass from the first Downsample on: images [0, B) are
the hint's, [B, 2B) x's, and each launch takes the ControlNet's weights for the lower half and the UNet's for the upper
half (grouped GEMM, GroupNorm and LayerNorm launches).  Every layer has one forward body; the UNet's layer, passed as
`other`, turns its launches into grouped ones.  The full-resolution blocks run at batch B per network.  The zero-convs
read the lower half, the decoder's skips are views of the upper half.  CTRLORA_TWIN_ENCODER=0 runs the two networks one
after the other.
"""
import os

import torch
import torch.nn as nn

from ctrlora_b200 import ops, prepare
from ctrlora_b200.runtime import CatSpec, Scaled, nchw_view, pixel_major, to_f16_rows, unwrap_scaled
from ldm.models.diffusion.ddpm import LatentDiffusion
from ldm.modules.attention import SpatialTransformer
from ldm.modules.diffusionmodules.openaimodel import (Downsample, ResBlock, TimestepEmbedSequential, UNetModel,  # noqa: F401
                                                      _Conv, _conv2d)
from ldm.modules.diffusionmodules.util import conv_nd, linear, timestep_embedding, zero_module  # noqa: F401
from ldm.util import exists, instantiate_from_config  # noqa: F401


def _ctx16(context):
    from ctrlora_b200.runtime import context_f16
    return context_f16(context)


class ControlledForward:
    """forward of ControlledUnetModel (reference cldm/cldm.py:22-45), shared with the IP-Adapter UNet of cldm/cldm_style.py"""

    @staticmethod
    def _context(context):
        return _ctx16(context)

    def forward(self, x, timesteps=None, context=None, control=None, only_mid_control=False, **kwargs):
        """`control`: list of 13 residual tensors (or runtime.Scaled pairs), consumed with pop() like the reference."""
        hs = []
        with torch.no_grad():  # the SD encoder never receives gradients (reference :25-32)
            emb = self.embed(timesteps)
            ctx = self._context(context)
            h = x
            for module in self.input_blocks:
                h = module(h, emb, ctx)
                hs.append(h)
            h = self.middle_block(h, emb, ctx)
        return self.decode(h, hs, emb, ctx, control, only_mid_control)

    def decode(self, h, hs, emb, ctx, control, only_mid_control):
        """the decoder half of forward: middle-block output h, encoder skips hs (consumed)"""
        add_mid, s_mid = (None, 1.0)
        if control is not None:
            add_mid, s_mid = unwrap_scaled(control.pop())
        for i, module in enumerate(self.output_blocks):
            skip = hs.pop()
            if only_mid_control or control is None:
                add, s = None, 1.0
            else:
                add, s = unwrap_scaled(control.pop())
            # `h += control.pop()` (reference :35) rides along as the addend of the first decoder block's input
            spec = CatSpec(h, add1=add_mid if i == 0 else None, s1=s_mid, x2=skip, add2=add, s2=s)
            h = module(spec, emb, ctx)
        return self.final(h)


class ControlledUnetModel(ControlledForward, UNetModel):
    pass


class ControlNet(nn.Module):
    """The ControlNet encoder copy (reference :48-305): same constructor kwargs and parameter names."""

    def __init__(self, image_size, in_channels, model_channels, hint_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, use_checkpoint=False, use_fp16=False,
                 num_heads=-1, num_head_channels=-1, num_heads_upsample=-1, use_scale_shift_norm=False,
                 resblock_updown=False, use_new_attention_order=False, use_spatial_transformer=False,
                 transformer_depth=1, context_dim=None, n_embed=None, legacy=True, disable_self_attentions=None,
                 num_attention_blocks=None, disable_middle_self_attn=False, use_linear_in_transformer=False):
        super().__init__()
        if not use_spatial_transformer or context_dim is None or dims != 2 or resblock_updown or use_scale_shift_norm:
            raise NotImplementedError("ControlNet: option outside the CtrLoRA configs")
        if type(context_dim).__name__ == "ListConfig":
            context_dim = list(context_dim)
        if num_heads == -1 and num_head_channels == -1:
            raise ValueError("Either num_heads or num_head_channels has to be set")
        self.dims = dims
        self.image_size = image_size
        self.in_channels = in_channels
        self.model_channels = model_channels
        self.num_res_blocks = len(channel_mult) * [num_res_blocks] if isinstance(num_res_blocks, int) else list(num_res_blocks)
        self.attention_resolutions = list(attention_resolutions)
        self.dropout = dropout
        self.channel_mult = tuple(channel_mult)
        self.conv_resample = conv_resample
        self.use_checkpoint = use_checkpoint
        self.dtype = torch.float32
        self.num_heads = num_heads
        self.num_head_channels = num_head_channels
        self.num_heads_upsample = num_heads if num_heads_upsample == -1 else num_heads_upsample
        self.predict_codebook_ids = n_embed is not None

        time_embed_dim = model_channels * 4
        self.time_embed = nn.Sequential(linear(model_channels, time_embed_dim), nn.SiLU(),
                                        linear(time_embed_dim, time_embed_dim))

        def transformer(ch, disable_sa=False):
            if num_head_channels == -1:
                nh, dh = num_heads, ch // num_heads
            else:
                nh, dh = ch // num_head_channels, num_head_channels
            if legacy:
                dh = ch // nh
            return SpatialTransformer(ch, nh, dh, depth=transformer_depth, context_dim=context_dim,
                                      disable_self_attn=disable_sa, use_linear=use_linear_in_transformer,
                                      use_checkpoint=use_checkpoint)

        def resblock(cin, cout):
            return ResBlock(cin, time_embed_dim, dropout, out_channels=cout, dims=dims, use_checkpoint=use_checkpoint,
                            use_scale_shift_norm=use_scale_shift_norm)

        self.input_blocks = nn.ModuleList([TimestepEmbedSequential(_conv2d(in_channels, model_channels, 3, padding=1))])
        self.zero_convs = nn.ModuleList([self.make_zero_conv(model_channels)])
        # image-space hint encoder of the vanilla ControlNet (8 convs, 3 -> model_channels at 1/8 resolution); every
        # CtrLoRA variant deletes it right after construction (cldm_ctrlora_finetune.py:19) and feeds VAE latents
        widths = [(hint_channels, 16, 1), (16, 16, 1), (16, 32, 2), (32, 32, 1), (32, 96, 2), (96, 96, 1), (96, 256, 2)]
        hint_layers = []
        for cin, cout, stride in widths:
            hint_layers += [nn.Conv2d(cin, cout, 3, padding=1, stride=stride), nn.SiLU()]
        hint_layers.append(zero_module(nn.Conv2d(256, model_channels, 3, padding=1)))
        self.input_hint_block = TimestepEmbedSequential(*hint_layers)

        self._feature_size = model_channels
        ch, ds = model_channels, 1
        for level, mult in enumerate(self.channel_mult):
            for nr in range(self.num_res_blocks[level]):
                layers = [resblock(ch, mult * model_channels)]
                ch = mult * model_channels
                if ds in self.attention_resolutions:
                    dsa = disable_self_attentions[level] if exists(disable_self_attentions) else False
                    if not exists(num_attention_blocks) or nr < num_attention_blocks[level]:
                        layers.append(transformer(ch, dsa))
                self.input_blocks.append(TimestepEmbedSequential(*layers))
                self.zero_convs.append(self.make_zero_conv(ch))
            if level != len(self.channel_mult) - 1:
                self.input_blocks.append(TimestepEmbedSequential(Downsample(ch, conv_resample, dims=dims, out_channels=ch)))
                self.zero_convs.append(self.make_zero_conv(ch))
                ds *= 2
        self.middle_block = TimestepEmbedSequential(resblock(ch, ch), transformer(ch, disable_middle_self_attn),
                                                    resblock(ch, ch))
        self.middle_block_out = self.make_zero_conv(ch)
        self._prep = prepare.PrepCache()

    def make_zero_conv(self, channels):
        return TimestepEmbedSequential(zero_module(_conv2d(channels, channels, 1, padding=0)))

    # ControlNet shares the batched time-embedding path with the UNet
    _resblocks = UNetModel._resblocks
    embed = UNetModel.embed

    def _zero_conv(self, seq, h):
        conv = prepare.effective(seq[0])
        w = seq[0]._cache().get(("w", id(conv)), [conv.weight], lambda: prepare.conv_weight(conv.weight))
        return nchw_view(ops.gemm(pixel_major(h), w, bias=prepare.bias_f32(conv.bias)))

    def _encode(self, h, emb, ctx):
        outs = []
        for module, zero_conv in zip(self.input_blocks, self.zero_convs):
            h = module(h, emb, ctx)
            outs.append(self._zero_conv(zero_conv, h))
        h = self.middle_block(h, emb, ctx)
        outs.append(self._zero_conv(self.middle_block_out, h))
        return outs

    def forward(self, x, hint, timesteps, context, **kwargs):
        """Vanilla ControlNet signature (reference :284-305) with an image-space hint."""
        if not hasattr(self, "input_hint_block"):
            raise RuntimeError("input_hint_block was deleted: use the CtrLoRA subclasses' forward(hint, timesteps, context)")
        raise NotImplementedError("the image-space hint encoder (stride-2 convs on 3-channel input) is outside the "
                                  "CtrLoRA path; all CtrLoRA variants feed the 4-channel VAE latent of the hint")

    def forward_latent_hint(self, hint, timesteps, context):
        """Shared body of ControlNet{Finetune,Pretrain,Inference}.forward (cldm_ctrlora_finetune.py:40-54)."""
        emb = self.embed(timesteps)
        return self._encode(hint, emb, _ctx16(context))


class ControlLDM(LatentDiffusion):
    def __init__(self, control_stage_config, control_key, only_mid_control, global_average_pooling=False, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.control_model = instantiate_from_config(control_stage_config)
        self.control_key = control_key
        self.only_mid_control = only_mid_control
        self.control_scales = [1.0] * 13
        self.global_average_pooling = global_average_pooling
        if global_average_pooling:
            raise NotImplementedError("global_average_pooling (shuffle ControlNet) is not on the CtrLoRA path")

    # -- shared by the CtrLoRA subclasses -------------------------------------------------------------------------
    def hint_latent(self, c_concat):
        """`0.18215 * VAE.encode(hint).sample()` (cldm_ctrlora_finetune.py:76-77).  A 4-channel tensor is taken to be
        that latent already (the reference would fail on it), which is how the post-VAE parity boundary and the
        benchmarks feed the path (SURVEY.md §0.6)."""
        hint = c_concat[0] if len(c_concat) == 1 else torch.cat(c_concat, 1)
        if hint.shape[1] == self.channels:
            return hint
        if getattr(self, "cache_hint_latent", False):
            # Opt-in (SURVEY.md §8 f1): the reference re-encodes the SAME condition image and re-draws posterior noise in
            # every apply_model -- 2 x S VAE passes of 1117 GFLOP per sampled image.  With the cache the latent is encoded
            # and sampled once per distinct hint tensor; that changes how much host RNG a sampling run consumes (one draw
            # instead of 2 x S), which is why it is not the default.
            key = (hint.data_ptr(), hint._version, tuple(hint.shape))
            hit = self.__dict__.get("_hint_cache")
            if hit is not None and hit[0] == key:
                return hit[1]
            lat = self.get_first_stage_encoding(self.encode_first_stage(hint))
            self.__dict__["_hint_cache"] = (key, lat)
            return lat
        return self.get_first_stage_encoding(self.encode_first_stage(hint))

    @torch.no_grad()
    def prepare_context(self, context):
        """Register `context` ([B, 77, 768], the tensor apply_model will receive as c_crossattn[0]) as step-invariant:
        its fp16 copy and the K / V^T projections of every cross-attention layer of the ControlNet and the UNet are
        computed now, into persistent buffers, and re-used by every following apply_model on this same tensor (identity +
        version checked; weight changes re-project).  Idempotent and cheap when nothing changed."""
        from ctrlora_b200 import runtime
        from ldm.modules.attention import CrossAttention
        if context is None or not context.is_cuda:
            return
        reg = runtime.CTX16
        if not runtime.context_registered(context):
            ctx16 = runtime.to_f16_rows(context).view(context.shape[0], context.shape[1], -1)
            old = reg["ctx16"]
            if old is not None and old.shape == ctx16.shape and old.device == ctx16.device:
                old.copy_(ctx16)  # keep the address: captured graphs read this buffer
                ctx16 = old
            reg.update(tensor=context, version=context._version, ctx16=ctx16, epoch=reg["epoch"] + 1)
        ctx16 = reg["ctx16"]
        key = reg["epoch"]
        ctx2d, nk = ctx16.view(-1, ctx16.shape[-1]), ctx16.shape[1]
        pairs = {}  # twin pass: a ControlNet layer and its UNet partner keep their K / V^T in one batch-2B buffer pair
        if self._twin_pairs() is not None:
            for ca, cb in self._twin_pairs()["cross"]:
                b, inner = ctx16.shape[0], ca.to_q.out_features
                nk_pad = (nk + 7) // 8 * 8
                buf = ca.__dict__.get("_kv_twin")
                if buf is None or buf[0].shape != (2 * b * nk, inner) or buf[0].device != ctx16.device:
                    buf = (torch.empty((2 * b * nk, inner), device=ctx16.device, dtype=torch.float16),
                           ops.zeros((2 * b, ca.heads, inner // ca.heads, nk_pad), ctx16.device))
                    ca.__dict__["_kv_twin"] = buf
                pairs[id(ca)] = (buf[0][:b * nk], buf[1][:b])
                pairs[id(cb)] = (buf[0][b * nk:], buf[1][b:])
        for net in (self.control_model, self.model.diffusion_model):
            for m in net.modules():
                if isinstance(m, CrossAttention) and m.to_k.in_features == ctx16.shape[-1] and m.to_k.in_features != m.to_q.in_features:
                    m.project_context(ctx2d, ctx16.shape[0], nk, key, out=pairs.get(id(m)))

    def _twin_pairs(self):
        """The layer pairs of the twin pass, or None when the ControlNet and the UNet encoder differ in structure (the
        style variant's IP-Adapter UNet, say).  Checked once per model: "cross" are the cross-attention pairs, "norms"
        the transformer norm pairs, whose effective layers (switch_lora re-points the inference ControlNet's) must have
        one eps when the pass runs.  The pass starts after the first Downsample, so a network without one has none."""
        from ldm.modules.attention import BasicTransformerBlock, CrossAttention
        if "_twin" in self.__dict__:
            return self.__dict__["_twin"]
        cn, un = self.control_model, self.model.diffusion_model

        def same(a, b):
            if type(a) is not type(b):
                return False
            if isinstance(a, ResBlock):
                return (a.channels, a.out_channels, type(a.skip_connection), a.in_layers[0].eps, a.out_layers[0].eps) == \
                    (b.channels, b.out_channels, type(b.skip_connection), b.in_layers[0].eps, b.out_layers[0].eps)
            if isinstance(a, SpatialTransformer):
                blocks = list(zip(a.transformer_blocks, b.transformer_blocks))
                return (a.in_channels, a.use_linear, len(a.transformer_blocks)) == \
                    (b.in_channels, b.use_linear, len(b.transformer_blocks)) and not a.use_linear and all(
                        type(x) is BasicTransformerBlock and type(y) is BasicTransformerBlock and not x.disable_self_attn and
                        not y.disable_self_attn and type(x.attn1) is CrossAttention and type(y.attn1) is CrossAttention and
                        type(x.attn2) is CrossAttention and type(y.attn2) is CrossAttention and
                        (x.attn1.heads, x.attn1.to_q.out_features, x.attn2.to_k.in_features) ==
                        (y.attn1.heads, y.attn1.to_q.out_features, y.attn2.to_k.in_features)
                        for x, y in blocks)
            if isinstance(a, Downsample):
                return (a.channels, a.out_channels) == (b.channels, b.out_channels)
            if isinstance(a, _Conv):
                return (a.in_channels, a.out_channels, a.kernel_size) == (b.in_channels, b.out_channels, b.kernel_size)
            return False

        seqs = list(zip(cn.input_blocks, un.input_blocks)) + [(cn.middle_block, un.middle_block)]
        ok = isinstance(un, ControlledForward) and len(cn.input_blocks) == len(un.input_blocks) and \
            cn.model_channels == un.model_channels and any(isinstance(m[0], Downsample) for m in cn.input_blocks) and all(
                len(a) == len(b) and all(same(x, y) for x, y in zip(a, b)) for a, b in seqs)
        res = None
        if ok:
            sts = [(la, lb) for a, b in seqs for la, lb in zip(a, b) if isinstance(la, SpatialTransformer)]
            blocks = [(x, y) for la, lb in sts for x, y in zip(la.transformer_blocks, lb.transformer_blocks)]
            res = {"cross": [(x.attn2, y.attn2) for x, y in blocks],
                   "norms": [(la.norm, lb.norm) for la, lb in sts] +
                            [(getattr(x, n), getattr(y, n)) for x, y in blocks for n in ("norm1", "norm2", "norm3")]}
        self.__dict__["_twin"] = res
        return res

    def twin_enabled(self):
        """Whether apply_model runs the ControlNet and the UNet encoder as one pass (the module docstring): inference
        only, on structurally equal networks, unless CTRLORA_TWIN_ENCODER=0."""
        if os.environ.get("CTRLORA_TWIN_ENCODER", "1") == "0" or self.training or torch.is_grad_enabled():
            return False
        pairs = self._twin_pairs()
        eff = prepare.effective
        return pairs is not None and all(eff(a).eps == eff(b).eps for a, b in pairs["norms"])

    @torch.no_grad()
    def _control_and_unet(self, x, hint, t, context):
        """The ControlNet's 13 control residuals and the UNet encoder + middle block as one batch-2B pass.
        Returns (control, h, hs, emb, ctx) for ControlledForward.decode."""
        cn, un = self.control_model, self.model.diffusion_model
        b = x.shape[0]
        # each network's time embedding, in rows of one common stride: a grouped GEMM reads both with one row stride
        wc = sum(r.out_channels for r in cn._resblocks())
        wu = sum(r.out_channels for r in un._resblocks())
        ld = max(wc, wu)
        emb_c = cn.embed(t, out_all=torch.empty((b, ld), device=x.device, dtype=torch.float32)[:, :wc])
        emb_u = un.embed(t, out_all=torch.empty((b, ld), device=x.device, dtype=torch.float32)[:, :wu])
        ctx = _ctx16(context)
        # the full-resolution blocks run at batch b per network (measured no faster twinned); the first Downsample
        # writes each network's output into its half of the batch-2b buffer, and the twin pass takes over from there
        down = next(i for i, m in enumerate(cn.input_blocks) if isinstance(m[0], Downsample))
        control, hs = [], []
        hc, hu = hint, x
        for i in range(down + 1):
            if i < down:
                hc = cn.input_blocks[i](hc, emb_c, ctx)
                hu = un.input_blocks[i](hu, emb_u, ctx)
            else:
                xc, xu = pixel_major(hc), pixel_major(hu)
                h16 = torch.empty((2 * b, xc.shape[1] // 2, xc.shape[2] // 2, cn.input_blocks[i][0].out_channels),
                                  device=x.device, dtype=torch.float16)
                cn.input_blocks[i][0].run(xc, out=h16[:b])
                un.input_blocks[i][0].run(xu, out=h16[b:])
                h = nchw_view(h16)
                hc, hu = h[:b], h[b:]
            control.append(cn._zero_conv(cn.zero_convs[i], hc))
            hs.append(hu)
        for i in range(down + 1, len(cn.input_blocks)):
            h = cn.input_blocks[i](h, emb_c, ctx, other=un.input_blocks[i], emb_other=emb_u)
            control.append(cn._zero_conv(cn.zero_convs[i], h[:b]))
            hs.append(h[b:])
        h = cn.middle_block(h, emb_c, ctx, other=un.middle_block, emb_other=emb_u)
        control.append(cn._zero_conv(cn.middle_block_out, h[:b]))
        return control, h[b:], hs, emb_u, ctx

    def control_and_unet(self, x, hint, t, cond_txt, control_of):
        """apply_model's body for one ControlNet pass: the twin pass when twin_enabled(), else the ControlNet then the
        UNet.  control_of(residuals) -> the control list the decoder consumes."""
        diffusion_model = self.model.diffusion_model
        if self.twin_enabled():
            control, h, hs, emb, ctx = self._control_and_unet(x, hint, t, cond_txt)
            return diffusion_model.decode(h, hs, emb, ctx, control_of(control), self.only_mid_control)
        control = self.control_model(hint=hint, timesteps=t, context=cond_txt)
        return diffusion_model(x=x, timesteps=t, context=cond_txt, control=control_of(control),
                               only_mid_control=self.only_mid_control)

    def scaled_control(self, control):
        return [Scaled(c, s) for c, s in zip(control, self.control_scales)]

    def apply_model(self, x_noisy, t, cond, *args, **kwargs):
        assert isinstance(cond, dict)
        diffusion_model = self.model.diffusion_model
        cond_txt = cond['c_crossattn'][0] if len(cond['c_crossattn']) == 1 else torch.cat(cond['c_crossattn'], 1)
        if cond['c_concat'] is None:
            return diffusion_model(x=x_noisy, timesteps=t, context=cond_txt, control=None,
                                   only_mid_control=self.only_mid_control)
        hint = cond['c_concat'][0] if len(cond['c_concat']) == 1 else torch.cat(cond['c_concat'], 1)
        control = self.control_model(x=x_noisy, hint=hint, timesteps=t, context=cond_txt)
        return diffusion_model(x=x_noisy, timesteps=t, context=cond_txt, control=self.scaled_control(control),
                               only_mid_control=self.only_mid_control)

    @torch.no_grad()
    def get_unconditional_conditioning(self, N):
        return self.get_learned_conditioning([""] * N)

    def configure_optimizers(self):
        lr = self.learning_rate
        params = list(self.control_model.parameters())
        if not getattr(self, "sd_locked", True):
            params += list(self.model.diffusion_model.output_blocks.parameters())
            params += list(self.model.diffusion_model.out.parameters())
        return torch.optim.AdamW(params, lr=lr)

    def low_vram_shift(self, is_diffusing):
        """Kept for API compatibility (reference :428-438): an 80 GB H100 holds every stage at once, nothing moves."""
        return None
