"""Drop-in for the reference's `cldm/cldm_ctrlora_inference.py`: a ControlNet with `lora_num` switchable sets of
(LoRA layers, zero-convs, norm layers) and an LDM whose apply_model sums the weighted control stacks."""
import copy

import torch
import torch.nn as nn

from ctrlora_b200 import ops

from cldm.cldm import ControlLDM, ControlNet
from cldm.ddim_hacked import DDIMSampler
from cldm.lora import LoRACompatibleLinear, LoRALinearLayer
from cldm.switchable import SwitchableConv2d, SwitchableGroupNorm, SwitchableLayerNorm
from cldm._inject import plain_linears, set_child, to_lora_linear
from ctrlora_b200.runtime import Scaled, unwrap_scaled


class ControlNetInference(ControlNet):
    def __init__(self, lora_rank=128, lora_num=1, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.lora_rank = lora_rank
        self.lora_num = lora_num
        del self.input_hint_block
        linears = plain_linears(self)
        zero_convs = [(n, m) for n, m in self.named_modules()
                      if ('zero_convs' in n or 'middle_block_out' in n) and isinstance(m, nn.Conv2d)]
        norms = [(n, m) for n, m in self.named_modules() if 'norm' in n and isinstance(m, (nn.GroupNorm, nn.LayerNorm))]
        self.loras_list = nn.ModuleList([
            nn.ModuleList([LoRALinearLayer(m.in_features, m.out_features, rank=lora_rank) for _, m in linears])
            for _ in range(lora_num)])
        self.zero_convs_list = nn.ModuleList([nn.ModuleList([copy.deepcopy(m) for _, m in zero_convs])
                                              for _ in range(lora_num)])
        self.norms_list = nn.ModuleList([nn.ModuleList([copy.deepcopy(m) for _, m in norms]) for _ in range(lora_num)])
        for n, m in linears:
            set_child(self, n, to_lora_linear(m))
        for n, m in zero_convs:
            set_child(self, n, SwitchableConv2d(m.in_channels, m.out_channels, m.kernel_size, m.stride, m.padding,
                                                m.dilation, m.groups, m.bias is not None))
        for n, m in norms:
            if isinstance(m, nn.GroupNorm):
                # note: the reference's switchable GroupNorm is built with the default eps (cldm_ctrlora_inference.py:88);
                # the swapped-in copies in norms_list keep the original eps and are the layers that get evaluated
                set_child(self, n, SwitchableGroupNorm(m.num_groups, m.num_channels))
            else:
                set_child(self, n, SwitchableLayerNorm(m.normalized_shape, m.eps, m.elementwise_affine))

    def forward(self, hint, timesteps, context, **kwargs):
        return self.forward_latent_hint(hint, timesteps, context)

    # ---- all LoRA sets in ONE pass (SURVEY.md §8 f2) ---------------------------------------------------------------
    def _switch_units(self):
        """{unit module: [(module, kind, index)]}: for every SpatialTransformer / zero-conv / the embedding MLP, the
        switchable children with the index `switch_lora` would give them (named_modules() order, reference :116-130)."""
        if self.__dict__.get("_units") is None:
            from ldm.modules.attention import SpatialTransformer
            from ldm.modules.diffusionmodules.openaimodel import ResBlock
            index, i, iz, inorm = {}, 0, 0, 0
            for n, m in self.named_modules():
                if any(tok in n for tok in ("loras_list", "zero_convs_list", "norms_list")):
                    continue
                if isinstance(m, LoRACompatibleLinear):
                    index[id(m)] = ("lora", i); i += 1
                elif isinstance(m, SwitchableConv2d):
                    index[id(m)] = ("conv", iz); iz += 1
                elif isinstance(m, (SwitchableGroupNorm, SwitchableLayerNorm)):
                    index[id(m)] = ("norm", inorm); inorm += 1
            units = {}
            roots = [m for m in self.modules() if isinstance(m, (SpatialTransformer, SwitchableConv2d))]
            emb_root = [self.time_embed] + [m.emb_layers for m in self.modules() if isinstance(m, ResBlock)]
            for root in roots + emb_root:
                units[id(root)] = [(m,) + index[id(m)] for m in root.modules() if id(m) in index]
            self.__dict__["_units"] = units
        return self.__dict__["_units"]

    def _attach(self, unit, g):
        for m, kind, idx in self._switch_units()[id(unit)]:
            if kind == "lora":
                m.set_lora_layer(self.loras_list[g][idx])
            elif kind == "conv":
                m.set_conv_layer(self.zero_convs_list[g][idx])
            else:
                m.set_norm_layer(self.norms_list[g][idx])

    def forward_grouped(self, hints, timesteps, context):
        """hints: `lora_num` tensors [B,4,H,W]; timesteps [B]; context [B,77,768].  Returns `lora_num` lists of 13 residuals,
        identical to running forward() once per set after switch_lora(i), from ONE pass over the batch [lora_num*B]: every
        conv / ResBlock GroupNorm (shared weights) sees the whole batch; LoRA linears, switchable norms and zero-convs run per
        slice with their set attached.  Ends with the last set attached, like the reference's loop."""
        from ldm.modules.attention import SpatialTransformer
        from ldm.modules.diffusionmodules.openaimodel import ResBlock
        from ctrlora_b200 import prepare
        from ctrlora_b200.runtime import EmbPack, context_f16, nchw_view, pixel_major
        n, b = len(hints), hints[0].shape[0]
        dev = hints[0].device
        # time embedding: time_embed and every emb_layers linear carry LoRA -> one batched GEMV per set, rows side by side
        blocks = self._resblocks()
        tdim = self.time_embed[2].out_features
        raw = torch.empty((n * b, tdim), device=dev, dtype=torch.float32)
        allout = torch.empty((n * b, sum(rb.out_channels for rb in blocks)), device=dev, dtype=torch.float32)
        for g in range(n):
            self._attach(self.time_embed, g)
            for rb in blocks:
                self._attach(rb.emb_layers, g)
            self.embed(timesteps, out_raw=raw[g * b:(g + 1) * b], out_all=allout[g * b:(g + 1) * b])
        slices, off = {}, 0
        for rb in blocks:
            slices[id(rb)] = allout[:, off:off + rb.out_channels]
            off += rb.out_channels
        emb = EmbPack(raw, slices)
        ctx16 = context_f16(context)  # [B, 77, D]: shared by the sets (reference :164), every slice attends to it
        cin = hints[0].shape[1]
        c_pad = (cin + 7) // 8 * 8
        hbuf = torch.empty((n * b, hints[0].shape[2], hints[0].shape[3], c_pad), device=dev, dtype=torch.float16)
        for g, hg in enumerate(hints):
            if hg.dtype == torch.float16:
                hbuf[g * b:(g + 1) * b].copy_(pixel_major(hg, c_pad if c_pad != cin else None))
            else:
                ops.nchw_to_nhwc_f16(hg.float().contiguous(), c_pad, out=hbuf[g * b:(g + 1) * b])
        h = nchw_view(hbuf)
        attach = lambda unit, g: self._attach(unit, g)
        outs = [[] for _ in range(n)]

        def zero(seq, hcur):
            sw = seq[0]
            for g in range(n):
                self._attach(sw, g)
                outs[g].append(self._zero_conv(seq, hcur[g * b:(g + 1) * b]))

        def run_seq(seq, hcur):
            for layer in seq:
                if isinstance(layer, ResBlock):
                    hcur = layer(hcur, emb)
                elif isinstance(layer, SpatialTransformer):
                    hcur = layer.forward_grouped(hcur, ctx16, n, attach)
                else:
                    hcur = layer(hcur)
            return hcur

        for module, zero_conv in zip(self.input_blocks, self.zero_convs):
            h = run_seq(module, h)
            zero(zero_conv, h)
        h = run_seq(self.middle_block, h)
        zero(self.middle_block_out, h)
        return outs

    def switch_lora(self, index: int):
        lora, zero_convs, norms = self.loras_list[index], self.zero_convs_list[index], self.norms_list[index]
        i = iz = inorm = 0
        for n, m in self.named_modules():
            if isinstance(m, LoRACompatibleLinear):
                m.set_lora_layer(lora[i])
                i += 1
            elif isinstance(m, SwitchableConv2d):
                m.set_conv_layer(zero_convs[iz])
                iz += 1
            elif isinstance(m, (SwitchableGroupNorm, SwitchableLayerNorm)):
                m.set_norm_layer(norms[inorm])
                inorm += 1

    def copy_weights_to_switchable(self):
        """Push the weights loaded into the switchable shells into the currently attached inner layers (call after
        switch_lora() and load_state_dict(), as in the reference :132-139)."""
        for n, m in self.named_modules():
            if isinstance(m, (SwitchableConv2d, SwitchableGroupNorm, SwitchableLayerNorm)):
                m.copy_weights()


class ControlInferenceLDM(ControlLDM):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.lora_weights = [1.0 / self.control_model.lora_num] * self.control_model.lora_num

    @torch.no_grad()
    def sample_log(self, cond, batch_size, ddim, ddim_steps, **kwargs):
        sampler = DDIMSampler(self)
        b, c, h, w = cond["c_concat"][0].shape
        shape = (self.channels, h // 8, w // 8) if c != self.channels else (self.channels, h, w)
        return sampler.sample(ddim_steps, batch_size, shape, cond, verbose=False, **kwargs)

    def apply_model(self, x_noisy, t, conds, *args, **kwargs):
        if isinstance(conds, dict):
            conds = [conds]
        assert isinstance(conds, (list, tuple))
        assert len(conds) == self.control_model.lora_num
        assert len(self.lora_weights) == self.control_model.lora_num
        diffusion_model = self.model.diffusion_model
        cc = conds[0]['c_crossattn']
        cond_txt = cc[0] if len(cc) == 1 else torch.cat(cc, 1)
        if len(conds) == 1:
            self.control_model.switch_lora(0)
            hint = self.hint_latent(conds[0]['c_concat'])
            return self.control_and_unet(x_noisy, hint, t, cond_txt, lambda st: [
                Scaled(c, s * self.lora_weights[0]) for c, s in zip(st, self.control_scales)])
        if getattr(self, "grouped_multi_lora", True):
            # all LoRA sets in one ControlNet pass (convs and ResBlock norms batched over the sets)
            hints = [self.hint_latent(cond['c_concat']) for cond in conds]
            stacks = self.control_model.forward_grouped(hints, t, cond_txt)
        else:
            stacks = []
            for i, cond in enumerate(conds):
                self.control_model.switch_lora(i)
                hint = self.hint_latent(cond['c_concat'])
                stacks.append(self.control_model(hint=hint, timesteps=t, context=cond_txt))
        # sum_i w_i * scale_j * control_i[j]  (reference :172-176): one n-ary kernel per residual, fp32 accumulate
        control = [ops.weighted_sum([st[j] for st in stacks], [s * w for w in self.lora_weights])
                   for j, s in enumerate(self.control_scales)]
        return diffusion_model(x=x_noisy, timesteps=t, context=cond_txt, control=control,
                               only_mid_control=self.only_mid_control)
