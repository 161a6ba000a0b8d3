"""Drop-in for the reference's `cldm/lora.py` (diffusers-style LoRA layers): same classes, attributes
(`down`, `up`, `rank`, `network_alpha`, `lora_layer`), methods (`set_lora_layer`, `_fuse_lora`, `_unfuse_lora`) and
state-dict keys (`<linear>.lora_layer.{down,up}.weight`).

At run time the reference evaluates `W x + b + scale * up(down(x))` as three GEMMs and an add per call
(lora.py:285-291).  Here the low-rank delta is folded into the fp16 kernel copy of the weight
(`ctrlora_b200.prepare.lora_folded_weight`, one wgmma GEMM per weight version), so a LoRA linear costs exactly one
GEMM per call; the fp32 master parameters (`weight`, `lora_layer.down/up.weight`) stay separate and trainable.
"""
from typing import Optional

import torch
from torch import nn

from ctrlora_b200 import ops, prepare
from ctrlora_b200.runtime import to_f16_rows
from ldm.modules.diffusionmodules.openaimodel import _Conv


class LoRALinearLayer(nn.Module):
    """Low-rank pair (down: in -> rank, up: rank -> out); init down ~ N(0, 1/rank), up = 0 (reference :26-80)."""

    def __init__(self, in_features, out_features, rank=4, network_alpha=None, device=None, dtype=None):
        super().__init__()
        self.down = nn.Linear(in_features, rank, bias=False, device=device, dtype=dtype)
        self.up = nn.Linear(rank, out_features, bias=False, device=device, dtype=dtype)
        self.network_alpha = network_alpha
        self.rank = rank
        self.out_features = out_features
        self.in_features = in_features
        nn.init.normal_(self.down.weight, std=1 / rank)
        nn.init.zeros_(self.up.weight)

    def delta_weight(self):
        """fp16 [out, 1, in] kernel copy of (alpha/rank) * up @ down."""
        scale = 1.0 if self.network_alpha is None else self.network_alpha / self.rank
        zero = torch.zeros((self.out_features, self.in_features), device=self.up.weight.device, dtype=torch.float32)
        return prepare.lora_folded_weight(zero, self.down.weight, self.up.weight, scale)

    def forward(self, hidden_states):
        shp = hidden_states.shape
        y = ops.gemm(to_f16_rows(hidden_states), self.delta_weight())
        return y.view(*shp[:-1], self.out_features).to(hidden_states.dtype)


class LoRAConv2dLayer(nn.Module):
    """API surface only: the reference defines it (:83-141) but no call site uses conv LoRA (SURVEY.md §0.2)."""

    def __init__(self, in_features, out_features, rank=4, kernel_size=(1, 1), stride=(1, 1), padding=0,
                 network_alpha=None):
        super().__init__()
        self.down = nn.Conv2d(in_features, rank, kernel_size=kernel_size, stride=stride, padding=padding, bias=False)
        self.up = nn.Conv2d(rank, out_features, kernel_size=(1, 1), stride=(1, 1), bias=False)
        self.network_alpha = network_alpha
        self.rank = rank
        nn.init.normal_(self.down.weight, std=1 / rank)
        nn.init.zeros_(self.up.weight)

    def forward(self, hidden_states):
        raise NotImplementedError("conv LoRA has no call site on the CtrLoRA path; fuse it with LoRACompatibleConv._fuse_lora")


def _fused(w_orig, w_up, w_down, alpha, rank, lora_scale, safe_fusing, owner):
    """W + lora_scale * (alpha/rank) * up @ down in fp32 (an offline weight-surgery step, not on the hot path)."""
    w_up = w_up.float()
    if alpha is not None:
        w_up = w_up * alpha / rank
    fusion = torch.mm(w_up.flatten(start_dim=1), w_down.float().flatten(start_dim=1)).reshape(w_orig.shape)
    fused = w_orig.float() + lora_scale * fusion
    if safe_fusing and torch.isnan(fused).any().item():
        raise ValueError("This LoRA weight seems to be broken. "
                         f"Encountered NaN values when trying to fuse LoRA weights for {owner}."
                         "LoRA weights will not be fused.")
    return fused, w_up


class _LoRAFuseMixin:
    def set_lora_layer(self, lora_layer):
        self.lora_layer = lora_layer

    def _fuse_lora(self, lora_scale: float = 1.0, safe_fusing: bool = False):
        if self.lora_layer is None:
            return
        dtype, device = self.weight.data.dtype, self.weight.data.device
        lora = self.lora_layer
        fused, w_up = _fused(self.weight.data, lora.up.weight.data, lora.down.weight.data, lora.network_alpha, lora.rank,
                             lora_scale, safe_fusing, self)
        self.weight.data = fused.to(device=device, dtype=dtype)
        prepare.bump_struct_version()
        self.lora_layer = None
        self.w_up = w_up.cpu()
        self.w_down = lora.down.weight.data.float().cpu()
        self._lora_scale = lora_scale

    def _unfuse_lora(self):
        if getattr(self, "w_up", None) is None or getattr(self, "w_down", None) is None:
            return
        fused = self.weight.data
        dtype, device = fused.dtype, fused.device
        w_up, w_down = self.w_up.to(device).float(), self.w_down.to(device).float()
        fusion = torch.mm(w_up.flatten(start_dim=1), w_down.flatten(start_dim=1)).reshape(fused.shape)
        self.weight.data = (fused.float() - self._lora_scale * fusion).to(device=device, dtype=dtype)
        prepare.bump_struct_version()
        self.w_up = None
        self.w_down = None


class LoRACompatibleLinear(_LoRAFuseMixin, nn.Linear):
    """nn.Linear with an optional `lora_layer` (reference :225-291)."""

    def __init__(self, *args, lora_layer: Optional[LoRALinearLayer] = None, **kwargs):
        super().__init__(*args, **kwargs)
        self.lora_layer = lora_layer

    def kernel_weight(self, scale=1.0):
        cache = self.__dict__.setdefault("_prep", prepare.PrepCache())
        lora = self.lora_layer
        if lora is None:
            return cache.get("plain", [self.weight], lambda: prepare.linear_weight(self.weight))
        s = scale * (1.0 if lora.network_alpha is None else lora.network_alpha / lora.rank)
        return cache.get(("lora", id(lora), s), [self.weight, lora.down.weight, lora.up.weight],
                         lambda: prepare.lora_folded_weight(self.weight, lora.down.weight, lora.up.weight, s))

    def forward(self, hidden_states, scale: float = 1.0):
        shp = hidden_states.shape
        y = ops.gemm(to_f16_rows(hidden_states), self.kernel_weight(scale), bias=prepare.bias_f32(self.bias))
        return y.view(*shp[:-1], self.out_features)


class LoRACompatibleConv(_LoRAFuseMixin, _Conv):
    """nn.Conv2d with an optional `lora_layer`; only the fuse / unfuse API is live (no call sites in the reference)."""

    def __init__(self, *args, lora_layer: Optional[LoRAConv2dLayer] = None, **kwargs):
        super().__init__(*args, **kwargs)
        self.lora_layer = lora_layer

    def forward(self, hidden_states, scale: float = 1.0):
        if self.lora_layer is not None:
            raise NotImplementedError("unfused conv LoRA is not on the CtrLoRA path: call _fuse_lora() first")
        return _Conv.forward(self, hidden_states)
