"""Glue shared by the drop-in modules: the internal activation convention and the small carrier objects that let
fused kernels see across module boundaries without changing the reference's call signatures.

Internal activations are fp16 "pixel-major" buffers [B, H, W, C]; between modules they travel as the zero-copy
logical-NCHW view of that buffer (`buf.permute(0, 3, 1, 2)`, i.e. a channels_last tensor), so every module still
receives and returns [B, C, H, W]-shaped tensors like the reference's.
"""
import torch

from . import ops


def pixel_major(x, c_pad=None):
    """[B,C,H,W] tensor (fp16 channels_last view, or fp32 NCHW from outside) -> fp16 [B,H,W,C] contiguous buffer."""
    if x.dim() != 4:
        raise ValueError(f"expected a [B,C,H,W] tensor, got {tuple(x.shape)}")
    if not x.is_cuda:
        raise RuntimeError("ctrlora_b200 runs on CUDA (sm_90a) only: move the model and inputs to the GPU")
    if x.dtype == torch.float16:
        v = x.permute(0, 2, 3, 1)
        if v.is_contiguous() and c_pad in (None, x.shape[1]):
            return v
        x = x.float()
    return ops.nchw_to_nhwc_f16(x.float().contiguous(), c_pad)


def nchw_view(buf):
    """fp16 [B,H,W,C] buffer -> logical [B,C,H,W] view (no copy)."""
    return buf.permute(0, 3, 1, 2)


# Step-invariant text conditioning (one sampling run = 50 DDIM steps over the SAME [B,77,768] context): the fp16 copy of the
# context and every cross-attention's K / V^T projections of it are computed once by `prepare_context` (called by the sampler)
# and found again here by tensor identity, instead of 32 small GEMMs + a cast per step (1.8 % of the DDIM step).
CTX16 = {"tensor": None, "version": -1, "ctx16": None, "epoch": 0}
# The registered tensor is held by reference (so its address cannot be recycled for another tensor while the cache lives) and
# matched by object identity + torch's in-place version counter.


def context_registered(context):
    return CTX16["tensor"] is context and CTX16["version"] == context._version


def context_f16(context):
    """[B, T, D] context -> fp16 [B, T, D]; the cached copy when `prepare_context` registered this very tensor."""
    if context is None:
        return None
    if context_registered(context):
        return CTX16["ctx16"]
    return to_f16_rows(context).view(context.shape[0], context.shape[1], -1)


def to_f16_rows(t):
    """fp32/fp16 [..., K] -> fp16 [rows, K] contiguous (context tokens)."""
    k = t.shape[-1]
    if t.dtype == torch.float16:
        return t.reshape(-1, k).contiguous()
    t = t.float().contiguous()
    return ops.cast_transpose(t, t.numel(), 1, 1).view(-1, k)


class Scaled:
    """A ControlNet residual with its control_scale (cldm/cldm_ctrlora_finetune.py:79): the multiply is applied where
    the residual is consumed (the GroupNorm kernel's addend scale) instead of as a separate pass."""
    __slots__ = ("tensor", "scale")

    def __init__(self, tensor, scale=1.0):
        self.tensor, self.scale = tensor, float(scale)


def unwrap_scaled(c):
    return (c.tensor, c.scale) if isinstance(c, Scaled) else (c, 1.0)


class CatSpec:
    """Deferred `cat([h (+ s1*add1), skip (+ s2*add2)], dim=1)` (cldm/cldm.py:34-42): consumed by the next ResBlock's
    GroupNorm kernel, which reads the pieces in place."""
    __slots__ = ("x1", "add1", "s1", "x2", "add2", "s2")

    def __init__(self, x1, add1=None, s1=1.0, x2=None, add2=None, s2=1.0):
        self.x1, self.add1, self.s1, self.x2, self.add2, self.s2 = x1, add1, s1, x2, add2, s2


class EmbPack:
    """Time embedding plus the per-ResBlock `emb_layers` outputs of a whole network, produced by one batched GEMV."""
    __slots__ = ("raw", "slices")

    def __init__(self, raw, slices=None):
        self.raw, self.slices = raw, slices or {}
