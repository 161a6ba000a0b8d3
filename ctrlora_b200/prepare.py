"""Kernel-layout weight copies (fp16, K-major, tap-major convs, LoRA folded in), cached per module and
re-derived whenever a source parameter changes (torch's `_version` counter / a new storage).

The fp32 nn.Parameters keep the reference's names and shapes, so `load_state_dict(strict=True)`, the optimizer
filters and the checkpoint tooling (SURVEY.md §5) see the reference's state dict; these copies are derived data.
"""
import contextlib

import torch

from . import ops


# Bumped by the trainer after every optimizer step: its fused AdamW kernel updates the flat parameter buffer behind
# torch's back, so `_version` does not move for parameters tagged `_ctrlora_trainable`.
TRAIN_VERSION = 0


def bump_train_version():
    global TRAIN_VERSION
    TRAIN_VERSION += 1


# Bumped whenever this package re-points a parameter's storage (`p.data = ...`: LoRA fuse / unfuse, a trainer adopting the
# parameters into its flat buffer) -- a change torch's `_version` counter does not see.  Captured-graph owners (the sampler)
# compare it every call and re-verify the storage pointers themselves only at the start of a sampling run.
STRUCT_VERSION = 0


def bump_struct_version():
    global STRUCT_VERSION
    STRUCT_VERSION += 1


def _ver(*params):
    return tuple((p.data_ptr(), p._version, tuple(p.shape), TRAIN_VERSION if getattr(p, "_ctrlora_trainable", False) else 0)
                 if p is not None else None for p in params)


# While a list is installed here, every PrepCache.get appends (cache, key, params, builder) to it: a trainer that
# accumulates gradients records which weight copies a micro-batch reads, so it can rebuild them in a graph of their own.
# A builder re-run that way must read its inputs from parameters or through other get() calls, never from a tensor it
# closed over, or it would rebuild from stale data.
RECORD = None


@contextlib.contextmanager
def record_builds():
    global RECORD
    log, prev = [], RECORD
    RECORD = log
    try:
        yield log
    finally:
        RECORD = prev


class PrepCache:
    """`get(key, params, builder)` returns builder() and re-runs it only when one of `params` changed."""

    def __init__(self):
        self._store = {}

    def get(self, key, params, builder):
        if RECORD is not None:
            RECORD.append((self, key, params, builder))
        ver = _ver(*params)
        hit = self._store.get(key)
        if hit is not None and hit[0] == ver:
            return hit[1]
        with torch.no_grad():
            val = builder()
        self._store[key] = (ver, val)
        return val

    def clear(self):
        self._store.clear()


def _f32c(p):
    t = p.detach()
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    return t


def linear_weight(weight, out=None):
    """nn.Linear weight fp32 [N, K] -> fp16 [N, 1, K] (written into `out`, a contiguous fp16 [N, 1, K] view, when given)"""
    n, k = weight.shape
    return ops.cast_transpose(_f32c(weight), n * k, 1, 1, out=out).view(n, 1, k)


def conv_weight(weight, pad_in=None, pad_out=None):
    """nn.Conv2d weight fp32 [Cout, Cin, kh, kw] -> fp16 [Cout(pad), kh*kw, Cin(pad)] (tap-major, channel-minor)."""
    co, ci, kh, kw = weight.shape
    wk = weight.detach().permute(0, 2, 3, 1)
    if weight.dtype == torch.float32 and wk.is_contiguous() and weight.is_cuda:
        # a trainer's GradSink already stores the parameter in kernel order [Cout, kh, kw, Cin]: the copy is a plain cast
        w = ops.cast_transpose(wk, co * kh * kw * ci, 1, 1).view(co, kh * kw, ci)
    else:
        w = ops.cast_transpose(_f32c(weight), co, ci, kh * kw)  # [Cout, taps, Cin]
    if pad_in or pad_out:
        full = torch.zeros((pad_out or co, kh * kw, pad_in or ci), device=w.device, dtype=torch.float16)
        full[:co, :, :ci] = w
        w = full
    return w


def flat_conv_weight(weight, k_multiple=1):
    """nn.Conv2d weight fp32 [Cout, Cin, kh, kw] -> fp16 [Cout, 1, K]: conv_weight's tap-major, channel-minor order as
    one row per output channel (the order of the tap gather and im2col_s2), zero-padded to a multiple of k_multiple."""
    w = conv_weight(weight)
    co, taps, ci = w.shape
    k = taps * ci
    w = w.view(co, 1, k)
    k_pad = (k + k_multiple - 1) // k_multiple * k_multiple
    if k_pad == k:
        return w
    full = torch.zeros((co, 1, k_pad), device=w.device, dtype=torch.float16)
    full[:, :, :k] = w
    return full


def lora_folded_weight(weight, down, up, scale=1.0, out=None):
    """W' = W + scale * up @ down as fp16 [N, 1, K]  (cldm/lora.py:250 `_fuse_lora`, evaluated in fp32 accumulate).

    One wgmma GEMM: A = up [N, r], B = down^T [K, r], epilogue adds the fp32 master W.  Cost 2*N*K*r flop, once per
    weight version (per optimizer step in training, once per checkpoint in sampling) instead of two skinny GEMMs and an
    add per forward call (cldm/lora.py:285-291)."""
    n, k = weight.shape
    r = down.shape[0]
    up16 = ops.cast_transpose(_f32c(up), n * r, 1, 1).view(n, r)
    down_t = ops.cast_transpose(_f32c(down), 1, r, k).view(k, 1, r)  # [K, r]
    if r % 8:  # TMA needs 16-byte rows: zero-pad the rank
        rp = (r + 7) // 8 * 8
        u2 = torch.zeros((n, rp), device=up16.device, dtype=torch.float16)
        u2[:, :r] = up16
        d2 = torch.zeros((k, 1, rp), device=up16.device, dtype=torch.float16)
        d2[:, :, :r] = down_t
        up16, down_t = u2, d2
    out = torch.empty((n, k), device=weight.device, dtype=torch.float16) if out is None else out.view(n, k)
    ops.gemm(up16, down_t, residual=_f32c(weight), out_scale=scale, out=out)
    return out.view(n, 1, k)


def effective_linear_weight(linear, out=None):
    """fp16 [N,1,K] weight of an nn.Linear or a LoRACompatibleLinear (LoRA folded when a lora_layer is attached)."""
    lora = getattr(linear, "lora_layer", None)
    if lora is None:
        return linear_weight(linear.weight, out=out)
    scale = 1.0
    if getattr(lora, "network_alpha", None) is not None:
        scale = lora.network_alpha / lora.rank  # cldm/lora.py:77-78
    return lora_folded_weight(linear.weight, lora.down.weight, lora.up.weight, scale * getattr(linear, "_lora_scale", 1.0),
                              out=out)


def linear_params(linear):
    """the parameters whose change invalidates effective_linear_weight(linear)"""
    lora = getattr(linear, "lora_layer", None)
    ps = [linear.weight]
    if lora is not None:
        ps += [lora.down.weight, lora.up.weight]
    return ps


def bias_f32(p):
    return None if p is None else _f32c(p)


def effective(module):
    """For the reference's Switchable* layers (cldm/switchable.py): the swapped-in inner layer's parameters are the
    live ones; any other module is its own effective layer."""
    inner = getattr(module, "norm_layer", None)
    if inner is None:
        inner = getattr(module, "conv_layer", None)
    return module if inner is None else inner


def lora_key(*linears):
    """cache-key component identifying which LoRA set is attached (switch_lora re-points `lora_layer`)"""
    return tuple(id(getattr(lin, "lora_layer", None)) for lin in linears)


def weight_T(w16):
    """fp16 kernel weight [N, 1, K] -> its transpose [K, 1, N] (dx = dy @ W uses the GEMM with this as the weight)."""
    n, _, k = w16.shape
    return ops.transpose_f16(w16.view(1, n, k).contiguous(), 1, n, k).view(k, 1, n)


def conv_dgrad_weight(w16):
    """fp16 conv kernel weight [Cout, taps, Cin] -> data-gradient weight [Cin, taps (flipped), Cout]:
    dx = conv(dy, W_d) with the same 'same' padding."""
    return ops.conv_dgrad_weight(w16.contiguous())
