"""Primitives of the denoising path, mirroring the names exported by the reference's
`ldm/modules/diffusionmodules/util.py`.  Schedules are host-side numpy (as in the reference); everything that touches
activations runs in the sm_90a kernels (ctrlora_b200.ops) — there is no torch/CPU fallback for those.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from ctrlora_b200 import ops


# ------------------------------------------------------------------------------------------------ schedules (host)
def make_beta_schedule(schedule, n_timestep, linear_start=1e-4, linear_end=2e-2, cosine_s=8e-3):
    """reference util.py:21-43.  float64 throughout, numpy out (DDPM.register_schedule casts to fp32)."""
    if schedule == "linear":
        # torch.linspace(float64), not np.linspace: the two can differ in the last bit and the reference uses torch
        betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=torch.float64) ** 2).numpy()
    elif schedule == "cosine":
        ts = torch.arange(n_timestep + 1, dtype=torch.float64) / n_timestep + cosine_s
        alphas = torch.cos(ts / (1 + cosine_s) * np.pi / 2).pow(2)
        alphas = alphas / alphas[0]
        betas = np.clip((1 - alphas[1:] / alphas[:-1]).numpy(), a_min=0, a_max=0.999)
    elif schedule == "sqrt_linear":
        betas = torch.linspace(linear_start, linear_end, n_timestep, dtype=torch.float64).numpy()
    elif schedule == "sqrt":
        betas = (torch.linspace(linear_start, linear_end, n_timestep, dtype=torch.float64) ** 0.5).numpy()
    else:
        raise ValueError(f"schedule '{schedule}' unknown.")
    return betas


def make_ddim_timesteps(ddim_discr_method, num_ddim_timesteps, num_ddpm_timesteps, verbose=True):
    """reference util.py:46-60: integer index arithmetic, +1 shift."""
    if ddim_discr_method == "uniform":
        stride = num_ddpm_timesteps // num_ddim_timesteps
        steps = np.arange(0, num_ddpm_timesteps, stride)
    elif ddim_discr_method == "quad":
        steps = (np.linspace(0, np.sqrt(num_ddpm_timesteps * .8), num_ddim_timesteps) ** 2).astype(int)
    else:
        raise NotImplementedError(f'There is no ddim discretization method called "{ddim_discr_method}"')
    steps = steps + 1
    if verbose:
        print(f"Selected timesteps for ddim sampler: {steps}")
    return steps


def make_ddim_sampling_parameters(alphacums, ddim_timesteps, eta, verbose=True):
    """reference util.py:63-74.  Mixed torch(fp32)/numpy arithmetic reproduced operand for operand so the per-step
    scalars are bit-identical to the reference's."""
    alphas = alphacums[ddim_timesteps]
    alphas_prev = np.asarray([alphacums[0]] + alphacums[ddim_timesteps[:-1]].tolist())
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    if verbose:
        print(f"Selected alphas for ddim sampler: a_t: {alphas}; a_(t-1): {alphas_prev}")
    return sigmas, alphas, alphas_prev


def extract_into_tensor(a, t, x_shape):
    """reference util.py:96-99: integer gather (bit-exact), reshaped for broadcasting."""
    b = t.shape[0]
    return a.gather(-1, t).reshape(b, *((1,) * (len(x_shape) - 1)))


def noise_like(shape, device, repeat=False):
    if repeat:
        return torch.randn((1, *shape[1:]), device=device).repeat(shape[0], *((1,) * (len(shape) - 1)))
    return torch.randn(shape, device=device)


# ------------------------------------------------------------------------------------------------ embeddings
_FREQS = {}


def embedding_freqs(dim, max_period, device):
    """exp(-ln(max_period) * k / half) computed with the reference's torch ops (util.py:163-166), cached on device."""
    key = (dim, max_period, str(device))
    if key not in _FREQS:
        half = dim // 2
        f = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
        _FREQS[key] = f.to(device)
    return _FREQS[key]


def timestep_embedding(timesteps, dim, max_period=10000, repeat_only=False):
    """reference util.py:154-174 -> ctrlora_timestep_embedding.  timesteps: [B] on a CUDA device.  Integer timesteps
    (the trainers, q_sample, DDIM) take the int64 kernel; floating ones (DPM-Solver's fractional model times) are
    embedded at their fp32 value, as the reference's `timesteps[:, None].float()` does (:168)."""
    if repeat_only or dim % 2:
        raise NotImplementedError("repeat_only / odd dims are not on the CtrLoRA path")
    if not timesteps.is_cuda:
        raise RuntimeError("ctrlora_b200: timestep_embedding needs CUDA tensors (no CPU path)")
    t = timesteps.to(torch.float32 if timesteps.is_floating_point() else torch.int64).contiguous()
    return ops.timestep_embedding(t, embedding_freqs(dim, max_period, timesteps.device))


# ------------------------------------------------------------------------------------------------ parameter holders
class GroupNorm32(nn.GroupNorm):
    """Parameter holder with the reference's name (util.py:217-219); the arithmetic is ctrlora_groupnorm_f16."""

    def forward(self, x):
        raise RuntimeError("GroupNorm32 is evaluated inside the fused blocks (ctrlora_groupnorm_f16), not standalone")


def normalization(channels):
    return GroupNorm32(32, channels)


def conv_nd(dims, *args, **kwargs):
    if dims != 2:
        raise ValueError(f"unsupported dimensions: {dims} (the CtrLoRA path is 2-D)")
    return nn.Conv2d(*args, **kwargs)


def linear(*args, **kwargs):
    return nn.Linear(*args, **kwargs)


def avg_pool_nd(dims, *args, **kwargs):
    raise NotImplementedError("conv_resample=False is not on the CtrLoRA path")


def zero_module(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


def checkpoint(func, inputs, params, flag):
    """The reference recomputes the forward inside backward (util.py:102-151) to save memory; results are identical
    (dropout p = 0).  An 80 GB H100 keeps the activations, so this is a plain call."""
    return func(*inputs)
