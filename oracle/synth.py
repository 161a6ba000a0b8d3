"""Deterministic synthetic weights and inputs (test infrastructure, shared by tools/make_golden.py, the tests,
smoke() and bench.py).  There are no checkpoints or datasets offline, and the reference's own init makes the whole
network output exactly 0 (zero-initialised out convs / proj_out / zero-convs / LoRA up, SURVEY.md §0.4), so every
tensor is drawn from numpy's frozen RandomState stream keyed by the parameter NAME: any process on any machine
regenerates bit-identical values from (name, shape, seed) and the golden fixtures only need to store outputs.
"""
import zlib

import numpy as np
import torch


def _rs(name, seed):
    return np.random.RandomState((zlib.crc32(name.encode()) ^ (seed * 2654435761)) & 0xFFFFFFFF)


def synth_param(name, shape, seed=0):
    """Variance-preserving scales so activations stay O(1) through ~60 layers."""
    shape = tuple(shape)
    g = _rs(name, seed).standard_normal(shape).astype(np.float32)
    if name.endswith("lora_layer.down.weight") or ".down.weight" in name and "lora" in name:
        g *= 1.0 / shape[0]                       # reference init: std 1/rank (cldm/lora.py:67)
    elif name.endswith("lora_layer.up.weight") or ".up.weight" in name and "lora" in name:
        g *= 0.05                                 # reference init is zeros (lora.py:68): re-randomised
    elif len(shape) >= 2:
        fan_in = int(np.prod(shape[1:]))
        g *= fan_in ** -0.5
    elif name.endswith(".weight"):                # 1-D weights are norm gains
        g = 1.0 + 0.1 * g
    else:                                         # biases
        g *= 0.1
    return torch.from_numpy(g)


def synth_state_dict(shapes, seed=0, prefix=""):
    """shapes: {name: shape}.  The RNG key is prefix + name so control_model.* and model.diffusion_model.* differ."""
    return {k: synth_param(prefix + k, s, seed) for k, s in shapes.items()}


def synth_input(name, shape, seed=0, scale=1.0):
    return torch.from_numpy(_rs("input." + name, seed).standard_normal(tuple(shape)).astype(np.float32) * scale)


def noise_image(name, seed, h, w, block, amp):
    """uint8 HWC [h, w, 3] test image: block x block squares of coarse noise (edges for a detector) plus fine noise in
    [-amp, amp)"""
    rs = _rs(name, seed)
    nh, nw = (h + block - 1) // block, (w + block - 1) // block
    coarse = rs.uniform(0, 1, (nh, nw, 3)).repeat(block, 0).repeat(block, 1)[:h, :w]
    fine = rs.uniform(-amp, amp, (h, w, 3))
    return np.clip((coarse + fine) * 255.0, 0, 255).astype(np.uint8)
