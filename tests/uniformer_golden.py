"""What tests/golden/uniformer_golden.pt is made of, shared by tools/make_uniformer_golden.py and the UniFormer tests.

Weights and images are regenerated from names by oracle/synth.py's frozen numpy stream, so the fixture holds the
reference's outputs, the state-dict keys and shapes, the palette and input checksums only.

synth_param alone gives every BatchNorm a running_var of about N(0, 0.1), mostly negative, so `weights` sets each
BatchNorm's statistics to running_mean ~ 0.2 N(0, 1) and running_var ~ 0.5 + U(0, 1), its scale to 1 + 0.1 N(0, 1)
and its bias to 0.1 N(0, 1): every ConvModule's ReLU then passes about half its inputs.  The residual branches' last
projections (CBlock conv2 and mlp.fc2, SABlock attn.proj and mlp.fc2) are scaled by BRANCH_SCALE so that 18 blocks
do not grow the stream by orders of magnitude, and conv_seg's weight by SEG_SCALE, so that the 150 logits of a pixel
spread over several units and the top-two margin is rarely near zero: the labels are then neither constant nor tied
everywhere.
"""
import functools

import numpy as np
import torch

import golden_io
from golden_io import unband  # noqa: F401
from oracle import synth

SEED = 47
PREFIX = "uniformer."
# input size -> network size: 256 x 320 -> 512 x 640; 512^2: the second logit resize is the identity; 384 x 640 ->
# 512 x 853 (odd levels: 213, 106, 53, 26 columns); 640 x 384: portrait; 200 x 1000: the 2048 long side binds -> 410 x 2048
SIZES = {"256x320": (256, 320), "512": (512, 512), "384x640": (384, 640), "640x384": (640, 384), "200x1000": (200, 1000)}
BRANCH_SCALE = 0.5
SEG_SCALE = 4.0
STAGE_FLOATS = 24 * 1024   # values stored per backbone stage and per logit map
MAP_BAND_ROWS = 64


def _bn(name, shape):
    rs = synth._rs(PREFIX + name + ".bn", SEED)
    c = shape[0]
    return {"weight": 1.0 + 0.1 * rs.standard_normal(c), "bias": 0.1 * rs.standard_normal(c),
            "running_mean": 0.2 * rs.standard_normal(c), "running_var": 0.5 + rs.uniform(0.0, 1.0, c)}


def weights(shapes, bn_names):
    """{name: shape}, the BatchNorm module names -> the fixture's fp32 state dict (see the module docstring)"""
    sd = synth.synth_state_dict(shapes, SEED, PREFIX)
    for m in bn_names:
        for k, v in _bn(m, shapes[m + ".weight"]).items():
            sd[f"{m}.{k}"] = torch.from_numpy(v.astype(np.float32))
        sd[f"{m}.num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    for k in sd:
        if k.startswith("backbone.blocks") and k.endswith(("conv2.weight", "mlp.fc2.weight", "attn.proj.weight")):
            sd[k] = sd[k] * BRANCH_SCALE
        if k.endswith("conv_seg.weight"):
            sd[k] = sd[k] * SEG_SCALE
    return sd


def image(size, tag=""):
    """uint8 HWC [H, W, 3] RGB test image: 16-pixel blocks of coarse noise plus fine noise"""
    h, w = SIZES[size] if size in SIZES else size
    return synth.noise_image(f"uniformer.image.{h}x{w}{tag}", SEED, h, w, 16, 0.15)


stage_positions = functools.partial(golden_io.stage_positions, "uniformer", SEED, STAGE_FLOATS)
sample_stage = golden_io.sample_stage
bands = functools.partial(golden_io.bands, rows=MAP_BAND_ROWS)
