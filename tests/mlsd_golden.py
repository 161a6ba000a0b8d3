"""What tests/golden/mlsd_golden.pt is made of, shared by tools/make_mlsd_golden.py and the M-LSD tests.

Weights and images are regenerated from names by oracle/synth.py's frozen numpy stream, so the fixture holds the
reference's outputs, the state-dict keys and shapes and input checksums only.

Every BatchNorm gets running_mean ~ 0.2 N(0, 1), running_var ~ 0.5 + U(0, 1), scale 1 + 0.1 N(0, 1) and bias
0.1 N(0, 1), so each ReLU / ReLU6 passes about half its inputs.  The head's conv3 is scaled per output column so that
the decode sees the spread a trained network gives: the centre column (7) by CENTER_SCALE with bias CENTER_BIAS, so
that the 3 x 3 peaks' scores spread over (0.1, 1), and the four displacement columns (8..11) by DISP_SCALE, so that the
segment lengths spread over about (0.1, 20) pixels at the half-size map.
"""
import functools

import numpy as np
import torch

import golden_io
from oracle import synth

SEED = 53
PREFIX = "mlsd."
# 512^2, 512 x 768 and 768 x 512; 497 x 513: H = 1 mod 16 (the levels 248, 124, 62, 31); 16 x 16: fewer than 200
# scores; 500 x 740: not 0 or 1 mod 16, the reference's decoder fails
SIZES = {"512": (512, 512), "512x768": (512, 768), "768x512": (768, 512), "497x513": (497, 513), "16": (16, 16),
         "500x740": (500, 740)}
ZERO_SIZES = ("16", "500x740")
FULL_SIZE = "512x768"          # the size whose full centre and displacement maps are stored
# (thr_v, thr_d) pairs of the stored maps: the apps' default 0.1 / 0.1, tool_make_cond_images-style draws, thr_v >= 1
THRESHOLDS = ((0.1, 0.1), (0.1, 5.0), (0.35, 2.5), (0.62, 11.0), (0.85, 0.5), (1.0, 0.1), (1.7, 3.0))
CENTER_SCALE = 42.0
CENTER_BIAS = -12.0
DISP_SCALE = 40.0
STAGE_FLOATS = 24 * 1024       # values stored per backbone feature and for the head map


def _bn(name, c):
    rs = synth._rs(PREFIX + name + ".bn", SEED)
    return {"weight": 1.0 + 0.1 * rs.standard_normal(c), "bias": 0.1 * rs.standard_normal(c),
            "running_mean": 0.2 * rs.standard_normal(c), "running_var": 0.5 + rs.uniform(0.0, 1.0, c)}


def weights(shapes, bn_names):
    """{name: shape}, the BatchNorm module names -> the fixture's fp32 state dict (see the module docstring)"""
    sd = synth.synth_state_dict(shapes, SEED, PREFIX)
    for m in bn_names:
        for k, v in _bn(m, shapes[m + ".weight"][0]).items():
            sd[f"{m}.{k}"] = torch.from_numpy(v.astype(np.float32))
        sd[f"{m}.num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    w, b = sd["block23.conv3.weight"].clone(), sd["block23.conv3.bias"].clone()
    w[7] *= CENTER_SCALE
    b[7] = CENTER_BIAS
    w[8:12] *= DISP_SCALE
    sd["block23.conv3.weight"], sd["block23.conv3.bias"] = w, b
    return sd


def image(size, tag=""):
    """uint8 HWC [H, W, 3] test image: 16-pixel blocks of coarse noise plus fine noise"""
    h, w = SIZES[size] if size in SIZES else size
    return synth.noise_image(f"mlsd.image.{h}x{w}{tag}", SEED, h, w, 16, 0.15)


stage_positions = functools.partial(golden_io.stage_positions, "mlsd", SEED, STAGE_FLOATS)
sample_stage = golden_io.sample_stage
