"""What tests/golden/midas_golden.pt is made of, shared by tools/make_midas_golden.py and the MiDaS tests.

Weights and images are regenerated from names by oracle/synth.py's frozen numpy stream, so the fixture holds the
reference's outputs, the state-dict keys and shapes, and input checksums only.

synth_param's variance-preserving scales alone leave the network's last ReLU with a depth that is zero everywhere
(the 32 -> 1 conv sums ReLU'd, hence positive, activations with random-sign weights, which lands far below 0), so the
comparison would be vacuous.  `weights` therefore takes the absolute value of that conv's weight
(scratch.output_conv.4.weight) and sets its bias to HEAD_BIAS, so that the depth is positive and varies with the
activations, and scales the ViT's residual-branch output projections (attn.proj, mlp.fc2) by BRANCH_SCALE, so that the
24 blocks do not grow the stream's norm by orders of magnitude.  The normal map then has structure: the depth has
edges at the image's 16-pixel blocks.
"""
import functools

import torch

import golden_io
from golden_io import unband  # noqa: F401
from oracle import synth

SEED = 31
# 384^2: the identity position resize; 512^2; 384 x 640 (non-square grid); 200 x 328: cropped to 192 x 320
SIZES = {"384": (384, 384), "512": (512, 512), "384x640": (384, 640), "200x328": (200, 328)}
STAGE_SIZE = (32, 64)   # block-level intermediates: a 2 x 4 grid
HEAD_BIAS = 0.1
BRANCH_SCALE = 0.25
MAP_BAND_ROWS = 32


def weights(shapes):
    """{name: shape} -> the fixture's fp32 state dict (see the module docstring for the two adjustments)"""
    sd = synth.synth_state_dict(shapes, SEED, "midas.")
    for k in sd:
        if k.endswith(("attn.proj.weight", "mlp.fc2.weight")):
            sd[k] = sd[k] * BRANCH_SCALE
    sd["model.scratch.output_conv.4.weight"] = sd["model.scratch.output_conv.4.weight"].abs()
    sd["model.scratch.output_conv.4.bias"] = torch.full_like(sd["model.scratch.output_conv.4.bias"], HEAD_BIAS)
    return sd


def image(size, tag=""):
    """uint8 HWC [H, W, 3] test image: 16-pixel blocks of coarse noise plus fine noise"""
    h, w = SIZES[size] if size in SIZES else size
    return synth.noise_image(f"midas.image.{h}x{w}{tag}", SEED, h, w, 16, 0.15)


def image_tensor(img):
    """MidasDetector.__call__'s network input: `float / 127.5 - 1`, 'h w c -> 1 c h w' (fp32, on the host)"""
    return (torch.from_numpy(img).float() / 127.5 - 1.0).permute(2, 0, 1).unsqueeze(0).contiguous()


bands = functools.partial(golden_io.bands, rows=MAP_BAND_ROWS)
