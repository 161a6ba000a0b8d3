"""What tests/golden/lineart_golden.pt is made of, shared by tools/make_lineart_golden.py and the line-art tests.

Weights and images are regenerated from names by oracle/synth.py's frozen numpy stream (any machine gives the same
bits), so the fixture holds the reference's outputs, the state-dict keys and shapes, and input checksums only.  Stage
activations (the outputs of model0 ... model3) are stored at a fixed sample of pixel positions with all their
channels: whole stages at 512 x 512 would be hundreds of MB.
"""
import functools

import numpy as np

import golden_io
from golden_io import sample_stage, unband  # noqa: F401 (sample_stage)
from oracle import synth

SEED = 11
N_RESIDUAL = 3                                       # LineartDetector builds Generator(3, 1, 3)
SIZES = {"512": (512, 512), "384x640": (384, 640), "64": (64, 64)}
STAGE_FLOATS = 32768                                 # per stored stage: positions = STAGE_FLOATS // channels
MAP_BAND_ROWS = 128                                  # the fp32 map is stored in bands of rows


def weights(shapes):
    """{name: shape} -> the fixture's fp32 state dict"""
    return synth.synth_state_dict(shapes, SEED, "lineart.")


def image(size, tag=""):
    """uint8 HWC [H, W, 3] test image: 16-pixel blocks of coarse noise (edges for the detector) plus fine noise"""
    h, w = SIZES[size] if size in SIZES else size
    return synth.noise_image(f"lineart.image.{h}x{w}{tag}", SEED, h, w, 16, 0.15)


stage_positions = functools.partial(golden_io.stage_positions, "lineart", SEED, STAGE_FLOATS)
map_bands = functools.partial(golden_io.bands, rows=MAP_BAND_ROWS)  # a 512 x 512 map is 1 MB, more than a part file


def golden_map(golden, size):
    """the fp32 [H, W] map of one size, reassembled from its bands"""
    return unband(golden[f"{size}.map"])


def quantise(line):
    """LineartDetector.__call__'s `(line * 255.0).clip(0, 255).astype(np.uint8)` on an fp32 numpy map"""
    return (line * 255.0).clip(0, 255).astype(np.uint8)
