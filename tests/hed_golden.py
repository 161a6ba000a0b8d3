"""What tests/golden/hed_golden.pt is made of, shared by tools/make_hed_golden.py and the HED tests.

Weights and images are regenerated from names by oracle/synth.py's frozen numpy stream (any machine gives the same
bits), so the fixture holds the reference's outputs, the state-dict keys and shapes, and input checksums only.  The
synthetic weights are adjusted so that the comparison is not vacuous: `norm` lies in 90 ... 150 (the input is RGB in
0 ... 255), the 3x3 convs are He-scaled (each ReLU halves the second moment, and 13 of them would otherwise shrink
the activations by 2^13), and the projections are scaled and offset so that the pre-sigmoid mean map is centred near 0 with a std of
about 2, which spreads the uint8 map and safe_step's bins.  Stage activations (the five blocks' outputs) are stored at a fixed sample
of pixel positions with all their channels.
"""
import functools

import cv2
import numpy as np
import torch

import golden_io
from golden_io import sample_stage, unband  # noqa: F401 (sample_stage)
from oracle import synth

SEED = 13
SIZES = {"512": (512, 512), "384x640": (384, 640), "200x328": (200, 328)}
STAGE_FLOATS = 16384                                 # per stored stage: positions = STAGE_FLOATS // channels
MAP_BAND_ROWS = 128                                  # full-size fp32 maps are stored in bands of rows
PROJ_SCALE = 0.12                                    # on top of synth's fan_in ** -0.5 (see the module docstring)
# projection biases that centre each side map of the test images near 0 (measured once at 200 x 328)
PROJ_BIAS = (2.0, -6.9, -4.6, 0.3, -13.3)
SKETCH_SEEDS = {"hed": (0, 1, 2), "dark": (0,)}  # HED-sketch cases: np.random.seed before each call


def weights(shapes):
    """{name: shape} -> the fixture's fp32 state dict"""
    sd = synth.synth_state_dict(shapes, SEED, "hed.")
    for k, v in sd.items():
        if k == "norm":
            sd[k] = torch.from_numpy(synth._rs("hed.norm", SEED).uniform(90.0, 150.0, tuple(v.shape)).astype(np.float32))
        elif ".convs." in k and k.endswith(".weight"):
            sd[k] = v * np.float32(2.0 ** 0.5)
        elif k.endswith("projection.weight"):
            sd[k] = v * np.float32(PROJ_SCALE)
        elif k.endswith("projection.bias"):
            sd[k] = torch.full_like(v, PROJ_BIAS[int(k[len("block")]) - 1])
    return sd


def image(size, tag=""):
    """uint8 HWC [H, W, 3] test image: 16-pixel blocks of coarse noise (edges for the detector) plus fine noise"""
    h, w = SIZES[size] if size in SIZES else size
    return synth.noise_image(f"hed.image.{h}x{w}{tag}", SEED, h, w, 16, 0.15)


stage_positions = functools.partial(golden_io.stage_positions, "hed", SEED, STAGE_FLOATS)
map_bands = functools.partial(golden_io.bands, rows=MAP_BAND_ROWS)  # a 512 x 512 map is 1 MB, more than a part file


def golden_map(golden, size, name):
    """a full-size fp32 [H, W] map ("mean" or "e1") of one size, reassembled from its bands"""
    return unband(golden[f"{size}.{name}"])


def dark(edge):
    """the HED-sketch cases' second input: the uint8 HED map at 45 % brightness, so that few pixels pass the first
    thresholds and the retry loop runs"""
    return (edge.astype(np.float32) * 0.45).astype(np.uint8)


def host_post(side_maps, safe=False):
    """HEDdetector's host post-process (annotator/hed/__init__.py:70-78) in numpy / cv2, on the five float32 [h_l, w_l]
    side maps: each map bilinearly resized to the first one's size (cv2 INTER_LINEAR), their float32 mean over the
    stacked last axis, the logistic function in float64, optionally annotator.util.safe_step (float32 x 3, int32
    truncation, / 2), and the uint8 cast of the map x 255 clipped to [0, 255].  Returns (float32 mean map, uint8 map)."""
    rows, cols = side_maps[0].shape
    stacked = np.stack([cv2.resize(np.asarray(m, dtype=np.float32), (cols, rows), interpolation=cv2.INTER_LINEAR)
                        for m in side_maps], axis=-1)
    mean = stacked.mean(axis=-1)
    prob = np.reciprocal(1.0 + np.exp(-mean.astype(np.float64)))
    if safe:
        prob = np.trunc(prob.astype(np.float32) * np.float32(3.0)).astype(np.int32).astype(np.float32) / np.float32(2.0)
    return mean, np.clip(prob * 255.0, 0, 255).astype(np.uint8)
