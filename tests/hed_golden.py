"""What tests/golden/hed_golden.pt is made of, shared by tools/make_hed_golden.py and the HED tests.

Weights and images are regenerated from names by oracle/synth.py's frozen numpy stream (any machine gives the same
bits), so the fixture holds the reference's outputs, the state-dict keys and shapes, and input checksums only.  The
synthetic weights are adjusted so that the comparison is not vacuous: `norm` lies in 90 ... 150 (the input is RGB in
0 ... 255), the 3x3 convs are He-scaled (each ReLU halves the second moment, and 13 of them would otherwise shrink
the activations by 2^13), and the projections are scaled and offset so that the pre-sigmoid mean map is centred near 0 with a std of
about 2, which spreads the uint8 map and safe_step's bins.  Stage activations (the five blocks' outputs) are stored at a fixed sample
of pixel positions with all their channels.
"""
import cv2
import numpy as np
import torch

from oracle import synth

SEED = 13
SIZES = {"512": (512, 512), "384x640": (384, 640), "200x328": (200, 328)}
STAGE_FLOATS = 16384                                 # per stored stage: positions = STAGE_FLOATS // channels
MAP_BAND_ROWS = 128                                  # full-size fp32 maps are stored in bands of rows (see map_bands)
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
    rs = synth._rs(f"hed.image.{h}x{w}{tag}", SEED)
    coarse = rs.uniform(0, 1, ((h + 15) // 16, (w + 15) // 16, 3)).repeat(16, 0).repeat(16, 1)[:h, :w]
    fine = rs.uniform(-0.15, 0.15, (h, w, 3))
    return np.clip((coarse + fine) * 255.0, 0, 255).astype(np.uint8)


def stage_positions(h, w, channels):
    """sorted flat pixel indices (row-major over h x w) at which a stage is stored"""
    n = min(h * w, STAGE_FLOATS // channels)
    rs = synth._rs(f"hed.positions.{h}x{w}x{channels}", SEED)
    return np.sort(rs.choice(h * w, n, replace=False))


def sample_stage(t, idx):
    """fp32 [1, C, h, w] stage -> [C, len(idx)] at the given flat pixel indices"""
    return t[0].reshape(t.shape[1], -1)[:, torch.as_tensor(idx, device=t.device)].float().cpu().contiguous()


def map_bands(m):
    """fp32 [H, W] map -> {band name: rows}: a 512 x 512 map is 1 MB, more than one fixture part file may hold, and the
    part splitter moves whole entries, so each band is an entry of its own"""
    return {f"rows{r:05d}": m[r:r + MAP_BAND_ROWS].clone() for r in range(0, m.shape[0], MAP_BAND_ROWS)}


def golden_map(golden, size, name):
    """a full-size fp32 [H, W] map ("mean" or "e1") of one size, reassembled from its bands"""
    bands = golden[f"{size}.{name}"]
    return torch.cat([bands[k] for k in sorted(bands)])


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
