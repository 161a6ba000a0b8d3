"""What tests/golden/lineart_golden.pt is made of, shared by tools/make_lineart_golden.py and the line-art tests.

Weights and images are regenerated from names by oracle/synth.py's frozen numpy stream (any machine gives the same
bits), so the fixture holds the reference's outputs, the state-dict keys and shapes, and input checksums only.  Stage
activations (the outputs of model0 ... model3) are stored at a fixed sample of pixel positions with all their
channels: whole stages at 512 x 512 would be hundreds of MB.
"""
import numpy as np
import torch

from oracle import synth

SEED = 11
N_RESIDUAL = 3                                       # LineartDetector builds Generator(3, 1, 3)
SIZES = {"512": (512, 512), "384x640": (384, 640), "64": (64, 64)}
STAGE_FLOATS = 32768                                 # per stored stage: positions = STAGE_FLOATS // channels
MAP_BAND_ROWS = 128                                  # the fp32 map is stored in bands of rows (see map_bands)


def weights(shapes):
    """{name: shape} -> the fixture's fp32 state dict"""
    return synth.synth_state_dict(shapes, SEED, "lineart.")


def image(size, tag=""):
    """uint8 HWC [H, W, 3] test image: 16-pixel blocks of coarse noise (edges for the detector) plus fine noise"""
    h, w = SIZES[size] if size in SIZES else size
    rs = synth._rs(f"lineart.image.{h}x{w}{tag}", SEED)
    coarse = rs.uniform(0, 1, ((h + 15) // 16, (w + 15) // 16, 3)).repeat(16, 0).repeat(16, 1)[:h, :w]
    fine = rs.uniform(-0.15, 0.15, (h, w, 3))
    return np.clip((coarse + fine) * 255.0, 0, 255).astype(np.uint8)


def stage_positions(h, w, channels):
    """sorted flat pixel indices (row-major over h x w) at which a stage is stored"""
    n = min(h * w, STAGE_FLOATS // channels)
    rs = synth._rs(f"lineart.positions.{h}x{w}x{channels}", SEED)
    return np.sort(rs.choice(h * w, n, replace=False))


def sample_stage(t, idx):
    """fp32 [1, C, h, w] stage -> [C, len(idx)] at the given flat pixel indices"""
    return t[0].reshape(t.shape[1], -1)[:, torch.as_tensor(idx, device=t.device)].float().cpu().contiguous()


def map_bands(line):
    """fp32 [H, W] map -> {band name: rows}: a 512 x 512 map is 1 MB, more than one fixture part file may hold, and the
    part splitter moves whole entries, so each band is an entry of its own"""
    return {f"rows{r:05d}": line[r:r + MAP_BAND_ROWS].clone() for r in range(0, line.shape[0], MAP_BAND_ROWS)}


def golden_map(golden, size):
    """the fp32 [H, W] map of one size, reassembled from its bands"""
    bands = golden[f"{size}.map"]
    return torch.cat([bands[k] for k in sorted(bands)])


def quantise(line):
    """LineartDetector.__call__'s `(line * 255.0).clip(0, 255).astype(np.uint8)` on an fp32 numpy map"""
    return (line * 255.0).clip(0, 255).astype(np.uint8)
