"""What tests/golden/lineart_anime_golden.pt is made of, shared by tools/make_lineart_anime_golden.py and the anime
line-art tests.

Weights and images are regenerated from names by oracle/synth.py's frozen numpy stream (any machine gives the same
bits), so the fixture holds the reference's outputs, the state-dict keys and shapes, and input checksums only.  Block
outputs (blocks 1 ... 7 of UnetGenerator(3, 1, 8)) are stored at a fixed sample of pixel positions with all their
channels: whole blocks at 512 x 768 would be hundreds of MB.
"""
import zlib

import numpy as np
import torch

from oracle import synth

SEED = 23
NUM_DOWNS = 8                                        # LineartAnimeDetector builds UnetGenerator(3, 1, 8, 64, ...)
# 256^2: the 1 x 1 bottleneck and 2 x 2 instance norms; 512 x 768: the app's size.  The detector pads to multiples of
# 256 with cv2.resize, which copies at these sizes.
SIZES = {"256": (256, 256), "512": (512, 512), "512x768": (512, 768)}
DETECTOR_SIZE = (500, 740)                           # not a multiple of 256: both cubic resizes run
STAGE_FLOATS = 16384                                 # per stored block output: positions = STAGE_FLOATS // channels
MAP_BAND_ROWS = 128                                  # the fp32 map is stored in bands of rows (see map_bands)
OUT_CONV = "model.model.3.weight"                    # block 0's ConvTranspose2d(128 -> 1)
OUT_CONV_SCALE = 0.125


def weights(shapes):
    """{name: shape} -> the fixture's fp32 state dict.  synth_param scales a transposed kernel [Cin, Cout, 4, 4] by
    (16 Cout)^-1/2, which for the 128 -> 1 output conv would drive tanh into saturation (a map of 0s and 255s); the
    extra OUT_CONV_SCALE keeps the map in tanh's graded range."""
    sd = synth.synth_state_dict(shapes, SEED, "lineart_anime.")
    sd[OUT_CONV] = sd[OUT_CONV] * OUT_CONV_SCALE
    return sd


def image(size, tag=""):
    """uint8 HWC [H, W, 3] test image: 16-pixel blocks of coarse noise (edges for the detector) plus fine noise"""
    h, w = SIZES[size] if size in SIZES else size
    rs = synth._rs(f"lineart_anime.image.{h}x{w}{tag}", SEED)
    coarse = rs.uniform(0, 1, ((h + 15) // 16, (w + 15) // 16, 3)).repeat(16, 0).repeat(16, 1)[:h, :w]
    fine = rs.uniform(-0.15, 0.15, (h, w, 3))
    return np.clip((coarse + fine) * 255.0, 0, 255).astype(np.uint8)


def image_tensor(img):
    """LineartAnimeDetector.__call__'s network input for an image whose sides are multiples of 256: `float / 127.5 -
    1`, 'h w c -> 1 c h w' (fp32, on the host)"""
    return (torch.from_numpy(img).float() / 127.5 - 1.0).permute(2, 0, 1).unsqueeze(0).contiguous()


def stage_positions(h, w, channels):
    """sorted flat pixel indices (row-major over h x w) at which a block output is stored"""
    n = min(h * w, max(1, STAGE_FLOATS // channels))
    rs = synth._rs(f"lineart_anime.positions.{h}x{w}x{channels}", SEED)
    return np.sort(rs.choice(h * w, n, replace=False))


def sample_stage(t, idx):
    """fp32 [1, C, h, w] block output -> [C, len(idx)] at the given flat pixel indices"""
    return t[0].reshape(t.shape[1], -1)[:, torch.as_tensor(idx, device=t.device)].float().cpu().contiguous()


def map_bands(line):
    """fp32 [H, W] map -> {band name: rows}: the part splitter moves whole entries, so each band is an entry of its own"""
    return {f"rows{r:05d}": line[r:r + MAP_BAND_ROWS].clone() for r in range(0, line.shape[0], MAP_BAND_ROWS)}


def golden_map(golden, size):
    """the fp32 [H, W] network output of one size, reassembled from its bands"""
    bands = golden[f"{size}.map"]
    return torch.cat([bands[k] for k in sorted(bands)])


# ---- the line-art kernels' existing calls, recorded from the library before 512-channel norms and strided gathers
PARITY_GOLDEN = "lineart_anime_parity.pt"
# instance norm: (name, batch, h, w, channels, phases, relu, residual)
PARITY_NORMS = [("n64", 1, 32, 32, 64, False, True, False), ("n128", 2, 12, 20, 128, False, False, True),
                ("n256", 1, 16, 16, 256, False, True, False), ("p64", 1, 8, 12, 64, True, True, False),
                ("p256", 2, 6, 4, 256, True, True, False)]
# tap gather: (name, source shape, fp32 NCHW, taps, reflect, k_pad)
PARITY_GATHERS = [("g7", (1, 3, 24, 32), True, [(ky - 3, kx - 3) for ky in range(7) for kx in range(7)], True, 160),
                  ("g3", (1, 6, 8, 256), False, [(ky - 1, kx - 1) for ky in range(3) for kx in range(3)], True, 2304),
                  ("gz", (1, 10, 14, 128), False, [(0, 0), (0, 1), (1, 0), (1, 1)], False, 512)]


def parity_input(name, shape):
    """a seeded fp16 input (fp32 for the NCHW gather source) of a parity case, made on the host"""
    g = torch.Generator().manual_seed(zlib.crc32(f"lineart_anime.parity.{name}".encode()))
    return torch.randn(*shape, generator=g) * 3 + 2


def parity_calls(ops, device):
    """{case name: output} of every parity case through `ops` (the library `_lib.load()` returns)"""
    res = {}
    for name, b, h, w, c, phases, relu, residual in PARITY_NORMS:
        x = parity_input(name, (4, b, h, w, c) if phases else (b, h, w, c)).half().to(device)
        res_t = parity_input(name + ".res", (b, h, w, c)).half().to(device) if residual else None
        res[name] = ops.instance_norm(x, relu=relu, residual=res_t, phases=phases).cpu()
    for name, shape, f32, taps, reflect, k_pad in PARITY_GATHERS:
        x = parity_input(name, shape).to(device)
        res[name] = ops.tap_gather(x if f32 else x.half(), taps, reflect=reflect, k_pad=k_pad).cpu()
    return res
