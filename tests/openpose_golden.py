"""What tests/golden/openpose_golden.pt is made of, shared by tools/make_openpose_golden.py and the OpenPose tests.

Weights, images and the planted stride-8 maps are regenerated from names by oracle/synth.py's frozen numpy stream and
closed-form geometry (any machine gives the same bits), so the fixture holds the reference's outputs only.

- Network cases: bodypose_model with synthetic He-scaled weights (every conv followed by a ReLU gets sqrt(2) on top of
  synth's fan_in ** -0.5, so six stages neither die out nor blow up) at the network inputs of four image sizes.
- Post-process cases: Body.__call__ and OpenposeDetector.__call__ with the network replaced by planted stride-8 maps:
  Gaussian keypoint blobs and PAF fields along the limbs of a few skeletons, plus distractors (a lone blob, a blob below
  the 0.1 threshold, a PAF patch with no parts).  Blob centres sit at asymmetric sub-pixel offsets.
"""
import math

import cv2
import numpy as np
import scipy.ndimage
import torch

from oracle import synth

SEED = 17
NET_SIZES = {"512": (512, 512), "384x640": (384, 640), "200x328": (200, 328), "120x200": (120, 200)}
BLOB_SIGMA = 0.85   # keypoint blobs, in stride-8 pixels
PAF_SIGMA = 1.0     # PAF tube half-width scale, in stride-8 pixels

# a standing person in units of its height, parts in the reference's order: nose, neck, r/l shoulder, elbow, wrist
# (right first), r/l hip, knee, ankle, r/l eye, r/l ear (the reference's 18 parts)
_TEMPLATE = ((0.013, -0.452), (0.0, -0.31), (-0.121, -0.303), (-0.163, -0.097), (-0.187, 0.081), (0.127, -0.301),
             (0.171, -0.093), (0.203, 0.072), (-0.083, 0.079), (-0.094, 0.297), (-0.106, 0.509), (0.081, 0.083),
             (0.103, 0.301), (0.117, 0.497), (-0.031, -0.487), (0.047, -0.484), (-0.069, -0.463), (0.081, -0.459))

# post-process cases: image size and people (centre x, centre y, height in stride-8 pixels, parts left out)
PP_CASES = {
    "320x448": {"size": (320, 448), "people": ((9.37, 11.61, 17.3, ()), (23.71, 11.23, 15.9, (7,)),
                                                (30.13, 17.42, 7.7, (0, 14, 15, 16, 17, 8, 9, 10))),
                "lone": (4, 29.41, 3.27), "weak": (6, 3.62, 20.84), "paf_patch": (2, 17.2, 20.9, 19.6, 21.3)},
    "512x384": {"size": (512, 384), "people": ((8.83, 11.37, 19.1, (3, 4)), (14.27, 7.61, 8.3, (9, 10, 12, 13))),
                "lone": (0, 15.63, 19.28), "weak": (11, 2.71, 2.46), "paf_patch": (10, 3.1, 19.2, 5.8, 21.7)},
}
WEAK_AMP = 0.06     # the blob below the peak threshold after smoothing


def weights(shapes):
    """{name: shape} -> the fixture's fp32 state dict (keys as bodypose_model's)"""
    from ctrlora_b200.annotator.openpose import no_relu_layers
    no_relu = set(no_relu_layers())
    sd = synth.synth_state_dict(shapes, SEED, "openpose.")
    for k, v in sd.items():
        layer = k.split(".")[1]
        if k.endswith(".weight") and layer not in no_relu:
            sd[k] = v * np.float32(2.0 ** 0.5)
    return sd


def image(size, tag=""):
    """uint8 HWC [H, W, 3] test image: 8-pixel blocks of coarse noise plus fine noise"""
    h, w = NET_SIZES[size] if size in NET_SIZES else size
    return synth.noise_image(f"openpose.image.{h}x{w}{tag}", SEED, h, w, 8, 0.2)


def _blob(h8, w8, cx, cy, amp=1.0):
    y, x = np.mgrid[0:h8, 0:w8].astype(np.float64)
    return amp * np.exp(-((x - cx) ** 2 + (y - cy) ** 2) / (2 * BLOB_SIGMA ** 2))


def _tube(h8, w8, ax, ay, bx, by):
    """(weight map, unit vector) of a PAF field along the segment A -> B"""
    y, x = np.mgrid[0:h8, 0:w8].astype(np.float64)
    vx, vy = bx - ax, by - ay
    n = max(np.hypot(vx, vy), 1e-9)
    ux, uy = vx / n, vy / n
    t = np.clip((x - ax) * ux + (y - ay) * uy, 0.0, n)
    d2 = (x - ax - t * ux) ** 2 + (y - ay - t * uy) ** 2
    return np.exp(-d2 / (2 * PAF_SIGMA ** 2)), ux, uy


def planted_maps(case):
    """fp32 (PAFs [1, 38, h8, w8], heatmaps [1, 19, h8, w8]) of a post-process case, at the network output size of its
    image"""
    from ctrlora_b200.annotator.openpose import LIMB_PAF, LIMB_PARTS, geometry
    spec = PP_CASES[case]
    h, w = spec["size"]
    _, _, ph, pw = geometry(h, w)
    h8, w8 = ph // 8, pw // 8
    heat = np.zeros((19, h8, w8))
    paf = np.zeros((38, h8, w8))
    for cx, cy, height, missing in spec["people"]:
        pts = [(cx + height * tx, cy + height * ty) for tx, ty in _TEMPLATE]
        for p, (x, y) in enumerate(pts):
            if p not in missing:
                heat[p] = np.maximum(heat[p], _blob(h8, w8, x, y, 0.93))
        for (a, b), (c0, c1) in zip(LIMB_PARTS, LIMB_PAF):
            if a - 1 in missing or b - 1 in missing:
                continue
            wt, ux, uy = _tube(h8, w8, *pts[a - 1], *pts[b - 1])
            paf[c0 - 19] += wt * ux
            paf[c1 - 19] += wt * uy
    p, x, y = spec["lone"]
    heat[p] = np.maximum(heat[p], _blob(h8, w8, x, y, 0.71))
    p, x, y = spec["weak"]
    heat[p] = np.maximum(heat[p], _blob(h8, w8, x, y, WEAK_AMP))
    k, ax, ay, bx, by = spec["paf_patch"]
    wt, ux, uy = _tube(h8, w8, ax, ay, bx, by)
    c0, c1 = LIMB_PAF[k]
    paf[c0 - 19] += wt * ux
    paf[c1 - 19] += wt * uy
    heat[18] = np.clip(1.0 - heat[:18].max(axis=0), 0, 1)
    return torch.from_numpy(paf[None].astype(np.float32)), torch.from_numpy(heat[None].astype(np.float32))


def dummy_image(case):
    """the uint8 image handed to the stubbed Body / OpenposeDetector (only its size matters to them)"""
    h, w = PP_CASES[case]["size"]
    return image((h, w), tag=".pp")


def pair_scores(paf, candidate, counts, img_h):
    """float64 restatement of body.py:107-131 on the full-size PAFs [H, W, 38]: per limb with peaks at both ends, the
    (i, j, score, samples) of every pair, with numpy's operations in the reference's order"""
    from ctrlora_b200.annotator import openpose as op
    first = np.concatenate([[0], np.cumsum(counts)])
    out = {}
    for k, ((a, b), (c0, c1)) in enumerate(zip(op.LIMB_PARTS, op.LIMB_PAF)):
        if not counts[a - 1] or not counts[b - 1]:
            continue
        ca, cb = candidate[first[a - 1]:first[a]], candidate[first[b - 1]:first[b]]
        rows = []
        for i, pa in enumerate(ca):
            for j, pb in enumerate(cb):
                vec = np.array([pb[0] - pa[0], pb[1] - pa[1]])
                norm = max(0.001, math.sqrt(vec[0] * vec[0] + vec[1] * vec[1]))
                vec = vec / norm
                xs, ys = np.linspace(pa[0], pb[0], num=op.MID_NUM), np.linspace(pa[1], pb[1], num=op.MID_NUM)
                pts = [(int(round(y)), int(round(x))) for x, y in zip(xs, ys)]
                vx = np.array([paf[y, x, c0 - 19] for y, x in pts], np.float64)
                vy = np.array([paf[y, x, c1 - 19] for y, x in pts], np.float64)
                samples = vx * vec[0] + vy * vec[1]
                score = sum(samples) / len(samples) + min(0.5 * img_h / norm - 1, 0)
                rows.append((i, j, score, samples))
        out[k] = rows
    return out


def host_postprocess(paf8, heat8, h, w):
    """Body's post-process on the host as the reference runs it (numpy / cv2 / scipy, one channel at a time), on
    stride-8 maps (numpy float32 [38, h8, w8] and [19, h8, w8]) for an h x w image -> (candidate, subset).  The
    baseline of tools/openpose_bench.py."""
    from ctrlora_b200.annotator import openpose as op
    rh, rw, ph, pw = op.geometry(h, w)
    interp = op.resize_interp(rh, rw, h, w)

    def full(maps):
        return np.stack([cv2.resize(cv2.resize(m, (pw, ph), interpolation=cv2.INTER_LANCZOS4)[:rh, :rw], (w, h),
                                    interpolation=interp) for m in maps], axis=2).astype(np.float64)
    heat, paf = full(heat8), full(paf8)
    px, py, sc, counts = [], [], [], []
    for part in range(op.N_PARTS):
        s = scipy.ndimage.gaussian_filter(heat[:, :, part], sigma=3)
        p = np.pad(s, 1)
        ys, xs = np.nonzero((s >= p[:-2, 1:-1]) & (s >= p[2:, 1:-1]) & (s >= p[1:-1, :-2]) & (s >= p[1:-1, 2:]) &
                            (s > op.THRE_PEAK))
        px += xs.tolist()
        py += ys.tolist()
        sc += heat[ys, xs, part].tolist()
        counts.append(len(xs))
    candidate = op.make_candidate(px, py, sc)
    limbs = [None] * len(op.LIMB_PARTS)
    for k, rows in pair_scores(paf, candidate, counts, h).items():
        limbs[k] = [(i, j, s) for i, j, s, smp in rows
                    if (smp > op.THRE_PAF).sum() > 0.8 * len(smp) and s > 0]
    return candidate, op.assemble(candidate, np.array(counts), limbs)
