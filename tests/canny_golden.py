"""What tests/golden/canny_golden.pt is made of, and a numpy / scipy restatement of cv2.Canny (apertureSize 3, L1
gradient) on uint8 H x W x 3 images, shared by tools/make_canny_golden.py and the Canny tests.  Test infrastructure
only: the product runs ctrlora_b200.annotator.canny.

The restatement's rules, in integer arithmetic:
1. per channel the 3 x 3 Sobel dx, dy with the border replicated, m = |dx| + |dy|; per pixel the (dx, dy, m) of the
   channel with the largest m, ties keeping the lowest channel;
2. lo = floor(low), hi = floor(high), swapped when lo > hi;
3. with x = |dx|, y = |dy| << 15: horizontal if y < x TG22, vertical if y > x TG22 + (x << 16), else diagonal;
4. magnitudes outside the image are 0; horizontal keeps m > m[left] && m >= m[right], vertical m > m[up] && m >=
   m[down], the diagonal with dx, dy of opposite sign m > m[up-right] && m > m[down-left], the other m > m[up-left] &&
   m > m[down-right];
5. candidate: kept and m > lo; strong: candidate and m > hi;
6. 255 at every candidate 8-connected through candidates to a strong pixel (scipy.ndimage.label), 0 elsewhere.
"""
import math

import cv2
import numpy as np
import scipy.ndimage

from oracle import synth

SEED = 61
TG22 = 13573
# the fixture: three kinds of content at four sizes, plus the spiral, each under every threshold pair
SIZES = {"512": (512, 512), "512x768": (512, 768), "768x512": (768, 512), "497x513": (497, 513)}
KINDS = ("smooth", "textured", "binary")
THRESHOLDS = ((100, 200), (1, 255), (200, 100), (150, 150), (100.5, 200.9))
SPIRAL_SIZE = (512, 512)


# ------------------------------------------------------------------------------------------------ the restatement
def thresholds(low, high):
    lo, hi = math.floor(low), math.floor(high)
    return (hi, lo) if lo > hi else (lo, hi)


def gradients(img):
    """uint8 [H, W, 3] -> int32 (dx, dy, m) [H, W] of the selected channel"""
    p = np.pad(img.astype(np.int32), ((1, 1), (1, 1), (0, 0)), mode="edge")
    dx = (p[:-2, 2:] + 2 * p[1:-1, 2:] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[1:-1, :-2] + p[2:, :-2])
    dy = (p[2:, :-2] + 2 * p[2:, 1:-1] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[:-2, 1:-1] + p[:-2, 2:])
    m = np.abs(dx) + np.abs(dy)
    c = m.argmax(-1)[..., None]  # the first of equal maxima: the lowest channel
    pick = lambda t: np.take_along_axis(t, c, -1)[..., 0]  # noqa: E731
    return pick(dx), pick(dy), pick(m)


def classes(img, lo, hi):
    """uint8 [H, W]: 0 none, 1 candidate, 2 strong (rules 1, 3-5) for integer thresholds lo <= hi"""
    dx, dy, m = gradients(img)
    h, w = m.shape
    mp = np.pad(m, 1)
    nb = lambda oy, ox: mp[1 + oy:1 + oy + h, 1 + ox:1 + ox + w]  # noqa: E731
    ax, ay = np.abs(dx).astype(np.int64), np.abs(dy).astype(np.int64) << 15
    tg22x = ax * TG22
    horiz = ay < tg22x
    vert = ~horiz & (ay > tg22x + (ax << 16))
    keep = np.where(horiz, (m > nb(0, -1)) & (m >= nb(0, 1)),
                    np.where(vert, (m > nb(-1, 0)) & (m >= nb(1, 0)),
                             np.where((dx ^ dy) < 0, (m > nb(-1, 1)) & (m > nb(1, -1)),
                                      (m > nb(-1, -1)) & (m > nb(1, 1)))))
    cand = keep & (m > lo)
    return cand.astype(np.uint8) + (cand & (m > hi)).astype(np.uint8)


def hysteresis(cls):
    """uint8 [H, W] classes -> uint8 [H, W] map: 255 on the 8-connected candidate components holding a strong pixel"""
    lab, _ = scipy.ndimage.label(cls > 0, structure=np.ones((3, 3), dtype=bool))
    strong = np.unique(lab[cls == 2])
    return np.where(np.isin(lab, strong[strong > 0]), 255, 0).astype(np.uint8)


def canny(img, low, high):
    """the restatement of cv2.Canny(img, low, high) on uint8 [H, W, 3]"""
    return hysteresis(classes(img, *thresholds(low, high)))


# ------------------------------------------------------------------------------------------------ content
def image(kind, h, w, tag=""):
    """a seeded uint8 [h, w, 3] image: smooth (a bilinearly upsampled coarse field), textured (coarse blocks plus fine
    noise on a few levels), binary (0 / 255 blocks and discs), random (uniform noise) or quantised (smooth on 4
    levels per channel)"""
    rs = synth._rs(f"canny.{kind}.{h}x{w}{tag}", SEED)
    if kind in ("smooth", "quantised"):
        coarse = rs.randint(0, 256, (h // 10 + 2, w // 10 + 2, 3)).astype(np.uint8)
        img = cv2.resize(coarse, (w, h), interpolation=cv2.INTER_LINEAR)
        return img if kind == "smooth" else (img // 64 * 85).astype(np.uint8)
    if kind == "textured":
        blocks = rs.randint(0, 256, (h // 12 + 1, w // 12 + 1, 3)).repeat(12, 0).repeat(12, 1)[:h, :w]
        fine = rs.randint(-1, 2, (h, w, 3)) * 12
        return np.clip(blocks + fine, 0, 255).astype(np.uint8)
    if kind == "binary":
        img = np.ascontiguousarray((rs.uniform(size=(h // 9 + 1, w // 9 + 1)) > 0.6).repeat(9, 0).repeat(9, 1)[:h, :w])
        img = img.astype(np.uint8) * 255
        for _ in range(max(1, h * w // 20000)):
            cx, cy, r = int(rs.randint(0, w)), int(rs.randint(0, h)), int(rs.randint(3, 40))
            cv2.circle(img, (cx, cy), r, int(rs.choice([0, 255])), -1)
        return np.repeat(img[..., None], 3, -1)
    if kind == "random":
        return rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    raise ValueError(kind)


def spiral(h=SPIRAL_SIZE[0], w=SPIRAL_SIZE[1], period=6, level=40):
    """a square spiral band at `level` on 0, 2 pixels wide with `period` pixels between turns, winding in from the
    border to the centre.  Under (100, 200) its edges form one 8-connected candidate component of about 87 000 pixels,
    strong only at the band's corners."""
    pts = []
    top, left, bottom, right = 2, 2, h - 3, w - 3
    while top < bottom and left < right:
        pts += [(left, top), (right, top), (right, bottom), (left, bottom), (left, top + period)]
        top, left, bottom, right = top + period, left + period, bottom - period, right - period
    img = np.zeros((h, w), dtype=np.uint8)
    cv2.polylines(img, [np.array(pts, dtype=np.int32)], False, level, 2)
    return np.repeat(img[..., None], 3, -1)


def pack(m):
    """uint8 0 / 255 map [H, W] -> the bit-packed bytes (np.packbits, row-major)"""
    return np.packbits(m.reshape(-1) > 0)


def unpack(bits, h, w):
    return (np.unpackbits(np.asarray(bits), count=h * w).reshape(h, w) * 255).astype(np.uint8)


def cases():
    """the fixture's images: [(name, uint8 [H, W, 3])]"""
    out = [(f"{kind}.{size}", image(kind, *hw)) for size, hw in SIZES.items() for kind in KINDS]
    return out + [("spiral", spiral())]


# ------------------------------------------------------------------------------------------------ seeded cases
CASE_KINDS = ("smooth", "textured", "binary", "random", "quantised")
# tiny, one-row and one-column images, sizes off the kernels' tiles and a few at tile multiples
CASE_SIZES = ((1, 1), (1, 13), (13, 1), (2, 3), (3, 2), (16, 32), (17, 33), (33, 65), (64, 96), (100, 37), (130, 257))
# swapped, fractional, zero, negative and out-of-range thresholds among the usual ones
CASE_THRESHOLDS = ((100, 200), (200, 100), (0, 0), (-5, 40), (0.5, 0.7), (150, 150), (1, 255), (2040, 2041),
                   (3000, 5000), (-10, -1), (37.9, 512.2), (100.5, 200.9), (-0.5, 60), (255, 1))
CASES_PER_IMAGE = 6


def seeded_cases():
    """[(name, uint8 [H, W, 3], low, high)]: every kind at every size under CASES_PER_IMAGE threshold pairs, 330 cases"""
    out, k = [], 0
    for kind in CASE_KINDS:
        for h, w in CASE_SIZES:
            img = image(kind, h, w, tag=".case")
            for _ in range(CASES_PER_IMAGE):
                lo, hi = CASE_THRESHOLDS[k % len(CASE_THRESHOLDS)]
                out.append((f"{kind}.{h}x{w}.{lo}_{hi}", img, lo, hi))
                k += 1
    return out
