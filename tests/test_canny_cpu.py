"""The Canny annotator without a GPU: tests/canny_golden.py's restatement against the reference's maps
(tests/golden/canny_golden.pt) and against live cv2.Canny, the detector's host-side thresholds and input checks, and
tests/canny_launches.py's launch references against index loops."""
import os
import sys

import cv2
import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_io import load_golden  # noqa: E402
import canny_golden as cg  # noqa: E402
import canny_launches as CL  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "canny_golden.pt")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def test_fixture_layout(golden):
    assert golden["seed"] == cg.SEED
    assert [tuple(t) for t in golden["thresholds"]] == list(cg.THRESHOLDS)
    assert golden["cases"] == [name for name, _ in cg.cases()]


def test_fixture_inputs_are_the_seeded_images(golden):
    for name, img in cg.cases():
        assert np.array_equal(cv2.imdecode(golden[f"{name}.png"].numpy(), cv2.IMREAD_UNCHANGED), img), name


def test_restatement_matches_the_fixture(golden):
    for name in golden["cases"]:
        img = cv2.imdecode(golden[f"{name}.png"].numpy(), cv2.IMREAD_UNCHANGED)
        h, w = golden[f"{name}.shape"]
        for i, (lo, hi) in enumerate(golden["thresholds"]):
            ref = cg.unpack(golden[f"{name}.map{i}"].numpy(), h, w)
            assert int((cg.canny(img, lo, hi) != ref).sum()) == 0, (name, lo, hi)


def test_restatement_matches_live_cv2():
    cases = cg.seeded_cases()
    assert len(cases) >= 300
    bad = [(name, int((cg.canny(img, lo, hi) != cv2.Canny(img, lo, hi)).sum()))
           for name, img, lo, hi in cases if not np.array_equal(cg.canny(img, lo, hi), cv2.Canny(img, lo, hi))]
    assert not bad, bad


def test_restatement_matches_cv2_on_the_spiral_and_a_large_image():
    for img in (cg.spiral(), cg.image("random", 1024, 1024)):
        for lo, hi in ((100, 200), (1, 255)):
            assert np.array_equal(cg.canny(img, lo, hi), cv2.Canny(img, lo, hi))


@pytest.mark.parametrize("low,high,want", [
    ((100, 200), None, (100, 200)), ((200, 100), None, (100, 200)), ((100.5, 200.9), None, (100, 200)),
    ((150, 150), None, (150, 150)), ((-0.5, 3.2), None, (-1, 3)), ((0.9, 0.1), None, (0, 0)),
    ((7.99, -2.01), None, (-3, 7)), ((3000, 5000.5), None, (3000, 5000)),
])
def test_thresholds_floor_and_swap(low, high, want):
    from ctrlora_b200.annotator.canny import thresholds
    assert thresholds(*low) == want == cg.thresholds(*low)


def test_thresholds_beyond_the_magnitudes_act_as_clamped():
    """ops.canny_classify clamps its integer thresholds to [-1, 2040] before the ABI; the classes do not change"""
    from ctrlora_b200 import ops
    assert ops.CANNY_MAX_MAG == 4 * 255 + 4 * 255
    img = cg.image("random", 40, 50)
    for lo, hi, clo, chi in ((-100, 5000, -1, 2040), (2040, 99999, 2040, 2040), (-7, -2, -1, -1)):
        assert np.array_equal(cg.classes(img, lo, hi), cg.classes(img, clo, chi))


def test_bad_input_raises():
    from ctrlora_b200.annotator.canny import CannyDetector
    det = CannyDetector()
    for bad in (np.zeros((8, 8), np.uint8), np.zeros((8, 8, 4), np.uint8), np.zeros((8, 8, 1), np.uint8),
                np.zeros((8, 8, 3), np.float32), np.zeros((8, 8, 3), np.int16), np.zeros((0, 8, 3), np.uint8),
                [[0, 0, 0]], torch.zeros(8, 8, 3, dtype=torch.uint8)):
        with pytest.raises(ValueError):
            det(bad, 100, 200)
    for bad in (torch.zeros(8, 8, 3, dtype=torch.uint8), torch.zeros(1, 8, 8, 4, dtype=torch.uint8),
                torch.zeros(1, 8, 8, 3, dtype=torch.float32)):
        with pytest.raises(ValueError):
            det.detect(bad, 100, 200)


def test_detector_is_built_without_arguments():
    from ctrlora_b200.annotator.canny import CannyDetector
    assert CannyDetector().device == torch.device("cuda")
    with pytest.raises(RuntimeError):
        CannyDetector(device="cpu")


# ------------------------------------------------------------------------------------------------ launch references
def _classes_loop(img, lo, hi):
    """rules 1, 3-5 pixel by pixel"""
    h, w, _ = img.shape
    px = lambda y, x, c: int(img[min(max(y, 0), h - 1), min(max(x, 0), w - 1), c])  # noqa: E731
    grad = {}
    for y in range(h):
        for x in range(w):
            best = None
            for c in range(3):
                dx = (px(y - 1, x + 1, c) + 2 * px(y, x + 1, c) + px(y + 1, x + 1, c)) - \
                     (px(y - 1, x - 1, c) + 2 * px(y, x - 1, c) + px(y + 1, x - 1, c))
                dy = (px(y + 1, x - 1, c) + 2 * px(y + 1, x, c) + px(y + 1, x + 1, c)) - \
                     (px(y - 1, x - 1, c) + 2 * px(y - 1, x, c) + px(y - 1, x + 1, c))
                if best is None or abs(dx) + abs(dy) > best[2]:
                    best = (dx, dy, abs(dx) + abs(dy))
            grad[y, x] = best
    mag = lambda y, x: grad[y, x][2] if 0 <= y < h and 0 <= x < w else 0  # noqa: E731
    out = np.zeros((h, w), np.uint8)
    for y in range(h):
        for x in range(w):
            dx, dy, m = grad[y, x]
            ax, ay = abs(dx), abs(dy) << 15
            if ay < ax * cg.TG22:
                keep = m > mag(y, x - 1) and m >= mag(y, x + 1)
            elif ay > ax * cg.TG22 + (ax << 16):
                keep = m > mag(y - 1, x) and m >= mag(y + 1, x)
            elif (dx < 0) != (dy < 0):
                keep = m > mag(y - 1, x + 1) and m > mag(y + 1, x - 1)
            else:
                keep = m > mag(y - 1, x - 1) and m > mag(y + 1, x + 1)
            if keep and m > lo:
                out[y, x] = 2 if m > hi else 1
    return out


def _hysteresis_loop(cls):
    """a flood fill from every strong pixel through 8-connected candidates"""
    h, w = cls.shape
    out = np.zeros((h, w), np.uint8)
    stack = [(y, x) for y in range(h) for x in range(w) if cls[y, x] == 2]
    while stack:
        y, x = stack.pop()
        if out[y, x]:
            continue
        out[y, x] = 255
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                yy, xx = y + dy, x + dx
                if 0 <= yy < h and 0 <= xx < w and cls[yy, xx] and not out[yy, xx]:
                    stack.append((yy, xx))
    return out


@pytest.mark.parametrize("kind", cg.CASE_KINDS)
def test_classify_reference_against_an_index_loop(kind):
    for h, w in ((1, 1), (1, 9), (7, 1), (13, 17)):
        imgs = np.stack([cg.image(kind, h, w, tag=f".loop{i}") for i in range(2)])
        for lo, hi in ((100, 200), (0, 0), (-1, 30), (20, 60)):
            got = CL.canny_classify(torch.from_numpy(imgs), lo, hi).numpy()
            for img, g in zip(imgs, got):
                assert np.array_equal(g, _classes_loop(img, lo, hi)), (kind, h, w, lo, hi)


def test_hysteresis_reference_against_an_index_loop():
    rs = np.random.RandomState(3)
    for h, w, p in ((1, 1, 0.9), (1, 30, 0.7), (30, 1, 0.7), (23, 29, 0.45), (40, 40, 0.3)):
        cls = np.stack([(rs.uniform(size=(h, w)) < p).astype(np.uint8) for _ in range(2)])
        cls[cls > 0] += (rs.uniform(size=int((cls > 0).sum())) < 0.05).astype(np.uint8)
        got = CL.canny_hysteresis(torch.from_numpy(cls)).numpy()
        for c, g in zip(cls, got):
            assert np.array_equal(g, _hysteresis_loop(c)), (h, w, p)
