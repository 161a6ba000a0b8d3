"""The Canny annotator on an H100, bit for bit: CannyDetector.__call__ against live cv2.Canny and against the reference's
maps (tests/golden/canny_golden.pt) on every fixture case, the seeded cases of tests/test_canny_cpu.py, the class map
against the restatement's, adversarial hysteresis inputs, batches, repeat calls, a CUDA-graph replay of `detect`, the
launch count and the launch shadow.  Every comparison counts mismatching pixels and requires 0."""
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

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "canny_golden.pt")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


@pytest.fixture(scope="module")
def det():
    from ctrlora_b200.annotator.canny import CannyDetector
    return CannyDetector()


def _mismatch(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, a.dtype, b.shape, b.dtype)
    return int((a != b).sum())


def _image(golden, name):
    return cv2.imdecode(golden[f"{name}.png"].numpy(), cv2.IMREAD_UNCHANGED)


def test_fixture_cases(golden, det):
    bad = []
    for name in golden["cases"]:
        img = _image(golden, name)
        h, w = golden[f"{name}.shape"]
        for i, (lo, hi) in enumerate(golden["thresholds"]):
            got = det(img, low_threshold=lo, high_threshold=hi)
            assert got.shape == (h, w) and got.dtype == np.uint8
            n_ref = _mismatch(got, cg.unpack(golden[f"{name}.map{i}"].numpy(), h, w))
            n_cv2 = _mismatch(got, cv2.Canny(img, lo, hi))
            if n_ref or n_cv2:
                bad.append((name, lo, hi, n_ref, n_cv2))
    assert not bad, f"pixels differing (fixture, cv2): {bad}"


def test_seeded_cases(det):
    bad = []
    for name, img, lo, hi in cg.seeded_cases():
        n = _mismatch(det(img, lo, hi), cv2.Canny(img, lo, hi))
        if n:
            bad.append((name, n))
    assert not bad, bad


@pytest.mark.parametrize("h,w", [(1, 1), (1, 40), (40, 1), (17, 33), (255, 257), (512, 768)])
def test_classes_against_the_restatement(h, w):
    """the class map alone, so that the hysteresis cannot hide a classification bug"""
    from ctrlora_b200 import ops
    for kind in cg.CASE_KINDS:
        img = cg.image(kind, h, w, tag=".classes")
        for lo, hi in ((100, 200), (0, 0), (-1, 2040), (20, 60)):
            got = ops.canny_classify(torch.from_numpy(img).cuda()[None], lo, hi)[0].cpu().numpy()
            assert _mismatch(got, cg.classes(img, lo, hi)) == 0, (kind, lo, hi)


def test_strided_rows():
    """a device batch whose rows are strided (a column crop of a wider buffer)"""
    from ctrlora_b200 import ops
    img = cg.image("textured", 70, 90, tag=".strided")
    wide = torch.from_numpy(img).cuda()[None]
    x = wide[:, :, 5:77]
    assert x.stride(1) == 90 * 3
    got = ops.canny_classify(x, 40, 120)[0].cpu().numpy()
    assert _mismatch(got, cg.classes(np.ascontiguousarray(img[:, 5:77]), 40, 120)) == 0


def _hyst(cls):
    from ctrlora_b200 import ops
    got = ops.canny_hysteresis(torch.from_numpy(np.ascontiguousarray(cls)).cuda()[None])[0].cpu().numpy()
    return got, cg.hysteresis(cls)


def test_spiral(det):
    s = cg.spiral()
    assert _mismatch(det(s, 100, 200), cv2.Canny(s, 100, 200)) == 0
    # the spiral's candidates with one strong pixel only, at the end of the longest chain
    cls = (cg.classes(s, 100, 200) > 0).astype(np.uint8)
    ys, xs = np.nonzero(cls)
    k = np.argmin(np.abs(ys - 256) + np.abs(xs - 256))
    cls[ys[k], xs[k]] = 2
    got, ref = _hyst(cls)
    assert (ref > 0).sum() > 80000
    assert _mismatch(got, ref) == 0


def test_serpentine_with_the_strong_pixel_at_the_far_end():
    h, w = 300, 420
    cls = np.zeros((h, w), np.uint8)
    for y in range(0, h, 4):
        cls[y, 1:w - 1] = 1
        x = w - 2 if (y // 4) % 2 == 0 else 1
        cls[y:min(y + 4, h), x] = 1
    cls[h - 1, w - 2] = 2                          # the last pixel of the chain that starts at (0, 1)
    got, ref = _hyst(cls)
    assert (ref > 0).sum() == (cls > 0).sum()
    assert _mismatch(got, ref) == 0


def test_staircase_through_tile_corners():
    """one-pixel diagonals and anti-diagonals, connected only through corners, that cross tile borders (32 x 16 and
    any other power-of-two tiling up to 64) exactly at tile corners; one strong pixel at one end of each"""
    h, w = 256, 320
    cls = np.zeros((h, w), np.uint8)
    for c in range(-192, 256, 64):                 # y = x + c
        ys = np.arange(h)
        xs = ys - c
        ok = (xs >= 0) & (xs < w)
        cls[ys[ok], xs[ok]] = 1
        cls[ys[ok][-1], xs[ok][-1]] = 2
    for c in range(63, h + w, 64):                 # y = c - x: (31, 32) -> (32, 31) and the like
        xs = np.arange(w)
        ys = c - xs
        ok = (ys >= 0) & (ys < h)
        cls[ys[ok], xs[ok]] = np.maximum(cls[ys[ok], xs[ok]], 1)
    cls[0, 63] = 2
    got, ref = _hyst(cls)
    assert _mismatch(got, ref) == 0
    assert ref.any() and not ref.all()


def test_candidates_without_a_strong_pixel_give_zeros(det):
    img = cg.image("textured", 200, 300, tag=".nostrong")
    cls = (cg.classes(img, 10, 20) > 0).astype(np.uint8)
    assert cls.sum() > 1000
    got, _ = _hyst(cls)
    assert not got.any()
    assert not det(img, 10, 5000).any()


def test_dense_binary_components():
    rs = np.random.RandomState(5)
    cls = (rs.uniform(size=(513, 771)) < 0.45).astype(np.uint8)
    cls[cls > 0] += (rs.uniform(size=int(cls.sum())) < 0.02).astype(np.uint8)
    import scipy.ndimage
    n = scipy.ndimage.label(cls > 0, structure=np.ones((3, 3)))[1]
    assert n > 2000
    got, ref = _hyst(cls)
    assert _mismatch(got, ref) == 0


def test_batch_equals_single_calls(det):
    imgs = [cg.image(k, 130, 257, tag=".batch") for k in ("smooth", "textured", "binary", "random")]
    x = torch.from_numpy(np.stack(imgs)).cuda()
    maps = det.detect(x, 100, 200).cpu().numpy()
    for img, m in zip(imgs, maps):
        assert _mismatch(m, det(img, 100, 200)) == 0
        assert _mismatch(m, cv2.Canny(img, 100, 200)) == 0


def test_repeat_calls_are_identical(det):
    img = cg.image("textured", 512, 768, tag=".repeat")
    assert _mismatch(det(img, 50, 150), det(img, 50, 150)) == 0


def test_noncontiguous_view(det):
    img = cg.image("smooth", 120, 90, tag=".view")
    view = img[:, ::-1]
    assert _mismatch(det(view, 100, 200), cv2.Canny(np.ascontiguousarray(view), 100, 200)) == 0


def test_detect_replays_from_a_cuda_graph(det):
    imgs = [cg.image("textured", 256, 384, tag=f".graph{i}") for i in range(3)] + [cg.spiral(256, 384)]
    x = torch.from_numpy(np.stack(imgs)).cuda()
    eager = det.detect(x, 100, 200)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        det.detect(x, 100, 200)                    # warm-up on the capture stream
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            out = det.detect(x, 100, 200)
        out.zero_()
        graph.replay()
    torch.cuda.current_stream().wait_stream(stream)
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_launch_count_does_not_depend_on_the_content(det):
    from ctrlora_b200 import ops
    blank = torch.zeros(1, 512, 512, 3, device="cuda", dtype=torch.uint8)
    spiral = torch.from_numpy(cg.spiral()).cuda()[None]
    n_blank = ops.count_launches(lambda: det.detect(blank, 100, 200))
    n_spiral = ops.count_launches(lambda: det.detect(spiral, 100, 200))
    assert n_blank == n_spiral == 5


def test_bad_input_raises(det):
    for bad in (np.zeros((8, 8), np.uint8), np.zeros((8, 8, 4), np.uint8), np.zeros((8, 8, 3), np.float32),
                np.zeros((0, 8, 3), np.uint8)):
        with pytest.raises(ValueError):
            det(bad, 100, 200)
    with pytest.raises(ValueError):
        det.detect(torch.zeros(1, 8, 8, 1, device="cuda", dtype=torch.uint8), 100, 200)


def test_detector_launches(det, monkeypatch):
    """every kernel launch of one CannyDetector call at 512 x 768 against its launch reference"""
    img = cg.image("textured", 512, 768, tag=".shadow")
    ref = det(img, 100, 200)
    sh = CL.shadow(monkeypatch)
    out = det(img, 100, 200)
    sh.check("CannyDetector at 512x768")
    assert np.array_equal(out, ref)
    assert sh.calls["canny_classify"] == 1 and sh.calls["canny_hysteresis"] == 1
