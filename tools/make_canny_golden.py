"""Generate tests/golden/canny_golden.pt: what the reference's Canny annotator computes, on the CPU.

    python tools/make_canny_golden.py

The unmodified reference `annotator.canny.CannyDetector` is imported from the reference tree and called as the apps
call it, `CannyDetector()(img, low_threshold=..., high_threshold=...)`.  The inputs are tests/canny_golden.py's seeded
images: smooth, textured and binary content at 512^2, 512 x 768, 768 x 512 and 497 x 513, and the spiral.  Each is
stored in the fixture as PNG bytes (lossless), and under every threshold pair of THRESHOLDS its map is stored
bit-packed (np.packbits of map > 0, row-major).  Running it twice writes identical bytes.
"""
import os
import sys

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from tools import ref_shims  # noqa: E402
from golden_io import save_golden  # noqa: E402
import canny_golden as cg  # noqa: E402


def main():
    if ref_shims.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shims.REFERENCE_ROOT)
    from annotator.canny import CannyDetector
    det = CannyDetector()
    g = {"seed": cg.SEED, "thresholds": [tuple(t) for t in cg.THRESHOLDS], "cv2": cv2.__version__, "cases": []}
    for name, img in cg.cases():
        ok, png = cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, 9])
        assert ok and np.array_equal(cv2.imdecode(png, cv2.IMREAD_UNCHANGED), img)
        g["cases"].append(name)
        g[f"{name}.png"] = torch.from_numpy(png.reshape(-1).copy())
        g[f"{name}.shape"] = tuple(img.shape[:2])
        counts = []
        for i, (lo, hi) in enumerate(cg.THRESHOLDS):
            m = det(img, low_threshold=lo, high_threshold=hi)
            assert m.shape == img.shape[:2] and m.dtype == np.uint8 and set(np.unique(m).tolist()) <= {0, 255}
            g[f"{name}.map{i}"] = torch.from_numpy(cg.pack(m))
            counts.append(int((m > 0).sum()))
        print(f"{name}: {img.shape[0]} x {img.shape[1]}, PNG {png.size} bytes, edge pixels per pair {counts}")
    path = os.path.join(ROOT, "tests", "golden", "canny_golden.pt")
    save_golden(g, path)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
