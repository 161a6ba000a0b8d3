"""The HED-sketch annotator (annotator/hedsketch/__init__.py) over the sm_90a HED.

`from ctrlora_b200.annotator.hedsketch import HEDSketchDetector` replaces the reference's.  The edge map comes from
ctrlora_b200.annotator.hed.HEDdetector.  The sketch search stays on the host, because each attempt decides there
whether to draw again: up to six attempts, each one np.random.randint draw, a binary threshold of the current image at
that level, its inverse and a 3x3 Gaussian blur, until enough of the image is dark.  It makes the reference's np.random
calls in the reference's order with the same cv2 operations, so it returns the reference's sketch for the same HED map
and leaves numpy's global RNG in the same state.
"""
import cv2
import numpy as np

from .hed import HEDdetector

THRESHOLD_LO, THRESHOLD_HI = 110, 160  # np.random.randint's range for the binarisation level
MAX_ATTEMPTS = 6                       # the first threshold and at most five redraws
DARK_LEVEL, DARK_SHARE = 5, 0.005      # a sketch is kept once more than 0.5 % of h * w values are below 5


class HEDSketchDetector:
    """__call__(HWC uint8 RGB image, safe=False) -> HWC uint8 sketch (3 equal channels)"""

    def __init__(self, ckpt_dir=None, device="cuda"):
        self.hed = HEDdetector(ckpt_dir=ckpt_dir, device=device)

    def __call__(self, input_image, safe=False):
        hed = self.hed(input_image, safe=safe)
        sketch = np.repeat(hed[:, :, None], 3, axis=2)  # annotator.util.HWC3 of an HW uint8 map
        h, w = hed.shape
        for _ in range(MAX_ATTEMPTS):
            # one draw per attempt: pixels above the threshold become black lines on white, softened by a 3x3 blur
            level = np.random.randint(THRESHOLD_LO, THRESHOLD_HI)
            _, lines = cv2.threshold(sketch, level, 255, cv2.THRESH_BINARY)
            sketch = cv2.GaussianBlur(cv2.bitwise_not(lines), (3, 3), 0)
            # enough dark pixels (counted over all three channels, against a share of h * w) ends the search
            if np.count_nonzero(sketch < DARK_LEVEL) > DARK_SHARE * h * w:
                break
        return sketch
