"""The Canny edge annotator (annotator/canny/__init__.py CannyDetector: one call of cv2.Canny(img, low, high)) on the
sm_90a kernels, bit for bit.

Switching a caller over is an import swap: `from ctrlora_b200.annotator.canny import CannyDetector`.  Two ops do the
work on the device:

- ops.canny_classify: per pixel the 3 x 3 Sobel of each channel (border replicated), the channel with the largest L1
  magnitude, cv2's fixed-point direction and asymmetric non-maximum suppression, and the two thresholds -> classes
  none / candidate / strong;
- ops.canny_hysteresis: the candidates 8-connected to a strong pixel, by union-find labelling in a fixed number of
  launches, so `detect` can be captured in a CUDA graph.

The thresholds are floored and swapped on the host as cv2 does (`thresholds`).  Inference only, on the current stream.
"""
import math

import numpy as np
import torch

from .. import ops


def thresholds(low_threshold, high_threshold):
    """cv2.Canny's integer thresholds: (floor(low), floor(high)), swapped when the first is the larger"""
    lo, hi = math.floor(low_threshold), math.floor(high_threshold)
    return (hi, lo) if lo > hi else (lo, hi)


def _check_image(img, what):
    if img.dim() != 4 or img.shape[3] != 3 or img.dtype != torch.uint8 or img.shape[1] < 1 or img.shape[2] < 1:
        raise ValueError(f"{what} takes uint8 [B, H, W, 3] images with H, W >= 1, got {img.dtype} {tuple(img.shape)}")


class CannyDetector:
    """The reference's CannyDetector: __call__(HWC uint8 RGB image, low_threshold, high_threshold) -> uint8 [H, W] edge
    map, 0 / 255, equal to cv2.Canny(img, low_threshold, high_threshold) bit for bit.  The one deliberate difference:
    an image that is not a uint8 H x W x 3 array raises ValueError (cv2 also takes 1- and 4-channel images; every
    caller converts with HWC3 first).  `detect` runs a device batch."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("CannyDetector runs on the sm_90a kernels only: pass a CUDA device")

    def __call__(self, img, low_threshold, high_threshold):
        if not isinstance(img, np.ndarray) or img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.uint8 or \
                img.shape[0] < 1 or img.shape[1] < 1:
            raise ValueError("CannyDetector takes an HWC uint8 RGB image, got "
                             f"{getattr(img, 'dtype', type(img))} {getattr(img, 'shape', '')}")
        x = torch.from_numpy(np.ascontiguousarray(img)).to(self.device)
        return self.detect(x[None], low_threshold, high_threshold)[0].cpu().numpy()

    def detect(self, x, low_threshold, high_threshold):
        """device uint8 [B, H, W, 3] -> device uint8 [B, H, W], each image's cv2.Canny map.  Five kernel launches
        whatever the images hold, no host synchronisation."""
        _check_image(x, "CannyDetector.detect")
        if x.stride(3) != 1 or x.stride(2) != 3 or x.stride(0) != x.shape[1] * x.stride(1):
            x = x.contiguous()
        lo, hi = thresholds(low_threshold, high_threshold)
        return ops.canny_hysteresis(ops.canny_classify(x, lo, hi))
