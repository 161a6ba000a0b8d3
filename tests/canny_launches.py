"""Launch references and the launch shadow for the ops wrappers of the Canny annotator (test infrastructure).

`canny_classify` and `canny_hysteresis` take the wrapper's arguments and compute with tests/canny_golden.py's
restatement: the classes per image, and the hysteresis as the closure of the 8-connected candidate components over
their strong pixels.  Both bounds are exact: the kernels must match bit for bit.  tests/test_canny_cpu.py checks each
reference against an index loop and tests/test_canny_gpu.py checks the kernels against them; `shadow(monkeypatch)`
returns a Shadow that checks every call of the two wrappers, registered for the duration of one test.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import canny_golden as cg  # noqa: E402
import launch_shadow as LS  # noqa: E402


def canny_classify(x, lo, hi):
    """uint8 [B, H, W, 3] (any device), integer lo <= hi -> uint8 [B, H, W] classes on x's device"""
    imgs = x.cpu().numpy()
    cls = np.stack([cg.classes(img, int(lo), int(hi)) for img in imgs])
    return torch.from_numpy(cls).to(x.device)


def canny_hysteresis(cls):
    """uint8 [B, H, W] classes -> uint8 [B, H, W] 0 / 255 maps on cls's device"""
    out = np.stack([cg.hysteresis(c) for c in cls.cpu().numpy()])
    return torch.from_numpy(out).to(cls.device)


NEW = ("canny_classify", "canny_hysteresis")
REFS = {name: globals()[name] for name in NEW}
IO = {"canny_classify": (("x",), ()), "canny_hysteresis": (("cls",), ())}


class CannyShadow(LS.Shadow):
    """checks the two Canny wrappers bit for bit against the references above"""

    def _compare(self, name, p, sub, got):
        if name not in NEW:
            return super()._compare(name, p, sub, got)
        torch.cuda.synchronize()
        return self._exact(got, REFS[name](**sub), "classes" if name == "canny_classify" else "map")


def shadow(monkeypatch):
    """a shadow over the Canny wrappers for the rest of the calling test"""
    for name, io in IO.items():
        monkeypatch.setitem(LS.IO, name, io)
    monkeypatch.setattr(LS, "_describe", _describe_with(LS._describe))
    return CannyShadow(monkeypatch, only=NEW)


def _describe_with(real):
    def describe(name, p):
        if name == "canny_classify":
            x = p["x"]
            return f"{LS._fmt_shape(x)}/ld{x.stride(1)} lo={p['lo']} hi={p['hi']}", ""
        if name == "canny_hysteresis":
            return LS._fmt_shape(p["cls"]), ""
        return real(name, p)
    return describe
