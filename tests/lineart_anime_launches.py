"""Launch references and the launch shadow for the two ops wrappers of the anime line-art annotator (test
infrastructure): `ops.tap_gather_act` and `ops.lineart_anime_out`.

tests/launch_refs.py holds a plain torch reference per `ops` wrapper and tests/launch_shadow.py checks every covered
call of a scenario against it.  This module adds references for the two wrappers the anime line-art path introduces,
in the same form (the wrapper's arguments, fp32 math, fp64 for fp64 operands), and `shadow(monkeypatch)`: a Shadow that
checks them too, registered for the duration of one test.  tests/test_lineart_anime_cpu.py pins the references at tiny
shapes on the host; tests/test_lineart_anime_gpu.py runs the shadow over a detector call.
"""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import launch_refs as R  # noqa: E402
import launch_shadow as LS  # noqa: E402

# lineart_anime_out: (max-abs guard as a fraction of max|ref|, norm-relative bound).  The norm-relative bound is
# test_lineart_anime_gpu.py's OUT_BOUND; the guard was measured on an H100 80GB HBM3 at 700 W over a detector call at
# 512 x 768: up to 3.97e-7 (fp32 sums of 512 products in another order than cuDNN's, then tanh and the scaling)
OUT_GUARD = (8e-7, 1e-6)


def _act(t, act):
    """the gather's activation on load, in fp32 (fp64 in fp64 mode), returned in t's dtype: an fp16 source is rounded
    once, as the kernel rounds act(value)"""
    if act is None:
        return t
    f = R._f(t)
    return (f.clamp_min(0) if act == "relu" else F.leaky_relu(f, 0.2)).to(t.dtype)


def tap_gather_act(x, taps, *, reflect, k_pad, stride=1, act=None, channels=None, out=None):
    """ops.tap_gather_act: launch_refs.tap_gather of act(x), at every stride-th output pixel in each direction ->
    fp16 [B, H / stride, W / stride, k_pad] (fp64 for an fp64 source)"""
    y = R.tap_gather(_act(x, act), taps, reflect=reflect, k_pad=k_pad, channels=channels)
    return y[:, ::stride, ::stride].contiguous()


def lineart_anime_out(skip, up, weight, bias, scale=1.0, shift=0.0):
    """ops.lineart_anime_out: tanh(bias + conv_transpose2d(relu([skip | up]), weight as [C, 1, 4, 4], stride 2,
    padding 1)) * scale + shift -> [B, 1, 2h, 2w]"""
    x = torch.cat([R._f(skip), R._f(up)], -1).clamp_min(0).permute(0, 3, 1, 2)
    wf = R._f(weight).to(x.dtype).view(-1, 1, 4, 4)
    with R.exact_fp32():
        y = F.conv_transpose2d(x, wf, R._f(bias).to(x.dtype).view(1), stride=2, padding=1)
    return torch.tanh(y) * scale + shift


class AnimeShadow(LS.Shadow):
    """launch_shadow.Shadow that also compares ops.tap_gather_act (bit for bit) and ops.lineart_anime_out"""

    def _compare(self, name, p, sub, got):
        if name == "tap_gather_act":
            torch.cuda.synchronize()
            return self._exact(got, tap_gather_act(**sub), "out")
        if name == "lineart_anime_out":
            torch.cuda.synchronize()
            ref = lineart_anime_out(**sub)
            return max(self._close(name, got[i], ref[i], f"y image {i}", OUT_GUARD) for i in range(got.shape[0]))
        return super()._compare(name, p, sub, got)


def _describe_with(real):
    def describe(name, p):
        if name == "tap_gather_act":
            x = p["x"]
            return (f"{LS._fmt_shape(x)} {'f32nchw' if x.dtype == torch.float32 else 'f16'} taps={len(p['taps'])} "
                    f"{'reflect' if p['reflect'] else 'zero'} k_pad={p['k_pad']} stride={p['stride']} act={p['act']}"), ""
        if name == "lineart_anime_out":
            return f"{LS._fmt_shape(p['skip'])}+{p['up'].shape[-1]} scale={p['scale']:g} shift={p['shift']:g}", ""
        return real(name, p)
    return describe


def shadow(monkeypatch):
    """a shadow over every covered `ops` wrapper and the two above, for the rest of the calling test"""
    monkeypatch.setitem(LS.IO, "tap_gather_act", (("x",), ("out",)))
    monkeypatch.setitem(LS.IO, "lineart_anime_out", (("skip", "up", "weight", "bias"), ()))
    monkeypatch.setattr(LS, "_describe", _describe_with(LS._describe))
    return AnimeShadow(monkeypatch, only=LS.COVERED + ("tap_gather_act", "lineart_anime_out"))
