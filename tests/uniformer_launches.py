"""Launch references and the launch shadow for the ops wrappers of the UniFormer annotator (test infrastructure).

This module adds fp32 references for the wrappers the UniFormer path introduces (`dwconv`, `resize_bilinear`,
`adaptive_avg_pool`, `seg_output`) to those of tests/midas_launches.py (patch_gather_hw, layernorm_rows, gelu_, the
d_head-64 attention) and reuses tests/lineart_anime_launches.py's `tap_gather_act`.  They take the wrapper's
arguments and compute in fp32 with torch's own operators; tests/test_uniformer_cpu.py checks each against an
index-loop restatement.  `shadow(monkeypatch)` returns a Shadow that checks them too, registered for the duration of one
test.  tests/test_uniformer_gpu.py runs it over a detector call.
"""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import launch_refs as R  # noqa: E402
import launch_shadow as LS  # noqa: E402
import lineart_anime_launches as AL  # noqa: E402
import midas_launches as ML  # noqa: E402

# norm-relative bounds (with a max-abs guard as a fraction of max|ref|): each kernel sums fp16 inputs in fp32 and rounds
# once to fp16, so it differs from the fp32 reference by the output rounding (2^-11 relative) and the summation order
BOUNDS = {
    "dwconv": (2e-3, 1e-3),
    "resize_bilinear": (2e-3, 1e-3),
    "adaptive_avg_pool": (2e-3, 1e-3),
}
# seg_output: the labels may differ from the fp32 reference only where its top-two margin is below SEG_MARGIN; the rgb
# map is palette[label] exactly
SEG_MARGIN = 1e-4
NEW = tuple(BOUNDS) + ("seg_output",)


def _nchw(x):
    return R._f(x).permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def dwconv(x, weight, bias, k, residual=None):
    c = x.shape[-1]
    w = R._f(weight).t().reshape(c, 1, k, k)
    y = _nhwc(F.conv2d(_nchw(x), w, R._f(bias), padding=k // 2, groups=c))
    return (y if residual is None else y + R._f(residual)).half()


def resize_bilinear(x, size=None, out=None, accumulate=False):
    """the resize in fp32; with out given, the values the wrapper leaves in out (its prior contents when accumulating,
    taken from the clone the shadow passes)"""
    ho, wo = size if out is None else out.shape[1:3]
    y = _nhwc(F.interpolate(_nchw(x), size=(ho, wo), mode="bilinear", align_corners=False))
    if accumulate:
        y = y + R._f(out)
    return y.half()


def adaptive_avg_pool(x, sizes):
    return [_nhwc(F.adaptive_avg_pool2d(_nchw(x), s)).reshape(-1, x.shape[-1]).half() for s in sizes]


def seg_logits(logits, classes, net_size, out_size):
    """fp32 [B, classes, H, W]: the logits resized to net_size and then to out_size, as the reference resizes them"""
    t = R._f(logits[..., :classes]).permute(0, 3, 1, 2)
    t = F.interpolate(t, size=tuple(net_size), mode="bilinear", align_corners=False)
    return F.interpolate(t, size=tuple(out_size), mode="bilinear", align_corners=False)


def seg_output(logits, classes, net_size, out_size, palette, want_labels=False):
    """(labels int64 [B, H, W], top-two margin [B, H, W], rgb uint8 [B, H, W, 3])"""
    up = seg_logits(logits, classes, net_size, out_size)
    top2 = up.topk(2, dim=1).values
    labels = up.argmax(1)
    return labels, top2[:, 0] - top2[:, 1], palette[labels]


def tap_gather_act(x, taps, *, reflect, k_pad, stride=1, act=None, channels=None, out=None):
    """lineart_anime_launches' reference cut to H // stride x W // stride: a stride-2 gather of an odd size drops the
    last row or column, as the stride-2 Conv2d of the patch embeds does"""
    h, w = x.shape[1:3]
    return AL.tap_gather_act(x, taps, reflect=reflect, k_pad=k_pad, stride=stride, act=act,
                             channels=channels)[:, :h // stride, :w // stride].contiguous()


REFS = {name: globals()[name] for name in NEW}


class UniformerShadow(ML.MidasShadow):
    """the MiDaS shadow (which covers patch_gather_hw, layernorm_rows, gelu_ and attention) plus the wrappers of NEW
    and tap_gather_act"""

    def _compare(self, name, p, sub, got):
        if name == "tap_gather_act":
            torch.cuda.synchronize()
            return self._exact(got, tap_gather_act(**sub), "out")
        if name not in NEW:
            return super()._compare(name, p, sub, got)
        torch.cuda.synchronize()
        ref = REFS[name](**sub)
        if name == "adaptive_avg_pool":
            return max(self._close(name, g, r, f"pool {s}", BOUNDS[name]) for g, r, s in zip(got, ref, p["sizes"]))
        if name == "resize_bilinear":
            return self._close(name, got, ref, "out", BOUNDS[name])
        if name == "seg_output":
            rgb, labels = got if p["want_labels"] else (got, None)
            ref_labels, margin, ref_rgb = ref
            if labels is not None:
                bad = (labels.long() != ref_labels) & (margin > SEG_MARGIN)
                assert not bad.any(), f"labels: {int(bad.sum())} pixels differ where the margin exceeds {SEG_MARGIN}"
            bad = (rgb != ref_rgb).any(-1) & (margin > SEG_MARGIN)
            assert not bad.any(), f"rgb: {int(bad.sum())} pixels differ where the margin exceeds {SEG_MARGIN}"
            return float((rgb != ref_rgb).any(-1).float().mean().item())
        return self._close(name, got, ref, "out", BOUNDS[name])


IO = {
    "dwconv": (("x", "weight", "bias", "residual"), ()),
    "resize_bilinear": (("x", "out"), ("out",)),
    "adaptive_avg_pool": (("x",), ()),
    "seg_output": (("logits", "palette"), ()),
    "tap_gather_act": (("x",), ("out",)),
}


def shadow(monkeypatch):
    """a shadow over every covered `ops` wrapper, MiDaS's and those above, for the rest of the calling test"""
    for name, io in list(ML.IO.items()) + list(IO.items()):
        monkeypatch.setitem(LS.IO, name, io)
    monkeypatch.setattr(LS, "_describe", _describe_with(AL._describe_with(ML._describe_with(LS._describe))))
    return UniformerShadow(monkeypatch, only=LS.COVERED + ML.NEW + NEW + ("tap_gather_act",))


def _describe_with(real):
    def describe(name, p):
        if name in NEW:
            shown = [f"{k}={LS._fmt_shape(v)}" if torch.is_tensor(v) else f"{k}={v}" for k, v in p.items()
                     if v is not None and k not in ("out", "taps")]
            if name == "resize_bilinear" and p["out"] is not None:
                shown.append(f"out={LS._fmt_shape(p['out'])}/ld{p['out'].stride(-2)}")
            return " ".join(shown), ""
        return real(name, p)
    return describe
