"""Launch references and the launch shadow for the ops wrappers the M-LSD annotator introduces (test infrastructure).

`gemm_relu6`, `gemm_relu_residual`, `dwconv_act`, `upsample_bilinear2x_into` and `mlsd_decode` take the wrapper's
arguments and compute with torch's own operators (the GEMM modes on tests/launch_refs.py's gemm reference);
tests/test_mlsd_cpu.py checks each against an index-loop restatement and tests/test_mlsd_gpu.py checks the kernels
against them.  `shadow(monkeypatch)` returns a Shadow that checks them too, on top of tests/uniformer_launches.py's
(gemm, gemm_relu, tap_gather, the depthwise conv, ...), registered for the duration of one test; `tap_gather_act` gets a
reference that also takes the stem's fp32 NCHW source.  tests/test_mlsd_gpu.py runs it over a detector call.
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
import uniformer_launches as UL  # noqa: E402

TOPK = 200


def _nchw(x):
    return R._f(x).permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def gemm_relu6(a, w, **kwargs):
    """ops.gemm_relu6: gemm's result, then min(max(., 0), 6) after the residual"""
    return R.gemm(a, w, **kwargs).clamp(0, 6)


def gemm_relu_residual(a, w, *, residual, **kwargs):
    """ops.gemm_relu_residual: max(gemm's result without the residual, 0) + residual"""
    y = R.gemm(a, w, **kwargs).clamp_min(0)
    m, n = y.reshape(-1, y.shape[-1]).shape
    return y + R._f(R._rows(residual, m, n)).reshape(y.shape)


def dwconv_act(x, weight, bias, k, *, stride=1, act=None, residual=None):
    """the depthwise conv in fp32: stride 1 pads k // 2; stride 2 pads (0, k - 2) on the bottom and right (TFLite),
    cut to H // 2 x W // 2; then residual and act"""
    c = x.shape[-1]
    wt = R._f(weight).t().reshape(c, 1, k, k)
    with R.exact_fp32():
        if stride == 1:
            y = F.conv2d(_nchw(x), wt, R._f(bias), padding=k // 2, groups=c)
        else:
            y = F.conv2d(F.pad(_nchw(x), (0, k - 2, 0, k - 2)), wt, R._f(bias), stride=2, groups=c)
            y = y[:, :, :x.shape[1] // 2, :x.shape[2] // 2]
    y = _nhwc(y)
    if residual is not None:
        y = y + R._f(residual)
    if act == "relu":
        y = y.clamp_min(0)
    elif act == "relu6":
        y = y.clamp(0, 6)
    return y


def upsample_bilinear2x_into(x, out):
    """the values the wrapper writes into `out` (an [B, 2h, 2w, C] view, checked): torch's F.interpolate on the fp16
    tensor itself, as tests/midas_launches.py's upsample_bilinear2x forms it (one fp16 unit apart at most)"""
    y = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    assert out is None or tuple(out.shape) == tuple(y.shape), (tuple(out.shape), tuple(y.shape))
    return y


def decode_scores(tp, c_center):
    """fp32 [B, h * w]: sigmoid(centre) where it equals its 3 x 3 window's maximum, else 0.  The sigmoid is formed as
    the kernel forms it, 1 / (1 + exp(-x)), so that equal inputs give equal scores on the device (torch.sigmoid may
    differ by an ulp, which would reorder near-ties)"""
    heat = 1.0 / (1.0 + torch.exp(-R._f(tp[..., c_center])))
    keep = F.max_pool2d(heat[:, None], 3, stride=1, padding=1)[:, 0] == heat
    return (heat * keep).reshape(tp.shape[0], -1)


def mlsd_decode(tp, c_center, c_disp):
    """(int64 [B, TOPK] indices, fp32 [B, TOPK, 6]) with the kernel's order: score descending, then index ascending
    (a stable sort of the negated scores)"""
    s = decode_scores(tp, c_center)
    order = torch.sort(-s, dim=1, stable=True).indices[:, :TOPK]
    b = tp.shape[0]
    d = R._f(tp[..., c_disp:c_disp + 4]).reshape(b, -1, 4).gather(1, order[..., None].expand(-1, -1, 4))
    ex, ey = d[..., 0] - d[..., 2], d[..., 1] - d[..., 3]
    dist = torch.sqrt(ex * ex + ey * ey)
    return order, torch.cat([s.gather(1, order)[..., None], dist[..., None], d], -1)


def tap_gather_act(x, taps, *, reflect, k_pad, stride=1, act=None, channels=None, out=None):
    """lineart_anime_launches' reference cut to H // stride x W // stride, with H, W read from an fp32 NCHW source
    ([B, C, H, W], the stem's) as well as from an fp16 pixel-major one"""
    h, w = x.shape[2:4] if x.dtype == torch.float32 else x.shape[1:3]
    return AL.tap_gather_act(x, taps, reflect=reflect, k_pad=k_pad, stride=stride, act=act,
                             channels=channels)[:, :h // stride, :w // stride].contiguous()


GEMMS = ("gemm_relu6", "gemm_relu_residual")
NEW = GEMMS + ("dwconv_act", "upsample_bilinear2x_into", "mlsd_decode")
REFS = {name: globals()[name] for name in NEW}
DWCONV_BOUND = UL.BOUNDS["dwconv"]
# mlsd_decode: indices and displacements exact; score and length within this relative error (fp32 sigmoid and sqrt
# of two libraries, an ulp or two)
DECODE_RTOL = 1e-6


class MLSDShadow(UL.UniformerShadow):
    """the UniFormer shadow (gemm, gemm_relu, tap_gather, tap_gather_act, ...) plus the wrappers of NEW, and
    tap_gather_act with an fp32 NCHW source"""

    def _compare(self, name, p, sub, got):
        if name == "tap_gather_act":
            torch.cuda.synchronize()
            return self._exact(got, tap_gather_act(**sub), "out")
        if name not in NEW:
            return super()._compare(name, p, sub, got)
        torch.cuda.synchronize()
        ref = REFS[name](**sub)
        if name in GEMMS:
            return self._compare_gemm(p, got, ref, name)
        if name == "dwconv_act":
            return self._close(name, got, ref, "out", DWCONV_BOUND)
        if name == "upsample_bilinear2x_into":
            ulps = ML.one_ulp_f16(got, ref)
            assert ulps <= 1.0, f"out: {ulps:.2f} fp16 units from torch's fp16 interpolation"
            return ulps
        idx, val = got
        ref_idx, ref_val = ref
        self._exact(idx.long(), ref_idx, "indices")
        self._exact(val[..., 2:], ref_val[..., 2:], "displacements")
        rel = ((val[..., :2] - ref_val[..., :2]).abs() / ref_val[..., :2].abs().clamp_min(1e-30)).max().item()
        assert rel <= DECODE_RTOL, f"score / length: relative error {rel:.2e}"
        return rel


IO = {
    "gemm_relu6": LS.IO["gemm"],
    "gemm_relu_residual": LS.IO["gemm"],
    "dwconv_act": (("x", "weight", "bias", "residual"), ()),
    "upsample_bilinear2x_into": (("x",), ("out",)),
    "mlsd_decode": (("tp",), ()),
}


def shadow(monkeypatch):
    """a shadow over every covered `ops` wrapper, UniFormer's and those above, for the rest of the calling test"""
    for name, io in list(ML.IO.items()) + list(UL.IO.items()) + list(IO.items()):
        monkeypatch.setitem(LS.IO, name, io)
    for name in GEMMS:
        monkeypatch.setitem(LS.BOUNDS, name, LS.BOUNDS["gemm"])
    real_sig = LS._signature
    # the two GEMM modes take gemm's arguments (gemm_relu_residual's residual among them): bind them by gemm's signature
    monkeypatch.setattr(LS, "_signature", lambda members, name: real_sig(members, "gemm" if name in GEMMS else name))
    monkeypatch.setattr(LS, "_describe", _describe_with(UL._describe_with(AL._describe_with(ML._describe_with(
        LS._describe)))))
    return MLSDShadow(monkeypatch, only=LS.COVERED + ML.NEW + UL.NEW + ("tap_gather_act",) + NEW)


def _describe_with(real):
    def describe(name, p):
        if name in GEMMS:
            return real("gemm", p)
        if name == "dwconv_act":
            return (f"{LS._fmt_shape(p['x'])} k={p['k']} stride={p['stride']} act={p['act']}" +
                    (",res" if p["residual"] is not None else "")), ""
        if name == "upsample_bilinear2x_into":
            x, out = p["x"], p["out"]
            return f"{LS._fmt_shape(x)}/ld{x.stride(-2)} -> {LS._fmt_shape(out)}/ld{out.stride(-2)}", ""
        if name == "mlsd_decode":
            return f"{LS._fmt_shape(p['tp'])} centre={p['c_center']} disp={p['c_disp']}", ""
        return real(name, p)
    return describe
