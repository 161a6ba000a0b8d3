"""Launch references and the launch shadow for the ops wrappers of the MiDaS annotator (test infrastructure).

tests/launch_refs.py holds a plain torch reference per `ops` wrapper, and tests/launch_shadow.py checks every covered
call of a scenario against it.  This module adds references for the wrappers the MiDaS path introduces
(`patch_gather_hw`, `depth_to_space_bias`, `add_relu`, `upsample_bilinear2x`, `midas_head_out`, `midas_maps`) and for the
existing wrappers the shared shadow leaves unchecked but this path calls with forms of its own (`small_linear` reading
the cls rows with row stride (P + 1) C, `cast_rows` with the same stride, `clip_vision_embed`, `layernorm_rows` at
eps 1e-6, `gelu_`).  They take the wrapper's arguments and compute in fp32.  `shadow(monkeypatch)` returns a Shadow that
checks them too, registered for the duration of one test.  tests/test_midas_gpu.py runs it over a detector call.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import launch_refs as R  # noqa: E402
import launch_shadow as LS  # noqa: E402

# (max-abs guard as a fraction of max|ref|, norm-relative bound) of the compared-with-tolerance wrappers.
# small_linear: the reference uses the same fp16 weights, so only the fp32 summation order differs; layernorm_rows
# and gelu_: the bounds of the shared shadow's layernorm and of test_conditioning_kernels_gpu.py's GELU; midas_head_out:
# 32 fp16 x fp32 products summed in fp32 in another order
BOUNDS = {
    "small_linear": (1e-5, 1e-5),
    "layernorm_rows": (3e-3, 1e-3),
    "gelu_": (2e-3, 1e-3),
    "midas_head_out": (1e-5, 1e-6),
}
# bit for bit: gathers, casts, fp32 adds, and an fp32 sum rounded once to fp16
EXACT = ("patch_gather_hw", "cast_rows", "clip_vision_embed", "depth_to_space_bias", "add_relu")
NEW = tuple(BOUNDS) + EXACT + ("upsample_bilinear2x", "midas_maps")


def patch_gather_hw(pixels, patch, k_pad, out=None):
    """F.unfold of the image cropped to whole patches, columns (c, kh, kw), zero beyond C * patch^2"""
    b, c, h, w = pixels.shape
    gh, gw = h // patch, w // patch
    cols = F.unfold(R._f(pixels[:, :, :gh * patch, :gw * patch]), patch, stride=patch)   # [B, C p p, gh gw]
    y = torch.zeros(b * gh * gw, k_pad, device=pixels.device, dtype=torch.float16)
    y[:, :c * patch * patch] = cols.transpose(1, 2).reshape(b * gh * gw, -1).half()
    return y


def cast_rows(src, rows, cols, lds):
    return torch.as_strided(src, (rows, cols), (lds, 1)).half()


def clip_vision_embed(patch_out, class_embedding, position_embedding, batch, out=None):
    cols = patch_out.shape[1]
    patches = patch_out.shape[0] // batch
    x = torch.cat([class_embedding.view(1, 1, cols).expand(batch, 1, cols), patch_out.view(batch, patches, cols)], 1)
    return (x + position_embedding).reshape(batch * (patches + 1), cols)


def small_linear(x, w, bias, silu_in=False, silu_out=False, out=None):
    assert not silu_in and not silu_out
    with R.exact_fp32():
        y = R._f(x) @ R._f(w).t()
    return y if bias is None else y + bias


def layernorm_rows(x, gamma, beta, eps=1e-5, out_f32=False, out=None):
    y = F.layer_norm(R._f(x), (x.shape[-1],), R._f(gamma), R._f(beta), eps)
    return y if (out_f32 or (out is not None and out.dtype == torch.float32)) else y.half()


def gelu_(x):
    return F.gelu(R._f(x)).half()


def depth_to_space_bias(src, bias, s):
    b, h, w, n = src.shape
    c = n // (s * s)
    return (src.view(b, h, w, s, s, c).permute(0, 1, 3, 2, 4, 5).reshape(b, h * s, w * s, c) + bias).half()


def add_relu(a, b=None):
    s = a if b is None else (a.float() + b.float()).half()
    return s.clamp_min(0) if b is None else (s, s.clamp_min(0))


def upsample_bilinear2x(x):
    """torch's F.interpolate on the fp16 CUDA tensor itself: its kernel forms the weights and the sums in fp32, as the
    restatement does, so the two may differ by one fp16 unit (FMA contraction).  An fp32 interpolation is not used:
    where neighbours cancel, its own weight rounding moves a small result by more than one unit of it."""
    return F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)


def midas_head_out(x, weight, bias):
    return F.relu(R._f(x) @ R._f(weight) + R._f(bias))


def midas_maps(depth, a, bg_th):
    """MidasDetector.__call__'s numpy / cv2 post-process, per image, on the depth the kernel received"""
    import cv2
    d8, n8 = [], []
    for dep in depth.cpu().numpy():
        depth_pt = dep.copy()
        depth_pt -= np.min(depth_pt)
        depth_pt /= np.max(depth_pt)
        d8.append((depth_pt * 255.0).clip(0, 255).astype(np.uint8))
        x = cv2.Sobel(dep, cv2.CV_32F, 1, 0, ksize=3)
        y = cv2.Sobel(dep, cv2.CV_32F, 0, 1, ksize=3)
        z = np.ones_like(x) * a
        x[depth_pt < bg_th] = 0
        y[depth_pt < bg_th] = 0
        normal = np.stack([x, y, z], axis=2)
        normal /= np.sum(normal ** 2.0, axis=2, keepdims=True) ** 0.5
        n8.append((normal * 127.5 + 127.5).clip(0, 255).astype(np.uint8))
    return torch.from_numpy(np.stack(d8)), torch.from_numpy(np.stack(n8))


REFS = {name: globals()[name] for name in NEW}


def one_ulp_f16(got, ref):
    """max over elements of |got - ref| in units of the fp16 spacing at ref (a correctly rounded result is <= 0.5)"""
    r = ref.float()
    _, e = torch.frexp(r)
    spacing = torch.where(r.abs() >= 2.0 ** -14, torch.ldexp(torch.ones_like(r), e - 11), torch.full_like(r, 2.0 ** -24))
    return ((got.float() - r).abs() / spacing).max().item()


class MidasShadow(LS.Shadow):
    """launch_shadow.Shadow that also compares the wrappers of NEW"""

    def _compare(self, name, p, sub, got):
        if name == "attention":
            return self._compare_attention(p, sub, got)
        if name not in NEW:
            return super()._compare(name, p, sub, got)
        torch.cuda.synchronize()
        ref = REFS[name](**sub)
        if name in EXACT:
            if name == "add_relu" and sub.get("b") is not None:
                return max(self._exact(g, r, w) for g, r, w in zip(got, ref, ("sum", "relu")))
            return self._exact(got, ref, "out")
        if name == "upsample_bilinear2x":
            ulps = one_ulp_f16(got, ref)
            assert ulps <= 1.0, f"out: {ulps:.2f} fp16 units from torch's fp16 interpolation"
            return ulps
        if name == "midas_maps":
            self._exact(got[0].cpu(), ref[0], "depth_u8")
            d = (got[1].cpu().int() - ref[1].int()).abs()
            assert d.max().item() <= 1, f"normal_u8: {d.max().item()} levels from the reference post-process"
            assert (d > 0).float().mean().item() < 1e-3, f"normal_u8: {(d > 0).float().mean().item():.2e} of it differs"
            return float((d > 0).float().mean().item())
        return self._close(name, got, ref, "out", BOUNDS[name])

    def _compare_attention(self, p, sub, got):
        """the shared comparison without its zero-padding assertion on V^T: the kernel's V^T tensor map ends at nk
        (attention_sm90.cu), so keys in [nk, nk_pad) are TMA zero fill and never read; run_layers leaves them unset"""
        torch.cuda.synchronize()
        ref = R.attention(**sub)
        ref_o = ref if p["lse"] is None else ref[0]
        return self._close_per_image("attention", got, ref_o, p["batch"], "out")


def _describe_with(real):
    def describe(name, p):
        if name in NEW:
            shown = [f"{k}={LS._fmt_shape(v)}" if torch.is_tensor(v) else f"{k}={v}" for k, v in p.items()
                     if v is not None and k != "out"]
            if name in ("small_linear", "cast_rows"):
                src = p["x" if name == "small_linear" else "src"]
                shown.append(f"ld={src.stride(0) if name == 'small_linear' else p['lds']}")
            return " ".join(shown), ""
        return real(name, p)
    return describe


IO = {
    "patch_gather_hw": (("pixels",), ("out",)),
    "cast_rows": (("src",), ()),
    "clip_vision_embed": (("patch_out", "class_embedding", "position_embedding"), ("out",)),
    "small_linear": (("x", "w", "bias"), ("out",)),
    "layernorm_rows": (("x", "gamma", "beta"), ("out",)),
    "gelu_": (("x",), ("x",)),
    "depth_to_space_bias": (("src", "bias"), ()),
    "add_relu": (("a", "b"), ()),
    "upsample_bilinear2x": (("x",), ()),
    "midas_head_out": (("x", "weight", "bias"), ()),
    "midas_maps": (("depth",), ()),
}


def shadow(monkeypatch):
    """a shadow over every covered `ops` wrapper and those above, for the rest of the calling test"""
    for name, io in IO.items():
        monkeypatch.setitem(LS.IO, name, io)
    monkeypatch.setattr(LS, "_describe", _describe_with(LS._describe))
    return MidasShadow(monkeypatch, only=LS.COVERED + NEW)
