"""GPU parity of the non-GEMM kernels against torch fp32 references computed on the same fp16-rounded inputs.

Tolerances: outputs are fp16 (2^-11 relative rounding) -> 2e-3 of the reference's max magnitude unless stated; the
DDIM update and the integer/index-driven kernels (layout conversion, upsample, stride-2 gather) are bit-exact.
"""
import math

import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


from tolerances import close as _close  # noqa: E402  (max-abs guard AND norm-relative <= 1e-3)


def _rand(*shape, s=1.0, dtype=torch.float16):
    return (torch.randn(*shape, device="cuda") * s).to(dtype)


@pytest.mark.parametrize("B,H,W,C,silu,eps", [(2, 16, 16, 320, True, 1e-5), (3, 8, 8, 32, False, 1e-6),
                                               (2, 32, 32, 640, True, 1e-5), (1, 64, 64, 320, True, 1e-5),
                                               (2, 8, 8, 1280, True, 1e-5)])
def test_groupnorm(B, H, W, C, silu, eps):
    from ctrlora_b200 import ops
    torch.manual_seed(0)
    x = _rand(B, H, W, C) + 0.5
    g, b = torch.randn(C, device="cuda"), torch.randn(C, device="cuda")
    y = ops.groupnorm(x, g, b, eps, silu)
    ref = F.group_norm(x.float().permute(0, 3, 1, 2), 32, g, b, eps)
    ref = (F.silu(ref) if silu else ref).permute(0, 2, 3, 1)
    _close(y, ref, 3e-3)


@pytest.mark.parametrize("C1,C2", [(1280, 1280), (1280, 640), (640, 320), (320, 320), (64, 32)])
def test_groupnorm_concat_with_control(C1, C2):
    """cat([h + s1*c_mid, hs + s2*ctrl], 1) -> GN -> SiLU, plus the raw concat for the skip conv (cldm/cldm.py:34-42)."""
    from ctrlora_b200 import ops
    torch.manual_seed(1)
    B, H, W = 2, 16, 16
    x1, a1, x2, a2 = _rand(B, H, W, C1), _rand(B, H, W, C1), _rand(B, H, W, C2), _rand(B, H, W, C2)
    C = C1 + C2
    g, b = torch.randn(C, device="cuda"), torch.randn(C, device="cuda")
    y, raw = ops.groupnorm(x1, g, b, 1e-5, True, add1=a1, add1_scale=0.7, x2=x2, add2=a2, add2_scale=1.3, want_raw=True)
    cat = torch.cat([x1.float() + 0.7 * a1.float(), x2.float() + 1.3 * a2.float()], dim=-1)
    _close(raw, cat, 1e-3)
    ref = F.silu(F.group_norm(cat.permute(0, 3, 1, 2), 32, g, b, 1e-5)).permute(0, 2, 3, 1)
    _close(y, ref, 3e-3)
    y2 = ops.groupnorm(x1, g, b, 1e-5, True, x2=x2)
    ref2 = F.silu(F.group_norm(torch.cat([x1, x2], -1).float().permute(0, 3, 1, 2), 32, g, b, 1e-5)).permute(0, 2, 3, 1)
    _close(y2, ref2, 3e-3)


@pytest.mark.parametrize("M,C", [(300, 320), (4096, 640), (77, 1280), (64, 32), (10, 2048)])
def test_layernorm(M, C):
    from ctrlora_b200 import ops
    torch.manual_seed(2)
    x = _rand(M, C) * 2 + 0.3
    g, b = torch.randn(C, device="cuda"), torch.randn(C, device="cuda")
    _close(ops.layernorm(x, g, b), F.layer_norm(x.float(), (C,), g, b, 1e-5), 3e-3)


def _attn_ref(q, k, v, B, H, Nq, Nk, d):
    qf = q.float().view(B, Nq, H, d).permute(0, 2, 1, 3)
    kf = k.float().view(B, Nk, H, d).permute(0, 2, 1, 3)
    vf = v.float().view(B, Nk, H, d).permute(0, 2, 1, 3)
    sim = (qf @ kf.transpose(-1, -2)) * d ** -0.5
    return (sim.softmax(-1) @ vf).permute(0, 2, 1, 3).reshape(B * Nq, H * d)


@pytest.mark.parametrize("B,H,Nq,Nk,d", [
    (2, 8, 4096, 4096, 40),   # 64x64 self-attention (online softmax, 32 KV tiles)
    (2, 8, 1024, 1024, 80),   # 32x32 self
    (2, 8, 256, 256, 160),    # 16x16 self (single 256-key tile)
    (2, 8, 64, 64, 160),      # 8x8 self
    (2, 8, 4096, 77, 40),     # cross-attention to 77 context tokens
    (2, 8, 1024, 77, 80),
    (2, 8, 256, 77, 160),
    (3, 4, 200, 300, 16),     # ragged sizes, tiny-config head dims
    (1, 4, 64, 520, 8),
    (2, 4, 256, 256, 32),
    (1, 2, 130, 129, 64),
    (1, 8, 600, 700, 40),     # ragged multi-tile: masked last key tile (keys beyond Nk masked)
    (1, 2, 300, 1000, 24),    # d16 = 32 < DPAD = 48
    (1, 2, 384, 640, 48),     # d a multiple of 16: row sums through the P x ones product
])
def test_attention(B, H, Nq, Nk, d):
    from ctrlora_b200 import ops
    torch.manual_seed(3)
    q, k, v = _rand(B * Nq, H * d), _rand(B * Nk, H * d), _rand(B * Nk, H * d)
    nk_pad = (Nk + 7) // 8 * 8
    vt = torch.zeros(B, H, d, nk_pad, device="cuda", dtype=torch.float16)
    vt[..., :Nk] = v.view(B, Nk, H, d).permute(0, 2, 3, 1)
    out = ops.attention(q, k, vt, B, H, Nq, Nk, d)
    _close(out, _attn_ref(q, k, v, B, H, Nq, Nk, d), 3e-3)


@pytest.mark.parametrize("Nq,Nk,d,hot", [(256, 1000, 40, "upper"), (256, 1000, 40, "lower"), (130, 290, 24, "upper"),
                                          (128, 4096, 40, "drift"), (64, 520, 8, "lower")])
def test_attention_split_key_streams_and_lse(Nq, Nk, d, hot):
    """The d < 48 streaming kernel runs two independent online-softmax streams per row (lower / upper 32 keys of every
    64-key tile) and merges them at the end: put the dominant logits into one half only / let the maximum drift upwards
    tile after tile, and check O and the saved log-sum-exp (base 2, scaled logits) against fp32 torch."""
    from ctrlora_b200 import ops
    torch.manual_seed(11)
    B, H = 1, 4
    q, k, v = _rand(B * Nq, H * d), _rand(B * Nk, H * d), _rand(B * Nk, H * d)
    kk = k.view(B, Nk, H, d)
    qq = q.view(B, Nq, H, d)
    idx = torch.arange(Nk, device="cuda")
    if hot in ("upper", "lower"):
        sel = ((idx % 64) >= 32) if hot == "upper" else ((idx % 64) < 32)
        kk[:, sel] += 1.5 * qq[:, :1].mean(1, keepdim=True).sign()  # logits of one key half stand well above the other
        kk[:, sel] *= 2.0
    else:
        kk *= (1.0 + 3.0 * idx.float() / Nk).view(1, Nk, 1, 1).half()  # keys grow: the row maximum keeps moving
    nk_pad = (Nk + 7) // 8 * 8
    vt = torch.zeros(B, H, d, nk_pad, device="cuda", dtype=torch.float16)
    vt[..., :Nk] = v.view(B, Nk, H, d).permute(0, 2, 3, 1)
    lse = torch.empty(B, H, Nq, device="cuda", dtype=torch.float32)
    out = ops.attention(q, k, vt, B, H, Nq, Nk, d, lse=lse)
    _close(out, _attn_ref(q, k, v, B, H, Nq, Nk, d), 3e-3)
    qf = q.float().view(B, Nq, H, d).permute(0, 2, 1, 3)
    kf = k.float().view(B, Nk, H, d).permute(0, 2, 1, 3)
    ref_lse = torch.logsumexp((qf @ kf.transpose(-1, -2)) * d ** -0.5, -1) * 1.4426950408889634
    assert (lse - ref_lse).abs().max().item() < 2e-3 * max(1.0, ref_lse.abs().max().item())


@pytest.mark.parametrize("B,H,Nq,Nk,d", [(1, 2, 130, 128, 64), (2, 3, 900, 100, 40), (1, 1, 128, 33, 8), (5, 8, 256, 77, 40),
                                         (1, 8, 4096, 77, 40), (3, 8, 1000, 77, 80), (20, 8, 64, 77, 80)])
def test_attention_short_context_persistent_kernel_and_lse(B, H, Nq, Nk, d):
    """Nk <= 128, d <= 80 runs the persistent cross-attention kernel (K / V^T resident, query tiles streamed, S and O
    double-buffered): ragged last query tile, 1 .. 32 tiles per CTA, full 128-key tile, more (head, image) pairs than SMs;
    output and saved log-sum-exp against fp32 torch."""
    from ctrlora_b200 import ops
    torch.manual_seed(B * Nq + Nk)
    q, k, v = _rand(B * Nq, H * d), _rand(B * Nk, H * d), _rand(B * Nk, H * d)
    nk_pad = (Nk + 7) // 8 * 8
    vt = torch.zeros(B, H, d, nk_pad, device="cuda", dtype=torch.float16)
    vt[..., :Nk] = v.view(B, Nk, H, d).permute(0, 2, 3, 1)
    lse = torch.empty(B, H, Nq, device="cuda", dtype=torch.float32)
    out = ops.attention(q, k, vt, B, H, Nq, Nk, d, lse=lse)
    _close(out, _attn_ref(q, k, v, B, H, Nq, Nk, d), 3e-3)
    qf = q.float().view(B, Nq, H, d).permute(0, 2, 1, 3)
    kf = k.float().view(B, Nk, H, d).permute(0, 2, 1, 3)
    ref_lse = torch.logsumexp((qf @ kf.transpose(-1, -2)) * d ** -0.5, -1) * 1.4426950408889634
    assert (lse - ref_lse).abs().max().item() < 2e-3 * max(1.0, ref_lse.abs().max().item())


def test_attention_sharp_softmax():
    """Large logits (|s| ~ 30): the online-softmax rescaling must stay exact across KV tiles."""
    from ctrlora_b200 import ops
    torch.manual_seed(4)
    B, H, Nq, Nk, d = 1, 8, 512, 2048, 40
    q, k, v = _rand(B * Nq, H * d, s=3.0), _rand(B * Nk, H * d, s=3.0), _rand(B * Nk, H * d)
    vt = v.view(B, Nk, H, d).permute(0, 2, 3, 1).contiguous()
    out = ops.attention(q, k, vt, B, H, Nq, Nk, d)
    _close(out, _attn_ref(q, k, v, B, H, Nq, Nk, d), 4e-3)


def test_layout_roundtrip_bit_exact():
    from ctrlora_b200 import ops
    torch.manual_seed(5)
    x = torch.randn(3, 4, 16, 16, device="cuda")
    y = ops.nchw_to_nhwc_f16(x, 8)
    assert y.shape == (3, 16, 16, 8)
    assert torch.equal(y[..., :4], x.permute(0, 2, 3, 1).half()) and (y[..., 4:] == 0).all()
    back = ops.nhwc_to_nchw_f32(y, 4)
    assert torch.equal(back, x.half().float())
    z = torch.randn(2, 8, 8, 16, device="cuda")
    assert torch.equal(ops.nhwc_to_nchw_f32(z, 4), z[..., :4].permute(0, 3, 1, 2).contiguous())


def test_timestep_embedding():
    from ctrlora_b200 import ops
    t = torch.tensor([0, 1, 21, 500, 981, 999], device="cuda")
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32) / half)
    out = ops.timestep_embedding(t, freqs.cuda())
    args = t.cpu()[:, None].float() * freqs[None]
    ref = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    assert (out.cpu() - ref).abs().max().item() < 2e-6  # same fp32 arguments; cos/sin differ by <= 2 ulp


@pytest.mark.parametrize("rows,K,N,si,so", [(4, 320, 1280, False, True), (8, 1280, 1280, False, False),
                                            (16, 1280, 6400, True, False), (2, 32, 128, True, False)])
def test_small_linear(rows, K, N, si, so):
    from ctrlora_b200 import ops
    torch.manual_seed(6)
    x = torch.randn(rows, K, device="cuda")
    w = _rand(N, K, s=K ** -0.5)
    b = torch.randn(N, device="cuda")
    y = ops.small_linear(x, w, b, silu_in=si, silu_out=so)
    xin = F.silu(x) if si else x
    ref = xin @ w.float().t() + b
    ref = F.silu(ref) if so else ref
    _close(y, ref, 1e-4)


def test_upsample_and_stride2_gather_bit_exact():
    from ctrlora_b200 import ops
    torch.manual_seed(7)
    x = _rand(2, 8, 8, 64)
    up = ops.upsample2x(x)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1).half()
    assert torch.equal(up, ref)
    col = ops.im2col_s2(x)  # [B, 4, 4, 9*C]
    w = _rand(48, 9, 64, s=(9 * 64) ** -0.5)
    y = ops.gemm(col.view(-1, 9 * 64), w.view(48, 1, 9 * 64))
    wt = w.float().view(48, 3, 3, 64).permute(0, 3, 1, 2)
    yref = F.conv2d(x.float().permute(0, 3, 1, 2), wt, stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, 48)
    _close(y, yref)


def test_cast_transpose_bit_exact():
    from ctrlora_b200 import ops
    torch.manual_seed(8)
    w = torch.randn(24, 16, 3, 3, device="cuda")  # Conv2d [Cout, Cin, kh, kw] -> [Cout, 9, Cin]
    out = ops.cast_transpose(w, 24, 16, 9)
    assert torch.equal(out, w.view(24, 16, 9).permute(0, 2, 1).half())
    lin = torch.randn(40, 64, device="cuda")
    assert torch.equal(ops.cast_transpose(lin, 40 * 64, 1, 1).view(40, 64), lin.half())
    assert torch.equal(ops.cast_transpose(lin, 1, 40, 64).view(64, 40), lin.t().half())


@pytest.mark.parametrize("cfg,eta_sigma", [(7.5, 0.0), (1.0, 0.0), (7.5, 0.3)])
def test_ddim_update_bit_exact(cfg, eta_sigma):
    """Same fp32 op order as cldm/ddim_hacked.py:190-231 -> bit-identical to torch on the same inputs."""
    from ctrlora_b200 import ops
    torch.manual_seed(9)
    B = 4
    x, ec, eu, nz = (torch.randn(B, 4, 64, 64, device="cuda") for _ in range(4))
    a_t, a_prev, sig, s1m = 0.0473, 0.0558, eta_sigma, math.sqrt(1 - 0.0473)
    use_u = cfg != 1.0
    stats = torch.empty(B, device="cuda")
    xp, p0 = ops.ddim_update(x, ec, eu if use_u else None, cfg, a_t, a_prev, sig, s1m, noise=nz if sig else None,
                             temperature=0.9, stats=stats)
    full = lambda v: torch.full((B, 1, 1, 1), v, device="cuda")
    e = eu + cfg * (ec - eu) if use_u else ec
    A, AP, S, SM = full(a_t), full(a_prev), full(sig), full(s1m)
    p0_ref = (x - SM * e) / A.sqrt()
    dir_xt = (1.0 - AP - S ** 2).sqrt() * e
    noise = S * nz * 0.9 if sig else torch.zeros_like(x)
    xp_ref = AP.sqrt() * p0_ref + dir_xt + noise
    assert torch.equal(p0, p0_ref)
    assert torch.equal(xp, xp_ref)
    _close(stats, (xp_ref ** 2).sum(dim=(1, 2, 3)), 1e-4)
