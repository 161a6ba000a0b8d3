"""GPU parity of the wgmma implicit GEMM (ctrlora_gemm_f16) against torch fp32 on the same fp16-rounded operands.

Tolerance: fp16 output rounding (2^-11 relative) + fp32 accumulation-order differences -> 2e-3 * max|ref| absolute.
"""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


from tolerances import close as _close  # noqa: E402  (max-abs guard AND norm-relative <= 1e-3)


def _rand(*shape, s=1.0):
    return (torch.randn(*shape, device="cuda") * s).half()


def _conv_ref(a, w, ksize):
    # a [B,H,W,C] fp16, w [N, taps, C] fp16 -> [B,H,W,N] fp32
    n = w.shape[0]
    wt = w.float().view(n, ksize, ksize, -1).permute(0, 3, 1, 2)
    y = F.conv2d(a.float().permute(0, 3, 1, 2), wt, padding=(ksize - 1) // 2)
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("simt", [True, False])
@pytest.mark.parametrize("M,K,N", [(300, 320, 320), (128, 64, 16), (1000, 768, 640), (77, 328, 48)])
def test_linear(M, K, N, simt):
    from ctrlora_b200 import ops
    torch.manual_seed(0)
    a, w = _rand(M, K), _rand(N, 1, K, s=K ** -0.5)
    bias = torch.randn(N, device="cuda")
    res = _rand(M, N)
    out = ops.gemm(a, w, bias=bias, residual=res, out_scale=0.5, simt=simt)
    ref = (a.float() @ w.float().view(N, K).t() + bias) * 0.5 + res.float()
    _close(out, ref)


@pytest.mark.parametrize("simt", [True, False])
@pytest.mark.parametrize("B,H,W,C,N", [(2, 16, 16, 64, 128), (3, 8, 8, 128, 64), (1, 32, 32, 72, 80), (5, 4, 4, 64, 32),
                                        (2, 64, 64, 8, 320)])
def test_conv3x3(B, H, W, C, N, simt):
    from ctrlora_b200 import ops
    torch.manual_seed(1)
    a, w = _rand(B, H, W, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
    bias = torch.randn(N, device="cuda")
    rowbias = torch.randn(B, N, device="cuda")
    out = ops.gemm(a, w, ksize=3, bias=bias, rowbias=rowbias, simt=simt)
    ref = _conv_ref(a, w, 3) + bias + rowbias[:, None, None, :]
    _close(out, ref)


@pytest.mark.parametrize("simt", [True, False])
def test_conv3x3_with_skip_operand(simt):
    from ctrlora_b200 import ops
    torch.manual_seed(2)
    B, H, W, C, C2, N = 2, 16, 16, 128, 192, 128
    a, w = _rand(B, H, W, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
    a2, w2 = _rand(B, H, W, C2), _rand(N, C2, s=C2 ** -0.5)
    bias = torch.randn(N, device="cuda")
    out = ops.gemm(a, w, ksize=3, bias=bias, a2=a2, w2=w2, simt=simt)
    ref = _conv_ref(a, w, 3) + bias + a2.float() @ w2.float().t()
    _close(out, ref)


@pytest.mark.parametrize("simt", [True, False])
def test_geglu(simt):
    from ctrlora_b200 import ops
    torch.manual_seed(3)
    M, K, N = 512, 320, 1280
    a, w = _rand(M, K), _rand(2 * N, 1, K, s=K ** -0.5)
    bias = torch.randn(2 * N, device="cuda")
    out = ops.gemm(a, w, bias=bias, geglu=True, simt=simt)
    y = a.float() @ w.float().view(2 * N, K).t() + bias
    ref = y[:, :N] * F.gelu(y[:, N:])
    _close(out, ref)


@pytest.mark.parametrize("simt", [True, False])
def test_qkv_segments_with_transposed_v(simt):
    from ctrlora_b200 import ops
    torch.manual_seed(4)
    Bimg, T, K, Cq, heads = 2, 256, 320, 320, 8
    d = Cq // heads
    a, w = _rand(Bimg * T, K), _rand(3 * Cq, 1, K, s=K ** -0.5)
    q = torch.empty(Bimg * T, Cq, device="cuda", dtype=torch.float16)
    k = torch.empty_like(q)
    vt = torch.zeros(Bimg, heads, d, T, device="cuda", dtype=torch.float16)
    ops.gemm(a, w, seg_outs=[q, k, vt], seg_width=Cq, transposed=(0, 0, 1), rows_per_img=T, head_dim=d, tok_pad=T,
             simt=simt)
    y = a.float() @ w.float().view(3 * Cq, K).t()
    _close(q, y[:, :Cq])
    _close(k, y[:, Cq:2 * Cq])
    v_ref = y[:, 2 * Cq:].view(Bimg, T, heads, d).permute(0, 2, 3, 1)
    _close(vt, v_ref)


def test_out_f32_small_n():
    from ctrlora_b200 import ops
    torch.manual_seed(5)
    B, H, W, C = 2, 64, 64, 320
    a = _rand(B, H, W, C)
    w = torch.zeros(16, 9, C, device="cuda", dtype=torch.float16)
    w[:4] = _rand(4, 9, C, s=(9 * C) ** -0.5)
    out = ops.gemm(a, w, ksize=3, out_f32=True)
    ref = _conv_ref(a, w, 3)
    _close(out, ref, tol=1e-4)


def test_sd_shapes_and_speed():
    """Full-size SD1.5 shapes: results against torch, and a first throughput reading (printed, not asserted)."""
    from ctrlora_b200 import ops
    torch.manual_seed(6)
    for (B, H, W, C, N, ks) in [(4, 64, 64, 320, 320, 3), (4, 32, 32, 640, 640, 3), (4, 16, 16, 1280, 1280, 3),
                                (4, 8, 8, 1280, 1280, 3), (4, 64, 64, 320, 320, 1), (4, 16, 16, 2560, 1280, 3)]:
        a, w = _rand(B, H, W, C), _rand(N, ks * ks, C, s=(ks * ks * C) ** -0.5)
        out = ops.gemm(a, w, ksize=ks)
        _close(out, _conv_ref(a, w, ks))
        for _ in range(3):
            ops.gemm(a, w, ksize=ks, out=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.gemm(a, w, ksize=ks, out=out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        fl = 2.0 * B * H * W * N * C * ks * ks
        print(f"conv{ks}x{ks} B{B} {H}x{W} {C}->{N}: {ms * 1e3:.1f} us  {fl / ms / 1e9:.1f} TFLOP/s")


@pytest.mark.parametrize("split", [2, 3, 4, 8])
@pytest.mark.parametrize("case", ["conv", "skip", "geglu", "qkv"])
def test_split_k(split, case):
    """Forced split-K: partial tiles are parked in fp32 workspace slices; the last CTA to arrive sums them (fixed order)
    and runs the epilogue."""
    from ctrlora_b200 import ops
    torch.manual_seed(10 + split)
    if case == "conv":
        B, H, W, C, N = 4, 8, 8, 640, 320
        a, w = _rand(B, H, W, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
        bias, rb, res = torch.randn(N, device="cuda"), torch.randn(B, N, device="cuda"), _rand(B * H * W, N)
        out = ops.gemm(a, w, ksize=3, bias=bias, rowbias=rb, residual=res, split_k=split)
        ref = _conv_ref(a, w, 3) + bias + rb[:, None, None, :] + res.float().view(B, H, W, N)
        _close(out, ref)
    elif case == "skip":
        B, H, W, C, C2, N = 2, 8, 8, 256, 512, 192
        a, w = _rand(B, H, W, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
        a2, w2 = _rand(B, H, W, C2), _rand(N, C2, s=C2 ** -0.5)
        out = ops.gemm(a, w, ksize=3, a2=a2, w2=w2, split_k=split)
        _close(out, _conv_ref(a, w, 3) + a2.float() @ w2.float().t())
    elif case == "geglu":
        M, K, N = 300, 1280, 640
        a, w = _rand(M, K), _rand(2 * N, 1, K, s=K ** -0.5)
        bias = torch.randn(2 * N, device="cuda")
        out = ops.gemm(a, w, bias=bias, geglu=True, split_k=split)
        y = a.float() @ w.float().view(2 * N, K).t() + bias
        _close(out, y[:, :N] * F.gelu(y[:, N:]))
    else:
        Bimg, T, K, Cq, heads = 2, 64, 1280, 320, 8
        d = Cq // heads
        a, w = _rand(Bimg * T, K), _rand(3 * Cq, 1, K, s=K ** -0.5)
        q = torch.empty(Bimg * T, Cq, device="cuda", dtype=torch.float16)
        k = torch.empty_like(q)
        vt = torch.zeros(Bimg, heads, d, T, device="cuda", dtype=torch.float16)
        ops.gemm(a, w, seg_outs=[q, k, vt], seg_width=Cq, transposed=(0, 0, 1), rows_per_img=T, head_dim=d, tok_pad=T,
                 split_k=split)
        y = a.float() @ w.float().view(3 * Cq, K).t()
        _close(q, y[:, :Cq])
        _close(k, y[:, Cq:2 * Cq])
        _close(vt, y[:, 2 * Cq:].view(Bimg, T, heads, d).permute(0, 2, 3, 1))
    ws, cnt = ops._splitk_buffers(torch.device("cuda", 0))
    assert cnt.abs().max().item() == 0  # counters are self-cleaning


def test_split_k_auto_small_m():
    """The selection model splits K on tile-starved problems (8x8 feature maps) and results do not change."""
    from ctrlora_b200 import ops
    torch.manual_seed(30)
    B, H, W, C, N = 8, 8, 8, 1280, 1280
    a, w = _rand(B, H, W, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
    out = ops.gemm(a, w, ksize=3)
    _close(out, _conv_ref(a, w, 3))
