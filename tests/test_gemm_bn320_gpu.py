"""320-column tiles of the wgmma implicit GEMM (ctrlora_gemm_f16): two m64n160 MMAs per k16 and two 160-row B boxes
per stage; GEGLU tiles carry 160 value + 160 gate columns.

Splitting N differently does not change the order in which an output element sums over K, so without a K split a
320-column tile is bit-identical to narrower tiles.  References are torch fp32 on the same fp16-rounded operands.
"""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from tolerances import close as _close  # noqa: E402
from test_gemm_persistent_gpu import _conv_ref, _rand, _step_shapes  # noqa: E402


def _run(a, w, ks, epi, N, block_n, split_k):
    """One launch of a _step_shapes() entry with an explicit tile width; returns the output tensors."""
    from ctrlora_b200 import ops
    M = a.numel() // a.shape[-1]
    if epi == "geglu":
        bias = torch.arange(2 * N, device="cuda", dtype=torch.float32) * 1e-3
        return [ops.gemm(a, w, bias=bias, geglu=True, block_n=block_n, split_k=split_k)]
    if epi == "qkv":
        cq, heads, imgs = N // 3, 8, 8
        T = M // imgs
        q = torch.empty(M, cq, device="cuda", dtype=torch.float16)
        k, v = torch.empty_like(q), torch.empty_like(q)
        vt = torch.zeros(imgs, heads, cq // heads, T, device="cuda", dtype=torch.float16)
        ops.gemm(a, w, seg_outs=[q, k, vt], seg_width=cq, transposed=(0, 0, 1), rows_per_img=T, head_dim=cq // heads,
                 tok_pad=T, dup_out=v, block_n=block_n, split_k=split_k)
        return [q, k, vt, v]
    bias = torch.arange(N, device="cuda", dtype=torch.float32) * 1e-3
    kw = {}
    g = torch.Generator(device="cuda").manual_seed(N + ks)
    if epi == "res":
        kw["residual"] = torch.randn(M, N, device="cuda", generator=g).half()
    elif epi.startswith("skip"):
        c2 = int(epi[4:])
        kw["a2"] = torch.randn(*a.shape[:-1], c2, device="cuda", generator=g).half()
        kw["w2"] = (torch.randn(N, c2, device="cuda", generator=g) * c2 ** -0.5).half()
    return [ops.gemm(a, w, ksize=ks, bias=bias, block_n=block_n, split_k=split_k, **kw)]


@pytest.mark.parametrize("B,H,W,C,N,ks,epi", _step_shapes())
def test_step_shapes_bn320_bit_identical(B, H, W, C, N, ks, epi):
    """Every distinct GEMM of the batch-8 step: 320-column tiles (GEGLU 160 + 160) equal 64-column tiles bit for bit
    when no tile is split, and match the fp32 reference."""
    torch.manual_seed(B * 7 + H + C + N + ks)
    M = B * H * W
    a = _rand(M, C) if H == 1 else _rand(B, H, W, C)
    kk = ks * ks
    rows = 2 * N if epi == "geglu" else N
    w = _rand(rows, kk, C, s=(kk * C) ** -0.5)
    wide = 160 if epi == "geglu" else 320
    narrow = 32 if epi == "geglu" else 64
    got = _run(a, w, ks, epi, N, wide, 1)
    base = _run(a, w, ks, epi, N, narrow, 1)
    for x, y in zip(got, base):
        assert torch.equal(x, y)
    if epi == "":
        ref = (a.float() @ w.float().view(N, C).t() if H == 1 else _conv_ref(a, w, ks).reshape(M, N))
        _close(got[0].reshape(M, N), ref + torch.arange(N, device="cuda") * 1e-3)


def test_bn320_equals_bn256():
    """N = 1280 at the 16x16 level: 4 tiles of 320 columns against 5 of 256, bit for bit."""
    from ctrlora_b200 import ops
    torch.manual_seed(50)
    a, w = _rand(8, 16, 16, 1280), _rand(1280, 9, 1280, s=(9 * 1280) ** -0.5)
    rb = torch.randn(8, 1280, device="cuda")
    o320 = ops.gemm(a, w, ksize=3, rowbias=rb, block_n=320, split_k=1)
    o256 = ops.gemm(a, w, ksize=3, rowbias=rb, block_n=256, split_k=1)
    assert torch.equal(o320, o256)
    _close(o320, _conv_ref(a, w, 3) + rb.view(8, 1, 1, 1280))


def test_bn320_partial_n_tile_and_odd_m():
    """N not a multiple of 320 (the second 160-row box is partly out of bounds) and a partial last M tile."""
    from ctrlora_b200 import ops
    torch.manual_seed(51)
    M, K, N = 128 * 7 + 37, 640, 320 + 168
    a, w = _rand(M, K), _rand(N, 1, K, s=K ** -0.5)
    res = torch.randn(M, N, device="cuda")
    out = ops.gemm(a, w, residual=res, out_f32=True, block_n=320, split_k=1)
    _close(out, a.float() @ w.float().view(N, K).t() + res, tol=1e-4)


@pytest.mark.parametrize("split", [2, 5])
def test_bn320_split_k(split):
    """Every tile split along K at 320 columns (workspace slices of 128 x 320): result, and counters back at zero."""
    from ctrlora_b200 import ops
    torch.manual_seed(52 + split)
    B, H, W, C, N = 8, 8, 8, 1280, 1280
    a, w = _rand(B, H, W, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
    a2, w2 = _rand(B, H, W, 640), _rand(N, 640, s=640 ** -0.5)
    ws, cnt = ops._splitk_buffers(torch.device("cuda", 0))
    out = ops.gemm(a, w, ksize=3, a2=a2, w2=w2, block_n=320, split_k=split)
    torch.cuda.synchronize()
    assert cnt.abs().max().item() == 0
    _close(out, _conv_ref(a, w, 3) + a2.float() @ w2.float().t())
    assert torch.equal(out, ops.gemm(a, w, ksize=3, a2=a2, w2=w2, block_n=320, split_k=split))


def test_bn320_sm_limit():
    """Under ctrlora_set_sm_limit(k) (7 CTAs walk 256 tiles each with the ring carried across them) 320-column tiles
    give the same bits."""
    from ctrlora_b200 import ops
    torch.manual_seed(55)
    a, w = _rand(8, 64, 64, 320), _rand(320, 9, 320, s=(9 * 320) ** -0.5)
    full = ops.gemm(a, w, ksize=3, block_n=320, split_k=1)
    for k in (7, 100):
        ops.set_sm_limit(k)
        try:
            out = ops.gemm(a, w, ksize=3, block_n=320, split_k=1)
        finally:
            ops.set_sm_limit(0)
        assert torch.equal(out, full)


def test_bn320_graph_replay():
    """The automatically planned launches (320-column tiles at these widths) replayed from a CUDA graph."""
    from ctrlora_b200 import ops
    torch.manual_seed(56)
    a, w = _rand(8, 32, 32, 640), _rand(640, 9, 640, s=(9 * 640) ** -0.5)
    ag, wg = _rand(8 * 32 * 32, 640), _rand(2 * 2560, 1, 640, s=640 ** -0.5)
    eager = [ops.gemm(a, w, ksize=3), ops.gemm(ag, wg, geglu=True)]
    out1 = torch.empty_like(eager[0])
    out2 = torch.empty_like(eager[1])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.gemm(a, w, ksize=3, out=out1)
        ops.gemm(ag, wg, geglu=True, out=out2)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.gemm(a, w, ksize=3, out=out1)
            ops.gemm(ag, wg, geglu=True, out=out2)
    torch.cuda.current_stream().wait_stream(s)
    out1.zero_()
    out2.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out1, eager[0]) and torch.equal(out2, eager[1])
    _close(out2, (lambda y: y[:, :2560] * F.gelu(y[:, 2560:]))(ag.float() @ wg.float().view(5120, 640).t()))
