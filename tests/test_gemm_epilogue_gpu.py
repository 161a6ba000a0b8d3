"""The TMA epilogue of the wgmma implicit GEMM (ctrlora_gemm_f16) and its 160-column tiles.

fp16 row-major outputs leave a tile through swizzled shared-memory slots that are stored by TMA, after the tile's
residual box has been loaded into the same slots ahead of time; the output and residual maps clip partial tiles and
column slices of wider buffers.  fp32 / transposed / unaligned outputs and split tiles keep the row-per-thread epilogue.
Both compute each element in the same order, and splitting N differently does not change the order of a K sum, so
unsplit results are bit-identical across tile widths and across the two epilogues.  References are torch fp32 on the
same fp16-rounded operands.
"""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from tolerances import close as _close  # noqa: E402
from test_gemm_persistent_gpu import _step_shapes  # noqa: E402

GUARD = 7.0


def _rand(*shape, s=1.0):
    return (torch.randn(*shape, device="cuda") * s).half()


def _conv_ref(a, w, ksize):
    n = w.shape[0]
    wt = w.float().view(n, ksize, ksize, -1).permute(0, 3, 1, 2)
    return F.conv2d(a.float().permute(0, 3, 1, 2), wt, padding=(ksize - 1) // 2).permute(0, 2, 3, 1)


def _guarded(rows, cols, ld, col0, guard_rows=3):
    """A [rows, cols] column slice at column col0 of a wider [rows + guard_rows, ld] buffer filled with GUARD."""
    buf = torch.full((rows + guard_rows, ld), GUARD, device="cuda", dtype=torch.float16)
    return buf, buf[:rows, col0:col0 + cols]


def _guards_intact(buf, rows, cols, col0):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[:rows, col0:col0 + cols] = False
    return bool((buf[mask] == GUARD).all())


_SHAPES_160 = [s for s in _step_shapes() if s[6] != "geglu" and (s[4] // 3 if s[6] == "qkv" else s[4]) % 160 == 0]


@pytest.mark.parametrize("B,H,W,C,N,ks,epi", _SHAPES_160)
def test_step_shapes_bn160_bit_identical(B, H, W, C, N, ks, epi):
    """Every GEMM of the batch-8 step whose width 160 divides: 160-column tiles equal 64-column tiles bit for bit."""
    from test_gemm_bn320_gpu import _run
    torch.manual_seed(B * 5 + H + C + N + ks)
    M = B * H * W
    a = _rand(M, C) if H == 1 else _rand(B, H, W, C)
    w = _rand(N, ks * ks, C, s=(ks * ks * C) ** -0.5)
    got, base = _run(a, w, ks, epi, N, 160, 1), _run(a, w, ks, epi, N, 64, 1)
    for x, y in zip(got, base):
        assert torch.equal(x, y)
    if epi == "":
        ref = a.float() @ w.float().view(N, C).t() if H == 1 else _conv_ref(a, w, ks).reshape(M, N)
        _close(got[0].reshape(M, N), ref + torch.arange(N, device="cuda") * 1e-3)


@pytest.mark.parametrize("block_n", [32, 64, 128, 160, 256, 320])
def test_column_slices_partial_tiles_and_guards(block_n):
    """Output and residual are column slices of wider buffers (ldc != ldr, both > N), N is no multiple of any tile
    width and M none of 128: guard columns and guard rows keep their fill, and every width gives the same bits."""
    from ctrlora_b200 import ops
    torch.manual_seed(60)
    M, K, N = 128 * 5 + 37, 320, 320 + 168
    a, w = _rand(M, K), _rand(N, 1, K, s=K ** -0.5)
    bias = torch.randn(N, device="cuda")
    rbuf, res = _guarded(M, N, 512, 16)
    res.copy_(_rand(M, N))
    obuf, out = _guarded(M, N, 520, 24)
    ops.gemm(a, w, bias=bias, residual=res, out=out, block_n=block_n, split_k=1)
    assert _guards_intact(obuf, M, N, 24) and _guards_intact(rbuf, M, N, 16)
    _close(out, a.float() @ w.float().view(N, K).t() + bias + res.float())
    obuf2, out2 = _guarded(M, N, 520, 24)
    ops.gemm(a, w, bias=bias, residual=res, out=out2, block_n=64, split_k=1)
    assert torch.equal(out, out2)


@pytest.mark.parametrize("block_n", [64, 160, 320])
def test_conv_24x24_partial_boxes_and_batch(block_n):
    """A 24x24 image (16-wide pixel boxes overhang the right and lower edges) and, at 8x8 (2 images per tile), a batch
    of 3 that does not fill the last tile; 3x3 conv with residual into a column slice."""
    from ctrlora_b200 import ops
    torch.manual_seed(61)
    for (B, H, C, N) in ((2, 24, 128, 320), (3, 8, 192, 320)):
        a, w = _rand(B, H, H, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
        res = _rand(B, H, H, N)
        M = B * H * H
        obuf, out = _guarded(M, N, N + 40, 8)
        ops.gemm(a, w, ksize=3, residual=res, out=out.view(B, H, H, N), block_n=block_n, split_k=1)
        assert _guards_intact(obuf, M, N, 8)
        _close(out.reshape(B, H, H, N), _conv_ref(a, w, 3) + res.float())


@pytest.mark.parametrize("block_n", [0, 64, 160, 256])
def test_rowbias_image_boundary_inside_tile(block_n):
    """The time-embedding row term where a 128-row tile spans two images: the 8x8 level, and a linear with 64 rows per
    image; together with out_scale != 1 and a residual.  Order per element: (acc + bias + rowbias) * scale + residual."""
    from ctrlora_b200 import ops
    torch.manual_seed(62)
    B, H, C, N = 6, 8, 320, 320
    a, w = _rand(B, H, H, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
    rb, bias, res = torch.randn(B, N, device="cuda"), torch.randn(N, device="cuda"), _rand(B, H, H, N)
    out = ops.gemm(a, w, ksize=3, bias=bias, rowbias=rb, residual=res, out_scale=0.625, block_n=block_n, split_k=1)
    _close(out, (_conv_ref(a, w, 3) + bias + rb.view(B, 1, 1, N)) * 0.625 + res.float())
    a2, w2 = a.view(B * 64, C), _rand(N, 1, C, s=C ** -0.5)
    out2 = ops.gemm(a2, w2, bias=bias, rowbias=rb, rows_per_img=64, residual=res.view(B * 64, N), out_scale=0.625,
                    block_n=block_n, split_k=1)
    ref2 = (a2.float() @ w2.float().view(N, C).t() + bias + rb.repeat_interleave(64, 0)) * 0.625 + res.view(B * 64, N).float()
    _close(out2, ref2)


def test_out_aliases_residual():
    """In place: a tile loads its residual box before it stores, and touches no other tile's box."""
    from ctrlora_b200 import ops
    torch.manual_seed(63)
    M, K, N = 8 * 1024 + 50, 1280, 320
    a, w = _rand(M, K), _rand(N, 1, K, s=K ** -0.5)
    res = _rand(M, N)
    want = ops.gemm(a, w, residual=res)
    buf = res.clone()
    ops.gemm(a, w, residual=buf, out=buf)
    assert torch.equal(buf, want)
    _close(buf, a.float() @ w.float().view(N, K).t() + res.float())


def test_fallback_next_to_tma_epilogue():
    """Argument sets the TMA epilogue does not cover (unaligned ldc, fp32 residual, fp32 output, V^T with a row-major
    copy) next to ones it does: all correct, and the fp16 ones bit-identical to each other."""
    from ctrlora_b200 import ops
    torch.manual_seed(64)
    M, K, N = 1024 + 19, 640, 320
    a, w = _rand(M, K), _rand(N, 1, K, s=K ** -0.5)
    res = _rand(M, N)
    ref = a.float() @ w.float().view(N, K).t()
    tma = ops.gemm(a, w, residual=res)
    obuf, odd = _guarded(M, N, N + 4, 0)   # ldc = 324: rows are not 16-byte aligned
    ops.gemm(a, w, residual=res, out=odd)
    assert torch.equal(odd, tma) and _guards_intact(obuf, M, N, 0)
    obuf, shifted = _guarded(M, N, N + 8, 4)  # base pointer 8 bytes off
    ops.gemm(a, w, residual=res, out=shifted)
    assert torch.equal(shifted, tma) and _guards_intact(obuf, M, N, 4)
    _close(tma, ref + res.float())
    _close(ops.gemm(a, w, residual=res.float()), ref + res.float())
    _close(ops.gemm(a, w, residual=res, out_f32=True), ref + res.float(), tol=1e-4)
    # q | k | V^T: q and k by TMA store, V^T and its row-major copy row per thread
    imgs, heads, T, cq = 4, 8, 256, 320
    a3, w3 = _rand(imgs * T, K), _rand(3 * cq, 1, K, s=K ** -0.5)
    y = a3.float() @ w3.float().view(3 * cq, K).t()
    for bn in (0, 64, 160, 320):
        q, k, v = (torch.empty(imgs * T, cq, device="cuda", dtype=torch.float16) for _ in range(3))
        vt = torch.zeros(imgs, heads, cq // heads, T, device="cuda", dtype=torch.float16)
        ops.gemm(a3, w3, seg_outs=[q, k, vt], seg_width=cq, transposed=(0, 0, 1), rows_per_img=T, head_dim=cq // heads,
                 tok_pad=T, dup_out=v, block_n=bn, split_k=1 if bn else 0)
        _close(q, y[:, :cq])
        _close(k, y[:, cq:2 * cq])
        _close(v, y[:, 2 * cq:])
        assert torch.equal(vt, v.view(imgs, T, heads, cq // heads).permute(0, 2, 3, 1))


@pytest.mark.parametrize("split", [0, 3])
def test_split_k_with_residual_and_rowbias(split):
    """Split tiles (explicit: every tile; automatic: the partial wave of 160 tiles on 132 SMs) keep the row-per-thread
    epilogue, in the same launch as whole tiles on the TMA epilogue."""
    from ctrlora_b200 import ops
    torch.manual_seed(65 + split)
    B, H, C, N = 8, 16, 1280, 1280
    a, w = _rand(B, H, H, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
    rb, res = torch.randn(B, N, device="cuda"), _rand(B, H, H, N)
    _, cnt = ops._splitk_buffers(torch.device("cuda", 0))
    out = ops.gemm(a, w, ksize=3, rowbias=rb, residual=res, block_n=128, split_k=split)
    torch.cuda.synchronize()
    assert cnt.abs().max().item() == 0
    _close(out, _conv_ref(a, w, 3) + rb.view(B, 1, 1, N) + res.float())
    assert torch.equal(out, ops.gemm(a, w, ksize=3, rowbias=rb, residual=res, block_n=128, split_k=split))


def test_graph_replay_and_sm_limit():
    """Residual GEMMs with automatic plans replayed from a CUDA graph, and on 7 / 100 CTAs (each CTA then walks many
    tiles through its slots): same bits as the eager full-grid launch."""
    from ctrlora_b200 import ops
    torch.manual_seed(66)
    a, w = _rand(8 * 4096, 320), _rand(320, 1, 320, s=320 ** -0.5)
    res = _rand(8 * 4096, 320)
    a2, w2 = _rand(8, 32, 32, 640), _rand(640, 9, 640, s=(9 * 640) ** -0.5)
    res2 = _rand(8, 32, 32, 640)
    eager = [ops.gemm(a, w, residual=res), ops.gemm(a2, w2, ksize=3, residual=res2)]
    _close(eager[0], a.float() @ w.float().view(320, 320).t() + res.float())
    _close(eager[1], _conv_ref(a2, w2, 3) + res2.float())
    whole = [ops.gemm(a, w, residual=res, block_n=64, split_k=1), ops.gemm(a2, w2, ksize=3, residual=res2, split_k=1)]
    for k in (7, 100):
        ops.set_sm_limit(k)
        try:
            lim = [ops.gemm(a, w, residual=res, block_n=160, split_k=1), ops.gemm(a2, w2, ksize=3, residual=res2, split_k=1)]
        finally:
            ops.set_sm_limit(0)
        assert torch.equal(lim[0], whole[0]) and torch.equal(lim[1], whole[1])
    o1, o2 = torch.empty_like(eager[0]), torch.empty_like(eager[1])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.gemm(a, w, residual=res, out=o1)
        ops.gemm(a2, w2, ksize=3, residual=res2, out=o2)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.gemm(a, w, residual=res, out=o1)
            ops.gemm(a2, w2, ksize=3, residual=res2, out=o2)
    torch.cuda.current_stream().wait_stream(s)
    o1.zero_()
    o2.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(o1, eager[0]) and torch.equal(o2, eager[1])
