"""Ping-pong tiles of the wgmma implicit GEMM (ctrlora_gemm_f16): each consumer warpgroup owns a whole 128-row tile
and runs its epilogue while the other warpgroup's MMAs run.

A launch runs ping-pong when all its units are whole tiles with the TMA epilogue and its K loop is short; an explicit
block_n of 64, 128 or 160 (GEGLU 64) with split_k=1 selects it, and block_n 256 / 320 (GEGLU 128 / 160) selects the
cooperative tile of the same launch.  Both compute every element in the same order, so they must agree bit for bit.
References are torch fp32 on the same fp16-rounded operands.
"""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

pytestmark = pytest.mark.gpu

from tolerances import close as _close  # noqa: E402

GUARD = 7.0


def _rand(*shape, s=1.0):
    return (torch.randn(*shape, device="cuda") * s).half()


def _launch(a, w, N, kind, block_n, split_k, **kw):
    from ctrlora_b200 import ops
    if kind == "geglu":
        bias = torch.arange(2 * N, device="cuda", dtype=torch.float32) * 1e-3
        return ops.gemm(a, w, bias=bias, geglu=True, block_n=block_n, split_k=split_k, **kw)
    bias = torch.arange(N, device="cuda", dtype=torch.float32) * 1e-3
    return ops.gemm(a, w, bias=bias, block_n=block_n, split_k=split_k, **kw)


def _ref(a, w, N, kind, residual=None, rowbias=None, rows_per_img=0):
    M, K = a.numel() // a.shape[-1], a.shape[-1]
    y = a.reshape(M, K).float() @ w.reshape(w.shape[0], K).float().t()
    if kind == "geglu":
        bias = torch.arange(2 * N, device="cuda", dtype=torch.float32) * 1e-3
        y = y + bias
        return y[:, :N] * torch.nn.functional.gelu(y[:, N:])
    y = y + torch.arange(N, device="cuda", dtype=torch.float32) * 1e-3
    if rowbias is not None:
        y = y + rowbias.repeat_interleave(rows_per_img, dim=0)
    if residual is not None:
        y = y + residual.reshape(M, N).float()
    return y


# (level, M, K, N, kind) of the batch-8 step's short-K GEMMs (linears and 1x1 convs: M = 8 * H * W rows)
_STEP = [
    ("64x64", 32768, 320, 320, ""), ("64x64", 32768, 320, 320, "res"), ("64x64", 32768, 320, 1280, "geglu"),
    ("64x64", 32768, 1280, 320, "res"), ("32x32", 8192, 640, 640, ""), ("32x32", 8192, 2560, 640, "res"),
    ("16x16", 2048, 1280, 1280, ""),
]


@pytest.mark.parametrize("level,M,K,N,kind", _STEP)
def test_step_shapes_pingpong_equals_cooperative(level, M, K, N, kind):
    torch.manual_seed(M + K + N)
    wr = 2 * N if kind == "geglu" else N
    a, w = _rand(M, K), _rand(wr, 1, K, s=K ** -0.5)
    kw = {"residual": _rand(M, N)} if kind == "res" else {}
    if kind == "geglu":
        pp_widths, coop = [64], 160
    else:
        pp_widths, coop = [64, 128, 160], 320
    base = _launch(a, w, N, kind, coop, 1, **kw)
    auto = _launch(a, w, N, kind, 0, 0, **kw)
    for bn in pp_widths:
        if N % bn:
            continue
        got = _launch(a, w, N, kind, bn, 1, **kw)
        assert torch.equal(got, base), (level, bn)
    assert torch.equal(_launch(a, w, N, kind, 0, 1, **kw), base)
    _close(auto, _ref(a, w, N, kind, residual=kw.get("residual")))
    _close(base, _ref(a, w, N, kind, residual=kw.get("residual")))


def test_rowbias_and_scale():
    """Time-embedding row term over images of 4096 rows on a 64x64 1x1 conv, with out_scale and a residual."""
    from ctrlora_b200 import ops
    torch.manual_seed(5)
    B, HW, C, N = 8, 64, 320, 320
    a, w = _rand(B, HW, HW, C), _rand(N, 1, C, s=C ** -0.5)
    rowbias = torch.randn(B, N, device="cuda")
    res = _rand(B, HW, HW, N)
    kw = dict(rowbias=rowbias, rows_per_img=HW * HW, residual=res, out_scale=0.5)
    bias = torch.randn(N, device="cuda")
    outs = [ops.gemm(a, w, bias=bias, block_n=bn, split_k=1, **kw) for bn in (160, 64, 320)]
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[2])
    M = B * HW * HW
    ref = (a.reshape(M, C).float() @ w.reshape(N, C).float().t() + bias + rowbias.repeat_interleave(HW * HW, 0)) * 0.5
    _close(outs[0].reshape(M, N), ref + res.reshape(M, N).float())


@pytest.mark.parametrize("m_tiles", [4, 5, 8, 12, 13, 29])
@pytest.mark.parametrize("rows_short", [0, 37])
def test_tiles_per_cta(m_tiles, rows_short):
    """8 SMs and 2 n tiles: 8 .. 58 tiles, i.e. 1, 2, 3 and 7-8 tiles per CTA, CTAs ending on either warpgroup."""
    from ctrlora_b200 import ops
    torch.manual_seed(m_tiles * 3 + rows_short)
    M, K, N = 128 * m_tiles - rows_short, 640, 320
    a, w, res = _rand(M, K), _rand(N, 1, K, s=K ** -0.5), _rand(M, N)
    ops.set_sm_limit(8)
    try:
        got = _launch(a, w, N, "", 160, 1, residual=res)
        again = _launch(a, w, N, "", 160, 1, residual=res)
        base = _launch(a, w, N, "", 320, 1, residual=res)
    finally:
        ops.set_sm_limit(0)
    assert torch.equal(got, base) and torch.equal(got, again)
    _close(got, _ref(a, w, N, "", residual=res))


@pytest.mark.parametrize("block_n", [64, 128, 160, 256, 320])
def test_partial_tiles_and_column_slices(block_n):
    """M no multiple of 128 and N of no width, output and residual column slices of wider buffers: the guards keep
    their fill and both schedules give the same bits."""
    from ctrlora_b200 import ops
    torch.manual_seed(61)
    M, K, N = 128 * 9 + 37, 320, 320 + 168
    a, w = _rand(M, K), _rand(N, 1, K, s=K ** -0.5)
    bias = torch.randn(N, device="cuda")
    rbuf = torch.full((M + 3, 512), GUARD, device="cuda", dtype=torch.float16)
    res = rbuf[:M, 16:16 + N]
    res.copy_(_rand(M, N))
    obuf = torch.full((M + 3, 520), GUARD, device="cuda", dtype=torch.float16)
    out = obuf[:M, 24:24 + N]
    ops.gemm(a, w, bias=bias, residual=res, out=out, block_n=block_n, split_k=1)
    mask = torch.ones_like(obuf, dtype=torch.bool)
    mask[:M, 24:24 + N] = False
    assert bool((obuf[mask] == GUARD).all())
    ref = a.float() @ w.reshape(N, K).float().t() + bias + res.float()
    _close(out, ref)
    coop = ops.gemm(a, w, bias=bias, residual=res, block_n=256, split_k=1)
    assert torch.equal(out, coop)


@pytest.mark.parametrize("block_n", [160, 64])
def test_out_aliases_residual(block_n):
    from ctrlora_b200 import ops
    torch.manual_seed(62)
    M, K, N = 128 * 40 + 5, 1280, 320
    a, w = _rand(M, K), _rand(N, 1, K, s=K ** -0.5)
    x = _rand(M, N)
    expect = ops.gemm(a, w, residual=x, block_n=320, split_k=1)
    y = x.clone()
    ops.gemm(a, w, residual=y, out=y, block_n=block_n, split_k=1)
    assert torch.equal(y, expect)


def test_pingpong_then_cooperative_in_one_graph():
    """A ping-pong launch feeding a cooperative one (a 3x3 conv) inside one CUDA graph, replayed."""
    from ctrlora_b200 import ops
    torch.manual_seed(63)
    B, HW, C, N = 8, 32, 640, 640
    a = _rand(B, HW, HW, C)
    w1, w2 = _rand(N, 1, C, s=C ** -0.5), _rand(N, 9, N, s=(9 * N) ** -0.5)
    res = _rand(B, HW, HW, N)

    def run():
        h = ops.gemm(a, w1, residual=res, block_n=160, split_k=1)
        return ops.gemm(h, w2, ksize=3)

    eager = run()
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        run()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            out = run()
        for _ in range(3):
            graph.replay()
    torch.cuda.current_stream().wait_stream(stream)
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
