"""The persistent wgmma implicit GEMM (ctrlora_gemm_f16): every distinct GEMM of the batch-8 sampling step at full size,
the edges of the persistent schedule, the SM budget, 256-column tiles, the tail split-K and run-to-run reproducibility.

References are torch fp32 on the same fp16-rounded operands, compared with tolerances.close.
"""
import json
import os
import sys
import tempfile

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from tolerances import close as _close  # noqa: E402


def _rand(*shape, s=1.0):
    return (torch.randn(*shape, device="cuda") * s).half()


def _conv_ref(a, w, ksize):
    n = w.shape[0]
    wt = w.float().view(n, ksize, ksize, -1).permute(0, 3, 1, 2)
    y = F.conv2d(a.float().permute(0, 3, 1, 2), wt, padding=(ksize - 1) // 2)
    return y.permute(0, 2, 3, 1)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _step_shapes():
    """(B, H, W, Cin, N, ksize, epilogue) of every distinct GEMM of one SD1.5 UNet + ControlNet pass at batch 8
    (512x512, latent 64x64).  Linears are B = H = 1, W = rows.  epilogue: "" | "res" (fp16 residual) | "geglu" |
    "qkv" (q / k / V^T segments) | "skip<C2>" (fused 1x1 skip convolution of a C2-channel input)."""
    shapes = []
    for hw, c in ((64, 320), (32, 640), (16, 1280), (8, 1280)):
        m = 8 * hw * hw
        # transformer blocks (levels 64 .. 16) and the mid block's (level 8): proj_in / proj_out, q / k / v, out, FF
        shapes += [(1, 1, m, c, c, 1, ""), (1, 1, m, c, c, 1, "res"), (1, 1, m, c, 3 * c, 1, "qkv"),
                   (1, 1, m, c, 8 * c, 1, "geglu"), (1, 1, m, 4 * c, c, 1, "res")]
        # ResBlocks: 3x3 convs with and without the residual, 1x1 convs (zero convs, proj)
        shapes += [(8, hw, hw, c, c, 3, ""), (8, hw, hw, c, c, 3, "res"), (8, hw, hw, c, c, 1, ""),
                   (8, hw, hw, c, c, 1, "res")]
    # decoder ResBlocks: concatenated skip inputs, second conv with the fused skip projection
    shapes += [(8, 64, 64, 640, 320, 3, ""), (8, 64, 64, 960, 320, 3, ""), (8, 64, 64, 320, 320, 3, "skip640"),
               (8, 64, 64, 320, 320, 3, "skip960"), (8, 32, 32, 960, 640, 3, ""), (8, 32, 32, 1280, 640, 3, ""),
               (8, 32, 32, 1920, 640, 3, ""), (8, 32, 32, 640, 640, 3, "skip960"), (8, 32, 32, 640, 640, 3, "skip1920"),
               (8, 16, 16, 1920, 1280, 3, ""), (8, 16, 16, 2560, 1280, 3, ""), (8, 16, 16, 1280, 1280, 3, "skip2560"),
               (8, 8, 8, 2560, 1280, 3, ""), (8, 8, 8, 1280, 1280, 3, "skip2560")]
    # downsampling-level convs, the input conv and the ControlNet hint / output convs
    shapes += [(8, 32, 32, 320, 640, 3, ""), (8, 16, 16, 640, 1280, 3, ""), (8, 32, 32, 640, 640, 3, "skip320"),
               (8, 16, 16, 1280, 1280, 3, "skip640"), (8, 16, 16, 1280, 1280, 3, "skip1920"),
               (8, 32, 32, 640, 640, 3, "skip1280"), (8, 32, 32, 1280, 1280, 3, ""), (8, 32, 32, 320, 320, 1, ""),
               (8, 16, 16, 640, 640, 1, ""), (8, 64, 64, 8, 320, 3, ""), (8, 64, 64, 320, 16, 3, ""),
               (8, 8, 8, 11520, 1280, 1, ""), (8, 16, 16, 5760, 640, 1, ""), (8, 32, 32, 2880, 320, 1, "")]
    return shapes


@pytest.mark.parametrize("B,H,W,C,N,ks,epi", _step_shapes())
def test_sampling_step_shapes(B, H, W, C, N, ks, epi):
    from ctrlora_b200 import ops
    torch.manual_seed(B * 7 + H + C + N + ks)
    M = B * H * W
    a = _rand(M, C) if H == 1 else _rand(B, H, W, C)
    kk = ks * ks
    if epi == "geglu":
        w = _rand(2 * N, kk, C, s=(kk * C) ** -0.5)
        bias = torch.randn(2 * N, device="cuda")
        out = ops.gemm(a, w, bias=bias, geglu=True)
        y = a.float() @ w.float().view(2 * N, C).t() + bias
        _close(out, y[:, :N] * F.gelu(y[:, N:]))
        return
    w = _rand(N, kk, C, s=(kk * C) ** -0.5)
    if epi == "qkv":
        cq, heads, imgs = N // 3, 8, 8
        T = M // imgs
        q = torch.empty(M, cq, device="cuda", dtype=torch.float16)
        k = torch.empty_like(q)
        vt = torch.zeros(imgs, heads, cq // heads, T, device="cuda", dtype=torch.float16)
        ops.gemm(a, w, seg_outs=[q, k, vt], seg_width=cq, transposed=(0, 0, 1), rows_per_img=T, head_dim=cq // heads,
                 tok_pad=T)
        y = a.float() @ w.float().view(N, C).t()
        _close(q, y[:, :cq])
        _close(k, y[:, cq:2 * cq])
        _close(vt, y[:, 2 * cq:].view(imgs, T, heads, cq // heads).permute(0, 2, 3, 1))
        return
    bias = torch.randn(N, device="cuda")
    ref = (a.float() @ w.float().view(N, C).t() if H == 1 else _conv_ref(a, w, ks).reshape(M, N)) + bias
    kw = {}
    if epi == "res":
        res = _rand(M, N)
        kw["residual"] = res
        ref = ref + res.float()
    elif epi.startswith("skip"):
        c2 = int(epi[4:])
        a2, w2 = _rand(B, H, W, c2), _rand(N, c2, s=c2 ** -0.5)
        kw.update(a2=a2, w2=w2)
        ref = ref + a2.float().reshape(M, c2) @ w2.float().t()
    out = ops.gemm(a, w, ksize=ks, bias=bias, **kw)
    _close(out.reshape(M, N), ref)


def _grids(fn):
    """Grid sizes of the gemm_wgmma_kernel launches of fn(), read from a torch.profiler trace."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
    return [e["args"]["grid"] for e in ev if e.get("cat") == "kernel" and "gemm_wgmma_kernel" in e.get("name", "")]


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_work_units_around_the_sm_budget(delta):
    """Tile counts one below, equal to and one above the SM count (64-column tiles, K = 1280)."""
    from ctrlora_b200 import ops
    torch.manual_seed(40 + delta)
    tiles = _sms() + delta
    M, K, N = 128 * tiles, 1280, 64
    a, w = _rand(M, K), _rand(N, 1, K, s=K ** -0.5)
    bias, res = torch.randn(N, device="cuda"), _rand(M, N)
    for split in (0, 1):
        out = ops.gemm(a, w, bias=bias, residual=res, block_n=64, split_k=split)
        _close(out, a.float() @ w.float().view(N, K).t() + bias + res.float())


def test_sm_limit_bounds_the_grid():
    """Under ctrlora_set_sm_limit(k) the persistent grid has at most k CTAs and the result does not change."""
    from ctrlora_b200 import ops
    torch.manual_seed(41)
    B, H, W, C, N = 8, 32, 32, 640, 640
    a, w = _rand(B, H, W, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
    ref = _conv_ref(a, w, 3)
    full = ops.gemm(a, w, ksize=3)
    assert max(g[0] for g in _grids(lambda: ops.gemm(a, w, ksize=3))) <= _sms()
    for k in (7, 100):
        ops.set_sm_limit(k)
        try:
            grids = _grids(lambda: ops.gemm(a, w, ksize=3))
            out = ops.gemm(a, w, ksize=3)
        finally:
            ops.set_sm_limit(0)
        assert grids and max(g[0] for g in grids) <= k, grids
        _close(out, ref)
        _close(out.float(), full.float())


def test_bn256_geglu_and_fp32_residual():
    from ctrlora_b200 import ops
    torch.manual_seed(42)
    M, K, N = 4096, 320, 1280
    a, w = _rand(M, K), _rand(2 * N, 1, K, s=K ** -0.5)
    bias = torch.randn(2 * N, device="cuda")
    out = ops.gemm(a, w, bias=bias, geglu=True, block_n=128)  # 256-column tile: 128 value + 128 gate columns
    y = a.float() @ w.float().view(2 * N, K).t() + bias
    _close(out, y[:, :N] * F.gelu(y[:, N:]))
    # fp32 residual and fp32 output (the fp32-master LoRA fold), 256-column tiles, with and without a split
    N2 = 768
    w2 = _rand(N2, 1, K, s=K ** -0.5)
    res = torch.randn(M, N2, device="cuda")
    for split in (0, 3):
        out = ops.gemm(a, w2, residual=res, out_f32=True, out_scale=0.25, block_n=256, split_k=split)
        _close(out, (a.float() @ w2.float().view(N2, K).t()) * 0.25 + res, tol=1e-4)


def test_bn256_skip_operand():
    from ctrlora_b200 import ops
    torch.manual_seed(43)
    B, H, W, C, C2, N = 8, 16, 16, 1280, 640, 1280
    a, w = _rand(B, H, W, C), _rand(N, 9, C, s=(9 * C) ** -0.5)
    a2, w2 = _rand(B, H, W, C2), _rand(N, C2, s=C2 ** -0.5)
    bias = torch.randn(N, device="cuda")
    out = ops.gemm(a, w, ksize=3, bias=bias, a2=a2, w2=w2, block_n=256)
    _close(out, _conv_ref(a, w, 3) + bias + a2.float() @ w2.float().t())


@pytest.mark.parametrize("split", [0, 4])
def test_transposed_v_with_dup_out(split):
    from ctrlora_b200 import ops
    torch.manual_seed(44)
    imgs, T, K, cq, heads = 8 if split == 0 else 2, 1024, 640, 640, 8  # a forced split of every tile must fit the workspace
    d = cq // heads
    a, w = _rand(imgs * T, K), _rand(3 * cq, 1, K, s=K ** -0.5)
    q = torch.empty(imgs * T, cq, device="cuda", dtype=torch.float16)
    k = torch.empty_like(q)
    v = torch.empty_like(q)
    vt = torch.zeros(imgs, heads, d, T, device="cuda", dtype=torch.float16)
    ops.gemm(a, w, seg_outs=[q, k, vt], seg_width=cq, transposed=(0, 0, 1), rows_per_img=T, head_dim=d, tok_pad=T,
             dup_out=v, split_k=split)
    y = a.float() @ w.float().view(3 * cq, K).t()
    _close(q, y[:, :cq])
    _close(k, y[:, cq:2 * cq])
    _close(vt, y[:, 2 * cq:].view(imgs, T, heads, d).permute(0, 2, 3, 1))
    _close(v, y[:, 2 * cq:])


@pytest.mark.parametrize("C,ks", [(1280, 3), (2560, 3)])
def test_auto_split_k_on_8x8_convs(C, ks):
    """The model splits the tail of the 8x8 level's long-K convs along K (the workspace is written) and the arrival
    counters are back at zero afterwards."""
    from ctrlora_b200 import ops
    torch.manual_seed(45)
    B, H, W, N = 8, 8, 8, 1280
    a, w = _rand(B, H, W, C), _rand(N, ks * ks, C, s=(ks * ks * C) ** -0.5)
    ws, cnt = ops._splitk_buffers(torch.device("cuda", 0))
    ws.zero_()
    out = ops.gemm(a, w, ksize=ks)
    torch.cuda.synchronize()
    assert ws.abs().max().item() > 0, "no split-K plan was chosen"
    assert cnt.abs().max().item() == 0
    _close(out, _conv_ref(a, w, ks))


@pytest.mark.parametrize("B,H,W,C,N,ks", [(8, 8, 8, 1280, 1280, 3), (8, 64, 64, 320, 320, 3), (8, 16, 16, 1280, 1280, 1)])
def test_bit_reproducible(B, H, W, C, N, ks):
    from ctrlora_b200 import ops
    torch.manual_seed(46)
    a, w = _rand(B, H, W, C), _rand(N, ks * ks, C, s=(ks * ks * C) ** -0.5)
    bias, rb = torch.randn(N, device="cuda"), torch.randn(B, N, device="cuda")
    o1 = ops.gemm(a, w, ksize=ks, bias=bias, rowbias=rb)
    o2 = ops.gemm(a, w, ksize=ks, bias=bias, rowbias=rb)
    assert torch.equal(o1, o2)
