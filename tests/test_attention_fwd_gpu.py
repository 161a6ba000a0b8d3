"""The warp-specialised, persistent attention forward (ctrlora_attention_f16): every distinct attention launch of the
batch-8 sampling step at full size, the edges of the query work unit (64 rows per consumer warpgroup; later warpgroups
empty or partial), work-unit counts around the SM count, partial last key tiles, reproducibility and CUDA-graph replay.

References are torch fp32 on the same fp16-rounded operands, computed one (image, head) at a time to bound memory; the
output is compared with tolerances.close, the saved base-2 log-sum-exp with the bound test_kernels_gpu.py uses.
"""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

pytestmark = pytest.mark.gpu

from tolerances import close as _close  # noqa: E402

LOG2E = 1.4426950408889634


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(B, H, Nq, Nk, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mk = lambda *s: torch.randn(*s, device="cuda", generator=g).half()
    q, k, v = mk(B * Nq, H * d), mk(B * Nk, H * d), mk(B * Nk, H * d)
    nk_pad = (Nk + 7) // 8 * 8
    vt = torch.zeros(B, H, d, nk_pad, device="cuda", dtype=torch.float16)
    vt[..., :Nk] = v.view(B, Nk, H, d).permute(0, 2, 3, 1)
    return q, k, v, vt


def _reference(q, k, v, B, H, Nq, Nk, d):
    """fp32 output [B * Nq, H * d] and base-2 log-sum-exp [B, H, Nq], one (image, head) at a time."""
    qv, kv, vv = q.view(B, Nq, H, d), k.view(B, Nk, H, d), v.view(B, Nk, H, d)
    out = torch.empty(B, Nq, H, d, device="cuda")
    lse = torch.empty(B, H, Nq, device="cuda")
    for b in range(B):
        for h in range(H):
            s = (qv[b, :, h].float() @ kv[b, :, h].float().T) * d ** -0.5
            out[b, :, h] = s.softmax(-1) @ vv[b, :, h].float()
            lse[b, h] = torch.logsumexp(s, -1) * LOG2E
    return out.view(B * Nq, H * d), lse


def _check(B, H, Nq, Nk, d, seed=0):
    from ctrlora_b200 import ops
    q, k, v, vt = _inputs(B, H, Nq, Nk, d, seed)
    lse = torch.empty(B, H, Nq, device="cuda", dtype=torch.float32)
    out = ops.attention(q, k, vt, B, H, Nq, Nk, d, lse=lse)
    ref, ref_lse = _reference(q, k, v, B, H, Nq, Nk, d)
    _close(out, ref, 3e-3, what=f"out {B}x{H}x{Nq}x{Nk} d{d}")
    assert (lse - ref_lse).abs().max().item() < 2e-3 * max(1.0, ref_lse.abs().max().item())


# self-attention at the 64 / 32 / 16 / 8 levels of the CFG batch, and cross-attention to the 77 context tokens
@pytest.mark.parametrize("Nq,Nk,d", [(4096, 4096, 40), (1024, 1024, 80), (256, 256, 160), (64, 64, 160),
                                     (4096, 77, 40), (1024, 77, 80), (256, 77, 160), (64, 77, 160)])
def test_step_launches_full_size(Nq, Nk, d):
    _check(8, 8, Nq, Nk, d, seed=Nq + Nk + d)


# work units of 192 query rows at d = 40 (three consumer warpgroups) and 128 at d = 80 / 160 (two): Nq = 64 leaves every
# warpgroup but the first without rows, 65 / 130 / 200 give a warpgroup a partial tile or no rows
@pytest.mark.parametrize("Nq", [64, 65, 130, 200])
@pytest.mark.parametrize("d", [40, 80, 160])
def test_partial_query_units(Nq, d):
    _check(2, 3, Nq, 300, d, seed=Nq * d)


# one work unit per (image, head): CTAs = units below, at and just above the SM count (then 2 units on some CTAs)
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_units_around_sm_count(delta):
    _check(_sms() + delta, 1, 128, 200, 40, seed=delta + 5)


# partial last 64-key tile, including a single tile shorter than 64 keys
@pytest.mark.parametrize("Nk", [1, 7, 63, 65, 127, 200])
@pytest.mark.parametrize("d", [8, 40, 80, 160])
def test_partial_key_tiles(Nk, d):
    _check(2, 2, 150, Nk, d, seed=Nk + d)


def test_sm_limit_many_units_per_cta():
    """A small SM budget makes every CTA walk many units; the ring and Q buffer carry across them."""
    from ctrlora_b200 import ops
    ops.set_sm_limit(5)
    try:
        _check(3, 4, 500, 700, 40, seed=9)
    finally:
        ops.set_sm_limit(0)


def test_repeated_calls_bit_identical():
    from ctrlora_b200 import ops
    B, H, Nq, Nk, d = 8, 8, 1024, 1024, 40
    q, k, _, vt = _inputs(B, H, Nq, Nk, d, 3)
    lse0 = torch.empty(B, H, Nq, device="cuda")
    out0 = ops.attention(q, k, vt, B, H, Nq, Nk, d, lse=lse0)
    for _ in range(3):
        lse = torch.empty_like(lse0)
        out = ops.attention(q, k, vt, B, H, Nq, Nk, d, lse=lse)
        assert torch.equal(out, out0) and torch.equal(lse, lse0)


def test_cuda_graph_replay_matches_eager():
    from ctrlora_b200 import ops
    B, H, Nq, Nk, d = 8, 8, 1024, 77, 80
    q, k, _, vt = _inputs(B, H, Nq, Nk, d, 4)
    eager = ops.attention(q, k, vt, B, H, Nq, Nk, d)
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.attention(q, k, vt, B, H, Nq, Nk, d, out=out)  # warm-up outside capture (function attributes)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.attention(q, k, vt, B, H, Nq, Nk, d, out=out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
