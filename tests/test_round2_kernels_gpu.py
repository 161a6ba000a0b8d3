"""GPU parity of the round-2 C-ABI entry points against torch fp32 references on the same inputs (bit-exact where the
arithmetic is integer / gather / separately-rounded fp32 products; norm-relative <= 1e-3 for fp16 outputs)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pytestmark = pytest.mark.gpu

from tolerances import close  # noqa: E402


def test_q_sample_and_ddim_encode_bit_exact():
    from ctrlora_b200 import ops
    torch.manual_seed(0)
    B = 5
    x0, noise = torch.randn(B, 4, 16, 16, device="cuda"), torch.randn(B, 4, 16, 16, device="cuda")
    tab_a, tab_s = torch.rand(1000, device="cuda"), torch.rand(1000, device="cuda")
    t = torch.tensor([0, 999, 21, 500, 981], device="cuda")
    got = ops.q_sample(x0, noise, t, tab_a, tab_s)
    ref = tab_a[t].view(-1, 1, 1, 1) * x0 + tab_s[t].view(-1, 1, 1, 1) * noise   # ldm/models/diffusion/ddpm.py:356-359
    assert torch.equal(got, ref)
    e_c, e_u = torch.randn_like(x0), torch.randn_like(x0)
    c1, c2 = torch.tensor(1.01234567), torch.tensor(-0.0456789)
    got = ops.ddim_encode_update(x0, e_c, e_u, 3.0, float(c1), float(c2))
    e = e_u + 3.0 * (e_c - e_u)                                                    # cldm/ddim_hacked.py:253-267
    assert torch.equal(got, c1.cuda() * x0 + c2.cuda() * e)
    assert torch.equal(ops.ddim_encode_update(x0, e_c, None, 1.0, float(c1), float(c2)), c1.cuda() * x0 + c2.cuda() * e_c)


def test_weighted_sum_and_memset():
    from ctrlora_b200 import ops
    torch.manual_seed(1)
    ts = [(torch.randn(2, 8, 8, 64, device="cuda")).half().permute(0, 3, 1, 2) for _ in range(3)]  # channels_last views
    w = [0.7, 0.3, -1.25]
    got = ops.weighted_sum(ts, w)
    assert got.stride() == ts[0].stride()
    close(got, sum(wi * t.float() for wi, t in zip(w, ts)), what="weighted_sum")
    z = ops.zeros((3, 5, 7), torch.device("cuda"))
    assert z.dtype == torch.float16 and float(z.abs().sum()) == 0.0


@pytest.mark.parametrize("rows,cols,scale", [(64, 256, 0.125), (300, 4096, 512 ** -0.5), (7, 1000, 1.0)])
def test_softmax_rows(rows, cols, scale):
    from ctrlora_b200 import ops
    torch.manual_seed(2)
    x = torch.randn(rows, cols, device="cuda") * 6
    close(ops.softmax_rows(x, scale), torch.softmax(x * scale, dim=-1), what="softmax_rows")


def test_im2col_gathers_bit_exact():
    from ctrlora_b200 import ops
    torch.manual_seed(3)
    x = torch.randn(2, 6, 8, 16, device="cuda").half()
    nchw = x.permute(0, 3, 1, 2).float()
    col = ops.im2col_3x3(x)                                                        # [B,H,W,9*C], tap-major
    ref = F.unfold(nchw, 3, padding=1).view(2, 16, 9, 6, 8).permute(0, 3, 4, 2, 1).reshape(2, 6, 8, 144)
    assert torch.equal(col.float(), ref)
    for pad_lo, padding in ((1, (1, 1, 1, 1)), (0, (0, 1, 0, 1))):                 # Conv2d(pad 1) vs the VAE's F.pad(0,1,0,1)
        col = ops.im2col_s2(x, pad_lo=pad_lo)
        ref = F.unfold(F.pad(nchw, padding), 3, stride=2).view(2, 16, 9, 3, 4).permute(0, 3, 4, 2, 1).reshape(2, 3, 4, 144)
        assert torch.equal(col.float(), ref), pad_lo


def test_small_mlp_backward_kernels():
    from ctrlora_b200 import ops
    torch.manual_seed(4)
    B, N, K = 6, 40, 72
    dy, x = torch.randn(B, N, device="cuda"), torch.randn(B, K, device="cuda")
    out = torch.randn(N, K, device="cuda")
    ref = 0.5 * out + 2.0 * dy.t() @ F.silu(x)
    ops.outer_accum(dy, x, out, alpha=2.0, beta=0.5, silu_x=True)
    close(out, ref, tol=1e-5, nrel=1e-6, what="outer_accum")
    xs = x.clone().requires_grad_(True)
    F.silu(xs).backward(dy[:, :K] if N >= K else torch.ones_like(xs))
    d = dy[:, :K] if N >= K else torch.ones_like(x)
    close(ops.silu_bwd(d.contiguous(), x), xs.grad, tol=1e-5, nrel=2e-6, what="silu_bwd")
    src = torch.randn(9, 8, device="cuda")
    dst = torch.zeros(9, 4, device="cuda")
    ops.copy2d(src, dst, 9, 4, 8, 4)
    ops.copy2d(src, dst, 9, 4, 8, 4, accumulate=True)
    assert torch.equal(dst, 2 * src[:, :4])


@pytest.mark.parametrize("rows,n,k,silu_in,silu_out", [(8, 1280, 320, False, True), (8, 1280, 1280, False, False),
                                                       (8, 20160, 1280, True, False), (16, 9600, 1280, True, False),
                                                       (2, 8, 128, True, False), (3, 100, 32, False, False), (16, 1280, 9600, False, False)])
def test_small_linear_shapes(rows, n, k, silu_in, silu_out):
    """time_embed (N = 1280), the batched emb_layers GEMV (N = 20 160 / 9 600), LoRA-rank-sized outputs and the long-K
    backward form (falls through to the unstaged kernel)."""
    from ctrlora_b200 import ops
    torch.manual_seed(5)
    x = torch.randn(rows, k, device="cuda")
    w = (torch.randn(n, k, device="cuda") * k ** -0.5).half()
    b = torch.randn(n, device="cuda")
    got = ops.small_linear(x, w, b, silu_in=silu_in, silu_out=silu_out)
    ref = F.linear(F.silu(x) if silu_in else x, w.float(), b)
    close(got, F.silu(ref) if silu_out else ref, tol=2e-4, nrel=5e-5, what="small_linear")


def test_gaussian_sample_and_adamw_step_counter():
    from ctrlora_b200 import ops
    torch.manual_seed(6)
    mom = torch.randn(2, 8, 4, 4, device="cuda") * 3
    mom[:, 4:] *= 10                                         # exercises the clamp(-30, 20) of the log-variance
    noise = torch.randn(2, 4, 4, 4, device="cuda")
    mean, logvar = mom[:, :4], mom[:, 4:].clamp(-30.0, 20.0)
    close(ops.gaussian_sample(mom, noise, 0.18215), 0.18215 * (mean + torch.exp(0.5 * logvar) * noise), tol=1e-5, nrel=1e-6)
    assert torch.equal(ops.gaussian_sample(mom, None, 0.18215), 0.18215 * mean)
    # device-side step bookkeeping: skipped steps do not advance AdamW's step (torch per-parameter `step` semantics)
    n = 1000
    p, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    pr = torch.nn.Parameter(p.clone())
    opt = torch.optim.AdamW([pr], lr=1e-2)
    step, bc = torch.zeros(1, device="cuda", dtype=torch.int32), torch.ones(2, device="cuda")
    flag, skipped = torch.zeros(1, device="cuda", dtype=torch.int32), torch.zeros(1, device="cuda", dtype=torch.int32)
    for it in range(4):
        flag.fill_(1 if it == 1 else 0)                      # the second step overflows
        gi = g * (it + 1)
        ops.adamw_begin(step, flag, (0.9, 0.999), bc, skipped)
        ops.adamw_step(p, gi, m, v, 0, lr=1e-2, skip_flag=flag, bc_dev=bc)
        if it != 1:
            pr.grad = gi.clone()
            opt.step()
    assert int(step.item()) == 3 and int(skipped.item()) == 1
    assert (p - pr.detach()).abs().max().item() < 1e-6
    bad = torch.zeros(1, device="cuda", dtype=torch.int32)
    ops.nonfinite_flag(torch.tensor([1.0, float("inf"), 2.0, 3.0, 4.0], device="cuda"), bad)
    assert int(bad.item()) == 1


@pytest.mark.parametrize("B,H,C,C2,silu", [(2, 8, 1280, 0, True), (3, 16, 1280, 0, True), (2, 32, 640, 0, False), (2, 64, 320, 0, True),
                                           (2, 16, 1280, 1280, True), (2, 64, 640, 320, True), (2, 2, 128, 128, True)])
def test_groupnorm_paths_are_deterministic_and_agree(B, H, C, C2, silu):
    """cluster kernel (bulk-staged / gathered) for slices that fit <= 8 CTAs, deterministic two-pass otherwise: same values as
    torch, bit-identical between calls, statistics buffer = {sum, sumsq} as the backward expects."""
    from ctrlora_b200 import ops
    torch.manual_seed(7)
    x1 = (torch.randn(B, H, H, C, device="cuda") + 0.3).half()
    x2 = (torch.randn(B, H, H, C2, device="cuda")).half() if C2 else None
    add2 = (torch.randn(B, H, H, C2, device="cuda")).half() if C2 else None
    g, b = torch.randn(C + C2, device="cuda"), torch.randn(C + C2, device="cuda")
    kw = dict(x2=x2, add2=add2, add2_scale=0.7) if C2 else {}
    y1, st1 = ops.groupnorm(x1, g, b, 1e-5, silu, want_stats=True, **kw)
    y2, st2 = ops.groupnorm(x1, g, b, 1e-5, silu, want_stats=True, **kw)
    assert torch.equal(y1, y2) and torch.equal(st1, st2)
    cat = x1.float() if not C2 else torch.cat([x1.float(), x2.float() + 0.7 * add2.float()], -1)
    ref = F.group_norm(cat.permute(0, 3, 1, 2), 32, g, b, 1e-5)
    ref = (F.silu(ref) if silu else ref).permute(0, 2, 3, 1)
    close(y1, ref, tol=4e-3, what="groupnorm")
    cpg = (C + C2) // 32
    sums = cat.view(B, H * H, 32, cpg).sum(dim=(1, 3))
    close(st1.view(B, 32, 2)[..., 0], sums, tol=2e-3, nrel=1e-4, what="gn stats")


@pytest.mark.gpu
@pytest.mark.parametrize("m,p,q,ldo_extra,alpha,beta", [
    (4096, 1280, 4096, 0, 1.0, 0.0),      # 160 tiles: one split, the epilogue writes the result itself
    (2048, 1280, 11520, 64, 0.5, 1.0),    # a dense 3x3 conv gradient of the 1280-wide stage, accumulated into a strided view
    (32768, 320, 2880, 0, 1.0, 1.0),      # few tiles: token splits + the tiled reduce kernel
    (8192, 136, 328, 8, 2.0, 1.0),        # ragged tile edges (P, Q multiples of 8 only)
])
def test_wgrad_direct_and_reduce_paths(m, p, q, ldo_extra, alpha, beta):
    """dense weight gradients of pretraining (reference: autograd of every ControlNet weight,
    cldm/cldm_ctrlora_pretrain.py:88-96): out = alpha * a^T b + beta * out, fp32 accumulate"""
    from ctrlora_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(m + p)
    a = (torch.randn(m, p, device="cuda", generator=g) * 0.5).half()
    b = (torch.randn(m, q, device="cuda", generator=g) * 0.5).half()
    buf = torch.randn(p, q + ldo_extra, device="cuda", generator=g)
    out = buf[:, :q]
    ref = alpha * (a.double().t() @ b.double()) + beta * out.double()
    keep = buf[:, q:].clone()
    ops.wgrad_tn(a, b, out=out, alpha=alpha, beta=beta)
    torch.cuda.synchronize()
    assert torch.equal(buf[:, q:], keep), "wrote outside the output view"
    err = ((out.double() - ref).norm() / ref.norm()).item()
    assert err < 3e-5, err  # fp32 tensor-core accumulation over up to 32768 tokens (measured <= 7.8e-6)


COLSUM_CASES = [(32768, 320, 320, torch.float16), (2048, 1280, 1280, torch.float16), (8192, 640, 1920, torch.float16),
                (77, 328, 328, torch.float16), (512, 8, 8, torch.float16),
                # fp32 input: the time-embedding MLP's bias gradients (rows = batch; emb_layers read a column slice of the
                # [B, 9600] d(rowbias) buffer), and a tall / ragged form of the same instance
                (2, 1280, 1280, torch.float32), (2, 320, 9600, torch.float32), (4096, 1280, 1280, torch.float32),
                (77, 1000, 1003, torch.float32)]


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,ld,dtype", COLSUM_CASES,
                         ids=[f"{r}-{c}-{ld}" + ("-fp32" if dt == torch.float32 else "") for r, c, ld, dt in COLSUM_CASES])
def test_colsum_vector_path(rows, cols, ld, dtype):
    from ctrlora_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(rows)
    x = torch.randn(rows, ld, device="cuda", generator=g).to(dtype)[:, :cols]
    out = torch.ones(cols, device="cuda")
    ops.colsum(x, out, scale=0.25)
    ref = 1.0 + 0.25 * x.double().sum(0)
    close(out, ref, tol=1e-5, nrel=1e-5, what="colsum")


@pytest.mark.gpu
@pytest.mark.parametrize("cout,taps,cin", [(320, 9, 320), (1280, 9, 640), (320, 9, 8), (640, 1, 320), (72, 9, 136)])
def test_conv_dgrad_weight_and_tiled_transpose_bit_exact(cout, taps, cin):
    from ctrlora_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(cout + cin)
    w = torch.randn(cout, taps, cin, device="cuda", generator=g).half()
    assert torch.equal(ops.conv_dgrad_weight(w), w.flip(1).permute(2, 1, 0).contiguous())
    w2 = w.view(1, cout, taps * cin)
    assert torch.equal(ops.transpose_f16(w2, 1, cout, taps * cin), w2.transpose(1, 2).contiguous())
    b3 = torch.randn(3, 66, 130, device="cuda", generator=g).half()
    assert torch.equal(ops.transpose_f16(b3, 3, 66, 130), b3.transpose(1, 2).contiguous())


@pytest.mark.gpu
@pytest.mark.parametrize("batch,rows,cols", [(1, 128, 1280), (320, 320, 9), (1, 1, 4096), (4099, 1, 1), (2, 66, 130), (1, 4, 77), (3, 5, 7)])
def test_cast_transpose_paths_bit_exact(batch, rows, cols):
    """fp32 master weight -> fp16 kernel layout (plain cast, tiled transpose, ragged fallback) == torch's rounding"""
    from ctrlora_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(rows * cols)
    src = torch.randn(batch, rows, cols, device="cuda", generator=g)
    got = ops.cast_transpose(src, batch, rows, cols).view(batch, cols, rows)
    assert torch.equal(got, src.transpose(1, 2).contiguous().half())
