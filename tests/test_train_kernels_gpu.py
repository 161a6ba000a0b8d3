"""GPU parity of the training-only kernels against torch fp32 on the same fp16-rounded operands."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

pytestmark = pytest.mark.gpu


from tolerances import close as _close  # noqa: E402  (max-abs guard AND norm-relative <= 1e-3)


def _rand(*shape, s=1.0):
    return (torch.randn(*shape, device="cuda") * s).half()


@pytest.mark.parametrize("M,P,Q", [(4096, 320, 128), (1000, 128, 320), (16384, 1280, 128), (300, 64, 64), (2048, 640, 640),
                                   (8192, 128, 2560), (77 * 4, 8, 768)])
def test_wgrad_tn(M, P, Q):
    """dW = A^T B over the token dim (LoRA up/down grads, zero-conv grads): MN-major wgmma operands."""
    from ctrlora_b200 import ops
    torch.manual_seed(0)
    a, b = _rand(M, P), _rand(M, Q, s=M ** -0.5)
    out = ops.wgrad_tn(a, b)
    ref = a.float().t() @ b.float()
    _close(out, ref, 1e-3)
    out2 = ops.wgrad_tn(a, b, out=out.clone(), alpha=0.5, beta=2.0)
    _close(out2, 0.5 * ref + 2.0 * out, 1e-3)


import torch.nn.functional as F  # noqa: E402


def _ids(cases, flags):
    """ids of the plain shapes stay the bare shape; the trainer's call forms append their flag names"""
    return ["-".join(str(v) for v in c[:len(c) - len(flags)]) + "".join(f"-{n}" for n, on in zip(flags, c[-len(flags):]) if on)
            for c in cases]


# (B, H, W, C1, C2, silu, res, add1): res = the skip-branch gradient added into d(input) (ResBlock: d_skip, SpatialTransformer:
# d_out); add1 = the mid-control addend on the first half of the first decoder block, with add1_scale and dx1_scale != 1
GN_BWD_CASES = [(2, 16, 16, 320, 0, True, False, False), (2, 8, 8, 64, 32, True, False, False), (3, 16, 16, 640, 0, False, False, False),
                (2, 16, 16, 1280, 640, True, False, False),
                (2, 64, 64, 320, 0, True, True, False),        # ControlNet / encoder ResBlock at 64x64
                (2, 64, 64, 320, 0, False, True, False),       # SpatialTransformer norm: no SiLU, residual gradient
                (2, 16, 16, 1280, 0, False, True, False),
                (2, 8, 8, 1280, 1280, True, True, True),       # decoder block 0: mid control, 2560 wide
                (2, 16, 16, 1280, 1280, True, True, False),    # decoder widths 2560 / 1920 / 960 at their resolutions
                (2, 32, 32, 1280, 640, True, True, False), (2, 32, 32, 640, 320, True, True, False),
                (2, 64, 64, 640, 320, True, True, False)]


@pytest.mark.parametrize("B,H,W,C1,C2,silu,res,add1", GN_BWD_CASES, ids=_ids(GN_BWD_CASES, ["res", "add1"]))
def test_groupnorm_backward(B, H, W, C1, C2, silu, res, add1):
    from ctrlora_b200 import ops
    torch.manual_seed(1)
    C = C1 + C2
    x1 = _rand(B, H, W, C1) + 0.3
    x2 = _rand(B, H, W, C2) if C2 else None
    a2 = _rand(B, H, W, C2) if C2 else None
    a1 = _rand(B, H, W, C1) if add1 else None
    s1, dx1_scale = (1.3, 0.6) if add1 else (1.0, 1.0)
    r = _rand(B, H, W, C) if res else None
    g, b = (1 + 0.2 * torch.randn(C, device="cuda")), 0.2 * torch.randn(C, device="cuda")
    dy = _rand(B, H, W, C)
    y, stats = ops.groupnorm(x1, g, b, 1e-5, silu, add1=a1, add1_scale=s1, x2=x2, add2=a2, add2_scale=0.7, want_stats=True)
    dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    bwd = lambda dgamma, dbeta: ops.groupnorm_bwd(dy, stats, x1, g, b, 1e-5, silu, add1=a1, add1_scale=s1, x2=x2, add2=a2,
                                                  add2_scale=0.7, want_dx2=bool(C2), dx2_scale=0.7, dgamma=dgamma, dbeta=dbeta,
                                                  res=r, dx1_scale=dx1_scale)
    out = bwd(dg, db)
    # the data gradient is bit-reproducible (fixed-order statistics): a rerun of the training step rounds every fp16
    # activation gradient the same way
    again = bwd(None, None)
    assert all(torch.equal(u, v) for u, v in zip(out if C2 else [out], again if C2 else [again]))
    # torch reference
    x1f = x1.float().requires_grad_(True)
    a2f = a2.float().requires_grad_(True) if C2 else None
    gf, bf = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    h1 = x1f + s1 * a1.float() if add1 else x1f
    cat = torch.cat([h1, x2.float() + 0.7 * a2f], -1) if C2 else h1
    z = F.group_norm(cat.permute(0, 3, 1, 2), 32, gf, bf, 1e-5).permute(0, 2, 3, 1)
    loss = ((F.silu(z) if silu else z) * dy.float()).sum()
    if res:
        loss = loss + (cat * r.float()).sum()
    loss.backward()
    if C2:
        _close(out[0], dx1_scale * x1f.grad, 4e-3)
        _close(out[1], a2f.grad, 4e-3)   # d(add2) = scale * d(x2 half)
    else:
        _close(out, dx1_scale * x1f.grad, 4e-3)
    _close(dg, gf.grad, 4e-3)
    _close(db, bf.grad, 4e-3)


# (M, C, res, frozen): the launcher's grid-stride loop first runs above 592 x 8 rows with dgamma and 1184 x 8 without
# (frozen: dgamma = dbeta = None, the UNet decoder's norms); every transformer LayerNorm backward passes `res`
LN_BWD_CASES = [(300, 320, False, False), (4096, 640, False, False), (1000, 1280, False, False), (64, 32, False, False)] + [
    (m, c, True, frozen) for m in (8192, 32768) for c in (320, 640, 1280) for frozen in (False, True)]


@pytest.mark.parametrize("M,C,res,frozen", LN_BWD_CASES, ids=_ids(LN_BWD_CASES, ["res", "frozen"]))
def test_layernorm_backward(M, C, res, frozen):
    from ctrlora_b200 import ops
    torch.manual_seed(2)
    x, dy = _rand(M, C) * 1.5 + 0.2, _rand(M, C)
    r = _rand(M, C) if res else None
    g = 1 + 0.2 * torch.randn(C, device="cuda")
    dg, db = (None, None) if frozen else (torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda"))
    dx = ops.layernorm_bwd(x, dy, g, 1e-5, dg, db, res=r)
    xf, gf = x.float().requires_grad_(True), g.clone().requires_grad_(True)
    bf = torch.zeros(C, device="cuda", requires_grad=True)
    loss = (F.layer_norm(xf, (C,), gf, bf, 1e-5) * dy.float()).sum()
    if res:
        loss = loss + (xf * r.float()).sum()
    loss.backward()
    _close(dx, xf.grad, 4e-3)
    if not frozen:
        _close(dg, gf.grad, 4e-3)
        _close(db, bf.grad, 4e-3)


def test_geglu_forward_backward():
    """500 x 640 and the trainer's feed-forward widths: rows = B * HW at each level, N = 4 * inner"""
    from ctrlora_b200 import ops
    torch.manual_seed(3)
    for M, N in ((500, 640), (8192, 1280), (2048, 2560), (512, 5120), (128, 5120)):
        h, dout = _rand(M, 2 * N), _rand(M, N)
        out = ops.geglu_fwd(h)
        hf = h.float().requires_grad_(True)
        ref = hf[:, :N] * F.gelu(hf[:, N:])
        _close(out, ref, what=f"geglu_fwd {M}x{N}")
        ref.backward(dout.float())
        _close(ops.geglu_bwd(h, dout), hf.grad, 3e-3, what=f"geglu_bwd {M}x{N}")


def test_colsums_and_adjoints():
    from ctrlora_b200 import ops
    torch.manual_seed(4)
    x = _rand(4 * 256, 320)
    out = torch.zeros(320, device="cuda")
    ops.colsum(x, out, 0.5)
    _close(out, 0.5 * x.float().sum(0), 1e-3)
    # the ResBlocks' time-embedding gradients: 256 rows per image, and the trainer's B = 2 at 64x64 ... 8x8 (4096 rows per
    # image is the row-split path with atomics)
    for images, rows, cols in ((4, 256, 320), (2, 4096, 320), (2, 1024, 640), (2, 256, 1280), (2, 64, 1280)):
        x = _rand(images * rows, cols)
        per = torch.zeros(images, cols, device="cuda")
        ops.image_colsum(x, images, per)
        _close(per, x.float().view(images, rows, cols).sum(1), 1e-3, what=f"image_colsum {images}x{rows}x{cols}")
    d = _rand(2, 16, 16, 64)
    up_ref = d.float().view(2, 8, 2, 8, 2, 64).sum(dim=(2, 4))
    _close(ops.upsample2x_bwd(d), up_ref, 2e-3)
    xin = _rand(2, 8, 8, 64)
    dcol = _rand(2, 4, 4, 9 * 64)
    xf = xin.float().requires_grad_(True)
    cols = F.unfold(xf.permute(0, 3, 1, 2), 3, padding=1, stride=2)  # [B, C*9, L] channel-major, tap-minor
    cols = cols.view(2, 64, 9, 16).permute(0, 3, 2, 1).reshape(2, 4, 4, 9 * 64)  # -> tap-major, channel-minor
    cols.backward(dcol.float())
    _close(ops.im2col_s2_bwd(dcol, 8, 8), xf.grad.detach(), 2e-3)


def test_mse_loss_and_adamw():
    from ctrlora_b200 import ops
    torch.manual_seed(5)
    # the default channel padding, and the trainer's call: 16 channels (the out conv's n_pad) with its loss scale
    for B, c_pad, scale in ((4, 8, 1.0), (2, 16, 2 * 4 * 64 * 64 / 16.0)):
        eps = torch.randn(B, 4, 64, 64, device="cuda", requires_grad=True)
        noise = torch.randn(B, 4, 64, 64, device="cuda")
        loss, grad = ops.mse_loss_grad(eps.detach(), noise, c_pad=c_pad, grad_scale=scale)
        ref = ((eps - noise) ** 2).mean(dim=[1, 2, 3]).mean()
        ref.backward()
        assert grad.shape == (B, 64, 64, c_pad)
        assert abs(loss.item() - ref.item()) < 1e-5 * abs(ref.item())
        _close(grad[..., :4], scale * eps.grad.permute(0, 2, 3, 1), 2e-3, what=f"mse grad c_pad {c_pad}")
        assert (grad[..., 4:] == 0).all()
    p = torch.randn(10000, device="cuda")
    p_ref = torch.nn.Parameter(p.clone())
    opt = torch.optim.AdamW([p_ref], lr=1e-2)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for step in range(1, 4):
        g = torch.randn(10000, device="cuda")
        p_ref.grad = g.clone()
        opt.step()
        ops.adamw_step(p, g, m, v, step, lr=1e-2)
    assert (p - p_ref.detach()).abs().max().item() < 1e-5


def _attention_bwd_reference(q, k, v, dout, B, H, Nq, Nk, d):
    """fp32 autograd one (image, head) at a time (bounded memory at 4096 x 4096): base-2 lse [B, H, Nq] and dQ, dK, dV"""
    qv, kv, vv, dv_ = (t.view(B, -1, H, d) for t in (q, k, v, dout))
    lse = torch.empty(B, H, Nq, device="cuda")
    grads = [torch.empty(B, n, H, d, device="cuda") for n in (Nq, Nk, Nk)]
    for b in range(B):
        for h in range(H):
            qf, kf, vf = (t[b, :, h].float().requires_grad_(True) for t in (qv, kv, vv))
            s = (qf @ kf.T) * d ** -0.5
            lse[b, h] = torch.logsumexp(s.detach(), -1) * 1.4426950408889634
            (s.softmax(-1) @ vf).backward(dv_[b, :, h].float())
            for g, t in zip(grads, (qf, kf, vf)):
                g[b, :, h] = t.grad
    return lse, [g.view(-1, H * d) for g in grads]


# (B, H, Nq, Nk, d, strided_out): strided_out = dQ / dK / dV written as column slices of one [B*N, 3*H*d + 8] buffer, as the
# trainer's self-attention backward does; the 8 guard columns past the last slice must keep their sentinel
ATTN_BWD_CASES = [(2, 8, 512, 512, 40, False), (1, 8, 1024, 1024, 80, False), (2, 8, 256, 256, 160, False), (2, 8, 256, 77, 40, False),
                  (2, 4, 200, 300, 16, False), (1, 8, 64, 64, 160, False), (2, 8, 1024, 77, 80, False), (1, 4, 130, 129, 32, False),
                  (1, 8, 600, 700, 40, False), (1, 2, 520, 1000, 24, False), (1, 2, 640, 576, 48, False),  # ragged
                  (2, 8, 4096, 77, 40, False), (2, 8, 256, 77, 160, False), (2, 8, 64, 77, 160, False),    # SD1.5 cross-attention
                  (2, 8, 4096, 4096, 40, True), (2, 8, 1024, 1024, 80, True), (2, 8, 256, 256, 160, True),  # SD1.5 self-attention
                  (2, 8, 64, 64, 160, True), (1, 4, 130, 130, 32, True)]


@pytest.mark.parametrize("B,H,Nq,Nk,d,strided_out", ATTN_BWD_CASES, ids=_ids(ATTN_BWD_CASES, ["strided"]))
def test_attention_backward(B, H, Nq, Nk, d, strided_out):
    """dQ, dK, dV of the fused attention against torch autograd on the same fp16-rounded inputs."""
    from ctrlora_b200 import ops
    torch.manual_seed(6)
    q, k, v = _rand(B * Nq, H * d), _rand(B * Nk, H * d), _rand(B * Nk, H * d)
    dout = _rand(B * Nq, H * d)
    nk_pad = (Nk + 7) // 8 * 8
    vt = torch.zeros(B, H, d, nk_pad, device="cuda", dtype=torch.float16)
    vt[..., :Nk] = v.view(B, Nk, H, d).permute(0, 2, 3, 1)
    lse = torch.empty(B, H, Nq, device="cuda", dtype=torch.float32)
    o = ops.attention(q, k, vt, B, H, Nq, Nk, d, lse=lse)
    c = H * d
    if strided_out:
        buf = torch.full((B * Nq, 3 * c + 8), -1234.0, device="cuda", dtype=torch.float16)
        dq, dk, dv = ops.attention_bwd(q, k, v, o, dout, lse, B, H, Nq, Nk, d, dq=buf[:, :c], dk=buf[:, c:2 * c],
                                       dv=buf[:, 2 * c:3 * c])
        torch.cuda.synchronize()
        assert (buf[:, 3 * c:] == -1234.0).all(), "a store ran past the last slice"
    else:
        dq, dk, dv = ops.attention_bwd(q, k, v, o, dout, lse, B, H, Nq, Nk, d)
    lse_ref, (dq_ref, dk_ref, dv_ref) = _attention_bwd_reference(q, k, v, dout, B, H, Nq, Nk, d)
    _close(lse, lse_ref, 1e-3)
    _close(dq, dq_ref, 5e-3, what="dq")
    _close(dk, dk_ref, 5e-3, what="dk")
    _close(dv, dv_ref, 5e-3, what="dv")
