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


@pytest.mark.parametrize("B,H,W,C1,C2,silu", [(2, 16, 16, 320, 0, True), (2, 8, 8, 64, 32, True), (3, 16, 16, 640, 0, False),
                                              (2, 16, 16, 1280, 640, True)])
def test_groupnorm_backward(B, H, W, C1, C2, silu):
    from ctrlora_b200 import ops
    torch.manual_seed(1)
    C = C1 + C2
    x1 = _rand(B, H, W, C1) + 0.3
    x2 = _rand(B, H, W, C2) if C2 else None
    a2 = _rand(B, H, W, C2) if C2 else None
    g, b = (1 + 0.2 * torch.randn(C, device="cuda")), 0.2 * torch.randn(C, device="cuda")
    dy = _rand(B, H, W, C)
    y, stats = ops.groupnorm(x1, g, b, 1e-5, silu, x2=x2, add2=a2, add2_scale=0.7, want_stats=True)
    dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    res = ops.groupnorm_bwd(dy, stats, x1, g, b, 1e-5, silu, x2=x2, add2=a2, add2_scale=0.7, want_dx2=bool(C2), dx2_scale=0.7,
                            dgamma=dg, dbeta=db)
    # torch reference
    x1f = x1.float().requires_grad_(True)
    a2f = a2.float().requires_grad_(True) if C2 else None
    gf, bf = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    cat = torch.cat([x1f, x2.float() + 0.7 * a2f], -1) if C2 else x1f
    z = F.group_norm(cat.permute(0, 3, 1, 2), 32, gf, bf, 1e-5).permute(0, 2, 3, 1)
    out = F.silu(z) if silu else z
    out.backward(dy.float())
    if C2:
        _close(res[0], x1f.grad, 4e-3)
        _close(res[1], a2f.grad, 4e-3)   # d(add2) = scale * d(x2 half)
    else:
        _close(res, x1f.grad, 4e-3)
    _close(dg, gf.grad, 4e-3)
    _close(db, bf.grad, 4e-3)


@pytest.mark.parametrize("M,C", [(300, 320), (4096, 640), (1000, 1280), (64, 32)])
def test_layernorm_backward(M, C):
    from ctrlora_b200 import ops
    torch.manual_seed(2)
    x, dy = _rand(M, C) * 1.5 + 0.2, _rand(M, C)
    g = 1 + 0.2 * torch.randn(C, device="cuda")
    dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    dx = ops.layernorm_bwd(x, dy, g, 1e-5, dg, db)
    xf, gf = x.float().requires_grad_(True), g.clone().requires_grad_(True)
    bf = torch.zeros(C, device="cuda", requires_grad=True)
    F.layer_norm(xf, (C,), gf, bf, 1e-5).backward(dy.float())
    _close(dx, xf.grad, 4e-3)
    _close(dg, gf.grad, 4e-3)
    _close(db, bf.grad, 4e-3)


def test_geglu_forward_backward():
    from ctrlora_b200 import ops
    torch.manual_seed(3)
    M, N = 500, 640
    h, dout = _rand(M, 2 * N), _rand(M, N)
    out = ops.geglu_fwd(h)
    hf = h.float().requires_grad_(True)
    ref = hf[:, :N] * F.gelu(hf[:, N:])
    _close(out, ref)
    ref.backward(dout.float())
    _close(ops.geglu_bwd(h, dout), hf.grad, 3e-3)


def test_colsums_and_adjoints():
    from ctrlora_b200 import ops
    torch.manual_seed(4)
    x = _rand(4 * 256, 320)
    out = torch.zeros(320, device="cuda")
    ops.colsum(x, out, 0.5)
    _close(out, 0.5 * x.float().sum(0), 1e-3)
    per = torch.zeros(4, 320, device="cuda")
    ops.image_colsum(x, 4, per)
    _close(per, x.float().view(4, 256, 320).sum(1), 1e-3)
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
    eps = torch.randn(4, 4, 64, 64, device="cuda", requires_grad=True)
    noise = torch.randn(4, 4, 64, 64, device="cuda")
    loss, grad = ops.mse_loss_grad(eps.detach(), noise)
    ref = ((eps - noise) ** 2).mean(dim=[1, 2, 3]).mean()
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5 * abs(ref.item())
    _close(grad[..., :4], eps.grad.permute(0, 2, 3, 1), 2e-3)
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


@pytest.mark.parametrize("B,H,Nq,Nk,d", [(2, 8, 512, 512, 40), (1, 8, 1024, 1024, 80), (2, 8, 256, 256, 160), (2, 8, 256, 77, 40),
                                         (2, 4, 200, 300, 16), (1, 8, 64, 64, 160), (2, 8, 1024, 77, 80), (1, 4, 130, 129, 32),
                                         (1, 8, 600, 700, 40), (1, 2, 520, 1000, 24), (1, 2, 640, 576, 48)])  # ragged
def test_attention_backward(B, H, Nq, Nk, d):
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
    dq, dk, dv = ops.attention_bwd(q, k, v, o, dout, lse, B, H, Nq, Nk, d)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    qh = qf.view(B, Nq, H, d).permute(0, 2, 1, 3)
    kh = kf.view(B, Nk, H, d).permute(0, 2, 1, 3)
    vh = vf.view(B, Nk, H, d).permute(0, 2, 1, 3)
    sim = (qh @ kh.transpose(-1, -2)) * d ** -0.5
    ref = (sim.softmax(-1) @ vh).permute(0, 2, 1, 3).reshape(B * Nq, H * d)
    lse_ref = torch.logsumexp(sim, -1) * 1.4426950408889634
    _close(lse, lse_ref, 1e-3)
    ref.backward(dout.float())
    _close(dq, qf.grad, 5e-3)
    _close(dk, kf.grad, 5e-3)
    _close(dv, vf.grad, 5e-3)
