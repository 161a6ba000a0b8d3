"""GroupNorm forward and backward at the widest channel count the entry points accept (C = 4096: one pixel lane of 512
threads per block, 64 KB of dynamic shared memory in the statistics kernels).  At 64x64 one image's slice does not fit
8 CTAs of the cluster kernel, so both directions run the two-pass pair."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pytestmark = pytest.mark.gpu

from tolerances import close  # noqa: E402


def test_groupnorm_two_pass_at_4096_channels():
    from ctrlora_b200 import ops
    torch.manual_seed(11)
    B, H, C = 1, 64, 4096
    x = (torch.randn(B, H, H, C, device="cuda") + 0.3).half()
    g, b = 1 + 0.2 * torch.randn(C, device="cuda"), 0.2 * torch.randn(C, device="cuda")
    dy = torch.randn(B, H, H, C, device="cuda").half()
    # forward: same values as torch, bit-identical between calls, statistics buffer = {sum, sumsq}
    y1, st1 = ops.groupnorm(x, g, b, 1e-5, True, want_stats=True)
    y2, st2 = ops.groupnorm(x, g, b, 1e-5, True, want_stats=True)
    assert torch.equal(y1, y2) and torch.equal(st1, st2)
    xf = x.float().requires_grad_(True)
    gf, bf = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    z = F.group_norm(xf.permute(0, 3, 1, 2), 32, gf, bf, 1e-5).permute(0, 2, 3, 1)
    close(y1, F.silu(z), tol=4e-3, what="groupnorm")
    sums = x.float().view(B, H * H, 32, C // 32).sum(dim=(1, 3))
    close(st1.view(B, 32, 2)[..., 0], sums, tol=2e-3, nrel=1e-4, what="gn stats")
    # backward: against autograd, dx bit-identical between calls
    dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    dx1 = ops.groupnorm_bwd(dy, st1, x, g, b, 1e-5, True, dgamma=dg, dbeta=db)
    dx2 = ops.groupnorm_bwd(dy, st1, x, g, b, 1e-5, True)
    assert torch.equal(dx1, dx2)
    (F.silu(z) * dy.float()).sum().backward()
    close(dx1, xf.grad, 4e-3, what="dx")
    close(dg, gf.grad, 4e-3, what="dgamma")
    close(db, bf.grad, 4e-3, what="dbeta")
