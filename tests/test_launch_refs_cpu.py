"""The per-call references of tests/launch_refs.py pinned at tiny shapes on the host, so that a wrong reference is not
mistaken for a wrong kernel: the 3x3 conv against a loop over its taps, the V^T segment layout and its row-major copy,
grouped calls against two plain calls on the halves, the row-term indexing, and every backward against central finite
differences of the forward reference in fp64."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import launch_refs as R  # noqa: E402


def _r(*shape, seed=0, dtype=torch.float32):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=dtype)


def _fd_grad(f, x, h=1e-6):
    """d f / d x by central differences (f: fp64 tensor -> fp64 scalar)"""
    g = torch.zeros_like(x)
    flat, gf = x.view(-1), g.view(-1)
    for i in range(flat.numel()):
        old = flat[i].item()
        flat[i] = old + h
        up = f(x).item()
        flat[i] = old - h
        dn = f(x).item()
        flat[i] = old
        gf[i] = (up - dn) / (2 * h)
    return g


def test_conv3x3_is_a_loop_over_taps():
    """tap t = 3 dy + dx reads pixel (y + dy - 1, x + dx - 1), zero outside; then bias, row term, scale, residual"""
    B, H, W, C, N = 2, 5, 6, 3, 4
    a, w = _r(B, H, W, C, seed=1), _r(N, 9, C, seed=2)
    bias, rb, res = _r(N, seed=3), _r(B, N, seed=4), _r(B, H, W, N, seed=5)
    got = R.gemm(a, w, ksize=3, bias=bias, rowbias=rb, residual=res, out_scale=0.5)
    ap = F.pad(a, (0, 0, 1, 1, 1, 1))
    ref = torch.zeros(B, H, W, N)
    for t in range(9):
        dy, dx = divmod(t, 3)
        ref += ap[:, dy:dy + H, dx:dx + W, :] @ w[:, t, :].t()
    ref = (ref + bias + rb.view(B, 1, 1, N)) * 0.5 + res
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5)


def test_skip_operand_geglu_and_fp16_inputs():
    M, K, K2, N = 10, 8, 5, 6
    a, a2 = _r(M, K, seed=1).half(), _r(M, K2, seed=2).half()
    w, w2, bias = _r(2 * N, K, seed=3).half(), _r(2 * N, K2, seed=4).half(), _r(2 * N, seed=5)
    y = a.float() @ w.float().t() + a2.float() @ w2.float().t() + bias
    ref = y[:, :N] * 0.5 * y[:, N:] * (1 + torch.erf(y[:, N:] / 2 ** 0.5))
    torch.testing.assert_close(R.gemm(a, w, bias=bias, a2=a2, w2=w2, geglu=True), ref, rtol=1e-5, atol=1e-5)


def test_transposed_segment_and_dup_out_round_trip():
    """q | k | V^T: V^T holds [image, head, d, token] with the padding tokens zero; dup_out is V row-major"""
    imgs, T, tok_pad, heads, d = 3, 5, 8, 2, 4
    c = heads * d
    a, w = _r(imgs * T, 6, seed=1), _r(3 * c, 6, seed=2)
    q, k = torch.empty(imgs * T, c), torch.empty(imgs * T, c)
    vt, v = torch.empty(imgs, heads, d, tok_pad), torch.empty(imgs * T, c)
    got = R.gemm(a, w, seg_outs=[q, k, vt], seg_width=c, transposed=(0, 0, 1), rows_per_img=T, head_dim=d,
                 tok_pad=tok_pad, dup_out=v)
    plain = R.gemm(a, w)
    assert len(got) == 4
    torch.testing.assert_close(got[0], plain[:, :c])
    torch.testing.assert_close(got[1], plain[:, c:2 * c])
    torch.testing.assert_close(got[3], plain[:, 2 * c:])
    for i in range(imgs):
        for h in range(heads):
            for tok in range(T):
                torch.testing.assert_close(got[2][i, h, :, tok], plain[i * T + tok, 2 * c + h * d:2 * c + (h + 1) * d])
    assert (got[2][..., T:] == 0).all()
    # K | V^T of a context (the transposed segment second, no copy)
    kk, vv = R.gemm(a, w[:2 * c], seg_outs=[k, vt], seg_width=c, transposed=(0, 1, 0), rows_per_img=T, head_dim=d,
                    tok_pad=tok_pad)
    torch.testing.assert_close(kk, plain[:, :c])
    torch.testing.assert_close(vv[..., :T], plain[:, c:2 * c].reshape(imgs, T, heads, d).permute(0, 2, 3, 1))


def test_grouped_conv_is_two_plain_calls():
    """4-D operand: images of the upper half take hi's weights, bias, skip weights and row terms (indexed from the
    half's first image); the residual and the skip operand are cut by image"""
    b, H, C, N = 2, 4, 3, 5
    a, a2, res = _r(2 * b, H, H, C, seed=1), _r(2 * b, H, H, 2, seed=2), _r(2 * b, H, H, N, seed=3)
    wl, wh, w2l, w2h = _r(N, 9, C, seed=4), _r(N, 9, C, seed=5), _r(N, 2, seed=6), _r(N, 2, seed=7)
    bl, bh = _r(N, seed=8), _r(N, seed=9)
    rbuf = _r(2 * b, 3 * N, seed=10)  # both halves' row terms: column slices of one wider buffer, one row stride
    rl, rh = rbuf[:b, :N], rbuf[b:, N:2 * N]
    g = R.gemm(a, wl, ksize=3, bias=bl, rowbias=rl, residual=res, a2=a2, w2=w2l, out_scale=0.75,
               hi={"w": wh, "bias": bh, "rowbias": rh, "w2": w2h})
    lo = R.gemm(a[:b], wl, ksize=3, bias=bl, rowbias=rl, residual=res[:b], a2=a2[:b], w2=w2l, out_scale=0.75)
    up = R.gemm(a[b:], wh, ksize=3, bias=bh, rowbias=rh, residual=res[b:], a2=a2[b:], w2=w2h, out_scale=0.75)
    torch.testing.assert_close(g, torch.cat([lo, up]))
    assert not torch.allclose(g[b:], R.gemm(a[b:], wh, ksize=3, bias=bl, rowbias=rh, residual=res[b:], a2=a2[b:],
                                            w2=w2h, out_scale=0.75))


def test_grouped_linear_is_two_plain_calls():
    """2-D operand: the halves are row halves -- GEGLU, and q | k | V^T with the images of each half"""
    T, c = 4, 6
    x = _r(4 * T, 5, seed=1)
    w1l, w1h, b1l, b1h = _r(2 * c, 5, seed=2), _r(2 * c, 5, seed=3), _r(2 * c, seed=4), _r(2 * c, seed=5)
    g = R.gemm(x, w1l, bias=b1l, geglu=True, hi={"w": w1h, "bias": b1h})
    torch.testing.assert_close(g, torch.cat([R.gemm(x[:2 * T], w1l, bias=b1l, geglu=True),
                                             R.gemm(x[2 * T:], w1h, bias=b1h, geglu=True)]))
    wl, wh = _r(3 * c, 5, seed=6), _r(3 * c, 5, seed=7)
    bufs = lambda n: [torch.empty(n * T, c), torch.empty(n * T, c), torch.empty(n, 2, 3, 8)]
    kw = dict(seg_width=c, transposed=(0, 0, 1), rows_per_img=T, head_dim=3, tok_pad=8)
    q, k, vt = R.gemm(x, wl, seg_outs=bufs(4), hi={"w": wh}, **kw)
    for half, ww, sl in ((x[:2 * T], wl, slice(0, 2)), (x[2 * T:], wh, slice(2, 4))):
        q1, k1, vt1 = R.gemm(half, ww, seg_outs=bufs(2), **kw)
        rows = slice(sl.start * T, sl.stop * T)
        torch.testing.assert_close(q[rows], q1)
        torch.testing.assert_close(k[rows], k1)
        torch.testing.assert_close(vt[sl], vt1)


def test_row_term_indexing():
    """rows_per_img different from H*W (a linear's rows), and a row stride wider than N (rowbias_ld, and a slice)"""
    M, K, N, rpi = 12, 4, 3, 4
    a, w = _r(M, K, seed=1), _r(N, K, seed=2)
    buf = _r(3, 10, seed=3)
    plain = a @ w.t()
    want = plain + buf[:, 2:2 + N].repeat_interleave(rpi, 0)
    torch.testing.assert_close(R.gemm(a, w, rowbias=buf[:, 2:2 + N], rows_per_img=rpi), want)
    flat = buf.reshape(-1)[2:]  # the same rows given as a flat tensor and an explicit row stride
    torch.testing.assert_close(R.gemm(a, w, rowbias=flat, rows_per_img=rpi, rowbias_ld=10), want)
    # 4-D: rows_per_img = 0 means H*W rows per image
    a4 = _r(3, 2, 2, K, seed=4)
    got = R.gemm(a4, w, rowbias=buf[:, :N])
    torch.testing.assert_close(got.reshape(M, N), a4.reshape(M, K) @ w.t() + buf[:, :N].repeat_interleave(4, 0))


def test_groupnorm_forward_grouped_raw_and_stats():
    B, H, c1, c2 = 4, 3, 4, 4
    x1, x2, add2 = _r(B, H, H, c1, seed=1).half(), _r(B, H, H, c2, seed=2).half(), _r(B, H, H, c2, seed=3).half()
    gl, bl, gh, bh = _r(8, seed=4), _r(8, seed=5), _r(8, seed=6), _r(8, seed=7)
    y, raw, st = R.groupnorm(x1, gl, bl, 1e-5, True, x2=x2, add2=add2, add2_scale=0.5, groups=4, want_raw=True,
                             want_stats=True, gamma_hi=gh, beta_hi=bh)
    cat = torch.cat([x1.float(), (x2.float() + 0.5 * add2.float()).half().float()], -1)
    torch.testing.assert_close(raw, cat)
    for sl, g, b in ((slice(0, 2), gl, bl), (slice(2, 4), gh, bh)):
        ref = F.silu(F.group_norm(cat[sl].permute(0, 3, 1, 2), 4, g, b, 1e-5)).permute(0, 2, 3, 1)
        torch.testing.assert_close(y[sl], ref, rtol=1e-5, atol=1e-5)
    st = st.view(B, 4, 2)
    torch.testing.assert_close(st[1, 2, 0].item(), cat[1, :, :, 4:6].double().sum().item())
    torch.testing.assert_close(st[3, 0, 1].item(), (cat[3, :, :, :2].double() ** 2).sum().item())


def test_layernorm_grouped_is_two_plain_calls():
    x = _r(6, 5, seed=1)
    g, b, gh, bh = _r(5, seed=2), _r(5, seed=3), _r(5, seed=4), _r(5, seed=5)
    y = R.layernorm(x, g, b, 1e-5, gamma_hi=gh, beta_hi=bh)
    torch.testing.assert_close(y[:3], F.layer_norm(x[:3], (5,), g, b, 1e-5))
    torch.testing.assert_close(y[3:], F.layer_norm(x[3:], (5,), gh, bh, 1e-5))


def test_attention_reads_keys_below_nk_and_lse_is_log2():
    B, Hh, nq, nk, d, pad = 2, 2, 3, 5, 4, 8
    q, k, v = _r(B * nq, Hh * d, seed=1), _r(B * nk, Hh * d, seed=2), _r(B * nk, Hh * d, seed=3)
    vt = torch.full((B, Hh, d, pad), 1e4)
    vt[..., :nk] = v.view(B, nk, Hh, d).permute(0, 2, 3, 1)
    out, lse = R.attention(q, k, vt, B, Hh, nq, nk, d, lse=torch.empty(B, Hh, nq))
    for b in range(B):
        for h in range(Hh):
            qs, ks, vs = (t.view(B, -1, Hh, d)[b, :, h] for t in (q, k, v))
            s = qs @ ks.t() / d ** 0.5
            torch.testing.assert_close(out.view(B, nq, Hh, d)[b, :, h], s.softmax(-1) @ vs)
            torch.testing.assert_close(lse[b, h], torch.log2(torch.exp(s).sum(-1)))


def test_wgrad_tn_accumulates_onto_out():
    a, b, out = _r(7, 3, seed=1), _r(7, 4, seed=2), _r(3, 4, seed=3)
    torch.testing.assert_close(R.wgrad_tn(a, b, out=out, alpha=0.5, beta=1.0), 0.5 * a.t() @ b + out)
    torch.testing.assert_close(R.wgrad_tn(a, b, out=out, alpha=2.0), 2.0 * a.t() @ b)


D = torch.float64


@pytest.mark.parametrize("silu,concat,res", [(True, False, False), (False, False, True), (True, True, True)])
def test_groupnorm_bwd_matches_finite_differences(silu, concat, res):
    """dx1 (with add1), dx2 and dgamma / dbeta (onto non-zero buffers), the `res` addend and both scales"""
    B, H, c1, c2, G = 2, 2, 4, 4 if concat else 0, 4
    C = c1 + c2
    x1, add1 = _r(B, H, H, c1, seed=1, dtype=D), _r(B, H, H, c1, seed=2, dtype=D)
    x2 = _r(B, H, H, c2, seed=3, dtype=D) if concat else None
    add2 = _r(B, H, H, c2, seed=4, dtype=D) if concat else None
    g, b = 1 + 0.3 * _r(C, seed=5, dtype=D), 0.3 * _r(C, seed=6, dtype=D)
    dy, r = _r(B, H, H, C, seed=7, dtype=D), (_r(B, H, H, C, seed=8, dtype=D) if res else None)
    dg0, db0 = _r(C, seed=9, dtype=D), _r(C, seed=10, dtype=D)
    kw = dict(add1=add1, add1_scale=1.3, x2=x2, add2=add2, add2_scale=0.7, groups=G)
    dx1, dx2, dg, db = R.groupnorm_bwd(dy, None, x1, g, b, 1e-5, silu, want_dx2=concat, dx2_scale=0.7, dgamma=dg0,
                                       dbeta=db0, res=r, dx1_scale=0.6, **kw)

    def loss(x1_=x1, x2_=x2, g_=g, b_=b):
        kk = dict(kw, x2=x2_)
        y = R.groupnorm(x1_, g_, b_, 1e-5, silu, **kk)
        cat = R._concat(x1_, add1, 1.3, x2_, add2, 0.7)
        return (y * dy).sum() + ((cat * r).sum() if res else 0.0)

    torch.testing.assert_close(dx1, 0.6 * _fd_grad(lambda t: loss(x1_=t), x1.clone()), rtol=1e-6, atol=1e-7)
    if concat:  # d(x2 half) = d(add2) / add2_scale, which the caller gets through dx2_scale = add2_scale
        torch.testing.assert_close(dx2, 0.7 * _fd_grad(lambda t: loss(x2_=t), x2.clone()), rtol=1e-6, atol=1e-7)
    else:
        assert dx2 is None
    torch.testing.assert_close(dg, dg0 + _fd_grad(lambda t: loss(g_=t), g.clone()), rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(db, db0 + _fd_grad(lambda t: loss(b_=t), b.clone()), rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("res", [False, True])
def test_layernorm_bwd_matches_finite_differences(res):
    x, dy, g = _r(3, 6, seed=1, dtype=D), _r(3, 6, seed=2, dtype=D), 1 + 0.3 * _r(6, seed=3, dtype=D)
    r = _r(3, 6, seed=4, dtype=D) if res else None
    dg0, db0 = _r(6, seed=5, dtype=D), _r(6, seed=6, dtype=D)
    dx, dg, db = R.layernorm_bwd(x, dy, g, 1e-5, dg0, db0, res=r)
    beta = 0.2 * _r(6, seed=7, dtype=D)

    def loss(x_=x, g_=g, b_=beta):
        return (R.layernorm(x_, g_, b_, 1e-5) * dy).sum() + ((x_ * r).sum() if res else 0.0)

    torch.testing.assert_close(dx, _fd_grad(lambda t: loss(x_=t), x.clone()), rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(dg, dg0 + _fd_grad(lambda t: loss(g_=t), g.clone()), rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(db, db0 + _fd_grad(lambda t: loss(b_=t), beta.clone()), rtol=1e-6, atol=1e-7)
    assert R.layernorm_bwd(x, dy, g, 1e-5)[1:] == (None, None)


def test_attention_bwd_matches_finite_differences():
    B, Hh, nq, nk, d = 2, 2, 3, 4, 2
    q, k, v = _r(B * nq, Hh * d, seed=1, dtype=D), _r(B * nk, Hh * d, seed=2, dtype=D), _r(B * nk, Hh * d, seed=3, dtype=D)
    dout = _r(B * nq, Hh * d, seed=4, dtype=D)
    dq, dk, dv = R.attention_bwd(q, k, v, None, dout, None, B, Hh, nq, nk, d)

    def loss(q_=q, k_=k, v_=v):
        vt = v_.view(B, nk, Hh, d).permute(0, 2, 3, 1)
        return (R.attention(q_, k_, vt, B, Hh, nq, nk, d) * dout).sum()

    torch.testing.assert_close(dq, _fd_grad(lambda t: loss(q_=t), q.clone()), rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(dk, _fd_grad(lambda t: loss(k_=t), k.clone()), rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(dv, _fd_grad(lambda t: loss(v_=t), v.clone()), rtol=1e-6, atol=1e-7)
    o = R.attention(q, k, v.view(B, nk, Hh, d).permute(0, 2, 3, 1), B, Hh, nq, nk, d)
    dq_o, dk_o = R.attention_dqk_given_o(q, k, v, o, dout, B, Hh, nq, nk, d)
    torch.testing.assert_close(dq_o, dq, rtol=1e-9, atol=1e-12)
    torch.testing.assert_close(dk_o, dk, rtol=1e-9, atol=1e-12)


def test_exact_fp32_restores_the_tf32_flags():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    with R.exact_fp32():
        assert not torch.backends.cuda.matmul.allow_tf32 and not torch.backends.cudnn.allow_tf32
    assert (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32) == old
