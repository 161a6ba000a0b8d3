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


# ---------------------------------------------------------------------- the sampling variants, VAE encoder, annotators
def test_gemm_relu_clamps_after_the_residual_and_on_every_segment():
    M, K, N = 9, 6, 8
    a, w, bias = _r(M, K, seed=1).half(), _r(2 * N, K, seed=2).half(), _r(2 * N, seed=3)
    res = _r(M, 2 * N, seed=4).half()
    plain = R.gemm(a, w, bias=bias, residual=res)
    assert (plain < 0).any()
    torch.testing.assert_close(R.gemm_relu(a, w, bias=bias, residual=res), plain.clamp_min(0), rtol=0, atol=0)
    segs = R.gemm_relu(a, w, seg_outs=[torch.empty(M, N), torch.empty(M, N)], seg_width=N, transposed=(0, 0))
    torch.testing.assert_close(torch.cat(segs, 1), R.gemm(a, w).clamp_min(0), rtol=0, atol=0)


def _mirror(i, n):
    return -i if i < 0 else (2 * (n - 1) - i if i >= n else i)


@pytest.mark.parametrize("reflect", [True, False])
@pytest.mark.parametrize("src", ["f16", "f16_ld", "f32_nchw"])
def test_tap_gather_is_a_loop_over_pixels_and_taps(reflect, src):
    """column t * C + c of pixel (y, x) = channel c at (y + dy_t, x + dx_t): mirrored without repeating the border, or
    zero outside; the columns past the taps zero; an fp32 NCHW source rounded to fp16"""
    B, H, W, C = 2, 5, 6, 3
    taps = [(ky - 3, kx - 3) for ky in range(7) for kx in range(7)] if src == "f32_nchw" else \
        [(0, 0), (0, 1), (1, 0), (1, 1), (-1, 2)]
    k_pad = (len(taps) * C + 15) // 16 * 16
    if src == "f32_nchw":
        x = _r(B, C, H, W, seed=1) * 3
        at = lambda b, y, xx, c: x[b, c, y, xx].half()
        got = R.tap_gather(x, taps, reflect=reflect, k_pad=k_pad)
    else:
        ld = C + 5 if src == "f16_ld" else C
        x = _r(B, H, W, ld, seed=2).half()
        at = lambda b, y, xx, c: x[b, y, xx, c]
        got = R.tap_gather(x, taps, reflect=reflect, k_pad=k_pad, channels=C)
    assert got.dtype == torch.float16 and got.shape == (B, H, W, k_pad)
    ref = torch.zeros(B, H, W, k_pad, dtype=torch.float16)
    for b in range(B):
        for y in range(H):
            for xx in range(W):
                for t, (dy, dx) in enumerate(taps):
                    sy, sx = y + dy, xx + dx
                    if reflect:
                        sy, sx = _mirror(sy, H), _mirror(sx, W)
                    elif not (0 <= sy < H and 0 <= sx < W):
                        continue
                    for c in range(C):
                        ref[b, y, xx, t * C + c] = at(b, sy, sx, c)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("mode", ["relu", "residual", "phases"])
def test_instance_norm_against_fp64_statistics(mode):
    """biased per (image, channel) statistics; with phases the output pixel (2m + py, 2n + px) of image b is phase
    2 py + px's pixel (m, n)"""
    B, H, W, C = 2, 3, 4, 5
    phases = mode == "phases"
    x = (_r(4, B, H, W, C, seed=1) if phases else _r(B, H, W, C, seed=1)) * 2 + 3
    res = _r(B, H, W, C, seed=2) if mode == "residual" else None
    got = R.instance_norm(x.half(), relu=mode != "residual", residual=None if res is None else res.half(),
                          phases=phases)
    xd = x.half().double()
    if phases:
        full = torch.zeros(B, 2 * H, 2 * W, C, dtype=D)
        for p in range(4):
            py, px = divmod(p, 2)
            for b in range(B):
                for m in range(H):
                    for n in range(W):
                        full[b, 2 * m + py, 2 * n + px] = xd[p, b, m, n]
        xd = full
    ref = torch.empty_like(xd)
    for b in range(B):
        for c in range(C):
            v = xd[b, :, :, c]
            mean = v.sum() / v.numel()
            var = ((v - mean) ** 2).sum() / v.numel()
            ref[b, :, :, c] = (v - mean) / torch.sqrt(var + 1e-5)
    ref = ref + res.half().double() if res is not None else ref.clamp_min(0)
    torch.testing.assert_close(got.double(), ref, rtol=1e-5, atol=1e-5)


def test_lineart_out_is_a_reflect_padded_conv_and_sigmoid():
    B, H, W, C = 2, 5, 7, 4
    x = _r(B, H, W, C, seed=1).half()
    conv_w, bias = _r(1, C, 7, 7, seed=2) * 0.3, _r(1, seed=3)
    weight = conv_w[0].permute(1, 2, 0).reshape(49, C).contiguous()  # tap-major, as the Generator prepares it
    y, u8 = R.lineart_out(x, weight, bias, want_u8=True)
    ref = torch.sigmoid(F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (3, 3, 3, 3), mode="reflect"), conv_w, bias))
    torch.testing.assert_close(y, ref, rtol=1e-5, atol=1e-6)
    assert torch.equal(u8, (ref[:, 0] * 255.0).clamp(0, 255).to(torch.uint8))
    assert torch.equal(R.lineart_out(x, weight, bias), y)


@pytest.mark.parametrize("h,w", [(6, 8), (7, 9)])
def test_hed_side_pool_and_max_pool(h, w):
    B, C = 2, 16
    x = _r(B, h, w, C, seed=1).half()
    weight, bias = _r(C, seed=2), _r(1, seed=3)
    side, pooled = R.hed_side_pool(x, weight, bias, pool=True)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), weight.double().view(1, C, 1, 1), bias.double())
    torch.testing.assert_close(side, ref.float(), rtol=1e-6, atol=1e-6)
    want = F.max_pool2d(x.float().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).half()
    assert torch.equal(pooled, want) and torch.equal(R.max_pool2x2(x), want)
    assert R.hed_side_pool(x, weight, bias, pool=False)[1] is None


@pytest.mark.parametrize("pad_lo", [0, 1])
@pytest.mark.parametrize("h,w", [(6, 8), (7, 9)])
def test_im2col_s2_is_a_loop_over_patches(pad_lo, h, w):
    """out[b, r, s, t C + c] = x[b, 2r + ky - pad_lo, 2s + kx - pad_lo, c] for tap t = 3 ky + kx, zero outside"""
    B, C = 2, 3
    x = _r(B, h, w, C, seed=1).half()
    got = R.im2col_s2(x, pad_lo=pad_lo)
    ref = torch.zeros(B, h // 2, w // 2, 9 * C, dtype=torch.float16)
    for r in range(h // 2):
        for s in range(w // 2):
            for t in range(9):
                ky, kx = divmod(t, 3)
                y, xx = 2 * r + ky - pad_lo, 2 * s + kx - pad_lo
                if 0 <= y < h and 0 <= xx < w:
                    ref[:, r, s, t * C:(t + 1) * C] = x[:, y, xx]
    assert got.dtype == torch.float16 and torch.equal(got, ref)


def test_upsample2x_is_nearest():
    x = _r(2, 3, 5, 4, seed=1).half()
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1).half()
    assert torch.equal(R.upsample2x(x), ref)


def test_softmax_weighted_sum_and_gaussian_sample_formulas():
    logits = _r(3, 7, seed=1) * 4
    e = torch.exp(logits.double() * 0.3 - (logits.double() * 0.3).max(-1, keepdim=True).values)
    torch.testing.assert_close(R.softmax_rows(logits, 0.3).double(), e / e.sum(-1, keepdim=True), rtol=1e-6, atol=1e-7)
    ts, wts = [_r(2, 4, 8, seed=i).half() for i in range(3)], (0.7, 0.45, -1.25)
    ref = 0.7 * ts[0].double() + 0.45 * ts[1].double() - 1.25 * ts[2].double()
    torch.testing.assert_close(R.weighted_sum(ts, wts).double(), ref, rtol=1e-6, atol=1e-6)
    mom = _r(2, 8, 3, 3, seed=5) * 3
    mom[0, 4] = 40.0                    # log-variances beyond clamp(-30, 20) on both sides
    mom[1, 5] = -50.0
    noise = _r(2, 4, 3, 3, seed=6)
    logvar = mom[:, 4:].double().clamp(-30, 20)
    ref = 0.18215 * (mom[:, :4].double() + torch.exp(0.5 * logvar) * noise.double())
    torch.testing.assert_close(R.gaussian_sample(mom, noise, 0.18215).double(), ref, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(R.gaussian_sample(mom, None, 0.18215).double(), 0.18215 * mom[:, :4].double())
