"""Plain torch references of single calls of the ctrlora_b200.ops wrappers (test infrastructure).

Each function takes exactly the arguments of the `ops` wrapper of the same name and returns what that call should have
written, computed in fp32 (fp64 when the operands are fp64) without tiling or any of the kernels' schemes.  Output
buffers among the arguments are read only for their shapes and for values the call accumulates onto (`wgrad_tn`'s
`out` when beta != 0, `groupnorm_bwd` / `layernorm_bwd`'s dgamma / dbeta); a caller checking a call that overwrites an
input passes that input's pre-call copy.  The semantics are those of include/ctrlora_b200.h.  Device-agnostic:
tests/test_launch_refs_cpu.py pins them at tiny shapes on the host; tests/test_step_launches_gpu.py and
tests/test_path_launches_gpu.py check every launch of the benchmarked steps, the sampling variants, the VAE encoder and
the annotators against them (through tests/launch_shadow.py).  Gathers, pools and copies return the kernel's dtype and
are compared bit for bit.
"""
import contextlib

import torch
import torch.nn.functional as F

LOG2E = 1.4426950408889634


@contextlib.contextmanager
def exact_fp32():
    """fp32 matmuls and convolutions without TF32 (restored afterwards)"""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _f(t):
    """fp64 stays fp64 (the host checks of the references), everything else computes in fp32"""
    return None if t is None else (t.double() if t.dtype == torch.float64 else t.float())


def _dtype(t):
    return torch.float64 if t.dtype == torch.float64 else torch.float32


def _round16(t, like):
    """the fp16 rounding a kernel applies to an intermediate it stores as fp16 (none in fp64 mode)"""
    return t if like.dtype == torch.float64 else t.half().float()


def _rows(t, m, cols):
    """[m, cols] view of a pixel-major / row-major tensor with a uniform row stride (stride(-2))"""
    return torch.as_strided(t, (m, cols), (t.stride(-2), 1))


# ------------------------------------------------------------------------------------------------------------ GEMM
def _product(a, w, ksize):
    """sum over the taps and channels: a [B, H, W, C] (conv, pad (k-1)/2) or [M, K] (linear) -> [M, N]"""
    n = w.shape[0]
    if ksize == 1:
        return _f(a).reshape(-1, a.shape[-1]) @ _f(w).reshape(n, -1).t()
    wt = _f(w).reshape(n, ksize, ksize, -1).permute(0, 3, 1, 2)
    y = F.conv2d(_f(a).permute(0, 3, 1, 2), wt, padding=(ksize - 1) // 2)
    return y.permute(0, 2, 3, 1).reshape(-1, n)


def _gemm_rows(a, w, ksize, bias, rowbias, rows_per_img, rowbias_ld, out_scale, a2, w2, geglu):
    """epilogue(conv_or_linear(a, w) [+ a2 w2^T]) of one (sub-)batch before the residual: fp32 [rows, n]"""
    y = _product(a, w, ksize)
    if a2 is not None:
        y = y + _f(a2).reshape(-1, a2.shape[-1]) @ _f(w2).reshape(w2.shape[0], -1).t()
    if bias is not None:
        y = y + _f(bias)
    if geglu:
        n = y.shape[1] // 2
        y = y[:, :n] * F.gelu(y[:, n:])
    if rowbias is not None:
        rows, n = y.shape
        hw = rows if a.dim() == 2 else a.shape[1] * a.shape[2]
        rpi = rows_per_img or hw
        imgs = rows // rpi
        rb = torch.as_strided(rowbias, (imgs, n), (rowbias_ld or rowbias.stride(0), 1))
        y = y + _f(rb).repeat_interleave(rpi, 0)
    return y * out_scale


def gemm(a, w, *, ksize=1, bias=None, rowbias=None, rows_per_img=0, rowbias_ld=0, residual=None, out_scale=1.0, a2=None,
         w2=None, geglu=False, out=None, out_f32=False, seg_outs=None, seg_width=0, transposed=(0, 0, 0), head_dim=0,
         tok_pad=0, block_n=0, split_k=0, dup_out=None, single_cta=False, simt=False, hi=None):
    """ops.gemm: the output tensor, or the list of segment outputs followed by dup_out's contents when dup_out is given.
    A transposed segment comes back in its [image, head, d, tok_pad] buffer shape with zeros in the padding tokens
    [rows_per_img, tok_pad), which the kernel does not write.  hi: the upper half of the batch (images of a 4-D `a`,
    rows of a 2-D one) takes hi's weights, bias, skip weights and row terms, the row terms indexed from that half's
    first image -- i.e. two plain calls on the halves.  block_n, split_k, single_cta and simt choose a plan, not a
    result."""
    m = a.shape[0] if a.dim() == 2 else a.shape[0] * a.shape[1] * a.shape[2]
    with exact_fp32():
        if hi is None:
            y = _gemm_rows(a, w, ksize, bias, rowbias, rows_per_img, rowbias_ld, out_scale, a2, w2, geglu)
        else:
            h = a.shape[0] // 2
            ld = rowbias_ld or (rowbias.stride(0) if rowbias is not None else 0)  # one row stride for both halves
            y = torch.cat([
                _gemm_rows(a[:h], w, ksize, bias, rowbias, rows_per_img, ld, out_scale,
                           None if a2 is None else a2[:h], w2, geglu),
                _gemm_rows(a[h:], hi["w"], ksize, hi.get("bias"), hi.get("rowbias"), rows_per_img, ld, out_scale,
                           None if a2 is None else a2[h:], hi.get("w2"), geglu)])
    n = y.shape[1]
    if residual is not None:
        y = y + _f(_rows(residual, m, n))
    if seg_outs is None:
        shape = out.shape if out is not None else a.shape[:-1] + (n,)
        return y.reshape(shape)
    rpi = rows_per_img or (m if a.dim() == 2 else a.shape[1] * a.shape[2])
    res, dup = [], None
    for i, o in enumerate(seg_outs):
        cols = y[:, i * seg_width:(i + 1) * seg_width]
        if transposed[i]:
            assert dup is None or dup_out is None, "dup_out copies one transposed segment"
            t = torch.zeros(o.shape, dtype=y.dtype, device=y.device)
            t.view(m // rpi, seg_width, -1)[:, :, :rpi] = cols.reshape(m // rpi, rpi, seg_width).transpose(1, 2)
            res.append(t)
            dup = cols
        else:
            res.append(cols.reshape(o.shape))
    if dup_out is not None:
        res.append(dup.reshape(dup_out.shape))
    return res


def gemm_relu(a, w, **kwargs):
    """ops.gemm_relu: gemm's result, then max(., 0) after the residual, on every segment and dup_out"""
    y = gemm(a, w, **kwargs)
    return [t.clamp_min(0) for t in y] if isinstance(y, list) else y.clamp_min(0)


# ------------------------------------------------------------------------------------------------------- GroupNorm
def _concat(x1, add1, add1_scale, x2, add2, add2_scale):
    """[x1 + s1 add1 | x2 + s2 add2] as the kernels stage it: each summed half rounded to fp16"""
    h1 = _f(x1) if add1 is None else _round16(_f(x1) + add1_scale * _f(add1), x1)
    if x2 is None:
        return h1
    h2 = _f(x2) if add2 is None else _round16(_f(x2) + add2_scale * _f(add2), x2)
    return torch.cat([h1, h2], -1)


def _per_image(p, p_hi, b, like):
    """affine parameter per image [b, C]: the upper half of the batch takes p_hi when given"""
    t = _f(p).to(like.dtype).expand(b, -1).clone()
    if p_hi is not None:
        t[b // 2:] = _f(p_hi).to(like.dtype)
    return t


def _gn_forward(cat, gamma, beta, eps, silu, groups, gamma_hi=None, beta_hi=None):
    b, c = cat.shape[0], cat.shape[-1]
    z = F.group_norm(cat.permute(0, 3, 1, 2), groups, eps=eps).permute(0, 2, 3, 1)
    y = z * _per_image(gamma, gamma_hi, b, cat).view(b, 1, 1, c) + _per_image(beta, beta_hi, b, cat).view(b, 1, 1, c)
    return F.silu(y) if silu else y


def groupnorm(x1, gamma, beta, eps, silu, *, add1=None, add1_scale=1.0, x2=None, add2=None, add2_scale=1.0, groups=32,
              want_raw=False, want_stats=False, out=None, gamma_hi=None, beta_hi=None):
    """ops.groupnorm: y (and the raw concatenation, and the fp64 {sum, sumsq} per (image, group) in the
    [batch * groups * 2] layout of its statistics), in the order ops.groupnorm returns them"""
    cat = _concat(x1, add1, add1_scale, x2, add2, add2_scale)
    y = _gn_forward(cat, gamma, beta, eps, silu, groups, gamma_hi, beta_hi)
    ret = [y]
    if want_raw:
        ret.append(cat)
    if want_stats:
        b, c = cat.shape[0], cat.shape[-1]
        g = cat.double().reshape(b, -1, groups, c // groups)
        ret.append(torch.stack([g.sum((1, 3)), (g * g).sum((1, 3))], -1).reshape(-1))
    return ret[0] if len(ret) == 1 else tuple(ret)


def layernorm(x, gamma, beta, eps=1e-5, gamma_hi=None, beta_hi=None):
    """ops.layernorm; with gamma_hi / beta_hi the upper half of the rows takes them"""
    c = x.shape[-1]
    x2 = _f(x).reshape(-1, c)
    rows = x2.shape[0]
    z = F.layer_norm(x2, (c,), eps=eps)
    if gamma_hi is None:
        return (z * _f(gamma) + _f(beta)).view(x.shape)
    h = rows // 2
    y = torch.cat([z[:h] * _f(gamma) + _f(beta), z[h:] * _f(gamma_hi) + _f(beta_hi)])
    return y.view(x.shape)


# ------------------------------------------------------------------------------------------------------- attention
def _heads(t, batch, n, heads, d):
    """[batch * n, heads * d] (row stride free) -> [batch, heads, n, d]"""
    return _f(t).reshape(batch, n, heads, d).transpose(1, 2)


def attention(q, k, vt, batch, heads, nq, nk, head_dim, out=None, lse=None):
    """ops.attention: out [batch * nq, heads * d], and with `lse` also the log2-domain log-sum-exp [batch, heads, nq].
    Keys are read from vt[..., :nk]; one image at a time (bounded memory)."""
    d = head_dim
    o = torch.empty(batch, nq, heads, d, dtype=_dtype(q), device=q.device)
    l2 = torch.empty(batch, heads, nq, dtype=o.dtype, device=q.device)
    with exact_fp32():
        for b in range(batch):
            qb = _heads(q[b * nq:(b + 1) * nq], 1, nq, heads, d)[0]
            kb = _heads(k[b * nk:(b + 1) * nk], 1, nk, heads, d)[0]
            vb = _f(vt[b, ..., :nk]).transpose(-1, -2)          # [heads, nk, d]
            s = (qb @ kb.transpose(-1, -2)) * d ** -0.5
            o[b] = (s.softmax(-1) @ vb).transpose(0, 1)
            l2[b] = torch.logsumexp(s, -1) * LOG2E
    o = o.reshape(batch * nq, heads * d)
    return o if lse is None else (o, l2)


def attention_bwd(q, k, v, o, dout, lse, batch, heads, nq, nk, head_dim, dq=None, dk=None, dv=None):
    """ops.attention_bwd: (dq, dk, dv) by autograd of the forward on q, k, v (natural layout); o and lse are the
    forward's outputs, which the reference recomputes"""
    d = head_dim
    grads = [torch.empty(batch, n, heads, d, dtype=_dtype(q), device=q.device) for n in (nq, nk, nk)]
    with exact_fp32(), torch.enable_grad():
        for b in range(batch):
            qb, kb, vb = (_heads(t[b * n:(b + 1) * n], 1, n, heads, d)[0].detach().requires_grad_(True)
                          for t, n in ((q, nq), (k, nk), (v, nk)))
            s = (qb @ kb.transpose(-1, -2)) * d ** -0.5
            ob = s.softmax(-1) @ vb
            ob.backward(_heads(dout[b * nq:(b + 1) * nq], 1, nq, heads, d)[0])
            for g, t in zip(grads, (qb, kb, vb)):
                g[b] = t.grad.transpose(0, 1)
    return tuple(g.reshape(-1, heads * d) for g in grads)


def attention_dqk_given_o(q, k, v, o, dout, batch, heads, nq, nk, head_dim):
    """(dq, dk) of attention_bwd with the softmax-gradient row term rowsum(dout * o) taken from the given forward output
    `o` instead of the exact one: dS = P (dout v^T - rowsum(dout * o)), dq = scale dS k, dk = scale dS^T q.  Equal to
    attention_bwd's when o is the exact forward output; with the fp16 o the kernels receive it isolates what that
    rounding contributes."""
    d = head_dim
    dq = torch.empty(batch, nq, heads, d, dtype=_dtype(q), device=q.device)
    dk = torch.empty(batch, nk, heads, d, dtype=_dtype(q), device=q.device)
    with exact_fp32():
        for b in range(batch):
            qb, kb, vb, ob, gb = (_heads(t[b * n:(b + 1) * n], 1, n, heads, d)[0]
                                  for t, n in ((q, nq), (k, nk), (v, nk), (o, nq), (dout, nq)))
            p = ((qb @ kb.transpose(-1, -2)) * d ** -0.5).softmax(-1)
            ds = p * (gb @ vb.transpose(-1, -2) - (gb * ob).sum(-1, keepdim=True))
            dq[b] = ((ds @ kb) * d ** -0.5).transpose(0, 1)
            dk[b] = ((ds.transpose(-1, -2) @ qb) * d ** -0.5).transpose(0, 1)
    return dq.reshape(-1, heads * d), dk.reshape(-1, heads * d)


# ------------------------------------------------------------------------------------------------------- training
def wgrad_tn(a, b, out=None, alpha=1.0, beta=0.0):
    """ops.wgrad_tn: alpha a^T b + beta out (out = its contents before the call)"""
    with exact_fp32():
        y = alpha * (_f(a).t() @ _f(b))
    return y if beta == 0.0 else y + beta * _f(out)


def groupnorm_bwd(dy, fwd_stats, x1, gamma, beta, eps, silu, *, add1=None, add1_scale=1.0, x2=None, add2=None,
                  add2_scale=1.0, groups=32, want_dx2=False, dx2_scale=1.0, dgamma=None, dbeta=None, res=None,
                  dx1_scale=1.0):
    """ops.groupnorm_bwd: (dx1, dx2 | None, dgamma | None, dbeta | None) by autograd of the forward reference.
    The concatenation's gradient plus `res` is scaled by dx1_scale (first half) and dx2_scale (second half); dgamma /
    dbeta are the given buffers' contents plus the parameter gradients.  fwd_stats is recomputed, not read."""
    c1 = x1.shape[-1]
    with torch.enable_grad():
        cat = _concat(x1, add1, add1_scale, x2, add2, add2_scale).detach().requires_grad_(True)
        g, b = _f(gamma).detach().requires_grad_(True), _f(beta).detach().requires_grad_(True)
        _gn_forward(cat, g, b, eps, silu, groups).backward(_f(dy))
    dcat = cat.grad
    if res is not None:
        dcat = dcat + _f(_rows(res, dcat[..., 0].numel(), dcat.shape[-1])).view(dcat.shape)
    dx1 = dx1_scale * dcat[..., :c1]
    dx2 = dx2_scale * dcat[..., c1:] if (want_dx2 and x2 is not None) else None
    return (dx1, dx2, None if dgamma is None else _f(dgamma) + g.grad, None if dbeta is None else _f(dbeta) + b.grad)


def layernorm_bwd(x, dy, gamma, eps=1e-5, dgamma=None, dbeta=None, res=None):
    """ops.layernorm_bwd: (dx (+ res), dgamma | None, dbeta | None), the parameter gradients accumulated onto the given
    buffers' contents"""
    c = x.shape[-1]
    with torch.enable_grad():
        xf = _f(x).reshape(-1, c).detach().requires_grad_(True)
        g = _f(gamma).detach().requires_grad_(True)
        b = torch.zeros_like(g, requires_grad=True)
        F.layer_norm(xf, (c,), g, b, eps).backward(_f(dy).reshape(-1, c))
    dx = xf.grad if res is None else xf.grad + _f(res).reshape(-1, c)
    return (dx.view(x.shape), None if dgamma is None else _f(dgamma) + g.grad,
            None if dbeta is None else _f(dbeta) + b.grad)


# ------------------------------------------------------------------------------------------- gathers and small kernels
def im2col_s2(x, pad_lo=1):
    """ops.im2col_s2: the 3x3 stride-2 patches of x [B, H, W, C] zero-padded by pad_lo on the top / left and 1 on the
    bottom / right, tap-major and channel-minor -> x.dtype [B, H // 2, W // 2, 9 C]"""
    b, h, w, c = x.shape
    xp = F.pad(_f(x).permute(0, 3, 1, 2), (pad_lo, 1, pad_lo, 1))
    cols = F.unfold(xp, 3, stride=2)                                     # [B, C * 9, L], channel-major
    oh, ow = (h + pad_lo - 2) // 2 + 1, (w + pad_lo - 2) // 2 + 1
    cols = cols.view(b, c, 9, oh, ow)[:, :, :, :h // 2, :w // 2]
    return cols.permute(0, 3, 4, 2, 1).reshape(b, h // 2, w // 2, 9 * c).to(x.dtype)


def upsample2x(x):
    """ops.upsample2x: nearest-neighbour x2 of x [B, H, W, C] -> [B, 2H, 2W, C]"""
    return x.repeat_interleave(2, 1).repeat_interleave(2, 2)


def softmax_rows(logits, scale=1.0):
    """ops.softmax_rows: softmax(scale * logits) over the last dim, fp32"""
    return (_f(logits) * scale).softmax(-1)


def weighted_sum(tensors, weights, out=None):
    """ops.weighted_sum: sum_i weights[i] tensors[i] in fp32"""
    y = torch.zeros(tensors[0].shape, dtype=_dtype(tensors[0]), device=tensors[0].device)
    for t, wt in zip(tensors, weights):
        y = y + float(wt) * _f(t)
    return y


def gaussian_sample(moments, noise=None, scale=1.0):
    """ops.gaussian_sample: scale (mean + exp(0.5 clamp(logvar, -30, 20)) noise), or scale mean without noise; moments
    [B, 2Z, H, W] = mean | logvar"""
    mean, logvar = _f(moments).chunk(2, dim=1)
    if noise is None:
        return scale * mean
    return scale * (mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * _f(noise))


# ------------------------------------------------------------------------------------------------------ annotators
TAPS7 = [(ky - 3, kx - 3) for ky in range(7) for kx in range(7)]


def _tap_index(n, d, reflect, device):
    """(source index, inside mask | None) of positions 0 .. n-1 shifted by d along an axis of length n: mirrored
    without repeating the border (nn.ReflectionPad2d, |d| < n), or clamped with the mask of those inside"""
    i = torch.arange(n, device=device) + d
    if reflect:
        i = i.abs()
        return torch.where(i >= n, 2 * (n - 1) - i, i), None
    return i.clamp(0, n - 1), (i >= 0) & (i < n)


def _shifted(src, dy, dx, reflect):
    """src [B, H, W, C] read at (y + dy, x + dx), reflected at the border or zero outside"""
    _, h, w, _ = src.shape
    iy, my = _tap_index(h, dy, reflect, src.device)
    ix, mx = _tap_index(w, dx, reflect, src.device)
    g = src[:, iy][:, :, ix]
    if reflect:
        return g
    inside = (my[:, None] & mx[None, :])[None, :, :, None]
    return torch.where(inside, g, torch.zeros((), dtype=g.dtype, device=g.device))


def tap_gather(x, taps, *, reflect, k_pad, channels=None, out=None):
    """ops.tap_gather: column t * C + c of pixel (y, x) = source channel c at (y + dy_t, x + dx_t), reflected or zero
    outside; columns >= len(taps) * C zero.  x fp16 pixel-major [B, H, W, ld] (the first `channels`), or fp32 NCHW
    [B, C, H, W], which the gather rounds to fp16.  -> fp16 [B, H, W, k_pad] (fp64 for an fp64 source)"""
    src = x[..., :channels or x.shape[-1]] if x.dtype == torch.float16 else x.permute(0, 2, 3, 1)
    b, h, w, c = src.shape
    y = torch.zeros((b, h, w, k_pad), dtype=torch.float64 if x.dtype == torch.float64 else torch.float16,
                    device=x.device)
    for t, (dy, dx) in enumerate(taps):
        y[..., t * c:(t + 1) * c] = _shifted(src, dy, dx, reflect)   # fp32 -> fp16: round to nearest even
    return y


def instance_norm(x, *, relu, residual=None, phases=False, eps=1e-5, out=None):
    """ops.instance_norm: per (image, channel) biased statistics over the image's pixels, y = relu?((x - mean) /
    sqrt(var + eps)) + residual?.  phases: x [4, B, H, W, C] holds sub-pixel phase 2 py + px, and y[b, 2m + py, 2n + px]
    = f(x[2 py + px, b, m, n]) -> [B, 2H, 2W, C]"""
    xf = _f(x)
    if phases:
        _, b, h, w, c = x.shape
        xf = xf.view(2, 2, b, h, w, c).permute(2, 3, 0, 4, 1, 5).reshape(b, 2 * h, 2 * w, c)
    mean = xf.mean((1, 2), keepdim=True)
    var = ((xf - mean) ** 2).mean((1, 2), keepdim=True)
    y = (xf - mean) / torch.sqrt(var + eps)
    if relu:
        y = y.clamp_min(0)
    return y if residual is None else y + _f(residual)


def _quantise(y):
    """LineartDetector's uint8 map of an fp32 map (lineart_golden.quantise, on the host)"""
    import lineart_golden
    return torch.from_numpy(lineart_golden.quantise(y.cpu().numpy())).to(y.device)


def lineart_out(x, weight, bias, want_u8=False):
    """ops.lineart_out: sigmoid(bias + the 7x7 taps of x [B, H, W, C] reflected by 3, weighted by weight [49, C]
    tap-major) -> [B, 1, H, W] (and with want_u8 the uint8 map of that reference)"""
    xf = _f(x)
    wf = _f(weight).to(xf.dtype)
    y = torch.zeros(x.shape[:3], dtype=xf.dtype, device=x.device)
    with exact_fp32():
        for t, (dy, dx) in enumerate(TAPS7):
            y += _shifted(xf, dy, dx, True) @ wf[t]
    y = torch.sigmoid(y + _f(bias).to(xf.dtype)).unsqueeze(1)
    return (y, _quantise(y[:, 0])) if want_u8 else y


def max_pool2x2(x):
    """ops.max_pool2x2: the 2x2 max of x [B, h, w, C], floor sizes -> x.dtype [B, h // 2, w // 2, C]"""
    b, h, w, c = x.shape
    return x[:, :h // 2 * 2, :w // 2 * 2].reshape(b, h // 2, 2, w // 2, 2, c).amax((2, 4))


def hed_side_pool(x, weight, bias, pool):
    """ops.hed_side_pool: (bias + x @ weight [B, 1, h, w], max_pool2x2(x) or None).  The projection sums in fp64, as its
    per-kernel test does: the bound is 1e-6, a few times fp32's rounding of a sum over C products"""
    side = (x.double() @ weight.double() + bias.double()).unsqueeze(1).to(_dtype(x))
    return side, (max_pool2x2(x) if pool else None)
