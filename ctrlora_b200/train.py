"""CtrLoRA finetune training step on the sm_90a kernels: forward with saved activations, hand-scheduled backward,
flat-buffer NCCL all-reduce of the trainable gradients and fused AdamW.

reference call stack (SURVEY.md §3.1): LatentDiffusion.p_losses (ldm/models/diffusion/ddpm.py:885-920) ->
ControlFinetuneLDM.apply_model (cldm/cldm_ctrlora_finetune.py:67-82) -> autograd backward -> DDP all-reduce ->
AdamW over {lora_layer.*, zero_convs.*, middle_block_out.*, *norm*} (cldm_ctrlora_finetune.py:84-108).

What is computed (SURVEY.md §0.7): the reference back-propagates weight gradients for every requires_grad parameter it
reaches (385 M ControlNet + UNet decoder weights it never uses).  Here only what the optimizer's parameter set needs:
  * activation gradients through the UNet decoder (frozen) -> the 13 control residuals,
  * activation gradients through the ControlNet,
  * weight gradients for LoRA down/up (factored: dUp = dY^T (X Down^T), dDown = (dY Up)^T X), zero-convs, and the
    'norm'-named GroupNorm / LayerNorm affine parameters.
The reference's activation checkpointing (util.py:102-151) is replaced by simply keeping the activations (they fit the 80 GB of an H100).
The M = batch time-embedding MLP (time_embed, emb_layers: 12 tiny LoRA linears) is differentiated with torch fp32
matmuls on [B, 1280] tensors -- negligible work, documented in DESIGN.md.

Gradient accumulation (the train scripts' --gradacc, Lightning's accumulate_grad_batches = k): step() takes one
micro-batch; k calls form a window whose gradients add into the flat buffer and are exchanged once, by the last
micro-batch, before one AdamW step with grad_scale 1 / (world * loss scale * k).  flush() applies a partial window.
"""
import numbers
import os

import torch
import torch.nn as nn

from . import checkpoint, ops, prepare
from .runtime import nchw_view, pixel_major, to_f16_rows

f32 = prepare.bias_f32


# ------------------------------------------------------------------------------------------------ gradient sink
class GradSink:
    """Flat fp32 buffers (params, grads, Adam moments) over an optimizer's parameter set.

    Default set: the finetune filter in the reference's order (cldm_ctrlora_finetune.py:88-100).  `named` overrides it
    (PretrainSink).  Conv weights are STORED in the kernels' [Cout, kh, kw, Cin] order -- the nn.Parameter keeps its
    reference shape [Cout, Cin, kh, kw] as a permuted view of that storage -- so the dense weight-gradient GEMM writes its
    [Cout, taps*Cin] result straight into the gradient buffer and the fp16 kernel copy is a plain cast; AdamW and the
    all-reduce are elementwise over the flat buffers and never see the difference."""

    def __init__(self, control_model, named=None):
        if named is None:
            from cldm.cldm_ctrlora_finetune import trainable_parameters
            if not getattr(control_model, "ft_with_lora", True):
                # full-ControlNet finetuning selects every parameter (cldm_ctrlora_finetune.py:101-104): that is the
                # dense-gradient trainer's job -- this sink's backward would leave conv/linear gradients at zero
                raise NotImplementedError("FinetuneTrainer covers ft_with_lora=True; use PretrainTrainer (dense weight "
                                          "gradients of every ControlNet parameter) for full-parameter training")
            named = trainable_parameters(control_model)
        self.names = [n for n, _ in named]
        self.params = [p for _, p in named]
        total = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat_p = torch.empty(total, device=dev, dtype=torch.float32)
        self.flat_g = torch.zeros(total, device=dev, dtype=torch.float32)
        self.exp_avg = torch.zeros_like(self.flat_g)
        self.exp_avg_sq = torch.zeros_like(self.flat_g)
        self._grad, self._api_grad, self.offsets = {}, {}, {}
        off = 0
        for name, p in zip(self.names, self.params):
            n = p.numel()
            seg_p, seg_g = self.flat_p[off:off + n], self.flat_g[off:off + n]
            if p.dim() == 4:
                co, ci, kh, kw = p.shape
                seg_p.view(co, kh, kw, ci).copy_(p.detach().permute(0, 2, 3, 1))
                p.data = seg_p.view(co, kh, kw, ci).permute(0, 3, 1, 2)   # reference shape, kernel-order storage
                self._grad[id(p)] = seg_g.view(co, kh * kw * ci)
                self._api_grad[id(p)] = seg_g.view(co, kh, kw, ci).permute(0, 3, 1, 2)
            else:
                seg_p.copy_(p.detach().reshape(-1))
                p.data = seg_p.view(p.shape)  # the module now reads the flat buffer
                self._grad[id(p)] = self._api_grad[id(p)] = seg_g.view(p.shape)
            p._ctrlora_trainable = True
            self.offsets[name] = (off, n)
            off += n
        self.numel = total
        prepare.bump_struct_version()  # parameter storages were re-pointed into the flat buffer

    def grad(self, param):
        """fp32 gradient view of a trainable parameter in STORAGE order (conv weights: [Cout, taps*Cin]), or None if the
        optimizer does not own it."""
        return self._grad.get(id(param)) if param is not None else None

    def named_grads(self):
        """{name: gradient} in the parameters' reference shapes"""
        return {n: self._api_grad[id(p)] for n, p in zip(self.names, self.params)}

    def zero(self):
        self.flat_g.zero_()


# ------------------------------------------------------------------------------------------------ weights
def _cache(mod):
    c = mod.__dict__.get("_tprep")
    if c is None:
        c = mod.__dict__["_tprep"] = prepare.PrepCache()
    return c


def lin_w(lin):
    return _cache(lin).get(("w", prepare.lora_key(lin)), prepare.linear_params(lin), lambda: prepare.effective_linear_weight(lin))


def lin_wT(lin):
    return _cache(lin).get(("wT", prepare.lora_key(lin)), prepare.linear_params(lin), lambda: prepare.weight_T(lin_w(lin)))


def cat_w(owner, key, lins):
    """the stacked [sum N, 1, K] weight of projections that share their input (q|k|v, k|v): each effective weight is
    produced straight into its row range"""
    params = [p for l in lins for p in prepare.linear_params(l)]

    def build():
        ns = [l.weight.shape[0] for l in lins]
        k = lins[0].weight.shape[1]
        out = torch.empty((sum(ns), 1, k), device=lins[0].weight.device, dtype=torch.float16)
        o = 0
        for l, n in zip(lins, ns):
            prepare.effective_linear_weight(l, out=out[o:o + n])
            o += n
        return out

    return _cache(owner).get((key, prepare.lora_key(*lins)), params, build)


def cat_wT(owner, key, lins):
    params = [p for l in lins for p in prepare.linear_params(l)]
    return _cache(owner).get((key + "T", prepare.lora_key(*lins)), params, lambda: prepare.weight_T(cat_w(owner, key, lins)))


def conv_w(conv):
    return _cache(conv).get("w", [conv.weight], lambda: prepare.conv_weight(conv.weight))


def conv_wd(conv):
    """data-gradient weight of a 'same' conv ([Cin, taps flipped, Cout]); for 1x1 convs it is the transpose"""
    return _cache(conv).get("wd", [conv.weight], lambda: prepare.conv_dgrad_weight(conv_w(conv)))


def lora_grads(lin, x2d, dy2d, G):
    """Accumulate dUp, dDown of a LoRACompatibleLinear (y = x W^T + up(down(x))): cldm/lora.py:70-80,285-291."""
    if G is None:
        return
    lora = getattr(lin, "lora_layer", None)
    if lora is None:
        return
    g_up, g_down = G.grad(lora.up.weight), G.grad(lora.down.weight)
    if g_up is None:
        return
    scale = 1.0 if lora.network_alpha is None else lora.network_alpha / lora.rank
    r, k = lora.down.weight.shape
    n = lora.up.weight.shape[0]
    rp = (r + 7) // 8 * 8  # the token-major operands need 16-byte rows: ranks that are not a multiple of 8 are zero-padded
    c = _cache(lora)

    def padded(w16, rows):  # fp16 [r, 1, cols] -> [rp, 1, cols] with zero rows
        if rp == r:
            return w16
        out = ops.zeros((rp, 1, rows), w16.device)
        out[:r].copy_(w16)
        return out

    d16 = c.get("d16", [lora.down.weight], lambda: padded(prepare.linear_weight(lora.down.weight), k))                       # [rp, 1, K]
    u16t = c.get("u16t", [lora.up.weight], lambda: padded(ops.cast_transpose(f32(lora.up.weight), 1, n, r).view(r, 1, n), n))  # [rp, 1, N]
    t1 = ops.gemm(x2d, d16)        # X Down^T   [M, rp]
    t2 = ops.gemm(dy2d, u16t)      # dY Up      [M, rp]
    if rp == r:
        ops.wgrad_tn(dy2d, t1, out=g_up, alpha=scale, beta=1.0)
        ops.wgrad_tn(t2, x2d, out=g_down, alpha=scale, beta=1.0)
    else:
        tmp_up = ops.wgrad_tn(dy2d, t1, alpha=scale)             # [N, rp]: columns r.. are zero
        ops.copy2d(tmp_up, g_up, n, r, rp, r, accumulate=True)
        tmp_down = ops.wgrad_tn(t2, x2d, alpha=scale)            # [rp, K]: rows r.. are zero
        ops.copy2d(tmp_down, g_down, r, k, k, k, accumulate=True)


def dense_lin_grads(lin, x2d, dy2d, G):
    """Dense dW = dY^T X and db = colsum(dY) of an nn.Linear when the optimizer owns them (pretraining: every ControlNet
    parameter, cldm_ctrlora_pretrain.py:174-182); no-op for the finetune set."""
    if G is None:
        return
    gw = G.grad(lin.weight)
    if gw is not None:
        ops.wgrad_tn(dy2d, x2d, out=gw, beta=1.0)
    gb = G.grad(getattr(lin, "bias", None))
    if gb is not None:
        ops.colsum(dy2d, gb)


def lin_grads(lin, x2d, dy2d, G):
    lora_grads(lin, x2d, dy2d, G)
    dense_lin_grads(lin, x2d, dy2d, G)


def dense_conv_grads(conv, xp, dyp, G, col=None):
    """Dense weight / bias gradients of a conv whose (pixel-major fp16) input was xp and output gradient is dyp.
    3x3: dW[Cout, tap, Cin] = dY^T im2col(x) -- exactly the gradient buffer's storage order (GradSink); 1x1: dY^T X.
    `col`: the already gathered operand (stride-2 Downsample keeps its forward gather)."""
    if G is None:
        return
    gw = G.grad(conv.weight)
    if gw is not None:
        b, h, w, co = dyp.shape
        d2d = dyp.reshape(b * h * w, co)
        if col is None:
            if conv.kernel_size[0] == 1:
                col = xp.reshape(b * h * w, -1)
            else:
                col = ops.im2col_3x3(xp.contiguous()).view(b * h * w, -1)
        else:
            col = col.reshape(b * h * w, -1)
        cin_store = gw.shape[1] // (conv.kernel_size[0] * conv.kernel_size[1])
        cin_x = col.shape[1] // (conv.kernel_size[0] * conv.kernel_size[1])
        if cin_x == cin_store:
            ops.wgrad_tn(d2d, col, out=gw, beta=1.0)
        else:  # channel-padded input (the 4-channel latent conv runs on 8): drop the padding columns
            tmp = ops.wgrad_tn(d2d, col)
            taps = conv.kernel_size[0] * conv.kernel_size[1]
            ops.copy2d(tmp, gw, co * taps, cin_store, cin_x, cin_store, accumulate=True)
    gb = G.grad(conv.bias)
    if gb is not None:
        ops.colsum(dyp.reshape(-1, dyp.shape[-1]), gb)


# ------------------------------------------------------------------------------------------------ transformer block
def tblock_fwd(blk, x2d, batch, n, ctx2d, nk):
    dev = x2d.device
    h16 = torch.float16
    a1m, a2m, ff = blk.attn1, blk.attn2, blk.ff
    inner = a1m.to_q.out_features
    heads, d = a1m.heads, inner // a1m.heads
    s = {"x": x2d, "batch": batch, "n": n, "nk": nk, "ctx": ctx2d}
    ln = lambda norm, t: ops.layernorm(t, f32(prepare.effective(norm).weight), f32(prepare.effective(norm).bias), norm.eps)
    # ---- self attention
    s["n1"] = n1 = ln(blk.norm1, x2d)
    np1 = (n + 7) // 8 * 8
    q = torch.empty((batch * n, inner), device=dev, dtype=h16)
    k, v = torch.empty_like(q), torch.empty_like(q)
    vt = torch.empty((batch, heads, d, np1), device=dev, dtype=h16)
    ops.gemm(n1, cat_w(a1m, "qkv", [a1m.to_q, a1m.to_k, a1m.to_v]), seg_outs=[q, k, vt], seg_width=inner, transposed=(0, 0, 1),
             rows_per_img=n, head_dim=d, tok_pad=np1, dup_out=v)
    s["lse1"] = torch.empty((batch, heads, n), device=dev, dtype=torch.float32)
    s["q1"], s["k1"], s["v1"] = q, k, v
    s["a1"] = ops.attention(q, k, vt, batch, heads, n, n, d, lse=s["lse1"])
    o1 = a1m.to_out[0]
    s["x1"] = x1 = ops.gemm(s["a1"], lin_w(o1), bias=f32(o1.bias), residual=x2d)
    # ---- cross attention
    s["n2"] = n2 = ln(blk.norm2, x1)
    npk = (nk + 7) // 8 * 8
    s["q2"] = ops.gemm(n2, lin_w(a2m.to_q))
    k2 = torch.empty((batch * nk, inner), device=dev, dtype=h16)
    v2 = torch.empty_like(k2)
    vt2 = ops.zeros((batch, heads, d, npk), dev) if npk != nk else torch.empty((batch, heads, d, npk), device=dev, dtype=h16)  # finite key padding
    ops.gemm(ctx2d, cat_w(a2m, "kv", [a2m.to_k, a2m.to_v]), seg_outs=[k2, vt2], seg_width=inner, transposed=(0, 1, 0),
             rows_per_img=nk, head_dim=d, tok_pad=npk, dup_out=v2)
    s["k2"], s["v2"] = k2, v2
    s["lse2"] = torch.empty((batch, heads, n), device=dev, dtype=torch.float32)
    s["a2"] = ops.attention(s["q2"], k2, vt2, batch, heads, n, nk, d, lse=s["lse2"])
    o2 = a2m.to_out[0]
    s["x2"] = x2 = ops.gemm(s["a2"], lin_w(o2), bias=f32(o2.bias), residual=x1)
    # ---- feed forward (GEGLU pre-activations are kept for the backward)
    s["n3"] = n3 = ln(blk.norm3, x2)
    proj, out = ff.net[0].proj, ff.net[2]
    s["h"] = h = ops.gemm(n3, lin_w(proj), bias=f32(proj.bias))
    s["g"] = g = ops.geglu_fwd(h)
    x3 = ops.gemm(g, lin_w(out), bias=f32(out.bias), residual=x2)
    return x3, s


def tblock_bwd(blk, s, d_x3, G):
    a1m, a2m, ff = blk.attn1, blk.attn2, blk.ff
    inner = a1m.to_q.out_features
    heads, d = a1m.heads, inner // a1m.heads
    batch, n, nk, ctx2d = s["batch"], s["n"], s["nk"], s["ctx"]

    def ln_bwd(norm, x, dy, res):
        m = prepare.effective(norm)
        gw, gb = (G.grad(m.weight), G.grad(m.bias)) if G is not None else (None, None)
        return ops.layernorm_bwd(x, dy, f32(m.weight), norm.eps, gw, gb, res=res)

    proj, out = ff.net[0].proj, ff.net[2]
    d_g = ops.gemm(d_x3, lin_wT(out))
    lin_grads(out, s["g"], d_x3, G)
    d_h = ops.geglu_bwd(s["h"], d_g)
    d_n3 = ops.gemm(d_h, lin_wT(proj))
    lin_grads(proj, s["n3"], d_h, G)
    d_x2 = ln_bwd(blk.norm3, s["x2"], d_n3, d_x3)
    # ---- cross attention
    o2 = a2m.to_out[0]
    d_a2 = ops.gemm(d_x2, lin_wT(o2))
    lin_grads(o2, s["a2"], d_x2, G)
    dq2, dk2, dv2 = ops.attention_bwd(s["q2"], s["k2"], s["v2"], s["a2"], d_a2, s["lse2"], batch, heads, n, nk, d)
    d_n2 = ops.gemm(dq2, lin_wT(a2m.to_q))
    lin_grads(a2m.to_q, s["n2"], dq2, G)
    lin_grads(a2m.to_k, ctx2d, dk2, G)
    lin_grads(a2m.to_v, ctx2d, dv2, G)
    d_x1 = ln_bwd(blk.norm2, s["x1"], d_n2, d_x2)
    # ---- self attention
    o1 = a1m.to_out[0]
    d_a1 = ops.gemm(d_x1, lin_wT(o1))
    lin_grads(o1, s["a1"], d_x1, G)
    dqkv = torch.empty((batch * n, 3 * inner), device=d_x3.device, dtype=torch.float16)
    ops.attention_bwd(s["q1"], s["k1"], s["v1"], s["a1"], d_a1, s["lse1"], batch, heads, n, n, d, dq=dqkv[:, :inner],
                      dk=dqkv[:, inner:2 * inner], dv=dqkv[:, 2 * inner:])
    d_n1 = ops.gemm(dqkv, cat_wT(a1m, "qkv", [a1m.to_q, a1m.to_k, a1m.to_v]))
    lin_grads(a1m.to_q, s["n1"], dqkv[:, :inner], G)
    lin_grads(a1m.to_k, s["n1"], dqkv[:, inner:2 * inner], G)
    lin_grads(a1m.to_v, s["n1"], dqkv[:, 2 * inner:], G)
    return ln_bwd(blk.norm1, s["x"], d_n1, d_x1)


# ------------------------------------------------------------------------------------------------ spatial transformer
def st_fwd(st, x, ctx):
    xp = pixel_major(x)
    b, h, w, c = xp.shape
    gn = prepare.effective(st.norm)
    xn, stats = ops.groupnorm(xp, f32(gn.weight), f32(gn.bias), gn.eps, False, groups=gn.num_groups, want_stats=True)
    y = ops.gemm(xn, conv_w(st.proj_in), bias=f32(st.proj_in.bias))
    y2d = y.view(b * h * w, -1)
    ctx2d, nk = to_f16_rows(ctx), ctx.shape[1]
    blocks = []
    for blk in st.transformer_blocks:
        y2d, bs = tblock_fwd(blk, y2d, b, h * w, ctx2d, nk)
        blocks.append(bs)
    out = ops.gemm(y2d.view(b, h, w, -1), conv_w(st.proj_out), bias=f32(st.proj_out.bias), residual=xp.view(b * h * w, c))
    return nchw_view(out), {"xp": xp, "stats": stats, "blocks": blocks, "shape": (b, h, w, c), "xn": xn, "y_last": y2d}


def st_bwd(st, s, d_out, G):
    b, h, w, c = s["shape"]
    dop = pixel_major(d_out)
    dense_conv_grads(st.proj_out, s["y_last"].view(b, h, w, -1), dop, G)
    d_y = ops.gemm(dop, conv_wd(st.proj_out)).view(b * h * w, -1)
    for blk, bs in zip(reversed(st.transformer_blocks), reversed(s["blocks"])):
        d_y = tblock_bwd(blk, bs, d_y, G)
    dense_conv_grads(st.proj_in, s["xn"], d_y.view(b, h, w, -1), G)
    d_xn = ops.gemm(d_y.view(b, h, w, -1), conv_wd(st.proj_in))
    gn = prepare.effective(st.norm)
    gw, gb = (G.grad(gn.weight), G.grad(gn.bias)) if G is not None else (None, None)
    dx = ops.groupnorm_bwd(d_xn, s["stats"], s["xp"], f32(gn.weight), f32(gn.bias), gn.eps, False, groups=gn.num_groups,
                           dgamma=gw, dbeta=gb, res=dop.view(b * h * w, c))
    return nchw_view(dx)


# ------------------------------------------------------------------------------------------------ res block
def res_fwd(rb, x, rowbias):
    """x: NCHW-view tensor or runtime.CatSpec; rowbias: fp32 [B, Cout] slice of the network's emb GEMV."""
    from .runtime import CatSpec
    gn1, conv1, gn2, conv2 = rb.in_layers[0], rb.in_layers[2], rb.out_layers[0], rb.out_layers[3]
    skip = None if isinstance(rb.skip_connection, nn.Identity) else rb.skip_connection
    s = {}
    if isinstance(x, CatSpec):
        src = dict(x1=pixel_major(x.x1), add1=None if x.add1 is None else pixel_major(x.add1), add1_scale=x.s1,
                   x2=None if x.x2 is None else pixel_major(x.x2), add2=None if x.add2 is None else pixel_major(x.add2),
                   add2_scale=x.s2)
        a, xp, stats1 = ops.groupnorm(src["x1"], f32(gn1.weight), f32(gn1.bias), gn1.eps, True, add1=src["add1"],
                                      add1_scale=x.s1, x2=src["x2"], add2=src["add2"], add2_scale=x.s2, want_raw=True,
                                      want_stats=True)
    else:
        xp = pixel_major(x)
        src = dict(x1=xp, add1=None, add1_scale=1.0, x2=None, add2=None, add2_scale=1.0)
        a, stats1 = ops.groupnorm(xp, f32(gn1.weight), f32(gn1.bias), gn1.eps, True, want_stats=True)
    b, h, w, cin = xp.shape
    hmid = ops.gemm(a, conv_w(conv1), ksize=3, bias=f32(conv1.bias), rowbias=rowbias)
    c, stats2 = ops.groupnorm(hmid, f32(gn2.weight), f32(gn2.bias), gn2.eps, True, want_stats=True)
    if skip is not None:
        wsk = _cache(skip).get("w2d", [skip.weight], lambda: prepare.conv_weight(skip.weight).view(rb.out_channels, cin))
        bsum = _cache(rb).get("bsum", [conv2.bias, skip.bias], lambda: (conv2.bias.float() + skip.bias.float()).contiguous())
        out = ops.gemm(c, conv_w(conv2), ksize=3, bias=bsum, a2=xp, w2=wsk)
    else:
        out = ops.gemm(c, conv_w(conv2), ksize=3, bias=f32(conv2.bias), residual=xp.view(b * h * w, cin))
    s.update(src=src, stats1=stats1, hmid=hmid, stats2=stats2, shape=(b, h, w, cin), a=a, c=c, xp=xp)
    return nchw_view(out), s


def res_bwd(rb, s, d_out, rowbias_grad=None, want_dx2=False, dx1_scale=1.0, G=None):
    """Returns dx1 (times dx1_scale) and, if want_dx2, the gradient of the second concat half times its add2_scale."""
    gn1, conv1, gn2, conv2 = rb.in_layers[0], rb.in_layers[2], rb.out_layers[0], rb.out_layers[3]
    skip = None if isinstance(rb.skip_connection, nn.Identity) else rb.skip_connection
    b, h, w, cin = s["shape"]
    dop = pixel_major(d_out)
    if G is not None:  # dense conv gradients + GroupNorm affine gradients (pretraining owns them; the finetune set owns
        # neither: ResBlock norms are named in_layers.0 / out_layers.0, which the 'norm' filter does not match)
        dense_conv_grads(conv2, s["c"], dop, G)
        if skip is not None:
            gw = G.grad(skip.weight)
            if gw is not None:
                ops.wgrad_tn(dop.reshape(b * h * w, -1), s["xp"].reshape(b * h * w, cin), out=gw, beta=1.0)
            # conv2.bias and skip.bias receive the same gradient (their sum is the fused epilogue bias)
            gb = G.grad(skip.bias)
            if gb is not None:
                ops.colsum(dop.reshape(b * h * w, -1), gb)
    d_c = ops.gemm(dop, conv_wd(conv2), ksize=3)
    d_skip = ops.gemm(dop, conv_wd(skip)).view(b * h * w, cin) if skip is not None else dop.view(b * h * w, cin)
    g2w, g2b = (G.grad(gn2.weight), G.grad(gn2.bias)) if G is not None else (None, None)
    d_hmid = ops.groupnorm_bwd(d_c, s["stats2"], s["hmid"], f32(gn2.weight), f32(gn2.bias), gn2.eps, True, dgamma=g2w, dbeta=g2b)
    if rowbias_grad is not None:
        ops.image_colsum(d_hmid.view(b * h * w, -1), b, rowbias_grad)
    if G is not None:
        dense_conv_grads(conv1, s["a"], d_hmid, G)
    d_a = ops.gemm(d_hmid, conv_wd(conv1), ksize=3)
    src = s["src"]
    g1w, g1b = (G.grad(gn1.weight), G.grad(gn1.bias)) if G is not None else (None, None)
    res = ops.groupnorm_bwd(d_a, s["stats1"], src["x1"], f32(gn1.weight), f32(gn1.bias), gn1.eps, True, add1=src["add1"],
                            add1_scale=src["add1_scale"], x2=src["x2"], add2=src["add2"], add2_scale=src["add2_scale"],
                            want_dx2=want_dx2, dx2_scale=src["add2_scale"], res=d_skip, dx1_scale=dx1_scale,
                            dgamma=g1w, dbeta=g1b)
    if want_dx2:
        return nchw_view(res[0]), nchw_view(res[1])
    return nchw_view(res)


# ------------------------------------------------------------------------------------------------ resampling
def down_fwd(ds, x):
    xp = pixel_major(x).contiguous()
    b, h, w, c = xp.shape
    col = ops.im2col_s2(xp)
    wk = _cache(ds).get("w", [ds.op.weight], lambda: prepare.conv_weight(ds.op.weight).view(ds.out_channels, 1, 9 * c))
    return nchw_view(ops.gemm(col, wk, bias=f32(ds.op.bias))), {"shape": (b, h, w, c), "col": col}


def down_bwd(ds, s, d_out, G=None):
    b, h, w, c = s["shape"]
    if G is not None:
        dense_conv_grads(ds.op, None, pixel_major(d_out), G, col=s["col"])
    # builders read their inputs through the caches (never a tensor fetched earlier): a recorded builder re-run inside a
    # preparation graph (FinetuneTrainer._capture_prep) must derive from the current parameters
    wk = lambda: _cache(ds).get("w", [ds.op.weight], lambda: prepare.conv_weight(ds.op.weight).view(ds.out_channels, 1, 9 * c))
    wt = _cache(ds).get("wT", [ds.op.weight], lambda: prepare.weight_T(wk()))
    d_col = ops.gemm(pixel_major(d_out), wt)  # [B, h/2, w/2, 9*C]
    return nchw_view(ops.im2col_s2_bwd(d_col, h, w))


def up_fwd(us, x):
    up = ops.upsample2x(pixel_major(x).contiguous())
    return nchw_view(ops.gemm(up, conv_w(us.conv), ksize=3, bias=f32(us.conv.bias))), {}


def up_bwd(us, s, d_out):
    d_up = ops.gemm(pixel_major(d_out), conv_wd(us.conv), ksize=3)
    return nchw_view(ops.upsample2x_bwd(d_up))


# ------------------------------------------------------------------------------------------------ block sequences
def seq_fwd(seq, x, emb, ctx):
    """TimestepEmbedSequential in training mode: returns (out, tape) with one (kind, module, saved) per child."""
    from ldm.modules.attention import SpatialTransformer
    from ldm.modules.diffusionmodules.openaimodel import Downsample, ResBlock, Upsample, _Conv
    tape = []
    for layer in seq:
        if isinstance(layer, ResBlock):
            x, s = res_fwd(layer, x, emb.slices[id(layer)])
            tape.append(("res", layer, s))
        elif isinstance(layer, SpatialTransformer):
            x, s = st_fwd(layer, x, ctx)
            tape.append(("st", layer, s))
        elif isinstance(layer, Downsample):
            x, s = down_fwd(layer, x)
            tape.append(("down", layer, s))
        elif isinstance(layer, Upsample):
            x, s = up_fwd(layer, x)
            tape.append(("up", layer, s))
        elif isinstance(layer, _Conv):
            cin = layer.in_channels
            c_pad = (cin + 7) // 8 * 8
            xin = pixel_major(x, c_pad if c_pad != cin else None)
            x = layer(nchw_view(xin))  # the 4-channel input conv: nothing upstream needs its data gradient
            tape.append(("stop", layer, {"xin": xin}))
        else:
            raise NotImplementedError(type(layer))
    return x, tape


def seq_bwd(tape, d, G, emb_grads=None, first_res_kw=None):
    """Backward through one block; returns the input gradient (or a tuple for a CatSpec-fed first ResBlock)."""
    for i in range(len(tape) - 1, -1, -1):
        kind, mod, s = tape[i]
        if kind == "res":
            kw = first_res_kw if (i == 0 and first_res_kw) else {}
            rg = emb_grads.get(id(mod)) if emb_grads is not None else None
            d = res_bwd(mod, s, d, rowbias_grad=rg, G=G, **kw)
        elif kind == "st":
            d = st_bwd(mod, s, d, G)
        elif kind == "down":
            d = down_bwd(mod, s, d, G)
        elif kind == "up":
            d = up_bwd(mod, s, d)
        elif kind == "stop":
            if G is not None:
                dense_conv_grads(mod, s["xin"], pixel_major(d), G)
            return None
    return d


# ------------------------------------------------------------------------------------------------ time-embedding MLP
def _small_lora_grads(lin, x, dy, G, silu_x=False):
    """LoRA (and, when owned, dense) gradients of a linear whose 'token' dimension is the batch: fp32 [B, K] input x
    (SiLU applied on the fly when silu_x), fp32 [B, N] output gradient dy.  cldm/lora.py:70-80,285-291."""
    gw, gb = G.grad(lin.weight), G.grad(getattr(lin, "bias", None))
    if gw is not None:
        ops.outer_accum(dy, x, gw, silu_x=silu_x)
    if gb is not None:
        ops.colsum(dy, gb)
    lora = getattr(lin, "lora_layer", None)
    if lora is None:
        return
    gu, gd = G.grad(lora.up.weight), G.grad(lora.down.weight)
    if gu is None:
        return
    sc = 1.0 if lora.network_alpha is None else lora.network_alpha / lora.rank
    r, k = lora.down.weight.shape
    n = lora.up.weight.shape[0]
    c = _cache(lora)
    d16 = c.get("d16s", [lora.down.weight], lambda: prepare.linear_weight(lora.down.weight).view(r, k))           # [r, K]
    u16t = c.get("u16ts", [lora.up.weight], lambda: ops.cast_transpose(f32(lora.up.weight), 1, n, r).view(r, n))  # [r, N]
    t1 = ops.small_linear(x, d16, None, silu_in=silu_x)      # (f(x)) Down^T  [B, r]
    ops.outer_accum(dy, t1, gu, alpha=sc)                    # dUp   += sc * dY^T (X Down^T)
    t2 = ops.small_linear(dy, u16t, None)                    # dY Up          [B, r]
    ops.outer_accum(t2, x, gd, alpha=sc, silu_x=silu_x)      # dDown += sc * (dY Up)^T X


def emb_mlp_backward(net, t_emb, emb, d_all, slices, G):
    """Backward of timestep_embedding -> time_embed (Linear, SiLU, Linear) -> every ResBlock's emb_layers (SiLU, Linear)
    (openaimodel.py:526-531, :208-215; LoRA-wrapped in the ControlNet) from d_all = d(rowbias) [B, sum Cout] (fp32; slices =
    {id(resblock): column view}).  M = batch rows: GEMV-shaped work on the small_linear / outer-product kernels."""
    from ldm.modules.diffusionmodules.openaimodel import ResBlock
    blocks = [m for m in net.modules() if isinstance(m, ResBlock)]
    l0, l2 = net.time_embed[0], net.time_embed[2]
    # weight / LoRA gradients of the emb_layers: input silu(emb), output gradient = the block's slice
    for rb in blocks:
        _small_lora_grads(rb.emb_layers[1], emb, slices[id(rb)], G, silu_x=True)
    # d silu(emb) = d_all @ Wcat  (the forward's batched [sum Cout, 1280] matrix, transposed once per weight version)
    lins = [b.emb_layers[1] for b in blocks]
    params = [p for lin in lins for p in prepare.linear_params(lin)]
    wcat_t = _cache(net).get("emb_cat_T", params, lambda: prepare.weight_T(
        torch.cat([b.emb_weight() for b in blocks], 0).contiguous().view(-1, 1, l2.out_features)).view(l2.out_features, -1))
    d_se = ops.small_linear(d_all, wcat_t, None)
    d_emb = ops.silu_bwd(d_se, emb)
    # time_embed.2: input hid = silu(hid_pre)
    w0 = _cache(l0).get("w2d", prepare.linear_params(l0), lambda: prepare.effective_linear_weight(l0).view(l0.out_features, -1))
    hid_pre = ops.small_linear(t_emb, w0, f32(l0.bias))
    _small_lora_grads(l2, hid_pre, d_emb, G, silu_x=True)
    w2t = _cache(l2).get("w2dT", prepare.linear_params(l2), lambda: prepare.weight_T(
        prepare.effective_linear_weight(l2)).view(l2.in_features, l2.out_features))
    d_hid = ops.small_linear(d_emb, w2t, None)
    d_hid_pre = ops.silu_bwd(d_hid, hid_pre)
    _small_lora_grads(l0, t_emb, d_hid_pre, G)


# ------------------------------------------------------------------------------------------------ networks
def controlnet_fwd(cn, hint, t, ctx):
    emb = cn.embed(t)
    ctx16 = to_f16_rows(ctx).view(ctx.shape[0], ctx.shape[1], -1)
    tapes, hs, outs = [], [], []
    h = hint
    for module, zc in zip(cn.input_blocks, cn.zero_convs):
        h, tape = seq_fwd(module, h, emb, ctx16)
        tapes.append(tape)
        hs.append(h)
        outs.append(cn._zero_conv(zc, h))
    h, tape = seq_fwd(cn.middle_block, h, emb, ctx16)
    tapes.append(tape)
    hs.append(h)
    outs.append(cn._zero_conv(cn.middle_block_out, h))
    return outs, {"tapes": tapes, "hs": hs, "emb": emb, "t": t}


def zero_conv_bwd(seq, h, d_out, G, upstream):
    """1x1 zero-conv: dW = dY^T H, db = colsum(dY), dH = dY W (+ the gradient arriving from the next block)."""
    conv = prepare.effective(seq[0])
    hp, dp = pixel_major(h), pixel_major(d_out)
    b, hh, ww, c = hp.shape
    h2d, d2d = hp.reshape(b * hh * ww, c), dp.reshape(b * hh * ww, c)
    gw, gb = G.grad(conv.weight), G.grad(conv.bias)
    if gw is not None:
        ops.wgrad_tn(d2d, h2d, out=gw.view(c, c), beta=1.0)
        ops.colsum(d2d, gb)
    wt = _cache(conv).get("wT", [conv.weight], lambda: prepare.weight_T(prepare.conv_weight(conv.weight)))
    up = None if upstream is None else pixel_major(upstream).reshape(b * hh * ww, c)
    return nchw_view(ops.gemm(dp, wt, residual=up))


STAGE_AFTER_BLOCK = {9: "ib9", 6: "ib6", 3: "ib3"}  # backward stages that close a gradient bucket (besides "middle")


def controlnet_bwd(cn, saved, d_outs, G, on_stage=None):
    """Backward through the ControlNet, last block first.  `on_stage(name)` fires when every gradient of a bucket is final
    ("middle": middle_block.*; "ib9"/"ib6"/"ib3": input_blocks 9-11 / 6-8 / 3-5) so the trainer can start that bucket's
    all-reduce while the remaining blocks are still being differentiated."""
    from ldm.modules.diffusionmodules.openaimodel import ResBlock
    emb = saved["emb"]
    bsz = emb.raw.shape[0]
    blocks = [m for m in cn.modules() if isinstance(m, ResBlock)]
    d_all = torch.zeros((bsz, sum(b.out_channels for b in blocks)), device=emb.raw.device, dtype=torch.float32)
    emb_grads, off = {}, 0
    for b in blocks:
        emb_grads[id(b)] = d_all[:, off:off + b.out_channels]
        off += b.out_channels
    tapes, hs = saved["tapes"], saved["hs"]
    d_h = zero_conv_bwd(cn.middle_block_out, hs[-1], d_outs[-1], G, None)
    d_h = seq_bwd(tapes[-1], d_h, G, emb_grads)
    if on_stage is not None:
        on_stage("middle")
    for i in range(len(cn.input_blocks) - 1, -1, -1):
        d_h = zero_conv_bwd(cn.zero_convs[i], hs[i], d_outs[i], G, d_h)
        d_h = seq_bwd(tapes[i], d_h, G, emb_grads)
        if on_stage is not None and i in STAGE_AFTER_BLOCK:
            on_stage(STAGE_AFTER_BLOCK[i])
    from ldm.modules.diffusionmodules.util import timestep_embedding
    t_emb = timestep_embedding(saved["t"], cn.model_channels)
    emb_mlp_backward(cn, t_emb, emb.raw, d_all, emb_grads, G)


def unet_fwd(unet, x, t, ctx, control, scales, only_mid_control=False):
    """ControlledUnetModel.forward (cldm/cldm.py:22-45) with the decoder taped; control: 13 tensors, scales: 13 floats."""
    from .runtime import CatSpec
    with torch.no_grad():
        emb = unet.embed(t)
        ctx16 = to_f16_rows(ctx).view(ctx.shape[0], ctx.shape[1], -1)
        hs = []
        h = x
        for module in unet.input_blocks:
            h = module(h, emb, ctx16)
            hs.append(h)
        h = unet.middle_block(h, emb, ctx16)
    ctrl = list(zip(control, scales))
    add_mid, s_mid = ctrl.pop()
    tapes = []
    for i, module in enumerate(unet.output_blocks):
        skip = hs.pop()
        add, sc = (None, 1.0) if only_mid_control else ctrl.pop()
        spec = CatSpec(h, add1=add_mid if i == 0 else None, s1=s_mid, x2=skip, add2=add, s2=sc)
        h, tape = seq_fwd(module, spec, emb, ctx16)
        tapes.append(tape)
    # out: GroupNorm32 -> SiLU -> conv3x3 (kept on the inference kernels, plus the saved statistics)
    gn, conv = unet.out[0], unet.out[2]
    hp = pixel_major(h)
    a, stats = ops.groupnorm(hp, f32(gn.weight), f32(gn.bias), gn.eps, True, want_stats=True)
    n_pad = (unet.out_channels + 15) // 16 * 16
    bias = unet._prep.get("out_bias", [conv.bias], lambda: torch.cat(
        [conv.bias.detach().float(), torch.zeros(n_pad - unet.out_channels, device=conv.bias.device)]).contiguous())
    y = ops.gemm(a, conv.kernel_weight(pad_out=n_pad), ksize=3, bias=bias, out_f32=True)
    eps = ops.nhwc_to_nchw_f32(y, unet.out_channels)
    return eps, {"tapes": tapes, "hp": hp, "stats": stats, "n_pad": n_pad, "only_mid": only_mid_control}


def unet_bwd(unet, saved, d_eps16):
    """d_eps16: fp16 pixel-major [B,H,W,16] gradient of eps (first 4 channels live).  Returns the 13 control gradients
    (already multiplied by their control_scales), in the ControlNet's output order."""
    gn, conv = unet.out[0], unet.out[2]
    wd = _cache(conv).get("wd_out", [conv.weight],
                          lambda: prepare.conv_dgrad_weight(conv.kernel_weight(pad_out=saved["n_pad"])))  # [320, 9, 16]
    d_a = ops.gemm(d_eps16, wd, ksize=3)
    d_h = nchw_view(ops.groupnorm_bwd(d_a, saved["stats"], saved["hp"], f32(gn.weight), f32(gn.bias), gn.eps, True))
    d_ctrl = []
    tapes = saved["tapes"]
    for i in range(len(tapes) - 1, -1, -1):
        want2 = not saved["only_mid"]
        if i == 0:
            # x1 = h_mid (+ s_mid * c_mid): only the control half of that sum needs a gradient
            src = tapes[0][0][2]["src"]
            res = seq_bwd(tapes[0], d_h, None, None, first_res_kw=dict(want_dx2=want2, dx1_scale=src["add1_scale"]))
        else:
            res = seq_bwd(tapes[i], d_h, None, None, first_res_kw=dict(want_dx2=want2))
        if want2:
            d_h, d2 = res
            d_ctrl.append(d2)
        else:
            d_h = res
    # d_ctrl holds gradients for control[11], ..., control[0] in pop() order reversed: decoder block i consumed control[11 - i]
    d_ctrl = d_ctrl[::-1] if d_ctrl else []  # now index j = decoder block j -> control[11 - j]
    ordered = [None] * 13
    for j, g in enumerate(d_ctrl):
        ordered[11 - j] = g
    ordered[12] = d_h  # scaled by s_mid inside the first decoder block's GroupNorm backward
    return ordered


# ------------------------------------------------------------------------------------------------ trainer
class FinetuneTrainer:
    """One data-parallel CtrLoRA finetune step per call (configs ctrlora_finetune_sd15_rank*.yaml)."""

    tasks = ()  # finetuning trains one LoRA set: no task to switch (PretrainTrainer: the ControlNet's tasks)

    def __init__(self, model, lr=1e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, process_group=None,
                 loss_scale=None, dynamic_loss_scale=True, accumulate_grad_batches=1, *, named=None):
        """named: the optimizer's parameter set, [(name, parameter)] as GradSink takes it; default: the finetune filter"""
        self._init_window(accumulate_grad_batches)
        self.model = model
        self.cn = model.control_model
        self.unet = model.model.diffusion_model
        self.G = GradSink(self.cn, named=named)
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.pg = process_group
        self.world, self.rank = 1, 0
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            self.world = torch.distributed.get_world_size(process_group)
            self.rank = torch.distributed.get_rank(process_group)
        if self.world > 1:
            # DDP's construction-time rank-0 broadcast (the reference relies on it: LoRA `down` is initialised
            # N(0, 1/r) without a seed, cldm/lora.py:67): every replica starts from rank 0's trainable parameters
            torch.distributed.broadcast(self.G.flat_p, src=0, group=process_group)
            prepare.bump_train_version()
        self.step_count = 0
        self.seg_steps = {}        # per-segment AdamW step counts (torch keeps `step` per parameter)
        # Loss scaling (the backward's activation gradients are fp16; the reference trains in fp32 and needs none):
        # d(loss)/d(eps) = 2 (eps - noise) / numel is ~1e-5 at batch 16 x 4 x 64 x 64 -- below fp16's normal range.  The
        # default scale makes it (eps - noise) / LOSS_SCALE_DIV independent of the batch shape; the AdamW kernel divides
        # it out of the fp32 gradient buffer.  `dynamic`: a non-finite gradient skips the update and halves the scale.
        self.loss_scale = loss_scale
        self.dynamic_loss_scale = dynamic_loss_scale
        dev = self.G.flat_p.device
        self.overflow_flag = torch.zeros(1, device=dev, dtype=torch.int32)
        self.skipped_steps = 0
        self._init_step_state(dev)
        self._graphs = None        # capture(): {"prep": {owner: graph}, "compute": {task: (graph(s), loss, scale)}}
        self._static = None        # the captured graphs' inputs
        self._on_stage = None      # backward-stage callback (the overlapped exchange)
        self._comm = None          # stream of the overlapped all-reduces

    LOSS_SCALE_DIV = 8.0
    CHECK_OVERFLOW_EVERY = 16   # host polls the device-side skipped-steps counter this often (no per-step sync)

    def _init_window(self, k):
        """Gradient accumulation (Lightning's accumulate_grad_batches): k consecutive step() calls form one window, one
        optimizer step.  micro_step = micro-batches already in the current window."""
        if isinstance(k, bool) or not isinstance(k, numbers.Integral) or k < 1:
            raise ValueError(f"accumulate_grad_batches must be an integer >= 1, got {k!r}")
        self.accumulate_grad_batches = int(k)
        self.micro_step = 0
        self._window_tasks = []

    def _init_step_state(self, dev):
        """AdamW's step counter lives on the device (ops.adamw_begin): a step skipped for a non-finite gradient does not
        count, and the host does not have to read the overflow flag before it may launch the next step."""
        self._step_dev = {}            # segment key -> int32 [1] step counter
        self._bc_dev = {}              # segment key -> fp32 [2] bias corrections of the current step
        self._skipped_dev = torch.zeros(1, device=dev, dtype=torch.int32)
        self._skipped_seen = 0
        self._launched = 0

    def _seg_state(self, key):
        if key not in self._step_dev:
            dev = self.G.flat_p.device
            self._step_dev[key] = torch.zeros(1, device=dev, dtype=torch.int32)
            self._bc_dev[key] = torch.ones(2, device=dev, dtype=torch.float32)
        return self._step_dev[key], self._bc_dev[key]

    def _poll_overflow(self, force=False):
        """True (after halving the loss scale and re-capturing) if the device skipped steps since the last poll."""
        self._launched += 1
        if not (force or (self.dynamic_loss_scale and self._launched % self.CHECK_OVERFLOW_EVERY == 0)):
            return False
        skipped = int(self._skipped_dev.item())
        if skipped == self._skipped_seen:
            return False
        self.skipped_steps += skipped - self._skipped_seen
        self._skipped_seen = skipped
        self.loss_scale = self._scale_used * 0.5
        return True

    def _scale_for(self, numel):
        return float(self.loss_scale) if self.loss_scale is not None else numel / (2.0 * self.LOSS_SCALE_DIV)

    def loss_and_grads(self, x0, hint_latent, context, t, noise, task=None, accumulate=False):
        """q_sample -> apply_model -> MSE -> backward into the flat gradient buffer.  Returns the loss (fp32 tensor).
        task: the LoRA set to attach first, when the trainer has tasks (None keeps the attached one).
        accumulate: add to the gradients already in the buffer (a continuing micro-batch of a window) and keep the window's
        loss scale and overflow flag; otherwise the buffer and the flag are zeroed first."""
        m = self.model
        if task is not None and self.tasks:
            self.cn.switch_lora(task)
            self.task = task
        if not accumulate:
            self.G.zero()
            self.overflow_flag.zero_()
            self._scale_used = self._scale_for(x0.numel())
        x_noisy = m.q_sample(x_start=x0, t=t, noise=noise)
        control, cn_saved = controlnet_fwd(self.cn, hint_latent, t, context)
        eps, un_saved = unet_fwd(self.unet, x_noisy, t, context, control, m.control_scales, m.only_mid_control)
        loss, d_eps = ops.mse_loss_grad(eps, noise, c_pad=un_saved["n_pad"], grad_scale=self._scale_used)
        d_ctrl = unet_bwd(self.unet, un_saved, d_eps)
        if m.only_mid_control:
            d_ctrl = [d if d is not None else torch.zeros_like(c) for d, c in zip(d_ctrl, control)]
        controlnet_bwd(self.cn, cn_saved, d_ctrl, self.G, on_stage=self._on_stage)
        self.last_eps = eps
        return loss

    def unscaled_grads(self):
        """{name: fp32 gradient} with the loss scale divided out (what the reference's autograd would hold)."""
        inv = 1.0 / self._scale_used
        return {n: g * inv for n, g in self.G.named_grads().items()}

    # -- the exchange step: all-reduce (SUM) of the flat trainable-gradient buffer (36.9 M fp32 elements for rank 128 =
    # 148 MB; the reference's DDP reduces ~10x more, SURVEY.md §0.7), split into buckets that follow the backward's order so
    # all but the last one overlap the remaining ControlNet backward.  1/world is folded into the AdamW kernel.
    STAGES = ("middle",) + tuple(STAGE_AFTER_BLOCK.values())  # backward stages that can close a bucket, in order
    # The active cuts come from the environment variable CUTS_ENV, default CUTS_DEFAULT (_overlap_cuts).  Finetuning:
    # none by default: every cut splits the CUDA graph and the collective's CTAs compete with the backward it overlaps,
    # which pays only for collectives longer than the finetune step's (more ranks, multi-node).
    CUTS_ENV, CUTS_DEFAULT = "CTRLORA_ALLREDUCE_CUTS", ""

    def gradient_buckets(self):
        """{stage: [(offset, numel)]}: contiguous flat-buffer ranges whose gradients are final when the backward reaches
        the stage (a block's zero-conv travels with its block); "final" is the rest: input_blocks.0-2 with their zero-convs and
        the time-embedding MLP -- ~4 M of the 36.9 M elements, the only part whose all-reduce cannot overlap the backward."""
        def stage_of(n):
            # the ResBlocks' emb_layers (and their LoRA layers) get their gradients from emb_mlp_backward, AFTER the last
            # block: they travel in the final bucket whatever block they sit in
            if ".emb_layers." in n:
                return "final"
            # zero_convs.i is differentiated right before input_blocks.i, middle_block_out right before middle_block
            if n.startswith(("middle_block.", "middle_block_out.")):
                return "middle"
            if n.startswith(("input_blocks.", "zero_convs.")):
                i = int(n.split(".")[1])
                for b0, st in STAGE_AFTER_BLOCK.items():
                    if b0 <= i < b0 + 3:
                        return st
            return "final"

        buckets = {k: [] for k in self.STAGES + ("final",)}
        for name in self.G.names:
            off, n = self.G.offsets[name]
            r = buckets[stage_of(name)]
            if r and r[-1][0] + r[-1][1] == off:
                r[-1] = (r[-1][0], r[-1][1] + n)
            else:
                r.append((off, n))
        return buckets

    def _overlap_cuts(self):
        """Backward stages after which a gradient bucket is closed and its all-reduce started, in backward order:
        `allreduce_cuts` when set, else the environment variable CUTS_ENV (default CUTS_DEFAULT); a comma-separated subset
        of middle,ib9,ib6,ib3, empty = one all-reduce after the backward."""
        cuts = getattr(self, "allreduce_cuts", None)
        if cuts is None:
            cuts = os.environ.get(self.CUTS_ENV, self.CUTS_DEFAULT)
        if isinstance(cuts, str):
            cuts = [c for c in cuts.split(",") if c]
        return [c for c in self.STAGES if c in cuts]

    def _segmented(self):
        """the exchange overlaps the backward: one graph per gradient bucket, each bucket reduced after its stage"""
        return self.world > 1 and bool(self._overlap_cuts())

    def merged_buckets(self):
        """[(stage, ranges)] in backward order for the active cuts + ("final", ranges): buckets of skipped stages are merged
        into the next active cut."""
        def coalesce(ranges):
            out = []
            for off, n in sorted(ranges):
                if out and out[-1][0] + out[-1][1] == off:
                    out[-1] = (out[-1][0], out[-1][1] + n)
                else:
                    out.append((off, n))
            return out

        b = self.gradient_buckets()
        cuts, out, pending = self._overlap_cuts(), [], []
        for st in self.STAGES:
            pending += b[st]
            if st in cuts:
                out.append((st, coalesce(pending)))
                pending = []
        out.append(("final", coalesce(pending + b["final"])))
        return out

    def exchange_plan(self, segs, bucket_ranges):
        """Ranges to all-reduce after each backward bucket, for a window's segments `segs` (window_segments): the bucket's
        part of the dense first segment ("all" / "base", at offset 0); the other segments (pretraining's LoRA sets, which
        live behind it in the flat buffer) travel with the LAST bucket.  Every element of `segs` appears exactly once in
        the plan."""
        dense_end = segs[0][1]
        rest = [(off, n) for off, n, _ in segs[1:]]
        plan = []
        for i, ranges in enumerate(bucket_ranges):
            r = [(off, min(n, dense_end - off)) for off, n in ranges if off < dense_end]
            plan.append(r + rest if i == len(bucket_ranges) - 1 else r)
        return plan

    def _reduce_ranges(self, ranges):
        """all-reduce `ranges` on the communication stream once everything enqueued so far on the compute stream is done"""
        if self.world <= 1 or not ranges:
            return
        if self._comm is None:
            self._comm = torch.cuda.Stream()
        ev = torch.cuda.Event()
        ev.record()
        self._comm.wait_event(ev)
        with torch.cuda.stream(self._comm):
            for off, n in ranges:
                torch.distributed.all_reduce(self.G.flat_g[off:off + n], group=self.pg)

    def reduce_gradients(self, ranges=None):
        """Un-overlapped form (also what the CPU/gloo tests drive): one all-reduce per (offset, numel) range, whole buffer
        by default."""
        if self.world > 1:
            for off, n in (ranges or [(0, self.G.numel)]):
                torch.distributed.all_reduce(self.G.flat_g[off:off + n], group=self.pg)

    # -- CUDA-graph replay of forward + backward (≈3 000 launches per step; Python cannot enqueue them fast enough)
    def capture(self, x0, hint_latent, context, t, noise, tasks=None, warmup=2):
        """Capture the step for these shapes: one compute graph per task (`tasks`: default every task of the trainer;
        finetuning's only task is None; the attached LoRA set is baked into the captured kernels' pointers), all in one
        memory pool -- only one of them is ever in flight.  A call replaces everything captured before: the inputs are
        cloned again and the earlier graphs dropped, so a re-capture passes every captured task.
          * k = 1: the trainable-weight copies (LoRA folds, fp16 / transposed / dgrad copies) are rebuilt inside the
            compute graph (they must re-run every step); the frozen-weight copies are built during warm-up and are not.
          * k > 1 (accumulate_grad_batches): the compute graph adds one micro-batch into the buffer, and the trainable
            copies are rebuilt once per window by preparation graphs (_capture_prep).
        A compute graph is one graph, or one per gradient bucket when the exchange overlaps the backward (_segmented)."""
        self._graphs = None
        self._static = [v.clone() for v in (x0, hint_latent, context, t, noise)]
        tasks = list(tasks or self.tasks or [None])
        accumulate = self.accumulate_grad_batches > 1
        cur = torch.cuda.current_stream()
        logs, compute, pool = {}, {}, None

        def capture_compute(task):
            nonlocal pool
            g, loss, pool = self._capture_compute(
                lambda: self.loss_and_grads(*self._static, task=task, accumulate=accumulate), pool)
            compute[task] = (g, loss, self._scale_used)

        for task in tasks:
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                for _ in range(warmup - 1 if accumulate else warmup):
                    self.loss_and_grads(*self._static, task=task)
                if accumulate:  # which copies a micro-batch reads, for the preparation graphs
                    prepare.bump_train_version()
                    with prepare.record_builds() as logs[task]:
                        self.loss_and_grads(*self._static, task=task)
            cur.wait_stream(side)
            if not accumulate:
                torch.cuda.synchronize()
                prepare.bump_train_version()  # force the trainable-weight preparation into the captured region
                capture_compute(task)
        prep = {}
        if accumulate:
            torch.cuda.synchronize()
            prep = self._capture_prep(tasks, logs)
            for task in tasks:
                capture_compute(task)
        self._graphs = {"prep": prep, "compute": compute}
        return self

    def _capture_prep(self, tasks, logs):
        """Preparation graphs of the accumulating path, from the copies each task's warm-up read (`logs`):
          * prep[None]: zero the gradient buffer and the overflow flag, rebuild every trainable-weight copy that does not
            depend on a task's LoRA set -- replayed at a window's start;
          * prep[task] (pretraining): rebuild the copies that depend on the task's LoRA set -- replayed on the task's first
            micro-batch in a window (a window mixes tasks, so not every fold can be built at its start).
        Each has a memory pool of its own, so no other graph's scratch can overwrite the copies it keeps."""
        builds, seen = {None: []}, set()
        for task in tasks:
            own = {id(p) for n, p in zip(self.G.names, self.G.params) if n.startswith(f"loras_dict.{task}.")}
            builds.setdefault(task, [])
            for entry in logs[task]:
                cache, key, params, _ = entry
                ps = [p for p in params if p is not None]
                if not any(getattr(p, "_ctrlora_trainable", False) for p in ps):
                    continue  # frozen copies are built once and never change
                owner = task if any(id(p) in own for p in ps) else None
                if (owner, id(cache), key) not in seen:
                    seen.add((owner, id(cache), key))
                    builds[owner].append(entry)

        prepare.bump_train_version()  # every recorded copy is rebuilt inside its prep graph
        prep = {}
        for owner, entries in builds.items():
            if owner is not None and not entries:
                continue
            if owner is not None:
                self.cn.switch_lora(owner)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                if owner is None:
                    self.G.zero()
                    self.overflow_flag.zero_()
                for cache, key, params, builder in entries:
                    cache.get(key, params, builder)
            prep[owner] = g
        return prep

    def _capture_compute(self, run, pool):
        """graph of run() in `pool`; one graph per gradient bucket when _segmented()"""
        kw = {} if pool is None else {"pool": pool}
        if not self._segmented():
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, **kw):
                loss = run()
            return g, loss, g.pool() if pool is None else pool
        # replay k, start bucket k's all-reduce on the communication stream, replay k+1 ... (NCCL stays outside the
        # captures)
        buckets = dict(self.merged_buckets())
        cur = torch.cuda.current_stream()
        segs, state = [], {"pool": pool}
        stream = torch.cuda.Stream()
        stream.wait_stream(cur)
        with torch.cuda.stream(stream):
            state["g"] = torch.cuda.CUDAGraph()
            state["g"].capture_begin(**kw)

            def on_stage(name):
                if name not in buckets:
                    return  # not an active cut
                state["g"].capture_end()
                state["pool"] = state["pool"] or state["g"].pool()
                segs.append((state["g"], buckets[name]))
                self._after_cut()
                state["g"] = torch.cuda.CUDAGraph()
                state["g"].capture_begin(pool=state["pool"])

            self._on_stage = on_stage
            try:
                loss = run()
            finally:
                self._on_stage = None
                ops.set_sm_limit(0)
            state["g"].capture_end()
            state["pool"] = state["pool"] or state["g"].pool()
            segs.append((state["g"], buckets["final"]))
        cur.wait_stream(stream)
        return segs, loss, state["pool"]

    def _after_cut(self):
        """hook while capturing the segments that follow a bucket cut (they run next to the bucket's all-reduce)"""

    def step(self, x0, hint_latent, context, t, noise):
        """One micro-batch; every accumulate_grad_batches-th call also exchanges the gradients and runs AdamW.  Returns
        this micro-batch's loss (its own mean, not divided by k)."""
        return self._micro_batch((x0, hint_latent, context, t, noise), None)

    def _update(self, segs):
        """Overflow check and AdamW over the exchanged gradients of the segments `segs` ([(offset, numel, key)]): the end
        of a window.  The window's 1/k enters AdamW's grad_scale, not the fp16 loss gradient."""
        G = self.G
        for off, n, _ in segs:
            ops.nonfinite_flag(G.flat_g[off:off + n], self.overflow_flag)  # after the all-reduce: every rank decides the same
        for i, (off, n, key) in enumerate(segs):
            step_dev, bc = self._seg_state(key)
            ops.adamw_begin(step_dev, self.overflow_flag, self.betas, bc, self._skipped_dev if i == 0 else None)
            ops.adamw_step(G.flat_p[off:off + n], G.flat_g[off:off + n], G.exp_avg[off:off + n], G.exp_avg_sq[off:off + n], 0,
                           lr=self.lr, betas=self.betas, eps=self.eps, weight_decay=self.wd,
                           grad_scale=1.0 / (self.world * self._scale_used * self.accumulate_grad_batches),
                           skip_flag=self.overflow_flag, bc_dev=bc)
            self.seg_steps[key] = self.seg_steps.get(key, 0) + 1
        prepare.bump_train_version()
        self.step_count += 1
        self.micro_step = 0
        if self._poll_overflow():
            self._after_skipped()

    def _after_skipped(self):
        """GradScaler semantics: the updates were skipped on the device; the scale is halved (re-capturing the graphs,
        whose loss kernel has the scale baked in) and the host step counts are re-read"""
        self.seg_steps = {k: int(v.item()) for k, v in self._step_dev.items()}
        self.step_count = self.seg_steps.get(self.segment_keys()[0], 0)
        self._recapture()

    def _recapture(self):
        if self._graphs is not None:
            self.capture(*self._static, tasks=list(self._graphs["compute"]), warmup=1)

    def _overflowed(self):
        return bool(self.overflow_flag.item())

    # -- checkpoints in the reference's Lightning layout (ctrlora_b200.checkpoint) ---------------------------------------
    def segment_keys(self):
        """the step-count segment of every optimizer parameter (GradSink order)"""
        return ["all"] * len(self.G.names)

    def _alias_key(self, key):
        """a state-dict key that names a parameter also stored under another key (checkpoint.checkpoint_weights)"""
        return False

    def _exact_counters(self):
        """Read the device's skipped-step counter now (the periodic poll, forced), so step_count, seg_steps,
        skipped_steps and loss_scale are exact on the host.  Refused inside an accumulation window."""
        if self.micro_step != 0:
            raise RuntimeError(f"cannot checkpoint inside an accumulation window ({self.micro_step} of "
                               f"{self.accumulate_grad_batches} micro-batches done): the partial gradient is not part of "
                               "the state; save between windows or after flush()")
        launched = self._launched
        try:
            if self._poll_overflow(force=True):
                self._after_skipped()
        finally:
            self._launched = launched  # the periodic poll keeps its cadence

    def state_dict(self):
        """The optimizer part of a checkpoint: {"optimizer": torch.optim.AdamW.state_dict() over the reference's
        parameter list (a Lightning checkpoint's optimizer_states[0]), checkpoint.EXTRA_KEY: loss scale, skipped steps,
        accumulate_grad_batches}.  Tensors are CPU copies."""
        self._exact_counters()
        return {"optimizer": checkpoint.optimizer_state_dict(self), checkpoint.EXTRA_KEY: checkpoint.trainer_extra(self)}

    def load_state_dict(self, sd):
        """Load state_dict()'s output, or a bare torch.optim.AdamW.state_dict(), in place: the flat moments, the host and
        device step counters and the file's hyper-parameters (lr, betas, eps, weight_decay).  A parameter without state
        is fresh (zero moments; its first step is AdamW step 1).  The current accumulation window is dropped.  Graphs
        whose baked-in loss scale no longer matches are re-captured."""
        if self._load_optimizer(sd):
            self._recapture()

    def _load_optimizer(self, sd):
        """load_state_dict without the re-capture; True if a captured graph's loss scale no longer matches"""
        opt, extra = (sd, None) if "param_groups" in sd else (sd["optimizer"], sd.get(checkpoint.EXTRA_KEY))
        scale, skipped = checkpoint.parse_extra(self, extra)
        checkpoint.load_optimizer_state_dict(self, opt)
        self.loss_scale, self.skipped_steps = scale, skipped
        self.micro_step, self._window_tasks = 0, []
        self.overflow_flag.zero_()
        self._skipped_dev.zero_()
        self._skipped_seen = 0
        return any(s != self._scale_for(self._static[0].numel()) for s in self._captured_scales())

    def _captured_scales(self):
        """loss scales baked into the captured graphs"""
        return [scale for _, _, scale in self._graphs["compute"].values()] if self._graphs is not None else []

    def save_checkpoint(self, path, epoch=0):
        """Write a checkpoint in the layout of the reference's `trainer.save_checkpoint` (cldm/logger.py:123):
        state_dict (model.state_dict(), contiguous CPU copies in the reference shapes), optimizer_states
        ([state_dict()["optimizer"]]), global_step (step_count: optimizer steps), epoch, and checkpoint.EXTRA_KEY.
        Under torch.distributed every rank syncs its counters, rank 0 writes, and all ranks leave together."""
        self._exact_counters()
        if self.rank == 0:
            ckpt = {"epoch": int(epoch), "global_step": int(self.step_count),
                    "state_dict": checkpoint.model_state_dict(self.model),
                    "optimizer_states": [checkpoint.optimizer_state_dict(self)],
                    checkpoint.EXTRA_KEY: checkpoint.trainer_extra(self)}
            torch.save(ckpt, path)
        if self.world > 1:
            torch.distributed.barrier(group=self.pg)

    def load_checkpoint(self, path):
        """Load a checkpoint written by save_checkpoint or by the reference's Lightning trainer into this trainer, in
        place: the weights through model.load_state_dict (keys of cond_stage_model are ignored unless the model was built
        with the text encoder), then load_state_dict of optimizer_states[0] and checkpoint.EXTRA_KEY.  Everything is
        validated before anything changes.  Trainable-weight copies are rebuilt, and captured graphs are re-captured (the frozen-weight
        copies they read are built outside the capture).  Every rank of a data-parallel run loads the same file.
        Returns {"epoch", "global_step"} of the file."""
        ckpt = torch.load(path, map_location="cpu", weights_only=True)
        weights = checkpoint.checkpoint_weights(ckpt["state_dict"], self.model.state_dict(), self._alias_key)
        opts = ckpt.get("optimizer_states") or []
        if len(opts) != 1:
            raise ValueError(f"expected one optimizer state in the checkpoint, found {len(opts)}")
        checkpoint.check_optimizer_state_dict(self, opts[0])
        checkpoint.parse_extra(self, ckpt.get(checkpoint.EXTRA_KEY))
        self.model.load_state_dict(weights, strict=False)
        prepare.bump_train_version()  # the flat parameter buffer was written behind the caches' version counters
        self._load_optimizer({"optimizer": opts[0], checkpoint.EXTRA_KEY: ckpt.get(checkpoint.EXTRA_KEY)})
        self._recapture()
        return {"epoch": ckpt.get("epoch", 0), "global_step": ckpt.get("global_step", self.step_count)}

    # -- gradient accumulation (accumulate_grad_batches = k; a plain step is k = 1) ---------------------------------------
    # A window of k micro-batches: the first zeroes the gradient buffer (and the overflow flag) and fixes the loss scale;
    # every micro-batch's backward adds into the buffer (every gradient write of the backward accumulates); with k > 1 the
    # trainable weight copies (LoRA folds, fp16 / transposed / dgrad copies) are built once per window: the caches are
    # keyed on the train version, which moves only when AdamW runs.  Only the last micro-batch exchanges the gradients.
    def window_segments(self, tasks):
        """[(offset, numel, key)] a window's update touches, given this rank's micro-batch tasks: the whole buffer."""
        return [(0, self.G.numel, "all")]

    def begin_micro_batch(self, task=None):
        """Window bookkeeping of one micro-batch, host only: records its task, and when it is the window's last one
        returns the window's segments (window_segments, which exchanges the used tasks across ranks).  Returns
        (window_start, first_use_of_task, segments or None)."""
        start = self.micro_step == 0
        if start:
            self._window_tasks = []
        first_use = task not in self._window_tasks
        self._window_tasks.append(task)
        self.micro_step += 1
        final = self.micro_step == self.accumulate_grad_batches
        return start, first_use, (self.window_segments(self._window_tasks) if final else None)

    def _micro_batch(self, args, task):
        """step(): replay the task's captured graphs, or run it eagerly; the window's last micro-batch exchanges the
        gradients -- bucket by bucket under its backward when the exchange is segmented -- and runs AdamW."""
        start, first_use, segs = self.begin_micro_batch(task)
        final = segs is not None
        compute = self._graphs["compute"] if self._graphs else {}
        overlapped = False
        if task in compute:
            for dst, src in zip(self._static, args):
                if dst.data_ptr() != src.data_ptr():
                    dst.copy_(src, non_blocking=True)
            if task is not None:
                self.cn.switch_lora(task)  # host-side pointers follow the graphs (weight caches are keyed on them)
                self.task = task
            prep = self._graphs["prep"]   # empty at k = 1: the compute graph rebuilds the copies
            if start and None in prep:
                prep[None].replay()       # zero the buffer and the overflow flag, rebuild the task-independent copies
            if first_use and task is not None and task in prep:
                prep[task].replay()       # the task's LoRA folds, once per window
            g, static_loss, self._scale_used = compute[task]
            if isinstance(g, list):
                plan = self.exchange_plan(segs, [r for _, r in g]) if final else [None] * len(g)
                for (graph, _), ranges in zip(g, plan):
                    graph.replay()
                    self._reduce_ranges(ranges)
                overlapped = final and self.world > 1
            else:
                g.replay()
            loss = static_loss.clone()    # the next replay overwrites the captured loss
        elif compute and self.accumulate_grad_batches > 1:
            # at k = 1 an uncaptured task runs eagerly; a window's micro-batches read its preparation graphs' copies
            raise KeyError(f"no graph captured for task {task!r}: pass it to capture()")
        elif final and self._segmented():
            merged = self.merged_buckets()
            plan = dict(zip([st for st, _ in merged], self.exchange_plan(segs, [r for _, r in merged])))
            self._on_stage = lambda name: self._reduce_ranges(plan.get(name))
            try:
                loss = self.loss_and_grads(*args, task=task, accumulate=not start)
            finally:
                self._on_stage = None
            self._reduce_ranges(plan["final"])
            overlapped = self.world > 1
        else:
            loss = self.loss_and_grads(*args, task=task, accumulate=not start)
        if final:
            if overlapped:
                torch.cuda.current_stream().wait_stream(self._comm)  # every bucket reduced before the overflow check / AdamW
            else:
                self.reduce_gradients([(off, n) for off, n, _ in segs])
            self._update(segs)
        return loss

    def flush(self):
        """Apply a partial window (fewer than k micro-batches, e.g. at the end of an epoch) with the same 1/k factor, as
        Lightning does on an epoch's last batch.  Nothing happens on an empty window."""
        if self.micro_step == 0:
            return
        segs = self.window_segments(self._window_tasks)
        self.reduce_gradients([(off, n) for off, n, _ in segs])
        self._update(segs)


# ------------------------------------------------------------------------------------------------ pretraining
def pretrain_parameters(control_model):
    """The pretrain optimizer's set: `list(control_model.parameters())` as the reference sees it in
    configure_optimizers (cldm_ctrlora_pretrain.py:174-182), i.e. before any switch_lora: the ControlNet's own parameters in
    module order, then every task's LoRA set under loras_dict.  (After a switch the attached set is ALSO reachable as
    `<linear>.lora_layer.*`; those aliases are skipped so the order does not depend on the attached task.)"""
    out, seen = [], set()
    for n, p in control_model.named_parameters(remove_duplicate=False):
        if ".lora_layer." in n or id(p) in seen:
            continue
        seen.add(id(p))
        out.append((n, p))
    return out


def active_segments(layout, tasks_on_ranks):
    """[(offset, numel, key)] of the flat buffer a step touches: the ControlNet's own parameters plus the LoRA sets of
    the tasks any rank trained this step.  A set no rank used keeps `grad is None` in the reference (DDP with
    find_unused_parameters leaves globally unused parameters untouched, and AdamW skips them -- no moment update, no
    weight decay), so it is neither reduced nor stepped here."""
    segs = [layout["base"] + ("base",)]
    for task in sorted(set(tasks_on_ranks), key=layout["tasks"].index):
        segs.append(layout["lora"][task] + (task,))
    return segs


class PretrainTrainer(FinetuneTrainer):
    """Base-ControlNet pretraining step (configs ctrlora_pretrain_sd15_9tasks_rank128.yaml): every ControlNet parameter
    and the mini-batch task's LoRA set are trained (cldm_ctrlora_pretrain.py:88-111,174-182); the task changes per
    mini-batch (datasets/multi_task_scheduler.py, mirrored by ctrlora_b200.scheduler.TaskSchedule).  Also covers
    ControlNetFinetune(ft_with_lora=False) (full-parameter finetuning, cldm_ctrlora_finetune.py:101-104)."""

    # The dense gradient buffer is 1.5 GB, so part of its exchange can hide under the backward; the rest is lost to the
    # collective's CTAs and HBM traffic competing with the backward it overlaps.  Default: all four cuts.
    CUTS_ENV, CUTS_DEFAULT = "CTRLORA_PRETRAIN_ALLREDUCE_CUTS", "middle,ib9,ib6,ib3"

    def __init__(self, model, lr=1e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, process_group=None,
                 loss_scale=None, dynamic_loss_scale=True, accumulate_grad_batches=1):
        super().__init__(model, lr, betas, eps, weight_decay, process_group, loss_scale, dynamic_loss_scale,
                         accumulate_grad_batches, named=pretrain_parameters(model.control_model))
        self.tasks = list(getattr(self.cn, "tasks", []))
        names = self.G.names
        first_lora = next((i for i, n in enumerate(names) if n.startswith("loras_dict.")), len(names))
        base_end = self.G.offsets[names[first_lora]][0] if first_lora < len(names) else self.G.numel
        self.layout = {"base": (0, base_end), "tasks": self.tasks, "lora": {}}
        for task in self.tasks:
            mine = [self.G.offsets[n] for n in names if n.startswith(f"loras_dict.{task}.")]
            start = mine[0][0]
            assert all(o == start + sum(m[1] for m in mine[:i]) for i, (o, _) in enumerate(mine)), "task set not contiguous"
            self.layout["lora"][task] = (start, sum(m[1] for m in mine))
        self.task = self.tasks[0] if self.tasks else None

    def _after_cut(self):
        """Segments after a cut run next to a collective: their persistent GEMM grids leave CTRLORA_OVERLAP_SM_RESERVE
        (default 16) SMs to its CTAs."""
        reserve = int(os.environ.get("CTRLORA_OVERLAP_SM_RESERVE", "16"))
        ops.set_sm_limit(max(2, torch.cuda.get_device_properties(self.G.flat_p.device).multi_processor_count - reserve))

    def step(self, x0, hint_latent, context, t, noise, task=None):
        """One micro-batch of `task` (default: the attached one); see FinetuneTrainer.step."""
        return self._micro_batch((x0, hint_latent, context, t, noise), task if task is not None else self.task)

    def window_segments(self, tasks):
        """Segments of a window whose micro-batches on this rank trained `tasks`: the ControlNet plus every LoRA set that
        any rank used in any micro-batch of the window.  The ranks exchange their used-task masks once per window (one
        all-reduce), before its last backward."""
        if not self.tasks:
            return [(0, self.G.numel, "base")]
        used = sorted({self.tasks.index(t) for t in tasks})
        if self.world > 1:
            mask = torch.zeros(len(self.tasks), device=self.G.flat_p.device, dtype=torch.int32)
            mask[used] = 1
            torch.distributed.all_reduce(mask, group=self.pg)
            used = [i for i, v in enumerate(mask.tolist()) if v]
        return active_segments(self.layout, [self.tasks[i] for i in used])

    def segment_keys(self):
        """"base" for the ControlNet's own parameters, the task for its LoRA set (active_segments)"""
        if not self.tasks:
            return ["base"] * len(self.G.names)
        return [n.split(".")[1] if n.startswith("loras_dict.") else "base" for n in self.G.names]

    def _alias_key(self, key):
        """`control_model.<linear>.lora_layer.*`: the attached task's set, whose data is saved under loras_dict.<task>.*
        (which set a file had attached, if any, does not matter on load)"""
        return bool(self.tasks) and key.startswith("control_model.") and ".lora_layer." in key
