"""Drop-in for the reference's `ldm/modules/attention.py`: same class names, constructor signatures, attribute tree
and state-dict keys; the arithmetic runs in the sm_90a kernels.

Kernel sequence of one SpatialTransformer (reference :321-340 and :271-275), all on pixel-major fp16 so the
'b c h w -> b (h w) c' rearranges (:330,:337) cost nothing:
    groupnorm(eps 1e-6) -> gemm proj_in ->
      layernorm -> gemm [q|k|v] (LoRA folded, V stored transposed) -> attention -> gemm to_out (+bias +residual) ->
      layernorm -> gemm q ; gemm [k|v](context) -> attention -> gemm to_out (+bias +residual) ->
      layernorm -> gemm GEGLU (value*gelu(gate) in the epilogue) -> gemm ff.net.2 (+bias +residual)
    -> gemm proj_out (+bias + x_in)
Each layer has one body.  Its optional `other`, the same layer of a second network, turns every launch into a grouped
one over the two halves of the batch (the twin pass of cldm/cldm.py); the attention launch covers the whole batch.
"""
from inspect import isfunction

import torch
import torch.nn as nn

from ctrlora_b200 import ops, prepare
from ctrlora_b200.runtime import nchw_view, pixel_major, to_f16_rows
from ldm.modules.diffusionmodules.util import checkpoint  # noqa: F401  (re-exported like the reference)

XFORMERS_IS_AVAILBLE = False  # name kept from the reference; the fused kernel supersedes both attention classes


def exists(val):
    return val is not None


def uniq(arr):
    return {el: True for el in arr}.keys()


def default(val, d):
    if exists(val):
        return val
    return d() if isfunction(d) else d


def zero_module(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


def Normalize(in_channels):
    return nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)


class GEGLU(nn.Module):
    """Parameter holder for `proj` (dim -> 2*dim_out); evaluated in the GEMM epilogue (reference :49-56)."""

    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        raise RuntimeError("GEGLU runs inside FeedForward's fused GEMM")


class FeedForward(nn.Module):
    def __init__(self, dim, dim_out=None, mult=4, glu=False, dropout=0.):
        super().__init__()
        if not glu:
            raise NotImplementedError("non-gated FeedForward is not on the CtrLoRA path (gated_ff=True everywhere)")
        if dropout != 0.:
            raise NotImplementedError("dropout > 0 is not on the CtrLoRA path")
        inner_dim = int(dim * mult)
        dim_out = default(dim_out, dim)
        self.net = nn.Sequential(GEGLU(dim, inner_dim), nn.Dropout(dropout), nn.Linear(inner_dim, dim_out))
        self._prep = prepare.PrepCache()

    def _kernel_params(self):
        proj, out = self.net[0].proj, self.net[2]
        lk = prepare.lora_key
        w1 = self._prep.get(("w1", lk(proj)), prepare.linear_params(proj), lambda: prepare.effective_linear_weight(proj))
        w2 = self._prep.get(("w2", lk(out)), prepare.linear_params(out), lambda: prepare.effective_linear_weight(out))
        return w1, prepare.bias_f32(proj.bias), w2, prepare.bias_f32(out.bias)

    def run(self, x2d, residual=None, out=None, other=None):
        """x2d fp16 [M, dim] -> fp16 [M, dim_out] (+ residual).  other: the same layer of a second network, applied to
        the upper half of the rows in the same launches."""
        w1, b1, w2, b2 = self._kernel_params()
        h1 = h2 = None
        if other is not None:
            ow1, ob1, ow2, ob2 = other._kernel_params()
            h1, h2 = {"w": ow1, "bias": ob1}, {"w": ow2, "bias": ob2}
        g = ops.gemm(x2d, w1, bias=b1, geglu=True, hi=h1)
        return ops.gemm(g, w2, bias=b2, residual=residual, out=out, hi=h2)

    def forward(self, x):
        shp = x.shape
        return self.run(to_f16_rows(x)).view(*shp[:-1], -1)


class CrossAttention(nn.Module):
    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.):
        super().__init__()
        inner_dim = dim_head * heads
        context_dim = default(context_dim, query_dim)
        self.scale = dim_head ** -0.5
        self.heads = heads
        self.to_q = nn.Linear(query_dim, inner_dim, bias=False)
        self.to_k = nn.Linear(context_dim, inner_dim, bias=False)
        self.to_v = nn.Linear(context_dim, inner_dim, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner_dim, query_dim), nn.Dropout(dropout))
        self._prep = prepare.PrepCache()

    def _cat_weight(self, key, linears):
        params = [p for lin in linears for p in prepare.linear_params(lin)]
        return self._prep.get((key, prepare.lora_key(*linears)), params,
                              lambda: torch.cat([prepare.effective_linear_weight(lin) for lin in linears], 0).contiguous())

    def _kv_weight_token(self):
        lins = [self.to_k, self.to_v]
        return prepare._ver(*[p for lin in lins for p in prepare.linear_params(lin)]) + prepare.lora_key(*lins)

    def project_context(self, ctx2d, batch, nk, ctx_key, out=None):
        """K and V^T of a step-invariant context, into persistent buffers (see ControlLDM.prepare_context); `out`:
        the (K, V^T) buffers to use."""
        inner = self.to_q.out_features
        h, d = self.heads, inner // self.heads
        nk_pad = (nk + 7) // 8 * 8
        token = (ctx_key, ctx2d.data_ptr(), self._kv_weight_token())
        hit = self.__dict__.get("_kv_cache")
        if hit is not None and hit[0] == token and (out is None or hit[1].data_ptr() == out[0].data_ptr()):
            return
        if out is not None:
            k, vt = out
        elif hit is not None and hit[1].shape == (batch * nk, inner) and hit[2].shape == (batch, h, d, nk_pad):
            k, vt = hit[1], hit[2]  # same addresses: captured graphs keep reading them
        else:
            k = torch.empty((batch * nk, inner), device=ctx2d.device, dtype=torch.float16)
            vt = ops.zeros((batch, h, d, nk_pad), ctx2d.device)
        w = self._cat_weight("kv", [self.to_k, self.to_v])
        ops.gemm(ctx2d, w, seg_outs=[k, vt], seg_width=inner, transposed=(0, 1, 0), rows_per_img=nk, head_dim=d, tok_pad=nk_pad)
        self.__dict__["_kv_cache"] = (token, k, vt)

    def _kv_hit(self, ctx2d, batch, nk):
        """(K, V^T) that project_context computed for this context and these weights, or None"""
        hit = self.__dict__.get("_kv_cache")
        if hit is not None and hit[0][1] == ctx2d.data_ptr() and hit[0][2] == self._kv_weight_token() and \
                hit[1].shape[0] == batch * nk:
            return hit[1], hit[2]
        return None

    def _q_weight(self):
        return self._prep.get(("q", prepare.lora_key(self.to_q)), prepare.linear_params(self.to_q),
                              lambda: prepare.effective_linear_weight(self.to_q))

    def _context_kv(self, ctx2d, batch, nk, other=None):
        """K [batch*nk, inner] and V^T [batch, heads, d, nk_pad] of the context: the buffers project_context filled when
        they are this context's, else projections into new buffers.  With `other` (the same layer of a second network)
        ctx2d holds batch/2 images' tokens; the lower half of K / V^T is this layer's projection of them, the upper half
        other's, and the buffers to re-use are the pair's one `_kv_twin` (ControlLDM.prepare_context)."""
        layers = (self,) if other is None else (self, other)
        per = batch // len(layers)
        if other is None:
            hit = self._kv_hit(ctx2d, batch, nk)
        else:
            hit, mine, theirs = self.__dict__.get("_kv_twin"), self._kv_hit(ctx2d, per, nk), other._kv_hit(ctx2d, per, nk)
            if hit is None or mine is None or theirs is None or mine[0].data_ptr() != hit[0].data_ptr() or \
                    theirs[0].data_ptr() != hit[0][per * nk:].data_ptr():
                hit = None
        if hit is not None:
            return hit
        inner = self.to_q.out_features
        h, d = self.heads, inner // self.heads
        nk_pad = (nk + 7) // 8 * 8
        dev = ctx2d.device
        k = torch.empty((batch * nk, inner), device=dev, dtype=torch.float16)
        # the key padding columns (77 -> 80) are never written by the projection, and ops.attention never reads
        # them: its V^T tensor map ends at key nk, so keys >= nk load as zeros.  The zero fill is not needed for
        # correctness.
        vt = ops.zeros((batch, h, d, nk_pad), dev) if nk_pad != nk else torch.empty((batch, h, d, nk_pad), device=dev, dtype=torch.float16)
        for i, m in enumerate(layers):
            rows, imgs = slice(i * per * nk, (i + 1) * per * nk), slice(i * per, (i + 1) * per)
            ops.gemm(ctx2d, m._cat_weight("kv", [m.to_k, m.to_v]), seg_outs=[k[rows], vt[imgs]], seg_width=inner,
                     transposed=(0, 1, 0), rows_per_img=nk, head_dim=d, tok_pad=nk_pad)
        return k, vt

    def run(self, x2d, batch, nq, ctx2d=None, nk=None, residual=None, other=None, **finish_kw):
        """x2d fp16 [batch*nq, C]; ctx2d fp16 [batch*nk, Cctx] or None (self-attention). Returns to_out(attn) (+residual).
        other: the same layer of a second network, applied to the upper half of the batch in the same launches (one
        attention launch over the whole batch); both halves attend the same context, so ctx2d then holds batch/2
        images' tokens.  finish_kw: handed on to _finish."""
        inner = self.to_q.out_features
        h, d = self.heads, inner // self.heads
        if ctx2d is None:
            nk = nq
            nk_pad = (nk + 7) // 8 * 8
            q = torch.empty((batch * nq, inner), device=x2d.device, dtype=torch.float16)
            k = torch.empty_like(q)
            vt = torch.empty((batch, h, d, nk_pad), device=x2d.device, dtype=torch.float16)
            w = self._cat_weight("qkv", [self.to_q, self.to_k, self.to_v])
            hi = None if other is None else {"w": other._cat_weight("qkv", [other.to_q, other.to_k, other.to_v])}
            ops.gemm(x2d, w, seg_outs=[q, k, vt], seg_width=inner, transposed=(0, 0, 1), rows_per_img=nk, head_dim=d,
                     tok_pad=nk_pad, hi=hi)
        else:
            q = ops.gemm(x2d, self._q_weight(), hi=None if other is None else {"w": other._q_weight()})
            k, vt = self._context_kv(ctx2d, batch, nk, other)
        return self._finish(ops.attention(q, k, vt, batch, h, nq, nk, d), q, batch, nq, residual, other, **finish_kw)

    def _out_weight(self):
        lin = self.to_out[0]
        return self._prep.get(("o", prepare.lora_key(lin)), prepare.linear_params(lin),
                              lambda: prepare.effective_linear_weight(lin))

    def _finish(self, o, q, batch, nq, residual, other=None):
        """to_out(attention output) (+ residual); `q` is handed on for variants that attend a second key set
        (ldm/modules/attention_ip.py)."""
        w, bias = self._out_weight(), prepare.bias_f32(self.to_out[0].bias)
        hi = None if other is None else {"w": other._out_weight(), "bias": prepare.bias_f32(other.to_out[0].bias)}
        return ops.gemm(o, w, bias=bias, residual=residual, hi=hi)

    def forward(self, x, context=None, mask=None):
        if mask is not None:
            raise NotImplementedError("attention masks are not on the CtrLoRA path")
        b, n, _ = x.shape
        ctx2d, nk = (None, None) if context is None else (to_f16_rows(context), context.shape[1])
        return self.run(to_f16_rows(x), b, n, ctx2d, nk).view(b, n, -1)


MemoryEfficientCrossAttention = CrossAttention  # the xformers variant (reference :197-243) is the same fused kernel here


class BasicTransformerBlock(nn.Module):
    ATTENTION_MODES = {"softmax": CrossAttention, "softmax-xformers": MemoryEfficientCrossAttention}
    attn2_cls = CrossAttention  # ldm/modules/attention_ip.py: IPCrossAttention

    def __init__(self, dim, n_heads, d_head, dropout=0., context_dim=None, gated_ff=True, checkpoint=True,
                 disable_self_attn=False):
        super().__init__()
        self.disable_self_attn = disable_self_attn
        self.attn1 = CrossAttention(query_dim=dim, heads=n_heads, dim_head=d_head, dropout=dropout,
                                    context_dim=context_dim if disable_self_attn else None)
        self.ff = FeedForward(dim, dropout=dropout, glu=gated_ff)
        self.attn2 = type(self).attn2_cls(query_dim=dim, context_dim=context_dim, heads=n_heads, dim_head=d_head,
                                          dropout=dropout)
        self.norm1 = nn.LayerNorm(dim)
        self.norm2 = nn.LayerNorm(dim)
        self.norm3 = nn.LayerNorm(dim)
        self.checkpoint = checkpoint

    @staticmethod
    def _ln(norm, x2d, other=None):
        """LayerNorm `norm` (of the upper half of the rows: `other`, the same layer of a second network)"""
        norm = prepare.effective(norm)
        hi = {} if other is None else {"gamma_hi": prepare.bias_f32(prepare.effective(other).weight),
                                       "beta_hi": prepare.bias_f32(prepare.effective(other).bias)}
        return ops.layernorm(x2d, prepare.bias_f32(norm.weight), prepare.bias_f32(norm.bias), norm.eps, **hi)

    def run(self, x2d, batch, n, ctx2d, nk, out=None, other=None, **attn2_kw):
        """x2d fp16 [batch*n, dim] -> same shape (reference _forward :271-275); `out`: optional destination buffer.
        other: the same block of a second network, applied to the upper half of the rows in the same launches.
        attn2_kw: further arguments of attn2.run (the IP-Adapter's image tokens)."""
        o = (None,) * 6 if other is None else (other.norm1, other.norm2, other.norm3, other.attn1, other.attn2, other.ff)
        c1 = (ctx2d, nk) if self.disable_self_attn else (None, None)
        x2d = self.attn1.run(self._ln(self.norm1, x2d, o[0]), batch, n, c1[0], c1[1], residual=x2d, other=o[3])
        x2d = self.attn2.run(self._ln(self.norm2, x2d, o[1]), batch, n, ctx2d, nk, residual=x2d, other=o[4], **attn2_kw)
        return self.ff.run(self._ln(self.norm3, x2d, o[2]), residual=x2d, out=out, other=o[5])

    def forward(self, x, context=None):
        b, n, _ = x.shape
        ctx2d, nk = (None, None) if context is None else (to_f16_rows(context), context.shape[1])
        return self.run(to_f16_rows(x), b, n, ctx2d, nk).view(b, n, -1)


class SpatialTransformer(nn.Module):
    block_cls = BasicTransformerBlock

    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0., context_dim=None, disable_self_attn=False,
                 use_linear=False, use_checkpoint=True):
        super().__init__()
        if exists(context_dim) and not isinstance(context_dim, list):
            context_dim = [context_dim]
        self.in_channels = in_channels
        inner_dim = n_heads * d_head
        self.norm = Normalize(in_channels)
        if not use_linear:
            self.proj_in = nn.Conv2d(in_channels, inner_dim, kernel_size=1, stride=1, padding=0)
        else:
            self.proj_in = nn.Linear(in_channels, inner_dim)
        self.transformer_blocks = nn.ModuleList(
            [type(self).block_cls(inner_dim, n_heads, d_head, dropout=dropout, context_dim=context_dim[d],
                                  disable_self_attn=disable_self_attn, checkpoint=use_checkpoint) for d in range(depth)])
        if not use_linear:
            self.proj_out = zero_module(nn.Conv2d(inner_dim, in_channels, kernel_size=1, stride=1, padding=0))
        else:
            self.proj_out = zero_module(nn.Linear(in_channels, inner_dim))
        self.use_linear = use_linear
        self._prep = prepare.PrepCache()

    def _w(self, key, mod):
        if isinstance(mod, nn.Linear):
            return self._prep.get((key, prepare.lora_key(mod)), prepare.linear_params(mod),
                                  lambda: prepare.effective_linear_weight(mod))
        return self._prep.get(key, [mod.weight], lambda: prepare.conv_weight(mod.weight))

    def forward_grouped(self, x, context, n_groups, attach):
        """One pass over a batch made of `n_groups` equal slices that use DIFFERENT LoRA / norm sets (multi-LoRA inference,
        cldm/cldm_ctrlora_inference.py:156-178 runs the ControlNet once per set): `attach(self, g)` re-points this module's
        LoRA layers and switchable norms to set g.  The 1x1 convs (no LoRA) run once over the whole batch; the GroupNorm and
        the transformer blocks run per slice, writing into shared buffers (no concatenation)."""
        xp = pixel_major(x)
        b, h, w, c = xp.shape
        bg = b // n_groups
        if not isinstance(context, list):
            context = [context]
        xn = torch.empty_like(xp)
        for g in range(n_groups):
            attach(self, g)
            gn = prepare.effective(self.norm)
            ops.groupnorm(xp[g * bg:(g + 1) * bg], prepare.bias_f32(gn.weight), prepare.bias_f32(gn.bias), gn.eps, False,
                          groups=gn.num_groups, out=xn[g * bg:(g + 1) * bg])
        y = ops.gemm(xn, self._w("in", self.proj_in), bias=prepare.bias_f32(self.proj_in.bias))
        y2d = y.view(b * h * w, -1)
        rows = bg * h * w
        y_out = torch.empty_like(y2d)
        for g in range(n_groups):
            attach(self, g)
            yg = y2d[g * rows:(g + 1) * rows]
            for i, block in enumerate(self.transformer_blocks):
                ctx = context[i] if i < len(context) else context[-1]
                ctx_g = None if ctx is None else (ctx if ctx.shape[0] == bg else ctx[g * bg:(g + 1) * bg])  # shared or per slice
                ctx2d, nk = (None, None) if ctx_g is None else (to_f16_rows(ctx_g), ctx_g.shape[1])
                last = i == len(self.transformer_blocks) - 1
                yg = block.run(yg, bg, h * w, ctx2d, nk, out=y_out[g * rows:(g + 1) * rows] if last else None)
        out = ops.gemm(y_out.view(b, h, w, -1), self._w("out", self.proj_out), bias=prepare.bias_f32(self.proj_out.bias),
                       residual=xp.view(b * h * w, c))
        return nchw_view(out)

    @staticmethod
    def block_context(ctx):
        """a transformer block's context entry -> (ctx2d, nk, further attn2.run arguments)"""
        return (None, None, {}) if ctx is None else (to_f16_rows(ctx), ctx.shape[1], {})

    def forward(self, x, context=None, other=None):
        """other: the same layer of a second network, applied to the upper half of the batch in the same launches;
        `context` then holds the images of one half, which both halves attend."""
        xp = pixel_major(x)  # [B, H, W, C]
        b, h, w, c = xp.shape
        if not isinstance(context, list):
            context = [context]
        f32 = prepare.bias_f32
        gn = prepare.effective(self.norm)
        ogn = None if other is None else prepare.effective(other.norm)
        hi = {} if other is None else {"gamma_hi": f32(ogn.weight), "beta_hi": f32(ogn.bias)}
        xn = ops.groupnorm(xp, f32(gn.weight), f32(gn.bias), gn.eps, False, groups=gn.num_groups, **hi)
        wi, bias = self._w("in", self.proj_in), f32(self.proj_in.bias)
        hi = None if other is None else {"w": other._w("in", other.proj_in), "bias": f32(other.proj_in.bias)}
        y = ops.gemm(xn, wi, bias=bias, hi=hi)
        y2d = y.view(b * h * w, -1)
        for i, block in enumerate(self.transformer_blocks):
            ctx2d, nk, attn2_kw = self.block_context(context[i] if i < len(context) else context[-1])
            y2d = block.run(y2d, b, h * w, ctx2d, nk, other=None if other is None else other.transformer_blocks[i],
                            **attn2_kw)
        wo, bias = self._w("out", self.proj_out), f32(self.proj_out.bias)
        hi = None if other is None else {"w": other._w("out", other.proj_out), "bias": f32(other.proj_out.bias)}
        out = ops.gemm(y2d.view(b, h, w, -1), wo, bias=bias, residual=xp.view(b * h * w, c), hi=hi)
        return nchw_view(out)
