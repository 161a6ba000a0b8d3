"""IP-Adapter / InstantStyle cross-attention (reference ldm/modules/attention_ip.py): a second key / value stream
`to_k_ip / to_v_ip` over the image-prompt tokens, attended with the same queries and added with `ip_scale`
(reference :196-289).  Everything else is ldm/modules/attention.py (the reference's file is a copy of it too).

    out = to_out( softmax(q k^T) v  +  ip_scale * softmax(q k_ip^T) v_ip )

Here the second stream reuses the projected queries, runs the single-tile attention kernel over the (4 .. 16) image
tokens, and its output enters `to_out` as the SECOND OPERAND PAIR of the same wgmma GEMM
(o @ Wo^T + o_ip @ (ip_scale Wo)^T accumulate in one register tile): no separate add pass, no extra rounding of the sum.
"""
import torch
import torch.nn as nn

from ctrlora_b200 import ops, prepare
from ctrlora_b200.runtime import nchw_view, pixel_major, to_f16_rows
from ldm.modules import attention as _base
from ldm.modules.attention import (GEGLU, CrossAttention, FeedForward, MemoryEfficientCrossAttention,  # noqa: F401
                                   Normalize, default, exists, uniq, zero_module)


def split_context(ctx):
    """`[text, ip]` (reference :222-231: a list is the pair, a tensor means no image prompt) -> (text, ip | None)"""
    if isinstance(ctx, (list, tuple)):
        if len(ctx) != 2:
            raise ValueError("an IP-Adapter context is the pair [text_tokens, image_tokens | None]")
        return ctx[0], ctx[1]
    return ctx, None


class IPCrossAttention(CrossAttention):
    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.):
        super().__init__(query_dim, context_dim=context_dim, heads=heads, dim_head=dim_head, dropout=dropout)
        inner_dim = dim_head * heads
        context_dim = default(context_dim, query_dim)
        # registration order of the reference (:207-215): to_q, to_k, to_v, to_k_ip, to_v_ip, ip_scale, to_out
        to_out = self._modules.pop("to_out")
        self.to_k_ip = nn.Linear(context_dim, inner_dim, bias=False)
        self.to_v_ip = nn.Linear(context_dim, inner_dim, bias=False)
        self.register_buffer("ip_scale", torch.tensor(0.0))
        self.to_out = to_out

    def _ip_scale_value(self):
        t = self.ip_scale
        key = (t.data_ptr(), t._version)
        hit = self.__dict__.get("_ip_scale_host")
        if hit is None or hit[0] != key:
            if t.is_cuda and torch.cuda.is_current_stream_capturing():
                raise RuntimeError("ip_scale changed under a CUDA-graph capture: run one eager step first")
            hit = self.__dict__["_ip_scale_host"] = (key, float(t))
        return hit[1]

    def run(self, x2d, batch, nq, ctx2d=None, nk=None, residual=None, ip2d=None, nk_ip=None):
        self.__dict__["_ip"] = None if ip2d is None else (ip2d, nk_ip)
        try:
            return super().run(x2d, batch, nq, ctx2d, nk, residual=residual)
        finally:
            self.__dict__["_ip"] = None

    def _finish(self, o, q, batch, nq, residual):
        ip = self.__dict__.get("_ip")
        scale = self._ip_scale_value() if ip is not None else 0.0
        if ip is None or scale == 0.0:  # `out + 0 * out_ip` (reference :287)
            return super()._finish(o, q, batch, nq, residual)
        ip2d, nk = ip
        inner = self.to_q.out_features
        h, d = self.heads, inner // self.heads
        nk_pad = (nk + 7) // 8 * 8
        k_ip = torch.empty((batch * nk, inner), device=q.device, dtype=torch.float16)
        # the key padding (4 -> 8) is neither written by the projection nor read by ops.attention (its V^T map ends at
        # key nk); the zero fill is not needed for correctness
        vt_ip = ops.zeros((batch, h, d, nk_pad), q.device)
        w = self._cat_weight("kv_ip", [self.to_k_ip, self.to_v_ip])
        ops.gemm(ip2d, w, seg_outs=[k_ip, vt_ip], seg_width=inner, transposed=(0, 1, 0), rows_per_img=nk, head_dim=d,
                 tok_pad=nk_pad)
        o_ip = ops.attention(q, k_ip, vt_ip, batch, h, nq, nk, d)
        lin = self.to_out[0]
        wo_s = self._prep.get(("o_ip", scale, prepare.lora_key(lin)), prepare.linear_params(lin),
                              lambda: (self._out_weight().float() * scale).half().contiguous())
        return ops.gemm(o, self._out_weight(), a2=o_ip, w2=wo_s, bias=prepare.bias_f32(lin.bias), residual=residual)

    def forward(self, x, context=None, mask=None):
        if mask is not None:
            raise NotImplementedError("attention masks are not on the CtrLoRA path")
        if context is None:
            raise AssertionError("IPCrossAttention needs a context (reference :236)")
        txt, ip = split_context(context)
        b, n, _ = x.shape
        ip2d, nk_ip = (None, None) if ip is None else (to_f16_rows(ip), ip.shape[1])
        return self.run(to_f16_rows(x), b, n, to_f16_rows(txt), txt.shape[1], ip2d=ip2d, nk_ip=nk_ip).view(b, n, -1)


IPMemoryEfficientCrossAttention = IPCrossAttention  # the xformers variant (reference :339-420): same kernels here


class BasicTransformerBlock(_base.BasicTransformerBlock):
    ATTENTION_MODES = {"softmax": CrossAttention, "softmax-ip": IPCrossAttention,
                       "softmax-xformers": MemoryEfficientCrossAttention, "softmax-xformers-ip": IPMemoryEfficientCrossAttention}

    attn2_cls = IPCrossAttention  # reference :434-441

    def run(self, x2d, batch, n, ctx2d, nk, out=None, ip2d=None, nk_ip=None):
        c1 = (ctx2d, nk) if self.disable_self_attn else (None, None)
        x2d = self.attn1.run(self._ln(self.norm1, x2d), batch, n, c1[0], c1[1], residual=x2d)
        x2d = self.attn2.run(self._ln(self.norm2, x2d), batch, n, ctx2d, nk, residual=x2d, ip2d=ip2d, nk_ip=nk_ip)
        return self.ff.run(self._ln(self.norm3, x2d), residual=x2d, out=out)

    def forward(self, x, context=None):
        txt, ip = split_context(context)
        b, n, _ = x.shape
        ctx2d, nk = (None, None) if txt is None else (to_f16_rows(txt), txt.shape[1])
        ip2d, nk_ip = (None, None) if ip is None else (to_f16_rows(ip), ip.shape[1])
        return self.run(to_f16_rows(x), b, n, ctx2d, nk, ip2d=ip2d, nk_ip=nk_ip).view(b, n, -1)


class SpatialTransformer(_base.SpatialTransformer):
    """reference :456-538; `context` is a tensor, a list with one entry per transformer block, and every entry may be
    the pair [text, ip] (cldm/cldm_ctrlora_style_inference.py:184-187)."""

    block_cls = BasicTransformerBlock

    def forward(self, x, context=None):
        xp = pixel_major(x)  # [B, H, W, C]
        b, h, w, c = xp.shape
        if not isinstance(context, list):
            context = [context]
        gn = prepare.effective(self.norm)
        xn = ops.groupnorm(xp, prepare.bias_f32(gn.weight), prepare.bias_f32(gn.bias), gn.eps, False, groups=gn.num_groups)
        y = ops.gemm(xn, self._w("in", self.proj_in), bias=prepare.bias_f32(self.proj_in.bias))
        y2d = y.view(b * h * w, -1)
        for i, block in enumerate(self.transformer_blocks):
            txt, ip = split_context(context[i] if i < len(context) else context[-1])
            ctx2d, nk = (None, None) if txt is None else (to_f16_rows(txt), txt.shape[1])
            ip2d, nk_ip = (None, None) if ip is None else (to_f16_rows(ip), ip.shape[1])
            y2d = block.run(y2d, b, h * w, ctx2d, nk, ip2d=ip2d, nk_ip=nk_ip)
        out = ops.gemm(y2d.view(b, h, w, -1), self._w("out", self.proj_out), bias=prepare.bias_f32(self.proj_out.bias),
                       residual=xp.view(b * h * w, c))
        return nchw_view(out)
