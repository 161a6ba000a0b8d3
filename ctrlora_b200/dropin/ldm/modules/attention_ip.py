"""IP-Adapter / InstantStyle cross-attention (reference ldm/modules/attention_ip.py): a second key / value stream
`to_k_ip / to_v_ip` over the image-prompt tokens, attended with the same queries and added with `ip_scale`
(reference :196-289).  Everything else is ldm/modules/attention.py (the reference's file is a copy of it too).

    out = to_out( softmax(q k^T) v  +  ip_scale * softmax(q k_ip^T) v_ip )

Here the second stream reuses the projected queries, runs the single-tile attention kernel over the (4 .. 16) image
tokens, and its output enters `to_out` as the SECOND OPERAND PAIR of the same wgmma GEMM
(o @ Wo^T + o_ip @ (ip_scale Wo)^T accumulate in one register tile): no separate add pass, no extra rounding of the sum.
The layers run the bodies of ldm/modules/attention.py: `SpatialTransformer.block_context` splits each block's context
entry into the text tokens and the image tokens, which reach `IPCrossAttention._finish` as arguments of `attn2.run`.
"""
import torch
import torch.nn as nn

from ctrlora_b200 import ops, prepare
from ctrlora_b200.runtime import to_f16_rows
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

    def _finish(self, o, q, batch, nq, residual, other=None, ip2d=None, nk_ip=None):
        """to_out(o + ip_scale * attention of q over the image tokens ip2d [batch*nk_ip, Cctx]) (+ residual)"""
        scale = self._ip_scale_value() if ip2d is not None else 0.0
        if ip2d is None or scale == 0.0:  # `out + 0 * out_ip` (reference :287)
            return super()._finish(o, q, batch, nq, residual, other)
        assert other is None, "the IP-Adapter cross-attention has no grouped (twin) variant"
        inner = self.to_q.out_features
        h, d = self.heads, inner // self.heads
        nk_pad = (nk_ip + 7) // 8 * 8
        k_ip = torch.empty((batch * nk_ip, inner), device=q.device, dtype=torch.float16)
        # the key padding (4 -> 8) is neither written by the projection nor read by ops.attention (its V^T map ends at
        # key nk); the zero fill is not needed for correctness
        vt_ip = ops.zeros((batch, h, d, nk_pad), q.device)
        w = self._cat_weight("kv_ip", [self.to_k_ip, self.to_v_ip])
        ops.gemm(ip2d, w, seg_outs=[k_ip, vt_ip], seg_width=inner, transposed=(0, 1, 0), rows_per_img=nk_ip, head_dim=d,
                 tok_pad=nk_pad)
        o_ip = ops.attention(q, k_ip, vt_ip, batch, h, nq, nk_ip, d)
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

    def forward(self, x, context=None):
        b, n, _ = x.shape
        ctx2d, nk, attn2_kw = SpatialTransformer.block_context(context)
        return self.run(to_f16_rows(x), b, n, ctx2d, nk, **attn2_kw).view(b, n, -1)


class SpatialTransformer(_base.SpatialTransformer):
    """reference :456-538; `context` is a tensor, a list with one entry per transformer block, and every entry may be
    the pair [text, ip] (cldm/cldm_ctrlora_style_inference.py:184-187)."""

    block_cls = BasicTransformerBlock

    @staticmethod
    def block_context(ctx):
        txt, ip = split_context(ctx)
        ctx2d, nk, _ = _base.SpatialTransformer.block_context(txt)
        return ctx2d, nk, {} if ip is None else {"ip2d": to_f16_rows(ip), "nk_ip": ip.shape[1]}
