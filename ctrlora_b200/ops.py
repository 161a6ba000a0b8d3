"""Tensor-level wrappers over the C ABI.  torch is used for device memory and the current stream only.

Layout convention: activations are fp16 "pixel-major" tensors, either [B, H, W, C] or [M, C]; the channel dim is
contiguous.  Weights are prepared once (see ctrlora_b200.prepare) as fp16 [N, taps, Cin].
"""
import ctypes as C

import torch

from . import _lib
from ._lib import GemmArgs, check


LAUNCHES = 0      # kernels launched through this module since the last reset (bench.py's gpu_launches)
_GEMM_PROFILE = None  # list of (flops, start_event, end_event) while profile_gemm() is active
_GEMM_SHAPES = None   # optional parallel list of problem shapes (tools/profile_step.py)
_GEMM_RECORD = None   # list of (args struct, flops, keep-alive tensors) while replay_gemms() records a step


def _count(n=1):
    global LAUNCHES
    LAUNCHES += n


def _ungraphed(fn, sampler):
    old = getattr(sampler, "use_cuda_graph", False)
    if sampler is not None:
        sampler.use_cuda_graph = False
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        if sampler is not None:
            sampler.use_cuda_graph = old


def count_launches(fn, sampler=None):
    """Kernel launches of one call of `fn` (run without CUDA-graph replay so every C-ABI call is seen)."""
    global LAUNCHES
    LAUNCHES = 0
    _ungraphed(fn, sampler)
    return LAUNCHES


def profile_gemm(fn, sampler=None):
    """Per-launch CUDA-event timing of every ctrlora_gemm_f16 launch inside `fn`: algorithmic flops and device ms."""
    global _GEMM_PROFILE
    _GEMM_PROFILE = []
    try:
        _ungraphed(fn, sampler)
        recs = _GEMM_PROFILE
    finally:
        _GEMM_PROFILE = None
    return {"launches": len(recs), "flops": float(sum(r[0] for r in recs)),
            "ms": float(sum(r[1].elapsed_time(r[2]) for r in recs))}


def replay_gemms(fn, sampler=None, reps=5):
    """Device time of the GEMM launches of `fn` replayed back to back from one CUDA graph.

    `fn` runs once un-graphed while every ctrlora_gemm_f16 argument block is recorded (its tensors are kept alive), then
    exactly those launches are captured into a graph and replayed `reps` times between two CUDA events on the capture
    stream.  Unlike per-launch events on an un-graphed step (host-bound: the GPU idles between launches, clocks and L2
    state differ from the real run) this times the kernels under the conditions they run in: PDL-chained, warm clocks.
    Returns {"launches", "flops", "ms"} for ONE pass over the step's GEMMs."""
    global _GEMM_RECORD
    _GEMM_RECORD = []
    try:
        _ungraphed(fn, sampler)
        recs = _GEMM_RECORD
    finally:
        _GEMM_RECORD = None
    lib = _lib.load()

    def launch_all():
        sp = _sp()
        for args, _, _ in recs:
            check(lib.ctrlora_gemm_f16(C.addressof(args), sp), "ctrlora_gemm_f16 (replay)")

    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        launch_all()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            launch_all()
        graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            graph.replay()
        e1.record()
    torch.cuda.current_stream().wait_stream(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    out = {"launches": len(recs), "flops": float(sum(r[1] for r in recs)), "ms": float(ms)}
    del graph, recs
    return out


_SPLITK = {}  # device index -> (fp32 workspace, uint32 counters); zero on entry and on exit of every GEMM launch
SPLITK_WS_BYTES = 128 << 20  # one fp32 [1280, 9*1280] dense-conv gradient slice is 59 MB
SPLITK_COUNTERS = 4096


def _splitk_buffers(device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    if key not in _SPLITK:
        _SPLITK[key] = (torch.zeros(SPLITK_WS_BYTES // 4, device=device, dtype=torch.float32),
                        torch.zeros(SPLITK_COUNTERS, device=device, dtype=torch.int32))
    return _SPLITK[key]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.CtrloraError("ctrlora_b200 ops need CUDA tensors (sm_90a); there is no CPU path")


def _as_bhwc(a):
    if a.dim() == 2:
        return 1, 1, a.shape[0], a.shape[1], a.stride(0)
    assert a.dim() == 4 and a.stride(3) == 1
    b, h, w, c = a.shape
    ld = a.stride(2)
    assert a.stride(1) == w * ld and a.stride(0) == h * w * ld, "pixel-major layout required"
    return b, h, w, c, ld


def gemm(a, w, *, ksize=1, bias=None, rowbias=None, rows_per_img=0, rowbias_ld=0, residual=None, out_scale=1.0, a2=None,
         w2=None,
         geglu=False, out=None, out_f32=False, seg_outs=None, seg_width=0, transposed=(0, 0, 0), head_dim=0,
         tok_pad=0, block_n=0, split_k=0, dup_out=None, single_cta=False, simt=False, hi=None):
    """out = epilogue(conv_or_linear(a, w) [+ a2 @ w2^T]); see `ctrlora_gemm_f16` in include/ctrlora_b200.h.

    a: fp16 [B,H,W,C] or [M,K]; w: fp16 [N(2N), ksize*ksize, C]; returns the output tensor ([..., N]).
    hi: grouped launch of two same-shaped layers over the two halves of the batch (images of a [B,H,W,C] `a`, rows of
    an [M,K] one): a dict with the upper half's "w" and, as the call has them, "bias", "rowbias" (indexed from the
    half's first image) and "w2".  A batch whose halves cannot be tiled apart runs as two launches.
    """
    return _gemm(a, w, ksize=ksize, bias=bias, rowbias=rowbias, rows_per_img=rows_per_img, rowbias_ld=rowbias_ld,
                 residual=residual, out_scale=out_scale, a2=a2, w2=w2, geglu=geglu, out=out, out_f32=out_f32,
                 seg_outs=seg_outs, seg_width=seg_width, transposed=transposed, head_dim=head_dim, tok_pad=tok_pad,
                 block_n=block_n, split_k=split_k, dup_out=dup_out, single_cta=single_cta, simt=simt, hi=hi)


def gemm_relu(a, w, **kwargs):
    """ops.gemm (same arguments) with max(., 0) as the epilogue's last step, before the output rounding: a conv + ReLU
    pair in one launch.  A function of its own, so that gemm's arguments stay those of its fp32 launch reference."""
    return _gemm(a, w, relu=True, **kwargs)


def gemm_relu6(a, w, **kwargs):
    """ops.gemm (same arguments) with min(max(., 0), 6) as the epilogue's last step, before the output rounding: a conv
    + BatchNorm + ReLU6 (MobileNetV2's ConvBNReLU) in one launch"""
    return _gemm(a, w, relu=2, **kwargs)


def gemm_relu_residual(a, w, *, residual, **kwargs):
    """ops.gemm (same arguments) with max(., 0) taken before the residual add: relu(conv(a)) + residual in one launch
    (M-LSD's BlockTypeB conv1)"""
    return _gemm(a, w, relu=3, residual=residual, **kwargs)


def _gemm(a, w, *, ksize=1, bias=None, rowbias=None, rows_per_img=0, rowbias_ld=0, residual=None, out_scale=1.0, a2=None,
          w2=None, geglu=False, out=None, out_f32=False, seg_outs=None, seg_width=0, transposed=(0, 0, 0), head_dim=0,
          tok_pad=0, block_n=0, split_k=0, dup_out=None, single_cta=False, simt=False, hi=None, relu=False):
    _require_cuda(a, w)
    assert a.dtype == torch.float16 and w.dtype == torch.float16 and w.is_contiguous()
    n_rows = w.shape[0]
    n = n_rows // 2 if geglu else n_rows
    if out is None and seg_outs is None:
        out = torch.empty(a.shape[:-1] + (n,), device=a.device, dtype=torch.float32 if out_f32 else torch.float16)
    a4, out4 = a, out
    if hi is not None:
        assert a.shape[0] % 2 == 0
        if a.dim() == 2:  # the two halves of the rows are two images
            a4 = a.view(2, 1, a.shape[0] // 2, a.shape[1])
            out4 = None if out is None else out.view(a4.shape[:3] + (out.shape[-1],))
    b, h, wd, c, ld = _as_bhwc(a4)
    assert w.numel() == n_rows * ksize * ksize * c, (w.shape, ksize, c)
    M = b * h * wd
    args = GemmArgs()
    args.a, args.a_b, args.a_h, args.a_w, args.a_c, args.a_ld = _ptr(a4), b, h, wd, c, ld
    args.w, args.kh, args.kw, args.pad = _ptr(w), ksize, ksize, (ksize - 1) // 2
    if a2 is not None:
        b2, h2, w2d, c2, ld2 = _as_bhwc(a2)
        assert (b2, h2, w2d) == (b, h, wd) and w2.dtype == torch.float16 and w2.is_contiguous()
        args.a2, args.a2_c, args.a2_ld, args.w2 = _ptr(a2), c2, ld2, _ptr(w2)
    args.n, args.block_n, args.geglu = n, block_n, int(geglu)
    if seg_outs is not None:
        ldc = seg_width
        for i, o in enumerate(seg_outs):
            args.out[i] = o.data_ptr()
            args.transposed[i] = int(transposed[i])
        ret = list(seg_outs)
    else:
        assert out4.stride(-1) == 1
        ldc = out4.stride(-2)
        args.out[0] = out4.data_ptr()
        ret = out
    args.seg_width, args.ldc, args.out_f32 = seg_width, ldc, int(out_f32)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == n_rows
    if rowbias is not None:
        assert rowbias.dtype == torch.float32 and rowbias.stride(-1) == 1
        rowbias_ld = rowbias_ld or rowbias.stride(0)
    args.bias, args.rowbias, args.rows_per_img, args.rowbias_ld = _ptr(bias), _ptr(rowbias), rows_per_img, rowbias_ld
    if residual is not None:
        assert residual.dtype in (torch.float16, torch.float32) and residual.stride(-1) == 1
        args.residual, args.ldr = _ptr(residual), residual.stride(-2)
        args.residual_f32 = int(residual.dtype == torch.float32)
    args.out_scale, args.head_dim, args.tok_pad, args.bf16 = float(out_scale), head_dim, tok_pad, 0
    ws, cnt = _splitk_buffers(a.device)
    args.split_k, args.splitk_ws, args.splitk_ws_bytes = split_k, ws.data_ptr(), SPLITK_WS_BYTES
    args.splitk_counters, args.splitk_counters_len = cnt.data_ptr(), SPLITK_COUNTERS
    if dup_out is not None:
        args.dup_out, args.dup_ld = dup_out.data_ptr(), dup_out.stride(0)
    args.force_single_cta = int(single_cta)
    args.relu = int(relu)
    if hi is not None:
        if hi.get("rowbias") is not None:  # the kernel reads both halves' row terms with the lower half's row stride
            assert rowbias is not None and hi["rowbias"].stride(0) == rowbias.stride(0) and \
                hi["rowbias"].stride(-1) == 1, "the two halves' row terms need one row stride"
        args.group_b, args.w_hi, args.w2_hi = b // 2, _ptr(hi["w"]), _ptr(hi.get("w2"))
        args.bias_hi, args.rowbias_hi = _ptr(hi.get("bias")), _ptr(hi.get("rowbias"))
    lib = _lib.load()
    shape = {"B": b, "H": h, "W": wd, "C": c, "N": n_rows, "ksize": ksize, "geglu": int(geglu),
             "c2": int(args.a2_c) if a2 is not None else 0, "segs": seg_width, "res": int(residual is not None)}
    keep = (a, w, a2, w2, bias, rowbias, residual, out, seg_outs, dup_out, ws, cnt, hi)
    if _launch_gemm(lib.ctrlora_gemm_f16_simt if simt else lib.ctrlora_gemm_f16, args, simt, shape, keep):
        return ret
    # a tile would straddle the halves: one plain launch per half, over the rows of the row-indexed operands and the
    # images of the V^T-layout segments
    half = a.shape[0] // 2
    rows = half if a.dim() == 2 else half * a.shape[1] * a.shape[2]
    imgs = rows // (rows_per_img or rows)

    def cut(t, lo, by_image=False):
        if t is None:
            return None
        n = imgs if by_image else (half if t.dim() == 4 else rows)
        return t[:n] if lo else t[n:]

    for lo in (True, False):
        segs = None if seg_outs is None else [cut(o, lo, by_image=bool(t)) for o, t in zip(seg_outs, transposed)]
        _gemm(cut(a, lo), w if lo else hi["w"], ksize=ksize, bias=bias if lo else hi.get("bias"),
              rowbias=rowbias if lo else hi.get("rowbias"), rows_per_img=rows_per_img, rowbias_ld=rowbias_ld,
              residual=cut(residual, lo), out_scale=out_scale, a2=cut(a2, lo), w2=w2 if lo else hi.get("w2"),
              geglu=geglu, out=cut(out, lo), out_f32=out_f32, seg_outs=segs, seg_width=seg_width, transposed=transposed,
              head_dim=head_dim, tok_pad=tok_pad, block_n=block_n, split_k=split_k, relu=relu)
    return ret


def _launch_gemm(fn, args, simt, shape, keep):
    """One ctrlora_gemm_f16 / ctrlora_gemm_f16_simt launch with its bookkeeping: the launch count, and for the wgmma
    kernel the replay_gemms record and the profile_gemm timing.  Returns False when a grouped launch is refused as
    UNSUPPORTED (nothing was launched); raises on any other error."""
    flops = 2.0 * shape["B"] * shape["H"] * shape["W"] * shape["N"] * (shape["ksize"] ** 2 * shape["C"] + shape["c2"])
    timed = _GEMM_PROFILE is not None and not simt
    if timed:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rc = fn(C.addressof(args), _sp())
    if rc == _lib.STATUS_UNSUPPORTED and args.group_b:
        return False
    check(rc, "ctrlora_gemm_f16")
    _count()
    if _GEMM_RECORD is not None and not simt:
        _GEMM_RECORD.append((args, flops, keep))
    if timed:
        e1.record()
        _GEMM_PROFILE.append((flops, e0, e1))
        if _GEMM_SHAPES is not None:
            _GEMM_SHAPES.append(shape)
    return True


def _dp(t):
    """raw device pointer (or NULL) for argtypes-declared entry points"""
    return t.data_ptr() if t is not None else None


def _sp():
    return torch.cuda.current_stream().cuda_stream


_GN_PARTIAL = {}  # device index -> (fp32 scratch for per-block partial statistics, uint32 self-cleaning arrival counters)
GN_PARTIAL_FLOATS = 1 << 19
GN_PARTIAL_COUNTERS = 256


def _gn_partial_buffers(device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    if key not in _GN_PARTIAL:
        if torch.cuda.is_current_stream_capturing():  # it would live in that graph's private pool
            raise _lib.CtrloraError("the GroupNorm partial-statistics scratch is allocated on the first call on a device; "
                                    "make one un-captured GroupNorm call before capturing a graph")
        _GN_PARTIAL[key] = (torch.empty(GN_PARTIAL_FLOATS, device=device, dtype=torch.float32),
                            torch.zeros(GN_PARTIAL_COUNTERS, device=device, dtype=torch.int32))
    return _GN_PARTIAL[key]


def _gn_args(x1, gamma, beta, eps, silu, add1, add1_scale, x2, add2, add2_scale, groups):
    """GroupNormArgs of a groupnorm / groupnorm_bwd call: the source description and the partial-statistics scratch
    (the forward's and the backward's are one buffer: bit-reproducible dx); the caller sets the statistics workspace"""
    b, h, w, c1, ld1 = _as_bhwc(x1)
    c2, ld2 = 0, 0
    if x2 is not None:
        b2, h2, w2, c2, ld2 = _as_bhwc(x2)
        assert (b2, h2, w2) == (b, h, w)
    a = _lib.GroupNormArgs()
    a.x1, a.add1, a.add1_scale, a.c1, a.ld1 = _dp(x1), _dp(add1), float(add1_scale), c1, ld1
    a.x2, a.add2, a.add2_scale, a.c2, a.ld2 = _dp(x2), _dp(add2), float(add2_scale), c2, ld2
    a.batch, a.hw, a.groups = b, h * w, groups
    a.gamma, a.beta, a.eps, a.silu = _dp(gamma), _dp(beta), float(eps), int(silu)
    pws, pcnt = _gn_partial_buffers(x1.device)
    a.partial_ws, a.partial_ws_floats = _dp(pws), GN_PARTIAL_FLOATS
    a.partial_counters, a.partial_counters_len = _dp(pcnt), GN_PARTIAL_COUNTERS
    return a, (b, h, w, c1, c2)


def groupnorm(x1, gamma, beta, eps, silu, *, add1=None, add1_scale=1.0, x2=None, add2=None, add2_scale=1.0,
              groups=32, want_raw=False, want_stats=False, out=None, gamma_hi=None, beta_hi=None):
    """GroupNorm(+SiLU) over [x1 (+s1*add1) | x2 (+s2*add2)], pixel-major fp16 [B,H,W,C*]; returns y (and raw concat).
    gamma_hi / beta_hi: the affine parameters of the upper half of the batch (two networks' layers in one launch)."""
    _require_cuda(x1, x2, add1, add2)
    a, (b, h, w, c1, c2) = _gn_args(x1, gamma, beta, eps, silu, add1, add1_scale, x2, add2, add2_scale, groups)
    for ad, ref in ((add1, x1), (add2, x2)):
        if ad is not None:
            assert ad.shape == ref.shape and ad.stride() == ref.stride() and ad.dtype == torch.float16
    ctot = c1 + c2
    y = torch.empty((b, h, w, ctot), device=x1.device, dtype=torch.float16) if out is None else out
    assert y.shape == (b, h, w, ctot) and y.is_contiguous() and y.dtype == torch.float16
    raw = torch.empty_like(y) if want_raw else None
    stats_ws = torch.empty(b * groups * 2, device=x1.device, dtype=torch.float32)
    a.stats_ws = _dp(stats_ws)
    assert gamma.dtype == torch.float32 and beta.dtype == torch.float32 and gamma.numel() == ctot
    if gamma_hi is not None:
        assert b % 2 == 0 and gamma_hi.numel() == ctot and beta_hi.numel() == ctot
        a.gamma_hi, a.beta_hi, a.group_b = _dp(gamma_hi), _dp(beta_hi), b // 2
    a.y, a.raw_out = _dp(y), _dp(raw)
    _count(2)
    check(_lib.load().ctrlora_groupnorm_f16(C.addressof(a), _sp()), "ctrlora_groupnorm_f16")
    if want_stats:
        return (y, raw, stats_ws) if want_raw else (y, stats_ws)
    return (y, raw) if want_raw else y


def zeros(shape, device, dtype=torch.float16):
    """torch.empty + cudaMemsetAsync (a memset node; torch.zeros launches an ATen fill kernel)"""
    t = torch.empty(shape, device=device, dtype=dtype)
    check(_lib.load().ctrlora_memset_zero(_dp(t), t.numel() * t.element_size(), _sp()), "memset_zero")
    return t


def layernorm(x, gamma, beta, eps=1e-5, gamma_hi=None, beta_hi=None):
    """x fp16 [..., C] with contiguous last dim and uniform row stride.  gamma_hi / beta_hi: the affine parameters of the
    upper half of the rows (two networks' layers in one launch)."""
    _require_cuda(x)
    cols = x.shape[-1]
    x2 = x.reshape(-1, cols)
    y = torch.empty((x2.shape[0], cols), device=x.device, dtype=torch.float16)
    _count(1)
    if gamma_hi is not None:
        assert x2.shape[0] % 2 == 0
        check(_lib.load().ctrlora_layernorm_grouped_f16(_dp(x2), x2.stride(0), _dp(y), cols, x2.shape[0], cols, _dp(gamma),
                                                        _dp(beta), _dp(gamma_hi), _dp(beta_hi), x2.shape[0] // 2,
                                                        float(eps), _sp()), "ctrlora_layernorm_grouped_f16")
        return y.view(x.shape)
    check(_lib.load().ctrlora_layernorm_f16(_dp(x2), x2.stride(0), _dp(y), cols, x2.shape[0], cols, _dp(gamma), _dp(beta),
                                            float(eps), _sp()), "ctrlora_layernorm_f16")
    return y.view(x.shape)


def attention(q, k, vt, batch, heads, nq, nk, head_dim, out=None, lse=None):
    """q [batch*nq, heads*d], k [batch*nk, heads*d], vt [batch, heads, d, nk_pad] (fp16) -> [batch*nq, heads*d]."""
    _require_cuda(q, k, vt)
    if out is None:
        out = torch.empty((batch * nq, heads * head_dim), device=q.device, dtype=torch.float16)
    _count(1)
    check(_lib.load().ctrlora_attention_f16(_dp(q), q.stride(0), _dp(k), k.stride(0), _dp(vt), vt.shape[-1], _dp(out),
                                            out.stride(0), _dp(lse), batch, heads, nq, nk, head_dim, _sp()),
          "ctrlora_attention_f16")
    return out


def nchw_to_nhwc_f16(x, c_pad=None, out=None):
    """fp32 [B,C,H,W] contiguous -> fp16 [B,H,W,c_pad] (zero-padded channels)."""
    _require_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous()
    b, c, h, w = x.shape
    c_pad = c_pad or c
    y = torch.empty((b, h, w, c_pad), device=x.device, dtype=torch.float16) if out is None else out
    assert y.shape == (b, h, w, c_pad) and y.is_contiguous() and y.dtype == torch.float16
    _count(1)
    check(_lib.load().ctrlora_nchw_f32_to_nhwc_f16(_dp(x), _dp(y), b, c, h * w, c_pad, _sp()), "nchw_to_nhwc")
    return y


def nhwc_to_nchw_f32(x, channels=None):
    """[B,H,W,ld] fp16/fp32 pixel-major -> fp32 [B,channels,H,W]."""
    _require_cuda(x)
    b, h, w, c, ld = _as_bhwc(x)
    channels = channels or c
    y = torch.empty((b, channels, h, w), device=x.device, dtype=torch.float32)
    _count(1)
    check(_lib.load().ctrlora_nhwc_to_nchw_f32(_dp(x), int(x.dtype == torch.float32), ld, _dp(y), b, channels, h * w,
                                               _sp()), "nhwc_to_nchw")
    return y


def timestep_embedding(t, freqs):
    """t int64 or fp32 [B] (device), freqs fp32 [half] (device) -> fp32 [B, 2*half].  int64 t takes the integer kernel;
    fp32 t (DPM-Solver's fractional model times) takes ctrlora_timestep_embedding_f32, never a truncation."""
    _require_cuda(t, freqs)
    assert t.dtype in (torch.int64, torch.float32) and freqs.dtype == torch.float32
    out = torch.empty((t.shape[0], 2 * freqs.shape[0]), device=t.device, dtype=torch.float32)
    fn = _lib.load().ctrlora_timestep_embedding if t.dtype == torch.int64 else _lib.load().ctrlora_timestep_embedding_f32
    _count(1)
    check(fn(_dp(t), _dp(freqs), _dp(out), t.shape[0], freqs.shape[0], _sp()), "timestep_embedding")
    return out


def small_linear(x, w, bias, silu_in=False, silu_out=False, out=None):
    """x fp32 [rows, K] (row stride free), w fp16 [N, K] -> fp32 [rows, N]"""
    _require_cuda(x, w)
    assert x.dtype == torch.float32 and w.dtype == torch.float16 and w.is_contiguous() and x.stride(1) == 1
    rows, k = x.shape
    n = w.shape[0]
    if out is None:
        out = torch.empty((rows, n), device=x.device, dtype=torch.float32)
    _count(1)
    check(_lib.load().ctrlora_small_linear(_dp(x), x.stride(0), _dp(w), _dp(bias), _dp(out), out.stride(0), rows, n, k,
                                           int(silu_in), int(silu_out), _sp()), "small_linear")
    return out


def upsample2x(x):
    _require_cuda(x)
    assert x.is_contiguous() and x.dtype == torch.float16
    b, h, w, c = x.shape
    y = torch.empty((b, 2 * h, 2 * w, c), device=x.device, dtype=torch.float16)
    _count(1)
    check(_lib.load().ctrlora_upsample2x_f16(_dp(x), _dp(y), b, h, w, c, _sp()), "upsample2x")
    return y


def im2col_s2(x, pad_lo=1):
    """stride-2 3x3 gather; pad_lo=1: Conv2d(padding=1); pad_lo=0: zeros on the right/bottom only (the VAE's Downsample)"""
    _require_cuda(x)
    assert x.is_contiguous() and x.dtype == torch.float16
    b, h, w, c = x.shape
    y = torch.empty((b, h // 2, w // 2, 9 * c), device=x.device, dtype=torch.float16)
    _count(1)
    check(_lib.load().ctrlora_im2col_s2_pad_f16(_dp(x), _dp(y), b, h, w, c, int(pad_lo), _sp()), "im2col_s2")
    return y


def softmax_rows(logits, scale=1.0):
    """fp32 [rows, cols] -> fp16 softmax(scale * logits) over the last dim"""
    _require_cuda(logits)
    assert logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
    out = torch.empty(logits.shape, device=logits.device, dtype=torch.float16)
    _count(1)
    check(_lib.load().ctrlora_softmax_rows_f32_to_f16(_dp(logits), logits.stride(0), _dp(out), out.stride(0), logits.shape[0],
                                                      logits.shape[1], float(scale), _sp()), "softmax_rows")
    return out


def gaussian_sample(moments, noise=None, scale=1.0):
    """moments fp32 [B, 2Z, H, W] -> scale * (mean + std * noise) (noise None: scale * mean), fp32 [B, Z, H, W]"""
    _require_cuda(moments, noise)
    moments = moments.float().contiguous()
    b, z2, h, w = moments.shape
    out = torch.empty((b, z2 // 2, h, w), device=moments.device, dtype=torch.float32)
    if noise is not None:
        noise = noise.float().contiguous()
        assert noise.shape == out.shape
    _count(1)
    check(_lib.load().ctrlora_gaussian_sample(_dp(moments), _dp(noise), _dp(out), b, z2 // 2, h * w, float(scale), _sp()),
          "gaussian_sample")
    return out


def cast_transpose(src, batch, rows, cols, out=None):
    """fp32 [batch, rows, cols] -> fp16 [batch, cols, rows]"""
    _require_cuda(src)
    assert src.dtype == torch.float32 and src.is_contiguous() and src.numel() == batch * rows * cols
    if out is None:
        out = torch.empty((batch, cols, rows), device=src.device, dtype=torch.float16)
    _count(1)
    check(_lib.load().ctrlora_cast_transpose_f32_to_f16(_dp(src), _dp(out), batch, rows, cols, _sp()), "cast_transpose")
    return out


def ddim_update(x, e_cond, e_uncond, cfg_scale, a_t, a_prev, sigma_t, sqrt_one_minus_at, noise=None, temperature=1.0,
                stats=None):
    """One DDIM update (cldm/ddim_hacked.py:190-231). fp32 [B,C,H,W] contiguous tensors; returns (x_prev, pred_x0)."""
    _require_cuda(x, e_cond, e_uncond, noise)
    for t in (x, e_cond, e_uncond, noise):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.shape == x.shape)
    x_prev, pred_x0 = torch.empty_like(x), torch.empty_like(x)
    b = x.shape[0]
    _count(1)
    check(_lib.load().ctrlora_ddim_update(_dp(x), _dp(e_cond), _dp(e_uncond), _dp(noise), _dp(x_prev), _dp(pred_x0),
                                          _dp(stats), b, x[0].numel(), float(cfg_scale), float(a_t), float(a_prev),
                                          float(sigma_t), float(sqrt_one_minus_at), float(temperature), _sp()),
          "ddim_update")
    return x_prev, pred_x0


def im2col_3x3(x):
    """fp16 [B,H,W,C] -> [B,H,W,9*C] (stride 1, pad 1; tap-major like the conv kernel weights)"""
    _require_cuda(x)
    assert x.is_contiguous() and x.dtype == torch.float16
    b, h, w, c = x.shape
    y = torch.empty((b, h, w, 9 * c), device=x.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_im2col_3x3_f16(_dp(x), _dp(y), b, h, w, c, _sp()), "im2col_3x3")
    return y


def outer_accum(dy, x, out, alpha=1.0, beta=1.0, silu_x=False):
    """out[n, k] = beta*out + alpha * sum_b dy[b, n] f(x[b, k])  (fp32 [B,N], [B,K] -> fp32 [N,K], row strides free)"""
    _require_cuda(dy, x, out)
    assert dy.dtype == x.dtype == out.dtype == torch.float32 and dy.stride(1) == 1 and x.stride(1) == 1 and out.stride(1) == 1
    rows, n = dy.shape
    k = x.shape[1]
    assert x.shape[0] == rows and out.shape == (n, k)
    _count()
    check(_lib.load().ctrlora_outer_accum_f32(_dp(dy), dy.stride(0), _dp(x), x.stride(0), _dp(out), out.stride(0), rows, n, k,
                                              float(alpha), float(beta), int(silu_x), _sp()), "outer_accum")
    return out


def copy2d(src, dst, rows, cols, lds, ldd, accumulate=False):
    """dst[r, c] (+)= src[r, c] over fp32 [rows, cols] blocks with explicit row strides"""
    _require_cuda(src, dst)
    assert src.dtype == dst.dtype == torch.float32
    _count()
    check(_lib.load().ctrlora_copy2d_f32(_dp(src), lds, _dp(dst), ldd, rows, cols, int(accumulate), _sp()), "copy2d")
    return dst


def silu_bwd(d, x):
    """d * silu'(x), fp32"""
    _require_cuda(d, x)
    d, x = d.contiguous(), x.contiguous()
    out = torch.empty_like(d)
    _count()
    check(_lib.load().ctrlora_silu_bwd_f32(_dp(d), _dp(x), _dp(out), d.numel(), _sp()), "silu_bwd")
    return out


def cast_rows(src, rows, cols, lds):
    """fp32 [rows, cols] with row stride lds -> dense fp16 [rows, cols]"""
    _require_cuda(src)
    out = torch.empty((rows, cols), device=src.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_cast_rows_f32_to_f16(_dp(src), lds, _dp(out), rows, cols, _sp()), "cast_rows")
    return out


def q_sample(x0, noise, t, tab_a, tab_s):
    """tab_a[t] * x0 + tab_s[t] * noise (fp32 [B,...] contiguous; t int64 [B]; tables fp32 on the device). Bit-exact."""
    _require_cuda(x0, noise, t, tab_a, tab_s)
    x0, noise = x0.float().contiguous(), noise.float().contiguous()
    assert t.dtype == torch.int64 and tab_a.dtype == torch.float32 and tab_s.dtype == torch.float32
    assert x0.shape == noise.shape and t.numel() == x0.shape[0]
    out = torch.empty_like(x0)
    _count()
    check(_lib.load().ctrlora_q_sample(_dp(x0), _dp(noise), _dp(t.contiguous()), _dp(tab_a.contiguous()),
                                       _dp(tab_s.contiguous()), _dp(out), x0.shape[0], x0[0].numel(), _sp()), "q_sample")
    return out


def ddim_encode_update(x, e_cond, e_uncond, cfg_scale, c1, c2):
    """x_next = c1 * x + c2 * cfg(e_cond, e_uncond)   (DDIM inversion, cldm/ddim_hacked.py:253-267)"""
    _require_cuda(x, e_cond, e_uncond)
    x, e_cond = x.float().contiguous(), e_cond.float().contiguous()
    e_uncond = None if e_uncond is None else e_uncond.float().contiguous()
    out = torch.empty_like(x)
    _count()
    check(_lib.load().ctrlora_ddim_encode_update(_dp(x), _dp(e_cond), _dp(e_uncond), _dp(out), x.numel(), float(cfg_scale),
                                                 float(c1), float(c2), _sp()), "ddim_encode_update")
    return out


def dpm_multistep_update(x, e_cond, e_uncond, m_prev, m_out, cfg_scale, sigma_s, alpha_s, c_x, c_m, c_d=0.0, inv_r0=0.0):
    """One DPM-Solver++ multistep step (ldm/models/diffusion/dpm_solver/dpm_solver.py): writes the data prediction
    (x - sigma_s * e) / alpha_s into m_out and returns x_next; order 2 when m_prev is given, order 1 otherwise.
    fp32 contiguous [B,C,H,W] tensors; the scalars come from ctrlora_b200.dpm_schedule."""
    _require_cuda(x, e_cond, e_uncond, m_prev, m_out)
    for t in (x, e_cond, e_uncond, m_prev, m_out):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.shape == x.shape)
    x_next = torch.empty_like(x)
    _count()
    check(_lib.load().ctrlora_dpm_multistep_update(_dp(x), _dp(e_cond), _dp(e_uncond), _dp(m_prev), _dp(m_out), _dp(x_next),
                                                   x.numel(), float(cfg_scale), float(sigma_s), float(alpha_s), float(c_x),
                                                   float(c_m), float(c_d), float(inv_r0), _sp()), "dpm_multistep_update")
    return x_next


def plms_update(x, e_cond, e_uncond, e_out, cfg_scale, sqrt_a_t, sqrt_one_minus_at, sqrt_a_prev, dir_coef, old=(),
                e_next=None):
    """One PLMS step (ldm/models/diffusion/plms.py:178-244): writes the guided eps e_t into e_out and returns
    (x_prev, pred_x0).  e_next = (e_next_cond, e_next_uncond | None) gives step 0's average with the eval at t_next
    (order 0); otherwise `old` = (old_eps[-1], old_eps[-2], ...) of up to 3 earlier e_t selects the Adams-Bashforth
    order len(old) + 1.  fp32 contiguous [B,C,H,W] tensors; the scalars come from ctrlora_b200.plms_schedule."""
    assert len(old) <= 3 and (e_next is None or not old)
    en_c, en_u = (None, None) if e_next is None else e_next
    o = list(old) + [None] * (3 - len(old))
    _require_cuda(x, e_cond, e_uncond, e_out, en_c, en_u, *o)
    for t in (x, e_cond, e_uncond, e_out, en_c, en_u, *o):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.shape == x.shape)
    x_prev, pred_x0 = torch.empty_like(x), torch.empty_like(x)
    order = 0 if e_next is not None else len(old) + 1
    _count()
    check(_lib.load().ctrlora_plms_update(_dp(x), _dp(e_cond), _dp(e_uncond), _dp(en_c), _dp(en_u), _dp(o[0]), _dp(o[1]),
                                          _dp(o[2]), _dp(e_out), _dp(x_prev), _dp(pred_x0), order, x.numel(),
                                          float(cfg_scale), float(sqrt_a_t), float(sqrt_one_minus_at), float(sqrt_a_prev),
                                          float(dir_coef), _sp()), "plms_update")
    return x_prev, pred_x0


DPM_NCOEF = 9
DPM_MODEL_TYPES = {"noise": 0, "x_start": 1, "v": 2}
DPM_UPDATE_MODES = {"first": 0, "diff": 1, "multistep2": 2, "multistep3": 3, "singlestep3_taylor": 4}


def _dpm_coef(coef):
    vals = [float(v) for v in coef] + [0.0] * (DPM_NCOEF - len(coef))
    assert len(vals) == DPM_NCOEF
    return (C.c_float * DPM_NCOEF)(*vals)


def _dpm_like(x, *ts):
    _require_cuda(x, *ts)
    for t in (x,) + ts:
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.shape == x.shape), \
            "DPM-Solver kernels take fp32 contiguous tensors of x's shape"


def dpm_model_output(x, out_cond, m_out, model_type="noise", out_uncond=None, grad=None, predict_x0=False,
                     scale=1.0, alpha_w=1.0, sigma_w=1.0, grad_coef=0.0, sigma_t=1.0, alpha_t=1.0):
    """One DPM_Solver model value into m_out (ldm/models/diffusion/dpm_solver/dpm_solver.py:257-312, :352-359): the
    model output converted to noise, guided by out_uncond (classifier-free) or grad (classifier), and with predict_x0
    the data prediction (x - sigma_t e) / alpha_t.  Scalars from ctrlora_b200.dpm_schedule."""
    _dpm_like(x, out_cond, m_out, out_uncond, grad)
    _count()
    check(_lib.load().ctrlora_dpm_model_output(
        _dp(x), _dp(out_cond), _dp(out_uncond), _dp(grad), _dp(m_out), x.numel(), DPM_MODEL_TYPES[model_type],
        int(bool(predict_x0)), _dpm_coef((scale, alpha_w, sigma_w, grad_coef, sigma_t, alpha_t)), _sp()),
        "dpm_model_output")
    return m_out


def dpm_solver_update(mode, x, m0, coef, m1=None, m2=None, out=None):
    """One DPM_Solver update of the given mode (first / diff / multistep2 / multistep3 / singlestep3_taylor, see
    include/ctrlora_b200.h) with coef = (a, b, c, d, k0, k1, k2, k3, rd) from ctrlora_b200.dpm_schedule; returns x_t."""
    out = torch.empty_like(x) if out is None else out
    _dpm_like(x, m0, m1, m2, out)
    _count()
    check(_lib.load().ctrlora_dpm_solver_update(_dp(x), _dp(m0), _dp(m1), _dp(m2), _dp(out), x.numel(),
                                                DPM_UPDATE_MODES[mode], _dpm_coef(coef), _sp()), "dpm_solver_update")
    return out


def dpm_threshold_(x0, k_lo, k_hi, weight, max_val, s_out=None):
    """Dynamic thresholding of x0 [B, ...] in place (dpm_solver.py:360-364); k_lo / k_hi / weight locate torch.quantile's
    0.995 order statistics (ctrlora_b200.dpm_schedule.quantile_rank).  s_out [B] receives the per-image s."""
    _require_cuda(x0, s_out)
    assert x0.dtype == torch.float32 and x0.is_contiguous()
    _count()
    check(_lib.load().ctrlora_dpm_threshold(_dp(x0), _dp(s_out), x0.shape[0], x0[0].numel(), int(k_lo), int(k_hi),
                                            float(weight), float(max_val), _sp()), "dpm_threshold")
    return x0


def dpm_adaptive_error(x_lower, x_prev, x_higher, atol, rtol, err=None):
    """The adaptive solver's E (dpm_solver.py:926-928) as a one-element fp32 device tensor."""
    _dpm_like(x_lower, x_prev, x_higher)
    err = torch.empty(1, device=x_lower.device, dtype=torch.float32) if err is None else err
    _count()
    check(_lib.load().ctrlora_dpm_adaptive_error(_dp(x_lower), _dp(x_prev), _dp(x_higher), _dp(err), x_lower.shape[0],
                                                 x_lower[0].numel(), float(atol), float(rtol), _sp()),
          "dpm_adaptive_error")
    return err


def wgrad_tn(a, b, out=None, alpha=1.0, beta=0.0):
    """out[p, q] = alpha * sum_m a[m, p] * b[m, q] + beta * out  (fp16 a [M,P], b [M,Q] -> fp32 [P,Q])."""
    _require_cuda(a, b)
    assert a.dtype == torch.float16 and b.dtype == torch.float16 and a.stride(1) == 1 and b.stride(1) == 1
    m, pd = a.shape
    qd = b.shape[1]
    assert b.shape[0] == m
    if out is None:
        assert beta == 0.0
        out = torch.empty((pd, qd), device=a.device, dtype=torch.float32)
    ws, _ = _splitk_buffers(a.device)
    _count(2)
    check(_lib.load().ctrlora_wgrad_tn_f16(_dp(a), a.stride(0), _dp(b), b.stride(0), m, pd, qd, _dp(out), out.stride(0),
                                           float(alpha), float(beta), _dp(ws), SPLITK_WS_BYTES, _sp()), "ctrlora_wgrad_tn_f16")
    return out


# ------------------------------------------------------------------------------------------------ training kernels
def groupnorm_bwd(dy, fwd_stats, x1, gamma, beta, eps, silu, *, add1=None, add1_scale=1.0, x2=None, add2=None,
                  add2_scale=1.0, groups=32, want_dx2=False, dx2_scale=1.0, dgamma=None, dbeta=None, res=None, dx1_scale=1.0):
    """Backward of ops.groupnorm (same source description).  Returns dx1 (and dx2 scaled by dx2_scale if want_dx2);
    dgamma/dbeta (fp32 [C]) are accumulated into when given."""
    _require_cuda(dy, x1)
    assert dy.dtype == torch.float16 and dy.is_contiguous()
    ws = torch.empty(fwd_stats.numel(), device=dy.device, dtype=torch.float32)
    a, (b, h, w, c1, c2) = _gn_args(x1, gamma, beta, eps, silu, add1, add1_scale, x2, add2, add2_scale, groups)
    a.stats_ws = _dp(ws)
    dx1 = torch.empty((b, h, w, c1), device=dy.device, dtype=torch.float16)
    dx2 = torch.empty((b, h, w, c2), device=dy.device, dtype=torch.float16) if (want_dx2 and c2) else None
    _count(2)
    if res is not None:
        assert res.dtype == torch.float16 and res.stride(-1) == 1 and res.shape[-1] == c1 + c2
    check(_lib.load().ctrlora_groupnorm_bwd_f16(C.addressof(a), _dp(dy), _dp(fwd_stats), _dp(dx1), c1, float(dx1_scale), _dp(dx2), c2,
                                                float(dx2_scale), _dp(res), res.stride(-2) if res is not None else 0,
                                                _dp(dgamma), _dp(dbeta), _sp()), "groupnorm_bwd")
    return (dx1, dx2) if want_dx2 else dx1


def layernorm_bwd(x, dy, gamma, eps=1e-5, dgamma=None, dbeta=None, res=None):
    _require_cuda(x, dy)
    cols = x.shape[-1]
    x2, d2 = x.reshape(-1, cols), dy.reshape(-1, cols)
    dx = torch.empty((x2.shape[0], cols), device=x.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_layernorm_bwd_f16(_dp(x2), x2.stride(0), _dp(d2), d2.stride(0), _dp(dx), cols, x2.shape[0],
                                                cols, _dp(gamma), float(eps), _dp(dgamma), _dp(dbeta), _dp(res),
                                                res.reshape(-1, cols).stride(0) if res is not None else 0, _sp()), "layernorm_bwd")
    return dx.view(x.shape)


def geglu_fwd(h):
    """h fp16 [M, 2N] = [value | gate] -> value * gelu(gate) [M, N]"""
    _require_cuda(h)
    m, n2 = h.shape
    out = torch.empty((m, n2 // 2), device=h.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_geglu_fwd_f16(_dp(h), _dp(out), m, n2 // 2, _sp()), "geglu_fwd")
    return out


def geglu_bwd(h, dout):
    _require_cuda(h, dout)
    m, n2 = h.shape
    dh = torch.empty_like(h)
    _count()
    check(_lib.load().ctrlora_geglu_bwd_f16(_dp(h), _dp(dout), _dp(dh), m, n2 // 2, _sp()), "geglu_bwd")
    return dh


def colsum(x, out, scale=1.0):
    """out[c] += scale * sum_rows x[row, c]; x fp16/fp32 [rows, cols] (row stride free), out fp32 [cols]"""
    _require_cuda(x, out)
    x2 = x.reshape(-1, x.shape[-1])
    _count()
    check(_lib.load().ctrlora_colsum(_dp(x2), int(x2.dtype == torch.float32), x2.stride(0), x2.shape[0], x2.shape[1],
                                     float(scale), _dp(out), _sp()), "colsum")
    return out


def image_colsum(x, images, out):
    """out[img, c] += sum over the image's rows of x (fp16 [images*rows, cols]); out fp32 [images, >=cols] (row stride free)"""
    _require_cuda(x, out)
    x2 = x.reshape(-1, x.shape[-1])
    _count()
    check(_lib.load().ctrlora_image_colsum_f16(_dp(x2), x2.stride(0), images, x2.shape[0] // images, x2.shape[1], _dp(out),
                                               out.stride(0), _sp()), "image_colsum")
    return out


def upsample2x_bwd(dout):
    _require_cuda(dout)
    b, h2, w2, c = dout.shape
    din = torch.empty((b, h2 // 2, w2 // 2, c), device=dout.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_upsample2x_bwd_f16(_dp(dout.contiguous()), _dp(din), b, h2 // 2, w2 // 2, c, _sp()), "upsample2x_bwd")
    return din


def im2col_s2_bwd(dcol, h, w):
    """dcol fp16 [B, h/2, w/2, 9*C] -> dx [B, h, w, C]"""
    _require_cuda(dcol)
    b = dcol.shape[0]
    c = dcol.shape[-1] // 9
    dx = torch.empty((b, h, w, c), device=dcol.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_im2col_s2_bwd_f16(_dp(dcol.contiguous()), _dp(dx), b, h, w, c, _sp()), "im2col_s2_bwd")
    return dx


def mse_loss_grad(eps, noise, c_pad=8, grad_scale=1.0):
    """eps, noise fp32 [B,C,H,W] -> (loss fp32 [1], grad fp16 pixel-major [B,H,W,c_pad])"""
    _require_cuda(eps, noise)
    b, c, h, w = eps.shape
    loss = torch.empty(1, device=eps.device, dtype=torch.float32)
    grad = torch.empty((b, h, w, c_pad), device=eps.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_mse_loss_grad(_dp(eps.contiguous()), _dp(noise.contiguous()), _dp(loss), _dp(grad), b, c, h * w,
                                            c_pad, float(grad_scale), _sp()), "mse_loss_grad")
    return loss, grad


def adamw_step(params, grads, exp_avg, exp_avg_sq, step, lr=1e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01,
               grad_scale=1.0, skip_flag=None, bc_dev=None):
    """In-place AdamW over flat fp32 buffers (torch.optim.AdamW semantics).  skip_flag: device int32 [1]; non-zero =
    the step is skipped (non-finite gradients under loss scaling).  bc_dev: device fp32 [2] bias corrections from
    adamw_begin (then `step` is ignored)."""
    _require_cuda(params, grads)
    _count()
    check(_lib.load().ctrlora_adamw_f32(_dp(params), _dp(grads), _dp(exp_avg), _dp(exp_avg_sq), params.numel(), float(lr),
                                        float(betas[0]), float(betas[1]), float(eps), float(weight_decay), int(step),
                                        float(grad_scale), _dp(skip_flag), _dp(bc_dev), _sp()), "adamw")


def adamw_begin(step_counter, skip_flag, betas, bc, skipped=None):
    """device-side step bookkeeping in front of adamw_step (see ctrlora_adamw_begin)"""
    _require_cuda(step_counter, bc)
    _count()
    check(_lib.load().ctrlora_adamw_begin(_dp(step_counter), _dp(skip_flag), float(betas[0]), float(betas[1]), _dp(bc),
                                          _dp(skipped), _sp()), "adamw_begin")


def nonfinite_flag(x, flag):
    """flag (int32 [1], device) |= any(!isfinite(x)); x fp32 flat."""
    _require_cuda(x, flag)
    assert x.dtype == torch.float32 and x.is_contiguous() and flag.dtype == torch.int32
    _count()
    check(_lib.load().ctrlora_nonfinite_flag_f32(_dp(x), x.numel(), _dp(flag), _sp()), "nonfinite_flag")
    return flag


def weighted_sum(tensors, weights, out=None):
    """sum_i weights[i] * tensors[i] over up to 8 same-shape, same-stride dense fp16 tensors (fp32 accumulate)."""
    _require_cuda(*tensors)
    t0 = tensors[0]
    n = len(tensors)
    assert 1 <= n <= 8 and len(weights) == n
    for t in tensors:
        assert t.dtype == torch.float16 and t.shape == t0.shape and t.stride() == t0.stride()
    dense = t0.is_contiguous() or t0.is_contiguous(memory_format=torch.channels_last)
    assert dense and t0.numel() % 8 == 0, "weighted_sum needs dense tensors with numel % 8 == 0"
    if out is None:
        out = torch.empty_like(t0)  # preserves the (dense) strides
    assert out.stride() == t0.stride()
    srcs = (C.c_void_p * n)(*[t.data_ptr() for t in tensors])
    ws = (C.c_float * n)(*[float(w) for w in weights])
    _count()
    check(_lib.load().ctrlora_weighted_sum_f16(srcs, ws, n, _dp(out), t0.numel(), _sp()), "weighted_sum")
    return out


def attention_bwd(q, k, v, o, dout, lse, batch, heads, nq, nk, head_dim, dq=None, dk=None, dv=None):
    """Backward of ops.attention.  q/o/dout [batch*nq, H*d], k/v natural [batch*nk, H*d] (fp16, row strides free),
    lse fp32 [batch, H, nq] from the forward.  Returns (dq, dk, dv) fp16."""
    _require_cuda(q, k, v, o, dout, lse)
    c = heads * head_dim
    dq = torch.empty((batch * nq, c), device=q.device, dtype=torch.float16) if dq is None else dq
    dk = torch.empty((batch * nk, c), device=q.device, dtype=torch.float16) if dk is None else dk
    dv = torch.empty((batch * nk, c), device=q.device, dtype=torch.float16) if dv is None else dv
    delta = torch.empty(batch * heads * nq, device=q.device, dtype=torch.float32)
    _count(3)
    check(_lib.load().ctrlora_attention_bwd_f16(_dp(q), q.stride(0), _dp(k), k.stride(0), _dp(v), v.stride(0), _dp(o), o.stride(0),
                                                _dp(dout), dout.stride(0), _dp(lse), _dp(delta), _dp(dq), dq.stride(0), _dp(dk),
                                                dk.stride(0), _dp(dv), dv.stride(0), batch, heads, nq, nk, head_dim, _sp()),
          "ctrlora_attention_bwd_f16")
    return dq, dk, dv


def transpose_f16(src, batch, rows, cols):
    """fp16 [batch, rows, cols] -> fp16 [batch, cols, rows]"""
    _require_cuda(src)
    assert src.dtype == torch.float16 and src.is_contiguous() and src.numel() == batch * rows * cols
    out = torch.empty((batch, cols, rows), device=src.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_transpose_f16(_dp(src), _dp(out), batch, rows, cols, _sp()), "transpose_f16")
    return out


def conv_dgrad_weight(w16):
    """fp16 conv kernel weight [Cout, taps, Cin] -> data-gradient weight [Cin, taps reversed, Cout]"""
    _require_cuda(w16)
    co, taps, ci = w16.shape
    out = torch.empty((ci, taps, co), device=w16.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_conv_dgrad_weight_f16(_dp(w16), _dp(out), co, taps, ci, _sp()), "conv_dgrad_weight")
    return out


# ------------------------------------------------------------------------------------------------ CLIP text encoder
def causal_attention(q, k, vt, batch, heads, n, out=None):
    """Causal self-attention, d_head 64, n <= 128: q, k [batch*n, heads*64] (row strides free), vt [batch, heads, 64,
    nk_pad] (fp16) -> [batch*n, heads*64]."""
    _require_cuda(q, k, vt)
    if out is None:
        out = torch.empty((batch * n, heads * 64), device=q.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_causal_attention_f16(_dp(q), q.stride(0), _dp(k), k.stride(0), _dp(vt), vt.shape[-1], _dp(out),
                                                   out.stride(0), batch, heads, n, 64, _sp()), "ctrlora_causal_attention_f16")
    return out


def clip_embed(ids, token_embedding, position_embedding, out_f32=True, out=None):
    """ids int64 [B, n] (device) -> token_embedding[ids] + position_embedding[:n], [B*n, C] fp32 (or fp16)"""
    _require_cuda(ids, token_embedding, position_embedding)
    assert ids.dtype == torch.int64 and ids.is_contiguous() and ids.dim() == 2
    assert token_embedding.dtype == position_embedding.dtype == torch.float32
    assert token_embedding.is_contiguous() and position_embedding.is_contiguous()
    b, n = ids.shape
    vocab, cols = token_embedding.shape
    assert position_embedding.shape[0] >= n and position_embedding.shape[1] == cols
    if out is None:
        out = torch.empty((b * n, cols), device=ids.device, dtype=torch.float32 if out_f32 else torch.float16)
    _count()
    check(_lib.load().ctrlora_clip_embed(_dp(ids), _dp(token_embedding), _dp(position_embedding), _dp(out),
                                         int(out.dtype == torch.float32), b, n, cols, vocab, _sp()), "clip_embed")
    return out


def quick_gelu_(x):
    """x * sigmoid(1.702 x) in place on a contiguous fp16 tensor"""
    _require_cuda(x)
    assert x.dtype == torch.float16 and x.is_contiguous()
    _count()
    check(_lib.load().ctrlora_quick_gelu_f16(_dp(x), x.numel(), _sp()), "quick_gelu")
    return x


def layernorm_rows(x, gamma, beta, eps=1e-5, out_f32=False, out=None):
    """LayerNorm over the last dim of x fp32 or fp16 [rows, C] (row stride free) -> fp32 or fp16 [rows, C]"""
    _require_cuda(x)
    assert x.dim() == 2 and x.stride(1) == 1 and x.dtype in (torch.float32, torch.float16)
    rows, cols = x.shape
    if out is None:
        out = torch.empty((rows, cols), device=x.device, dtype=torch.float32 if out_f32 else torch.float16)
    _count()
    check(_lib.load().ctrlora_layernorm_rows(_dp(x), int(x.dtype == torch.float32), x.stride(0), _dp(out),
                                             int(out.dtype == torch.float32), out.stride(0), rows, cols, _dp(gamma), _dp(beta),
                                             float(eps), _sp()), "layernorm_rows")
    return out


# ------------------------------------------------------------------------------------------------ CLIP image encoder
def clip_patch_gather(pixels, patch, k_pad, out=None):
    """pixels fp32 or fp16 [B, C, S, S] (contiguous) -> fp16 patch rows [B * (S/patch)^2, k_pad] in the Conv2d weight's
    (c, kh, kw) column order, zero beyond C * patch^2"""
    _require_cuda(pixels)
    assert pixels.dim() == 4 and pixels.is_contiguous() and pixels.dtype in (torch.float32, torch.float16)
    b, c, s, s2 = pixels.shape
    assert s == s2 and s % patch == 0
    rows = b * (s // patch) ** 2
    if out is None:
        out = torch.empty((rows, k_pad), device=pixels.device, dtype=torch.float16)
    assert out.shape == (rows, k_pad) and out.is_contiguous() and out.dtype == torch.float16
    _count()
    check(_lib.load().ctrlora_clip_patch_gather(_dp(pixels), int(pixels.dtype == torch.float32), _dp(out), b, c, s, patch,
                                                k_pad, _sp()), "clip_patch_gather")
    return out


def patch_gather_hw(pixels, patch, k_pad, out=None):
    """pixels fp32 or fp16 [B, C, H, W] (contiguous) -> fp16 patch rows [B * gh * gw, k_pad], gh = H // patch, gw =
    W // patch (rows and columns beyond the last whole patch are not read), in clip_patch_gather's column order"""
    _require_cuda(pixels)
    assert pixels.dim() == 4 and pixels.is_contiguous() and pixels.dtype in (torch.float32, torch.float16)
    b, c, h, w = pixels.shape
    rows = b * (h // patch) * (w // patch)
    if out is None:
        out = torch.empty((rows, k_pad), device=pixels.device, dtype=torch.float16)
    assert out.shape == (rows, k_pad) and out.is_contiguous() and out.dtype == torch.float16
    _count()
    check(_lib.load().ctrlora_patch_gather_hw(_dp(pixels), int(pixels.dtype == torch.float32), _dp(out), b, c, h, w, patch,
                                              k_pad, _sp()), "patch_gather_hw")
    return out


def clip_vision_embed(patch_out, class_embedding, position_embedding, batch, out=None):
    """patch_out fp32 [batch * P, C] (row stride free) -> fp32 [batch * (P + 1), C]: per image the class embedding, then
    its P patch rows, each plus its position embedding"""
    _require_cuda(patch_out, class_embedding, position_embedding)
    assert patch_out.dtype == class_embedding.dtype == position_embedding.dtype == torch.float32 and patch_out.stride(1) == 1
    assert class_embedding.is_contiguous() and position_embedding.is_contiguous()
    rows, cols = patch_out.shape
    patches = rows // batch
    assert rows == batch * patches and position_embedding.shape == (patches + 1, cols) and class_embedding.numel() == cols
    if out is None:
        out = torch.empty((batch * (patches + 1), cols), device=patch_out.device, dtype=torch.float32)
    assert out.shape == (batch * (patches + 1), cols) and out.is_contiguous() and out.dtype == torch.float32
    _count()
    check(_lib.load().ctrlora_clip_vision_embed(_dp(patch_out), patch_out.stride(0), _dp(class_embedding),
                                                _dp(position_embedding), _dp(out), batch, patches, cols, _sp()),
          "clip_vision_embed")
    return out


def gelu_(x):
    """exact GELU 0.5 x (1 + erf(x / sqrt 2)) in place on a contiguous fp16 tensor"""
    _require_cuda(x)
    assert x.dtype == torch.float16 and x.is_contiguous()
    _count()
    check(_lib.load().ctrlora_gelu_f16(_dp(x), x.numel(), _sp()), "gelu")
    return x


# ------------------------------------------------------------------------------------------------ line-art annotator
def _gather_source(x, taps, channels):
    """(batch, h, w, channels, ld, src_f32_nchw, host tap array) of a tap gather's source"""
    _require_cuda(x)
    if x.dtype == torch.float32:
        assert x.dim() == 4 and x.is_contiguous()
        b, c, h, w = x.shape
        ld, f32 = 0, 1
    else:
        assert x.dtype == torch.float16
        b, h, w, c, ld = _as_bhwc(x)
        c, f32 = channels or c, 0
    flat = (C.c_int * (2 * len(taps)))(*[int(v) for t in taps for v in t])
    return b, h, w, c, ld, f32, flat


def _gather_out(out, shape, device):
    if out is None:
        out = torch.empty(shape, device=device, dtype=torch.float16)
    assert out.shape == shape and out.is_contiguous() and out.dtype == torch.float16
    return out


def tap_gather(x, taps, *, reflect, k_pad, channels=None, out=None):
    """Gather the (dy, dx) taps of every pixel into GEMM rows: fp16 [B, H, W, k_pad], column t * C + c = x at (y + dy_t,
    x + dx_t), reflected at the border (nn.ReflectionPad2d) or zero outside, zero beyond len(taps) * C.
    x: fp16 pixel-major [B, H, W, ld] (channels <= ld, default ld) or fp32 NCHW [B, C, H, W] contiguous."""
    b, h, w, c, ld, f32, flat = _gather_source(x, taps, channels)
    out = _gather_out(out, (b, h, w, k_pad), x.device)
    _count()
    check(_lib.load().ctrlora_tap_gather_f16(_dp(x), f32, ld, _dp(out), b, h, w, c, C.cast(flat, C.c_void_p), len(taps),
                                             int(bool(reflect)), k_pad, _sp()), "tap_gather")
    return out


GATHER_ACTS = {None: 0, "relu": 1, "leaky": 2}  # ctrlora_tap_gather_act_f16's act codes; "leaky" is LeakyReLU(0.2)


def tap_gather_act(x, taps, *, reflect, k_pad, stride=1, act=None, channels=None, out=None):
    """tap_gather with an output stride and an activation on load: fp16 [B, H // stride, W // stride, k_pad], column
    t * C + c of output pixel (y, x) = act(x at (stride y + dy_t, stride x + dx_t)), reflected or zero outside.
    stride 1 or 2; act None, "relu" or "leaky" (LeakyReLU(0.2)), applied in fp32 before the fp16 rounding."""
    b, h, w, c, ld, f32, flat = _gather_source(x, taps, channels)
    out = _gather_out(out, (b, h // stride, w // stride, k_pad), x.device)
    _count()
    check(_lib.load().ctrlora_tap_gather_act_f16(_dp(x), f32, ld, _dp(out), b, h, w, c, C.cast(flat, C.c_void_p),
                                                 len(taps), int(bool(reflect)), k_pad, stride, GATHER_ACTS[act], _sp()),
          "tap_gather_act")
    return out


INSTANCE_NORM_MAX_CHUNKS = 1024  # per-image statistics chunks (annotator_sm90.cu kNormMaxChunks)


def instance_norm(x, *, relu, residual=None, phases=False, eps=1e-5, out=None):
    """InstanceNorm2d (affine=False) + optional ReLU + optional residual add, fp16 pixel-major.
    phases=False: x [B, H, W, C] -> [B, H, W, C].  phases=True: x [4, B, H, W, C], the four sub-pixel phase outputs
    (2 py + px) of a stride-2 transposed conv -> [B, 2H, 2W, C] interleaved.  residual: y's shape, added last."""
    _require_cuda(x, residual)
    assert x.dtype == torch.float16 and x.is_contiguous()
    if phases:
        assert x.dim() == 5 and x.shape[0] == 4
        _, b, h, w, c = x.shape
        shape = (b, 2 * h, 2 * w, c)
    else:
        b, h, w, c = x.shape
        shape = (b, h, w, c)
    if out is None:
        out = torch.empty(shape, device=x.device, dtype=torch.float16)
    assert out.shape == shape and out.is_contiguous() and out.dtype == torch.float16
    if residual is not None:
        assert residual.shape == shape and residual.is_contiguous() and residual.dtype == torch.float16
    ws_floats = 2 * b * c * (INSTANCE_NORM_MAX_CHUNKS + 1)
    ws = torch.empty(ws_floats, device=x.device, dtype=torch.float32)
    _count(3)
    check(_lib.load().ctrlora_instance_norm_f16(_dp(x), _dp(residual), _dp(out), _dp(ws), ws_floats, b, h, w, c,
                                                int(bool(phases)), int(bool(relu)), float(eps), _sp()), "instance_norm")
    return out


def lineart_out(x, weight, bias, want_u8=False):
    """ReflectionPad2d(3) + Conv2d(C -> 1, 7) + Sigmoid: x fp16 [B, H, W, C], weight fp32 [49, C] (tap-major), bias fp32
    [1] (device) -> fp32 [B, 1, H, W] (and with want_u8 the uint8 [B, H, W] map (uint8)clip(y * 255, 0, 255))."""
    _require_cuda(x, weight, bias)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4
    b, h, w, c = x.shape
    assert weight.dtype == torch.float32 and weight.is_contiguous() and weight.shape == (49, c)
    assert bias.dtype == torch.float32 and bias.numel() == 1
    out = torch.empty((b, 1, h, w), device=x.device, dtype=torch.float32)
    u8 = torch.empty((b, h, w), device=x.device, dtype=torch.uint8) if want_u8 else None
    _count()
    check(_lib.load().ctrlora_lineart_out_f16(_dp(x), _dp(weight), _dp(bias), _dp(out), _dp(u8), b, h, w, c, _sp()),
          "lineart_out")
    return (out, u8) if want_u8 else out


def lineart_anime_out(skip, up, weight, bias, scale=1.0, shift=0.0):
    """Anime2Sketch's outermost up path: tanh(bias + ConvTranspose2d(C -> 1, 4, stride 2, padding 1)(ReLU([skip | up]))
    ) * scale + shift.  skip, up: fp16 [B, h, w, C / 2] each; weight fp32 [C, 16] (the transposed kernel [C, 1, 4, 4]);
    bias fp32 [1] (device) -> fp32 [B, 1, 2h, 2w]"""
    _require_cuda(skip, up, weight, bias)
    assert skip.dtype == up.dtype == torch.float16 and skip.is_contiguous() and up.is_contiguous()
    assert skip.dim() == 4 and up.shape == skip.shape
    b, h, w, half = skip.shape
    assert weight.dtype == torch.float32 and weight.is_contiguous() and weight.shape == (2 * half, 16)
    assert bias.dtype == torch.float32 and bias.numel() == 1
    out = torch.empty((b, 1, 2 * h, 2 * w), device=skip.device, dtype=torch.float32)
    _count()
    check(_lib.load().ctrlora_lineart_anime_out_f16(_dp(skip), _dp(up), _dp(weight), _dp(bias), _dp(out), b, h, w,
                                                    2 * half, float(scale), float(shift), _sp()), "lineart_anime_out")
    return out


# ------------------------------------------------------------------------------------------------ HED annotator
def hed_side_pool(x, weight, bias, pool):
    """A HED block's 1x1 side projection (C -> 1) and, with pool, the 2x2 max-pool (floor) that feeds the next block, in
    one read of x fp16 [B, h, w, C].  weight fp32 [C], bias fp32 [1] (device).  Returns (fp32 [B, 1, h, w] side map,
    fp16 [B, h // 2, w // 2, C] pooled or None)."""
    _require_cuda(x, weight, bias)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4
    b, h, w, c = x.shape
    assert weight.dtype == torch.float32 and weight.is_contiguous() and weight.numel() == c
    assert bias.dtype == torch.float32 and bias.numel() == 1
    side = torch.empty((b, 1, h, w), device=x.device, dtype=torch.float32)
    pooled = torch.empty((b, h // 2, w // 2, c), device=x.device, dtype=torch.float16) if pool else None
    _count()
    check(_lib.load().ctrlora_hed_side_pool_f16(_dp(x), _dp(weight), _dp(bias), _dp(side), _dp(pooled), b, h, w, c, _sp()),
          "hed_side_pool")
    return side, pooled


def hed_fuse(sides, tables, safe):
    """HEDdetector's post-process on the device.  sides: the five fp32 [B, 1, h_l, w_l] side maps, the first at the
    output size H x W; tables: for levels 1..4, (int32 [H + W] source index, fp32 [H + W] fraction) device pairs (rows
    then columns, annotator.hed.resize_tables).  Returns (fp32 [B, H, W] mean map, uint8 [B, H, W] edge map)."""
    _require_cuda(*sides)
    assert len(sides) == 5 and len(tables) == 4
    b, _, h, w = sides[0].shape
    for s in sides:
        assert s.dtype == torch.float32 and s.is_contiguous() and s.shape[:2] == (b, 1)
    for idx, frac in tables:
        _require_cuda(idx, frac)
        assert idx.dtype == torch.int32 and frac.dtype == torch.float32 and idx.numel() == frac.numel() == h + w
    mean = torch.empty((b, h, w), device=sides[0].device, dtype=torch.float32)
    u8 = torch.empty((b, h, w), device=sides[0].device, dtype=torch.uint8)
    ptrs = (C.c_void_p * 5)(*[s.data_ptr() for s in sides])
    hw = (C.c_int * 10)(*[v for s in sides for v in s.shape[2:]])
    idx_p = (C.c_void_p * 5)(None, *[t[0].data_ptr() for t in tables])
    frac_p = (C.c_void_p * 5)(None, *[t[1].data_ptr() for t in tables])
    _count()
    check(_lib.load().ctrlora_hed_fuse(C.cast(ptrs, C.c_void_p), C.cast(hw, C.c_void_p), C.cast(idx_p, C.c_void_p),
                                       C.cast(frac_p, C.c_void_p), _dp(mean), _dp(u8), b, h, w, int(bool(safe)), _sp()),
          "hed_fuse")
    return mean, u8


def max_pool2x2(x):
    """nn.MaxPool2d(2, 2) (floor) on fp16 [B, h, w, C] (C in {64, 128, 256, 512}) -> fp16 [B, h // 2, w // 2, C]:
    ctrlora_hed_side_pool_f16 without its projection"""
    _require_cuda(x)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4
    b, h, w, c = x.shape
    pooled = torch.empty((b, h // 2, w // 2, c), device=x.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_hed_side_pool_f16(_dp(x), None, None, None, _dp(pooled), b, h, w, c, _sp()), "max_pool2x2")
    return pooled


# ------------------------------------------------------------------------------------------------ OpenPose annotator
def _openpose_tabs(tables):
    ys, yw, xs, xw = tables
    _require_cuda(ys, yw, xs, xw)
    assert ys.dtype == xs.dtype == torch.int32 and yw.dtype == xw.dtype == torch.float64
    assert yw.dim() == xw.dim() == 2 and yw.shape[0] == ys.numel() and xw.shape[0] == xs.numel()
    return [_dp(ys), _dp(yw), yw.shape[1], _dp(xs), _dp(xw), xw.shape[1]]


def _pixel_maps(maps):
    """fp32 pixel-major [h8, w8, ld] (one image) -> (h8, w8, ld)"""
    assert maps.dtype == torch.float32 and maps.dim() == 3 and maps.stride(2) == 1
    h8, w8, ld = maps.shape[0], maps.shape[1], maps.stride(1)
    assert maps.stride(0) == w8 * ld
    return h8, w8, ld


def openpose_resample(maps, tables, channels):
    """Channels 0 .. channels - 1 of one image's stride-8 maps (fp32 pixel-major [h8, w8, ld]) resampled to the image
    through `tables` = (int32 [H] row starts, float64 [H, ty] row weights, int32 [W], float64 [W, tx]) -> fp32
    [channels, H, W]"""
    _require_cuda(maps)
    h8, w8, ld = _pixel_maps(maps)
    tab = _openpose_tabs(tables)
    h, w = tables[0].numel(), tables[2].numel()
    out = torch.empty((channels, h, w), device=maps.device, dtype=torch.float32)
    _count()
    check(_lib.load().ctrlora_openpose_resample(_dp(maps), ld, h8, w8, channels, *tab, _dp(out), h, w, _sp()),
          "openpose_resample")
    return out


def openpose_smooth(heat, weights):
    """scipy.ndimage.gaussian_filter(mode='reflect') of each fp32 [H, W] map of heat [maps, H, W], in float64, with the
    symmetric kernel `weights` (host sequence, centre tap first) -> float64 [maps, H, W]"""
    _require_cuda(heat)
    assert heat.dtype == torch.float32 and heat.is_contiguous() and heat.dim() == 3
    tmp = torch.empty(heat.shape, device=heat.device, dtype=torch.float64)
    out = torch.empty(heat.shape, device=heat.device, dtype=torch.float64)
    wts = (C.c_double * len(weights))(*[float(v) for v in weights])
    _count(2)
    check(_lib.load().ctrlora_openpose_smooth(_dp(heat), _dp(tmp), _dp(out), heat.shape[0], heat.shape[1],
                                              heat.shape[2], C.cast(wts, C.c_void_p), len(weights) - 1, _sp()),
          "openpose_smooth")
    return out


OPENPOSE_PEAK_CHUNK = 2048  # map elements per block of the peak passes (openpose_sm90.cu kPeakChunk)


def openpose_peaks(smoothed, heat, thre, capacity=1024):
    """The peaks of smoothed float64 [maps, H, W] (>= the four neighbours, > thre) in (map, y, x) order -> device (int32
    x, int32 y, int32 part, fp32 score = heat at the peak), each [number of peaks].  Reads the count on the host."""
    _require_cuda(smoothed, heat)
    assert smoothed.dtype == torch.float64 and smoothed.is_contiguous() and smoothed.dim() == 3
    assert heat.dtype == torch.float32 and heat.is_contiguous() and heat.shape == smoothed.shape
    m, h, w = smoothed.shape
    blocks = (m * h * w + OPENPOSE_PEAK_CHUNK - 1) // OPENPOSE_PEAK_CHUNK
    ws = torch.empty(blocks + 1, device=smoothed.device, dtype=torch.int32)
    while True:
        pk = torch.empty((3, capacity), device=smoothed.device, dtype=torch.int32)
        score = torch.empty(capacity, device=smoothed.device, dtype=torch.float32)
        _count(3)
        check(_lib.load().ctrlora_openpose_peaks(_dp(smoothed), _dp(heat), m, h, w, float(thre), _dp(ws), ws.numel(),
                                                 _dp(pk[0]), _dp(pk[1]), _dp(pk[2]), _dp(score), capacity, _sp()),
              "openpose_peaks")
        n = int(ws[blocks].item())
        if n <= capacity:
            return pk[0, :n], pk[1, :n], pk[2, :n], score[:n]
        capacity = n


def openpose_limbs(paf, tables, px, py, limbs, img_h, thre):
    """Score every candidate pair of every limb.  paf: fp32 pixel-major [h8, w8, ld] stride-8 PAF maps; tables: as for
    openpose_resample; px, py: int32 peak coordinates (device); limbs: host rows (first pair, first A peak, nA, first B
    peak, nB, x channel, y channel).  Returns device (float64 score, uint8 ok) per pair."""
    _require_cuda(paf, px, py)
    h8, w8, ld = _pixel_maps(paf)
    tab = _openpose_tabs(tables)
    pairs = sum(r[2] * r[4] for r in limbs)
    score = torch.empty(pairs, device=paf.device, dtype=torch.float64)
    ok = torch.empty(pairs, device=paf.device, dtype=torch.uint8)
    if pairs == 0:
        return score, ok
    assert px.dtype == py.dtype == torch.int32
    flat = (C.c_int * (7 * len(limbs)))(*[int(v) for r in limbs for v in r])
    _count()
    check(_lib.load().ctrlora_openpose_limbs(_dp(paf), ld, h8, w8, *tab, _dp(px), _dp(py), C.cast(flat, C.c_void_p),
                                             len(limbs), pairs, int(img_h), float(thre), _dp(score), _dp(ok), _sp()),
          "openpose_limbs")
    return score, ok


# ------------------------------------------------------------------------------------------------ MiDaS annotator
def depth_to_space_bias(src, bias, s):
    """src fp32 [B, h, w, s * s * C] (a kernel = stride ConvTranspose2d as one GEMM, column (ky * s + kx) * C + c), bias
    fp32 [C] -> fp16 [B, h * s, w * s, C], the bias added before the one rounding"""
    _require_cuda(src, bias)
    assert src.dtype == torch.float32 and src.is_contiguous() and src.dim() == 4
    assert bias.dtype == torch.float32 and bias.is_contiguous()
    b, h, w, n = src.shape
    c = n // (s * s)
    assert c * s * s == n and bias.numel() == c
    out = torch.empty((b, h * s, w * s, c), device=src.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_depth_to_space_bias(_dp(src), _dp(bias), _dp(out), b, h, w, c, s, _sp()),
          "depth_to_space_bias")
    return out


def add_relu(a, b=None):
    """fp16 tensors of one shape (contiguous) -> (s, relu(s)) with s = a + b rounded to fp16 once; b None: relu(a) only"""
    _require_cuda(a, b)
    assert a.dtype == torch.float16 and a.is_contiguous()
    if b is not None:
        assert b.dtype == torch.float16 and b.is_contiguous() and b.shape == a.shape
    s = torch.empty_like(a) if b is not None else None
    r = torch.empty_like(a)
    _count()
    check(_lib.load().ctrlora_add_relu_f16(_dp(a), _dp(b), _dp(s), _dp(r), a.numel(), _sp()), "add_relu")
    return r if b is None else (s, r)


def upsample_bilinear2x(x):
    """F.interpolate(scale_factor=2, mode="bilinear", align_corners=True) on fp16 [B, h, w, C] -> [B, 2h, 2w, C]"""
    _require_cuda(x)
    assert x.is_contiguous() and x.dtype == torch.float16 and x.dim() == 4
    b, h, w, c = x.shape
    y = torch.empty((b, 2 * h, 2 * w, c), device=x.device, dtype=torch.float16)
    _count()
    check(_lib.load().ctrlora_upsample_bilinear2x_f16(_dp(x), _dp(y), b, h, w, c, _sp()), "upsample_bilinear2x")
    return y


def upsample_bilinear2x_into(x, out):
    """upsample_bilinear2x from fp16 [B, h, w, C] into `out`, an fp16 [B, 2h, 2w, C] view; either may be a channel slice
    of a wider pixel-major buffer"""
    _require_cuda(x, out)
    assert x.dtype == torch.float16 and out.dtype == torch.float16
    b, h, w, c, ld = _as_bhwc(x)
    bo, ho, wo, co, ldo = _as_bhwc(out)
    assert (bo, ho, wo, co) == (b, 2 * h, 2 * w, c), (tuple(x.shape), tuple(out.shape))
    _count()
    check(_lib.load().ctrlora_upsample_bilinear2x_ld_f16(_dp(x), ld, _dp(out), ldo, b, h, w, c, _sp()),
          "upsample_bilinear2x_into")
    return out


def midas_head_out(x, weight, bias):
    """the DPT head's Conv2d(C -> 1, 1) + ReLU: x fp16 [B, H, W, C], weight fp32 [C], bias fp32 [1] -> fp32 [B, H, W]"""
    _require_cuda(x, weight, bias)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4
    b, h, w, c = x.shape
    assert weight.dtype == torch.float32 and weight.is_contiguous() and weight.numel() == c
    assert bias.dtype == torch.float32 and bias.numel() == 1
    out = torch.empty((b, h, w), device=x.device, dtype=torch.float32)
    _count()
    check(_lib.load().ctrlora_midas_head_out_f16(_dp(x), _dp(weight), _dp(bias), _dp(out), b * h * w, c, _sp()),
          "midas_head_out")
    return out


def midas_maps(depth, a, bg_th):
    """MidasDetector's post-process: depth fp32 [B, H, W] -> (uint8 [B, H, W] depth map, uint8 [B, H, W, 3] normal map)"""
    _require_cuda(depth)
    assert depth.dtype == torch.float32 and depth.is_contiguous() and depth.dim() == 3
    b, h, w = depth.shape
    minmax = torch.empty((b, 2), device=depth.device, dtype=torch.float32)
    d8 = torch.empty((b, h, w), device=depth.device, dtype=torch.uint8)
    n8 = torch.empty((b, h, w, 3), device=depth.device, dtype=torch.uint8)
    _count(2)
    check(_lib.load().ctrlora_midas_maps(_dp(depth), _dp(minmax), _dp(d8), _dp(n8), b, h, w, float(a), float(bg_th), _sp()),
          "midas_maps")
    return d8, n8


# ------------------------------------------------------------------------------------------------ UniFormer annotator
def dwconv(x, weight, bias, k, residual=None):
    """depthwise Conv2d(C, C, k, padding k // 2, groups=C) (k = 3 or 5) on fp16 [B, H, W, C] (contiguous), weight fp32
    [k * k, C] tap-major, bias fp32 [C] -> fp16 [B, H, W, C] = (residual +) bias + conv, rounded once"""
    _require_cuda(x, weight, bias, residual)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4
    b, h, w, c = x.shape
    assert weight.dtype == torch.float32 and weight.is_contiguous() and weight.shape == (k * k, c)
    assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == c
    if residual is not None:
        assert residual.dtype == torch.float16 and residual.is_contiguous() and residual.shape == x.shape
    out = torch.empty_like(x)
    _count()
    check(_lib.load().ctrlora_dwconv_f16(_dp(x), _dp(weight), _dp(bias), _dp(residual), _dp(out), b, h, w, c, k, _sp()),
          "dwconv")
    return out


DWCONV_ACTS = {None: 0, "relu": 1, "relu6": 2}  # ctrlora_dwconv_act_f16's act codes


def dwconv_act(x, weight, bias, k, *, stride=1, act=None, residual=None):
    """dwconv with a stride and an activation: stride 1 pads k // 2 -> fp16 [B, H, W, C]; stride 2 uses the TFLite
    padding (output pixel (y, x) reads rows 2y .. 2y + k - 1 and the same columns, zero outside) -> fp16 [B, H // 2,
    W // 2, C].  act None, "relu" or "relu6", applied after bias and residual (shaped like the output).  Stride 2 and
    an activation take k = 3 only."""
    _require_cuda(x, weight, bias, residual)
    assert x.dtype == torch.float16 and x.is_contiguous() and x.dim() == 4
    b, h, w, c = x.shape
    assert weight.dtype == torch.float32 and weight.is_contiguous() and weight.shape == (k * k, c)
    assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == c
    out = torch.empty((b, h // stride, w // stride, c), device=x.device, dtype=torch.float16)
    if residual is not None:
        assert residual.dtype == torch.float16 and residual.is_contiguous() and residual.shape == out.shape
    _count()
    check(_lib.load().ctrlora_dwconv_act_f16(_dp(x), _dp(weight), _dp(bias), _dp(residual), _dp(out), b, h, w, c, k,
                                             stride, DWCONV_ACTS[act], _sp()), "dwconv_act")
    return out


def resize_bilinear(x, size=None, out=None, accumulate=False):
    """F.interpolate(x, size, mode="bilinear", align_corners=False) on fp16 [B, h, w, C] (channels may be a slice of a
    wider buffer) -> fp16 [B, H, W, C]: into `out` (an fp16 [B, H, W, C] view, channel slices allowed) when given,
    adding to its contents when accumulate; otherwise a new tensor of `size`"""
    _require_cuda(x, out)
    assert x.dtype == torch.float16 and (out is None or out.dtype == torch.float16)
    b, hi, wi, c, ld = _as_bhwc(x)
    if out is None:
        assert not accumulate
        out = torch.empty((b, size[0], size[1], c), device=x.device, dtype=torch.float16)
    bo, ho, wo, co, ldo = _as_bhwc(out)
    assert (bo, co) == (b, c) and (size is None or tuple(size) == (ho, wo))
    _count()
    check(_lib.load().ctrlora_resize_bilinear_f16(_dp(x), ld, _dp(out), ldo, b, hi, wi, ho, wo, c, int(bool(accumulate)),
                                                  _sp()), "resize_bilinear")
    return out


def adaptive_avg_pool(x, sizes):
    """AdaptiveAvgPool2d(s) for every s in sizes (<= 4) in one launch on fp16 [B, H, W, C] (channels may be a slice of a
    wider buffer) -> [fp16 [B * s * s, C] rows (b, i, j) per size], views of one buffer"""
    _require_cuda(x)
    assert x.dtype == torch.float16
    b, h, w, c, ld = _as_bhwc(x)
    rows = [b * s * s for s in sizes]
    out = torch.empty((sum(rows), c), device=x.device, dtype=torch.float16)
    arr = (C.c_int * len(sizes))(*[int(s) for s in sizes])
    _count()
    check(_lib.load().ctrlora_adaptive_avg_pool_f16(_dp(x), ld, _dp(out), b, h, w, c, C.cast(arr, C.c_void_p), len(sizes),
                                                    _sp()), "adaptive_avg_pool")
    return list(torch.split(out, rows))


def seg_output(logits, classes, net_size, out_size, palette, want_labels=False):
    """logits fp32 [B, h4, w4, ld] (ld % 4 == 0) -> uint8 [B, H, W, 3] = palette[argmax over the first `classes`
    channels of the logits resized to net_size and then to out_size = (H, W)] (and the int32 labels [B, H, W])"""
    _require_cuda(logits, palette)
    assert logits.dtype == torch.float32 and logits.is_contiguous() and logits.dim() == 4
    assert palette.dtype == torch.uint8 and palette.is_contiguous() and palette.shape == (classes, 3)
    b, h4, w4, ld = logits.shape
    ho, wo = out_size
    rgb = torch.empty((b, ho, wo, 3), device=logits.device, dtype=torch.uint8)
    labels = torch.empty((b, ho, wo), device=logits.device, dtype=torch.int32) if want_labels else None
    _count()
    check(_lib.load().ctrlora_seg_output(_dp(logits), ld, classes, b, h4, w4, net_size[0], net_size[1], ho, wo,
                                         _dp(palette), _dp(rgb), _dp(labels), _sp()), "seg_output")
    return (rgb, labels) if want_labels else rgb


# ------------------------------------------------------------------------------------------------ M-LSD annotator
MLSD_TOPK = 200  # CTRLORA_MLSD_TOPK


def mlsd_decode(tp, c_center, c_disp):
    """M-LSD's line decode on the head's fp32 map [B, h, w, ld] (contiguous): per image the MLSD_TOPK largest of
    sigmoid(centre) * (3 x 3 peak mask), descending, ties by the lower flat index -> (int32 [B, TOPK] flat indices
    y * w + x, fp32 [B, TOPK, 6] (score, segment length, the four displacements)).  h * w >= MLSD_TOPK."""
    _require_cuda(tp)
    assert tp.dtype == torch.float32 and tp.is_contiguous() and tp.dim() == 4
    b, h, w, ld = tp.shape
    ws = torch.empty((b, h, w), device=tp.device, dtype=torch.float32)
    idx = torch.empty((b, MLSD_TOPK), device=tp.device, dtype=torch.int32)
    val = torch.empty((b, MLSD_TOPK, 6), device=tp.device, dtype=torch.float32)
    _count(2)
    check(_lib.load().ctrlora_mlsd_decode(_dp(tp), ld, c_center, c_disp, b, h, w, _dp(ws), _dp(idx), _dp(val), _sp()),
          "mlsd_decode")
    return idx, val


# ------------------------------------------------------------------------------------------------ Canny annotator
CANNY_MAX_MAG = 2040  # the largest L1 Sobel magnitude of uint8 input: 4 * 255 + 4 * 255


def canny_classify(x, lo, hi):
    """cv2.Canny's gradient, non-maximum suppression and thresholds on uint8 [B, H, W, 3] (rows may be strided, pixels
    and channels packed) with integer thresholds lo <= hi -> uint8 [B, H, W] classes: 0 none, 1 candidate (kept by the
    suppression and m > lo), 2 strong (also m > hi).  Thresholds beyond the magnitudes' range [0, 2040] act as -1 or
    2040, so they are clamped there before they cross the int32 ABI."""
    _require_cuda(x)
    assert x.dtype == torch.uint8 and x.dim() == 4 and x.shape[3] == 3
    assert x.stride(3) == 1 and x.stride(2) == 3 and x.stride(0) == x.shape[1] * x.stride(1), "packed pixels required"
    lo, hi = int(lo), int(hi)
    assert lo <= hi, (lo, hi)
    b, h, w, _ = x.shape
    cls = torch.empty((b, h, w), device=x.device, dtype=torch.uint8)
    clamp = lambda t: max(-1, min(t, CANNY_MAX_MAG))  # noqa: E731
    _count()
    check(_lib.load().ctrlora_canny_classify(_dp(x), x.stride(1), b, h, w, clamp(lo), clamp(hi), _dp(cls), _sp()),
          "canny_classify")
    return cls


def canny_hysteresis(cls):
    """cv2.Canny's hysteresis on the classes of canny_classify (uint8 [B, H, W], contiguous) -> uint8 [B, H, W]: 255 at
    every candidate 8-connected through candidates to a strong pixel, else 0.  Four launches whatever the content."""
    _require_cuda(cls)
    assert cls.dtype == torch.uint8 and cls.is_contiguous() and cls.dim() == 3
    b, h, w = cls.shape
    ws = torch.empty((b, h, w), device=cls.device, dtype=torch.int32)
    out = torch.empty_like(cls)
    _count(4)
    check(_lib.load().ctrlora_canny_hysteresis(_dp(cls), b, h, w, _dp(ws), _dp(out), _sp()), "canny_hysteresis")
    return out


def set_sm_limit(limit):
    """persistent GEMM grids use at most `limit` SMs (0 = all); baked into CUDA graphs at capture"""
    check(_lib.load().ctrlora_set_sm_limit(int(limit)), "set_sm_limit")
