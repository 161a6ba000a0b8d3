"""The conditioning-side kernels called directly, each against a plain torch reference of the same operation:

* the K | V^T projection of a cross-attention context (`ctrlora_gemm_f16` with seg_outs [k, V^T], transposed (0, 1, 0))
  at 77 tokens padded to 80 and at the IP-Adapter's 4 (and 1) tokens padded to 8, and q | k | V^T with tok_pad >
  rows_per_img (the text encoder's 77 -> 80, the vision tower's 257 -> 264): 128-row tiles that hold the end of one
  image and the start of the next, partial last tiles, every tile width that divides the segment, explicit and
  automatic split-K, the trainer's row-major V copy (dup_out), and the SIMT twin.  Guard values around every output
  show that nothing is written into V^T's key padding or past any buffer;
* the DPM-Solver++ multistep update, bit for bit against the torch fp32 expression of the reference's formula;
* the CLIP token + position embedding, quick-GELU over every finite fp16 value, the fp32 / fp16 row LayerNorm at
  both sides of each of its register-tile limits, and the two casts / gathers no other test calls.

References are torch on the same fp16-rounded operands (fp32, or fp64 where it is cheap).  Bounds are about 20 %
above what an NVIDIA H100 80GB HBM3 measured (rounding error, independent of clocks), written beside them; the errors
are printed under `pytest -s`.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tolerances import close

pytestmark = pytest.mark.gpu

GUARD = -1234.0     # finite fp16 sentinel in every location a launch must not write
GUARD_ROWS = 3      # rows of GUARD after each row-major output
GUARD_TAIL = 4096   # elements of GUARD after V^T
# norm-relative error of every projection output against fp32 torch on the same fp16 operands: one fp16 rounding of
# an fp32 sum; worst measured 2.27e-4 (k | V^T at one token per image, inner 320 and 64)
PROJ_NREL = 2.8e-4


def _rand(*shape, s=1.0, gen=None):
    return (torch.randn(*shape, device="cuda", generator=gen) * s).half()


def _sp():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ K | V^T projections
class _Proj:
    """One projection launch into GUARD-filled buffers: `segs` row-major segments (k, or q and k) then V^T
    [images, heads, d, tok_pad], plus an optional row-major copy of V (dup_out)."""

    def __init__(self, a, w, segs, heads, rows, tok_pad, bias=None, block_n=0, split_k=0, dup=True, simt=False):
        from ctrlora_b200 import ops
        dev = a.device
        self.M, self.inner = a.shape[0], w.shape[0] // (segs + 1)
        self.segs, self.heads, self.rows, self.tok_pad = segs, heads, rows, tok_pad
        self.imgs, self.d = self.M // rows, self.inner // heads
        assert self.imgs * rows == self.M and self.d * heads == self.inner
        self.bufs = [torch.full((self.M + GUARD_ROWS, self.inner), GUARD, device=dev, dtype=torch.float16)
                     for _ in range(segs)]
        self.vt_n = self.imgs * heads * self.d * tok_pad
        self.vt_buf = torch.full((self.vt_n + GUARD_TAIL,), GUARD, device=dev, dtype=torch.float16)
        self.vt = self.vt_buf[:self.vt_n].view(self.imgs, heads, self.d, tok_pad)
        self.dup_buf = torch.full((self.M + GUARD_ROWS, self.inner), GUARD, device=dev, dtype=torch.float16) if dup else None
        transposed = (0, 1, 0) if segs == 1 else (0, 0, 1)
        ops.gemm(a, w, bias=bias, seg_outs=[b[:self.M] for b in self.bufs] + [self.vt], seg_width=self.inner,
                 transposed=transposed, rows_per_img=rows, head_dim=self.d, tok_pad=tok_pad,
                 dup_out=self.dup_buf[:self.M] if dup else None, block_n=block_n, split_k=split_k, simt=simt)

    def seg(self, i):
        return self.bufs[i][:self.M]

    def vt_tokens(self):
        return self.vt[..., :self.rows]

    def permute_rows(self, v):
        """row-major [M, inner] -> [images, heads, d, rows]"""
        return v.reshape(self.imgs, self.rows, self.heads, self.d).permute(0, 2, 3, 1)

    def check(self, ref, what):
        """every output against the fp32 reference [M, (segs + 1) * inner]; the guards intact; returns the worst
        norm-relative error"""
        inner, M = self.inner, self.M
        errs = []
        for i in range(self.segs):
            errs.append(close(self.seg(i), ref[:, i * inner:(i + 1) * inner], nrel=PROJ_NREL, what=f"{what} seg {i}"))
            assert (self.bufs[i][M:] == GUARD).all(), f"{what}: rows after segment {i} written"
        errs.append(close(self.vt_tokens(), self.permute_rows(ref[:, self.segs * inner:]), nrel=PROJ_NREL,
                          what=f"{what} V^T"))
        assert (self.vt[..., self.rows:] == GUARD).all(), f"{what}: V^T key padding written"
        assert (self.vt_buf[self.vt_n:] == GUARD).all(), f"{what}: written past V^T"
        if self.dup_buf is not None:
            assert torch.equal(self.vt_tokens(), self.permute_rows(self.dup_buf[:M])), f"{what}: dup_out != V^T"
            assert (self.dup_buf[M:] == GUARD).all(), f"{what}: rows after dup_out written"
        return max(errs)

    def outputs(self):
        return [self.seg(i) for i in range(self.segs)] + [self.vt_tokens()]


def _widths(seg_width):
    """the explicit tile widths that divide a segment"""
    return [bn for bn in (32, 64, 128, 160, 256, 320) if seg_width % bn == 0]


def _sweep(a, w, segs, heads, rows, tok_pad, bias, tag):
    """every (block_n, split_k) against the reference; unsplit launches bit-identical to each other; the SIMT twin;
    and with V's weights equal to k's, V^T equal to k bit for bit (same sums, the two epilogues round alike)"""
    M, K = a.shape
    n_out = w.shape[0]
    inner = n_out // (segs + 1)
    ref = a.float() @ w.float().view(n_out, K).t()
    if bias is not None:
        ref = ref + bias
    worst, unsplit = 0.0, []
    for bn in [0] + _widths(inner):
        for sk in (0, 1, 3):
            p = _Proj(a, w, segs, heads, rows, tok_pad, bias=bias, block_n=bn, split_k=sk)
            worst = max(worst, p.check(ref, f"{tag} block_n {bn} split_k {sk}"))
            if sk == 1:
                unsplit.append((bn, p.outputs()))
    bn0, base = unsplit[0]
    for bn, outs in unsplit[1:]:
        for x, y in zip(outs, base):
            assert torch.equal(x, y), f"{tag}: block_n {bn} differs from block_n {bn0} (both unsplit)"
    simt = _Proj(a, w, segs, heads, rows, tok_pad, bias=bias, simt=True)
    worst = max(worst, simt.check(ref, f"{tag} simt"))
    w_same = w.clone()
    w_same[segs * inner:] = w[(segs - 1) * inner:segs * inner]
    b_same = None
    if bias is not None:
        b_same = bias.clone()
        b_same[segs * inner:] = bias[(segs - 1) * inner:segs * inner]
    p = _Proj(a, w_same, segs, heads, rows, tok_pad, bias=b_same, split_k=1, dup=False)
    assert torch.equal(p.vt_tokens(), p.permute_rows(p.seg(segs - 1))), f"{tag}: V^T rounds unlike k"
    print(f"{tag}: worst norm-relative error {worst:.2e} over {len(unsplit) * 3 + 1} launches")
    return worst


# (inner, heads, context width): SD1.5's cross-attention at its three widths, and the tiny test model's
_KV_WIDTHS = [(320, 8, 768), (640, 8, 768), (1280, 8, 768), (32, 4, 64), (64, 4, 64), (128, 4, 64)]


@pytest.mark.parametrize("inner,heads,ctx", _KV_WIDTHS)
@pytest.mark.parametrize("batch", [1, 2, 8, 16])
@pytest.mark.parametrize("rows,tok_pad", [(77, 80), (4, 8), (1, 8)])
def test_k_vt_projection(rows, tok_pad, batch, inner, heads, ctx):
    """K | V^T of a context, as every cross-attention (77 text tokens) and the IP-Adapter branch (4 image tokens)
    project it: k by the TMA epilogue, V^T row per thread, in the same launch"""
    gen = torch.Generator(device="cuda").manual_seed(rows * 1000 + batch * 10 + inner)
    a = _rand(batch * rows, ctx, gen=gen)
    w = _rand(2 * inner, 1, ctx, s=ctx ** -0.5, gen=gen)
    _sweep(a, w, 1, heads, rows, tok_pad, None, f"k|V^T {rows}->{tok_pad} x{batch} inner {inner}")


# (tokens, tok_pad, width, heads, batches): the CLIP text encoder (SD1.5's ViT-L/14 and the tiny fixture's) and the
# IP-Adapter's vision tower (ViT-H/14 and the tiny one), with the layers' qkv bias
_QKV_SHAPES = [(77, 80, 768, 12, (1, 2, 8)), (77, 80, 64, 1, (1, 2, 8)), (257, 264, 1280, 16, (1, 3)),
               (257, 264, 160, 2, (1, 3))]


@pytest.mark.parametrize("rows,tok_pad,width,heads,batch",
                         [(r, t, c, h, b) for r, t, c, h, bs in _QKV_SHAPES for b in bs])
def test_qkv_projection_padded_tokens(rows, tok_pad, width, heads, batch):
    gen = torch.Generator(device="cuda").manual_seed(rows + batch * 7 + width)
    a = _rand(batch * rows, width, gen=gen)
    w = _rand(3 * width, 1, width, s=width ** -0.5, gen=gen)
    bias = 0.1 * torch.randn(3 * width, device="cuda", generator=gen)
    _sweep(a, w, 2, heads, rows, tok_pad, bias, f"q|k|V^T {rows}->{tok_pad} x{batch} C {width}")


# ------------------------------------------------------------------------------------------------ DPM-Solver++ update
DPM_F64_TOL = 1.5e-7   # fp32 kernel vs fp64 evaluation of the same formula, norm-relative: 1.21e-7 measured


def _sd15_alphas_cumprod():
    """make_beta_schedule('linear', 1000, 0.00085, 0.012) of the configs (ldm/modules/diffusionmodules/util.py)"""
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float64) ** 2
    return torch.cumprod(1.0 - betas, 0).float()


def _dpm_ref(x, c, u, m_prev, cfg, st, dtype):
    s = lambda v: torch.tensor([v], device="cuda", dtype=dtype)  # noqa: E731  (a device tensor: true division)
    x, c = x.to(dtype), c.to(dtype)
    e = c if u is None else u.to(dtype) + s(cfg) * (c - u.to(dtype))
    m = (x - s(st.sigma_s) * e) / s(st.alpha_s)
    xn = s(st.c_x) * x - s(st.c_m) * m
    if m_prev is not None:
        xn = xn - s(st.c_d) * (s(st.inv_r0) * (m - m_prev.to(dtype)))
    return xn, m


@pytest.mark.parametrize("shape", [(2, 4, 64, 64), (3, 4, 9, 7)])
@pytest.mark.parametrize("guided", [True, False])
def test_dpm_multistep_update_bit_exact(shape, guided):
    """Each step of a 20-step plan (order 1, then order 2) and of a 10-step one (whose last step falls back to order 1),
    chained as the sampler chains them: x_next and the data prediction equal the torch fp32 expression of
    dpm_solver.py:311-312, 359, 494-497, 751-758 bit for bit, and stay within DPM_F64_TOL of an fp64 evaluation"""
    from ctrlora_b200 import dpm_schedule, ops
    ac = _sd15_alphas_cumprod()
    gen = torch.Generator(device="cuda").manual_seed(11 + guided)
    cfg = 7.5 if guided else 1.0
    worst = 0.0
    for steps in (20, 10):
        plan = dpm_schedule.multistep_plan(ac, steps)
        assert plan[0].order == 1 and plan[1].order == 2 and plan[-1].order == (2 if steps >= 15 else 1)
        x = torch.randn(shape, device="cuda", generator=gen)
        hist = [torch.empty_like(x), torch.empty_like(x)]
        for i, st in enumerate(plan):
            c = torch.randn(shape, device="cuda", generator=gen)
            u = torch.randn(shape, device="cuda", generator=gen) if guided else None
            m_prev = hist[(i - 1) % 2] if st.order == 2 else None
            inputs = [t.clone() for t in (x, c, u, m_prev) if t is not None]
            xn = ops.dpm_multistep_update(x, c, u, m_prev, hist[i % 2], cfg, **st.kernel_args())
            for t, t0 in zip([t for t in (x, c, u, m_prev) if t is not None], inputs):
                assert torch.equal(t, t0), "an input of the update changed"
            rx, rm = _dpm_ref(x, c, u, m_prev, cfg, st, torch.float32)
            assert torch.equal(hist[i % 2], rm), f"{steps} steps, step {i}: data prediction"
            assert torch.equal(xn, rx), f"{steps} steps, step {i} (order {st.order}): x_next"
            dx, dm = _dpm_ref(x, c, u, m_prev, cfg, st, torch.float64)
            worst = max(worst, ((xn.double() - dx).norm() / dx.norm()).item(), ((rm.double() - dm).norm() / dm.norm()).item())
            x = xn
    print(f"dpm update {shape} guided={guided}: bit-exact to fp32 torch; vs fp64 worst norm-relative {worst:.2e}")
    assert worst < DPM_F64_TOL


# ------------------------------------------------------------------------------------------------ CLIP embedding
@pytest.mark.parametrize("cols,vocab", [(768, 49408), (64, 1000)])
@pytest.mark.parametrize("batch,n", [(3, 77), (2, 5)])
def test_clip_embed(cols, vocab, batch, n):
    """token_embedding[ids] + position_embedding[:n]: one fp32 add (bit-exact), or that sum rounded once to fp16; an
    id outside the vocabulary turns its own row into NaN and no other"""
    from ctrlora_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(cols + n)
    tok = torch.randn((vocab, cols), device="cuda", generator=gen)
    pos = torch.randn((77, cols), device="cuda", generator=gen)
    ids = torch.randint(0, vocab, (batch, n), device="cuda", generator=gen)
    ids[0, 0], ids[-1, -1], ids[0, n // 2] = 0, vocab - 1, vocab - 1
    ref = (tok[ids] + pos[:n]).reshape(batch * n, cols)
    got = ops.clip_embed(ids, tok, pos)
    assert got.dtype == torch.float32 and torch.equal(got, ref)
    got16 = ops.clip_embed(ids, tok, pos, out_f32=False)
    assert got16.dtype == torch.float16 and torch.equal(got16, ref.half())
    bad = ids.clone()
    mid = batch // 2
    bad[mid, n // 2] = -1
    bad[mid, n - 1] = vocab
    for f32 in (True, False):
        out = ops.clip_embed(bad, tok, pos, out_f32=f32).view(batch, n, cols)
        want = (ref if f32 else ref.half()).view(batch, n, cols)
        nan_rows = torch.zeros((batch, n), dtype=torch.bool, device="cuda")
        nan_rows[mid, n // 2] = nan_rows[mid, n - 1] = True
        assert torch.isnan(out[nan_rows]).all()
        assert torch.equal(out[~nan_rows], want[~nan_rows])


# ------------------------------------------------------------------------------------------------ quick-GELU
def _all_finite_f16():
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    x = bits[torch.isfinite(bits)]
    return x[: x.numel() // 8 * 8].cuda().contiguous()


def test_quick_gelu_every_fp16_value():
    """x * sigmoid(1.702 x) over every finite fp16 value against fp64.  The kernel evaluates x / (1 + __expf(-1.702 x))
    in fp32: __expf is within 2 + 1.173 |a| ulp of exp(a) (CUDA math API), the fp32 argument -1.702 x carries about
    |a| ulp more, and the add and the divide one half ulp each, so before its one fp16 rounding the result is within
    (5 + 4 |x|) * 2^-23 of the exact value relatively; the rounding adds 2^-11 relatively (2^-25 absolutely for fp16
    subnormal results).  Large |x| gives exactly x (x > 0) or a zero of x's sign, never NaN."""
    from ctrlora_b200 import ops
    x = _all_finite_f16()
    got = ops.quick_gelu_(x.clone())
    assert torch.equal(got.view(torch.int16), ops.quick_gelu_(x.clone()).view(torch.int16))
    xd = x.double()
    ref = xd * torch.sigmoid(1.702 * xd)
    err = (got.double() - ref).abs()
    bound = ref.abs() * (2.0 ** -11 + (5 + 4 * xd.abs()) * 2.0 ** -23) + 2.0 ** -25
    ratio = (err / bound).max().item()
    print(f"quick-GELU over {x.numel()} fp16 values: max abs err {err.max():.2e}, worst err / bound {ratio:.6f}")
    assert (err <= bound).all(), x[err > bound][:8]
    sub = xd.abs() < 2.0 ** -14
    assert (err[sub] <= 2.0 ** -25).all()  # subnormal inputs: x / 2 to the nearest fp16
    big = xd.abs() >= 12
    want = torch.where(x > 0, x, torch.zeros_like(x).copysign(x))
    assert torch.equal(got[big].view(torch.int16), want[big].view(torch.int16))
    assert not torch.isnan(got).any()


def test_quick_gelu_grid_stride_second_lap():
    """more vectors than one grid of 4096 x 256 threads covers: the elements of the second lap get the same values"""
    from ctrlora_b200 import ops
    x = _all_finite_f16()
    table = torch.empty(65536, device="cuda", dtype=torch.float16)
    table[x.view(torch.int16).long() & 0xFFFF] = ops.quick_gelu_(x.clone())
    gen = torch.Generator(device="cuda").manual_seed(5)
    n = 4096 * 256 * 8 + 8 * 1237
    big = x[torch.randint(0, x.numel(), (n,), device="cuda", generator=gen)]
    got = ops.quick_gelu_(big.clone())
    assert torch.equal(got.view(torch.int16), table[big.view(torch.int16).long() & 0xFFFF].view(torch.int16))


# ------------------------------------------------------------------------------------------------ row LayerNorm
# norm-relative error against F.layer_norm in fp64, by output type and whether the rows sit on a large common offset;
# measured (worst over the columns and input types below) in the comments.  At mean ~1e3 the fp32 mean itself is
# rounded to 6e-5 (one ulp of 1e3) against a std of 1, hence the offset rows' 5e-5 with fp32 output.
LN_TOL = {
    (torch.float32, False): 9.7e-8,   # 8.06e-8
    (torch.float32, True): 5.8e-5,    # 4.83e-5 (fp16 input: 1.67e-5)
    (torch.float16, False): 2.75e-4,  # 2.27e-4: one fp16 rounding (4 columns, 52 values)
    (torch.float16, True): 2.75e-4,   # 2.28e-4
}
LN_COLS = [4, 64, 256, 260, 768, 1024, 1028, 1280, 2048]


@pytest.mark.parametrize("cols", LN_COLS)
@pytest.mark.parametrize("x_dtype,y_dtype", [(torch.float32, torch.float32), (torch.float32, torch.float16),
                                             (torch.float16, torch.float32), (torch.float16, torch.float16)])
@pytest.mark.parametrize("offset", [False, True])
def test_layernorm_rows(cols, x_dtype, y_dtype, offset):
    """13 rows (not a multiple of the 8 per CTA) read from a column slice of a wider buffer and written into one, whose
    guard columns and rows keep their fill; rows of mean ~1e3 and std ~1 catch a variance that cancels"""
    from ctrlora_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(cols + 3 * offset)
    rows = 13
    xs = torch.randn((rows, cols + 12), device="cuda", generator=gen) + (1000.0 if offset else 0.0)
    x = xs.to(x_dtype)[:, 4:4 + cols]
    gamma = 1 + 0.1 * torch.randn(cols, device="cuda", generator=gen)
    beta = 0.1 * torch.randn(cols, device="cuda", generator=gen)
    ybuf = torch.full((rows + GUARD_ROWS, cols + 16), GUARD, device="cuda", dtype=y_dtype)
    y = ybuf[:rows, 8:8 + cols]
    ops.layernorm_rows(x, gamma, beta, 1e-5, out=y)
    ref = F.layer_norm(x.double(), (cols,), gamma.double(), beta.double(), 1e-5)
    err = ((y.double() - ref).norm() / ref.norm()).item()
    print(f"layernorm_rows {x_dtype} -> {y_dtype}, {cols} cols, offset {offset}: norm-relative {err:.2e}")
    assert err < LN_TOL[(y_dtype, offset)]
    mask = torch.ones_like(ybuf, dtype=torch.bool)
    mask[:rows, 8:8 + cols] = False
    assert (ybuf[mask] == GUARD).all()
    assert torch.equal(ops.layernorm_rows(x, gamma, beta, 1e-5, out_f32=y_dtype == torch.float32), y)


def test_layernorm_rows_pooled_rows():
    """the vision tower's pooled class rows: one row per image at a stride of 257 rows (image_encoder.py post_layernorm)"""
    from ctrlora_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(9)
    b, c = 5, 1280
    h = torch.randn((b * 257, c), device="cuda", generator=gen)
    gamma = 1 + 0.1 * torch.randn(c, device="cuda", generator=gen)
    beta = 0.1 * torch.randn(c, device="cuda", generator=gen)
    pooled = h.view(b, 257, c)[:, 0]
    y = ops.layernorm_rows(pooled, gamma, beta, 1e-5, out_f32=True)
    ref = F.layer_norm(pooled.double(), (c,), gamma.double(), beta.double(), 1e-5)
    err = ((y.double() - ref).norm() / ref.norm()).item()
    print(f"layernorm_rows pooled rows: norm-relative {err:.2e}")
    assert err < LN_TOL[(torch.float32, False)]
    assert torch.equal(y, ops.layernorm_rows(pooled.contiguous(), gamma, beta, 1e-5, out_f32=True))


def test_layernorm_rows_rejects_unsupported_widths():
    from ctrlora_b200 import _lib
    lib = _lib.load()
    x = torch.zeros((2, 2056), device="cuda")
    g = torch.ones(2056, device="cuda")
    y = torch.empty_like(x)

    def call(cols):
        return lib.ctrlora_layernorm_rows(x.data_ptr(), 1, 2056, y.data_ptr(), 1, 2056, 2, cols, g.data_ptr(), g.data_ptr(),
                                          1e-5, _sp())
    assert call(2052) == 4  # CTRLORA_STATUS_UNSUPPORTED: more columns than the widest register tile holds
    assert call(766) == 1   # CTRLORA_STATUS_BAD_ARGUMENT: cols % 4 != 0
    assert call(2048) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ casts and gathers
def test_cast_rows():
    from ctrlora_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(12)
    rows, cols, lds = 37, 300, 328
    src = torch.randn((rows, lds), device="cuda", generator=gen) * 300
    src[0, :6] = torch.tensor([7e4, -7e4, 3e-8, -3e-8, 65519.0, 2.0 ** -24 * 1.5], device="cuda")  # overflow, subnormals, ties
    got = ops.cast_rows(src, rows, cols, lds)
    assert torch.equal(got.view(torch.int16), src[:, :cols].half().view(torch.int16))


def test_im2col_s2_pad_lo_1_entry_point():
    """ctrlora_im2col_s2_f16 is the pad_lo = 1 case of ctrlora_im2col_s2_pad_f16"""
    from ctrlora_b200 import _lib, ops
    gen = torch.Generator(device="cuda").manual_seed(13)
    x = _rand(3, 10, 14, 24, gen=gen)
    want = ops.im2col_s2(x, pad_lo=1)
    got = torch.full_like(want, GUARD)
    assert _lib.load().ctrlora_im2col_s2_f16(x.data_ptr(), got.data_ptr(), 3, 10, 14, 24, _sp()) == 0
    assert torch.equal(got, want)
    xp = F.pad(x.float().permute(0, 3, 1, 2), (1, 1, 1, 1))
    cols = F.unfold(xp, 3, stride=2).view(3, 24, 9, 5, 7).permute(0, 3, 4, 2, 1).reshape(3, 5, 7, 9 * 24)
    assert torch.equal(got.float(), cols)
