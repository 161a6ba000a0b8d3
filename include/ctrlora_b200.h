/* ctrlora_b200 C ABI — the drop-in boundary underneath the reference's Python module contract.
 *
 * The reference (xyfJASON/ctrlora) has no FFI of its own: its hot path is torch calls (SURVEY.md §8b).  Every entry
 * point below replaces one group of those torch call sites with a hand-written sm_90a kernel; the reference file:line
 * each one stands in for is cited on the declaration.  Conventions: plain pointers and sizes, device pointers unless
 * stated, no allocation inside (workspaces are passed in), the launch goes on `stream` (a cudaStream_t passed as
 * void*), the return value is a status code (0 = ok), no exceptions cross the boundary.
 *
 * Activations are NHWC fp16 ("pixel-major"): a [B, H, W, C] tensor is a [B*H*W, C] row-major matrix, so the
 * transformer's 'b c h w -> b (h w) c' rearranges (reference ldm/modules/attention.py:330,337) are no-ops.
 */
#ifndef CTRLORA_B200_H
#define CTRLORA_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define CTRLORA_ABI_VERSION 3

/* status codes */
#define CTRLORA_STATUS_OK 0
#define CTRLORA_STATUS_BAD_ARGUMENT 1
#define CTRLORA_STATUS_CUDA_ERROR 2
#define CTRLORA_STATUS_TENSORMAP_ERROR 3
#define CTRLORA_STATUS_UNSUPPORTED 4

int ctrlora_abi_version(void);
/* Last CUDA error string seen by this library on the calling thread's device (host pointer, static storage). */
const char* ctrlora_last_cuda_error(void);

/* cudaMemsetAsync(ptr, 0, bytes) on `stream`: a memset node, not a kernel (zero-initialised key padding of V^T etc.) */
int ctrlora_memset_zero(void* ptr, long long bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Implicit GEMM on the Hopper tensor cores (wgmma, accumulators in registers, operands staged by TMA):
 *   out[m, n] = epilogue( sum_{tap, c} A[pixel(m) + tap_offset, c] * W[n, tap, c]  (+ sum_c A2[pixel(m), c] * W2[n, c]) )
 * replaces  nn.Linear / F.linear              ldm/modules/attention.py:154-161,52,72; cldm/lora.py:287-290
 *           nn.Conv2d 1x1 and 3x3 stride 1    ldm/modules/diffusionmodules/openaimodel.py:196,228-240,729; cldm/cldm.py:281-282
 *           GEGLU                             ldm/modules/attention.py:49-56      (geglu = 1)
 *           the ResBlock skip connection      openaimodel.py:233-240,272-274      (a2/w2 = 1x1 skip conv, or residual)
 *           h + emb_out[..., None, None]      openaimodel.py:263-270              (rowbias)
 *           control_i * control_scales[i]     cldm/cldm_ctrlora_finetune.py:79    (out_scale)
 * A plain [M, K] matrix is a_b = 1, a_h = 1, a_w = M, a_c = K, kh = kw = 1, pad = 0.
 */
typedef struct ctrlora_gemm_args {
    const void* a;          /* fp16 activations, pixel-major; channel stride 1, pixel stride a_ld elements */
    int a_b, a_h, a_w, a_c;
    long long a_ld;
    const void* w;          /* fp16 weights [n (2n for GEGLU), kh*kw, a_c], dense */
    int kh, kw, pad;        /* 1x1 (pad 0), 3x3 (pad 1) or 7x7 (pad 3), stride 1 */
    const void* a2;         /* optional second activation operand with the same B,H,W (1x1), or NULL */
    int a2_c;
    long long a2_ld;
    const void* w2;         /* [n, a2_c] */
    int n;                  /* output columns */
    int block_n;            /* 0 = choose automatically */
    int geglu;
    void* out[3];           /* out[0] always; out[1..2] when seg_width > 0 */
    int seg_width;          /* 0 = single output; else column n is stored to out[n / seg_width] at column n % seg_width */
    int transposed[3];      /* segment stored as [image, seg_width, tok_pad] (i.e. [image, head, d, token]) */
    int ldc;                /* row stride (elements) of the non-transposed outputs */
    int out_f32;            /* 0: fp16 outputs, 1: fp32 outputs */
    const float* bias;      /* [n] ([2n] for GEGLU) or NULL */
    const float* rowbias;   /* [images, n] fp32 or NULL */
    int rows_per_img;       /* rows per image for rowbias / transposed stores; 0 = a_h * a_w */
    int rowbias_ld;         /* row stride of rowbias (0 = n): lets one batched time-embedding GEMV feed every ResBlock */
    const void* residual;   /* [M, ldr] added after scaling, or NULL; fp16 unless residual_f32 */
    int ldr;
    int residual_f32;
    float out_scale;        /* applied to (acc + bias + rowbias) */
    int head_dim, tok_pad;  /* for transposed stores */
    int bf16;               /* must be 0 (fp16 operands) in this ABI version */
    int split_k;            /* 0 = choose automatically (needs the workspace below), 1 = never split */
    float* splitk_ws;       /* fp32 scratch for the per-split partial tiles (no initial contents required) */
    long long splitk_ws_bytes;
    unsigned int* splitk_counters;   /* arrival counters: all zero on entry, left all zero on exit */
    int splitk_counters_len;
    void* dup_out;          /* optional: transposed segments are also stored row-major here (fp16, row stride dup_ld) */
    int dup_ld;
    int force_single_cta;   /* accepted for ABI compatibility; every tile is one CTA */
    /* Grouped launch: two same-shaped layers of two networks over one batch (the ControlNet and the UNet encoder run as
     * one pass).  group_b > 0: images (a_b index) >= group_b take w_hi, w2_hi, bias_hi and rowbias_hi, whose rows are
     * indexed from image img - group_b * a_h * a_w / rows_per_img.  Every tile must lie in one group: when group_b is
     * not a multiple of the images one tile covers, the call returns CTRLORA_STATUS_UNSUPPORTED and launches nothing. */
    int group_b;
    const void* w_hi;
    const float* bias_hi;
    const float* rowbias_hi;
    const void* w2_hi;
    /* relu = 1: max(v, 0) as the last step before the output rounding, after bias, row term, scale and residual (split
     * tiles: after the split-K sum).  The ReLU of HED's conv + ReLU pairs (annotator/hed/__init__.py:30-31).
     * relu = 2: min(max(v, 0), 6) as that last step: the ReLU6 of M-LSD's ConvBNReLU (annotator/mlsd/models/
     * mbv2_mlsd_large.py:107).  relu = 3: max((acc + bias + row term) * scale, 0) + residual, the ReLU before the
     * residual add: BlockTypeB's relu(bn(conv1(x))) + x (mbv2_mlsd_large.py:47).  Other values are rejected. */
    int relu;
} ctrlora_gemm_args;

int ctrlora_gemm_f16(const ctrlora_gemm_args* args, void* stream);

/* Bring-up / bisecting twin of ctrlora_gemm_f16 on the CUDA cores (same arguments, same results up to fp32
 * summation order).  Only the tests call it. */
int ctrlora_gemm_f16_simt(const ctrlora_gemm_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * GroupNorm (+SiLU) over pixel-major fp16, fp32 statistics, optionally over the channel concatenation
 * [x1 (+ add1_scale*add1) | x2 (+ add2_scale*add2)].
 * replaces  GroupNorm32 + SiLU              ldm/modules/diffusionmodules/util.py:202-219, openaimodel.py:190-197,221-231,726-730
 *           Normalize (eps 1e-6)            ldm/modules/attention.py:88-89,327
 *           h += control.pop(); cat([h, hs.pop() + control.pop()], 1)    cldm/cldm.py:34-42
 */
typedef struct ctrlora_groupnorm_args {
    const void* x1; const void* add1; float add1_scale; int c1; long long ld1;
    const void* x2; const void* add2; float add2_scale; int c2; long long ld2;   /* x2 = NULL: single source */
    int batch, hw, groups;
    const float* gamma; const float* beta; float eps; int silu;
    void* y;          /* fp16 [batch*hw, c1+c2] */
    void* raw_out;    /* optional fp16 [batch*hw, c1+c2]: the concatenated (and summed) input itself, or NULL */
    void* stats_ws;   /* fp32 workspace [batch * groups * 2] */
    float* partial_ws;   /* required: scratch for per-block partial statistics (any contents), so that the forward and the
                            backward's dx are bit-reproducible: no fp32 atomics in the statistics, the last block of an image
                            sums the partials in a fixed order (the backward's dgamma/dbeta still accumulate atomically).
                            The call returns CTRLORA_STATUS_BAD_ARGUMENT and launches nothing when partial_ws or
                            partial_counters is NULL, when batch > partial_counters_len, or when the two-pass launch's
                            partials (batch * blocks per image * groups * 2 floats) exceed partial_ws_floats. */
    long long partial_ws_floats;
    unsigned int* partial_counters;   /* [>= batch] arrival counters: all zero on entry, left all zero on exit */
    int partial_counters_len;
    /* Grouped forward (two networks' GroupNorms over one batch): images >= group_b (0 = off) take gamma_hi / beta_hi.
     * Statistics stay per image and are computed as by a call over images [0, group_b) and one over the rest. */
    const float* gamma_hi; const float* beta_hi; int group_b;
} ctrlora_groupnorm_args;
int ctrlora_groupnorm_f16(const ctrlora_groupnorm_args* args, void* stream);

/* LayerNorm over the last dim (eps 1e-5 in the reference: ldm/modules/attention.py:263-265), fp16 in/out. */
int ctrlora_layernorm_f16(const void* x, long long ldx, void* y, long long ldy, int rows, int cols,
                          const float* gamma, const float* beta, float eps, void* stream);
/* The same LayerNorm over the rows of two networks' layers in one launch: rows >= split_rows take gamma_hi / beta_hi. */
int ctrlora_layernorm_grouped_f16(const void* x, long long ldx, void* y, long long ldy, int rows, int cols,
                                  const float* gamma, const float* beta, const float* gamma_hi, const float* beta_hi,
                                  int split_rows, float eps, void* stream);

/* Fused attention forward: out[b, i, h*d:(h+1)*d] = softmax_j(q_i . k_j * d^-1/2) v_j   (fp32 logits / softmax).
 * replaces CrossAttention.forward   ldm/modules/attention.py:163-194 (and MemoryEfficientCrossAttention :197-243).
 * q [batch, nq, heads*d] (row stride ldq), k [batch, nk, heads*d] (ldk), vt = V transposed [batch, heads, d, nk_pad]. */
int ctrlora_attention_f16(const void* q, long long ldq, const void* k, long long ldk, const void* vt, int nk_pad,
                          void* out, long long ldo, float* lse /* optional [batch, heads, nq], log2 domain */, int batch,
                          int heads, int nq, int nk, int head_dim, void* stream);

/* Module-boundary layout/dtype conversion (the reference's tensors are NCHW fp32). */
int ctrlora_nchw_f32_to_nhwc_f16(const float* src, void* dst, int batch, int channels, int hw, int c_pad, void* stream);
int ctrlora_nhwc_to_nchw_f32(const void* src, int src_is_f32, long long ld, float* dst, int batch, int channels, int hw,
                             void* stream);

/* timestep_embedding   ldm/modules/diffusionmodules/util.py:154-174: out[b] = [cos(t_b * f) | sin(t_b * f)];
 * freqs (fp32 [half]) are computed on the host exactly as the reference does; t is int64. */
int ctrlora_timestep_embedding(const long long* t, const float* freqs, float* out, int batch, int half, void* stream);
/* timestep_embedding   ldm/modules/diffusionmodules/util.py:154-174 at fp32 t (the reference embeds `t[:, None].float()`,
 * :168): DPM-Solver's model times (t_continuous - 1/N) * 1000 (ldm/models/diffusion/dpm_solver/dpm_solver.py:246-253)
 * are fractional.  arg = t[b] * freqs[k] rounded once, then accurate cosf / sinf; integer-valued t gives the bits of
 * ctrlora_timestep_embedding. */
int ctrlora_timestep_embedding_f32(const float* t, const float* freqs, float* out, int batch, int half, void* stream);

/* y = act_out(act_in(x) W^T + b) for M = batch rows, fp32 activations, fp16 weights [n, k].
 * replaces time_embed (Linear-SiLU-Linear, openaimodel.py:526-531) and every ResBlock emb_layers (SiLU-Linear, :208-215). */
int ctrlora_small_linear(const float* x, int ldx, const void* w, const float* bias, float* y, int ldy, int rows, int n,
                         int k, int silu_in, int silu_out, void* stream);

/* F.interpolate(scale_factor=2, mode='nearest')   openaimodel.py:115 */
int ctrlora_upsample2x_f16(const void* src, void* dst, int batch, int h, int w, int channels, void* stream);
/* gather for Downsample's conv3x3 stride 2 pad 1 (openaimodel.py:148-159): dst [batch, h/2, w/2, 9, channels] */
int ctrlora_im2col_s2_f16(const void* src, void* dst, int batch, int h, int w, int channels, void* stream);
/* same gather with the zero padding only on the right/bottom when pad_lo = 0: the first-stage VAE's
 * F.pad(x, (0,1,0,1)) + Conv2d(stride 2, padding 0), ldm/modules/diffusionmodules/model.py:80-84 */
int ctrlora_im2col_s2_pad_f16(const void* src, void* dst, int batch, int h, int w, int channels, int pad_lo, void* stream);
/* softmax(scale * src) over rows, fp32 logits -> fp16 probabilities: the VAE's d = 512 single-head AttnBlock
 * (model.py:179-203), whose logits come from ctrlora_gemm_f16 with out_f32 = 1 */
int ctrlora_softmax_rows_f32_to_f16(const float* src, long long lds, void* dst, long long ldd, long long rows, int cols,
                                    float scale, void* stream);
/* DiagonalGaussianDistribution.sample() / .mode() times scale_factor (ldm/modules/distributions/distributions.py:24-37,
 * ldm/models/diffusion/ddpm.py get_first_stage_encoding): moments fp32 [batch, 2*z, hw]; noise NULL = mode. */
int ctrlora_gaussian_sample(const float* moments, const float* noise, float* out, int batch, int z_channels, int hw, float scale,
                            void* stream);
/* weight preparation: fp32 [batch, rows, cols] -> fp16 [batch, cols, rows] */
int ctrlora_cast_transpose_f32_to_f16(const float* src, void* dst, long long batch, int rows, int cols, void* stream);

/* fp16 [batch, rows, cols] -> fp16 [batch, cols, rows] (transposed weight copies for the data-gradient GEMMs) */
int ctrlora_transpose_f16(const void* src, void* dst, long long batch, int rows, int cols, void* stream);

/* conv kernel weight fp16 [cout, taps, cin] -> data-gradient weight [cin, taps reversed, cout]: dx = conv(dy, W_d) with the
 * same padding -- the adjoint of torch.nn.Conv2d (ldm/modules/diffusionmodules/util.py:224 conv_nd) that autograd applies;
 * rebuilt every step in pretraining, where the conv weights train (cldm/cldm_ctrlora_pretrain.py:88-96). */
int ctrlora_conv_dgrad_weight_f16(const void* src, void* dst, int cout, int taps, int cin, void* stream);

/* Persistent GEMM and attention-forward grids use at most `limit` SMs from now on (0 = all of them): the gradient all-reduce that overlaps the
 * ControlNet backward (the reference's DDP does the same overlap by buckets, pytorch_lightning strategy "ddp",
 * train_ctrlora_pretrain.py) owns a few SMs, and a 148-CTA persistent grid would wait for them.  Read at launch time. */
int ctrlora_set_sm_limit(int limit);

/* DDIM update in one pass   cldm/ddim_hacked.py:190-192 (CFG, e_uncond may be NULL), :208-231 (pred_x0, x_prev).
 * fp32, round-to-nearest ops in the reference's order. stats (optional, [batch]) receives sum(x_prev^2) per image. */
int ctrlora_ddim_update(const float* x, const float* e_cond, const float* e_uncond, const float* noise, float* x_prev,
                        float* pred_x0, float* stats, int batch, int per_image, float cfg_scale, float a_t, float a_prev,
                        float sigma_t, float sqrt_one_minus_at, float temperature, void* stream);

/* q_sample (ldm/models/diffusion/ddpm.py:356-359) and DDIMSampler.stochastic_encode (cldm/ddim_hacked.py:281-296):
 * out[b] = tab_a[t[b]] * x0[b] + tab_s[t[b]] * noise[b]; t int64 [batch] (device), tables fp32 (device).  Bit-exact. */
int ctrlora_q_sample(const float* x0, const float* noise, const long long* t, const float* tab_a, const float* tab_s,
                     float* out, int batch, int per_image, void* stream);
/* DDIM inversion step (cldm/ddim_hacked.py:253-267): e = e_uncond + cfg*(e_cond - e_uncond) (e_uncond may be NULL), then
 * x_next = c1 * x + c2 * e with c1 = sqrt(a_next/a), c2 = sqrt(a_next) * (sqrt(1/a_next - 1) - sqrt(1/a - 1)) evaluated
 * by the caller in fp32 like the reference's 0-dim tensor arithmetic. */
int ctrlora_ddim_encode_update(const float* x, const float* e_cond, const float* e_uncond, float* x_next, int total,
                               float cfg_scale, float c1, float c2, void* stream);
/* One step of DPMSolverSampler (ldm/models/diffusion/dpm_solver/sampler.py:72-85: DPM-Solver++, multistep, data
 * prediction), all fp32 with round-to-nearest ops in the reference's order (dpm_solver.py):
 *   e = e_uncond + cfg * (e_cond - e_uncond)                 :311-312 (e_uncond may be NULL: no guidance)
 *   m_out = (x - sigma_s * e) / alpha_s                      :356-359 (data prediction at the step's start time)
 *   x_next = c_x * x - c_m * m_out                           order 1, :490-497 (m_prev NULL)
 *            - c_d * (inv_r0 * (m_out - m_prev))             order 2, :748-758
 * The per-step scalars (c_x = sigma_t / sigma_s, c_m = alpha_t * expm1(-h) or alpha_t * (exp(-h) - 1),
 * c_d = 0.5 * c_m, inv_r0 = 1 / r0) are computed by the caller from NoiseScheduleVP('discrete') (:60-160). */
int ctrlora_dpm_multistep_update(const float* x, const float* e_cond, const float* e_uncond, const float* m_prev, float* m_out,
                                 float* x_next, int total, float cfg_scale, float sigma_s, float alpha_s, float c_x, float c_m,
                                 float c_d, float inv_r0, void* stream);
/* One step of PLMSSampler (ldm/models/diffusion/plms.py:178-244, eta 0), fp32 with round-to-nearest ops in torch's order:
 *   e = e_uncond + cfg * (e_cond - e_uncond) -> e_out               :184-192 (e_uncond may be NULL: no guidance); the
 *                                                                   guided e_t the caller keeps as old_eps (:164-167)
 *   e' = (e + e_next) / 2                       order 0             :227-231 (e_next guided from e_next_cond /
 *                                                                   e_next_uncond, the eval at t_next on the provisional
 *                                                                   x_prev that ctrlora_ddim_update gives)
 *        e                                      order 1             (a DDIM step; PLMSSampler does not use it)
 *        (3 e - o1) / 2                         order 2             :232-234
 *        (23 e - 16 o1 + 5 o2) / 12             order 3             :235-237
 *        (55 e - 59 o1 + 37 o2 - 9 o3) / 24     order 4             :238-240   (o1 = old_eps[-1], o2 = [-2], o3 = [-3])
 *   pred_x0 = (x - sqrt_one_minus_at * e') / sqrt_a_t               :207-213
 *   x_prev = sqrt_a_prev * pred_x0 + dir_coef * e'                  :219-223 (dir_coef = sqrt(1 - a_prev - sigma_t^2))
 * The divisions are products with the fp32 reciprocal, as torch computes a CUDA tensor divided by a Python number.
 * Inputs an order does not read must be NULL.  The scalars are computed by the caller in torch CPU fp32 ops, the
 * reference's values as run on a CPU (whose sqrt is not always correctly rounded, unlike the sqrtf of
 * ctrlora_ddim_update). */
int ctrlora_plms_update(const float* x, const float* e_cond, const float* e_uncond, const float* e_next_cond,
                        const float* e_next_uncond, const float* old1, const float* old2, const float* old3, float* e_out,
                        float* x_prev, float* pred_x0, int order, int total, float cfg_scale, float sqrt_a_t,
                        float sqrt_one_minus_at, float sqrt_a_prev, float dir_coef, void* stream);

/* DPM_Solver (ldm/models/diffusion/dpm_solver/dpm_solver.py), every method and order.  fp32 contiguous tensors, all
 * arithmetic round-to-nearest in the reference's order; `coef` is a host array of CTRLORA_DPM_NCOEF floats formed by
 * ctrlora_b200.dpm_schedule on the CPU (unused entries are ignored). */
#define CTRLORA_DPM_NCOEF 9
#define CTRLORA_DPM_MODEL_NOISE 0
#define CTRLORA_DPM_MODEL_X_START 1
#define CTRLORA_DPM_MODEL_V 2
/* One model value, written to the caller's history slot m_out (model_wrapper :257-312, data_prediction_fn :352-359):
 *   e = to_noise(out_cond), to_noise by model_type: out | (x - alpha_w out) / sigma_w | alpha_w out + sigma_w x
 *   e = u + coef[0] * (e - u)                 u = to_noise(out_uncond), classifier-free guidance  (NULL: none)
 *   e = e - coef[3] * grad                    classifier guidance, coef[3] = scale * sigma_t      (NULL: none)
 *   m_out = (x - coef[4] * e) / coef[5]       predict_x0: sigma_t, alpha_t of the solver's schedule
 * coef[1] = alpha_w, coef[2] = sigma_w (the wrapper's schedule at t). */
int ctrlora_dpm_model_output(const float* x, const float* out_cond, const float* out_uncond, const float* grad,
                             float* m_out, long long total, int model_type, int predict_x0, const float* coef,
                             void* stream);
#define CTRLORA_DPM_UPDATE_FIRST 0
#define CTRLORA_DPM_UPDATE_DIFF 1
#define CTRLORA_DPM_UPDATE_MULTISTEP2 2
#define CTRLORA_DPM_UPDATE_MULTISTEP3 3
#define CTRLORA_DPM_UPDATE_SINGLESTEP3_TAYLOR 4
/* One update, out = a x - b m0 + ... with (a, b, c, d, k0, k1, k2, k3, rd) = coef[0..8]; c and d carry their sign:
 *   FIRST                 a x - b m0                                          dpm_solver_first_update :469-513, and
 *                                                                             every singlestep x_s1
 *   DIFF                  a x - b m0 + c (m1 - m0)                            singlestep-2 :553-593, singlestep-3 x_s2
 *                                                                             :655-698 and 'dpm_solver' x_t :661-705
 *   MULTISTEP2            D = k0 (m0 - m1); a x - b m0 + c D                  :751-777 (m0 newest, m1 previous)
 *   MULTISTEP3            D0 = k0 (m0 - m1), D1 = k1 (m1 - m2), G = D0 - D1;  :807-824
 *                         a x - b m0 + c (D0 + k2 G) + d (k3 G)
 *   SINGLESTEP3_TAYLOR    D0 = k0 (m1 - m0), D1 = k1 (m2 - m0);               'taylor' x_t :668-677, :707-716
 *                         a x - b m0 + c ((k3 D0 - k2 D1) / rd) + d ((2 (D1 - D0)) / rd)
 * m1 / m2 are NULL exactly when the mode does not read them. */
int ctrlora_dpm_solver_update(const float* x, const float* m0, const float* m1, const float* m2, float* out,
                              long long total, int mode, const float* coef, void* stream);
/* Dynamic thresholding in place (data_prediction_fn :360-364), x0 [batch, per_image]: per image, the order statistics
 * k_lo / k_hi of |x0| joined as torch.quantile's lerp with `weight` (the fractional part of fp32(0.995) * (n - 1)),
 * s = max(that, max_val), x0 = clamp(x0, -s, s) / s.  s_out (optional, [batch]) receives s.  Radix select in shared
 * memory when the image fits, in global memory otherwise. */
int ctrlora_dpm_threshold(float* x0, float* s_out, int batch, long long per_image, long long k_lo, long long k_hi,
                          float weight, float max_val, void* stream);
/* Adaptive solver's error (dpm_solver_adaptive :926-928) into the device scalar err:
 * max over images of sqrt(mean(((x_higher - x_lower) / max(atol, rtol * max(|x_lower|, |x_prev|)))^2)).
 * The sum's order is a fixed tree, not torch's: E agrees with the reference to rounding, not to the bit. */
int ctrlora_dpm_adaptive_error(const float* x_lower, const float* x_prev, const float* x_higher, float* err, int batch,
                               long long per_image, float atol, float rtol, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Training (backward of the trainable set; reference: autograd over cldm/lora.py:70-80,285-291 and cldm/cldm.py:281-282,
 * parameters selected by cldm/cldm_ctrlora_finetune.py:88-100).
 *
 * Weight-gradient GEMM over the token dimension: out[p, q] = alpha * sum_m a[m, p] * b[m, q] + beta * out[p, q],
 * fp16 a [m, p_dim] (row stride lda), b [m, q_dim] (ldb), fp32 out (row stride ldo).  ws: fp32 scratch (any contents).
 */
int ctrlora_wgrad_tn_f16(const void* a, long long lda, const void* b, long long ldb, int m, int p_dim, int q_dim, float* out,
                         long long ldo, float alpha, float beta, float* ws, long long ws_bytes, void* stream);

/* Attention backward (autograd of ldm/modules/attention.py:163-194): v is the NATURAL [batch*nk, heads*d] layout; lse is
 * what ctrlora_attention_f16 wrote; delta_ws: fp32 scratch [batch*heads*nq].  dq/dk/dv: fp16, same layouts as q/k/v. */
int ctrlora_attention_bwd_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                              const void* o, long long ldo, const void* dout, long long lddo, const float* lse,
                              float* delta_ws, void* dq, long long lddq, void* dk, long long lddk, void* dv, long long lddv,
                              int batch, int heads, int nq, int nk, int head_dim, void* stream);

/* GroupNorm(+SiLU) backward: same source description as the forward (`args`, not grouped; its stats_ws is a scratch buffer for the
 * backward statistics); fwd_stats = the {sum, sumsq} buffer the forward left in ITS stats_ws.  dx1 / dx2: gradients of
 * the two concat halves (fp16, row strides ldd1 / ldd2, scaled by dx*_scale; dx2 may be NULL).  dgamma/dbeta (fp32 [C],
 * accumulated into) may be NULL. */
int ctrlora_groupnorm_bwd_f16(const ctrlora_groupnorm_args* args, const void* dy, const void* fwd_stats, void* dx1,
                              long long ldd1, float dx1_scale, void* dx2, long long ldd2, float dx2_scale,
                              const void* res /* optional fp16 [rows, ldres]: added to the concat gradient */, long long ldres,
                              float* dgamma, float* dbeta, void* stream);
/* LayerNorm backward (statistics recomputed from x); dgamma/dbeta accumulated into (may be NULL). */
int ctrlora_layernorm_bwd_f16(const void* x, long long ldx, const void* dy, long long ldy, void* dx, long long lddx, int rows,
                              int cols, const float* gamma, float eps, float* dgamma, float* dbeta,
                              const void* res /* optional fp16 residual-branch gradient added to dx */, long long ldres,
                              void* stream);
/* GEGLU on the stored projection h = [value | gate] ([rows, 2n]): out = value * gelu(gate), and its backward. */
int ctrlora_geglu_fwd_f16(const void* h, void* out, long long rows, int n, void* stream);
int ctrlora_geglu_bwd_f16(const void* h, const void* dout, void* dh, long long rows, int n, void* stream);
/* out[c] += scale * sum_rows x[row, c]  (bias gradients); out[img, c] += per-image column sums (time-embedding gradients) */
int ctrlora_colsum(const void* x, int x_is_f32, long long ld, long long rows, int cols, float scale, float* out, void* stream);
int ctrlora_image_colsum_f16(const void* x, long long ld, int images, int rows_per_img, int cols, float* out, long long ldo,
                             void* stream);
/* Pretraining (every ControlNet parameter trainable, cldm/cldm_ctrlora_pretrain.py:174-182): dense weight gradients.
 * dW[Cout, tap, Cin] of a 3x3 stride-1 conv = ctrlora_wgrad_tn_f16(dY [M, Cout], col [M, 9*Cin]) with
 * col[b, h, w, tap, c] = x[b, h+kh-1, w+kw-1, c]: */
int ctrlora_im2col_3x3_f16(const void* src, void* dst, int batch, int h, int w, int channels, void* stream);
/* out[n, k] = beta*out + alpha * sum_b dy[b, n] * f(x[b, k]) (fp32; b = batch rows; f = SiLU when silu_x): time_embed /
 * emb_layers weight gradients */
int ctrlora_outer_accum_f32(const float* dy, int lddy, const float* x, int ldx, float* out, long long ldo, int rows, int n, int k,
                            float alpha, float beta, int silu_x, void* stream);
/* dst[r, c] (+)= src[r, c], fp32, row strides lds / ldd */
int ctrlora_copy2d_f32(const float* src, long long lds, float* dst, long long ldd, long long rows, int cols, int accumulate,
                       void* stream);
/* out = d * silu'(x) (fp32): backward of the SiLU in the time-embedding MLP (openaimodel.py:526-531, :208-215) */
int ctrlora_silu_bwd_f32(const float* d, const float* x, float* out, long long n, void* stream);
/* fp32 [rows, cols] (row stride lds) -> dense fp16 [rows, cols] */
int ctrlora_cast_rows_f32_to_f16(const float* src, long long lds, void* dst, long long rows, int cols, void* stream);
/* adjoints of ctrlora_upsample2x_f16 and ctrlora_im2col_s2_f16 */
int ctrlora_upsample2x_bwd_f16(const void* dout, void* din, int batch, int h, int w, int channels, void* stream);
int ctrlora_im2col_s2_bwd_f16(const void* dcol, void* dx, int batch, int h, int w, int channels, void* stream);
/* loss = mean((eps - noise)^2)  (ldm/models/diffusion/ddpm.py:902-918, logvar = 0) and its gradient, written as
 * pixel-major fp16 [batch, hw, c_pad] (times grad_scale); eps / noise are fp32 NCHW. */
int ctrlora_mse_loss_grad(const float* eps, const float* noise, float* loss, void* grad, int batch, int channels, int hw,
                          int c_pad, float grad_scale, void* stream);
/* torch.optim.AdamW step over one flat fp32 buffer (cldm/cldm_ctrlora_finetune.py:105: lr 1e-5, betas .9/.999, eps 1e-8,
 * weight decay 0.01); grads are multiplied by grad_scale first (1/(world_size * loss_scale) after an all-reduce SUM).
 * skip_flag (device int, may be NULL): when non-zero the step is skipped (loss-scale overflow, see below). */
int ctrlora_adamw_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr, float beta1,
                      float beta2, float eps, float weight_decay, int step, float grad_scale, const int* skip_flag,
                      const float* bc_dev /* optional device {1-beta1^step, 1-beta2^step} from ctrlora_adamw_begin; then `step`
                                             is ignored */,
                      void* stream);
/* In front of an AdamW step: ++*step_counter unless *skip_flag (then ++*skipped), bc[0..1] = 1 - beta^step.  Keeps torch's
 * per-parameter `step` semantics (skipped steps do not count) without a host read of the overflow flag every step. */
int ctrlora_adamw_begin(int* step_counter, const int* skip_flag, float beta1, float beta2, float* bc, int* skipped, void* stream);
/* *flag |= 1 if any element of x is NaN/Inf: the overflow check of the loss-scaled fp16 backward (the reference trains in
 * fp32 and has no such step; torch.cuda.amp.GradScaler semantics: skip the update, lower the scale). */
int ctrlora_nonfinite_flag_f32(const float* x, long long n, int* flag, void* stream);
/* out = sum_i weights[i] * srcs[i] over `count` (<= 8) fp16 tensors of n elements (n % 8 == 0), fp32 accumulation:
 * the weighted control sum of multi-LoRA inference, cldm/cldm_ctrlora_inference.py:172-176.  srcs / weights: HOST arrays. */
int ctrlora_weighted_sum_f16(const void* const* srcs, const float* weights, int count, void* out, long long n, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * CLIP text encoder (FrozenCLIPEmbedder, ldm/modules/encoders/modules.py:88-135, running transformers' CLIPTextModel).
 * Causal self-attention of CLIPAttention with its causal mask and no padding mask (the embedder passes no
 * attention_mask, :118-121): out[b, i, h*64:(h+1)*64] = sum_{j <= i} softmax_j(q_i . k_j / 8) v_j, fp32 logits and
 * softmax.  Operands as for ctrlora_attention_f16 (q, k [batch, n, heads*64], V^T [batch, heads, 64, nk_pad]); only
 * keys < n of V^T are read.  head_dim != 64 or n > 128: CTRLORA_STATUS_UNSUPPORTED. */
int ctrlora_causal_attention_f16(const void* q, long long ldq, const void* k, long long ldk, const void* vt, int nk_pad,
                                 void* out, long long ldo, int batch, int heads, int n, int head_dim, void* stream);
/* CLIPTextEmbeddings: out[b*n + t, :] = token_embedding[ids[b, t], :] + position_embedding[t, :] (fp32 tables [*, cols],
 * ids int64 [batch, n]); out fp32 or fp16 [batch*n, cols].  An id outside [0, vocab) fills its row with NaN. */
int ctrlora_clip_embed(const long long* ids, const float* token_embedding, const float* position_embedding, void* out,
                       int out_f32, int batch, int n, int cols, int vocab, void* stream);
/* quick-GELU x * sigmoid(1.702 x) (CLIP's hidden_act), fp32 math, in place on fp16 [n] (n % 8 == 0) */
int ctrlora_quick_gelu_f16(void* x, long long n, void* stream);
/* LayerNorm over the last dim with fp32 or fp16 input and output (x_f32 / y_f32): the CLIP encoder's layer_norm1/2 and
 * final_layer_norm on its fp32 residual stream.  cols % 4 == 0, cols <= 2048. */
int ctrlora_layernorm_rows(const void* x, int x_f32, long long ldx, void* y, int y_f32, long long ldy, int rows, int cols,
                           const float* gamma, const float* beta, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * IP-Adapter image encoder (app/gradio_ctrlora_style_transfer.py:385-409, running transformers'
 * CLIPVisionModelWithProjection and, for the negative content prompt, CLIPTextModelWithProjection).
 * Patch gather for CLIPVisionEmbeddings.patch_embedding (transformers models/clip/modeling_clip.py, Conv2d with
 * kernel = stride = patch and no bias), which then runs as one ctrlora_gemm_f16 with a [C, 1, k_pad] weight:
 * pixels fp32 (pixels_f32 = 1) or fp16 NCHW [batch, channels, image, image] -> fp16 [batch * P, k_pad], P = (image/patch)^2,
 * row b * P + py * (image/patch) + px, column c * patch^2 + kh * patch + kw; columns >= channels * patch^2 are zero.
 * image % patch == 0, k_pad % 8 == 0. */
int ctrlora_clip_patch_gather(const void* pixels, int pixels_f32, void* out, int batch, int channels, int image, int patch,
                              int k_pad, void* stream);
/* The same gather over a rectangular NCHW [batch, channels, h, w] image (MiDaS' ViT-L/16 patch embedding, forward_flex in
 * annotator/midas/midas/vit.py): a grid of gh = h / patch by gw = w / patch patches, rows and columns beyond patch * gh,
 * patch * gw are not read (the stride-patch Conv2d ignores them); row b * gh * gw + py * gw + px.  h = w is
 * ctrlora_clip_patch_gather, bit for bit (both run one kernel). */
int ctrlora_patch_gather_hw(const void* pixels, int pixels_f32, void* out, int batch, int channels, int h, int w, int patch,
                            int k_pad, void* stream);
/* CLIPVisionEmbeddings.forward after the conv: out[b * (P+1) + t, :] = (t == 0 ? class_embedding : patch_out[b * P + t-1, :])
 * + position_embedding[t, :], fp32 throughout (patch_out row stride ldp); pre_layrnorm follows as ctrlora_layernorm_rows. */
int ctrlora_clip_vision_embed(const float* patch_out, long long ldp, const float* class_embedding,
                              const float* position_embedding, float* out, int batch, int patches, int cols, void* stream);
/* exact GELU 0.5 x (1 + erf(x / sqrt 2)) (transformers' GELUActivation, hidden_act "gelu" of the ViT-H/14 image and text
 * towers), fp32 math, in place on fp16 [n] (n % 8 == 0) */
int ctrlora_gelu_f16(void* x, long long n, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Line-art annotator (annotator/lineart/__init__.py:36-91, informative-drawings' Generator, as
 * LineartDetector.__call__ :111-122 runs it).  Its convs become ctrlora_gemm_f16 launches over gathered operands.
 *
 * Tap gather: dst[b, y, x, t * channels + c] = src[b, Y(y + dy_t), X(x + dx_t), c] for the n_taps (dy, dx) pairs of the
 * host array `taps` (n_taps <= 64), fp16 [batch, h, w, k_pad]; columns >= n_taps * channels are zero.  reflect = 1: Y / X
 * mirror without repeating the border (nn.ReflectionPad2d, :21,25,41,77; |dy| < h, |dx| < w); reflect = 0: outside taps
 * read 0 (the sub-pixel phases of ConvTranspose2d(3, stride 2, padding 1, output_padding 1), :69).  src: fp16 pixel-major
 * [batch, h, w, ld] (src_f32_nchw = 0), or fp32 NCHW [batch, channels, h, w] (src_f32_nchw = 1, ld unused: the network
 * input of :116-119).  k_pad % 8 == 0.
 */
int ctrlora_tap_gather_f16(const void* src, int src_f32_nchw, long long ld, void* dst, int batch, int h, int w, int channels,
                           const int* taps, int n_taps, int reflect, int k_pad, void* stream);
/* ctrlora_tap_gather_f16 with an output stride and an activation on load (Anime2Sketch's UnetGenerator,
 * annotator/lineart_anime/__init__.py:73-99): dst is [batch, h / stride, w / stride, k_pad] and output pixel (y, x)
 * reads (stride y + dy, stride x + dx); stride 1 or 2, h / stride and w / stride rounded down (a stride-2 Conv2d's
 * truncation of odd sizes), at least 1.  act: 0 none, 1 ReLU (uprelu), 2
 * LeakyReLU(0.2) (downrelu), applied in fp32 to each gathered value before the fp16 rounding (zero-masked taps stay
 * 0).  stride = 1, act = 0 is ctrlora_tap_gather_f16, bit for bit. */
int ctrlora_tap_gather_act_f16(const void* src, int src_f32_nchw, long long ld, void* dst, int batch, int h, int w,
                               int channels, const int* taps, int n_taps, int reflect, int k_pad, int stride, int act,
                               void* stream);
/* InstanceNorm2d(affine = False, track_running_stats = False) (:14): per (image, channel) biased statistics over the
 * image's rows, then y = relu?((x - mean) / sqrt(var + eps)) + residual?, fp16 in and out, fp32 math (the ReLU of :24,44,54,71
 * and ResidualBlock's x + conv_block(x), :33).  phases = 0: x and y are [batch, h, w, channels].  phases = 1: x holds the
 * four sub-pixel phase outputs of a stride-2 transposed conv, [4, batch, h, w, channels] with phase 2 py + px, and y is
 * [batch, 2h, 2w, channels], y[b, 2m + py, 2n + px] = f(x[2 py + px, b, m, n]).  residual (or NULL) has y's layout.
 * Statistics: fixed per-image row chunks and a fixed summation order, no atomics (bit-reproducible, and independent of
 * the batch).  ws: fp32 scratch of at least 2 * batch * channels * 1025 floats.  channels in {64, 128, 256, 512}. */
int ctrlora_instance_norm_f16(const void* x, const void* residual, void* y, float* ws, long long ws_floats, int batch, int h,
                              int w, int channels, int phases, int relu, float eps, void* stream);
/* The output layer (:77-80): ReflectionPad2d(3) + Conv2d(channels -> 1, 7) + Sigmoid on fp16 [batch, h, w, channels]
 * (channels % 16 == 0, h, w > 3), fp32 accumulation.  weight: fp32 [49, channels] (tap-major), bias: fp32 [1] (device).
 * out: fp32 [batch, h, w]; out_u8 (or NULL): uint8 [batch, h, w] = (uint8)clip(out * 255, 0, 255) with an fp32 multiply
 * and truncation, as LineartDetector's `(line * 255.0).clip(0, 255).astype(np.uint8)` (:122). */
int ctrlora_lineart_out_f16(const void* x, const float* weight, const float* bias, float* out, unsigned char* out_u8,
                            int batch, int h, int w, int channels, void* stream);
/* Anime2Sketch's outermost up path (annotator/lineart_anime/__init__.py:85,112, as LineartAnimeDetector.__call__
 * :144 scales it): out = tanh(bias + ConvTranspose2d(channels -> 1, 4, stride 2, padding 1)(ReLU([skip | up]))) *
 * scale + shift, a multiply then an add in fp32.  skip and up: fp16 [batch, h, w, channels / 2] each (4-byte aligned),
 * the concatenation's two halves, never materialised; channels % 4 == 0, <= 128.  weight: fp32 [channels, 16], the
 * transposed kernel's [channels, 1, 4, 4]; bias: fp32 [1] (device).  out: fp32 [batch, 2h, 2w], fp32 accumulation. */
int ctrlora_lineart_anime_out_f16(const void* skip, const void* up, const float* weight, const float* bias, float* out,
                                  int batch, int h, int w, int channels, float scale, float shift, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * HED annotator (annotator/hed/__init__.py, ControlNetHED_Apache2 :36-52 as HEDdetector.__call__ :65-79 runs it).  Its
 * 3x3 conv + ReLU pairs (:28-31) are ctrlora_gemm_f16 launches with relu = 1.
 *
 * Side projection and pool: x is a block's output, fp16 [batch, h, w, channels] (channels in {64, 128, 256, 512}, 16-byte
 * aligned), read once.  side: fp32 [batch, h, w] = bias[0] + sum_c weight[c] * x[.., c], fp32 accumulation in a fixed
 * order (DoubleConvBlock.projection, :32).  pooled (or NULL): fp16 [batch, h / 2, w / 2, channels], the 2x2 max of x,
 * floor sizes (the next block's max_pool2d(2, 2), :28); a max is exact, so it equals max_pool2d on x bit for bit.
 * weight: fp32 [channels], bias: fp32 [1] (device).  weight = bias = side = NULL runs the pool alone (pooled is then
 * required): OpenPose's max pools (annotator/openpose/model.py:10-13).
 */
int ctrlora_hed_side_pool_f16(const void* x, const float* weight, const float* bias, float* side, void* pooled, int batch,
                              int h, int w, int channels, void* stream);
/* The detector's post-process (:70-78) for the five side maps at once.  sides[l]: fp32 [batch, side_hw[2l], side_hw[2l+1]];
 * level 0 is h x w and is taken as is (cv2.resize to its own size is a copy).  Levels 1..4 are resized bilinearly to
 * h x w through host-built tables (cv2's INTER_LINEAR coordinate rule): idx[l] int32 [h + w], the source row of each
 * output row then the source column of each output column, and frac[l] fp32 [h + w], their fractional weights (the
 * neighbour index is clamped to the map).  mean: fp32 [batch, h, w] = ((((e1 + e2) + e3) + e4) + e5) / 5 in fp32;
 * then edge = 1 / (1 + exp(-mean)) in float64, with safe = 1 safe_step's (float)(int)((float)edge * 3) / 2
 * (annotator/util.py:78-81), and out_u8 = (uint8)clip(edge * 255, 0, 255).  idx and frac of level 0 are unused. */
int ctrlora_hed_fuse(const float* const* sides, const int* side_hw, const int* const* idx, const float* const* frac,
                     float* mean, unsigned char* out_u8, int batch, int h, int w, int safe, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * OpenPose body estimator (annotator/openpose/body.py, Body.__call__ :24-138 with the single scale 0.5).  bodypose_model's
 * 3x3 and 7x7 conv + ReLU pairs are ctrlora_gemm_f16 launches with relu = 1; its max pools are
 * ctrlora_hed_side_pool_f16 with weight = side = NULL.  The host keeps the input resize, the greedy matching and the
 * assembly of people; these run the rest.
 *
 * Resampling tables: the reference resizes each stride-8 map by 8 (cv2 LANCZOS4), crops the padding and resizes to the
 * image (LANCZOS4 or INTER_AREA, annotator/openpose/util.py:10-35).  Both are linear and separable, so each axis is one
 * banded float64 matrix built on the host: output row y reads source rows y_start[y] ... y_start[y] + ty - 1 with
 * weights y_w[y * ty + i] (source rows < h8), and the same for columns (x_start, x_w, tx).  A resampled value is
 * sum_i y_w_i * (sum_j x_w_j * map) in float64, rounded once to fp32.
 *
 * Resample: maps fp32 pixel-major [h8, w8, map_ld] (one image); out: fp32 [channels, h, w], channels 0 .. channels - 1.
 */
int ctrlora_openpose_resample(const float* maps, int map_ld, int h8, int w8, int channels, const int* y_start,
                              const double* y_w, int ty, const int* x_start, const double* x_w, int tx, float* out, int h,
                              int w, void* stream);
/* scipy.ndimage.gaussian_filter with mode 'reflect' (body.py:84) on `maps` fp32 [h, w] maps, in float64: first along the
 * rows (axis 0) into tmp, then along the columns into out (both float64 [maps, h, w]), each as scipy's correlate1d
 * computes a symmetric kernel: in[0] * w[0], then + (in[-j] + in[+j]) * w[j] for j = radius ... 1.  weights: host array
 * of radius + 1 doubles (centre first), radius <= 16. */
int ctrlora_openpose_smooth(const float* in, double* tmp, double* out, int maps, int h, int w, const double* weights,
                            int radius, void* stream);
/* Peaks (body.py:86-100): element (m, y, x) of smoothed float64 [maps, h, w] is a peak when it is >= its four neighbours
 * (0 outside the map) and > thre.  Peaks are numbered in (m, y, x) order by a prefix sum: peak id gets px, py, part
 * (= m) and score = heat[m, y, x] (heat: the unsmoothed fp32 [maps, h, w]) when id < capacity.  ws: int32 scratch of at
 * least ceil(maps * h * w / 2048) + 1 ints; its last used entry, ws[ceil(maps * h * w / 2048)], receives the number of
 * peaks (which may exceed capacity: the caller then calls again with more room). */
int ctrlora_openpose_peaks(const double* smoothed, const float* heat, int maps, int h, int w, double thre, int* ws,
                           long long ws_ints, int* px, int* py, int* part, float* score, int capacity, void* stream);
/* Limb scores (body.py:107-131): for each of n_limbs (<= 32) limbs, limbs[7 k ...] = {first pair index, first peak of
 * part A, peaks of A (>= 1), first peak of part B, peaks of B (>= 1), PAF channel of x, PAF channel of y}, the pair
 * ranges consecutive and summing to `pairs`.  Pair (i, j) of a limb (index first + i * nB + j) samples the resampled
 * PAF (paf: fp32 pixel-major [h8, w8, paf_ld], the same tables as above) at the 10 points of np.linspace from peak A to
 * peak B rounded half to even, and gets, in float64 as numpy computes it: score = sum(dot(PAF, unit vector)) / 10 +
 * min(0.5 * img_h / max(0.001, norm) - 1, 0), and ok = (more than 8 of the 10 dots > thre) and score > 0. */
int ctrlora_openpose_limbs(const float* paf, int paf_ld, int h8, int w8, const int* y_start, const double* y_w, int ty,
                           const int* x_start, const double* x_w, int tx, const int* px, const int* py, const int* limbs,
                           int n_limbs, long long pairs, int img_h, double thre, double* score, unsigned char* ok,
                           void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * MiDaS DPT-Large depth annotator (annotator/midas/__init__.py MidasDetector, midas/dpt_depth.py, blocks.py, vit.py).
 * The ViT-L/16 runs on ctrlora_patch_gather_hw, ctrlora_gemm_f16, ctrlora_clip_vision_embed, ctrlora_layernorm_rows,
 * ctrlora_attention_f16 (d_head 64) and ctrlora_gelu_f16; the reassemble and fusion convs on ctrlora_gemm_f16 and
 * ctrlora_im2col_s2_pad_f16.
 *
 * ConvTranspose2d(kernel = stride = s) computed as one GEMM with N = s * s * channels (column (ky * s + kx) * channels + c)
 * and fp32 output: dst[b, y * s + ky, x * s + kx, c] = fp16(src[b, y, x, (ky * s + kx) * channels + c] + bias[c]).
 * src fp32 [batch, h, w, s * s * channels] dense, dst fp16 [batch, h * s, w * s, channels]; channels % 4 == 0, s <= 8. */
int ctrlora_depth_to_space_bias(const float* src, const float* bias, void* dst, int batch, int h, int w, int channels, int s,
                                void* stream);
/* sum = fp16(a + b) and relu = max(sum, 0) in one pass over fp16 [n] (n % 8 == 0, 16-byte aligned): the fusion block's
 * skip_add.add followed by its RCU's input ReLU.  b = NULL: relu = max(a, 0) only (sum must be NULL then); either output
 * may be NULL.  The ReLU is of the rounded sum. */
int ctrlora_add_relu_f16(const void* a, const void* b, void* sum, void* relu, long long n, void* stream);
/* F.interpolate(scale_factor=2, mode="bilinear", align_corners=True) on fp16 NHWC [batch, h, w, channels] -> [batch, 2h,
 * 2w, channels], fp32 weights and sums (source index ((in - 1) / (out - 1)) * dst, as torch's kernel forms it);
 * channels % 8 == 0.  FeatureFusionBlock_custom's and the DPT head's upsample. */
int ctrlora_upsample_bilinear2x_f16(const void* src, void* dst, int batch, int h, int w, int channels, void* stream);
/* ctrlora_upsample_bilinear2x_f16 with pixel strides src_ld and dst_ld (halves, % 8 == 0, >= channels), so that either
 * side may be a channel slice of a wider buffer: M-LSD's BlockTypeA upsamples into its half of the concatenation
 * (annotator/mlsd/models/mbv2_mlsd_large.py:27-29).  ld = channels on both sides is ctrlora_upsample_bilinear2x_f16. */
int ctrlora_upsample_bilinear2x_ld_f16(const void* src, int src_ld, void* dst, int dst_ld, int batch, int h, int w,
                                       int channels, void* stream);
/* The DPT head's Conv2d(channels -> 1, 1) + ReLU: out[p] = max(bias[0] + sum_c weight[c] * x[p, c], 0), fp32 sums in
 * channel order.  x fp16 [pixels, channels] dense, channels % 8 == 0, <= 64; weight fp32 [channels]; bias fp32 [1]
 * (device); out fp32 [pixels]. */
int ctrlora_midas_head_out_f16(const void* x, const float* weight, const float* bias, float* out, long long pixels,
                               int channels, void* stream);
/* MidasDetector.__call__'s post-process on fp32 depth [batch, h, w] (h, w >= 2), two launches: per image the min and max
 * into minmax fp32 [batch, 2] (exact, so independent of the reduction order), then per pixel, in fp32 with each
 * operation rounded on its own as numpy and cv2 compute it:
 *   dn = (d - min) / (max - min);  depth_u8 = u8(dn * 255)
 *   x, y = cv2.Sobel(d, CV_32F, 1, 0 / 0, 1, ksize=3), BORDER_REFLECT_101, on the raw depth; x = y = 0 where dn < bg_th
 *   n = sqrt(x^2 + y^2 + a^2);  normal_u8[.., 0..2] = u8([x, y, a] / n * 127.5 + 127.5)
 * u8(v) is numpy's clip(0, 255).astype(uint8).  depth_u8 uint8 [batch, h, w]; normal_u8 uint8 [batch, h, w, 3]. */
int ctrlora_midas_maps(const float* depth, float* minmax, unsigned char* depth_u8, unsigned char* normal_u8, int batch,
                       int h, int w, float a, float bg_th, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * UniFormer-S + UPerNet segmentation annotator (annotator/uniformer: mmseg's EncoderDecoder, UniFormer backbone,
 * UPerHead).  The patch embeds, 1x1 and 3x3 convs and linears run on ctrlora_patch_gather_hw, ctrlora_tap_gather_act_f16
 * and ctrlora_gemm_f16, the attention on ctrlora_attention_f16 (d_head 64), the norms on ctrlora_layernorm_rows.
 *
 * Depthwise Conv2d(channels, channels, k, padding k / 2, groups=channels), k = 3 or 5, on fp16 NHWC x [batch, h, w,
 * channels] (dense): out = fp16(residual + bias + sum over the taps of weight[ky * k + kx, c] * x), zero padding, fp32
 * sums.  weight fp32 [k * k, channels] (tap-major), bias fp32 [channels]; residual NULL or fp16 like out (it may be x:
 * x + dw(x) in one launch); out must not be x.  channels % 8 == 0. */
int ctrlora_dwconv_f16(const void* x, const float* weight, const float* bias, const void* residual, void* out, int batch,
                       int h, int w, int channels, int k, void* stream);
/* ctrlora_dwconv_f16 with a stride and an activation; stride 2 and act != 0 take k = 3 only (k = 5 with either returns
 * CTRLORA_STATUS_BAD_ARGUMENT).  stride 1: padding k / 2, the output is h x w (stride 1, act 0 is ctrlora_dwconv_f16).
 * stride 2: the TFLite padding of M-LSD's ConvBNReLU (F.pad(x, (0, 1, 0, 1)) then padding 0,
 * annotator/mlsd/models/mbv2_mlsd_large.py:98-100, 113-115): output pixel (y, x) reads rows 2y .. 2y + 2 and the same
 * columns, zero outside, and the output is floor(h / 2) x floor(w / 2).  act 0 none, 1 ReLU, 2 ReLU6
 * (min(max(v, 0), 6)), applied after bias and residual, before the one fp16 rounding; residual is shaped like out. */
int ctrlora_dwconv_act_f16(const void* x, const float* weight, const float* bias, const void* residual, void* out,
                           int batch, int h, int w, int channels, int k, int stride, int act, void* stream);
/* F.interpolate(size=(ho, wo), mode="bilinear", align_corners=False) on fp16 NHWC: src [batch, hi, wi] with pixel stride
 * src_ld (halves), dst [batch, ho, wo] with pixel stride dst_ld, `channels` channels from each pointer (so dst may be a
 * channel slice of a wider buffer).  torch's source rule (scale = in / out in fp32, r = max(scale (d + 0.5) - 0.5, 0)),
 * fp32 weights and sums; accumulate != 0: dst = fp16(dst + resized), one rounding.  channels, src_ld, dst_ld % 8 == 0;
 * dst must not overlap src. */
int ctrlora_resize_bilinear_f16(const void* src, int src_ld, void* dst, int dst_ld, int batch, int hi, int wi, int ho,
                                int wo, int channels, int accumulate, void* stream);
/* AdaptiveAvgPool2d(s) for each of n_sizes (<= 4) sizes (host array) in one launch, torch's bins (rows floor(i h / s) ..
 * ceil((i + 1) h / s) - 1, the same for columns), fp32 sums: src fp16 [batch, h, w] with pixel stride src_ld, dst fp16
 * rows of `channels`: size k's block starts at row batch * (sum of the squares of the sizes before it), row
 * (b * s + i) * s + j within it.  channels, src_ld % 8 == 0. */
int ctrlora_adaptive_avg_pool_f16(const void* src, int src_ld, void* dst, int batch, int h, int w, int channels,
                                  const int* sizes, int n_sizes, void* stream);
/* The segmentor's output from fp32 logits [batch, h4, w4, ld] (ld % 4 == 0, ld >= classes rounded up to 4): per pixel
 * of [batch, ho, wo], the logits resized to the network size [hn, wn] and then to [ho, wo] (two bilinear steps with
 * align_corners=False, as ctrlora_resize_bilinear_f16 computes them, in fp32; the network-size logits are evaluated
 * where the second step reads them and never stored), the first class with the largest value, rgb uint8 [batch, ho,
 * wo, 3] = palette[label] (uint8 [classes, 3], device) and, unless NULL, labels int32 [batch, ho, wo]. */
int ctrlora_seg_output(const float* logits, int ld, int classes, int batch, int h4, int w4, int hn, int wn, int ho, int wo,
                       const unsigned char* palette, unsigned char* rgb, int* labels, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * M-LSD line detector (annotator/mlsd/__init__.py MLSDdetector, models/mbv2_mlsd_large.py, utils.py pred_lines).  The
 * MobileNetV2 backbone and the decoder run on ctrlora_tap_gather_act_f16, ctrlora_gemm_f16 (relu = 2, 3),
 * ctrlora_dwconv_act_f16 and ctrlora_upsample_bilinear2x_ld_f16.
 *
 * The line decode (utils.py:19-41, deccode_output_score_and_ptss with ksize 3 and topk_n = CTRLORA_MLSD_TOPK): on the
 * head's fp32 map tp [batch, h, w, ld] (centre at column c_center, the four displacements at c_disp .. c_disp + 3),
 * per image: heat = sigmoid(centre) in fp32; score = heat where it equals the maximum of its 3 x 3 window (pixels
 * outside the map skipped, max_pool2d's -inf padding), else 0; the CTRLORA_MLSD_TOPK largest scores in descending
 * order, ties broken by the lower flat index y * w + x (so zero scores fill the slots left over, lowest indices first).
 * Per candidate: out_idx int32 [batch, TOPK] the flat index, out_val fp32 [batch, TOPK, 6] = (score, dist, d0, d1, d2,
 * d3) with d the displacements and dist = sqrt((d0 - d2)^2 + (d1 - d3)^2), each step rounded to fp32 as numpy does
 * (utils.py:66).  score_ws: fp32 [batch, h, w] workspace.  Two launches: the scores, then one CTA per image (a radix
 * select on the scores' bits and a rank sort, no atomics), so the result is deterministic and does not depend on the
 * batch.  h * w < TOPK returns CTRLORA_STATUS_BAD_ARGUMENT (torch.topk fails there too). */
#define CTRLORA_MLSD_TOPK 200
int ctrlora_mlsd_decode(const float* tp, int ld, int c_center, int c_disp, int batch, int h, int w, float* score_ws,
                        int* out_idx, float* out_val, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Canny edges (annotator/canny/__init__.py CannyDetector: cv2.Canny(img, low, high) with apertureSize 3 and the L1
 * gradient), bit for bit, in integer arithmetic.
 *
 * Classification: img uint8 [batch, h, w, 3] with row stride ld bytes (image stride h * ld, pixel stride 3) -> cls
 * uint8 [batch, h, w]: 0 none, 1 candidate, 2 strong.  Per channel the 3 x 3 Sobel dx, dy with the border replicated
 * and m = |dx| + |dy|; per pixel the (dx, dy, m) of the channel with the largest m (ties keep the lower channel).  With
 * x = |dx|, y = |dy| << 15 and TG22 = 13573 the direction is horizontal if y < x TG22, vertical if y > x TG22 +
 * (x << 16), else diagonal; magnitudes outside the image are 0 and a pixel is kept when m > m[left] && m >= m[right]
 * (horizontal), m > m[up] && m >= m[down] (vertical), m > m[up-right] && m > m[down-left] (diagonal, dx and dy of
 * opposite sign) or m > m[up-left] && m > m[down-right] (the other diagonal).  Candidate: kept and m > lo; strong:
 * candidate and m > hi.  lo <= hi, both already floored (and swapped) on the host.  One launch.
 *
 * Hysteresis: cls as above -> out uint8 [batch, h, w], 255 at every candidate 8-connected through candidates to a
 * strong pixel, else 0.  Union-find labelling in labels_ws (int32 [batch * h * w]) in four launches whatever the
 * content (tile-local union, union across tile borders, flatten and flag the roots with a strong member, output), no
 * host synchronisation, so the pair can be captured in a CUDA graph.  The atomics may link components in any order;
 * the output does not depend on it.
 *
 * Both: batch * h * w < 2^31, batch <= 65535, else CTRLORA_STATUS_BAD_ARGUMENT. */
int ctrlora_canny_classify(const unsigned char* img, long long ld, int batch, int h, int w, int lo, int hi,
                           unsigned char* cls, void* stream);
int ctrlora_canny_hysteresis(const unsigned char* cls, int batch, int h, int w, int* labels_ws, unsigned char* out,
                             void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CTRLORA_B200_H */
