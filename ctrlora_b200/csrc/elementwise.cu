// Small HBM/latency-bound kernels of the hot path: layout/dtype conversion at the module boundary, timestep embedding,
// the M = batch linears of the time-embedding MLP, nearest-2x upsample, the stride-2 gather, weight preparation and
// the DDIM and DPM-Solver++ updates.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

// ---- NCHW fp32 (reference tensor layout) -> pixel-major fp16 with the channel dim zero-padded to c_pad
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, __half* __restrict__ dst, int B, int C, int HW, int c_pad) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(B) * HW * c_pad;
    if (i >= total) return;
    const int c = static_cast<int>(i % c_pad);
    const long long pix = i / c_pad;
    const int b = static_cast<int>(pix / HW), p = static_cast<int>(pix % HW);
    dst[i] = c < C ? __float2half_rn(src[(static_cast<long long>(b) * C + c) * HW + p]) : __float2half_rn(0.f);
}

// ---- pixel-major (fp16 or fp32, row stride ld) -> NCHW fp32, first C channels
template <typename T>
__global__ void nhwc_to_nchw_kernel(const T* __restrict__ src, long long ld, float* __restrict__ dst, int B, int C, int HW) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(B) * C * HW;
    if (i >= total) return;
    const int p = static_cast<int>(i % HW);
    const int c = static_cast<int>((i / HW) % C);
    const int b = static_cast<int>(i / (static_cast<long long>(HW) * C));
    dst[i] = static_cast<float>(src[(static_cast<long long>(b) * HW + p) * ld + c]);
}

// ---- timestep_embedding: out[b] = [cos(t*f) | sin(t*f)], freqs computed on the host exactly like the reference
__global__ void timestep_embedding_kernel(const long long* __restrict__ t, const float* __restrict__ freqs,
                                          float* __restrict__ out, int B, int half) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half) return;
    const int b = i / half, k = i % half;
    const float arg = __fmul_rn(static_cast<float>(t[b]), freqs[k]);
    out[b * 2 * half + k] = cosf(arg);
    out[b * 2 * half + half + k] = sinf(arg);
}

// ---- same embedding at fp32 t (DPM-Solver's fractional model times, e.g. 949.05): the product is rounded once and fed
// to the accurate cosf / sinf (the __cosf / __sinf intrinsics are far off at |arg| ~ 1000)
__global__ void timestep_embedding_f32_kernel(const float* __restrict__ t, const float* __restrict__ freqs,
                                              float* __restrict__ out, int B, int half) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * half) return;
    const int b = i / half, k = i % half;
    const float arg = __fmul_rn(t[b], freqs[k]);
    out[b * 2 * half + k] = cosf(arg);
    out[b * 2 * half + half + k] = sinf(arg);
}

// ---- y[b, n] = act_out( sum_k act_in(x[b, k]) * W[n, k] + bias[n] ),  b < rows <= 8 per pass; one warp per n.
// fp32 activations (the time embedding stays fp32 end to end), fp16 weights.
__global__ void __launch_bounds__(256)
small_linear_kernel(const float* __restrict__ x, int ldx, const __half* __restrict__ w, const float* __restrict__ bias,
                    float* __restrict__ y, int ldy, int rows, int N, int K, int silu_in, int silu_out) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    for (int r0 = 0; r0 < rows; r0 += 8) {
        float acc[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) acc[r] = 0.f;
        for (int k = lane * 8; k < K; k += 256) {
            uint4 u = *reinterpret_cast<const uint4*>(w + static_cast<long long>(n) * K + k);
            const __half2* h = reinterpret_cast<const __half2*>(&u);
            float wv[8];
#pragma unroll
            for (int e = 0; e < 4; ++e) { float2 f = __half22float2(h[e]); wv[2 * e] = f.x; wv[2 * e + 1] = f.y; }
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                if (r0 + r < rows) {
                    const float* xp = x + static_cast<long long>(r0 + r) * ldx + k;
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        float xv = xp[e];
                        if (silu_in) xv = silu_f(xv);
                        acc[r] += xv * wv[e];
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
        }
        if (lane == 0) {
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                if (r0 + r < rows) {
                    float v = acc[r] + (bias ? bias[n] : 0.f);
                    if (silu_out) v = silu_f(v);
                    y[static_cast<long long>(r0 + r) * ldy + n] = v;
                }
            }
        }
    }
}

// ---- nearest-neighbour 2x upsample (F.interpolate(scale_factor=2, mode='nearest')), pixel-major fp16, 16 B vectors
__global__ void upsample2x_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int B, int H, int W, int vecs) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(B) * 4 * H * W * vecs;
    if (i >= total) return;
    const int v = static_cast<int>(i % vecs);
    long long pix = i / vecs;
    const int ow = static_cast<int>(pix % (2 * W));
    pix /= 2 * W;
    const int oh = static_cast<int>(pix % (2 * H));
    const int b = static_cast<int>(pix / (2 * H));
    dst[i] = src[((static_cast<long long>(b) * H + (oh >> 1)) * W + (ow >> 1)) * vecs + v];
}

// ---- stride-2 3x3 pad-1 gather: col[b, oh, ow, tap, c] = x[b, 2*oh + kh - 1, 2*ow + kw - 1, c] (0 outside)
__global__ void im2col_s2_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int B, int H, int W, int vecs,
                                 int pad_lo) {
    const int Ho = H / 2, Wo = W / 2;
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(B) * Ho * Wo * 9 * vecs;
    if (i >= total) return;
    const int v = static_cast<int>(i % vecs);
    long long r = i / vecs;
    const int tap = static_cast<int>(r % 9);
    r /= 9;
    const int ow = static_cast<int>(r % Wo);
    r /= Wo;
    const int oh = static_cast<int>(r % Ho);
    const int b = static_cast<int>(r / Ho);
    // pad_lo = 1: Conv2d(stride 2, padding 1) (openaimodel.py Downsample); pad_lo = 0: the VAE's F.pad(x, (0,1,0,1)) + Conv2d(
    // stride 2, padding 0) (ldm/modules/diffusionmodules/model.py:80-84) -- zeros only on the right / bottom
    const int ih = 2 * oh + tap / 3 - pad_lo, iw = 2 * ow + tap % 3 - pad_lo;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) val = src[((static_cast<long long>(b) * H + ih) * W + iw) * vecs + v];
    dst[i] = val;
}

// ---- row softmax of fp32 logits -> fp16 probabilities (the VAE's single-head AttnBlock at d = 512, model.py:179-203: logits
// stay fp32 like the reference's bmm; one warp per row, two passes over a row that stays in L1/L2)
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ src, long long lds, __half* __restrict__ dst, long long ldd, long long rows,
                    int cols, float scale) {
    const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* x = src + row * lds;
    float m = -3.0e38f;
    for (int c = lane * 4; c < cols; c += 128) {
        const float4 v = *reinterpret_cast<const float4*>(x + c);
        m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const float ms = m * scale;
    float sum = 0.f;
    for (int c = lane * 4; c < cols; c += 128) {
        const float4 v = *reinterpret_cast<const float4*>(x + c);
        sum += __expf(v.x * scale - ms) + __expf(v.y * scale - ms) + __expf(v.z * scale - ms) + __expf(v.w * scale - ms);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.0f / sum;
    __half* y = dst + row * ldd;
    for (int c = lane * 4; c < cols; c += 128) {
        const float4 v = *reinterpret_cast<const float4*>(x + c);
        __half2 h0 = __floats2half2_rn(__expf(v.x * scale - ms) * inv, __expf(v.y * scale - ms) * inv);
        __half2 h1 = __floats2half2_rn(__expf(v.z * scale - ms) * inv, __expf(v.w * scale - ms) * inv);
        uint2 u;
        u.x = *reinterpret_cast<uint32_t*>(&h0);
        u.y = *reinterpret_cast<uint32_t*>(&h1);
        *reinterpret_cast<uint2*>(y + c) = u;
    }
}

// ---- DiagonalGaussianDistribution (ldm/modules/distributions/distributions.py:24-37) on fp32 NCHW moments [B, 2Z, HW]:
// mean = first Z channels, logvar = clamp(second Z channels, -30, 20); out = scale * (mean + exp(0.5 logvar) * noise), or
// scale * mean when noise == NULL (.mode()).
__global__ void gaussian_sample_kernel(const float* __restrict__ moments, const float* __restrict__ noise, float* __restrict__ out,
                                       int B, int Z, int HW, float scale) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(B) * Z * HW;
    if (i >= total) return;
    const long long b = i / (static_cast<long long>(Z) * HW), r = i % (static_cast<long long>(Z) * HW);
    const float mean = moments[b * 2 * Z * HW + r];
    float v = mean;
    if (noise) {
        const float lv = fminf(fmaxf(moments[b * 2 * Z * HW + static_cast<long long>(Z) * HW + r], -30.0f), 20.0f);
        v = __fadd_rn(mean, __fmul_rn(expf(0.5f * lv), noise[i]));
    }
    out[i] = __fmul_rn(scale, v);
}

// ---- weight preparation: fp32 [batch, R, C] -> fp16 [batch, C, R]  (Conv2d [Cout, Cin, 3*3] -> [Cout, 9, Cin];
// R == 1 is a plain cast), optional zero padding of C_out dim handled by the caller's buffer.
__global__ void cast_transpose_kernel(const float* __restrict__ src, __half* __restrict__ dst, long long batch, int R, int C) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = batch * R * C;
    if (i >= total) return;
    const int r = static_cast<int>(i % R);  // dst index: [b][c][r]
    const int c = static_cast<int>((i / R) % C);
    const long long b = i / (static_cast<long long>(R) * C);
    dst[i] = __float2half_rn(src[(b * R + r) * C + c]);
}

// ---- fp16 [batch, R, C] -> fp16 [batch, C, R]  (transposed kernel copies of weights for the dgrad GEMMs)
__global__ void transpose_f16_kernel(const __half* __restrict__ src, __half* __restrict__ dst, long long batch, int R, int C) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = batch * R * C;
    if (i >= total) return;
    const int r = static_cast<int>(i % R);
    const int c = static_cast<int>((i / R) % C);
    const long long b = i / (static_cast<long long>(R) * C);
    dst[i] = src[(b * R + r) * C + c];
}

// ---- tiled fp16 transpose with free outer strides: dst[z', j, i] = src[z, i, j], 64 x 64 tiles through shared memory,
// 128-byte row segments on both sides.  z' = Z-1-z when `flip` (the tap reversal of a convolution's data-gradient weight).
__device__ __forceinline__ __half2 load_pair(const __half* p) { return *reinterpret_cast<const __half2*>(p); }
__device__ __forceinline__ __half2 load_pair(const float* p) {
    const float2 v = *reinterpret_cast<const float2*>(p);
    return __floats2half2_rn(v.x, v.y);
}

template <typename S>
__global__ void __launch_bounds__(256)
tiled_transpose_f16_kernel(const S* __restrict__ src, __half* __restrict__ dst, int I, int J, long long s_i,
                           long long d_j, long long src_z, long long dst_z, int flip) {
    __shared__ __half tile[64][66];
    const int z = blockIdx.z, zo = flip ? static_cast<int>(gridDim.z) - 1 - z : z;
    src += z * src_z;
    dst += zo * dst_z;
    const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int i = i0 + ty + 8 * k, j = j0 + 2 * tx;
        __half2 v = __floats2half2_rn(0.f, 0.f);
        if (i < I && j < J) v = load_pair(src + i * s_i + j);
        tile[ty + 8 * k][2 * tx] = __low2half(v);
        tile[ty + 8 * k][2 * tx + 1] = __high2half(v);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int j = j0 + ty + 8 * k, i = i0 + 2 * tx;
        if (j < J && i < I)
            *reinterpret_cast<__half2*>(dst + j * d_j + i) = __halves2half2(tile[2 * tx][ty + 8 * k], tile[2 * tx + 1][ty + 8 * k]);
    }
}

static bool tiled_transpose_ok(const void* src, const void* dst, int I, int J, long long s_i, long long d_j, long long src_z,
                               long long dst_z, long long Z, int src_align = 3) {
    return !((I | J) & 1) && !((s_i | d_j | src_z | dst_z) & 1) && Z <= 65535 && (J + 63) / 64 > 0 && (I + 63) / 64 <= 65535 &&
           !(reinterpret_cast<uintptr_t>(src) & src_align) && !(reinterpret_cast<uintptr_t>(dst) & 3);
}

// fp32 -> fp16 plain cast, 8 elements per thread (the per-step fp16 copies of the trainable fp32 master weights)
__global__ void __launch_bounds__(256) cast_vec8_kernel(const float* __restrict__ src, __half* __restrict__ dst, long long vecs) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= vecs) return;
    const float4 a = reinterpret_cast<const float4*>(src)[2 * i], b = reinterpret_cast<const float4*>(src)[2 * i + 1];
    uint4 o;
    __half2* h = reinterpret_cast<__half2*>(&o);
    h[0] = __floats2half2_rn(a.x, a.y); h[1] = __floats2half2_rn(a.z, a.w);
    h[2] = __floats2half2_rn(b.x, b.y); h[3] = __floats2half2_rn(b.z, b.w);
    reinterpret_cast<uint4*>(dst)[i] = o;
}

// ---- DDIM update, one pass: CFG combine + pred_x0 + x_prev; explicit round-to-nearest ops in the reference's
// order (cldm/ddim_hacked.py:192,215,226-230) so that no FMA contraction changes the fp32 results.
// stats[b] += sum(x_prev^2) of image b (warp-reduced), a per-step scalar the host can read back.
__global__ void __launch_bounds__(256)
ddim_update_kernel(const float* __restrict__ x, const float* __restrict__ e_cond, const float* __restrict__ e_uncond,
                   const float* __restrict__ noise, float* __restrict__ x_prev, float* __restrict__ pred_x0,
                   float* __restrict__ stats, int per_image, int total, float cfg_scale, float sqrt_a_t,
                   float sqrt_a_prev, float dir_coef, float sigma_t, float temperature, float sqrt_one_minus_at) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float sq = 0.f;
    int img = 0;
    if (i < total) {
        float e = e_cond[i];
        if (e_uncond) {
            const float u = e_uncond[i];
            e = __fadd_rn(u, __fmul_rn(cfg_scale, __fsub_rn(e, u)));
        }
        const float p0 = __fdiv_rn(__fsub_rn(x[i], __fmul_rn(sqrt_one_minus_at, e)), sqrt_a_t);
        const float dir = __fmul_rn(dir_coef, e);
        float xp = __fadd_rn(__fmul_rn(sqrt_a_prev, p0), dir);
        xp = __fadd_rn(xp, noise ? __fmul_rn(__fmul_rn(sigma_t, noise[i]), temperature) : 0.f);
        x_prev[i] = xp;
        pred_x0[i] = p0;
        sq = xp * xp;
        img = i / per_image;
    }
    if (stats) {
        // per_image is a multiple of 32 for every latent shape on this path, so a warp never straddles two images
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
        if ((threadIdx.x & 31) == 0 && i < total) atomicAdd(&stats[img], sq);
    }
}

// q_sample / stochastic_encode (ldm/models/diffusion/ddpm.py:356-359, cldm/ddim_hacked.py:281-296): integer gather of the two
// per-timestep coefficients, then a*x0 + s*noise with separately rounded products (bit-identical to the reference's fp32
// tensor expression).
__global__ void __launch_bounds__(256)
q_sample_kernel(const float* __restrict__ x0, const float* __restrict__ noise, const long long* __restrict__ t,
                const float* __restrict__ tab_a, const float* __restrict__ tab_s, float* __restrict__ out, int per_image,
                int total) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const long long ti = t[i / per_image];
    out[i] = __fadd_rn(__fmul_rn(tab_a[ti], x0[i]), __fmul_rn(tab_s[ti], noise[i]));
}

// DDIM inversion step (cldm/ddim_hacked.py:253-267): optional CFG combine, then x_next = c1*x + c2*e, products rounded
// separately like the reference's tensor expression.
__global__ void __launch_bounds__(256)
ddim_encode_kernel(const float* __restrict__ x, const float* __restrict__ e_cond, const float* __restrict__ e_uncond,
                   float* __restrict__ x_next, int total, float cfg_scale, float c1, float c2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    float e = e_cond[i];
    if (e_uncond) {
        const float u = e_uncond[i];
        e = __fadd_rn(u, __fmul_rn(cfg_scale, __fsub_rn(e, u)));
    }
    x_next[i] = __fadd_rn(__fmul_rn(c1, x[i]), __fmul_rn(c2, e));
}

// DPM-Solver++ multistep step (ldm/models/diffusion/dpm_solver/dpm_solver.py, data prediction, solver_type 'dpm_solver'):
// CFG combine (:311-312), data prediction m = (x - sigma_s e) / alpha_s (:356-359) written to m_out, then the order-1
// (:490-497) or order-2 (:748-758) update.  Explicit round-to-nearest ops in the reference's order: no FMA contraction.
__global__ void __launch_bounds__(256)
dpm_multistep_kernel(const float* __restrict__ x, const float* __restrict__ e_cond, const float* __restrict__ e_uncond,
                     const float* __restrict__ m_prev, float* __restrict__ m_out, float* __restrict__ x_next, int total,
                     float cfg_scale, float sigma_s, float alpha_s, float c_x, float c_m, float c_d, float inv_r0) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    float e = e_cond[i];
    if (e_uncond) {
        const float u = e_uncond[i];
        e = __fadd_rn(u, __fmul_rn(cfg_scale, __fsub_rn(e, u)));
    }
    const float xi = x[i];
    const float m = __fdiv_rn(__fsub_rn(xi, __fmul_rn(sigma_s, e)), alpha_s);
    float xn = __fsub_rn(__fmul_rn(c_x, xi), __fmul_rn(c_m, m));
    if (m_prev) xn = __fsub_rn(xn, __fmul_rn(c_d, __fmul_rn(inv_r0, __fsub_rn(m, m_prev[i]))));
    m_out[i] = m;
    x_next[i] = xn;
}

// PLMS step (ldm/models/diffusion/plms.py:178-244): guided e_t (:184-192) written to e_out, e' of the given order
// (:226-240), then DDIM's pred_x0 / x_prev with e' (:205-223, sigma_t = 0).  Explicit round-to-nearest ops in torch's
// order; the divisions by 2 / 12 / 24 are products with the fp32 reciprocal, which is what torch does on a CUDA tensor
// divided by a Python number.
__device__ __forceinline__ float guided_eps(const float* __restrict__ e_cond, const float* __restrict__ e_uncond, int i,
                                            float cfg_scale) {
    const float e = e_cond[i];
    if (!e_uncond) return e;
    const float u = e_uncond[i];
    return __fadd_rn(u, __fmul_rn(cfg_scale, __fsub_rn(e, u)));
}

__global__ void __launch_bounds__(256)
plms_update_kernel(const float* __restrict__ x, const float* __restrict__ e_cond, const float* __restrict__ e_uncond,
                   const float* __restrict__ e_next_cond, const float* __restrict__ e_next_uncond,
                   const float* __restrict__ old1, const float* __restrict__ old2, const float* __restrict__ old3,
                   float* __restrict__ e_out, float* __restrict__ x_prev, float* __restrict__ pred_x0, int order, int total,
                   float cfg_scale, float sqrt_a_t, float sqrt_one_minus_at, float sqrt_a_prev, float dir_coef) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const float e = guided_eps(e_cond, e_uncond, i, cfg_scale);
    float ep;
    switch (order) {
    case 0:   // (e_t + e_t_next) / 2
        ep = __fmul_rn(__fadd_rn(e, guided_eps(e_next_cond, e_next_uncond, i, cfg_scale)), 0.5f);
        break;
    case 1:
        ep = e;
        break;
    case 2:   // (3 e - o1) / 2
        ep = __fmul_rn(__fsub_rn(__fmul_rn(3.f, e), old1[i]), 0.5f);
        break;
    case 3:   // (23 e - 16 o1 + 5 o2) / 12
        ep = __fmul_rn(__fadd_rn(__fsub_rn(__fmul_rn(23.f, e), __fmul_rn(16.f, old1[i])), __fmul_rn(5.f, old2[i])),
                       1.f / 12.f);
        break;
    default:  // (55 e - 59 o1 + 37 o2 - 9 o3) / 24
        ep = __fmul_rn(__fsub_rn(__fadd_rn(__fsub_rn(__fmul_rn(55.f, e), __fmul_rn(59.f, old1[i])),
                                           __fmul_rn(37.f, old2[i])),
                                 __fmul_rn(9.f, old3[i])),
                       1.f / 24.f);
    }
    const float p0 = __fdiv_rn(__fsub_rn(x[i], __fmul_rn(sqrt_one_minus_at, ep)), sqrt_a_t);
    e_out[i] = e;
    pred_x0[i] = p0;
    x_prev[i] = __fadd_rn(__fmul_rn(sqrt_a_prev, p0), __fmul_rn(dir_coef, ep));
}

static inline unsigned blocks_for(long long total, int threads) { return static_cast<unsigned>((total + threads - 1) / threads); }

}  // namespace ctrl

using namespace ctrl;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)
#define LAUNCH_OK() (cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA)

extern "C" int ctrlora_nchw_f32_to_nhwc_f16(const float* src, void* dst, int batch, int channels, int hw, int c_pad,
                                            void* stream) {
    if (!src || !dst || c_pad < channels) return CTRLORA_ERR_ARG;
    const long long total = static_cast<long long>(batch) * hw * c_pad;
    nchw_to_nhwc_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(src, reinterpret_cast<__half*>(dst), batch,
                                                                           channels, hw, c_pad);
    return LAUNCH_OK();
}

extern "C" int ctrlora_nhwc_to_nchw_f32(const void* src, int src_is_f32, long long ld, float* dst, int batch,
                                        int channels, int hw, void* stream) {
    if (!src || !dst) return CTRLORA_ERR_ARG;
    const long long total = static_cast<long long>(batch) * channels * hw;
    if (src_is_f32)
        nhwc_to_nchw_kernel<float><<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(
            reinterpret_cast<const float*>(src), ld, dst, batch, channels, hw);
    else
        nhwc_to_nchw_kernel<__half><<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(
            reinterpret_cast<const __half*>(src), ld, dst, batch, channels, hw);
    return LAUNCH_OK();
}

extern "C" int ctrlora_timestep_embedding(const long long* t, const float* freqs, float* out, int batch, int half,
                                          void* stream) {
    if (!t || !freqs || !out) return CTRLORA_ERR_ARG;
    timestep_embedding_kernel<<<blocks_for(static_cast<long long>(batch) * half, 128), 128, 0, STREAM(stream)>>>(
        t, freqs, out, batch, half);
    return LAUNCH_OK();
}

extern "C" int ctrlora_timestep_embedding_f32(const float* t, const float* freqs, float* out, int batch, int half,
                                              void* stream) {
    if (!t || !freqs || !out) return CTRLORA_ERR_ARG;
    timestep_embedding_f32_kernel<<<blocks_for(static_cast<long long>(batch) * half, 128), 128, 0, STREAM(stream)>>>(
        t, freqs, out, batch, half);
    return LAUNCH_OK();
}

// Same contract, for rows * K <= 40960 (e.g. 32 rows of 1280): the block stages act_in(x) ([rows][K] fp32) in shared memory once
// (the first version re-evaluated SiLU(emb) for every output feature: 206 M evaluations per UNet call, MUFU-bound), then every
// warp sweeps F output features AT A TIME against it: a lane owns 4 consecutive k per 128-wide chunk, so the activation reads
// are conflict-free 16-byte shared loads shared by the F features (round 1 read shared memory once per feature with a 2-way
// bank conflict and ran at ~0.4 TB/s of weight traffic), and the F weight rows are F independent 8-byte global loads per chunk.
// Features per block follow N so that small layers (time_embed: N = 1280) still fill the machine.
template <int F>
__global__ void __launch_bounds__(256)
small_linear_staged_kernel(const float* __restrict__ x, int ldx, const __half* __restrict__ w, const float* __restrict__ bias,
                           float* __restrict__ y, int ldy, int rows, int N, int K, int silu_in, int silu_out, int groups_per_warp) {
    extern __shared__ float sx[];  // [rows][K]
    {
        // staging: 16-byte loads, four in flight per thread (the scalar one-load-per-iteration loop of round 1 was a chain of
        // dependent global-load latencies: 20-40 us for 16 x 1280 activations, most of this kernel's time)
        const int k4 = K >> 2, total4 = rows * k4;
        const bool vec_ok = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
        int i = threadIdx.x;
        if (vec_ok) {
            for (; i + 3 * static_cast<int>(blockDim.x) < total4; i += 4 * blockDim.x) {
                float4 v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int j = i + u * blockDim.x, r = j / k4, c = j - r * k4;
                    v[u] = *reinterpret_cast<const float4*>(x + static_cast<long long>(r) * ldx + 4 * c);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    if (silu_in) { v[u].x = silu_f(v[u].x); v[u].y = silu_f(v[u].y); v[u].z = silu_f(v[u].z); v[u].w = silu_f(v[u].w); }
                    *reinterpret_cast<float4*>(sx + 4 * (i + u * blockDim.x)) = v[u];
                }
            }
            for (; i < total4; i += blockDim.x) {
                const int r = i / k4, c = i - r * k4;
                float4 v = *reinterpret_cast<const float4*>(x + static_cast<long long>(r) * ldx + 4 * c);
                if (silu_in) { v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w); }
                *reinterpret_cast<float4*>(sx + 4 * i) = v;
            }
        } else {
            for (int e = threadIdx.x; e < rows * K; e += blockDim.x) {
                const int r = e / K, k = e - r * K;
                const float v = x[static_cast<long long>(r) * ldx + k];
                sx[e] = silu_in ? silu_f(v) : v;
            }
        }
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = (K + 127) >> 7;
    for (int gidx = 0; gidx < groups_per_warp; ++gidx) {
        const int n0 = ((blockIdx.x * 8 + warp) * groups_per_warp + gidx) * F;
        if (n0 >= N) break;
        for (int r0 = 0; r0 < rows; r0 += 8) {
            float acc[F][8];
#pragma unroll
            for (int f = 0; f < F; ++f)
#pragma unroll
                for (int r = 0; r < 8; ++r) acc[f][r] = 0.f;
            for (int c = 0; c < chunks; ++c) {
                const int k = (c << 7) + lane * 4;
                const bool kin = k < K;  // K % 8 == 0 and k % 4 == 0: a 4-vector is either inside or outside
                uint2 uw[F];
#pragma unroll
                for (int f = 0; f < F; ++f)
                    uw[f] = (kin && n0 + f < N) ? __ldg(reinterpret_cast<const uint2*>(w + static_cast<long long>(n0 + f) * K + k))
                                                : make_uint2(0u, 0u);
                if (!kin) continue;
                float wv[F][4];
#pragma unroll
                for (int f = 0; f < F; ++f) {
                    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&uw[f].x));
                    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&uw[f].y));
                    wv[f][0] = a.x; wv[f][1] = a.y; wv[f][2] = b.x; wv[f][3] = b.y;
                }
#pragma unroll
                for (int r = 0; r < 8; ++r) {
                    if (r0 + r < rows) {
                        const float4 xv = *reinterpret_cast<const float4*>(sx + (r0 + r) * K + k);
#pragma unroll
                        for (int f = 0; f < F; ++f)
                            acc[f][r] += xv.x * wv[f][0] + xv.y * wv[f][1] + xv.z * wv[f][2] + xv.w * wv[f][3];
                    }
                }
            }
#pragma unroll
            for (int f = 0; f < F; ++f)
#pragma unroll
                for (int r = 0; r < 8; ++r)
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) acc[f][r] += __shfl_xor_sync(0xffffffffu, acc[f][r], o);
            if (lane == 0) {
#pragma unroll
                for (int f = 0; f < F; ++f) {
                    if (n0 + f < N) {
                        const float bv = bias ? bias[n0 + f] : 0.f;
#pragma unroll
                        for (int r = 0; r < 8; ++r) {
                            if (r0 + r < rows) {
                                float v = acc[f][r] + bv;
                                if (silu_out) v = silu_f(v);
                                y[static_cast<long long>(r0 + r) * ldy + n0 + f] = v;
                            }
                        }
                    }
                }
            }
        }
    }
}

extern "C" int ctrlora_small_linear(const float* x, int ldx, const void* w, const float* bias, float* y, int ldy,
                                    int rows, int n, int k, int silu_in, int silu_out, void* stream) {
    if (!x || !w || !y || k % 8 != 0 || ldx % 4 != 0) return CTRLORA_ERR_ARG;
    if (static_cast<long long>(rows) * k <= 40960 && k <= 2048) {
        const size_t sm = static_cast<size_t>(rows) * k * sizeof(float);
        static bool attr = false;
        if (!attr) {
            if (cudaFuncSetAttribute(small_linear_staged_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 40960 * 4) != cudaSuccess ||
                cudaFuncSetAttribute(small_linear_staged_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 40960 * 4) != cudaSuccess)
                return CTRLORA_ERR_CUDA;
            attr = true;
        }
        const __half* wp = reinterpret_cast<const __half*>(w);
        if (n >= 4096) {  // 4 features per warp pass, 2 passes: 64 features per block (e.g. 20 160 emb_layers rows -> 315 blocks)
            small_linear_staged_kernel<4><<<(n + 63) / 64, 256, sm, STREAM(stream)>>>(x, ldx, wp, bias, y, ldy, rows, n, k,
                                                                                     silu_in, silu_out, 2);
        } else {          // one feature per warp: 8 per block (time_embed N = 1280 -> 160 blocks)
            small_linear_staged_kernel<1><<<(n + 7) / 8, 256, sm, STREAM(stream)>>>(x, ldx, wp, bias, y, ldy, rows, n, k, silu_in,
                                                                                   silu_out, 1);
        }
        return LAUNCH_OK();
    }
    small_linear_kernel<<<(n + 7) / 8, 256, 0, STREAM(stream)>>>(x, ldx, reinterpret_cast<const __half*>(w), bias, y, ldy,
                                                                 rows, n, k, silu_in, silu_out);
    return LAUNCH_OK();
}

extern "C" int ctrlora_upsample2x_f16(const void* src, void* dst, int batch, int h, int w, int channels, void* stream) {
    if (!src || !dst || channels % 8 != 0) return CTRLORA_ERR_ARG;
    const int vecs = channels / 8;
    const long long total = static_cast<long long>(batch) * 4 * h * w * vecs;
    upsample2x_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(reinterpret_cast<const uint4*>(src),
                                                                        reinterpret_cast<uint4*>(dst), batch, h, w, vecs);
    return LAUNCH_OK();
}

extern "C" int ctrlora_im2col_s2_f16(const void* src, void* dst, int batch, int h, int w, int channels, void* stream) {
    if (!src || !dst || channels % 8 != 0 || (h & 1) || (w & 1)) return CTRLORA_ERR_ARG;
    const int vecs = channels / 8;
    const long long total = static_cast<long long>(batch) * (h / 2) * (w / 2) * 9 * vecs;
    im2col_s2_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(reinterpret_cast<const uint4*>(src),
                                                                       reinterpret_cast<uint4*>(dst), batch, h, w, vecs, 1);
    return LAUNCH_OK();
}

extern "C" int ctrlora_im2col_s2_pad_f16(const void* src, void* dst, int batch, int h, int w, int channels, int pad_lo,
                                         void* stream) {
    if (!src || !dst || channels % 8 != 0 || (h & 1) || (w & 1) || pad_lo < 0 || pad_lo > 1) return CTRLORA_ERR_ARG;
    const int vecs = channels / 8;
    const long long total = static_cast<long long>(batch) * (h / 2) * (w / 2) * 9 * vecs;
    im2col_s2_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(reinterpret_cast<const uint4*>(src),
                                                                       reinterpret_cast<uint4*>(dst), batch, h, w, vecs, pad_lo);
    return LAUNCH_OK();
}

extern "C" int ctrlora_softmax_rows_f32_to_f16(const float* src, long long lds, void* dst, long long ldd, long long rows,
                                               int cols, float scale, void* stream) {
    if (!src || !dst || cols % 4 != 0 || lds % 4 != 0 || ldd % 4 != 0) return CTRLORA_ERR_ARG;
    softmax_rows_kernel<<<blocks_for(rows, 8), 256, 0, STREAM(stream)>>>(src, lds, reinterpret_cast<__half*>(dst), ldd, rows,
                                                                       cols, scale);
    return LAUNCH_OK();
}

extern "C" int ctrlora_gaussian_sample(const float* moments, const float* noise, float* out, int batch, int z_channels, int hw,
                                       float scale, void* stream) {
    if (!moments || !out) return CTRLORA_ERR_ARG;
    const long long total = static_cast<long long>(batch) * z_channels * hw;
    gaussian_sample_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(moments, noise, out, batch, z_channels, hw, scale);
    return LAUNCH_OK();
}

extern "C" int ctrlora_cast_transpose_f32_to_f16(const float* src, void* dst, long long batch, int rows, int cols,
                                                 void* stream) {
    if (!src || !dst) return CTRLORA_ERR_ARG;
    const long long total = batch * rows * cols;
    if (total <= 0) return CTRLORA_OK;
    const bool aligned = !(reinterpret_cast<uintptr_t>(src) & 15) && !(reinterpret_cast<uintptr_t>(dst) & 15);
    if ((rows == 1 || cols == 1) && total % 8 == 0 && aligned) {
        cast_vec8_kernel<<<blocks_for(total / 8, 256), 256, 0, STREAM(stream)>>>(src, reinterpret_cast<__half*>(dst), total / 8);
        return LAUNCH_OK();
    }
    if (rows > 1 && cols > 1 &&
        tiled_transpose_ok(src, dst, rows, cols, cols, rows, (long long)rows * cols, (long long)rows * cols, batch, 7)) {
        tiled_transpose_f16_kernel<float><<<dim3((cols + 63) / 64, (rows + 63) / 64, (unsigned)batch), 256, 0, STREAM(stream)>>>(
            src, reinterpret_cast<__half*>(dst), rows, cols, cols, rows, (long long)rows * cols, (long long)rows * cols, 0);
        return LAUNCH_OK();
    }
    cast_transpose_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(src, reinterpret_cast<__half*>(dst), batch,
                                                                            rows, cols);
    return LAUNCH_OK();
}

// conv kernel weight [Cout, taps, Cin] -> data-gradient weight [Cin, taps reversed, Cout]  (dx = conv(dy, W_d), same padding)
extern "C" int ctrlora_conv_dgrad_weight_f16(const void* src, void* dst, int cout, int taps, int cin, void* stream) {
    if (!src || !dst || cout <= 0 || taps <= 0 || cin <= 0) return CTRLORA_ERR_ARG;
    if (!tiled_transpose_ok(src, dst, cout, cin, (long long)taps * cin, (long long)taps * cout, cin, cout, taps)) return CTRLORA_ERR_ARG;
    tiled_transpose_f16_kernel<__half><<<dim3((cin + 63) / 64, (cout + 63) / 64, taps), 256, 0, STREAM(stream)>>>(
        reinterpret_cast<const __half*>(src), reinterpret_cast<__half*>(dst), cout, cin, (long long)taps * cin,
        (long long)taps * cout, cin, cout, 1);
    return LAUNCH_OK();
}

extern "C" int ctrlora_transpose_f16(const void* src, void* dst, long long batch, int rows, int cols, void* stream) {
    if (src && dst && tiled_transpose_ok(src, dst, rows, cols, cols, rows, (long long)rows * cols, (long long)rows * cols, batch) &&
        batch > 0) {
        tiled_transpose_f16_kernel<__half><<<dim3((cols + 63) / 64, (rows + 63) / 64, (unsigned)batch), 256, 0, STREAM(stream)>>>(
            reinterpret_cast<const __half*>(src), reinterpret_cast<__half*>(dst), rows, cols, cols, rows,
            (long long)rows * cols, (long long)rows * cols, 0);
        return LAUNCH_OK();
    }
    if (!src || !dst) return CTRLORA_ERR_ARG;
    const long long total = batch * rows * cols;
    transpose_f16_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(reinterpret_cast<const __half*>(src),
                                                                           reinterpret_cast<__half*>(dst), batch, rows, cols);
    return LAUNCH_OK();
}

extern "C" int ctrlora_ddim_update(const float* x, const float* e_cond, const float* e_uncond, const float* noise,
                                   float* x_prev, float* pred_x0, float* stats, int batch, int per_image,
                                   float cfg_scale, float a_t, float a_prev, float sigma_t, float sqrt_one_minus_at,
                                   float temperature, void* stream) {
    if (!x || !e_cond || !x_prev || !pred_x0 || (stats && per_image % 32 != 0)) return CTRLORA_ERR_ARG;
    // per-step scalars exactly as the reference forms them from fp32 tensors (cldm/ddim_hacked.py:208-227):
    // a_t.sqrt(), a_prev.sqrt(), (1 - a_prev - sigma_t**2).sqrt(), sigma_t * temperature
    const float sqrt_a_t = sqrtf(a_t), sqrt_a_prev = sqrtf(a_prev);
    const float dir_coef = sqrtf((1.0f - a_prev) - sigma_t * sigma_t);
    const int total = batch * per_image;
    if (stats && cudaMemsetAsync(stats, 0, sizeof(float) * batch, STREAM(stream)) != cudaSuccess) return CTRLORA_ERR_CUDA;
    ddim_update_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(
        x, e_cond, e_uncond, noise, x_prev, pred_x0, stats, per_image, total, cfg_scale, sqrt_a_t, sqrt_a_prev, dir_coef,
        sigma_t, temperature, sqrt_one_minus_at);
    return LAUNCH_OK();
}

extern "C" int ctrlora_q_sample(const float* x0, const float* noise, const long long* t, const float* tab_a,
                                const float* tab_s, float* out, int batch, int per_image, void* stream) {
    if (!x0 || !noise || !t || !tab_a || !tab_s || !out) return CTRLORA_ERR_ARG;
    const int total = batch * per_image;
    q_sample_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(x0, noise, t, tab_a, tab_s, out, per_image, total);
    return LAUNCH_OK();
}

extern "C" int ctrlora_ddim_encode_update(const float* x, const float* e_cond, const float* e_uncond, float* x_next,
                                          int total, float cfg_scale, float c1, float c2, void* stream) {
    if (!x || !e_cond || !x_next) return CTRLORA_ERR_ARG;
    ddim_encode_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(x, e_cond, e_uncond, x_next, total, cfg_scale, c1, c2);
    return LAUNCH_OK();
}

extern "C" int ctrlora_dpm_multistep_update(const float* x, const float* e_cond, const float* e_uncond, const float* m_prev,
                                            float* m_out, float* x_next, int total, float cfg_scale, float sigma_s,
                                            float alpha_s, float c_x, float c_m, float c_d, float inv_r0, void* stream) {
    if (!x || !e_cond || !m_out || !x_next || total < 0) return CTRLORA_ERR_ARG;
    dpm_multistep_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(
        x, e_cond, e_uncond, m_prev, m_out, x_next, total, cfg_scale, sigma_s, alpha_s, c_x, c_m, c_d, inv_r0);
    return LAUNCH_OK();
}

extern "C" int ctrlora_plms_update(const float* x, const float* e_cond, const float* e_uncond, const float* e_next_cond,
                                   const float* e_next_uncond, const float* old1, const float* old2, const float* old3,
                                   float* e_out, float* x_prev, float* pred_x0, int order, int total, float cfg_scale,
                                   float sqrt_a_t, float sqrt_one_minus_at, float sqrt_a_prev, float dir_coef,
                                   void* stream) {
    if (!x || !e_cond || !e_out || !x_prev || !pred_x0 || total < 0 || order < 0 || order > 4) return CTRLORA_ERR_ARG;
    // exactly the inputs the order reads: a stray pointer means the caller's history bookkeeping is wrong
    const bool ok = order == 0 ? (e_next_cond && !old1 && !old2 && !old3 && !e_next_uncond == !e_uncond)
                               : (!e_next_cond && !e_next_uncond && !old1 == (order < 2) && !old2 == (order < 3) &&
                                  !old3 == (order < 4));
    if (!ok) return CTRLORA_ERR_ARG;
    plms_update_kernel<<<blocks_for(total, 256), 256, 0, STREAM(stream)>>>(
        x, e_cond, e_uncond, e_next_cond, e_next_uncond, old1, old2, old3, e_out, x_prev, pred_x0, order, total,
        cfg_scale, sqrt_a_t, sqrt_one_minus_at, sqrt_a_prev, dir_coef);
    return LAUNCH_OK();
}
