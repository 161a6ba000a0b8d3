// DPM_Solver (ldm/models/diffusion/dpm_solver/dpm_solver.py) on the device: the model-output conversion, dynamic
// thresholding, every first / singlestep / multistep update, and the adaptive solver's error norm.  Every scalar is
// formed on the host by ctrlora_b200.dpm_schedule (torch CPU fp32, the reference's operation order) and arrives as a
// float; the kernels apply the reference's elementwise expression trees with explicit round-to-nearest ops, so no FMA
// contraction changes a rounding and, given the same model values, the result is the reference's to the bit.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

struct DpmCoef {
    float v[CTRLORA_DPM_NCOEF];
};

// ---- model output: model_wrapper's noise_pred_fn / model_fn (:257-312) and data_prediction_fn (:352-359)
__device__ __forceinline__ float dpm_to_noise(float out, float x, int model_type, float alpha, float sigma) {
    switch (model_type) {
    case CTRLORA_DPM_MODEL_X_START:   // (x - alpha_t * out) / sigma_t                       :270
        return __fdiv_rn(__fsub_rn(x, __fmul_rn(alpha, out)), sigma);
    case CTRLORA_DPM_MODEL_V:         // alpha_t * out + sigma_t * x                          :274
        return __fadd_rn(__fmul_rn(alpha, out), __fmul_rn(sigma, x));
    default:                          // noise                                                :266
        return out;
    }
}

__global__ void __launch_bounds__(256)
dpm_model_output_kernel(const float* __restrict__ x, const float* __restrict__ out_cond,
                        const float* __restrict__ out_uncond, const float* __restrict__ grad, float* __restrict__ m_out,
                        long long total, int model_type, int predict_x0, DpmCoef k) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const float xi = x[i];
    const float scale = k.v[0], alpha_w = k.v[1], sigma_w = k.v[2];
    float e = dpm_to_noise(out_cond[i], xi, model_type, alpha_w, sigma_w);
    if (out_uncond) {   // noise_uncond + scale * (noise - noise_uncond)                          :312
        const float u = dpm_to_noise(out_uncond[i], xi, model_type, alpha_w, sigma_w);
        e = __fadd_rn(u, __fmul_rn(scale, __fsub_rn(e, u)));
    }
    if (grad) e = __fsub_rn(e, __fmul_rn(k.v[3], grad[i]));   // noise - (scale * sigma_t) * cond_grad   :303
    if (predict_x0) e = __fdiv_rn(__fsub_rn(xi, __fmul_rn(k.v[4], e)), k.v[5]);   // (x - sigma_t noise) / alpha_t  :359
    m_out[i] = e;
}

// ---- one update: x_t from x and up to three model values.  c and d carry the sign of their term (t - c*v and
// t + (-c)*v round identically), so each mode is one tree for both predict_x0 values and both solver types.
__global__ void __launch_bounds__(256)
dpm_update_kernel(const float* __restrict__ x, const float* __restrict__ m0, const float* __restrict__ m1,
                  const float* __restrict__ m2, float* __restrict__ out, long long total, int mode, DpmCoef k) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const float a = k.v[0], b = k.v[1], c = k.v[2], d = k.v[3];
    const float v0 = m0[i];
    float r = __fsub_rn(__fmul_rn(a, x[i]), __fmul_rn(b, v0));   // a x - b m0: every update's first two terms
    switch (mode) {
    case CTRLORA_DPM_UPDATE_DIFF:         // + c (m1 - m0): singlestep-2 final, singlestep-3 x_s2 and final
        r = __fadd_rn(r, __fmul_rn(c, __fsub_rn(m1[i], v0)));
        break;
    case CTRLORA_DPM_UPDATE_MULTISTEP2: { // D1_0 = k0 (m0 - m1); + c D1_0                               :751-777
        const float d10 = __fmul_rn(k.v[4], __fsub_rn(v0, m1[i]));
        r = __fadd_rn(r, __fmul_rn(c, d10));
        break;
    }
    case CTRLORA_DPM_UPDATE_MULTISTEP3: { // :807-824
        const float v1 = m1[i];
        const float d10 = __fmul_rn(k.v[4], __fsub_rn(v0, v1));
        const float d11 = __fmul_rn(k.v[5], __fsub_rn(v1, m2[i]));
        const float diff = __fsub_rn(d10, d11);
        const float d1 = __fadd_rn(d10, __fmul_rn(k.v[6], diff));
        const float d2 = __fmul_rn(k.v[7], diff);
        r = __fadd_rn(__fadd_rn(r, __fmul_rn(c, d1)), __fmul_rn(d, d2));
        break;
    }
    case CTRLORA_DPM_UPDATE_SINGLESTEP3_TAYLOR: {   // :668-677, :707-716 (k0 = 1/r1, k1 = 1/r2, k2 = r1, k3 = r2)
        const float d10 = __fmul_rn(k.v[4], __fsub_rn(m1[i], v0));
        const float d11 = __fmul_rn(k.v[5], __fsub_rn(m2[i], v0));
        const float d1 = __fdiv_rn(__fsub_rn(__fmul_rn(k.v[7], d10), __fmul_rn(k.v[6], d11)), k.v[8]);
        const float d2 = __fdiv_rn(__fmul_rn(2.f, __fsub_rn(d11, d10)), k.v[8]);
        r = __fadd_rn(__fadd_rn(r, __fmul_rn(c, d1)), __fmul_rn(d, d2));
        break;
    }
    default:                              // first order: a x - b m0                                   :494-509
        break;
    }
    out[i] = r;
}

// ---- dynamic thresholding (:360-364): s = max(quantile(|x0|, 0.995), max_val) per image, x0 = clamp(x0, -s, s) / s.
// torch.quantile sorts and joins the order statistics floor(rank) and ceil(rank), rank = fp32(0.995) * (n - 1) in fp32,
// with torch's lerp (a fused multiply-add on the CPU).  Here a 4-pass, 8-bit radix select on the bit patterns of |x0|
// (non-negative floats order like their bits) finds each order statistic; one block per image.
constexpr int kThreshThreads = 1024;

__device__ unsigned radix_select(const float* __restrict__ v, long long n, long long kth, unsigned* hist,
                                 unsigned* sh_prefix, long long* sh_k) {
    unsigned prefix = 0, mask = 0;
    long long k = kth;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int j = threadIdx.x; j < 256; j += blockDim.x) hist[j] = 0;
        __syncthreads();
        for (long long j = threadIdx.x; j < n; j += blockDim.x) {
            const unsigned u = __float_as_uint(v[j]) & 0x7fffffffu;
            if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 0xffu], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long acc = 0;
            int digit = 0;
            for (; digit < 255; ++digit) {
                if (acc + hist[digit] > k) break;
                acc += hist[digit];
            }
            *sh_prefix = prefix | (static_cast<unsigned>(digit) << shift);
            *sh_k = k - acc;
        }
        __syncthreads();
        prefix = *sh_prefix;
        k = *sh_k;
        mask |= 0xffu << shift;
        __syncthreads();
    }
    return prefix;
}

__global__ void __launch_bounds__(kThreshThreads)
dpm_threshold_kernel(float* __restrict__ x0, long long per_image, int use_smem, long long k_lo, long long k_hi,
                     float weight, float max_val, float* __restrict__ s_out) {
    extern __shared__ float sh_vals[];
    __shared__ unsigned hist[256];
    __shared__ unsigned sh_prefix;
    __shared__ long long sh_k;
    float* img = x0 + static_cast<long long>(blockIdx.x) * per_image;
    const float* src = img;
    if (use_smem) {
        for (long long j = threadIdx.x; j < per_image; j += blockDim.x) sh_vals[j] = img[j];
        __syncthreads();
        src = sh_vals;
    }
    const float lo = __uint_as_float(radix_select(src, per_image, k_lo, hist, &sh_prefix, &sh_k));
    const float hi = k_hi == k_lo ? lo : __uint_as_float(radix_select(src, per_image, k_hi, hist, &sh_prefix, &sh_k));
    const float diff = __fsub_rn(hi, lo);
    const float q = fabsf(weight) < 0.5f ? __fmaf_rn(weight, diff, lo) : __fmaf_rn(-diff, __fsub_rn(1.f, weight), hi);
    const float s = fmaxf(q, max_val);
    if (s_out && threadIdx.x == 0) s_out[blockIdx.x] = s;
    for (long long j = threadIdx.x; j < per_image; j += blockDim.x)
        img[j] = __fdiv_rn(fminf(fmaxf(src[j], -s), s), s);
}

// ---- adaptive solver error (:926-928): delta = max(atol, rtol * max(|x_lower|, |x_prev|)),
// E = max over images of sqrt(mean(((x_higher - x_lower) / delta)^2)).  One block, images in turn: the per-thread fp32
// partial sums are joined by a fixed tree, so E is deterministic but its rounding is not torch's cascade sum.
constexpr int kErrThreads = 1024;

__global__ void __launch_bounds__(kErrThreads)
dpm_adaptive_error_kernel(const float* __restrict__ x_lower, const float* __restrict__ x_prev,
                          const float* __restrict__ x_higher, float* __restrict__ err, int batch, long long per_image,
                          float atol, float rtol) {
    __shared__ float warp_sums[kErrThreads / 32];
    float e_max = 0.f;
    for (int b = 0; b < batch; ++b) {
        const long long base = static_cast<long long>(b) * per_image;
        float acc = 0.f;
        for (long long j = threadIdx.x; j < per_image; j += blockDim.x) {
            const float xl = x_lower[base + j];
            const float delta = fmaxf(atol, __fmul_rn(rtol, fmaxf(fabsf(xl), fabsf(x_prev[base + j]))));
            const float v = __fdiv_rn(__fsub_rn(x_higher[base + j], xl), delta);
            acc = __fadd_rn(acc, __fmul_rn(v, v));
        }
        for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
        if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x < 32) {
            float w = threadIdx.x < (blockDim.x >> 5) ? warp_sums[threadIdx.x] : 0.f;
            for (int o = 16; o > 0; o >>= 1) w = __fadd_rn(w, __shfl_xor_sync(0xffffffffu, w, o));
            if (threadIdx.x == 0) e_max = fmaxf(e_max, __fsqrt_rn(__fdiv_rn(w, static_cast<float>(per_image))));
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *err = e_max;
}

}  // namespace ctrl

using namespace ctrl;

static inline unsigned dpm_blocks(long long total) { return static_cast<unsigned>((total + 255) / 256); }
#define DPM_STREAM(s) reinterpret_cast<cudaStream_t>(s)
#define DPM_LAUNCH_OK() (cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA)

static DpmCoef dpm_coef(const float* coef) {
    DpmCoef k;
    for (int j = 0; j < CTRLORA_DPM_NCOEF; ++j) k.v[j] = coef[j];
    return k;
}

extern "C" int ctrlora_dpm_model_output(const float* x, const float* out_cond, const float* out_uncond,
                                        const float* grad, float* m_out, long long total, int model_type,
                                        int predict_x0, const float* coef, void* stream) {
    if (!x || !out_cond || !m_out || !coef || total < 0 || model_type < CTRLORA_DPM_MODEL_NOISE ||
        model_type > CTRLORA_DPM_MODEL_V)
        return CTRLORA_ERR_ARG;
    if (total == 0) return CTRLORA_OK;
    dpm_model_output_kernel<<<dpm_blocks(total), 256, 0, DPM_STREAM(stream)>>>(
        x, out_cond, out_uncond, grad, m_out, total, model_type, predict_x0, dpm_coef(coef));
    return DPM_LAUNCH_OK();
}

extern "C" int ctrlora_dpm_solver_update(const float* x, const float* m0, const float* m1, const float* m2, float* out,
                                         long long total, int mode, const float* coef, void* stream) {
    if (!x || !m0 || !out || !coef || total < 0) return CTRLORA_ERR_ARG;
    // exactly the model values the mode reads: a missing or stray one means the caller's bookkeeping is wrong
    const bool need1 = mode != CTRLORA_DPM_UPDATE_FIRST;
    const bool need2 = mode == CTRLORA_DPM_UPDATE_MULTISTEP3 || mode == CTRLORA_DPM_UPDATE_SINGLESTEP3_TAYLOR;
    if (mode < CTRLORA_DPM_UPDATE_FIRST || mode > CTRLORA_DPM_UPDATE_SINGLESTEP3_TAYLOR || !m1 != !need1 || !m2 != !need2)
        return CTRLORA_ERR_ARG;
    if (total == 0) return CTRLORA_OK;
    dpm_update_kernel<<<dpm_blocks(total), 256, 0, DPM_STREAM(stream)>>>(x, m0, m1, m2, out, total, mode, dpm_coef(coef));
    return DPM_LAUNCH_OK();
}

extern "C" int ctrlora_dpm_threshold(float* x0, float* s_out, int batch, long long per_image, long long k_lo,
                                     long long k_hi, float weight, float max_val, void* stream) {
    if (!x0 || batch < 0 || per_image <= 0 || k_lo < 0 || k_hi < k_lo || k_hi >= per_image) return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    // the image in shared memory when it fits (64 KB at a 64x64x4 latent); larger images are selected from global memory
    static const int smem_cap = [] {
        int dev = 0, cap = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        return cap - 4096;   // the histogram and the select's scalars
    }();
    const long long bytes = per_image * static_cast<long long>(sizeof(float));
    const int use_smem = bytes <= smem_cap;
    const size_t dyn = use_smem ? static_cast<size_t>(bytes) : 0;
    if (use_smem && cudaFuncSetAttribute(dpm_threshold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(dyn)) != cudaSuccess)
        return CTRLORA_ERR_CUDA;
    dpm_threshold_kernel<<<batch, kThreshThreads, dyn, DPM_STREAM(stream)>>>(x0, per_image, use_smem, k_lo, k_hi, weight,
                                                                            max_val, s_out);
    return DPM_LAUNCH_OK();
}

extern "C" int ctrlora_dpm_adaptive_error(const float* x_lower, const float* x_prev, const float* x_higher, float* err,
                                          int batch, long long per_image, float atol, float rtol, void* stream) {
    if (!x_lower || !x_prev || !x_higher || !err || batch <= 0 || per_image <= 0) return CTRLORA_ERR_ARG;
    dpm_adaptive_error_kernel<<<1, kErrThreads, 0, DPM_STREAM(stream)>>>(x_lower, x_prev, x_higher, err, batch, per_image,
                                                                        atol, rtol);
    return DPM_LAUNCH_OK();
}
