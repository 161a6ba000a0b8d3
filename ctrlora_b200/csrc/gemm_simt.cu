// CUDA-core twin of the wgmma implicit GEMM (same argument block, same epilogue semantics).  It exists to bisect
// tensor-core / TMA descriptor bugs on the GPU box; the product path never calls it.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

__global__ void gemm_simt_kernel(ctrlora_gemm_args a, int M, int rows_per_img) {
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= static_cast<long long>(M) * a.n) return;
    const int n = static_cast<int>(idx % a.n);
    const long long m = idx / a.n;
    const int w = static_cast<int>(m % a.a_w);
    const int h = static_cast<int>((m / a.a_w) % a.a_h);
    const int b = static_cast<int>(m / (static_cast<long long>(a.a_w) * a.a_h));
    const __half* A = reinterpret_cast<const __half*>(a.a);
    const __half* Wt = reinterpret_cast<const __half*>(a.w);
    const int taps = a.kh * a.kw;
    auto dot = [&](int wrow) {
        float acc = 0.f;
        for (int t = 0; t < taps; ++t) {
            const int hh = h + t / a.kw - a.pad, ww = w + t % a.kw - a.pad;
            if (hh < 0 || hh >= a.a_h || ww < 0 || ww >= a.a_w) continue;
            const __half* ap = A + ((static_cast<long long>(b) * a.a_h + hh) * a.a_w + ww) * a.a_ld;
            const __half* wp = Wt + (static_cast<long long>(wrow) * taps + t) * a.a_c;
            for (int c = 0; c < a.a_c; ++c) acc += __half2float(ap[c]) * __half2float(wp[c]);
        }
        return acc;
    };
    float v = dot(n);
    if (a.a2) {
        const __half* ap = reinterpret_cast<const __half*>(a.a2) + m * a.a2_ld;
        const __half* wp = reinterpret_cast<const __half*>(a.w2) + static_cast<long long>(n) * a.a2_c;
        for (int c = 0; c < a.a2_c; ++c) v += __half2float(ap[c]) * __half2float(wp[c]);
    }
    if (a.bias) v += a.bias[n];
    if (a.geglu) {
        float g = dot(a.n + n);
        if (a.bias) g += a.bias[a.n + n];
        v *= gelu_erf_f(g);
    }
    const int img = static_cast<int>(m / rows_per_img), tok = static_cast<int>(m % rows_per_img);
    if (a.rowbias) v += a.rowbias[static_cast<long long>(img) * (a.rowbias_ld > 0 ? a.rowbias_ld : a.n) + n];
    v *= a.out_scale;
    if (a.residual) v += a.residual_f32 ? reinterpret_cast<const float*>(a.residual)[m * a.ldr + n]
                                         : __half2float(reinterpret_cast<const __half*>(a.residual)[m * a.ldr + n]);
    int seg = 0, nloc = n;
    if (a.seg_width > 0) { seg = n / a.seg_width; nloc = n % a.seg_width; }
    if (a.transposed[seg]) {
        reinterpret_cast<__half*>(a.out[seg])[(static_cast<long long>(img) * a.seg_width + nloc) * a.tok_pad + tok] =
            __float2half_rn(v);
        if (a.dup_out) reinterpret_cast<__half*>(a.dup_out)[m * a.dup_ld + nloc] = __float2half_rn(v);
    } else if (a.out_f32) {
        reinterpret_cast<float*>(a.out[seg])[m * a.ldc + nloc] = v;
    } else {
        reinterpret_cast<__half*>(a.out[seg])[m * a.ldc + nloc] = __float2half_rn(v);
    }
}

}  // namespace ctrl

extern "C" int ctrlora_gemm_f16_simt(const ctrlora_gemm_args* a, void* stream_) {
    if (!a || !a->a || !a->w || !a->out[0]) return CTRLORA_ERR_ARG;
    if (a->group_b > 0) return CTRLORA_ERR_UNSUPPORTED;
    const long long M = static_cast<long long>(a->a_b) * a->a_h * a->a_w;
    const long long total = M * a->n;
    const int rows = a->rows_per_img > 0 ? a->rows_per_img : a->a_h * a->a_w;
    const int threads = 256;
    const long long blocks = (total + threads - 1) / threads;
    ctrl::gemm_simt_kernel<<<static_cast<unsigned>(blocks), threads, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
        *a, static_cast<int>(M), rows);
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}
