// Training-only elementwise / reduction kernels (HBM-bound): GEGLU forward+backward on stored pre-activations, column
// sums (bias gradients), nearest-upsample and stride-2-gather adjoints, the eps-MSE loss with its gradient, fused AdamW.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

__device__ __forceinline__ void ld8(const __half* p, float* v) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { float2 f = __half22float2(h[e]); v[2 * e] = f.x; v[2 * e + 1] = f.y; }
}
__device__ __forceinline__ void st8(__half* p, const float* v) {
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
    *reinterpret_cast<uint4*>(p) = u;
}

// GEGLU on the stored projection h = [value | gate] ([M, 2N]): out = value * gelu(gate)   (attention.py:49-56)
__global__ void geglu_fwd_kernel(const __half* __restrict__ h, __half* __restrict__ out, long long M, int N) {
    pdl_launch_dependents();
    pdl_wait();
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // one 8-vector
    const int nv = N >> 3;
    if (i >= M * nv) return;
    const long long row = i / nv;
    const int c = static_cast<int>(i % nv) * 8;
    float v[8], g[8];
    ld8(h + row * 2 * N + c, v);
    ld8(h + row * 2 * N + N + c, g);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] *= gelu_erf_f(g[e]);
    st8(out + row * N + c, v);
}

// dh = [dout * gelu(gate) | dout * value * gelu'(gate)],  gelu'(g) = Phi(g) + g * phi(g)
__global__ void geglu_bwd_kernel(const __half* __restrict__ h, const __half* __restrict__ dout, __half* __restrict__ dh,
                                 long long M, int N) {
    pdl_launch_dependents();
    pdl_wait();
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int nv = N >> 3;
    if (i >= M * nv) return;
    const long long row = i / nv;
    const int c = static_cast<int>(i % nv) * 8;
    float v[8], g[8], d[8], dv[8], dg[8];
    ld8(h + row * 2 * N + c, v);
    ld8(h + row * 2 * N + N + c, g);
    ld8(dout + row * N + c, d);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const float cdf = 0.5f * (1.0f + erff(g[e] * 0.70710678118654752f));
        const float pdf = 0.3989422804014327f * __expf(-0.5f * g[e] * g[e]);
        dv[e] = d[e] * g[e] * cdf;
        dg[e] = d[e] * v[e] * (cdf + g[e] * pdf);
    }
    st8(dh + row * 2 * N + c, dv);
    st8(dh + row * 2 * N + N + c, dg);
}

// out[c] (+)= scale * sum_rows x[row, c]     (bias gradients); fp16 or fp32 input, fp32 atomics once per block per column
template <typename T>
__global__ void colsum_kernel(const T* __restrict__ x, long long ld, long long rows, int cols, float scale, float* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    const long long r0 = static_cast<long long>(blockIdx.y) * ((rows + gridDim.y - 1) / gridDim.y);
    const long long r1 = min(rows, r0 + (rows + gridDim.y - 1) / gridDim.y);
    float acc = 0.f;
    for (long long r = r0; r < r1; ++r) acc += static_cast<float>(x[r * ld + c]);
    atomicAdd(&out[c], scale * acc);
}

// fp16 rows of 8-column vectors: block (32 vectors, 8 row lanes), 16-byte loads four rows deep, row lanes combined in
// shared memory, one atomic per column per block
__global__ void __launch_bounds__(256)
colsum_vec_kernel(const __half* __restrict__ x, long long ld, long long rows, int vecs, float scale, float* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float red[8][32][9];
    const int vx = threadIdx.x & 31, ry = threadIdx.x >> 5;
    const int v = blockIdx.x * 32 + vx;
    const long long chunk = (rows + gridDim.y - 1) / gridDim.y;
    const long long r0 = static_cast<long long>(blockIdx.y) * chunk, r1 = min(rows, r0 + chunk);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (v < vecs) {
        const __half* base = x + 8 * v;
        long long r = r0 + ry;
        for (; r + 24 < r1; r += 32) {
            uint4 q[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) q[u] = *reinterpret_cast<const uint4*>(base + (r + 8 * u) * ld);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const __half2* h = reinterpret_cast<const __half2*>(&q[u]);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(h[j]);
                    acc[2 * j] += f.x;
                    acc[2 * j + 1] += f.y;
                }
            }
        }
        for (; r < r1; r += 8) {
            const uint4 q = *reinterpret_cast<const uint4*>(base + r * ld);
            const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(h[j]);
                acc[2 * j] += f.x;
                acc[2 * j + 1] += f.y;
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) red[ry][vx][j] = acc[j];
    __syncthreads();
    // 256 threads = 32 vectors x 8 columns
    const int col = threadIdx.x & 7, vec = threadIdx.x >> 3;
    const int vo = blockIdx.x * 32 + vec;
    if (vo >= vecs) return;
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][vec][col];
    atomicAdd(&out[8 * vo + col], scale * t);
}

// per-image column sums: out[img, c] = sum over the image's rows (time-embedding gradient of a ResBlock conv)
__global__ void rowgroup_colsum_kernel(const __half* __restrict__ x, long long ld, int rows_per_img, int cols, float* __restrict__ out,
                                       long long ldo) {
    pdl_launch_dependents();
    pdl_wait();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int img = blockIdx.y;
    if (c >= cols) return;
    const int chunk = (rows_per_img + gridDim.z - 1) / gridDim.z;
    const int r0 = blockIdx.z * chunk, r1 = min(rows_per_img, r0 + chunk);
    float acc = 0.f;
    for (int r = r0; r < r1; ++r) acc += __half2float(x[(static_cast<long long>(img) * rows_per_img + r) * ld + c]);
    atomicAdd(&out[img * ldo + c], acc);
}

// adjoint of nearest-2x upsample: din[b,h,w,:] = sum of the 2x2 output block
__global__ void upsample2x_bwd_kernel(const __half* __restrict__ dout, __half* __restrict__ din, int B, int H, int W, int vecs) {
    pdl_launch_dependents();
    pdl_wait();
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<long long>(B) * H * W * vecs) return;
    const int v = static_cast<int>(i % vecs);
    long long pix = i / vecs;
    const int w = static_cast<int>(pix % W);
    pix /= W;
    const int h = static_cast<int>(pix % H);
    const int b = static_cast<int>(pix / H);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            float t[8];
            ld8(dout + (((static_cast<long long>(b) * 2 * H + 2 * h + dy) * 2 * W + 2 * w + dx) * vecs + v) * 8, t);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] += t[e];
        }
    st8(din + i * 8, acc);
}

// adjoint of the stride-2 3x3 pad-1 gather: dx[b,ih,iw,:] = sum over (oh, ow, tap) that read it of dcol[b,oh,ow,tap,:]
__global__ void im2col_s2_bwd_kernel(const __half* __restrict__ dcol, __half* __restrict__ dx, int B, int H, int W, int vecs) {
    pdl_launch_dependents();
    pdl_wait();
    const int Ho = H / 2, Wo = W / 2;
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<long long>(B) * H * W * vecs) return;
    const int v = static_cast<int>(i % vecs);
    long long pix = i / vecs;
    const int iw = static_cast<int>(pix % W);
    pix /= W;
    const int ih = static_cast<int>(pix % H);
    const int b = static_cast<int>(pix / H);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int kh = 0; kh < 3; ++kh) {
        const int t = ih + 1 - kh;  // 2*oh = ih + 1 - kh
        if (t < 0 || (t & 1)) continue;
        const int oh = t >> 1;
        if (oh >= Ho) continue;
        for (int kw = 0; kw < 3; ++kw) {
            const int u = iw + 1 - kw;
            if (u < 0 || (u & 1)) continue;
            const int ow = u >> 1;
            if (ow >= Wo) continue;
            float tv[8];
            ld8(dcol + ((((static_cast<long long>(b) * Ho + oh) * Wo + ow) * 9 + kh * 3 + kw) * vecs + v) * 8, tv);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] += tv[e];
        }
    }
    st8(dx + i * 8, acc);
}

// loss = mean((eps - noise)^2) over everything (== mean over images of per-image means, ddpm.py:902-918 with logvar 0);
// grad (pixel-major fp16 [B, HW, c_pad]) = 2 (eps - noise) / numel * grad_scale.  eps, noise: fp32 NCHW.
__global__ void mse_loss_grad_kernel(const float* __restrict__ eps, const float* __restrict__ noise, float* __restrict__ loss,
                                     __half* __restrict__ grad, int B, int C, int HW, int c_pad, float grad_scale) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = static_cast<long long>(B) * C * HW;
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    float sq = 0.f;
    if (i < total) {
        const int p = static_cast<int>(i % HW);
        const int c = static_cast<int>((i / HW) % C);
        const int b = static_cast<int>(i / (static_cast<long long>(HW) * C));
        const float d = eps[i] - noise[i];
        sq = d * d;
        grad[(static_cast<long long>(b) * HW + p) * c_pad + c] = __float2half_rn(2.0f * d / static_cast<float>(total) * grad_scale);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if ((threadIdx.x & 31) == 0 && sq != 0.f) atomicAdd(loss, sq / static_cast<float>(total));
}

// torch.optim.AdamW semantics (decoupled weight decay, bias correction), fp32 master params, one flat buffer.
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             long long n, float lr, float beta1, float beta2, float eps, float wd, float bc1, float bc2,
                             float grad_scale, const int* __restrict__ skip_flag, const float* __restrict__ bc_dev) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (skip_flag && *skip_flag) return;  // a non-finite gradient was seen this step (loss-scale overflow): no update
    if (bc_dev) { bc1 = bc_dev[0]; bc2 = bc_dev[1]; }  // bias corrections of the DEVICE-side step counter (adamw_begin)
    const float gi = g[i] * grad_scale;
    float pi = p[i] * (1.0f - lr * wd);
    const float mi = beta1 * m[i] + (1.0f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.0f - beta2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / sqrtf(bc2) + eps;
    pi -= (lr / bc1) * (mi / denom);
    p[i] = pi;
}

// flag |= any(!isfinite(x)): the overflow check of static/dynamic loss scaling (fp16 activation gradients)
__global__ void nonfinite_flag_kernel(const float* __restrict__ x, long long n, int* __restrict__ flag) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
    bool bad = false;
    for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
        if (i + 4 <= n) {
            const float4 v = *reinterpret_cast<const float4*>(x + i);
            bad |= !(isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && isfinite(v.w));
        } else {
            for (long long j = i; j < n; ++j) bad |= !isfinite(x[j]);
        }
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1);
}

// out = sum_i w[i] * src[i]  (fp16 tensors of n elements, fp32 accumulate): the multi-LoRA control sum
// (cldm/cldm_ctrlora_inference.py:172-176) in one pass
struct WeightedSumArgs {
    const __half* src[8];
    float w[8];
    int count;
};
__global__ void weighted_sum_kernel(const __grid_constant__ WeightedSumArgs a, __half* __restrict__ out, long long nvec) {
    pdl_launch_dependents();
    pdl_wait();
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= nvec) return;
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = 0; s < a.count; ++s) {
        float t[8];
        ld8(a.src[s] + i * 8, t);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] += a.w[s] * t[e];
    }
    st8(out + i * 8, acc);
}

// stride-1 3x3 pad-1 gather: col[b, h, w, tap, c] = x[b, h + kh - 1, w + kw - 1, c] (0 outside): the token-major operand
// of the dense conv weight gradient dW[Cout, tap, Cin] = dY^T col (pretraining: every ControlNet conv is trainable)
__global__ void im2col_3x3_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int B, int H, int W, int vecs) {
    pdl_launch_dependents();
    pdl_wait();
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(B) * H * W * 9 * vecs;
    if (i >= total) return;
    const int v = static_cast<int>(i % vecs);
    long long r = i / vecs;
    const int tap = static_cast<int>(r % 9);
    r /= 9;
    const int w = static_cast<int>(r % W);
    r /= W;
    const int h = static_cast<int>(r % H);
    const int b = static_cast<int>(r / H);
    const int ih = h + tap / 3 - 1, iw = w + tap % 3 - 1;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) val = src[((static_cast<long long>(b) * H + ih) * W + iw) * vecs + v];
    dst[i] = val;
}

// out[n, k] (+)= alpha * sum_b dy[b, n] * x[b, k]   (fp32, b = batch rows <= 64): weight gradients of the time-embedding
// MLP / emb_layers linears, where the "token" dimension is just the batch
__global__ void __launch_bounds__(256)
outer_accum_kernel(const float* __restrict__ dy, int lddy, const float* __restrict__ x, int ldx, float* __restrict__ out,
                   long long ldo, int rows, int N, int K, float alpha, float beta, int silu_x) {
    pdl_launch_dependents();
    pdl_wait();
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = blockIdx.y;
    if (k >= K) return;
    float acc = 0.f;
    for (int b = 0; b < rows; ++b) {
        float xv = x[b * ldx + k];
        if (silu_x) xv = xv / (1.0f + __expf(-xv));
        acc += dy[b * lddy + n] * xv;
    }
    float* o = out + n * ldo + k;
    *o = beta * (*o) + alpha * acc;
}

// out = d * silu'(x)  (fp32)
__global__ void silu_bwd_kernel(const float* __restrict__ d, const float* __restrict__ x, float* __restrict__ out, long long n) {
    pdl_launch_dependents();
    pdl_wait();
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float z = x[i];
    const float s = 1.0f / (1.0f + __expf(-z));
    out[i] = d[i] * s * (1.0f + z * (1.0f - s));
}

// dst[r, c] (+)= src[r, c] over [rows, cols] with row strides (fp32): sub-block extraction of padded gradient tiles
__global__ void copy2d_kernel(const float* __restrict__ src, long long lds, float* __restrict__ dst, long long ldd, long long rows,
                              int cols, int accumulate) {
    pdl_launch_dependents();
    pdl_wait();
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const long long r = i / cols;
    const int c = static_cast<int>(i % cols);
    const float v = src[r * lds + c];
    float* d = dst + r * ldd + c;
    *d = accumulate ? *d + v : v;
}

// fp32 [rows, cols] with arbitrary row stride -> fp16 dense (weight copies of parameters stored in kernel layout)
__global__ void cast_rows_kernel(const float* __restrict__ src, long long lds, __half* __restrict__ dst, long long rows, int cols) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    dst[i] = __float2half_rn(src[(i / cols) * lds + (i % cols)]);
}

// One thread, in front of an AdamW step: advances the device-side step counter unless the step is being skipped (then the
// skipped-steps counter), and leaves the two bias corrections 1 - beta^step in bc[0..1].  With the counter on the device the
// host never has to read the overflow flag before launching the next step (it polls `skipped` now and then to lower the loss
// scale), and torch's `step` semantics -- a skipped step does not count -- hold exactly.
__global__ void adamw_begin_kernel(int* __restrict__ step_counter, const int* __restrict__ skip_flag, float beta1, float beta2,
                                   float* __restrict__ bc, int* __restrict__ skipped) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (skip_flag && *skip_flag) {
        if (skipped) ++*skipped;
        return;
    }
    const int st = ++*step_counter;
    bc[0] = 1.0f - powf(beta1, static_cast<float>(st));
    bc[1] = 1.0f - powf(beta2, static_cast<float>(st));
}

static inline unsigned nblk(long long total, int threads) { return static_cast<unsigned>((total + threads - 1) / threads); }

}  // namespace ctrl

using namespace ctrl;
#define STREAM(s) reinterpret_cast<cudaStream_t>(s)
#define LAUNCH_OK() (cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA)

extern "C" int ctrlora_geglu_fwd_f16(const void* h, void* out, long long rows, int n, void* stream) {
    if (!h || !out || n % 8) return CTRLORA_ERR_ARG;
    launch_pdl(geglu_fwd_kernel, dim3(nblk(rows * (n / 8), 256)), dim3(256), (size_t)0, STREAM(stream),
               reinterpret_cast<const __half*>(h), reinterpret_cast<__half*>(out), rows, n);
    return LAUNCH_OK();
}

extern "C" int ctrlora_geglu_bwd_f16(const void* h, const void* dout, void* dh, long long rows, int n, void* stream) {
    if (!h || !dout || !dh || n % 8) return CTRLORA_ERR_ARG;
    launch_pdl(geglu_bwd_kernel, dim3(nblk(rows * (n / 8), 256)), dim3(256), (size_t)0, STREAM(stream),
               reinterpret_cast<const __half*>(h), reinterpret_cast<const __half*>(dout), reinterpret_cast<__half*>(dh), rows, n);
    return LAUNCH_OK();
}

extern "C" int ctrlora_colsum(const void* x, int x_is_f32, long long ld, long long rows, int cols, float scale, float* out,
                              void* stream) {
    if (!x || !out) return CTRLORA_ERR_ARG;
    if (!x_is_f32 && cols % 8 == 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
        const int vecs = cols / 8, xb = (vecs + 31) / 32;
        long long ys = (2 * 132 + xb - 1) / xb;  // about two blocks per SM of an H100
        if (ys > rows / 64) ys = rows / 64;
        if (ys < 1) ys = 1;
        launch_pdl(colsum_vec_kernel, dim3(xb, (unsigned)ys), dim3(256), (size_t)0, STREAM(stream),
                   reinterpret_cast<const __half*>(x), ld, rows, vecs, scale, out);
        return LAUNCH_OK();
    }
    int ysplit = static_cast<int>(rows / 256);
    if (ysplit < 1) ysplit = 1;
    if (ysplit > 64) ysplit = 64;
    dim3 grid((cols + 127) / 128, ysplit);
    if (x_is_f32)
        launch_pdl(colsum_kernel<float>, grid, dim3(128), (size_t)0, STREAM(stream), reinterpret_cast<const float*>(x), ld, rows, cols, scale, out);
    else
        launch_pdl(colsum_kernel<__half>, grid, dim3(128), (size_t)0, STREAM(stream), reinterpret_cast<const __half*>(x), ld, rows, cols, scale, out);
    return LAUNCH_OK();
}

extern "C" int ctrlora_image_colsum_f16(const void* x, long long ld, int images, int rows_per_img, int cols, float* out,
                                        long long ldo, void* stream) {
    if (!x || !out) return CTRLORA_ERR_ARG;
    int z = rows_per_img / 128;
    if (z < 1) z = 1;
    if (z > 32) z = 32;
    dim3 grid((cols + 127) / 128, images, z);
    launch_pdl(rowgroup_colsum_kernel, grid, dim3(128), (size_t)0, STREAM(stream), reinterpret_cast<const __half*>(x), ld,
               rows_per_img, cols, out, ldo);
    return LAUNCH_OK();
}

extern "C" int ctrlora_upsample2x_bwd_f16(const void* dout, void* din, int batch, int h, int w, int channels, void* stream) {
    if (!dout || !din || channels % 8) return CTRLORA_ERR_ARG;
    const int vecs = channels / 8;
    launch_pdl(upsample2x_bwd_kernel, dim3(nblk(static_cast<long long>(batch) * h * w * vecs, 256)), dim3(256), (size_t)0,
               STREAM(stream), reinterpret_cast<const __half*>(dout), reinterpret_cast<__half*>(din), batch, h, w, vecs);
    return LAUNCH_OK();
}

extern "C" int ctrlora_im2col_s2_bwd_f16(const void* dcol, void* dx, int batch, int h, int w, int channels, void* stream) {
    if (!dcol || !dx || channels % 8 || (h & 1) || (w & 1)) return CTRLORA_ERR_ARG;
    const int vecs = channels / 8;
    launch_pdl(im2col_s2_bwd_kernel, dim3(nblk(static_cast<long long>(batch) * h * w * vecs, 256)), dim3(256), (size_t)0,
               STREAM(stream), reinterpret_cast<const __half*>(dcol), reinterpret_cast<__half*>(dx), batch, h, w, vecs);
    return LAUNCH_OK();
}

extern "C" int ctrlora_mse_loss_grad(const float* eps, const float* noise, float* loss, void* grad, int batch, int channels,
                                     int hw, int c_pad, float grad_scale, void* stream) {
    if (!eps || !noise || !loss || !grad || c_pad < channels) return CTRLORA_ERR_ARG;
    if (cudaMemsetAsync(loss, 0, sizeof(float), STREAM(stream)) != cudaSuccess) return CTRLORA_ERR_CUDA;
    if (cudaMemsetAsync(grad, 0, static_cast<size_t>(batch) * hw * c_pad * 2, STREAM(stream)) != cudaSuccess) return CTRLORA_ERR_CUDA;
    const long long total = static_cast<long long>(batch) * channels * hw;
    mse_loss_grad_kernel<<<nblk(total, 256), 256, 0, STREAM(stream)>>>(eps, noise, loss, reinterpret_cast<__half*>(grad), batch,
                                                                       channels, hw, c_pad, grad_scale);
    return LAUNCH_OK();
}

extern "C" int ctrlora_adamw_f32(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr,
                                 float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                                 const int* skip_flag, const float* bc_dev, void* stream) {
    if (!params || !grads || !exp_avg || !exp_avg_sq || (step < 1 && !bc_dev)) return CTRLORA_ERR_ARG;
    const float bc1 = 1.0f - powf(beta1, static_cast<float>(step)), bc2 = 1.0f - powf(beta2, static_cast<float>(step));
    adamw_kernel<<<nblk(n, 256), 256, 0, STREAM(stream)>>>(params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps,
                                                           weight_decay, bc1, bc2, grad_scale, skip_flag, bc_dev);
    return LAUNCH_OK();
}

extern "C" int ctrlora_adamw_begin(int* step_counter, const int* skip_flag, float beta1, float beta2, float* bc, int* skipped,
                                   void* stream) {
    if (!step_counter || !bc) return CTRLORA_ERR_ARG;
    adamw_begin_kernel<<<1, 32, 0, STREAM(stream)>>>(step_counter, skip_flag, beta1, beta2, bc, skipped);
    return LAUNCH_OK();
}

extern "C" int ctrlora_nonfinite_flag_f32(const float* x, long long n, int* flag, void* stream) {
    if (!x || !flag || (reinterpret_cast<uintptr_t>(x) & 15)) return CTRLORA_ERR_ARG;
    long long blocks = (n / 4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) blocks = 1;
    nonfinite_flag_kernel<<<static_cast<unsigned>(blocks), 256, 0, STREAM(stream)>>>(x, n, flag);
    return LAUNCH_OK();
}

extern "C" int ctrlora_weighted_sum_f16(const void* const* srcs, const float* weights, int count, void* out, long long n,
                                        void* stream) {
    if (!srcs || !weights || !out || count < 1 || count > 8 || n % 8) return CTRLORA_ERR_ARG;
    WeightedSumArgs a;
    a.count = count;
    for (int i = 0; i < count; ++i) {
        if (!srcs[i] || (reinterpret_cast<uintptr_t>(srcs[i]) & 15)) return CTRLORA_ERR_ARG;
        a.src[i] = reinterpret_cast<const __half*>(srcs[i]);
        a.w[i] = weights[i];
    }
    launch_pdl(weighted_sum_kernel, dim3(nblk(n / 8, 256)), dim3(256), (size_t)0, STREAM(stream), a,
               reinterpret_cast<__half*>(out), n / 8);
    return LAUNCH_OK();
}

extern "C" int ctrlora_im2col_3x3_f16(const void* src, void* dst, int batch, int h, int w, int channels, void* stream) {
    if (!src || !dst || channels % 8 != 0) return CTRLORA_ERR_ARG;
    const int vecs = channels / 8;
    const long long total = static_cast<long long>(batch) * h * w * 9 * vecs;
    launch_pdl(im2col_3x3_kernel, dim3(nblk(total, 256)), dim3(256), (size_t)0, STREAM(stream),
               reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), batch, h, w, vecs);
    return LAUNCH_OK();
}

extern "C" int ctrlora_outer_accum_f32(const float* dy, int lddy, const float* x, int ldx, float* out, long long ldo, int rows,
                                       int n, int k, float alpha, float beta, int silu_x, void* stream) {
    if (!dy || !x || !out || rows < 1 || n < 1 || k < 1) return CTRLORA_ERR_ARG;
    launch_pdl(outer_accum_kernel, dim3((k + 255) / 256, n), dim3(256), (size_t)0, STREAM(stream), dy, lddy, x, ldx, out, ldo,
               rows, n, k, alpha, beta, silu_x);
    return LAUNCH_OK();
}

extern "C" int ctrlora_copy2d_f32(const float* src, long long lds, float* dst, long long ldd, long long rows, int cols,
                                  int accumulate, void* stream) {
    if (!src || !dst) return CTRLORA_ERR_ARG;
    launch_pdl(copy2d_kernel, dim3(nblk(rows * cols, 256)), dim3(256), (size_t)0, STREAM(stream), src, lds, dst, ldd, rows, cols,
               accumulate);
    return LAUNCH_OK();
}

extern "C" int ctrlora_silu_bwd_f32(const float* d, const float* x, float* out, long long n, void* stream) {
    if (!d || !x || !out) return CTRLORA_ERR_ARG;
    launch_pdl(silu_bwd_kernel, dim3(nblk(n, 256)), dim3(256), (size_t)0, STREAM(stream), d, x, out, n);
    return LAUNCH_OK();
}

extern "C" int ctrlora_cast_rows_f32_to_f16(const float* src, long long lds, void* dst, long long rows, int cols, void* stream) {
    if (!src || !dst) return CTRLORA_ERR_ARG;
    cast_rows_kernel<<<nblk(rows * cols, 256), 256, 0, STREAM(stream)>>>(src, lds, reinterpret_cast<__half*>(dst), rows, cols);
    return LAUNCH_OK();
}
