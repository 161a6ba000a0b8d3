// The CLIP text encoder's own kernels (reference: ldm/modules/encoders/modules.py:88-135 FrozenCLIPEmbedder, which runs
// transformers' CLIPTextModel): causal self-attention over <= 128 tokens, the token + position embedding gather, quick-GELU,
// and a LayerNorm that reads and writes either precision (the encoder keeps its residual stream in fp32).  The
// projections and the MLP are ctrlora_gemm_f16 launches.
#include "common.cuh"
#include "ctrlora_b200.h"
#include "wgmma.cuh"
#include <math.h>

namespace ctrl {

// ------------------------------------------------------------------------------------------ causal attention, d = 64
// One CTA per (image, head) holds every query, key and value of the head in shared memory:
//   Q [128 queries][64 d], K [128 keys][64 d], V^T [64 d][128 keys] as two 64-key halves, all in the SWIZZLE_128B layout
//   wgmma_desc_kmajor expects (rows of 128 B, 16-byte chunks XOR-permuted by row & 7), rows / keys >= n zero-filled.
// Warpgroup w owns query rows [64w, 64w + 64): S = Q K^T is one m64n128k16 chain, the causal mask and the softmax run on
// the fragment in registers (fp32, full rows: no online rescaling), P goes back into the wgmma as the A fragment and
// O = P V^T^T is an m64n64k16 chain over 128 keys.  Warpgroup 1 has nothing to do when n <= 64.
constexpr int CA_N = 128, CA_D = 64;
constexpr int CA_TILE = CA_N * 128;  // bytes of one [128][64] fp16 tile
constexpr int CA_SMEM = 3 * CA_TILE + 1024;

__device__ __forceinline__ uint32_t swz128(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

__global__ void __launch_bounds__(256, 1)
causal_attention_d64_kernel(const __half* __restrict__ q, long long ldq, const __half* __restrict__ k, long long ldk,
                            const __half* __restrict__ vt, int nk_pad, __half* __restrict__ out, long long ldo, int heads,
                            int n, float scale_log2e) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = smem + CA_TILE;
    uint8_t* sV = smem + 2 * CA_TILE;
    const int img = blockIdx.x / heads, head = blockIdx.x % heads;
    pdl_launch_dependents();
    pdl_wait();
    // ---- gather: 1024 16-byte chunks per operand, four per thread each
    const uint4 zero = make_uint4(0, 0, 0, 0);
    for (int i = threadIdx.x; i < CA_N * 8; i += blockDim.x) {
        const int row = i >> 3, ch = i & 7;
        uint4 qv = zero, kv = zero;
        if (row < n) {
            const long long tok = static_cast<long long>(img) * n + row;
            qv = __ldg(reinterpret_cast<const uint4*>(q + tok * ldq + head * CA_D + ch * 8));
            kv = __ldg(reinterpret_cast<const uint4*>(k + tok * ldk + head * CA_D + ch * 8));
        }
        *reinterpret_cast<uint4*>(sQ + swz128(row, ch)) = qv;
        *reinterpret_cast<uint4*>(sK + swz128(row, ch)) = kv;
        // V^T: row d of the head, keys [8 c16, 8 c16 + 8) with c16 = 0..15 -> half (c16 >> 3), chunk (c16 & 7)
        const int d = i >> 4, c16 = i & 15, key0 = c16 * 8;
        uint4 vv = zero;
        if (key0 < n) {
            const __half* src = vt + ((static_cast<long long>(img) * heads + head) * CA_D + d) * nk_pad + key0;
            if (key0 + 8 <= n) {
                vv = __ldg(reinterpret_cast<const uint4*>(src));
            } else {  // the keys in [n, nk_pad) are not ours to trust: zeros, so that P = 0 times them stays 0
                __half* h = reinterpret_cast<__half*>(&vv);
                for (int e = 0; e < n - key0; ++e) h[e] = src[e];
            }
        }
        *reinterpret_cast<uint4*>(sV + (c16 >> 3) * (CA_TILE / 2) + swz128(d, c16 & 7)) = vv;
    }
    fence_proxy_async_smem();  // generic-proxy stores -> wgmma operand reads
    __syncthreads();

    const int wg = threadIdx.x >> 7;
    if (wg * 64 >= n) return;
    const int lane = threadIdx.x & 31, warp_in_wg = (threadIdx.x >> 5) & 3;
    const uint32_t aQ = smem_u32(sQ) + wg * 64 * 128, aK = smem_u32(sK), aV = smem_u32(sV);
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < CA_D / 16; ++kk)
        WgmmaSS<128, 0, 0>::mma(s, wgmma_desc_kmajor(aQ + kk * 32), wgmma_desc_kmajor(aK + kk * 32), kk ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<64>(s);

    // ---- causal softmax of rows r0 and r0 + 8: key j > query i (and j >= n) is -inf before the row max
    const int r0 = wg * 64 + warp_in_wg * 16 + (lane >> 2), r1 = r0 + 8, kq = 2 * (lane & 3);
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int col = 8 * i + kq + e;
            s[4 * i + e] = (col <= r0 && col < n) ? s[4 * i + e] * scale_log2e : -INFINITY;
            s[4 * i + 2 + e] = (col <= r1 && col < n) ? s[4 * i + 2 + e] * scale_log2e : -INFINITY;
            mx0 = fmaxf(mx0, s[4 * i + e]);
            mx1 = fmaxf(mx1, s[4 * i + 2 + e]);
        }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    // rows >= n (never stored) have finite maxima too: key 0 is always visible
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            s[4 * i + e] = exp2f(s[4 * i + e] - mx0);
            s[4 * i + 2 + e] = exp2f(s[4 * i + 2 + e] - mx1);
            l0 += s[4 * i + e];
            l1 += s[4 * i + 2 + e];
        }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);

    // ---- O = P V: the S fragment of 16 columns is the A fragment of one k16 step
    uint32_t pa[32];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        pa[4 * (i >> 1) + 2 * (i & 1)] = pack_half2(s[4 * i], s[4 * i + 1]);
        pa[4 * (i >> 1) + 2 * (i & 1) + 1] = pack_half2(s[4 * i + 2], s[4 * i + 3]);
    }
    float o[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < CA_N / 16; ++kk)
        WgmmaRS<64, 0>::mma(o, pa + 4 * kk, wgmma_desc_kmajor(aV + (kk >> 2) * (CA_TILE / 2) + (kk & 3) * 32), kk ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<32>(o);
    wgmma_fence_regs<32>(pa);

    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    const long long base = static_cast<long long>(img) * n;
    __half* o0 = out + (base + r0) * ldo + head * CA_D;
    __half* o1 = out + (base + r1) * ldo + head * CA_D;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int col = 8 * i + kq;
        if (r0 < n) *reinterpret_cast<__half2*>(o0 + col) = __floats2half2_rn(o[4 * i] * inv0, o[4 * i + 1] * inv0);
        if (r1 < n) *reinterpret_cast<__half2*>(o1 + col) = __floats2half2_rn(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
    }
}

// ------------------------------------------------------------------------------------------ embeddings
// out[b * n + t, :] = token_embedding[ids[b, t], :] + position_embedding[t, :]   (CLIPTextEmbeddings, fp32 tables, one
// rounded add as in the reference).  An id outside the vocabulary writes NaN into its row rather than reading out of bounds.
__global__ void __launch_bounds__(256)
clip_embed_kernel(const long long* __restrict__ ids, const float* __restrict__ tok, const float* __restrict__ pos,
                  void* __restrict__ out, int out_f32, int rows, int n, int cols, int vocab) {
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const long long id = ids[row];
    const bool ok = id >= 0 && id < vocab;
    const float* te = tok + (ok ? id : 0) * cols;
    const float* pe = pos + static_cast<long long>(row % n) * cols;
    for (int c = lane * 4; c < cols; c += 128) {
        const float4 a = *reinterpret_cast<const float4*>(te + c), p = *reinterpret_cast<const float4*>(pe + c);
        float4 r = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
        if (!ok) r = make_float4(NAN, NAN, NAN, NAN);
        if (out_f32) {
            *reinterpret_cast<float4*>(static_cast<float*>(out) + static_cast<long long>(row) * cols + c) = r;
        } else {
            __half2 h[2] = {__floats2half2_rn(r.x, r.y), __floats2half2_rn(r.z, r.w)};
            *reinterpret_cast<uint2*>(static_cast<__half*>(out) + static_cast<long long>(row) * cols + c) =
                *reinterpret_cast<uint2*>(h);
        }
    }
}

// ------------------------------------------------------------------------------------------ quick-GELU
// x * sigmoid(1.702 x) in fp32, in place on fp16 (transformers' QuickGELUActivation, CLIP's hidden_act)
__global__ void __launch_bounds__(256) quick_gelu_kernel(__half* __restrict__ x, long long vecs) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < vecs; v += (long long)gridDim.x * blockDim.x) {
        uint4 u = reinterpret_cast<uint4*>(x)[v];
        __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h[e]);
            h[e] = __floats2half2_rn(f.x / (1.0f + __expf(-1.702f * f.x)), f.y / (1.0f + __expf(-1.702f * f.y)));
        }
        reinterpret_cast<uint4*>(x)[v] = u;
    }
}

// ------------------------------------------------------------------------------------------ LayerNorm, fp32 or fp16
// One warp per row, the row in registers between the mean and the variance pass (the arithmetic of
// ctrlora_layernorm_f16: mean, then the mean of squared deviations, rsqrtf(var + eps)).  Four columns per vector.
__device__ __forceinline__ void load4(const void* p, int f32, long long off, float* v) {
    if (f32) {
        const float4 a = *reinterpret_cast<const float4*>(static_cast<const float*>(p) + off);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    } else {
        const uint2 u = *reinterpret_cast<const uint2*>(static_cast<const __half*>(p) + off);
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
        const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
    }
}

template <int MAXV>
__global__ void __launch_bounds__(256)
layernorm_rows_kernel(const void* __restrict__ x, int x_f32, long long ldx, void* __restrict__ y, int y_f32, long long ldy,
                      int M, int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps) {
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= M) return;
    const int vecs = C >> 2;
    float v[MAXV][4];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vi = lane + i * 32;
        if (vi < vecs) {
            load4(x, x_f32, row * ldx + vi * 4, v[i]);
            sum += v[i][0] + v[i][1] + v[i][2] + v[i][3];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / C;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
        if (lane + i * 32 < vecs)
#pragma unroll
            for (int e = 0; e < 4; ++e) { const float d = v[i][e] - mean; sq += d * d; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq / C + eps);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vi = lane + i * 32;
        if (vi >= vecs) continue;
        const float4 g = *reinterpret_cast<const float4*>(gamma + vi * 4), b = *reinterpret_cast<const float4*>(beta + vi * 4);
        const float r0 = (v[i][0] - mean) * rstd * g.x + b.x, r1 = (v[i][1] - mean) * rstd * g.y + b.y;
        const float r2 = (v[i][2] - mean) * rstd * g.z + b.z, r3 = (v[i][3] - mean) * rstd * g.w + b.w;
        if (y_f32) {
            *reinterpret_cast<float4*>(static_cast<float*>(y) + row * ldy + vi * 4) = make_float4(r0, r1, r2, r3);
        } else {
            __half2 h[2] = {__floats2half2_rn(r0, r1), __floats2half2_rn(r2, r3)};
            *reinterpret_cast<uint2*>(static_cast<__half*>(y) + row * ldy + vi * 4) = *reinterpret_cast<uint2*>(h);
        }
    }
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_causal_attention_f16(const void* q, long long ldq, const void* k, long long ldk, const void* vt,
                                            int nk_pad, void* out, long long ldo, int batch, int heads, int n, int head_dim,
                                            void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!q || !k || !vt || !out || batch < 0 || heads < 1 || n < 1) return CTRLORA_ERR_ARG;
    if (head_dim != CA_D || n > CA_N) return CTRLORA_ERR_UNSUPPORTED;
    if (ldq % 8 || ldk % 8 || ldo % 2 || nk_pad % 8 || nk_pad < n || ldq < heads * CA_D || ldk < heads * CA_D ||
        ldo < heads * CA_D)
        return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(causal_attention_d64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CA_SMEM) !=
            cudaSuccess)
            return CTRLORA_ERR_CUDA;
        attr = true;
    }
    const float scale_log2e = 0.125f * 1.4426950408889634f;  // d^-1/2 = 1/8
    return launched(launch_pdl(causal_attention_d64_kernel, dim3(batch * heads), dim3(256), (size_t)CA_SMEM, stream,
                               static_cast<const __half*>(q), ldq, static_cast<const __half*>(k), ldk,
                               static_cast<const __half*>(vt), nk_pad, static_cast<__half*>(out), ldo, heads, n, scale_log2e));
}

extern "C" int ctrlora_clip_embed(const long long* ids, const float* token_embedding, const float* position_embedding,
                                  void* out, int out_f32, int batch, int n, int cols, int vocab, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!ids || !token_embedding || !position_embedding || !out || batch < 0 || n < 1 || cols < 4 || cols % 4 || vocab < 1)
        return CTRLORA_ERR_ARG;
    const int rows = batch * n;
    if (rows == 0) return CTRLORA_OK;
    return launched(launch_pdl(clip_embed_kernel, dim3((rows + 7) / 8), dim3(256), (size_t)0, stream, ids, token_embedding,
                               position_embedding, out, out_f32, rows, n, cols, vocab));
}

extern "C" int ctrlora_quick_gelu_f16(void* x, long long n, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || n < 0 || n % 8) return CTRLORA_ERR_ARG;
    const long long vecs = n / 8;
    if (vecs == 0) return CTRLORA_OK;
    long long blocks = (vecs + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    return launched(launch_pdl(quick_gelu_kernel, dim3((unsigned)blocks), dim3(256), (size_t)0, stream,
                               static_cast<__half*>(x), vecs));
}

extern "C" int ctrlora_layernorm_rows(const void* x, int x_f32, long long ldx, void* y, int y_f32, long long ldy, int rows,
                                      int cols, const float* gamma, const float* beta, float eps, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !y || !gamma || !beta || rows < 0 || cols < 4 || cols % 4 || ldx % 4 || ldy % 4) return CTRLORA_ERR_ARG;
    if (cols > 2048) return CTRLORA_ERR_UNSUPPORTED;
    if (rows == 0) return CTRLORA_OK;
    const dim3 grid((rows + 7) / 8), block(256);
    cudaError_t e;
    if (cols <= 256)
        e = launch_pdl(layernorm_rows_kernel<2>, grid, block, (size_t)0, stream, x, x_f32, ldx, y, y_f32, ldy, rows, cols, gamma,
                       beta, eps);
    else if (cols <= 1024)
        e = launch_pdl(layernorm_rows_kernel<8>, grid, block, (size_t)0, stream, x, x_f32, ldx, y, y_f32, ldy, rows, cols, gamma,
                       beta, eps);
    else
        e = launch_pdl(layernorm_rows_kernel<16>, grid, block, (size_t)0, stream, x, x_f32, ldx, y, y_f32, ldy, rows, cols,
                       gamma, beta, eps);
    return launched(e);
}
