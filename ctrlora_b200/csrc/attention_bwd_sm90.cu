// Attention backward on wgmma (training): given Q, K, V, O, dO and the forward's log-sum-exp, produce dQ, dK, dV.
// reference: autograd through CrossAttention.forward, ldm/modules/attention.py:163-194.
//
// Two kernels, no atomics; each CTA is one warpgroup that owns 64 rows and streams 64-row tiles of the other side by
// TMA into a double buffer:
//   attn_bwd_dq_kernel    CTA = 64 queries of one (image, head); loops over key tiles:
//                           S = Q K^T, dP = dO V^T -> P = exp2(S c - lse), dS = P (dP - D) (registers)
//                           -> dQ += dS K (A = dS from registers, the K tile re-read as an MN-major B operand)
//   attn_bwd_dkdv_kernel  CTA = 64 keys of one (image, head); loops over query tiles:
//                           S^T = K Q^T, dP^T = V dO^T -> P^T, dS^T (lse / D per column)
//                           -> dV += P^T dO, dK += dS^T Q (the dO / Q tiles re-read as MN-major B operands)
// The same [rows][64-col] SWIZZLE_128B TMA tiles serve both as K-major operands (contraction over d) and as MN-major
// operands (contraction over tokens); only the descriptor differs.  D = rowsum(dO * O) comes from a small pre-pass.
#include "common.cuh"
#include "ctrlora_b200.h"
#include "wgmma.cuh"
#include <math.h>
#include <string.h>

namespace ctrl {

int make_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box);

struct AttnBwdParams {
    int Nq, Nk, heads, d;
    float scale, scale_log2e;
    const float* lse;    // [B, H, Nq]  log2-domain: P = exp2(s * scale_log2e - lse)
    const float* delta;  // [B, H, Nq]  rowsum(dO * O)
    __half* dq; long long lddq;
    __half* dk; long long lddk;
    __half* dv; long long lddv;
};

constexpr int AB_ROWS = 64, AB_THREADS = 128;

// ================================================================================================ D = rowsum(dO * O)
__global__ void attn_bwd_delta_kernel(const __half* __restrict__ o, long long ldo, const __half* __restrict__ dout, long long lddo,
                                      float* __restrict__ delta, int batch, int heads, int nq, int d) {
    pdl_launch_dependents();
    pdl_wait();
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;  // (b, q, h)
    if (i >= static_cast<long long>(batch) * nq * heads) return;
    const int h = static_cast<int>(i % heads);
    const long long row = i / heads;  // b * nq + q
    const int b = static_cast<int>(row / nq), q = static_cast<int>(row % nq);
    const __half* op = o + row * ldo + h * d;
    const __half* dp = dout + row * lddo + h * d;
    float acc = 0.f;
    for (int c = 0; c < d; c += 8) {
        uint4 u = *reinterpret_cast<const uint4*>(op + c), w = *reinterpret_cast<const uint4*>(dp + c);
        const __half2* a = reinterpret_cast<const __half2*>(&u);
        const __half2* bb = reinterpret_cast<const __half2*>(&w);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 x = __half22float2(a[e]), y = __half22float2(bb[e]);
            acc += x.x * y.x + x.y * y.y;
        }
    }
    delta[(static_cast<long long>(b) * heads + h) * nq + q] = acc;
}

template <int DP>
struct AbSmem {
    static constexpr int NKC = (DP + 63) / 64;
    static constexpr int TILE = NKC * AB_ROWS * 128;  // one [nkc][64 rows][128 B] token tile
    static constexpr int OWN = 2 * TILE;              // the CTA's own two tiles (Q, dO  or  K, V)
    static constexpr int STAGE = 2 * TILE;            // the streamed pair
    static constexpr int STAT = OWN + 2 * STAGE;      // dkdv: [2 stages][lse 64 | delta 64] fp32
    static constexpr int DATA = STAT + 2 * 2 * AB_ROWS * 4;
    static constexpr int TOTAL = DATA + 64 + 1024;
};

__device__ __forceinline__ void ab_pack(const float* x, uint32_t* a) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        a[4 * (i >> 1) + 2 * (i & 1)] = pack_half2(x[4 * i], x[4 * i + 1]);
        a[4 * (i >> 1) + 2 * (i & 1) + 1] = pack_half2(x[4 * i + 2], x[4 * i + 3]);
    }
}

// acc[64 x 64] = X[64 rows x d] Y[64 rows x d]^T over the DP / 16 k-steps of two K-major token tiles (the columns beyond
// d are TMA zero fill; a compile-time trip count keeps the accumulators in place between the wgmmas)
template <int DP>
__device__ __forceinline__ void ab_dot(float* acc, uint32_t x, uint32_t y) {
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {
        const uint32_t off = (kk >> 2) * (AB_ROWS * 128) + (kk & 3) * 32;
        WgmmaSS<64, 0, 0>::mma(acc, wgmma_desc_kmajor(x + off), wgmma_desc_kmajor(y + off), kk ? 1u : 0u);
    }
}

// store rows r0 / r0 + 8 (columns < d) of a [64 x DP] accumulator, times `scale`
template <int DP>
__device__ __forceinline__ void ab_store(const float* acc, float scale, __half* base, long long ld, int row0, int nrows, int d) {
    const int lane = threadIdx.x & 31;
    const int r0 = row0 + (threadIdx.x >> 5) * 16 + (lane >> 2), r1 = r0 + 8, cq = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
        const int c = 8 * i + cq;
        if (c >= d) continue;
        if (r0 < nrows) *reinterpret_cast<__half2*>(base + r0 * ld + c) = __floats2half2_rn(acc[4 * i] * scale, acc[4 * i + 1] * scale);
        if (r1 < nrows) *reinterpret_cast<__half2*>(base + r1 * ld + c) = __floats2half2_rn(acc[4 * i + 2] * scale, acc[4 * i + 3] * scale);
    }
}

// ================================================================================================ dQ
template <int DP>
__global__ void __launch_bounds__(AB_THREADS)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmDO,
                   const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                   const __grid_constant__ AttnBwdParams p) {
    using L = AbSmem<DP>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::DATA);
    pdl_launch_dependents();
    const int tid = threadIdx.x, lane = tid & 31;
    const int q0 = blockIdx.x * AB_ROWS, head = blockIdx.y, img = blockIdx.z;
    const int n_tiles = (p.Nk + AB_ROWS - 1) / AB_ROWS;
    const uint32_t s0 = smem_u32(smem);
    auto load_kv = [&](int stage, int tile) {
        uint64_t* bar = &bars[1 + stage];
        uint8_t* dst = smem + L::OWN + stage * L::STAGE;
        mbar_expect_tx(bar, L::STAGE);
#pragma unroll
        for (int c = 0; c < L::NKC; ++c) {
            tma_load_4d(dst + c * AB_ROWS * 128, &tmK, bar, c * 64, head, tile * AB_ROWS, img);
            tma_load_4d(dst + L::TILE + c * AB_ROWS * 128, &tmV, bar, c * 64, head, tile * AB_ROWS, img);
        }
    };
    if (tid == 0) {
        for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    if (tid == 0) {
        mbar_expect_tx(&bars[0], L::OWN);
#pragma unroll
        for (int c = 0; c < L::NKC; ++c) {
            tma_load_4d(smem + c * AB_ROWS * 128, &tmQ, &bars[0], c * 64, head, q0, img);
            tma_load_4d(smem + L::TILE + c * AB_ROWS * 128, &tmDO, &bars[0], c * 64, head, q0, img);
        }
        for (int s = 0; s < 2 && s < n_tiles; ++s) load_kv(s, s);
    }
    const int r0 = q0 + (tid >> 5) * 16 + (lane >> 2), r1 = r0 + 8;
    const long long stat = (static_cast<long long>(img) * p.heads + head) * p.Nq;
    const float lse0 = r0 < p.Nq ? p.lse[stat + r0] : 0.f, lse1 = r1 < p.Nq ? p.lse[stat + r1] : 0.f;
    const float dl0 = r0 < p.Nq ? p.delta[stat + r0] : 0.f, dl1 = r1 < p.Nq ? p.delta[stat + r1] : 0.f;
    float dq[DP / 2];
#pragma unroll
    for (int i = 0; i < DP / 2; ++i) dq[i] = 0.f;
    mbar_wait_nocall(&bars[0], 0);
    for (int t = 0; t < n_tiles; ++t) {
        const int st = t & 1;
        const uint32_t sK = s0 + L::OWN + st * L::STAGE, sV = sK + L::TILE;
        mbar_wait_nocall(&bars[1 + st], (t >> 1) & 1);
        float s[32], dp[32];
        wgmma_fence();
        ab_dot<DP>(s, s0, sK);
        ab_dot<DP>(dp, s0 + L::TILE, sV);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<32>(s);
        wgmma_fence_regs<32>(dp);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const bool ok = t * AB_ROWS + 8 * i + 2 * (lane & 3) + e < p.Nk;
                const float pa = ok ? fast_exp2(fmaf(s[4 * i + e], p.scale_log2e, -lse0)) : 0.f;
                const float pb = ok ? fast_exp2(fmaf(s[4 * i + 2 + e], p.scale_log2e, -lse1)) : 0.f;
                s[4 * i + e] = pa * (dp[4 * i + e] - dl0);
                s[4 * i + 2 + e] = pb * (dp[4 * i + 2 + e] - dl1);
            }
        uint32_t ds[16];
        ab_pack(s, ds);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) WgmmaRS<DP, 1>::mma(dq, ds + 4 * kk, wgmma_desc_mnmajor(sK + kk * 2048, AB_ROWS * 128), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<DP / 2>(dq);
        wgmma_fence_regs<16>(ds);
        __syncthreads();
        if (tid == 0 && t + 2 < n_tiles) load_kv(st, t + 2);
    }
    ab_store<DP>(dq, p.scale, p.dq + static_cast<long long>(img) * p.Nq * p.lddq + head * p.d, p.lddq, q0, p.Nq, p.d);
}

// ================================================================================================ dK, dV
// WHICH: 0 = dK and dV, 1 = dV only, 2 = dK only (d_head 160: the two accumulators would not fit the register file)
template <int DP, int WHICH>
__global__ void __launch_bounds__(AB_THREADS)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmDO,
                     const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                     const __grid_constant__ AttnBwdParams p) {
    using L = AbSmem<DP>;
    constexpr bool DO_V = WHICH != 2, DO_K = WHICH != 1;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::DATA);
    float* sStat = reinterpret_cast<float*>(smem + L::STAT);
    pdl_launch_dependents();
    const int tid = threadIdx.x, lane = tid & 31;
    const int k0 = blockIdx.x * AB_ROWS, head = blockIdx.y, img = blockIdx.z;
    const int n_tiles = (p.Nq + AB_ROWS - 1) / AB_ROWS;
    const uint32_t s0 = smem_u32(smem);
    auto load_q = [&](int stage, int tile) {
        uint64_t* bar = &bars[1 + stage];
        uint8_t* dst = smem + L::OWN + stage * L::STAGE;
        mbar_expect_tx(bar, L::STAGE);
#pragma unroll
        for (int c = 0; c < L::NKC; ++c) {
            tma_load_4d(dst + c * AB_ROWS * 128, &tmQ, bar, c * 64, head, tile * AB_ROWS, img);
            tma_load_4d(dst + L::TILE + c * AB_ROWS * 128, &tmDO, bar, c * 64, head, tile * AB_ROWS, img);
        }
    };
    if (tid == 0) {
        for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    if (tid == 0) {
        mbar_expect_tx(&bars[0], L::OWN);
#pragma unroll
        for (int c = 0; c < L::NKC; ++c) {
            tma_load_4d(smem + c * AB_ROWS * 128, &tmK, &bars[0], c * 64, head, k0, img);
            tma_load_4d(smem + L::TILE + c * AB_ROWS * 128, &tmV, &bars[0], c * 64, head, k0, img);
        }
        for (int s = 0; s < 2 && s < n_tiles; ++s) load_q(s, s);
    }
    const long long stat = (static_cast<long long>(img) * p.heads + head) * p.Nq;
    float dk[DO_K ? DP / 2 : 1], dv[DO_V ? DP / 2 : 1];
#pragma unroll
    for (int i = 0; i < DP / 2; ++i) {
        if (DO_K) dk[i] = 0.f;
        if (DO_V) dv[i] = 0.f;
    }
    mbar_wait_nocall(&bars[0], 0);
    for (int t = 0; t < n_tiles; ++t) {
        const int st = t & 1;
        const uint32_t sQ = s0 + L::OWN + st * L::STAGE, sDO = sQ + L::TILE;
        float* sl = sStat + st * 2 * AB_ROWS;
        {
            const int q = t * AB_ROWS + (tid & 63);
            sl[tid] = q < p.Nq ? (tid < 64 ? p.lse[stat + q] : p.delta[stat + q]) : 0.f;
        }
        __syncthreads();
        mbar_wait_nocall(&bars[1 + st], (t >> 1) & 1);
        float s[32], dp[DO_K ? 32 : 1];
        wgmma_fence();
        ab_dot<DP>(s, s0, sQ);
        if (DO_K) ab_dot<DP>(dp, s0 + L::TILE, sDO);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<32>(s);
        if (DO_K) wgmma_fence_regs<32>(dp);
        // column = query: P^T[key][q] = exp2(S^T c - lse[q]), dS^T = P^T (dP^T - D[q])
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int ql = 8 * i + 2 * (lane & 3) + e;
                const bool ok = t * AB_ROWS + ql < p.Nq;
                const float lse = sl[ql], dl = sl[AB_ROWS + ql];
                const float pa = ok ? fast_exp2(fmaf(s[4 * i + e], p.scale_log2e, -lse)) : 0.f;
                const float pb = ok ? fast_exp2(fmaf(s[4 * i + 2 + e], p.scale_log2e, -lse)) : 0.f;
                s[4 * i + e] = pa;
                s[4 * i + 2 + e] = pb;
                if (DO_K) {
                    dp[4 * i + e] = pa * (dp[4 * i + e] - dl);
                    dp[4 * i + 2 + e] = pb * (dp[4 * i + 2 + e] - dl);
                }
            }
        uint32_t pt[16], dst[16];
        if (DO_V) ab_pack(s, pt);
        if (DO_K) ab_pack(dp, dst);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if (DO_V) WgmmaRS<DP, 1>::mma(dv, pt + 4 * kk, wgmma_desc_mnmajor(sDO + kk * 2048, AB_ROWS * 128), 1u);
            if (DO_K) WgmmaRS<DP, 1>::mma(dk, dst + 4 * kk, wgmma_desc_mnmajor(sQ + kk * 2048, AB_ROWS * 128), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        if (DO_V) { wgmma_fence_regs<DP / 2>(dv); wgmma_fence_regs<16>(pt); }
        if (DO_K) { wgmma_fence_regs<DP / 2>(dk); wgmma_fence_regs<16>(dst); }
        __syncthreads();
        if (tid == 0 && t + 2 < n_tiles) load_q(st, t + 2);
    }
    if (DO_V) ab_store<DP>(dv, 1.0f, p.dv + static_cast<long long>(img) * p.Nk * p.lddv + head * p.d, p.lddv, k0, p.Nk, p.d);
    if (DO_K) ab_store<DP>(dk, p.scale, p.dk + static_cast<long long>(img) * p.Nk * p.lddk + head * p.d, p.lddk, k0, p.Nk, p.d);
}

template <typename K>
static int ab_launch(K kernel, int smem, const CUtensorMap& tq, const CUtensorMap& tdo, const CUtensorMap& tk, const CUtensorMap& tv,
                     const AttnBwdParams& p, dim3 grid, cudaStream_t s) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return CTRLORA_ERR_CUDA;
    return launch_pdl(kernel, grid, dim3(AB_THREADS), (size_t)smem, s, tq, tdo, tk, tv, p) == cudaSuccess ? CTRLORA_OK
                                                                                                       : CTRLORA_ERR_CUDA;
}

template <int DP>
static int launch_bwd(const CUtensorMap& tq, const CUtensorMap& tdo, const CUtensorMap& tk, const CUtensorMap& tv,
                      const AttnBwdParams& p, int batch, cudaStream_t s) {
    const int smem = AbSmem<DP>::TOTAL;
    int rc = ab_launch(attn_bwd_dq_kernel<DP>, smem, tq, tdo, tk, tv, p, dim3((p.Nq + AB_ROWS - 1) / AB_ROWS, p.heads, batch), s);
    if (rc) return rc;
    const dim3 grid((p.Nk + AB_ROWS - 1) / AB_ROWS, p.heads, batch);
    if (DP <= 80) return ab_launch(attn_bwd_dkdv_kernel<DP, 0>, smem, tq, tdo, tk, tv, p, grid, s);
    rc = ab_launch(attn_bwd_dkdv_kernel<DP, 1>, smem, tq, tdo, tk, tv, p, grid, s);
    if (rc) return rc;
    return ab_launch(attn_bwd_dkdv_kernel<DP, 2>, smem, tq, tdo, tk, tv, p, grid, s);
}

static int tmap_tokens(CUtensorMap* m, const void* base, long long ld, int d, int heads, int n, int batch) {
    uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)n, (uint64_t)batch};
    uint64_t str[3] = {(uint64_t)d * 2, (uint64_t)ld * 2, (uint64_t)ld * 2 * n};
    uint32_t box[4] = {64, 1, (uint32_t)AB_ROWS, 1};
    return make_tmap_f16(m, base, 4, dims, str, box);
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_attention_bwd_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v,
                                         long long ldv, const void* o, long long ldo, const void* dout, long long lddo,
                                         const float* lse, float* delta_ws, void* dq, long long lddq, void* dk, long long lddk,
                                         void* dv, long long lddv, int batch, int heads, int nq, int nk, int head_dim,
                                         void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!q || !k || !v || !o || !dout || !lse || !delta_ws || !dq || !dk || !dv) return CTRLORA_ERR_ARG;
    const int d = head_dim;
    if (d % 8 || d > 160 || ldq % 8 || ldk % 8 || ldv % 8 || ldo % 8 || lddo % 8 || lddq % 8 || lddk % 8 || lddv % 8)
        return CTRLORA_ERR_ARG;
    {
        const long long total = static_cast<long long>(batch) * nq * heads;
        launch_pdl(attn_bwd_delta_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), (size_t)0, stream,
                   reinterpret_cast<const __half*>(o), ldo, reinterpret_cast<const __half*>(dout), lddo, delta_ws, batch, heads, nq, d);
    }
    AttnBwdParams p;
    memset(&p, 0, sizeof(p));
    p.Nq = nq; p.Nk = nk; p.heads = heads; p.d = d;
    p.scale = 1.0f / sqrtf(static_cast<float>(d));
    p.scale_log2e = p.scale * 1.4426950408889634f;
    p.lse = lse; p.delta = delta_ws;
    p.dq = reinterpret_cast<__half*>(dq); p.lddq = lddq;
    p.dk = reinterpret_cast<__half*>(dk); p.lddk = lddk;
    p.dv = reinterpret_cast<__half*>(dv); p.lddv = lddv;
    CUtensorMap tq, tdo, tk, tv;
    int rc = tmap_tokens(&tq, q, ldq, d, heads, nq, batch);
    if (!rc) rc = tmap_tokens(&tdo, dout, lddo, d, heads, nq, batch);
    if (!rc) rc = tmap_tokens(&tk, k, ldk, d, heads, nk, batch);
    if (!rc) rc = tmap_tokens(&tv, v, ldv, d, heads, nk, batch);
    if (rc) return rc;
    if (d <= 48) rc = launch_bwd<48>(tq, tdo, tk, tv, p, batch, stream);
    else if (d <= 80) rc = launch_bwd<80>(tq, tdo, tk, tv, p, batch, stream);
    else rc = launch_bwd<160>(tq, tdo, tk, tv, p, batch, stream);
    if (rc) return rc;
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}
