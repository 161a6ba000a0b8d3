// Fused attention forward on wgmma for sm_90a:  O = softmax(Q K^T * d^-1/2) V  per (image, head, 64-query tile).
// reference: CrossAttention.forward, ldm/modules/attention.py:163-194 (fp32 logits and softmax, scale d_head^-0.5);
// the [8B, N, N] fp32 `sim` matrix the reference materialises (512 MiB per image at N = 4096) never exists here.
//
// One warpgroup per CTA owns 64 query rows; thread 0 streams 64-key tiles of K and V^T by TMA into a double buffer.
//   S = Q K^T      wgmma m64n64k16, both operands K-major in shared memory (SWIZZLE_128B TMA tiles), S in registers
//   softmax        online (running max / sum per row, fp32, exp2 domain); a row lives in the 4 threads of a quad
//   O += P V       wgmma with A = P straight from registers (the S accumulator fragment is the A fragment layout) and
//                  B = the V^T tile ([d x 64 keys], K-major; the V projection GEMM stores V transposed for this)
#include "common.cuh"
#include "ctrlora_b200.h"
#include "wgmma.cuh"
#include <math.h>
#include <string.h>

namespace ctrl {

int make_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box);

struct AttnParams {
    int Nq, Nk, heads, d;
    int n_kv_tiles;
    float scale_log2e;           // d^-1/2 * log2(e)
    __half* out;
    long long ldo;
    float* lse;                  // optional [B, H, Nq]: log2-domain log-sum-exp, for the backward
};

constexpr int ATT_BQ = 64, ATT_BKV = 64, ATT_THREADS = 128;

template <int DP>  // DP = d rounded up to 48 / 80 / 160: the wgmma N of P V
struct AttnSmem {
    static constexpr int NKC = (DP + 63) / 64;
    static constexpr int Q_BYTES = NKC * ATT_BQ * 128;   // [nkc][64 q][128 B]
    static constexpr int K_BYTES = NKC * ATT_BKV * 128;  // [nkc][64 keys][128 B]
    static constexpr int V_BYTES = DP * 128;             // V^T [DP][64 keys]
    static constexpr int STAGE = K_BYTES + V_BYTES;
    static constexpr int DATA = Q_BYTES + 2 * STAGE;
    static constexpr int TOTAL = DATA + 64 + 1024;
};

// pack the 64-column accumulator fragment x (two rows per thread) into the A fragments of four k16 steps
__device__ __forceinline__ void pack_a_frags(const float* x, uint32_t* a) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        a[4 * (i >> 1) + 2 * (i & 1)] = pack_half2(x[4 * i], x[4 * i + 1]);
        a[4 * (i >> 1) + 2 * (i & 1) + 1] = pack_half2(x[4 * i + 2], x[4 * i + 3]);
    }
}

template <int DP>
__global__ void __launch_bounds__(ATT_THREADS)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ AttnParams p) {
    using L = AttnSmem<DP>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::DATA);  // [0] Q, [1..2] K/V stages
    pdl_launch_dependents();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q0 = blockIdx.x * ATT_BQ, head = blockIdx.y, img = blockIdx.z;
    const uint32_t sQ = smem_u32(smem), sKV = sQ + L::Q_BYTES;
    auto load_kv = [&](int stage, int tile) {
        uint64_t* bar = &bars[1 + stage];
        uint8_t* dst = smem + L::Q_BYTES + stage * L::STAGE;
        mbar_expect_tx(bar, L::STAGE);
#pragma unroll
        for (int c = 0; c < L::NKC; ++c) tma_load_4d(dst + c * ATT_BKV * 128, &tmK, bar, c * 64, head, tile * ATT_BKV, img);
        tma_load_4d(dst + L::K_BYTES, &tmV, bar, tile * ATT_BKV, 0, head, img);
    };
    if (tid == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    if (tid == 0) {
        mbar_expect_tx(&bars[0], L::Q_BYTES);
#pragma unroll
        for (int c = 0; c < L::NKC; ++c) tma_load_4d(smem + c * ATT_BQ * 128, &tmQ, &bars[0], c * 64, head, q0, img);
        for (int s = 0; s < 2 && s < p.n_kv_tiles; ++s) load_kv(s, s);
    }
    float o[DP / 2];
#pragma unroll
    for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows r0 = 16 warp + lane / 4 and r0 + 8
    mbar_wait(&bars[0], 0);
    for (int t = 0; t < p.n_kv_tiles; ++t) {
        const int st = t & 1;
        const uint32_t sK = sKV + st * L::STAGE, sV = sK + L::K_BYTES;
        mbar_wait(&bars[1 + st], (t >> 1) & 1);
        float s[32];
        wgmma_fence();
        // all DP / 16 k-steps, a compile-time count (the columns beyond d are TMA zero fill): a runtime trip count would
        // move the accumulators between wgmmas and make the compiler serialise the warpgroup
#pragma unroll
        for (int kk = 0; kk < DP / 16; ++kk) {
            const uint32_t off = (kk >> 2) * 8192 + (kk & 3) * 32;
            WgmmaSS<64, 0, 0>::mma(s, wgmma_desc_kmajor(sQ + off), wgmma_desc_kmajor(sK + off), kk ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<32>(s);
        // ---- online softmax in the exp2 domain
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const bool ok = t * ATT_BKV + 8 * i + 2 * (lane & 3) + e < p.Nk;
                s[4 * i + e] = ok ? s[4 * i + e] * p.scale_log2e : -INFINITY;
                s[4 * i + 2 + e] = ok ? s[4 * i + 2 + e] * p.scale_log2e : -INFINITY;
                mx0 = fmaxf(mx0, s[4 * i + e]);
                mx1 = fmaxf(mx1, s[4 * i + 2 + e]);
            }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float a0 = fast_exp2(m0 - mx0), a1 = fast_exp2(m1 - mx1);
        m0 = mx0;
        m1 = mx1;
        float ls0 = 0.f, ls1 = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                s[4 * i + e] = fast_exp2(s[4 * i + e] - m0);
                s[4 * i + 2 + e] = fast_exp2(s[4 * i + 2 + e] - m1);
                ls0 += s[4 * i + e];
                ls1 += s[4 * i + 2 + e];
            }
        l0 = l0 * a0 + ls0;
        l1 = l1 * a1 + ls1;
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            o[4 * i] *= a0; o[4 * i + 1] *= a0;
            o[4 * i + 2] *= a1; o[4 * i + 3] *= a1;
        }
        uint32_t pa[16];
        pack_a_frags(s, pa);
        // ---- O += P V
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) WgmmaRS<DP, 0>::mma(o, pa + 4 * kk, wgmma_desc_kmajor(sV + 32 * kk), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<DP / 2>(o);
        wgmma_fence_regs<16>(pa);
        __syncthreads();  // every warp is done with this stage
        if (tid == 0 && t + 2 < p.n_kv_tiles) load_kv(st, t + 2);
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8, cq = 2 * (lane & 3);
    __half* o0 = p.out + (static_cast<long long>(img) * p.Nq + r0) * p.ldo + head * p.d;
    __half* o1 = p.out + (static_cast<long long>(img) * p.Nq + r1) * p.ldo + head * p.d;
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
        const int c = 8 * i + cq;
        if (c >= p.d) continue;
        if (r0 < p.Nq) *reinterpret_cast<__half2*>(o0 + c) = __floats2half2_rn(o[4 * i] * inv0, o[4 * i + 1] * inv0);
        if (r1 < p.Nq) *reinterpret_cast<__half2*>(o1 + c) = __floats2half2_rn(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
    }
    if (p.lse && (lane & 3) == 0) {
        float* lrow = p.lse + (static_cast<long long>(img) * p.heads + head) * p.Nq;
        if (r0 < p.Nq) lrow[r0] = m0 + log2f(l0);
        if (r1 < p.Nq) lrow[r1] = m1 + log2f(l1);
    }
}

template <int DP>
static int launch_attn(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnParams& p, dim3 grid,
                       cudaStream_t stream) {
    using L = AttnSmem<DP>;
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(attention_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL) != cudaSuccess)
            return CTRLORA_ERR_CUDA;
        attr = true;
    }
    if (launch_pdl(attention_kernel<DP>, grid, dim3(ATT_THREADS), (size_t)L::TOTAL, stream, tq, tk, tv, p) != cudaSuccess)
        return CTRLORA_ERR_CUDA;
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_attention_f16(const void* q, long long ldq, const void* k, long long ldk, const void* vt,
                                     int nk_pad, void* out, long long ldo, float* lse, int batch, int heads, int nq,
                                     int nk, int head_dim, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!q || !k || !vt || !out) return CTRLORA_ERR_ARG;
    const int d = head_dim;
    if (d % 8 != 0 || d > 160 || nk_pad % 8 != 0 || nk_pad < nk || ldq % 8 != 0 || ldk % 8 != 0 || ldo % 8 != 0 || nk < 1)
        return CTRLORA_ERR_ARG;
    const int dp = d <= 48 ? 48 : d <= 80 ? 80 : 160;
    AttnParams p;
    memset(&p, 0, sizeof(p));
    p.Nq = nq; p.Nk = nk; p.heads = heads; p.d = d;
    p.n_kv_tiles = (nk + ATT_BKV - 1) / ATT_BKV;
    p.scale_log2e = (1.0f / sqrtf(static_cast<float>(d))) * 1.4426950408889634f;
    p.out = reinterpret_cast<__half*>(out); p.ldo = ldo; p.lse = lse;
    CUtensorMap tq, tk, tv;
    {
        uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)nq, (uint64_t)batch};
        uint64_t str[3] = {(uint64_t)d * 2, (uint64_t)ldq * 2, (uint64_t)ldq * 2 * nq};
        uint32_t box[4] = {64, 1, ATT_BQ, 1};
        int rc = make_tmap_f16(&tq, q, 4, dims, str, box);
        if (rc) return rc;
    }
    {
        uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)nk, (uint64_t)batch};
        uint64_t str[3] = {(uint64_t)d * 2, (uint64_t)ldk * 2, (uint64_t)ldk * 2 * nk};
        uint32_t box[4] = {64, 1, ATT_BKV, 1};
        int rc = make_tmap_f16(&tk, k, 4, dims, str, box);
        if (rc) return rc;
    }
    {
        uint64_t dims[4] = {(uint64_t)nk, (uint64_t)d, (uint64_t)heads, (uint64_t)batch};
        uint64_t str[3] = {(uint64_t)nk_pad * 2, (uint64_t)nk_pad * 2 * d, (uint64_t)nk_pad * 2 * d * heads};
        uint32_t box[4] = {ATT_BKV, (uint32_t)dp, 1, 1};
        int rc = make_tmap_f16(&tv, vt, 4, dims, str, box);
        if (rc) return rc;
    }
    dim3 grid((nq + ATT_BQ - 1) / ATT_BQ, heads, batch);
    if (dp == 48) return launch_attn<48>(tq, tk, tv, p, grid, stream);
    if (dp == 80) return launch_attn<80>(tq, tk, tv, p, grid, stream);
    return launch_attn<160>(tq, tk, tv, p, grid, stream);
}
