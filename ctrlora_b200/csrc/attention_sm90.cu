// Fused attention forward on wgmma for sm_90a:  O = softmax(Q K^T * d^-1/2) V  per (image, head, query tile).
// reference: CrossAttention.forward, ldm/modules/attention.py:163-194 (fp32 logits and softmax, scale d_head^-0.5);
// the [8B, N, N] fp32 `sim` matrix the reference materialises (512 MiB per image at N = 4096) never exists here.
//
// Warp-specialised and persistent (the FlashAttention-3 schedule):
//   warpgroup 0     one thread streams Q (64 rows per consumer warpgroup per work unit) and 64-key tiles of K and V^T
//                   by TMA into a ring of stages with full / empty mbarriers; the warpgroup gives its registers away
//   warpgroups 1..  64 query rows each (three consumer warpgroups at d <= 48, two above); all read every K / V stage,
//                   which is refilled once all have released it
//   S = Q K^T       wgmma m64n64k16, both operands K-major in shared memory (SWIZZLE_128B TMA tiles), S in registers
//   softmax         online, exp2 domain: per score one scale, one subtract, one ex2; only a partial last key tile
//                   masks (a warp-uniform branch); O is rescaled only when a row max moved
//   O += P V        A = P straight from registers (the S accumulator fragment is the A fragment layout), B = the V^T
//                   tile ([d x 64 keys], K-major; the V projection GEMM stores V transposed for this)
// Per key tile t a consumer warpgroup issues S_t = Q K_t^T and O += P_{t-1} V_{t-1} back to back and runs the softmax of
// S_t while the PV wgmma is in flight.  Named barriers pass the right to issue round robin between the consumer
// warpgroups, so one warpgroup's softmax runs under another's wgmmas (ping-pong).  Every wait is mbar_wait_nocall: a function call
// in the kernel would make ptxas serialise all of its wgmmas.  Per row and key tile the arithmetic is
// that of the earlier one-warpgroup kernel, so the results are bit-identical to it.
// CTA b runs work units b, b + gridDim.x, ... with the query tile fastest, so CTAs running at the same time read the
// same K / V from L2.  The producer loads the next unit's Q as soon as all warpgroups have finished their last QK^T,
// under the last PV and the epilogue.  CTAs never wait on each other.
#include "common.cuh"
#include "ctrlora_b200.h"
#include "wgmma.cuh"
#include <math.h>
#include <string.h>

namespace ctrl {

int make_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box);
int persistent_sms();

struct AttnParams {
    int Nq, Nk, heads, d;
    int n_kv_tiles, q_tiles, units;
    float scale_log2e;           // d^-1/2 * log2(e)
    __half* out;
    long long ldo;
    float* lse;                  // optional [B, H, Nq]: log2-domain log-sum-exp, for the backward
};

constexpr int ATT_BKV = 64;

template <int DP>  // DP = d rounded up to 48 / 80 / 160: the wgmma N of P V
struct AttnSmem {
    // consumer warpgroups: three at DP = 48, where the softmax dominates and a third warp per scheduler hides its
    // latency chain (S wait, row max, shuffles, packing); two where the O accumulator needs the registers
    static constexpr int NWG = DP <= 48 ? 3 : 2;
    static constexpr int BQ = 64 * NWG;                   // query rows of a work unit
    static constexpr int THREADS = 128 * (NWG + 1), CONSUMERS = 128 * NWG;
    static constexpr int PRODUCER_REGS = NWG == 3 ? 24 : 40, CONSUMER_REGS = NWG == 3 ? 160 : 232;
    static constexpr int NKC = (DP + 63) / 64;            // 64-column (128-byte) chunks of a Q / K row
    static constexpr int STAGES = DP <= 48 ? 6 : DP <= 80 ? 4 : 3;
    static constexpr int Q_CHUNK = BQ * 128;              // [BQ q][128 B] per chunk
    static constexpr int Q_BYTES = NKC * Q_CHUNK;
    static constexpr int K_CHUNK = ATT_BKV * 128;         // [64 keys][128 B] per chunk
    static constexpr int K_BYTES = NKC * K_CHUNK;
    static constexpr int V_BYTES = DP * 128;              // V^T [DP][64 keys]
    static constexpr int STAGE = K_BYTES + V_BYTES;
    static constexpr int DATA = Q_BYTES + STAGES * STAGE;
    static constexpr int TOTAL = DATA + (2 + 2 * STAGES) * 8 + 1024;
};

// S = Q K^T of one warpgroup: all DP / 16 k-steps, a compile-time count (the columns beyond d are TMA zero fill)
template <int DP>
__device__ __forceinline__ void issue_qk(float* s, uint32_t sQ, uint32_t sK) {
    using L = AttnSmem<DP>;
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk)
        WgmmaSS<64, 0, 0>::mma(s, wgmma_desc_kmajor(sQ + (kk >> 2) * L::Q_CHUNK + (kk & 3) * 32),
                               wgmma_desc_kmajor(sK + (kk >> 2) * L::K_CHUNK + (kk & 3) * 32), kk ? 1u : 0u);
    wgmma_commit();
}

template <int DP>
__device__ __forceinline__ void issue_pv(float* o, const uint32_t* pa, uint32_t sV) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) WgmmaRS<DP, 0>::mma(o, pa + 4 * kk, wgmma_desc_kmajor(sV + 32 * kk), 1u);
    wgmma_commit();
}

// Online softmax of one 64-key tile of S (rows r0 and r0 + 8 of the thread, 16 columns each); s becomes P (unnormalised),
// m / l the running row max (scaled, exp2 domain) and row sum, a the factor the previous O and l are scaled by.  MASK:
// keys from `key0 + column` onwards that are >= nk are -inf.  The arithmetic (scale, then subtract the max; row sums
// in column order) is the one the sampling and training results were validated with: a different rounding pattern
// moves the ill-conditioned LoRA gradients of the time-embedding layers by up to 1e-3 relative.
template <bool MASK>
__device__ __forceinline__ void softmax_tile(float* s, float (&m)[2], float (&l)[2], float (&a)[2], float c, int key0,
                                             int nk) {
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const bool ok = !MASK || key0 + 8 * i + e < nk;
            s[4 * i + e] = ok ? s[4 * i + e] * c : -INFINITY;
            s[4 * i + 2 + e] = ok ? s[4 * i + 2 + e] * c : -INFINITY;
            mx[0] = fmaxf(mx[0], s[4 * i + e]);
            mx[1] = fmaxf(mx[1], s[4 * i + 2 + e]);
        }
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        a[h] = fast_exp2(m[h] - mx[h]);  // exactly 1 when the max has not moved; 0 on the first tile
        m[h] = mx[h];
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            s[4 * i + e] = fast_exp2(s[4 * i + e] - m[0]);
            s[4 * i + 2 + e] = fast_exp2(s[4 * i + 2 + e] - m[1]);
            ls[0] += s[4 * i + e];
            ls[1] += s[4 * i + 2 + e];
        }
    l[0] = l[0] * a[0] + ls[0];
    l[1] = l[1] * a[1] + ls[1];
}

// pack the 64-column accumulator fragment x (two rows per thread) into the A fragments of four k16 steps
__device__ __forceinline__ void pack_a_frags(const float* x, uint32_t* a) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        a[4 * (i >> 1) + 2 * (i & 1)] = pack_half2(x[4 * i], x[4 * i + 1]);
        a[4 * (i >> 1) + 2 * (i & 1) + 1] = pack_half2(x[4 * i + 2], x[4 * i + 3]);
    }
}

template <int DP>
__global__ void __launch_bounds__(AttnSmem<DP>::THREADS, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ AttnParams p) {
    using L = AttnSmem<DP>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + L::DATA);
    uint64_t* q_empty = q_full + 1;
    uint64_t* full = q_full + 2;
    uint64_t* empty = full + L::STAGES;
    pdl_launch_dependents();
    const int warp = uniform_warp_idx();
    const int n_kv = p.n_kv_tiles;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        mbar_init(q_full, 1);
        mbar_init(q_empty, L::CONSUMERS);
        for (int i = 0; i < L::STAGES; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], L::CONSUMERS);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    if (warp < 4) {
        // ---------------------------------------------------- TMA producer: one thread of warpgroup 0
        setmaxnreg_dec<L::PRODUCER_REGS>();
        if (warp == 0 && elect_one()) {
            int s = 0;
            uint32_t phase = 0, qphase = 0;
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                const int qt = u % p.q_tiles, hi = u / p.q_tiles, head = hi % p.heads, img = hi / p.heads;
                mbar_wait_nocall(q_empty, qphase ^ 1);  // all warpgroups are done with the previous unit's Q
                qphase ^= 1;
                mbar_expect_tx(q_full, L::Q_BYTES);
#pragma unroll
                for (int c = 0; c < L::NKC; ++c)
                    tma_load_4d(smem + c * L::Q_CHUNK, &tmQ, q_full, c * 64, head, qt * L::BQ, img);
                for (int t = 0; t < n_kv; ++t) {
                    mbar_wait_nocall(&empty[s], phase ^ 1);
                    uint8_t* dst = smem + L::Q_BYTES + s * L::STAGE;
                    mbar_expect_tx(&full[s], L::STAGE);
#pragma unroll
                    for (int c = 0; c < L::NKC; ++c)
                        tma_load_4d(dst + c * L::K_CHUNK, &tmK, &full[s], c * 64, head, t * ATT_BKV, img);
                    tma_load_4d(dst + L::K_BYTES, &tmV, &full[s], t * ATT_BKV, 0, head, img);
                    if (++s == L::STAGES) { s = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // -------------------------------------------------------- consumers: query rows [64 wg, 64 wg + 64) of every unit
    setmaxnreg_inc<L::CONSUMER_REGS>();
    const int ct = threadIdx.x - 128, wg = ct >> 7, lane = threadIdx.x & 31;
    const uint32_t sQ = smem_u32(smem) + wg * 64 * 128, sKV = smem_u32(smem) + L::Q_BYTES;
    const float c = p.scale_log2e;
    const bool ragged = (p.Nk % ATT_BKV) != 0;
    const int kq = 2 * (lane & 3);  // the thread's first column in every 8-column group of S
    // ping-pong: warpgroup wg issues its wgmmas after bar.sync on barrier 1 + wg, then arrives on the next warpgroup's
    // (round robin).  Warpgroup 0 goes first; the last warpgroup's opening arrival is consumed by warpgroup 0's final
    // sync.  A named barrier counts the threads of the two warpgroups that meet on it.
    const int bar_own = 1 + wg, bar_next = 1 + (wg + 1) % L::NWG;
    if (wg == L::NWG - 1) named_bar_arrive(1, 256);
    int s = 0;
    uint32_t phase = 0, qphase = 0;
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        const int qt = u % p.q_tiles, hi = u / p.q_tiles, head = hi % p.heads, img = hi / p.heads;
        float o[DP / 2];
#pragma unroll
        for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
        float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, a[2];
        float sc[32];
        uint32_t pa[16];
        mbar_wait_nocall(q_full, qphase);
        qphase ^= 1;

        // ---- key tile 0: S only
        mbar_wait_nocall(&full[s], phase);
        named_bar_sync(bar_own, 256);
        wgmma_fence();
        issue_qk<DP>(sc, sQ, sKV + s * L::STAGE);
        named_bar_arrive(bar_next, 256);
        wgmma_wait<0>();
        wgmma_fence_regs<32>(sc);
        if (n_kv == 1) mbar_arrive(q_empty);
        if (ragged && n_kv == 1) softmax_tile<true>(sc, m, l, a, c, kq, p.Nk);
        else softmax_tile<false>(sc, m, l, a, c, kq, p.Nk);
        pack_a_frags(sc, pa);
        int prev = s;
        if (++s == L::STAGES) { s = 0; phase ^= 1; }

        // ---- key tiles 1 ..: S_t and P_{t-1} V_{t-1} in flight together, softmax of S_t under the PV wgmma
        for (int t = 1; t < n_kv; ++t) {
            mbar_wait_nocall(&full[s], phase);
            named_bar_sync(bar_own, 256);
            wgmma_fence();
            issue_qk<DP>(sc, sQ, sKV + s * L::STAGE);
            issue_pv<DP>(o, pa, sKV + prev * L::STAGE + L::K_BYTES);
            named_bar_arrive(bar_next, 256);
            wgmma_wait<1>();
            wgmma_fence_regs<32>(sc);
            if (t == n_kv - 1) mbar_arrive(q_empty);
            if (ragged && t == n_kv - 1) softmax_tile<true>(sc, m, l, a, c, t * ATT_BKV + kq, p.Nk);
            else softmax_tile<false>(sc, m, l, a, c, t * ATT_BKV + kq, p.Nk);
            wgmma_wait<0>();
            wgmma_fence_regs<DP / 2>(o);
            wgmma_fence_regs<16>(pa);
            mbar_arrive(&empty[prev]);
            if (__any_sync(0xffffffffu, a[0] != 1.f || a[1] != 1.f)) {
#pragma unroll
                for (int i = 0; i < DP / 8; ++i) {
                    o[4 * i] *= a[0]; o[4 * i + 1] *= a[0];
                    o[4 * i + 2] *= a[1]; o[4 * i + 3] *= a[1];
                }
            }
            pack_a_frags(sc, pa);
            prev = s;
            if (++s == L::STAGES) { s = 0; phase ^= 1; }
        }
        wgmma_fence();
        issue_pv<DP>(o, pa, sKV + prev * L::STAGE + L::K_BYTES);
        wgmma_wait<0>();
        wgmma_fence_regs<DP / 2>(o);
        mbar_arrive(&empty[prev]);

        // ---- epilogue: rows r0 and r0 + 8 of the thread, straight from the fragment
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
            l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
        }
        const float inv0 = 1.0f / l[0], inv1 = 1.0f / l[1];
        const int r0 = qt * L::BQ + wg * 64 + ((ct >> 5) & 3) * 16 + (lane >> 2), r1 = r0 + 8;
        __half* o0 = p.out + (static_cast<long long>(img) * p.Nq + r0) * p.ldo + head * p.d;
        __half* o1 = p.out + (static_cast<long long>(img) * p.Nq + r1) * p.ldo + head * p.d;
#pragma unroll
        for (int i = 0; i < DP / 8; ++i) {
            const int col = 8 * i + kq;
            if (col >= p.d) continue;
            if (r0 < p.Nq) *reinterpret_cast<__half2*>(o0 + col) = __floats2half2_rn(o[4 * i] * inv0, o[4 * i + 1] * inv0);
            if (r1 < p.Nq) *reinterpret_cast<__half2*>(o1 + col) = __floats2half2_rn(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
        }
        if (p.lse && (lane & 3) == 0) {
            float* lrow = p.lse + (static_cast<long long>(img) * p.heads + head) * p.Nq;
            if (r0 < p.Nq) lrow[r0] = m[0] + log2f(l[0]);
            if (r1 < p.Nq) lrow[r1] = m[1] + log2f(l[1]);
        }
    }
    if (wg == 0) named_bar_sync(1, 256);
}

template <int DP>
static int launch_attn(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnParams& p, int grid,
                       cudaStream_t stream) {
    using L = AttnSmem<DP>;
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(attention_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL) != cudaSuccess)
            return CTRLORA_ERR_CUDA;
        attr = true;
    }
    if (launch_pdl(attention_kernel<DP>, dim3(grid), dim3(L::THREADS), (size_t)L::TOTAL, stream, tq, tk, tv, p) !=
        cudaSuccess)
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
    const int bq = dp == 48 ? AttnSmem<48>::BQ : dp == 80 ? AttnSmem<80>::BQ : AttnSmem<160>::BQ;
    AttnParams p;
    memset(&p, 0, sizeof(p));
    p.Nq = nq; p.Nk = nk; p.heads = heads; p.d = d;
    p.n_kv_tiles = (nk + ATT_BKV - 1) / ATT_BKV;
    p.q_tiles = (nq + bq - 1) / bq;
    p.units = p.q_tiles * heads * batch;
    p.scale_log2e = (1.0f / sqrtf(static_cast<float>(d))) * 1.4426950408889634f;
    p.out = reinterpret_cast<__half*>(out); p.ldo = ldo; p.lse = lse;
    if (p.units == 0) return CTRLORA_OK;
    const int sms = persistent_sms();
    if (sms <= 0) return CTRLORA_ERR_CUDA;
    CUtensorMap tq, tk, tv;
    {
        uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)nq, (uint64_t)batch};
        uint64_t str[3] = {(uint64_t)d * 2, (uint64_t)ldq * 2, (uint64_t)ldq * 2 * nq};
        uint32_t box[4] = {64, 1, (uint32_t)bq, 1};
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
    const int grid = p.units < sms ? p.units : sms;
    if (dp == 48) return launch_attn<48>(tq, tk, tv, p, grid, stream);
    if (dp == 80) return launch_attn<80>(tq, tk, tv, p, grid, stream);
    return launch_attn<160>(tq, tk, tv, p, grid, stream);
}
