// GroupNorm(+SiLU) and LayerNorm for pixel-major fp16 activations (HBM-bound kernels; fp32 statistics).
//   GroupNorm32 -> SiLU before every ResBlock conv    reference: ldm/modules/diffusionmodules/openaimodel.py:190-197,
//                                                     221-231 with GroupNorm32 = fp32 statistics, util.py:202-219
//   GroupNorm(eps 1e-6) at the SpatialTransformer     reference: ldm/modules/attention.py:88-89,327
//   LayerNorm(eps 1e-5)                               reference: ldm/modules/attention.py:263-265,272-274
// The GroupNorm input may be the channel concatenation [x1 (+ s1*add1) | x2 (+ s2*add2)]: that is the UNet decoder's
// `cat([h, hs.pop() + control.pop()], 1)` (cldm/cldm.py:34-42) read in place — the concat and the ControlNet residual
// adds never make a round trip through HBM on their own.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

struct GnSrc {
    const __half* x1; const __half* add1; float s1; int c1; long long ld1;
    const __half* x2; const __half* add2; float s2; int c2; long long ld2;
};

__device__ __forceinline__ void load8(const GnSrc& s, long long pix, int c, float* v) {
    // c is a multiple of 8; c1 is a multiple of 8, so a vector never straddles the two sources
    const __half* x; const __half* ad; float sc; long long off;
    if (c < s.c1) { x = s.x1; ad = s.add1; sc = s.s1; off = pix * s.ld1 + c; }
    else { x = s.x2; ad = s.add2; sc = s.s2; off = pix * s.ld2 + (c - s.c1); }
    uint4 u = *reinterpret_cast<const uint4*>(x + off);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { float2 f = __half22float2(h[e]); v[2 * e] = f.x; v[2 * e + 1] = f.y; }
    if (ad) {
        uint4 w = *reinterpret_cast<const uint4*>(ad + off);
        const __half2* g = reinterpret_cast<const __half2*>(&w);
#pragma unroll
        for (int e = 0; e < 4; ++e) { float2 f = __half22float2(g[e]); v[2 * e] += sc * f.x; v[2 * e + 1] += sc * f.y; }
    }
}

// Statistics of the two-pass pair (gn_stats_det_kernel + gn_apply_kernel), deterministic: per-thread partials are reduced
// through shared memory in a fixed order, every block stores its per-group partial {sum, sumsq} (no atomics), and the LAST
// block of an image to arrive (one self-cleaning counter per image) adds the partials up in block order and writes the totals.
__global__ void __launch_bounds__(512)
gn_stats_det_kernel(GnSrc s, int C, int HW, int groups, int pix_per_block, float* __restrict__ stats, float* __restrict__ partial,
                    unsigned int* __restrict__ counters) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sm[];  // [lanes][2][C] scratch, then [2][C] channel sums
    __shared__ int is_last;
    const int b = blockIdx.y;
    const int vecs = C >> 3;
    const int lanes = blockDim.x / vecs;  // blockDim.x == vecs * lanes exactly
    const int vec = threadIdx.x % vecs, pl = threadIdx.x / vecs;
    float* csum = sm + static_cast<size_t>(lanes) * 2 * C;
    const int p0 = blockIdx.x * pix_per_block;
    const int p1 = min(HW, p0 + pix_per_block);
    float a[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { a[e] = 0.f; q[e] = 0.f; }
    int p = p0 + pl;
    for (; p + 3 * lanes < p1; p += 4 * lanes) {
        float v[4][8];
#pragma unroll
        for (int u = 0; u < 4; ++u) load8(s, static_cast<long long>(b) * HW + p + u * lanes, vec * 8, v[u]);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
#pragma unroll
            for (int e = 0; e < 8; ++e) { a[e] += v[u][e]; q[e] += v[u][e] * v[u][e]; }
        }
    }
    for (; p < p1; p += lanes) {
        float v[8];
        load8(s, static_cast<long long>(b) * HW + p, vec * 8, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) { a[e] += v[e]; q[e] += v[e] * v[e]; }
    }
    float* sp = sm + static_cast<size_t>(pl) * 2 * C + vec * 8;
    *reinterpret_cast<float4*>(sp) = make_float4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<float4*>(sp + 4) = make_float4(a[4], a[5], a[6], a[7]);
    *reinterpret_cast<float4*>(sp + C) = make_float4(q[0], q[1], q[2], q[3]);
    *reinterpret_cast<float4*>(sp + C + 4) = make_float4(q[4], q[5], q[6], q[7]);
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
        float t = 0.f;
        for (int l = 0; l < lanes; ++l) t += sm[static_cast<size_t>(l) * 2 * C + i];
        csum[i] = t;
    }
    __syncthreads();
    const int cpg = C / groups;
    const int nblk = gridDim.x;
    float* mine = partial + (static_cast<size_t>(b) * nblk + blockIdx.x) * groups * 2;
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
        float su = 0.f, sq = 0.f;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) { su += csum[c]; sq += csum[C + c]; }
        mine[2 * g] = su;
        mine[2 * g + 1] = sq;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int old = atomicAdd(&counters[b], 1u);
        is_last = (old == static_cast<unsigned int>(nblk - 1));
        if (is_last) counters[b] = 0;  // self-cleaning: ready for the next launch
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) {
        float t = 0.f;
        const float* src = partial + static_cast<size_t>(b) * nblk * groups * 2 + i;
        for (int k = 0; k < nblk; ++k) t += __ldcg(src + static_cast<size_t>(k) * groups * 2);  // block order: fixed
        stats[b * groups * 2 + i] = t;
    }
}

__global__ void __launch_bounds__(512, 2)  // <= 64 registers: four 240..256-thread blocks per SM, the whole grid in one wave
gn_apply_kernel(GnSrc s, int C, int HW, int groups, int pix_per_block, const float* __restrict__ stats,
                const float* __restrict__ gamma_lo, const float* __restrict__ beta_lo, const float* __restrict__ gamma_hi,
                const float* __restrict__ beta_hi, int group_b, float eps, int silu, __half* __restrict__ y,
                __half* __restrict__ raw) {
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.y;
    const bool hi = group_b > 0 && b >= group_b;  // grouped launch: the second network's affine parameters
    const float* __restrict__ gamma = hi ? gamma_hi : gamma_lo;
    const float* __restrict__ beta = hi ? beta_hi : beta_lo;
    const int vecs = C >> 3;
    const int lanes = blockDim.x / vecs;
    const int vec = threadIdx.x % vecs, pl = threadIdx.x / vecs;
    if (pl >= lanes) return;
    const int cpg = C / groups;
    const float inv_n = 1.0f / (static_cast<float>(cpg) * HW);
    float sc[8], sh[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int c = vec * 8 + e;
        const int g = c / cpg;
        const float mean = stats[(b * groups + g) * 2] * inv_n;
        const float var = fmaxf(stats[(b * groups + g) * 2 + 1] * inv_n - mean * mean, 0.f);
        const float rstd = rsqrtf(var + eps);
        sc[e] = rstd * gamma[c];
        sh[e] = beta[c] - mean * sc[e];
    }
    const int p0 = blockIdx.x * pix_per_block;
    const int p1 = min(HW, p0 + pix_per_block);
    auto emit = [&](long long pix, float* v) {
        if (raw) {
            uint4 u;
            __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
            *reinterpret_cast<uint4*>(raw + pix * C + vec * 8) = u;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float t = v[e] * sc[e] + sh[e];
            v[e] = silu ? silu_f(t) : t;
        }
        uint4 u;
        __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
        *reinterpret_cast<uint4*>(y + pix * C + vec * 8) = u;
    };
    int p = p0 + pl;
    for (; p + lanes < p1; p += 2 * lanes) {  // two vectors in flight per thread, four blocks per SM
        float v[2][8];
#pragma unroll
        for (int u = 0; u < 2; ++u) load8(s, static_cast<long long>(b) * HW + p + u * lanes, vec * 8, v[u]);
#pragma unroll
        for (int u = 0; u < 2; ++u) emit(static_cast<long long>(b) * HW + p + u * lanes, v[u]);
    }
    for (; p < p1; p += lanes) {
        float v[8];
        load8(s, static_cast<long long>(b) * HW + p, vec * 8, v);
        emit(static_cast<long long>(b) * HW + p, v);
    }
}

// ---- single-pass GroupNorm on a thread-block CLUSTER: the image's activations are read from HBM/L2 ONCE, parked in the
// shared memory of the `cs` CTAs of a cluster (one cluster per image, each CTA holds HW/cs pixels x C channels, <= 200 KB),
// the per-group {sum, sumsq} partials are exchanged through distributed shared memory, and every CTA normalises its own
// slice out of shared memory.  Replaces the two-pass pair (gn_stats_det_kernel + gn_apply_kernel: two launches, the tensor
// read twice) wherever the slice fits -- every GroupNorm of the 512x512 path except the decoder's widest concat inputs.
__device__ __forceinline__ float ld_dsmem_f32(const float* local_ptr, uint32_t cta_rank) {
    uint32_t remote;
    float v;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_ptr)), "r"(cta_rank));
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
    return v;
}

__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// BULK: the slice of this CTA is one contiguous block of global memory (single source, no addend, dense rows): it is
// brought in by the TMA engine (cp.async.bulk, 32 KiB pieces on one mbarrier) with no registers in the way; otherwise (the
// UNet decoder's `cat([h, hs.pop() + control.pop()])` inputs) the threads gather it with 16-byte loads, four in flight each.
// Determinism: no atomics anywhere -- per-thread partials go through a shared scratch array and are summed in a fixed order,
// CTA partials are summed in rank order -- so a forward pass is bit-reproducible.  (With fp16 storage this matters more than
// it sounds: a 1e-7 perturbation of one statistic flips a few fp16 roundings, and every following rounding stage amplifies
// the difference towards the rounding-noise level itself; fp32 atomics in the statistics made two identical SD1.5
// passes differ by 1.6e-3, tools/debug_determinism.py.)
template <int MODE>  // 0: register-gathered tile, 1: TMA bulk-staged tile
__global__ void __launch_bounds__(512, 1)
gn_cluster_kernel(GnSrc s, int C, int HW, int groups, int ppc, int cs, const float* __restrict__ gamma_lo,
                  const float* __restrict__ beta_lo, const float* __restrict__ gamma_hi, const float* __restrict__ beta_hi,
                  int group_b, float eps, int silu, __half* __restrict__ y, __half* __restrict__ raw,
                  float* __restrict__ stats_out) {
    constexpr bool BULK = MODE == 1;
    pdl_launch_dependents();
    extern __shared__ __align__(128) uint8_t gsm[];
    __half* tile = reinterpret_cast<__half*>(gsm);                                    // [ppc][C]
    float* scratch = reinterpret_cast<float*>(gsm + static_cast<size_t>(ppc) * C * 2);  // [lanes][2][C]
    float* csum = scratch + static_cast<size_t>(blockDim.x / (C >> 3)) * 2 * C;      // [2][C]: per-channel sum, sumsq
    float* part = csum + 2 * C;                                                       // [groups][2]: this CTA's group partials
    float* mr = part + 2 * groups;                                                    // [groups][2]: mean, rstd
    uint64_t* bar = reinterpret_cast<uint64_t*>(mr + 2 * groups);
    const int b = blockIdx.y;
    const uint32_t rank = cluster_ctarank();
    const int vecs = C >> 3;
    const int lanes = blockDim.x / vecs;
    const int vec = threadIdx.x % vecs, pl = threadIdx.x / vecs;
    const int p0 = static_cast<int>(rank) * ppc, p1 = min(HW, p0 + ppc);
    const int npix = max(p1 - p0, 0);
    if (BULK && threadIdx.x == 0) {
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    float a[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { a[e] = 0.f; q[e] = 0.f; }
    if (BULK) {
        const uint32_t total = static_cast<uint32_t>(npix) * C * 2;  // multiple of 16
        if (threadIdx.x == 0 && total > 0) {
            mbar_expect_tx(bar, total);
            const uint8_t* src = reinterpret_cast<const uint8_t*>(s.x1 + (static_cast<long long>(b) * HW + p0) * C);
            for (uint32_t off = 0; off < total; off += 32768u)
                bulk_g2s(gsm + off, src + off, min(32768u, total - off), bar);
        }
        if (total > 0) mbar_wait(bar, 0);
        if (pl < lanes) {
            for (int p = pl; p < npix; p += lanes) {
                const uint4 w = *reinterpret_cast<const uint4*>(tile + static_cast<size_t>(p) * C + vec * 8);
                const __half2* h = reinterpret_cast<const __half2*>(&w);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(h[e]);
                    a[2 * e] += f.x; q[2 * e] += f.x * f.x;
                    a[2 * e + 1] += f.y; q[2 * e + 1] += f.y * f.y;
                }
            }
        }
    } else if (pl < lanes) {
        int p = pl;
        for (; p + 3 * lanes < npix; p += 4 * lanes) {  // four 16-byte loads (eight with an addend) in flight per thread
            float v[4][8];
#pragma unroll
            for (int u = 0; u < 4; ++u) load8(s, static_cast<long long>(b) * HW + p0 + p + u * lanes, vec * 8, v[u]);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                uint4 w;
                __half2* h = reinterpret_cast<__half2*>(&w);
#pragma unroll
                for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[u][2 * e], v[u][2 * e + 1]);
                *reinterpret_cast<uint4*>(tile + static_cast<size_t>(p + u * lanes) * C + vec * 8) = w;
#pragma unroll
                for (int e = 0; e < 8; ++e) { a[e] += v[u][e]; q[e] += v[u][e] * v[u][e]; }
            }
        }
        for (; p < npix; p += lanes) {
            float v[8];
            load8(s, static_cast<long long>(b) * HW + p0 + p, vec * 8, v);
            uint4 w;
            __half2* h = reinterpret_cast<__half2*>(&w);
#pragma unroll
            for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
            *reinterpret_cast<uint4*>(tile + static_cast<size_t>(p) * C + vec * 8) = w;
#pragma unroll
            for (int e = 0; e < 8; ++e) { a[e] += v[e]; q[e] += v[e] * v[e]; }
        }
    }
    if (pl < lanes) {  // fixed-order reduction over the pixel lanes (no atomics: bit-reproducible statistics)
        float* sp = scratch + static_cast<size_t>(pl) * 2 * C + vec * 8;
        *reinterpret_cast<float4*>(sp) = make_float4(a[0], a[1], a[2], a[3]);
        *reinterpret_cast<float4*>(sp + 4) = make_float4(a[4], a[5], a[6], a[7]);
        *reinterpret_cast<float4*>(sp + C) = make_float4(q[0], q[1], q[2], q[3]);
        *reinterpret_cast<float4*>(sp + C + 4) = make_float4(q[4], q[5], q[6], q[7]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
        float t = 0.f;
        for (int l = 0; l < lanes; ++l) t += scratch[static_cast<size_t>(l) * 2 * C + i];
        csum[i] = t;
    }
    __syncthreads();
    const int cpg = C / groups;
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) {  // one thread per (group, statistic), fixed channel order
        const int g = i >> 1, which = i & 1;
        float t = 0.f;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) t += csum[which * C + c];
        part[i] = t;
    }
    cluster_sync_all();  // every CTA's partials are visible cluster-wide (release / acquire)
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
        // all remote loads are issued before the first add (a dependent load -> add chain would serialise ~0.7 us of
        // DSMEM latency per CTA of the cluster); the adds run in rank order: every CTA gets bit-identical statistics
        float rs[16], rq[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            rs[r] = r < cs ? ld_dsmem_f32(part + 2 * g, r) : 0.f;
            rq[r] = r < cs ? ld_dsmem_f32(part + 2 * g + 1, r) : 0.f;
        }
        float su = 0.f, sq = 0.f;
#pragma unroll
        for (int r = 0; r < 16; ++r) { su += rs[r]; sq += rq[r]; }
        const float inv_n = 1.0f / (static_cast<float>(cpg) * HW);
        const float mean = su * inv_n;
        const float var = fmaxf(sq * inv_n - mean * mean, 0.f);
        mr[2 * g] = mean;
        mr[2 * g + 1] = rsqrtf(var + eps);
        if (rank == 0 && stats_out) {  // {sum, sumsq}: what the backward kernels expect from the forward
            stats_out[(b * groups + g) * 2] = su;
            stats_out[(b * groups + g) * 2 + 1] = sq;
        }
    }
    cluster_sync_all();  // remote reads of this CTA's partials are done (it may exit); mr[] visible to the whole block
    if (pl >= lanes) return;
    const bool hi = group_b > 0 && b >= group_b;  // grouped launch: the second network's affine parameters
    const float* __restrict__ gamma = hi ? gamma_hi : gamma_lo;
    const float* __restrict__ beta = hi ? beta_hi : beta_lo;
    float sc[8], sh[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int c = vec * 8 + e, g = c / cpg;
        sc[e] = mr[2 * g + 1] * gamma[c];
        sh[e] = beta[c] - mr[2 * g] * sc[e];
    }
    for (int p = pl; p < npix; p += lanes) {
        const long long pix = static_cast<long long>(b) * HW + p0 + p;
        const uint4 w = *reinterpret_cast<const uint4*>(tile + static_cast<size_t>(p) * C + vec * 8);
        if (raw) *reinterpret_cast<uint4*>(raw + pix * C + vec * 8) = w;
        const __half2* h = reinterpret_cast<const __half2*>(&w);
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h[e]);
            float t0 = f.x * sc[2 * e] + sh[2 * e], t1 = f.y * sc[2 * e + 1] + sh[2 * e + 1];
            if (silu) { t0 = silu_f(t0); t1 = silu_f(t1); }
            oh[e] = __floats2half2_rn(t0, t1);
        }
        *reinterpret_cast<uint4*>(y + pix * C + vec * 8) = o;
    }
}

// one warp per row; the row stays in registers between the mean and variance passes (C <= 2048)
template <int MAXV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy, int M, int C,
                 const float* __restrict__ gamma_lo, const float* __restrict__ beta_lo, const float* __restrict__ gamma_hi,
                 const float* __restrict__ beta_hi, int split_rows, float eps) {
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= M) return;
    const float* __restrict__ gamma = row >= split_rows ? gamma_hi : gamma_lo;
    const float* __restrict__ beta = row >= split_rows ? beta_hi : beta_lo;
    const int vecs = C >> 3;
    float v[MAXV][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vi = lane + i * 32;
        if (vi < vecs) {
            uint4 u = *reinterpret_cast<const uint4*>(x + row * ldx + vi * 8);
            const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) { float2 f = __half22float2(h[e]); v[i][2 * e] = f.x; v[i][2 * e + 1] = f.y; }
#pragma unroll
            for (int e = 0; e < 8; ++e) sum += v[i][e];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / C;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        if (lane + i * 32 < vecs) {
#pragma unroll
            for (int e = 0; e < 8; ++e) { const float d = v[i][e] - mean; sq += d * d; }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq / C + eps);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int vi = lane + i * 32;
        if (vi < vecs) {
            float4 g0 = *reinterpret_cast<const float4*>(gamma + vi * 8), g1 = *reinterpret_cast<const float4*>(gamma + vi * 8 + 4);
            float4 b0 = *reinterpret_cast<const float4*>(beta + vi * 8), b1 = *reinterpret_cast<const float4*>(beta + vi * 8 + 4);
            const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            uint4 u;
            __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e)
                h[e] = __floats2half2_rn((v[i][2 * e] - mean) * rstd * g[2 * e] + bb[2 * e],
                                         (v[i][2 * e + 1] - mean) * rstd * g[2 * e + 1] + bb[2 * e + 1]);
            *reinterpret_cast<uint4*>(y + row * ldy + vi * 8) = u;
        }
    }
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_groupnorm_f16(const ctrlora_groupnorm_args* a, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || !a->x1 || !a->y || !a->stats_ws || !a->gamma || !a->beta) return CTRLORA_ERR_ARG;
    if (a->group_b < 0 || a->group_b >= a->batch || (a->group_b > 0 && (!a->gamma_hi || !a->beta_hi))) return CTRLORA_ERR_ARG;
    const float* gamma_hi = a->group_b > 0 ? a->gamma_hi : a->gamma;
    const float* beta_hi = a->group_b > 0 ? a->beta_hi : a->beta;
    const int C = a->c1 + (a->x2 ? a->c2 : 0);
    if (C % 8 != 0 || a->c1 % 8 != 0 || C % a->groups != 0 || C / 8 > 512) return CTRLORA_ERR_ARG;
    if (a->ld1 % 8 != 0 || (a->x2 && a->ld2 % 8 != 0)) return CTRLORA_ERR_ARG;
    GnSrc s;
    s.x1 = reinterpret_cast<const __half*>(a->x1); s.add1 = reinterpret_cast<const __half*>(a->add1); s.s1 = a->add1_scale;
    s.c1 = a->c1; s.ld1 = a->ld1;
    s.x2 = reinterpret_cast<const __half*>(a->x2); s.add2 = reinterpret_cast<const __half*>(a->add2); s.s2 = a->add2_scale;
    s.c2 = a->x2 ? a->c2 : 0; s.ld2 = a->ld2;
    const int HW = a->hw, B = a->batch;
    // two-pass geometry: ~4 blocks per SM in total, at least 8 pixels per block; a grouped launch splits each image as a
    // call over the larger group would, so that its statistics are summed in the same order
    const int B_split = a->group_b > 0 ? (a->group_b > B - a->group_b ? a->group_b : B - a->group_b) : B;
    int chunks = (592 + B_split - 1) / B_split;
    int ppb = (HW + chunks - 1) / chunks;
    if (ppb < 8) ppb = 8;
    chunks = (HW + ppb - 1) / ppb;
    if (!a->partial_ws || !a->partial_counters || B > a->partial_counters_len ||
        static_cast<long long>(B) * chunks * a->groups * 2 > a->partial_ws_floats)
        return CTRLORA_ERR_ARG;
    // ---- single-pass cluster kernel where one image's slice fits the shared memory of 1, 2, 4 or 8 CTAs
    {
        const int vecs = C / 8;
        const int lanes_max = vecs <= 512 ? 512 / vecs : 0;
        auto fixed_for = [&](int lanes) {  // scratch [lanes][2C] + csum [2C] + part/mr [4 groups] + the staging mbarrier
            return static_cast<size_t>((lanes + 1) * 2 * C + 4 * a->groups) * sizeof(float) + 16;
        };
        const size_t budget = 216 * 1024;
        int cs = 0;
        for (int c = 1; c <= 8 && lanes_max > 0; c *= 2) {  // 16-CTA clusters measured slower than the two-pass pair
            const int ppc = (HW + c - 1) / c;
            if (c > HW) break;
            const int lanes = lanes_max < ppc ? lanes_max : ppc;
            if (static_cast<size_t>(ppc) * C * 2 + fixed_for(lanes) <= budget) { cs = c; break; }
        }
        if (cs > 0) {
            const int ppc = (HW + cs - 1) / cs;
            int lanes = lanes_max;
            if (lanes > ppc) lanes = ppc;
            if (lanes < 1) lanes = 1;
            const size_t fixed = fixed_for(lanes);
            const int threads = vecs * lanes;  // exact: the scratch layout is indexed by blockDim.x / vecs
            // contiguous slice -> TMA bulk staging (needs 16-byte aligned base, dense rows)
            const bool bulk = !a->x2 && !a->add1 && a->ld1 == C && (reinterpret_cast<uintptr_t>(a->x1) & 15) == 0;
            const size_t smem = static_cast<size_t>(ppc) * C * 2 + fixed;
            static bool attr = false;
            if (!attr) {
                if (cudaFuncSetAttribute(gn_cluster_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess ||
                    cudaFuncSetAttribute(gn_cluster_kernel<0>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
                    cudaFuncSetAttribute(gn_cluster_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess ||
                    cudaFuncSetAttribute(gn_cluster_kernel<1>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess)
                    return CTRLORA_ERR_CUDA;
                attr = true;
            }
            const cudaError_t rc = launch_cluster_pdl(bulk ? gn_cluster_kernel<1> : gn_cluster_kernel<0>, dim3(cs, B),
                                                      dim3(threads), smem, stream, (unsigned)cs, s, C, HW, (int)a->groups, ppc, cs,
                                                      a->gamma, a->beta, gamma_hi, beta_hi, (int)a->group_b, a->eps,
                                                      (int)a->silu, reinterpret_cast<__half*>(a->y),
                                                      reinterpret_cast<__half*>(a->raw_out), reinterpret_cast<float*>(a->stats_ws));
            if (rc == cudaSuccess) return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
            (void)cudaGetLastError();  // fall through to the two-pass pair
        }
    }
    dim3 grid(chunks, B);
    const int vecs = C / 8;
    const int lanes = vecs >= 256 ? 1 : 256 / vecs;
    const int threads = vecs * lanes;  // every thread owns one 8-channel vector of one pixel lane
    static bool det_attr = false;  // (lanes + 1) * 2 * C floats: up to 64 KB (C = 4096, one lane), over the default 48 KB
    if (!det_attr) {
        if (cudaFuncSetAttribute(gn_stats_det_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024) != cudaSuccess)
            return CTRLORA_ERR_CUDA;
        det_attr = true;
    }
    launch_pdl(gn_stats_det_kernel, grid, dim3(threads), (size_t)((lanes + 1) * 2 * C * sizeof(float)), stream, s, C, HW,
               (int)a->groups, ppb, reinterpret_cast<float*>(a->stats_ws), a->partial_ws, a->partial_counters);
    launch_pdl(gn_apply_kernel, grid, dim3(threads), (size_t)0, stream, s, C, HW, (int)a->groups, ppb,
               reinterpret_cast<const float*>(a->stats_ws), a->gamma, a->beta, gamma_hi, beta_hi, (int)a->group_b, a->eps,
               (int)a->silu, reinterpret_cast<__half*>(a->y), reinterpret_cast<__half*>(a->raw_out));
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}

extern "C" int ctrlora_layernorm_grouped_f16(const void* x, long long ldx, void* y, long long ldy, int rows, int cols,
                                             const float* gamma, const float* beta, const float* gamma_hi,
                                             const float* beta_hi, int split_rows, float eps, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !y || cols % 8 != 0 || cols > 2048 || ldx % 8 != 0 || ldy % 8 != 0) return CTRLORA_ERR_ARG;
    if (split_rows < 0 || (split_rows < rows && (!gamma_hi || !beta_hi))) return CTRLORA_ERR_ARG;
    const int grid = (rows + 7) / 8;
    const __half* xp = reinterpret_cast<const __half*>(x);
    __half* yp = reinterpret_cast<__half*>(y);
    const float* gh = split_rows < rows ? gamma_hi : gamma;
    const float* bh = split_rows < rows ? beta_hi : beta;
    if (cols <= 512) launch_pdl(layernorm_kernel<2>, dim3(grid), dim3(256), (size_t)0, stream, xp, ldx, yp, ldy, rows, cols, gamma, beta, gh, bh, split_rows, eps);
    else if (cols <= 768) launch_pdl(layernorm_kernel<3>, dim3(grid), dim3(256), (size_t)0, stream, xp, ldx, yp, ldy, rows, cols, gamma, beta, gh, bh, split_rows, eps);
    else if (cols <= 1280) launch_pdl(layernorm_kernel<5>, dim3(grid), dim3(256), (size_t)0, stream, xp, ldx, yp, ldy, rows, cols, gamma, beta, gh, bh, split_rows, eps);
    else launch_pdl(layernorm_kernel<8>, dim3(grid), dim3(256), (size_t)0, stream, xp, ldx, yp, ldy, rows, cols, gamma, beta, gh, bh, split_rows, eps);
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}

extern "C" int ctrlora_layernorm_f16(const void* x, long long ldx, void* y, long long ldy, int rows, int cols,
                                     const float* gamma, const float* beta, float eps, void* stream) {
    return ctrlora_layernorm_grouped_f16(x, ldx, y, ldy, rows, cols, gamma, beta, nullptr, nullptr, rows, eps, stream);
}

// ================================================================================================ backward (training)
// GroupNorm(+SiLU) backward.  Forward: z = xhat * gamma + beta, y = silu(z) (or z); xhat = (x - mu) * rstd per (image,
// group).  With dz = dy * silu'(z):  dx = rstd * (dz*gamma - mean_g(dz*gamma) - xhat * mean_g(dz*gamma*xhat)),
// dgamma_c = sum dz*xhat, dbeta_c = sum dz.  x is re-read through the same (concat, addend) source description as the
// forward; mu/rstd come from the forward's saved {sum, sumsq}.
namespace ctrl {

__device__ __forceinline__ float dsilu_f(float z) {
    const float s = sigmoid_f(z);
    return s * (1.0f + z * (1.0f - s));
}

__device__ __forceinline__ void load8h(const __half* p, float* v) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) { float2 f = __half22float2(h[e]); v[2 * e] = f.x; v[2 * e + 1] = f.y; }
}

// bstats[b][g] = {sum dz*gamma, sum dz*gamma*xhat}, the backward twin of gn_stats_det_kernel: per-lane channel sums reduced through shared memory in lane order, one per-group partial per block
// (no atomics), and the last block of an image to arrive adds the partials up in block order.  bstats -- and with them every
// dx the apply kernel writes -- are then bit-reproducible; dgamma/dbeta still accumulate with fp32 atomics (one per
// channel per block): they feed only the fp32 gradient buffer, never an fp16 activation.
__global__ void __launch_bounds__(512)
gn_bwd_stats_det_kernel(GnSrc s, const __half* __restrict__ dy, int C, int HW, int groups, int pix_per_block,
                        const float* __restrict__ fstats, const float* __restrict__ gamma, const float* __restrict__ beta,
                        float eps, int silu, float* __restrict__ bstats, float* __restrict__ dgamma, float* __restrict__ dbeta,
                        float* __restrict__ partial, unsigned int* __restrict__ counters) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sm[];  // [lanes][2][C] scratch, then [2][C] channel sums (dz, dz*xhat)
    __shared__ int is_last;
    const int b = blockIdx.y;
    const int vecs = C >> 3, lanes = blockDim.x / vecs;  // blockDim.x == vecs * lanes exactly
    const int vec = threadIdx.x % vecs, pl = threadIdx.x / vecs;
    float* c_dz = sm + static_cast<size_t>(lanes) * 2 * C;
    float* c_dzx = c_dz + C;
    const int cpg = C / groups;
    const float inv_n = 1.0f / (static_cast<float>(cpg) * HW);
    float mu[8], rs[8], ga[8], be[8], a[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int c = vec * 8 + e, g = c / cpg;
        const float mean = fstats[(b * groups + g) * 2] * inv_n;
        const float var = fmaxf(fstats[(b * groups + g) * 2 + 1] * inv_n - mean * mean, 0.f);
        mu[e] = mean; rs[e] = rsqrtf(var + eps); ga[e] = gamma[c]; be[e] = beta[c]; a[e] = 0.f; q[e] = 0.f;
    }
    const int p0 = blockIdx.x * pix_per_block, p1 = min(HW, p0 + pix_per_block);
    auto accum = [&](const float* x, const float* d) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float xh = (x[e] - mu[e]) * rs[e];
            const float dz = silu ? d[e] * dsilu_f(xh * ga[e] + be[e]) : d[e];
            a[e] += dz; q[e] += dz * xh;
        }
    };
    int p = p0 + pl;
    for (; p + lanes < p1; p += 2 * lanes) {  // two pixels (four 16-byte loads) in flight per thread
        const long long pix = static_cast<long long>(b) * HW + p;
        float x0[8], d0[8], x1[8], d1[8];
        load8(s, pix, vec * 8, x0);
        load8h(dy + pix * C + vec * 8, d0);
        load8(s, pix + lanes, vec * 8, x1);
        load8h(dy + (pix + lanes) * C + vec * 8, d1);
        accum(x0, d0);
        accum(x1, d1);
    }
    for (; p < p1; p += lanes) {
        const long long pix = static_cast<long long>(b) * HW + p;
        float x[8], d[8];
        load8(s, pix, vec * 8, x);
        load8h(dy + pix * C + vec * 8, d);
        accum(x, d);
    }
    float* sp = sm + static_cast<size_t>(pl) * 2 * C + vec * 8;
    *reinterpret_cast<float4*>(sp) = make_float4(a[0], a[1], a[2], a[3]);
    *reinterpret_cast<float4*>(sp + 4) = make_float4(a[4], a[5], a[6], a[7]);
    *reinterpret_cast<float4*>(sp + C) = make_float4(q[0], q[1], q[2], q[3]);
    *reinterpret_cast<float4*>(sp + C + 4) = make_float4(q[4], q[5], q[6], q[7]);
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
        float t = 0.f;
        for (int l = 0; l < lanes; ++l) t += sm[static_cast<size_t>(l) * 2 * C + i];
        c_dz[i] = t;  // i >= C lands in c_dzx
    }
    __syncthreads();
    const int nblk = gridDim.x;
    float* mine = partial + (static_cast<size_t>(b) * nblk + blockIdx.x) * groups * 2;
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
        float g1 = 0.f, g2 = 0.f;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) { g1 += gamma[c] * c_dz[c]; g2 += gamma[c] * c_dzx[c]; }
        mine[2 * g] = g1;
        mine[2 * g + 1] = g2;
    }
    if (dgamma) {
        for (int c = threadIdx.x; c < C; c += blockDim.x) { atomicAdd(&dgamma[c], c_dzx[c]); atomicAdd(&dbeta[c], c_dz[c]); }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int old = atomicAdd(&counters[b], 1u);
        is_last = (old == static_cast<unsigned int>(nblk - 1));
        if (is_last) counters[b] = 0;  // self-cleaning: ready for the next launch
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) {
        float t = 0.f;
        const float* src = partial + static_cast<size_t>(b) * nblk * groups * 2 + i;
        for (int k = 0; k < nblk; ++k) t += __ldcg(src + static_cast<size_t>(k) * groups * 2);  // block order: fixed
        bstats[b * groups * 2 + i] = t;
    }
}

__global__ void __launch_bounds__(512)
gn_bwd_apply_kernel(GnSrc s, const __half* __restrict__ dy, int C, int HW, int groups, int pix_per_block,
                    const float* __restrict__ fstats, const float* __restrict__ bstats, const float* __restrict__ gamma,
                    const float* __restrict__ beta, float eps, int silu, __half* __restrict__ dx1, long long ldd1, float scale1,
                    __half* __restrict__ dx2, long long ldd2, float scale2, const __half* __restrict__ res, long long ldres) {
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.y;
    const int vecs = C >> 3, lanes = blockDim.x / vecs;
    const int vec = threadIdx.x % vecs, pl = threadIdx.x / vecs;
    if (pl >= lanes) return;
    const int cpg = C / groups;
    const float inv_n = 1.0f / (static_cast<float>(cpg) * HW);
    float mu[8], rs[8], ga[8], be[8], m1[8], m2[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const int c = vec * 8 + e, g = c / cpg;
        const float mean = fstats[(b * groups + g) * 2] * inv_n;
        const float var = fmaxf(fstats[(b * groups + g) * 2 + 1] * inv_n - mean * mean, 0.f);
        mu[e] = mean; rs[e] = rsqrtf(var + eps); ga[e] = gamma[c]; be[e] = beta[c];
        m1[e] = bstats[(b * groups + g) * 2] * inv_n; m2[e] = bstats[(b * groups + g) * 2 + 1] * inv_n;
    }
    const bool first = vec * 8 < s.c1;
    __half* dst = first ? dx1 : dx2;
    if (!dst) return;
    const long long ldd = first ? ldd1 : ldd2;
    const int coff = first ? vec * 8 : vec * 8 - s.c1;
    const float osc = first ? scale1 : scale2;
    const int p0 = blockIdx.x * pix_per_block, p1 = min(HW, p0 + pix_per_block);
    auto one = [&](long long pix, const float* x, const float* d, const float* rr) {
        uint4 u;
        __half2* h = reinterpret_cast<__half2*>(&u);
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float xh = (x[e] - mu[e]) * rs[e];
            const float dz = silu ? d[e] * dsilu_f(xh * ga[e] + be[e]) : d[e];
            o[e] = (rs[e] * (dz * ga[e] - m1[e] - xh * m2[e]) + rr[e]) * osc;
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(o[2 * e], o[2 * e + 1]);
        *reinterpret_cast<uint4*>(dst + pix * ldd + coff) = u;
    };
    int p = p0 + pl;
    for (; p + lanes < p1; p += 2 * lanes) {  // two pixels in flight per thread
        const long long pix = static_cast<long long>(b) * HW + p;
        float x0[8], d0[8], x1[8], d1[8];
        float r0[8] = {0, 0, 0, 0, 0, 0, 0, 0}, r1[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        load8(s, pix, vec * 8, x0);
        load8h(dy + pix * C + vec * 8, d0);
        load8(s, pix + lanes, vec * 8, x1);
        load8h(dy + (pix + lanes) * C + vec * 8, d1);
        if (res) {  // gradient arriving over the block's skip path (identity residual or the 1x1 skip conv's dgrad)
            load8h(res + pix * ldres + vec * 8, r0);
            load8h(res + (pix + lanes) * ldres + vec * 8, r1);
        }
        one(pix, x0, d0, r0);
        one(pix + lanes, x1, d1, r1);
    }
    for (; p < p1; p += lanes) {
        const long long pix = static_cast<long long>(b) * HW + p;
        float x[8], d[8];
        load8(s, pix, vec * 8, x);
        load8h(dy + pix * C + vec * 8, d);
        uint4 u;
        __half2* h = reinterpret_cast<__half2*>(&u);
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const float xh = (x[e] - mu[e]) * rs[e];
            const float dz = silu ? d[e] * dsilu_f(xh * ga[e] + be[e]) : d[e];
            o[e] = rs[e] * (dz * ga[e] - m1[e] - xh * m2[e]);
        }
        if (res) {  // gradient arriving over the block's skip path (identity residual or the 1x1 skip conv's dgrad)
            float rr[8];
            load8h(res + pix * ldres + vec * 8, rr);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] += rr[e];
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] *= osc;
#pragma unroll
        for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(o[2 * e], o[2 * e + 1]);
        *reinterpret_cast<uint4*>(dst + pix * ldd + coff) = u;
    }
}

// LayerNorm backward: one warp per row (grid-stride), dgamma/dbeta accumulated per lane then once per block.
// DG = false (frozen norms: the UNet's): no per-lane dgamma / dbeta accumulators -> ~80 fewer registers, 2-3x the occupancy
// of a kernel whose time is the per-row latency chain (load -> 3 warp reductions -> store).
template <int MAXV, bool DG>
__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const __half* __restrict__ x, long long ldx, const __half* __restrict__ dy, long long ldy,
                     __half* __restrict__ dx, long long lddx, int M, int C, const float* __restrict__ gamma, float eps,
                     float* __restrict__ dgamma, float* __restrict__ dbeta, const __half* __restrict__ res, long long ldres) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sm[];  // [2][C] when dgamma
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    const int vecs = C >> 3;
    float agam[DG ? MAXV : 1][8], abet[DG ? MAXV : 1][8];
#pragma unroll
    for (int i = 0; i < (DG ? MAXV : 1); ++i)
#pragma unroll
        for (int e = 0; e < 8; ++e) { agam[i][e] = 0.f; abet[i][e] = 0.f; }
    for (int row = blockIdx.x * wpb + warp; row < M; row += gridDim.x * wpb) {
        float v[MAXV][8], d[MAXV][8];
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int vi = lane + i * 32;
            if (vi < vecs) {
                load8h(x + row * ldx + vi * 8, v[i]);
                load8h(dy + row * ldy + vi * 8, d[i]);
#pragma unroll
                for (int e = 0; e < 8; ++e) sum += v[i][e];
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
                for (int e = 0; e < 8; ++e) { const float t = v[i][e] - mean; sq += t * t; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
        const float rstd = rsqrtf(sq / C + eps);
        float s1 = 0.f, s2 = 0.f;  // sum dz, sum dz*xhat with dz = dy*gamma
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int vi = lane + i * 32;
            if (vi < vecs) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const float xh = (v[i][e] - mean) * rstd;
                    const float dz = d[i][e] * gamma[vi * 8 + e];
                    s1 += dz; s2 += dz * xh;
                    if (DG) { agam[DG ? i : 0][e] += d[i][e] * xh; abet[DG ? i : 0][e] += d[i][e]; }
                    v[i][e] = xh; d[i][e] = dz;
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
        s1 /= C; s2 /= C;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int vi = lane + i * 32;
            if (vi < vecs) {
                float rr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                if (res) load8h(res + row * ldres + vi * 8, rr);  // gradient of the residual branch
                uint4 u;
                __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    h[e] = __floats2half2_rn(rstd * (d[i][2 * e] - s1 - v[i][2 * e] * s2) + rr[2 * e],
                                             rstd * (d[i][2 * e + 1] - s1 - v[i][2 * e + 1] * s2) + rr[2 * e + 1]);
                *reinterpret_cast<uint4*>(dx + row * lddx + vi * 8) = u;
            }
        }
    }
    if (DG && dgamma) {
        for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) sm[i] = 0.f;
        __syncthreads();
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int vi = lane + i * 32;
            if (vi < vecs)
#pragma unroll
                for (int e = 0; e < 8; ++e) { atomicAdd(&sm[vi * 8 + e], agam[DG ? i : 0][e]); atomicAdd(&sm[C + vi * 8 + e], abet[DG ? i : 0][e]); }
        }
        __syncthreads();
        for (int c = threadIdx.x; c < C; c += blockDim.x) { atomicAdd(&dgamma[c], sm[c]); atomicAdd(&dbeta[c], sm[C + c]); }
    }
}

}  // namespace ctrl

extern "C" int ctrlora_groupnorm_bwd_f16(const ctrlora_groupnorm_args* a, const void* dy, const void* fwd_stats, void* dx1,
                                         long long ldd1, float dx1_scale, void* dx2, long long ldd2, float dx2_scale,
                                         const void* res, long long ldres, float* dgamma, float* dbeta, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || !a->x1 || !dy || !fwd_stats || !a->stats_ws || !a->gamma || !a->beta) return CTRLORA_ERR_ARG;
    if (a->group_b != 0) return CTRLORA_ERR_UNSUPPORTED;
    const int C = a->c1 + (a->x2 ? a->c2 : 0);
    if (C % 8 != 0 || a->c1 % 8 != 0 || C % a->groups != 0 || C / 8 > 512) return CTRLORA_ERR_ARG;
    GnSrc s;
    s.x1 = reinterpret_cast<const __half*>(a->x1); s.add1 = reinterpret_cast<const __half*>(a->add1); s.s1 = a->add1_scale;
    s.c1 = a->c1; s.ld1 = a->ld1;
    s.x2 = reinterpret_cast<const __half*>(a->x2); s.add2 = reinterpret_cast<const __half*>(a->add2); s.s2 = a->add2_scale;
    s.c2 = a->x2 ? a->c2 : 0; s.ld2 = a->ld2;
    const int HW = a->hw, B = a->batch;
    int chunks = (592 + B - 1) / B;
    int ppb = (HW + chunks - 1) / chunks;
    if (ppb < 8) ppb = 8;
    chunks = (HW + ppb - 1) / ppb;
    dim3 grid(chunks, B);
    const int vecs = C / 8;
    const int lanes = vecs >= 256 ? 1 : 256 / vecs;
    const int threads = vecs * lanes;
    if (!a->partial_ws || !a->partial_counters || B > a->partial_counters_len ||
        static_cast<long long>(B) * chunks * a->groups * 2 > a->partial_ws_floats)
        return CTRLORA_ERR_ARG;
    static bool attr = false;  // (lanes + 1) * 2 * C floats: up to 64 KB (C = 4096, one lane), over the default 48 KB
    if (!attr) {
        if (cudaFuncSetAttribute(gn_bwd_stats_det_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024) != cudaSuccess)
            return CTRLORA_ERR_CUDA;
        attr = true;
    }
    launch_pdl(gn_bwd_stats_det_kernel, grid, dim3(threads), (size_t)((lanes + 1) * 2 * C * sizeof(float)), stream, s,
               reinterpret_cast<const __half*>(dy), C, HW, (int)a->groups, ppb, reinterpret_cast<const float*>(fwd_stats),
               a->gamma, a->beta, a->eps, (int)a->silu, reinterpret_cast<float*>(a->stats_ws), dgamma, dbeta,
               a->partial_ws, a->partial_counters);
    launch_pdl(gn_bwd_apply_kernel, grid, dim3(threads), (size_t)0, stream, s, reinterpret_cast<const __half*>(dy), C, HW,
               (int)a->groups, ppb, reinterpret_cast<const float*>(fwd_stats), reinterpret_cast<const float*>(a->stats_ws),
               a->gamma, a->beta, a->eps, (int)a->silu, reinterpret_cast<__half*>(dx1), ldd1, dx1_scale,
               reinterpret_cast<__half*>(dx2), ldd2, dx2_scale, reinterpret_cast<const __half*>(res), ldres);
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}

extern "C" int ctrlora_layernorm_bwd_f16(const void* x, long long ldx, const void* dy, long long ldy, void* dx, long long lddx,
                                         int rows, int cols, const float* gamma, float eps, float* dgamma, float* dbeta,
                                         const void* res, long long ldres, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !dy || !dx || !gamma || cols % 8 != 0 || cols > 1280 || (dgamma && !dbeta)) return CTRLORA_ERR_ARG;
    int grid = (rows + 7) / 8;
    const int cap = dgamma ? 592 : 1184;  // resident blocks: the accumulator-free variant fits twice as many
    if (grid > cap) grid = cap;
    const size_t sm = dgamma ? 2 * cols * sizeof(float) : 0;
    const __half* xp = reinterpret_cast<const __half*>(x);
    const __half* dp = reinterpret_cast<const __half*>(dy);
    __half* op = reinterpret_cast<__half*>(dx);
    const __half* rp = reinterpret_cast<const __half*>(res);
    if (cols <= 512) {
        if (dgamma) launch_pdl(layernorm_bwd_kernel<2, true>, dim3(grid), dim3(256), sm, stream, xp, ldx, dp, ldy, op, lddx, rows, cols, gamma, eps, dgamma, dbeta, rp, ldres);
        else launch_pdl(layernorm_bwd_kernel<2, false>, dim3(grid), dim3(256), sm, stream, xp, ldx, dp, ldy, op, lddx, rows, cols, gamma, eps, dgamma, dbeta, rp, ldres);
    } else if (cols <= 768) {
        if (dgamma) launch_pdl(layernorm_bwd_kernel<3, true>, dim3(grid), dim3(256), sm, stream, xp, ldx, dp, ldy, op, lddx, rows, cols, gamma, eps, dgamma, dbeta, rp, ldres);
        else launch_pdl(layernorm_bwd_kernel<3, false>, dim3(grid), dim3(256), sm, stream, xp, ldx, dp, ldy, op, lddx, rows, cols, gamma, eps, dgamma, dbeta, rp, ldres);
    } else {
        if (dgamma) launch_pdl(layernorm_bwd_kernel<5, true>, dim3(grid), dim3(256), sm, stream, xp, ldx, dp, ldy, op, lddx, rows, cols, gamma, eps, dgamma, dbeta, rp, ldres);
        else launch_pdl(layernorm_bwd_kernel<5, false>, dim3(grid), dim3(256), sm, stream, xp, ldx, dp, ldy, op, lddx, rows, cols, gamma, eps, dgamma, dbeta, rp, ldres);
    }
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}
