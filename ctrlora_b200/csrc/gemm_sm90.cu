// wgmma implicit-GEMM for sm_90a: one warp-specialised kernel that serves
//   * every nn.Linear of the hot path            (reference: ldm/modules/attention.py:154-161, cldm/lora.py:285-291)
//   * every 1x1 / 3x3 stride-1 Conv2d in NHWC    (reference: ldm/modules/diffusionmodules/openaimodel.py:162-274)
// D[M, N] = sum_taps A_shifted[M, Cin] * W[N, tap, Cin]^T  (+ optional second 1x1 operand pair: the ResBlock skip conv)
// A tiles are TMA boxes over the (C, W, H, B) activation tensor: a filter tap is a coordinate shift and the conv zero
// padding is the TMA out-of-bounds fill, so no im2col buffer exists in HBM.  The grid is persistent: each CTA walks a
// static list of 128 x BN output tiles (BN up to 320), a producer thread fills a ring of TMA stages, and two consumer
// warpgroups (64 rows each) run wgmma with accumulators in registers, then run the epilogue while the producer already
// loads the next tile.  fp16 row-major outputs leave through shared-memory slots that a second thread of the producer
// warpgroup stores by TMA and into which it has loaded the tile's residual ahead of time, so that epilogue never waits
// on global memory; everything else (fp32, transposed or unaligned outputs, split tiles) takes a row-per-thread
// epilogue through a staging buffer.  Tiles of a last, partial wave may be split along K.
// Launches of whole tiles that all take the TMA epilogue and have a short K loop may run ping-pong instead: each
// consumer warpgroup owns whole 128-row tiles and runs its epilogue while the other's MMAs run.
#include "gemm_sm90.cuh"
#include "wgmma.cuh"
#include "ctrlora_b200.h"
#include <stdio.h>
#include <string.h>

namespace ctrl {

__device__ __forceinline__ bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }
// The last step of the epilogue for relu = 1 (ReLU) and 2 (ReLU6); relu = 3 (ReLU before the residual) is applied
// before the residual add instead.
__device__ __forceinline__ float act_last(int relu, float v) {
    return relu == 2 ? fminf(fmaxf(v, 0.f), 6.f) : fmaxf(v, 0.f);
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// One CW-column chunk (CW = 16 or 32) of the epilogue for one output row, after bias (and GEGLU): time-embedding row
// term (of the tile's group: `hi`), scale, residual, then the store (row-major fp16 / fp32, or the transposed V^T
// layout).
template <int CW>
__device__ __forceinline__ void epilogue_chunk(const GemmKParams& p, float* v, int c, int bn_out, int n0, bool row_ok,
                                               long long m, int img, int tok, bool hi) {
    const int nbase = n0 + c;
    const bool full_chunk = (c + CW <= bn_out) && (nbase + CW <= p.N);
    if (!row_ok) return;
    if (p.rowbias) {
        const float* rb = p.rowbias_g[hi] + static_cast<long long>(img - hi * p.rb_img_off) * p.rowbias_ld + nbase;
        if (full_chunk && aligned16(rb)) {
#pragma unroll
            for (int q = 0; q < CW / 4; ++q) {
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(rb) + q);
                v[4 * q] += b4.x; v[4 * q + 1] += b4.y; v[4 * q + 2] += b4.z; v[4 * q + 3] += b4.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < CW; ++j)
                if (nbase + j < p.N) v[j] += __ldg(rb + j);
        }
    }
    if (p.out_scale != 1.0f) {
#pragma unroll
        for (int j = 0; j < CW; ++j) v[j] *= p.out_scale;
    }
    if (p.relu == 3) {
#pragma unroll
        for (int j = 0; j < CW; ++j) v[j] = fmaxf(v[j], 0.f);
    }
    if (p.residual && p.residual_f32) {
        const float* rp = reinterpret_cast<const float*>(p.residual) + m * p.ldr + nbase;
        if (full_chunk && aligned16(rp)) {  // LoRA folds: W (fp32 master) + s * up . down
#pragma unroll
            for (int q = 0; q < CW / 4; ++q) {
                const float4 r4 = __ldg(reinterpret_cast<const float4*>(rp) + q);
                v[4 * q] += r4.x; v[4 * q + 1] += r4.y; v[4 * q + 2] += r4.z; v[4 * q + 3] += r4.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < CW; ++j)
                if (c + j < bn_out && nbase + j < p.N) v[j] += rp[j];
        }
    } else if (p.residual) {
        const __half* rp = p.residual + m * p.ldr + nbase;
        if (full_chunk && aligned16(rp)) {
            uint4 u[CW / 8];
#pragma unroll
            for (int q = 0; q < CW / 8; ++q) u[q] = __ldg(reinterpret_cast<const uint4*>(rp) + q);
#pragma unroll
            for (int q = 0; q < CW / 8; ++q) {
                const __half2* h = reinterpret_cast<const __half2*>(&u[q]);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(h[e]);
                    v[q * 8 + e * 2] += f.x;
                    v[q * 8 + e * 2 + 1] += f.y;
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < CW; ++j)
                if (c + j < bn_out && nbase + j < p.N) v[j] += __half2float(rp[j]);
        }
    }
    if (p.relu == 1 || p.relu == 2) {
#pragma unroll
        for (int j = 0; j < CW; ++j) v[j] = act_last(p.relu, v[j]);
    }
    int seg = 0, nloc = nbase;
    if (p.seg_width > 0) { seg = nbase / p.seg_width; nloc = nbase - seg * p.seg_width; }
    if (p.transposed[seg]) {
        __half* o = reinterpret_cast<__half*>(p.out[seg]) + (static_cast<long long>(img) * p.seg_width + nloc) * p.tok_pad + tok;
#pragma unroll
        for (int j = 0; j < CW; ++j)
            if (c + j < bn_out && nbase + j < p.N) o[static_cast<long long>(j) * p.tok_pad] = __float2half_rn(v[j]);
        if (p.dup_out) {
            __half* o2 = p.dup_out + m * p.dup_ld + nloc;
#pragma unroll
            for (int j = 0; j < CW; ++j)
                if (c + j < bn_out && nbase + j < p.N) o2[j] = __float2half_rn(v[j]);
        }
    } else if (p.out_f32) {
        float* o = reinterpret_cast<float*>(p.out[seg]) + m * p.ldc + nloc;
        if (full_chunk && aligned16(o)) {
#pragma unroll
            for (int q = 0; q < CW / 4; ++q)
                reinterpret_cast<float4*>(o)[q] = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < CW; ++j)
                if (c + j < bn_out && nbase + j < p.N) o[j] = v[j];
        }
    } else {
        __half* o = reinterpret_cast<__half*>(p.out[seg]) + m * p.ldc + nloc;
        if (full_chunk && aligned16(o)) {
#pragma unroll
            for (int q = 0; q < CW / 8; ++q) {
                uint4 u;
                u.x = pack_h2(v[q * 8 + 0], v[q * 8 + 1]);
                u.y = pack_h2(v[q * 8 + 2], v[q * 8 + 3]);
                u.z = pack_h2(v[q * 8 + 4], v[q * 8 + 5]);
                u.w = pack_h2(v[q * 8 + 6], v[q * 8 + 7]);
                reinterpret_cast<uint4*>(o)[q] = u;
            }
        } else {
#pragma unroll
            for (int j = 0; j < CW; ++j)
                if (c + j < bn_out && nbase + j < p.N) o[j] = __float2half_rn(v[j]);
        }
    }
}

// Grouped launch: does m tile mt hold images of the second group (its weights, bias and row term)?
__device__ __forceinline__ bool tile_hi(const GemmKParams& p, int mt) {
    return p.group_b > 0 && (mt / (p.tiles_w * p.tiles_h)) * p.nb >= p.group_b;
}

// One work unit: an output tile (m tile, n tile) and its k-iteration range.  `slot` >= 0 marks a split tile: its
// workspace slices and arrival counter.
struct GemmUnit {
    int mt, nt, it0, it1, ks, slot;
};
__device__ __forceinline__ GemmUnit gemm_unit(const GemmKParams& p, int u, int m_tiles, int k_iters) {
    GemmUnit w;
    int tile;
    if (u < p.tiles_whole) {
        tile = u;
        w.ks = 0; w.slot = -1; w.it0 = 0; w.it1 = k_iters;
    } else {
        const int v = u - p.tiles_whole;
        w.slot = v / p.splits;
        w.ks = v - w.slot * p.splits;
        tile = p.tiles_whole + w.slot;
        w.it0 = w.ks * p.kiters_per_split;
        w.it1 = min(k_iters, w.it0 + p.kiters_per_split);
    }
    w.mt = tile % m_tiles;  // M fastest: CTAs that run at the same time share the B (weight) tile
    w.nt = tile / m_tiles;
    return w;
}

// fp32 epilogue slab of one warpgroup: [64 rows][64 columns], 16-byte chunk j of row r stored at chunk j ^ (r & 7)
__device__ __forceinline__ uint32_t epi_addr(uint32_t base, int r, int col) {
    return base + static_cast<uint32_t>(r * (GEMM_EPI_COLS * 4) + ((((col >> 2) ^ (r & 7)) << 4) | ((col & 3) << 2)));
}

// Persistent: CTA b runs work units b, b + gridDim.x, ...  The producer thread walks the same sequence, so it fills
// the ring for the next unit while the consumers run the epilogue of the current one; the ring position (stage,
// phase) carries across units.  CTAs never wait on each other, so correctness does not depend on co-residency.
//
// TMA epilogue.  A tile's output is cut into slabs of SW = 64 (32 where 64 does not divide the tile) columns; slab j of
// the CTA's q-th such tile is number q * NSLAB + j of one sequence that the consumers and the epilogue thread both walk,
// through p.epi_slots slots.  The epilogue thread opens a slot (loads the residual slab into it, or just marks it free:
// slot_ready), the consumers add it to their fragment, write the fp16 result over it and arrive on slot_done, the
// epilogue thread stores the slot through the output map and opens it for the slab epi_slots further on once the
// store has read it.  A tile reads only its own residual box and stores after that box has arrived, so the output may
// alias the residual.  The tiles that take this epilogue come first in every CTA's list (p.tma_tiles); the
// row-per-thread epilogue of the later units reuses the slots' memory after `drained`.
// In a slot, row r is SW * 2 bytes and its 16-byte chunk c sits at chunk c ^ (r & 7) (SW = 64, SWIZZLE_128B) or
// c ^ ((r >> 1) & 3) (SW = 32, SWIZZLE_64B).
__host__ __device__ constexpr int gemm_slab_cols(int bn_out) { return bn_out % 64 == 0 ? 64 : 32; }
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ float2 h2_to_f2(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); }

// Entry `idx` of a ring of n barriers walked in order from 0: barrier idx % n, in the phase of parity (idx / n) & 1.
// The producer and the epilogue thread step through consecutive entries (slot + 1, wrapping with a phase flip); the
// ping-pong consumers jump to the first entry of each of their tiles.  A tile is k_iters ring entries and NSLAB_TMA
// slot entries, so tile q of a CTA starts at entry q * k_iters (q * NSLAB_TMA).
struct RingPos {
    int slot;
    uint32_t phase;
};
__host__ __device__ __forceinline__ RingPos ring_pos(uint32_t idx, int n) {
    return RingPos{static_cast<int>(idx % static_cast<uint32_t>(n)), (idx / static_cast<uint32_t>(n)) & 1u};
}

// Ping-pong consumers: every unit of the launch is a whole tile with the TMA epilogue.  Warpgroup wg owns the CTA's
// tiles q = wg, wg + 2, ... (unit blockIdx.x + q * gridDim.x) and all 128 rows of each: two m64nBNk16 per k16, BN
// accumulators per thread.  The K loops take turns (named barrier 4 + wg: the other warpgroup has issued the MMAs of
// tile q - 1), so one warpgroup's epilogue runs while the other's MMAs occupy the tensor cores.  Each element of the
// epilogue is computed as in the cooperative schedule, so the two give the same bits.
template <bool GEGLU, int BN>
__device__ __forceinline__ void gemm_pingpong_consumers(const GemmKParams& p, uint8_t* ring, uint64_t* full,
                                                        uint64_t* empty, uint64_t* slot_ready, uint64_t* slot_done,
                                                        int m_tiles, int k_iters) {
    constexpr int BN_OUT = GEGLU ? BN / 2 : BN;
    constexpr int HALF = BN / 2;  // accumulators of one 64-row half of the tile
    constexpr int SW = gemm_slab_cols(BN_OUT);
    constexpr int NSLAB_TMA = BN_OUT / SW;
    constexpr int SLOT = GEMM_BM * SW * 2;
    static_assert(BN <= 160, "ping-pong tiles hold BN accumulators per thread");
    const int ct = threadIdx.x - 128;
    const int wg = ct >> 7, t = ct & 127, lane = threadIdx.x & 31;
    const uint32_t ring0 = smem_u32(ring);
    const int fr = ((t >> 5) << 4) + (lane >> 2), cq = 2 * (lane & 3);
    const int n_local = (p.units - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
    for (int q = wg; q < n_local; q += 2) {
        const int u = blockIdx.x + q * gridDim.x;
        const int mt = u % m_tiles, nt = u / m_tiles;
        float acc[BN];
#pragma unroll
        for (int i = 0; i < BN; ++i) acc[i] = 0.f;
        if (q > 0) named_bar_sync(4 + wg, 256);
        RingPos rp = ring_pos(static_cast<uint32_t>(q) * k_iters, p.stages);
        int s = rp.slot, prev = -1;
        uint32_t phase = rp.phase;
        for (int it = 0; it < k_iters; ++it) {
            mbar_wait_nocall(&full[s], phase);
            const uint32_t a_base = ring0 + s * p.stage_bytes;
            const uint32_t b_base = a_base + GEMM_A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < GEMM_BK / 16; ++k) {
                const uint32_t sc = (it > 0 || k > 0) ? 1u : 0u;
                const uint64_t db = wgmma_desc_kmajor(b_base + 32 * k);
                WgmmaSS<BN, 0, 0>::mma(acc, wgmma_desc_kmajor(a_base + 32 * k), db, sc);
                WgmmaSS<BN, 0, 0>::mma(acc + HALF, wgmma_desc_kmajor(a_base + 64 * 128 + 32 * k), db, sc);
            }
            wgmma_commit();
            wgmma_wait<1>();  // the previous stage's MMAs have finished reading it
            if (prev >= 0) mbar_arrive(&empty[prev]);
            prev = s;
            if (++s == p.stages) { s = 0; phase ^= 1; }
        }
        if (q + 1 < n_local) named_bar_arrive(4 + (wg ^ 1), 256);  // the other warpgroup may issue tile q + 1's MMAs
        wgmma_wait<0>();
        wgmma_fence_regs<BN>(acc);
        mbar_arrive(&empty[prev]);

        // ---- the TMA epilogue of the cooperative schedule, over both row halves: h = 0 holds rows fr, fr + 8 of the
        // tile in acc[0, HALF), h = 1 rows 64 + fr, 72 + fr in acc[HALF, BN)
        const int n0 = nt * BN_OUT;
        const bool hi = tile_hi(p, mt);
        const float* bias = p.bias_g[hi];  // once per tile: a per-chunk lookup slows the short-K epilogues
        auto bias_geglu = [&](float* a, int i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int n = n0 + 8 * i + cq + e;
                float bv = 0.f, bg = 0.f;
                if (bias && n < p.N) {
                    bv = __ldg(bias + n);
                    if (GEGLU) bg = __ldg(bias + p.N + n);
                }
                a[4 * i + e] += bv;
                a[4 * i + 2 + e] += bv;
                if (GEGLU) {
                    a[4 * i + e] *= gelu_erf_f(a[4 * (i + BN_OUT / 8) + e] + bg);
                    a[4 * i + 2 + e] *= gelu_erf_f(a[4 * (i + BN_OUT / 8) + 2 + e] + bg);
                }
            }
        };
        if (GEGLU) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < BN_OUT / 8; ++i) bias_geglu(acc + h * HALF, i);
        }
        const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h, tb = mt / (p.tiles_w * p.tiles_h);
        const uint32_t row_x = SW == 64 ? (fr & 7) : ((fr >> 1) & 3);  // the same for rows fr, 64 + fr
        const float* rb[4] = {nullptr, nullptr, nullptr, nullptr};     // rows fr, fr + 8, 64 + fr, 72 + fr
        if (p.rowbias) {
            const float* rowbias = p.rowbias_g[hi];
            const int img_off = hi * p.rb_img_off;
            auto row_img = [&](int r) {
                const int iw = r % p.bw, ih = (r / p.bw) % p.bh, ib = r / (p.bw * p.bh);
                const int gw = tw * p.bw + iw, gh = th * p.bh + ih, gb = tb * p.nb + ib;
                if (gw >= p.W || gh >= p.H || gb >= p.Bn) return 0LL;
                return ((static_cast<long long>(gb) * p.H + gh) * p.W + gw) / p.rows_per_img - img_off;
            };
#pragma unroll
            for (int r = 0; r < 4; ++r) rb[r] = rowbias + row_img((r >> 1) * 64 + fr + (r & 1) * 8) * p.rowbias_ld;
        }
#pragma unroll
        for (int j = 0; j < NSLAB_TMA; ++j) {
            const uint32_t idx = static_cast<uint32_t>(q) * NSLAB_TMA + j;
            const RingPos sp = ring_pos(idx, p.epi_slots);
            // The slot's previous slab may be the other warpgroup's, still unopened: slot_ready would then be a whole
            // phase behind and its parity would pass.  Wait until that slab is written (slot_done); with epi_slots >=
            // NSLAB_TMA the one before it is a finished tile's, so this parity cannot alias either.
            if (idx >= static_cast<uint32_t>(p.epi_slots)) mbar_wait_nocall(&slot_done[sp.slot], sp.phase ^ 1);
            mbar_wait_nocall(&slot_ready[sp.slot], sp.phase);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float* a = acc + h * HALF;
                const uint32_t sb = ring0 - (p.epi_slots - sp.slot) * SLOT + (h * 64 + fr) * (SW * 2) + cq * 2;
#pragma unroll
                for (int c = 0; c < SW / 8; ++c) {
                    const int i = j * (SW / 8) + c;
                    if (!GEGLU) bias_geglu(a, i);
                    float v00 = a[4 * i], v01 = a[4 * i + 1], v10 = a[4 * i + 2], v11 = a[4 * i + 3];
                    const int n = n0 + 8 * i + cq;
                    if (rb[0]) {
                        const float* r0 = rb[2 * h];
                        const float* r1 = rb[2 * h + 1];
                        if (n < p.N) { v00 = __fadd_rn(v00, __ldg(r0 + n)); v10 = __fadd_rn(v10, __ldg(r1 + n)); }
                        if (n + 1 < p.N) { v01 = __fadd_rn(v01, __ldg(r0 + n + 1)); v11 = __fadd_rn(v11, __ldg(r1 + n + 1)); }
                    }
                    if (p.out_scale != 1.0f) {
                        v00 = __fmul_rn(v00, p.out_scale); v01 = __fmul_rn(v01, p.out_scale);
                        v10 = __fmul_rn(v10, p.out_scale); v11 = __fmul_rn(v11, p.out_scale);
                    }
                    const uint32_t a0 = sb + ((static_cast<uint32_t>(c) ^ row_x) << 4);
                    const uint32_t a1 = a0 + 8 * SW * 2;
                    if (p.relu == 3) {
                        v00 = fmaxf(v00, 0.f); v01 = fmaxf(v01, 0.f);
                        v10 = fmaxf(v10, 0.f); v11 = fmaxf(v11, 0.f);
                    }
                    if (p.residual) {
                        const float2 r0 = h2_to_f2(lds32(a0)), r1 = h2_to_f2(lds32(a1));
                        v00 = __fadd_rn(v00, r0.x); v01 = __fadd_rn(v01, r0.y);
                        v10 = __fadd_rn(v10, r1.x); v11 = __fadd_rn(v11, r1.y);
                    }
                    if (p.relu == 1 || p.relu == 2) {
                        v00 = act_last(p.relu, v00); v01 = act_last(p.relu, v01);
                        v10 = act_last(p.relu, v10); v11 = act_last(p.relu, v11);
                    }
                    sts32(a0, pack_h2(v00, v01));
                    sts32(a1, pack_h2(v10, v11));
                }
            }
            fence_proxy_async_smem();  // the slot is stored by TMA
            mbar_arrive(&slot_done[sp.slot]);
        }
    }
}

// PP: the ping-pong schedule (gemm_pingpong_consumers); the producer and the epilogue thread are the same for both,
// only the arrival counts of `empty` and `slot_done` differ (one warpgroup consumes a stage or fills a slot, not two).
template <bool GEGLU, int BN, bool PP>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                  const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmO0,
                  const __grid_constant__ CUtensorMap tmO1, const __grid_constant__ CUtensorMap tmO2,
                  const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmB2h,
                  const __grid_constant__ GemmKParams p) {
    constexpr int BN_OUT = GEGLU ? BN / 2 : BN;
    constexpr int NACC = BN / 2;  // fp32 accumulators per consumer thread (64 rows x BN per warpgroup)
    constexpr int BOX = GEGLU || BN > 256 ? BN / 2 : BN;  // rows of one B TMA box: a tile is one box or two
    constexpr int SW = gemm_slab_cols(BN_OUT);            // columns of a TMA epilogue slab
    constexpr int NSLAB_TMA = BN_OUT / SW;
    constexpr int SLOT = GEMM_BM * SW * 2;                // bytes of a slot
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* ring = smem + p.epi_slots * SLOT;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + GEMM_SMEM_DATA);
    uint64_t* full = bars;
    uint64_t* empty = bars + GEMM_MAX_STAGES;
    uint64_t* slot_ready = bars + 2 * GEMM_MAX_STAGES;
    uint64_t* slot_done = slot_ready + GEMM_MAX_SLOTS;
    uint64_t* drained = slot_done + GEMM_MAX_SLOTS;
    volatile int* last_flag = reinterpret_cast<volatile int*>(drained + 1);

    pdl_launch_dependents();
    const int warp = uniform_warp_idx();
    const int lane = threadIdx.x & 31;
    const int nstages = p.stages;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (p.kchunks2 > 0) {
            tma_prefetch_desc(&tmA2);
            tma_prefetch_desc(&tmB2);
        }
        if (p.group_b > 0) {
            tma_prefetch_desc(&tmBh);
            if (p.kchunks2 > 0) tma_prefetch_desc(&tmB2h);
        }
        for (int i = 0; i < nstages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], PP ? 128 : GEMM_CONSUMERS);
        }
        for (int i = 0; i < p.epi_slots; ++i) {
            mbar_init(&slot_ready[i], 1);
            mbar_init(&slot_done[i], PP ? 128 : GEMM_CONSUMERS);
        }
        mbar_init(drained, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();  // everything above overlapped the previous kernel's tail; operands are read only from here on

    const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_b;
    const int main_iters = p.taps * p.kchunks;
    const int k_iters = main_iters + p.kchunks2;

    if (warp < 4) {
        // ---------------------------------------------------- TMA producer: one thread of warpgroup 0
        setmaxnreg_dec<GEMM_PRODUCER_REGS>();
        if (warp == 0 && elect_one()) {
            const uint32_t tx_bytes = GEMM_A_BYTES + BN * 128;
            int s = 0;
            uint32_t phase = 0;
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                const GemmUnit w = gemm_unit(p, u, m_tiles, k_iters);
                const int tw = w.mt % p.tiles_w, th = (w.mt / p.tiles_w) % p.tiles_h, tb = w.mt / (p.tiles_w * p.tiles_h);
                const int w0 = tw * p.bw - p.pad, h0 = th * p.bh - p.pad, b0 = tb * p.nb, n0 = w.nt * BN_OUT;
                const bool hi = p.group_b > 0 && b0 >= p.group_b;  // the tile's weights: the second group's maps
                const CUtensorMap* mB = hi ? &tmBh : &tmB;
                const CUtensorMap* mB2 = hi ? &tmB2h : &tmB2;
                for (int it = w.it0; it < w.it1; ++it) {
                    mbar_wait_nocall(&empty[s], phase ^ 1);
                    uint8_t* dst = ring + s * p.stage_bytes;
                    mbar_expect_tx(&full[s], tx_bytes);
                    if (it < main_iters) {
                        const int tap = it / p.kchunks, kc = it - tap * p.kchunks, ky = tap / p.kw, kx = tap - ky * p.kw;
                        tma_load_4d(dst, &tmA, &full[s], kc * GEMM_BK, w0 + kx, h0 + ky, b0);
                        tma_load_3d(dst + GEMM_A_BYTES, mB, &full[s], kc * GEMM_BK, tap, n0);
                        if (BOX < BN)  // GEGLU: the gate rows start at N
                            tma_load_3d(dst + GEMM_A_BYTES + BOX * 128, mB, &full[s], kc * GEMM_BK, tap, GEGLU ? p.N + n0 : n0 + BOX);
                    } else {  // second operand pair (fused 1x1 skip convolution)
                        const int c0 = (it - main_iters) * GEMM_BK;
                        tma_load_4d(dst, &tmA2, &full[s], c0, w0 + p.pad, h0 + p.pad, b0);
                        tma_load_3d(dst + GEMM_A_BYTES, mB2, &full[s], c0, 0, n0);
                        if (BOX < BN) tma_load_3d(dst + GEMM_A_BYTES + BOX * 128, mB2, &full[s], c0, 0, n0 + BOX);
                    }
                    if (++s == nstages) { s = 0; phase ^= 1; }
                }
            }
        } else if (warp == 1 && p.tma_tiles > 0 && elect_one()) {
            // ------------------------------------------------ epilogue thread: residual loads and output stores
            const int nslots = p.epi_slots;
            // slab (u, j): open its slot
            auto open = [&](int u, int j, int slot) {
                if (!p.residual) { mbar_arrive(&slot_ready[slot]); return; }
                const int mt = u % m_tiles, nt = u / m_tiles;
                const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h, tb = mt / (p.tiles_w * p.tiles_h);
                mbar_expect_tx(&slot_ready[slot], GEMM_BM * SW * 2);
                tma_load_4d(smem + slot * SLOT, &tmR, &slot_ready[slot], nt * BN_OUT + j * SW, tw * p.bw, th * p.bh,
                            tb * p.nb);
            };
            int ou = blockIdx.x, oj = 0;  // the next slab to open
            for (int k = 0; k < nslots && ou < p.tma_tiles; ++k) {
                open(ou, oj, k);
                if (++oj == NSLAB_TMA) { oj = 0; ou += gridDim.x; }
            }
            int slot = 0, prev_slot = -1;
            uint32_t phase = 0;
            for (int u = blockIdx.x; u < p.tma_tiles; u += gridDim.x) {
                const int mt = u % m_tiles, nt = u / m_tiles;
                const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h, tb = mt / (p.tiles_w * p.tiles_h);
                for (int j = 0; j < NSLAB_TMA; ++j) {
                    int col = nt * BN_OUT + j * SW, seg = 0;
                    if (p.seg_width > 0) { seg = col / p.seg_width; col -= seg * p.seg_width; }
                    mbar_wait_nocall(&slot_done[slot], phase);
                    tma_store_4d(seg == 0 ? &tmO0 : seg == 1 ? &tmO1 : &tmO2, smem_u32(smem + slot * SLOT), col,
                                 tw * p.bw, th * p.bh, tb * p.nb);
                    bulk_commit_group();
                    if (prev_slot >= 0) {
                        bulk_wait_group_read<1>();  // the store before this one has read its slot
                        if (ou < p.tma_tiles) {
                            open(ou, oj, prev_slot);
                            if (++oj == NSLAB_TMA) { oj = 0; ou += gridDim.x; }
                        }
                    }
                    prev_slot = slot;
                    if (++slot == nslots) { slot = 0; phase ^= 1; }
                }
            }
            bulk_wait_group<0>();
            mbar_arrive(drained);
        }
        return;  // the consumers synchronise among themselves only (named barriers 1-3)
    }

    // -------------------------------------------------------- consumers: rows [64 wg, 64 wg + 64) of every tile
    setmaxnreg_inc<GEMM_CONSUMER_REGS>();
    if constexpr (PP) {
        gemm_pingpong_consumers<GEGLU, BN>(p, ring, full, empty, slot_ready, slot_done, m_tiles, k_iters);
        return;
    }
    const int ct = threadIdx.x - 128;  // 0..255
    const int wg = ct >> 7, t = ct & 127;
    const uint32_t ring0 = smem_u32(ring);
    const int fr = ((t >> 5) << 4) + (lane >> 2), cq = 2 * (lane & 3);  // accumulator fragment: rows fr, fr + 8
    const int er = t & 63, eh = t >> 6;                                  // epilogue: row er, 32-column half eh of a slab
    const long long slice = static_cast<long long>(GEMM_BM) * BN;       // floats of one split-K workspace slice
    int s = 0;
    uint32_t phase = 0, slot_pos = 0;  // slot_pos: the TMA epilogue's slot, its phase in bit 16
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        const GemmUnit w = gemm_unit(p, u, m_tiles, k_iters);
        float acc[NACC];
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int it = w.it0; it < w.it1; ++it) {
            mbar_wait_nocall(&full[s], phase);
            const uint32_t a_base = ring0 + s * p.stage_bytes + wg * 64 * 128;
            const uint32_t b_base = ring0 + s * p.stage_bytes + GEMM_A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < GEMM_BK / 16; ++k) {
                const uint32_t sc = (it > w.it0 || k > 0) ? 1u : 0u;
                if constexpr (BN > 256) {  // columns [0, 160) and [160, 320): the fragment stays in column order
                    WgmmaSS<BN / 2, 0, 0>::mma(acc, wgmma_desc_kmajor(a_base + 32 * k), wgmma_desc_kmajor(b_base + 32 * k), sc);
                    WgmmaSS<BN / 2, 0, 0>::mma(acc + NACC / 2, wgmma_desc_kmajor(a_base + 32 * k),
                                               wgmma_desc_kmajor(b_base + (BN / 2) * 128 + 32 * k), sc);
                } else {
                    WgmmaSS<BN, 0, 0>::mma(acc, wgmma_desc_kmajor(a_base + 32 * k), wgmma_desc_kmajor(b_base + 32 * k), sc);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();  // the previous stage's MMAs have finished reading it
            if (prev >= 0) mbar_arrive(&empty[prev]);
            prev = s;
            if (++s == nstages) { s = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs<NACC>(acc);
        mbar_arrive(&empty[prev]);  // the producer may refill the ring for the next unit during this epilogue

        if (w.slot >= 0) {
            // ---- split-K: park this split's partial tile in its own fp32 workspace slice in fragment order (each
            // warp stores 512 contiguous bytes per instruction); the last CTA to arrive sums the slices in slice order
            float* frag0 = p.ws + static_cast<long long>(w.slot) * p.splits * slice + ct * 4;
#pragma unroll
            for (int i = 0; i < NACC / 4; ++i)
                __stcg(reinterpret_cast<float4*>(frag0 + w.ks * slice + i * (GEMM_CONSUMERS * 4)),
                       make_float4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]));
            __threadfence();
            named_bar_sync(1, GEMM_CONSUMERS);
            if (ct == 0) {
                const unsigned int old = atomicAdd(&p.counters[w.slot], 1u);
                const int last = (old == static_cast<unsigned int>(p.splits - 1));
                if (last) p.counters[w.slot] = 0;  // self-cleaning: ready for the next launch
                *last_flag = last;
            }
            named_bar_sync(1, GEMM_CONSUMERS);
            if (!*last_flag) continue;
            __threadfence();
#pragma unroll
            for (int i = 0; i < NACC / 4; ++i) {
                float4 t4 = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int sl = 0; sl < p.splits; ++sl) {  // fixed order: deterministic sums
                    const float4 x4 = __ldcg(reinterpret_cast<const float4*>(frag0 + sl * slice + i * (GEMM_CONSUMERS * 4)));
                    t4.x += x4.x; t4.y += x4.y; t4.z += x4.z; t4.w += x4.w;
                }
                acc[4 * i] = t4.x; acc[4 * i + 1] = t4.y; acc[4 * i + 2] = t4.z; acc[4 * i + 3] = t4.w;
            }
        }

        // ---- bias and GEGLU on the fragment: a thread holds value column c and its gate column c + BN_OUT
        const int n0 = w.nt * BN_OUT;
        const bool hi = tile_hi(p, w.mt);
        // the group's bias: looked up once per tile, except in the 320-column tiles, which have no register to hold it
        const float* bias_tile = BN > 256 ? nullptr : p.bias_g[hi];
        auto bias_geglu = [&](int i) {
            const float* bias = BN > 256 ? p.bias_g[hi] : bias_tile;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int n = n0 + 8 * i + cq + e;
                float bv = 0.f, bg = 0.f;
                if (bias && n < p.N) {
                    bv = __ldg(bias + n);
                    if (GEGLU) bg = __ldg(bias + p.N + n);
                }
                acc[4 * i + e] += bv;
                acc[4 * i + 2 + e] += bv;
                if (GEGLU) {
                    acc[4 * i + e] *= gelu_erf_f(acc[4 * (i + BN_OUT / 8) + e] + bg);
                    acc[4 * i + 2 + e] *= gelu_erf_f(acc[4 * (i + BN_OUT / 8) + 2 + e] + bg);
                }
            }
        };
        // GEGLU: all at once, which frees the gate accumulators.  Otherwise per slab as it is staged, so only one
        // slab's bias loads are in flight next to the accumulators
        if (GEGLU) {
#pragma unroll
            for (int i = 0; i < BN_OUT / 8; ++i) bias_geglu(i);
        }
        const int tw = w.mt % p.tiles_w, th = (w.mt / p.tiles_w) % p.tiles_h, tb = w.mt / (p.tiles_w * p.tiles_h);
        if (u < p.tma_tiles) {
            // ---- TMA epilogue on the fragment: time-embedding row term, scale, residual, one rounding, each in the
            // order of the row-per-thread epilogue.  A thread owns rows fr and fr + 8 of its warpgroup's 64; a warp's
            // 4-byte accesses to one 16-byte chunk of 8 rows fall on 8 different chunk positions: no bank conflicts.
            const uint32_t row_off = (wg * 64 + fr) * (SW * 2) + cq * 2, row_x = SW == 64 ? (fr & 7) : ((fr >> 1) & 3);
            const float* rb0 = nullptr;
            const float* rb1 = nullptr;
            const float* rowbias = p.rowbias_g[hi];
            const int img_off = hi * p.rb_img_off;
            if (rowbias) {
                auto row_img = [&](int r) {  // row term row of tile row r (a tile can span several images); 0 past the end
                    const int iw = r % p.bw, ih = (r / p.bw) % p.bh, ib = r / (p.bw * p.bh);
                    const int gw = tw * p.bw + iw, gh = th * p.bh + ih, gb = tb * p.nb + ib;
                    if (gw >= p.W || gh >= p.H || gb >= p.Bn) return 0LL;
                    return ((static_cast<long long>(gb) * p.H + gh) * p.W + gw) / p.rows_per_img - img_off;
                };
                rb0 = rowbias + row_img(wg * 64 + fr) * p.rowbias_ld;
                rb1 = rowbias + row_img(wg * 64 + fr + 8) * p.rowbias_ld;
            }
#pragma unroll
            for (int j = 0; j < NSLAB_TMA; ++j) {
                const int slot = slot_pos & 0xffff;
                mbar_wait_nocall(&slot_ready[slot], slot_pos >> 16);
                const uint32_t sb = ring0 - (p.epi_slots - slot) * SLOT + row_off;
#pragma unroll
                for (int c = 0; c < SW / 8; ++c) {
                    const int i = j * (SW / 8) + c;
                    if (!GEGLU) bias_geglu(i);
                    float v00 = acc[4 * i], v01 = acc[4 * i + 1], v10 = acc[4 * i + 2], v11 = acc[4 * i + 3];
                    const int n = n0 + 8 * i + cq;
                    if (rb0) {
                        if (n < p.N) { v00 = __fadd_rn(v00, __ldg(rb0 + n)); v10 = __fadd_rn(v10, __ldg(rb1 + n)); }
                        if (n + 1 < p.N) { v01 = __fadd_rn(v01, __ldg(rb0 + n + 1)); v11 = __fadd_rn(v11, __ldg(rb1 + n + 1)); }
                    }
                    if (p.out_scale != 1.0f) {
                        v00 = __fmul_rn(v00, p.out_scale); v01 = __fmul_rn(v01, p.out_scale);
                        v10 = __fmul_rn(v10, p.out_scale); v11 = __fmul_rn(v11, p.out_scale);
                    }
                    const uint32_t a0 = sb + ((static_cast<uint32_t>(c) ^ row_x) << 4);
                    const uint32_t a1 = a0 + 8 * SW * 2;
                    if (p.relu == 3) {
                        v00 = fmaxf(v00, 0.f); v01 = fmaxf(v01, 0.f);
                        v10 = fmaxf(v10, 0.f); v11 = fmaxf(v11, 0.f);
                    }
                    if (p.residual) {
                        const float2 r0 = h2_to_f2(lds32(a0)), r1 = h2_to_f2(lds32(a1));
                        v00 = __fadd_rn(v00, r0.x); v01 = __fadd_rn(v01, r0.y);
                        v10 = __fadd_rn(v10, r1.x); v11 = __fadd_rn(v11, r1.y);
                    }
                    if (p.relu == 1 || p.relu == 2) {
                        v00 = act_last(p.relu, v00); v01 = act_last(p.relu, v01);
                        v10 = act_last(p.relu, v10); v11 = act_last(p.relu, v11);
                    }
                    sts32(a0, pack_h2(v00, v01));
                    sts32(a1, pack_h2(v10, v11));
                }
                fence_proxy_async_smem();  // the slot is stored by TMA
                mbar_arrive(&slot_done[slot]);
                slot_pos = slot + 1 == p.epi_slots ? (slot_pos & 0x10000) ^ 0x10000 : slot_pos + 1;
            }
            continue;
        }
        // ---- the rest of the epilogue, one 64-column slab at a time through this warpgroup's staging buffer
        // the staging buffer is slot memory: the TMA epilogue's last stores have left it (the barrier completes once)
        if (p.tma_tiles > 0) mbar_wait_nocall(drained, 0);
        const uint32_t stg = ring0 - p.epi_slots * SLOT + wg * (64 * GEMM_EPI_COLS * 4);
        const int r = wg * 64 + er;
        const int iw = r % p.bw, ih = (r / p.bw) % p.bh, ib = r / (p.bw * p.bh);
        const int gw = tw * p.bw + iw, gh = th * p.bh + ih, gb = tb * p.nb + ib;
        const bool row_ok = gw < p.W && gh < p.H && gb < p.Bn;
        const long long m = (static_cast<long long>(gb) * p.H + gh) * p.W + gw;
        const int img = row_ok ? static_cast<int>(m / p.rows_per_img) : 0;
        const int tok = row_ok ? static_cast<int>(m % p.rows_per_img) : 0;
        constexpr int NSLAB = (BN_OUT + GEMM_EPI_COLS - 1) / GEMM_EPI_COLS;
#pragma unroll
        for (int sl = 0; sl < NSLAB; ++sl) {
            const int s0 = sl * GEMM_EPI_COLS;
#pragma unroll
            for (int j = 0; j < GEMM_EPI_COLS / 8; ++j) {
                const int i = sl * (GEMM_EPI_COLS / 8) + j;
                if (i >= BN_OUT / 8) break;
                if (!GEGLU) bias_geglu(i);
                const int col = 8 * j + cq;
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(epi_addr(stg, fr, col)), "f"(acc[4 * i]), "f"(acc[4 * i + 1])
                             : "memory");
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(epi_addr(stg, fr + 8, col)), "f"(acc[4 * i + 2]),
                             "f"(acc[4 * i + 3])
                             : "memory");
            }
            named_bar_sync(2 + wg, 128);
            // a thread takes 32 columns of its row, in chunks of CW (16 with wider tiles: the accumulators of the
            // later slabs are still live)
            constexpr int CW = BN_OUT > 128 ? 16 : 32;
#pragma unroll
            for (int c1 = 0; c1 < 32; c1 += CW) {
                const int c = s0 + 32 * eh + c1;
                if (c < BN_OUT) {
                    float v[CW];
#pragma unroll
                    for (int q = 0; q < CW / 4; ++q) {
                        const float4 x = lds128f(epi_addr(stg, er, 32 * eh + c1 + 4 * q));
                        v[4 * q] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
                    }
                    epilogue_chunk<CW>(p, v, c, BN_OUT, n0, row_ok, m, img, tok, hi);
                }
            }
            named_bar_sync(2 + wg, 128);  // the slab is free for the next one
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_tmapEncodeTiled get_tmap_encoder() {
    static PFN_tmapEncodeTiled fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<PFN_tmapEncodeTiled>(ptr);
    }
    return fn;
}

// fp16 tensor map with SWIZZLE_128B, zero OOB fill; dims innermost first; strides (bytes) for dims 1..rank-1.
static int make_tmap_f16_sw(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                            const uint32_t* box, CUtensorMapSwizzle swz);
int make_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box) {
    return make_tmap_f16_sw(map, base, rank, dims, strides_bytes, box, CU_TENSOR_MAP_SWIZZLE_128B);
}
static int make_tmap_f16_sw(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                            const uint32_t* box, CUtensorMapSwizzle swz) {
    PFN_tmapEncodeTiled enc = get_tmap_encoder();
    if (!enc) return CTRLORA_ERR_TMAP;
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bx[5], es[5];
    for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstr, bx, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr, "ctrlora: cuTensorMapEncodeTiled failed (%d) rank %d dims", (int)r, rank);
        for (int i = 0; i < rank; ++i) fprintf(stderr, " %llu", (unsigned long long)dims[i]);
        fprintf(stderr, " box");
        for (int i = 0; i < rank; ++i) fprintf(stderr, " %u", box[i]);
        fprintf(stderr, "\n");
        return CTRLORA_ERR_TMAP;
    }
    return CTRLORA_OK;
}

static int pow2_floor(int x) {
    int p = 1;
    while (p * 2 <= x) p *= 2;
    return p;
}

static int g_num_sms = 0;
static int g_sm_limit = 0;  // > 0: SM budget of the persistent grids and the tile model (ctrlora_set_sm_limit)

// SMs a persistent grid may occupy: the device's count, capped by ctrlora_set_sm_limit; 0 if the count is unavailable
int persistent_sms() {
    if (g_num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_num_sms <= 0) return 0;
    }
    return g_sm_limit > 0 && g_sm_limit < g_num_sms ? g_sm_limit : g_num_sms;
}

// constants of the tile model (cycles of one SM): estimates from the data-sheet rates, not yet fitted to a sweep;
// tools/sweep_gemm.py times every (block_n, split_k) of the step's shapes against the model's choice
constexpr double GEMM_L2_BPC = 40.0;          // operand bytes per cycle an SM streams from L2 with all SMs busy
constexpr double GEMM_EPI_FIXED = 600.0;      // per tile: drain, row setup
constexpr double GEMM_EPI_PER_COL = 12.0;     // per output column of a tile (128 rows: stores, residual reads)
constexpr double GEMM_SPLIT_PER_COL = 12.0;   // per accumulator column and slice moved through the workspace (512 B)
constexpr int GEMM_MAX_AUTO_SPLIT = 8;
// 320-column tiles leave room for only 3 ring stages, and the model does not price what that costs a short K loop: on
// the batch-8 step (H100 80GB HBM3, 400 W, tools/gemm_classes.py) they took 10-45 % longer than the narrower tiles
// the model picks on every 1x1 GEMM with K <= 1280 (5-20 k-steps), and 10-40 % less time on the 3x3 convs (45+)
static constexpr int GEMM_WIDE_MIN_KITERS = 40;
// Ping-pong tiles (gemm_pingpong_consumers) are offered to launches of whole tiles that all take the TMA epilogue and
// whose K loop is shorter than this.  One warpgroup runs a whole tile's epilogue, so its per-column cost is twice the
// cooperative one; a CTA's tiles cost max(K loop, epilogue) each, and the last epilogue is exposed.
static constexpr int GEMM_PP_MAX_KITERS = GEMM_WIDE_MIN_KITERS;
static bool g_attr_set = false;

template <bool GEGLU, int BN, bool PP = false>
static cudaError_t launch_gemm(dim3 grid, cudaStream_t stream, const CUtensorMap* tm, const GemmKParams& p) {
    return launch_pdl(gemm_wgmma_kernel<GEGLU, BN, PP>, grid, dim3(GEMM_THREADS), (size_t)GEMM_SMEM_BYTES, stream, tm[0], tm[1],
                      tm[2], tm[3], tm[4], tm[5], tm[6], tm[7], tm[8], tm[9], p);
}
template <bool GEGLU, int BN, bool PP = false>
static bool set_smem_attr() {
    return cudaFuncSetAttribute(gemm_wgmma_kernel<GEGLU, BN, PP>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_BYTES) ==
           cudaSuccess;
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_gemm_f16(const ctrlora_gemm_args* a, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || !a->a || !a->w || !a->out[0]) return CTRLORA_ERR_ARG;
    if (a->a_c % 8 != 0 || a->a_ld % 8 != 0) return CTRLORA_ERR_ARG;
    if (a->relu < 0 || a->relu > 3) return CTRLORA_ERR_ARG;
    // square 1x1, 3x3 and 7x7 taps (7x7: OpenPose's CPM stages); the box origin goes down to -pad, which the tensor
    // map's out-of-bounds fill reads as zero padding
    if (a->kh != a->kw || (a->kh != 1 && a->kh != 3 && a->kh != 7)) return CTRLORA_ERR_UNSUPPORTED;
    if (a->bf16) return CTRLORA_ERR_UNSUPPORTED;
    GemmKParams p;
    memset(&p, 0, sizeof(p));
    p.W = a->a_w; p.H = a->a_h; p.Bn = a->a_b;
    p.bw = pow2_floor(p.W < 128 ? p.W : 128);
    p.bh = pow2_floor(p.H < 128 / p.bw ? p.H : 128 / p.bw);
    p.nb = 128 / (p.bw * p.bh);
    p.tiles_w = (p.W + p.bw - 1) / p.bw;
    p.tiles_h = (p.H + p.bh - 1) / p.bh;
    p.tiles_b = (p.Bn + p.nb - 1) / p.nb;
    p.N = a->n;
    p.taps = a->kh * a->kw; p.kw = a->kw; p.pad = a->pad;
    p.kchunks = (a->a_c + GEMM_BK - 1) / GEMM_BK;
    p.kchunks2 = a->a2 ? (a->a2_c + GEMM_BK - 1) / GEMM_BK : 0;
    p.geglu = a->geglu;
    if (a->group_b > 0) {
        // a grouped launch: every tile's images lie on one side of group_b (the tile model plans on the whole batch)
        if (!a->w_hi || a->group_b >= p.Bn || (a->a2 && !a->w2_hi) || (a->bias && !a->bias_hi) || (a->rowbias && !a->rowbias_hi))
            return CTRLORA_ERR_ARG;
        if (a->group_b % p.nb != 0) return CTRLORA_ERR_UNSUPPORTED;
        p.group_b = a->group_b;
    }
    const int sms = persistent_sms();
    if (sms <= 0) return CTRLORA_ERR_CUDA;
    const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_b;
    // ---- which tiles take the TMA epilogue: fp16 row-major outputs and an fp16 (or no) residual that tensor maps can
    // address.  The segments it serves must come first (q and k of a q | k | V^T launch), so that every CTA runs its
    // TMA-epilogue tiles before the others; split tiles keep the row-per-thread epilogue (only the CTA that arrives
    // last knows that it needs the residual).
    const int n_segs = a->seg_width > 0 ? (p.N + a->seg_width - 1) / a->seg_width : 1;
    if (n_segs > 3) return CTRLORA_ERR_ARG;
    auto tma_ok = [](const void* ptr, long long ld) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && ld % 8 == 0; };
    int tma_segs = 0;
    while (tma_segs < n_segs && !a->transposed[tma_segs]) ++tma_segs;
    bool tma_epi = !a->out_f32 && tma_segs > 0 && (!a->residual || (!a->residual_f32 && tma_ok(a->residual, a->ldr)));
    for (int i = 0; i < n_segs; ++i) {
        if (i < tma_segs ? !a->out[i] || !tma_ok(a->out[i], a->ldc) : !a->transposed[i]) tma_epi = false;
    }
    const int k_iters = p.taps * p.kchunks + p.kchunks2;
    // ---- pick the N tile (wgmma N = 32 ... 256 columns; GEGLU tiles carry value + gate) and the split of the tail with
    // a cycle model of the persistent schedule over `sms` CTAs.  A k-step of a 128 x BN tile costs max(MMA: 4 BN cycles
    // at the dense fp16 rate of one SM, operand bytes / GEMM_L2_BPC from L2); a tile adds its epilogue.  Full waves of
    // tiles run whole; the tiles of the last, partial wave may be split along K so that their work units fill it.
    // A plan that does not fit the split-K workspace or counters is not considered.  An explicit block_n / split_k
    // overrides the model (split_k then splits every tile).  Ping-pong plans (GEMM_PP_MAX_KITERS) are priced next to
    // the cooperative ones; with an explicit block_n a qualifying width runs its whole tiles ping-pong.
    const bool explicit_split = a->split_k > 0;
    const bool pp_launch = tma_epi && tma_segs == n_segs && k_iters < GEMM_PP_MAX_KITERS && a->split_k <= 1;
    auto plan = [&](int cand, int S, int* s_eff, int* whole) -> double {
        const int bnt = p.geglu ? 2 * cand : cand;
        const long long tiles = (long long)m_tiles * ((p.N + cand - 1) / cand);
        const int kps = (k_iters + S - 1) / S;
        *s_eff = (k_iters + kps - 1) / kps;
        long long w = *s_eff == 1 ? tiles : explicit_split ? 0 : (tiles / sms) * sms;
        const long long tail = tiles - w;
        if (*s_eff > 1 && (!a->splitk_ws || !a->splitk_counters || tail == 0 ||
                           tail * *s_eff * GEMM_BM * bnt * 4 > a->splitk_ws_bytes || tail > a->splitk_counters_len))
            return -1.0;
        *whole = (int)w;
        const double step = fmax(4.0 * bnt, (double)(GEMM_A_BYTES + bnt * 128) / GEMM_L2_BPC);
        const double epi = GEMM_EPI_FIXED + GEMM_EPI_PER_COL * cand;
        const double t_whole = k_iters * step + epi;
        const double t_split = kps * step + epi + GEMM_SPLIT_PER_COL * bnt * (1 + *s_eff);
        return (double)((w + sms - 1) / sms) * t_whole + (double)((tail * *s_eff + sms - 1) / sms) * t_split;
    };
    auto plan_pp = [&](int cand) -> double {
        const int bnt = p.geglu ? 2 * cand : cand;
        const long long per_cta = ((long long)m_tiles * ((p.N + cand - 1) / cand) + sms - 1) / sms;
        const double step = fmax(4.0 * bnt, (double)(GEMM_A_BYTES + bnt * 128) / GEMM_L2_BPC);
        const double epi = GEMM_EPI_FIXED + 2.0 * GEMM_EPI_PER_COL * cand;
        return (double)per_cta * fmax(k_iters * step, epi) + epi;
    };
    int bn_out = 0, splits = 1, tiles_whole = 0;
    bool pingpong = false;
    double best_cost = -1;
    // tile widths; GEGLU tiles carry half as many outputs (and have no 80 + 80 tile)
    static const int kWidths[] = {GEMM_MAX_BN, 256, 160, 128, 64, 32};
    for (int wi = 0; wi < 6; ++wi) {
        const int cand = p.geglu ? kWidths[wi] / 2 : kWidths[wi];
        if (cand < 32 || (p.geglu && kWidths[wi] == 160)) continue;
        if (a->block_n > 0 && cand != a->block_n) continue;
        if (a->block_n <= 0 && kWidths[wi] > 256 && k_iters < GEMM_WIDE_MIN_KITERS) continue;
        // 160 columns are the exact tile of N = 320 on the short loops that exclude 320; on long ones the model chose
        // them for split tiles of the 8x8 level, which measured 30-40 % slower than its choice without them
        if (a->block_n <= 0 && kWidths[wi] == 160 && k_iters >= GEMM_WIDE_MIN_KITERS) continue;
        if (a->seg_width > 0 && a->seg_width % cand != 0) continue;
        // ping-pong widths: 64, 128, 160 columns, GEGLU 64 + 64 (BN accumulators per thread)
        const bool pp_width = pp_launch && (p.geglu ? cand == 64 : cand >= 64 && cand <= 160);
        if (pp_width) {
            const double cost = plan_pp(cand);
            if (best_cost < 0 || cost < best_cost || a->block_n > 0) {
                best_cost = cost; bn_out = cand; splits = 1; pingpong = true;
                tiles_whole = m_tiles * ((p.N + cand - 1) / cand);
            }
            if (a->block_n > 0) break;
        }
        for (int S = explicit_split ? a->split_k : 1; S <= (explicit_split ? a->split_k : GEMM_MAX_AUTO_SPLIT); ++S) {
            int s_eff, whole;
            const double cost = plan(cand, S, &s_eff, &whole);
            if (cost < 0) continue;
            if (best_cost < 0 || cost < best_cost) {
                best_cost = cost; bn_out = cand; splits = s_eff; tiles_whole = whole; pingpong = false;
            }
        }
    }
    if (bn_out <= 0) {
        // no tile width divides seg_width, the explicit width is not a wgmma width, or an explicit split does not fit
        // the workspace
        return CTRLORA_ERR_ARG;
    }
    p.BN = p.geglu ? 2 * bn_out : bn_out;
    p.n_tiles = (p.N + bn_out - 1) / bn_out;
    p.kiters_per_split = (k_iters + splits - 1) / splits;
    p.splits = (k_iters + p.kiters_per_split - 1) / p.kiters_per_split;
    p.tiles_whole = tiles_whole;
    p.units = tiles_whole + (m_tiles * p.n_tiles - tiles_whole) * p.splits;
    if (p.splits > 1) {
        p.ws = a->splitk_ws;
        p.counters = a->splitk_counters;
    }
    for (int i = 0; i < 3; ++i) { p.out[i] = a->out[i]; p.transposed[i] = a->transposed[i]; }
    if (tma_epi) {
        const long long t = tma_segs == n_segs ? (long long)m_tiles * p.n_tiles : (long long)m_tiles * tma_segs * (a->seg_width / bn_out);
        p.tma_tiles = (int)(t < tiles_whole ? t : tiles_whole);
    }
    // shared memory: slots for one tile's slabs if the ring keeps 3 stages, and what is left over after whole stages
    const int slab_cols = gemm_slab_cols(bn_out);
    const int slot_bytes = GEMM_BM * slab_cols * 2;
    int epi_want = p.tma_tiles > 0 ? (bn_out / slab_cols) * slot_bytes : GEMM_EPI_BYTES;
    if (epi_want < GEMM_EPI_BYTES) epi_want = GEMM_EPI_BYTES;
    p.stage_bytes = GEMM_A_BYTES + ((p.BN * 128 + 1023) / 1024) * 1024;
    p.stages = (GEMM_SMEM_DATA - epi_want) / p.stage_bytes;
    if (p.stages < 3) p.stages = 3;
    if (p.stages > GEMM_MAX_STAGES) p.stages = GEMM_MAX_STAGES;
    p.epi_slots = (GEMM_SMEM_DATA - p.stages * p.stage_bytes) / slot_bytes;
    if (p.epi_slots > GEMM_MAX_SLOTS) p.epi_slots = GEMM_MAX_SLOTS;
    p.seg_width = a->seg_width;
    p.ldc = a->ldc; p.out_f32 = a->out_f32;
    p.bias = a->bias; p.rowbias = a->rowbias;
    p.bias_g[0] = a->bias;
    p.bias_g[1] = p.group_b > 0 ? a->bias_hi : a->bias;
    p.rowbias_g[0] = a->rowbias;
    p.rowbias_g[1] = p.group_b > 0 ? a->rowbias_hi : a->rowbias;
    p.rows_per_img = a->rows_per_img > 0 ? a->rows_per_img : p.W * p.H;
    if (p.group_b > 0 && p.rowbias) {
        const long long rows_lo = (long long)p.group_b * p.H * p.W;
        if (rows_lo % p.rows_per_img != 0) return CTRLORA_ERR_ARG;
        p.rb_img_off = (int)(rows_lo / p.rows_per_img);
    }
    p.residual = reinterpret_cast<const __half*>(a->residual); p.ldr = a->ldr;
    p.residual_f32 = a->residual_f32;
    p.rowbias_ld = a->rowbias_ld > 0 ? a->rowbias_ld : a->n;
    p.out_scale = a->out_scale;
    p.head_dim = a->head_dim; p.tok_pad = a->tok_pad;
    p.dup_out = reinterpret_cast<__half*>(a->dup_out); p.dup_ld = a->dup_ld;
    p.relu = a->relu;

    const int b_box = p.geglu || p.BN > 256 ? p.BN / 2 : p.BN;  // rows of a B box (the kernel's BOX)
    CUtensorMap tm[10];  // A, B, A2, B2, residual, out[0..2], B and B2 of the second group
    CUtensorMap &tmA = tm[0], &tmB = tm[1], &tmA2 = tm[2], &tmB2 = tm[3];
    {
        uint64_t dims[4] = {(uint64_t)a->a_c, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.Bn};
        uint64_t str[3] = {(uint64_t)a->a_ld * 2, (uint64_t)a->a_ld * 2 * p.W, (uint64_t)a->a_ld * 2 * p.W * p.H};
        uint32_t box[4] = {GEMM_BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.nb};
        int rc = make_tmap_f16(&tmA, a->a, 4, dims, str, box);
        if (rc) return rc;
        const uint64_t rows = p.geglu ? 2ull * p.N : (uint64_t)p.N;
        uint64_t wd[3] = {(uint64_t)a->a_c, (uint64_t)p.taps, rows};
        uint64_t ws[2] = {(uint64_t)a->a_c * 2, (uint64_t)a->a_c * 2 * p.taps};
        uint32_t wb[3] = {GEMM_BK, 1, (uint32_t)b_box};
        rc = make_tmap_f16(&tmB, a->w, 3, wd, ws, wb);
        if (rc) return rc;
        if (p.group_b > 0) {
            rc = make_tmap_f16(&tm[8], a->w_hi, 3, wd, ws, wb);
            if (rc) return rc;
        }
    }
    if (a->a2) {
        if (!a->w2 || a->a2_c % 8 != 0 || a->a2_ld % 8 != 0 || p.geglu) return CTRLORA_ERR_ARG;
        uint64_t dims[4] = {(uint64_t)a->a2_c, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.Bn};
        uint64_t str[3] = {(uint64_t)a->a2_ld * 2, (uint64_t)a->a2_ld * 2 * p.W, (uint64_t)a->a2_ld * 2 * p.W * p.H};
        uint32_t box[4] = {GEMM_BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.nb};
        int rc = make_tmap_f16(&tmA2, a->a2, 4, dims, str, box);
        if (rc) return rc;
        uint64_t wd[3] = {(uint64_t)a->a2_c, 1, (uint64_t)p.N};
        uint64_t ws[2] = {(uint64_t)a->a2_c * 2, (uint64_t)a->a2_c * 2};
        uint32_t wb[3] = {GEMM_BK, 1, (uint32_t)b_box};
        rc = make_tmap_f16(&tmB2, a->w2, 3, wd, ws, wb);
        if (rc) return rc;
        if (p.group_b > 0) {
            rc = make_tmap_f16(&tm[9], a->w2_hi, 3, wd, ws, wb);
            if (rc) return rc;
        }
    } else {
        tmA2 = tmA;
        tmB2 = tmB;
    }
    if (p.group_b == 0) tm[8] = tmB;
    if (p.group_b == 0 || !a->a2) tm[9] = tmB2;
    for (int i = 4; i < 8; ++i) tm[i] = tmA;
    if (p.tma_tiles > 0) {
        // the residual and the outputs have the geometry of A with C = N (a segment: seg_width): the map clips partial
        // tiles, and a column slice of a wider buffer (ld > N) keeps its neighbours
        const CUtensorMapSwizzle swz = slab_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
        const uint32_t box[4] = {(uint32_t)slab_cols, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.nb};
        auto pixel_map = [&](CUtensorMap* m, const void* base, int cols, long long ld) {
            uint64_t dims[4] = {(uint64_t)cols, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.Bn};
            uint64_t str[3] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * p.W, (uint64_t)ld * 2 * p.W * p.H};
            return make_tmap_f16_sw(m, base, 4, dims, str, box, swz);
        };
        if (a->residual) {
            int rc = pixel_map(&tm[4], a->residual, p.N, a->ldr);
            if (rc) return rc;
        }
        for (int i = 0; i < tma_segs; ++i) {
            const int cols = a->seg_width > 0 ? (p.N - i * a->seg_width < a->seg_width ? p.N - i * a->seg_width : a->seg_width) : p.N;
            int rc = pixel_map(&tm[5 + i], a->out[i], cols, a->ldc);
            if (rc) return rc;
        }
    }
    if (!g_attr_set) {
        if (!set_smem_attr<false, 32>() || !set_smem_attr<false, 64>() || !set_smem_attr<false, 128>() ||
            !set_smem_attr<false, 160>() || !set_smem_attr<false, 256>() || !set_smem_attr<false, 320>() || !set_smem_attr<true, 64>() ||
            !set_smem_attr<true, 128>() || !set_smem_attr<true, 256>() || !set_smem_attr<true, 320>() ||
            !set_smem_attr<false, 64, true>() || !set_smem_attr<false, 128, true>() || !set_smem_attr<false, 160, true>() ||
            !set_smem_attr<true, 128, true>())
            return CTRLORA_ERR_CUDA;
        g_attr_set = true;
    }
    const dim3 grid((unsigned)(p.units < sms ? p.units : sms));
    cudaError_t lrc;
    if (pingpong) {
        // unreachable (the plan's conditions and the slot count of every ping-pong width), but the schedule relies on it
        if (p.tma_tiles != p.units || p.splits != 1 || p.epi_slots < 2 || p.epi_slots < bn_out / slab_cols)
            return CTRLORA_ERR_ARG;
        lrc = p.geglu      ? launch_gemm<true, 128, true>(grid, stream, tm, p)
            : p.BN == 64  ? launch_gemm<false, 64, true>(grid, stream, tm, p)
            : p.BN == 128 ? launch_gemm<false, 128, true>(grid, stream, tm, p)
                          : launch_gemm<false, 160, true>(grid, stream, tm, p);
    } else if (p.geglu) lrc = p.BN == 64  ? launch_gemm<true, 64>(grid, stream, tm, p)
                     : p.BN == 128 ? launch_gemm<true, 128>(grid, stream, tm, p)
                     : p.BN == 256 ? launch_gemm<true, 256>(grid, stream, tm, p)
                                   : launch_gemm<true, 320>(grid, stream, tm, p);
    else lrc = p.BN == 32  ? launch_gemm<false, 32>(grid, stream, tm, p)
             : p.BN == 64  ? launch_gemm<false, 64>(grid, stream, tm, p)
             : p.BN == 128 ? launch_gemm<false, 128>(grid, stream, tm, p)
             : p.BN == 160 ? launch_gemm<false, 160>(grid, stream, tm, p)
             : p.BN == 256 ? launch_gemm<false, 256>(grid, stream, tm, p)
                           : launch_gemm<false, 320>(grid, stream, tm, p);
    if (lrc != cudaSuccess) return CTRLORA_ERR_CUDA;
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}

// The persistent grid of ctrlora_gemm_f16 uses at most `limit` CTAs, one per SM, and its tile model plans with that
// many SMs (0 = all).  A communication kernel that runs
// next to the backward (the overlapped gradient all-reduce) owns a few SMs.  The limit is read at launch time, i.e. it
// is baked into a CUDA graph at capture.
extern "C" int ctrlora_set_sm_limit(int limit) {
    if (limit < 0) return CTRLORA_ERR_ARG;
    g_sm_limit = limit;
    return CTRLORA_OK;
}
