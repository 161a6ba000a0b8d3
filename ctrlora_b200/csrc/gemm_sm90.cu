// wgmma implicit-GEMM for sm_90a: one warp-specialised kernel that serves
//   * every nn.Linear of the hot path            (reference: ldm/modules/attention.py:154-161, cldm/lora.py:285-291)
//   * every 1x1 / 3x3 stride-1 Conv2d in NHWC    (reference: ldm/modules/diffusionmodules/openaimodel.py:162-274)
// D[M, N] = sum_taps A_shifted[M, Cin] * W[N, tap, Cin]^T  (+ optional second 1x1 operand pair: the ResBlock skip conv)
// A tiles are TMA boxes over the (C, W, H, B) activation tensor: a filter tap is a coordinate shift and the conv zero
// padding is the TMA out-of-bounds fill, so no im2col buffer exists in HBM.  One CTA owns one 128 x BN output tile: a
// producer thread fills a ring of TMA stages, two consumer warpgroups (64 rows each) run wgmma with accumulators in
// registers, then stage the fp32 tile in shared memory for a row-per-thread epilogue.
#include "gemm_sm90.cuh"
#include "wgmma.cuh"
#include "ctrlora_b200.h"
#include <stdio.h>
#include <string.h>

namespace ctrl {

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// One 32-column chunk of the epilogue for one accumulator row: bias, GEGLU, time-embedding row term, scale, residual,
// then the store (row-major fp16 / fp32, or the transposed V^T layout).  v = value columns, g = gate columns (GEGLU).
template <bool GEGLU>
__device__ __forceinline__ void epilogue_chunk(const GemmKParams& p, float* v, const float* g, int c, int bn_out, int n0,
                                               bool row_ok, long long m, int img, int tok, const float* sb,
                                               const uint4* rpre = nullptr) {
    const int nbase = n0 + c;
    const bool full_chunk = (c + 32 <= bn_out) && (nbase + 32 <= p.N);
    // sb: this tile's bias staged in shared memory (zeros where there is no bias / beyond N): broadcast 16-byte reads
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const float4 b4 = lds128f(smem_u32(sb + c + 4 * q));
        v[4 * q] += b4.x; v[4 * q + 1] += b4.y; v[4 * q + 2] += b4.z; v[4 * q + 3] += b4.w;
    }
    if (GEGLU) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 b4 = lds128f(smem_u32(sb + 256 + c + 4 * q));
            v[4 * q] *= gelu_erf_f(g[4 * q] + b4.x);
            v[4 * q + 1] *= gelu_erf_f(g[4 * q + 1] + b4.y);
            v[4 * q + 2] *= gelu_erf_f(g[4 * q + 2] + b4.z);
            v[4 * q + 3] *= gelu_erf_f(g[4 * q + 3] + b4.w);
        }
    }
    if (!row_ok) return;
    if (p.rowbias) {
        const float* rb = p.rowbias + static_cast<long long>(img) * p.rowbias_ld + nbase;
        if (full_chunk && (p.rowbias_ld & 3) == 0) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(rb) + q);
                v[4 * q] += b4.x; v[4 * q + 1] += b4.y; v[4 * q + 2] += b4.z; v[4 * q + 3] += b4.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
                if (nbase + j < p.N) v[j] += __ldg(rb + j);
        }
    }
    if (p.out_scale != 1.0f) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] *= p.out_scale;
    }
    if (p.residual && p.residual_f32) {
        const float* rp = reinterpret_cast<const float*>(p.residual) + m * p.ldr + nbase;
        if (full_chunk && (p.ldr & 3) == 0) {  // LoRA folds: W (fp32 master) + s * up . down
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 r4 = __ldg(reinterpret_cast<const float4*>(rp) + q);
                v[4 * q] += r4.x; v[4 * q + 1] += r4.y; v[4 * q + 2] += r4.z; v[4 * q + 3] += r4.w;
            }
        } else {
            for (int j = 0; j < 32; ++j)
                if (c + j < bn_out && nbase + j < p.N) v[j] += rp[j];
        }
    } else if (p.residual) {
        const __half* rp = p.residual + m * p.ldr + nbase;
        if (full_chunk && (p.ldr & 7) == 0) {
            uint4 u[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) u[q] = rpre ? rpre[q] : __ldg(reinterpret_cast<const uint4*>(rp) + q);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const __half2* h = reinterpret_cast<const __half2*>(&u[q]);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(h[e]);
                    v[q * 8 + e * 2] += f.x;
                    v[q * 8 + e * 2 + 1] += f.y;
                }
            }
        } else {
            for (int j = 0; j < 32; ++j)
                if (c + j < bn_out && nbase + j < p.N) v[j] += __half2float(rp[j]);
        }
    }
    int seg = 0, nloc = nbase;
    if (p.seg_width > 0) { seg = nbase / p.seg_width; nloc = nbase - seg * p.seg_width; }
    if (p.transposed[seg]) {
        __half* o = reinterpret_cast<__half*>(p.out[seg]) + (static_cast<long long>(img) * p.seg_width + nloc) * p.tok_pad + tok;
        for (int j = 0; j < 32; ++j)
            if (c + j < bn_out && nbase + j < p.N) o[static_cast<long long>(j) * p.tok_pad] = __float2half_rn(v[j]);
        if (p.dup_out) {
            __half* o2 = p.dup_out + m * p.dup_ld + nloc;
            for (int j = 0; j < 32; ++j)
                if (c + j < bn_out && nbase + j < p.N) o2[j] = __float2half_rn(v[j]);
        }
    } else if (p.out_f32) {
        float* o = reinterpret_cast<float*>(p.out[seg]) + m * p.ldc + nloc;
        if (full_chunk && (p.ldc & 3) == 0) {
#pragma unroll
            for (int q = 0; q < 8; ++q)
                reinterpret_cast<float4*>(o)[q] = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
        } else {
            for (int j = 0; j < 32; ++j)
                if (c + j < bn_out && nbase + j < p.N) o[j] = v[j];
        }
    } else {
        __half* o = reinterpret_cast<__half*>(p.out[seg]) + m * p.ldc + nloc;
        if (full_chunk && (p.ldc & 7) == 0) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                uint4 u;
                u.x = pack_h2(v[q * 8 + 0], v[q * 8 + 1]);
                u.y = pack_h2(v[q * 8 + 2], v[q * 8 + 3]);
                u.z = pack_h2(v[q * 8 + 4], v[q * 8 + 5]);
                u.w = pack_h2(v[q * 8 + 6], v[q * 8 + 7]);
                reinterpret_cast<uint4*>(o)[q] = u;
            }
        } else {
            for (int j = 0; j < 32; ++j)
                if (c + j < bn_out && nbase + j < p.N) o[j] = __float2half_rn(v[j]);
        }
    }
}

template <bool GEGLU, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                  const __grid_constant__ GemmKParams p) {
    constexpr int LD = BN + 4;  // fp32 pitch of the staged tile (float4-aligned rows)
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + GEMM_SMEM_DATA);
    uint64_t* full = bars;
    uint64_t* empty = bars + GEMM_MAX_STAGES;
    volatile int* last_flag = reinterpret_cast<volatile int*>(bars + 2 * GEMM_MAX_STAGES);
    float* sb = reinterpret_cast<float*>(smem + GEMM_SMEM_DATA + 256);  // [value 256 | gate 256]

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
        for (int i = 0; i < nstages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], GEMM_CONSUMERS);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();  // everything above overlapped the previous kernel's tail; operands are read only from here on

    const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_b;
    const int main_iters = p.taps * p.kchunks;
    const int k_iters = main_iters + p.kchunks2;
    const int bn_out = GEGLU ? (BN >> 1) : BN;
    // tile -> (m tile, split, n tile); the k range of a split is [ks * kiters_per_split, ...)
    const int mt = static_cast<int>(blockIdx.x) % m_tiles;
    const int rest = static_cast<int>(blockIdx.x) / m_tiles;
    const int ks = rest % p.splits, nt = rest / p.splits;
    const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h, tb = mt / (p.tiles_w * p.tiles_h);
    const int n0 = nt * bn_out;
    const int it0 = ks * p.kiters_per_split, it1 = min(k_iters, it0 + p.kiters_per_split);
    const int nit = it1 - it0;

    if (warp < 4) {
        // ---------------------------------------------------- TMA producer: one thread of warpgroup 0
        if (warp == 0 && elect_one()) {
            const int w0 = tw * p.bw - p.pad, h0 = th * p.bh - p.pad, b0 = tb * p.nb;
            const uint32_t tx_bytes = GEMM_A_BYTES + BN * 128;
            for (int j = 0; j < nit; ++j) {
                const int it = it0 + j, s = j % nstages;
                mbar_wait(&empty[s], ((j / nstages) & 1) ^ 1);
                uint8_t* dst = smem + s * p.stage_bytes;
                mbar_expect_tx(&full[s], tx_bytes);
                if (it < main_iters) {
                    const int tap = it / p.kchunks, kc = it - tap * p.kchunks, ky = tap / p.kw, kx = tap - ky * p.kw;
                    tma_load_4d(dst, &tmA, &full[s], kc * GEMM_BK, w0 + kx, h0 + ky, b0);
                    tma_load_3d(dst + GEMM_A_BYTES, &tmB, &full[s], kc * GEMM_BK, tap, n0);
                    if (GEGLU) tma_load_3d(dst + GEMM_A_BYTES + bn_out * 128, &tmB, &full[s], kc * GEMM_BK, tap, p.N + n0);
                } else {  // second operand pair (fused 1x1 skip convolution)
                    const int c0 = (it - main_iters) * GEMM_BK;
                    tma_load_4d(dst, &tmA2, &full[s], c0, w0 + p.pad, h0 + p.pad, b0);
                    tma_load_3d(dst + GEMM_A_BYTES, &tmB2, &full[s], c0, 0, n0);
                }
            }
        }
        return;  // the consumers synchronise among themselves only (named barrier 1)
    }

    // -------------------------------------------------------- consumers: wgmma main loop, rows [64 wg, 64 wg + 64)
    const int ct = threadIdx.x - 128;  // 0..255
    const int wg = ct >> 7;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    const uint32_t smem0 = smem_u32(smem);
    for (int j = 0; j < nit; ++j) {
        const int s = j % nstages;
        mbar_wait(&full[s], (j / nstages) & 1);
        const uint32_t a_base = smem0 + s * p.stage_bytes + wg * 64 * 128;
        const uint32_t b_base = smem0 + s * p.stage_bytes + GEMM_A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k)
            WgmmaSS<BN, 0, 0>::mma(acc, wgmma_desc_kmajor(a_base + 32 * k), wgmma_desc_kmajor(b_base + 32 * k), (j | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous stage's MMAs have finished reading it
        if (j > 0) mbar_arrive(&empty[(j - 1) % nstages]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs<BN / 2>(acc);

    // ---- stage the fp32 tile over the (now idle) operand ring, and this tile's bias
    named_bar_sync(1, GEMM_CONSUMERS);  // both warpgroups are done reading the ring
    float* stg = reinterpret_cast<float*>(smem);
    {
        const int r0 = wg * 64 + ((ct & 127) >> 5) * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
            *reinterpret_cast<float2*>(stg + r0 * LD + 8 * i + cq) = make_float2(acc[4 * i], acc[4 * i + 1]);
            *reinterpret_cast<float2*>(stg + (r0 + 8) * LD + 8 * i + cq) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
        }
        float bv = 0.f, bg = 0.f;
        if (p.bias && ct < bn_out && n0 + ct < p.N) {
            bv = __ldg(p.bias + n0 + ct);
            if (GEGLU) bg = __ldg(p.bias + p.N + n0 + ct);
        }
        sb[ct] = bv;
        sb[256 + ct] = bg;
    }
    named_bar_sync(1, GEMM_CONSUMERS);

    // ---- epilogue: thread = row, the two threads of a row take alternate 32-column chunks
    const int r = ct & 127, half = ct >> 7;
    const int iw = r % p.bw, ih = (r / p.bw) % p.bh, ib = r / (p.bw * p.bh);
    const int gw = tw * p.bw + iw, gh = th * p.bh + ih, gb = tb * p.nb + ib;
    const bool row_ok = gw < p.W && gh < p.H && gb < p.Bn;
    const long long m = (static_cast<long long>(gb) * p.H + gh) * p.W + gw;
    const int img = row_ok ? static_cast<int>(m / p.rows_per_img) : 0;
    const int tok = row_ok ? static_cast<int>(m % p.rows_per_img) : 0;
    const float* srow = stg + r * LD;
    if (p.splits == 1) {
        for (int c = 32 * half; c < bn_out; c += 64) {
            float v[32], g[GEGLU ? 32 : 1];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 x = *reinterpret_cast<const float4*>(srow + c + 4 * q);
                v[4 * q] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
                if (GEGLU) {
                    const float4 y = *reinterpret_cast<const float4*>(srow + bn_out + c + 4 * q);
                    g[4 * q] = y.x; g[4 * q + 1] = y.y; g[4 * q + 2] = y.z; g[4 * q + 3] = y.w;
                }
            }
            epilogue_chunk<GEGLU>(p, v, g, c, bn_out, n0, row_ok, m, img, tok, sb);
        }
    } else {
        // ---- split-K: park this split's partial tile in its own fp32 workspace slice (plain stores)
        const int tile_mn = nt * m_tiles + mt;
        const long long slice = static_cast<long long>(GEMM_BM) * BN;
        // slice layout [BN / 4][128 rows][4 floats]: thread = row, so the 32 lanes of a warp touch 32 consecutive
        // 16-byte slots (512 contiguous bytes per instruction) both when parking and when reducing
        float* wrow0 = p.ws + static_cast<long long>(tile_mn) * p.splits * slice + static_cast<long long>(r) * 4;
        float* wrow = wrow0 + ks * slice;
        auto wofs = [](int col) { return static_cast<long long>(col >> 2) * (GEMM_BM * 4); };
        for (int c = 32 * half; c < BN; c += 64) {
#pragma unroll
            for (int q = 0; q < 8; ++q)
                __stcg(reinterpret_cast<float4*>(wrow + wofs(c + 4 * q)), *reinterpret_cast<const float4*>(srow + c + 4 * q));
        }
        __threadfence();
        named_bar_sync(1, GEMM_CONSUMERS);
        if (ct == 0) {
            const unsigned int old = atomicAdd(&p.counters[tile_mn], 1u);
            const int last = (old == static_cast<unsigned int>(p.splits - 1));
            if (last) p.counters[tile_mn] = 0;  // self-cleaning: ready for the next launch
            *last_flag = last;
        }
        named_bar_sync(1, GEMM_CONSUMERS);
        if (*last_flag) {
            __threadfence();
            for (int c = 32 * half; c < bn_out; c += 64) {
                float v[32], g[32];
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    float4 t4 = make_float4(0.f, 0.f, 0.f, 0.f), g4 = t4;
                    for (int sl = 0; sl < p.splits; ++sl) {  // fixed order: deterministic sums
                        const float4 x4 = __ldcg(reinterpret_cast<const float4*>(wrow0 + sl * slice + wofs(c + 4 * q)));
                        t4.x += x4.x; t4.y += x4.y; t4.z += x4.z; t4.w += x4.w;
                        if (GEGLU) {
                            const float4 y4 = __ldcg(reinterpret_cast<const float4*>(wrow0 + sl * slice + wofs(bn_out + c + 4 * q)));
                            g4.x += y4.x; g4.y += y4.y; g4.z += y4.z; g4.w += y4.w;
                        }
                    }
                    v[4 * q] = t4.x; v[4 * q + 1] = t4.y; v[4 * q + 2] = t4.z; v[4 * q + 3] = t4.w;
                    g[4 * q] = g4.x; g[4 * q + 1] = g4.y; g[4 * q + 2] = g4.z; g[4 * q + 3] = g4.w;
                }
                epilogue_chunk<GEGLU>(p, v, g, c, bn_out, n0, row_ok, m, img, tok, sb);
            }
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
static int g_sm_limit = 0;  // > 0: SM budget the tile-size model plans with (ctrlora_set_sm_limit)
static bool g_attr_set = false;

template <bool GEGLU, int BN>
static cudaError_t launch_gemm(dim3 grid, cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB,
                               const CUtensorMap& tmA2, const CUtensorMap& tmB2, const GemmKParams& p) {
    return launch_pdl(gemm_wgmma_kernel<GEGLU, BN>, grid, dim3(GEMM_THREADS), (size_t)GEMM_SMEM_BYTES, stream, tmA, tmB, tmA2,
                      tmB2, p);
}
template <bool GEGLU, int BN>
static bool set_smem_attr() {
    return cudaFuncSetAttribute(gemm_wgmma_kernel<GEGLU, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_BYTES) ==
           cudaSuccess;
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_gemm_f16(const ctrlora_gemm_args* a, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || !a->a || !a->w || !a->out[0]) return CTRLORA_ERR_ARG;
    if (a->a_c % 8 != 0 || a->a_ld % 8 != 0) return CTRLORA_ERR_ARG;
    if (a->kh != a->kw || (a->kh != 1 && a->kh != 3)) return CTRLORA_ERR_UNSUPPORTED;
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
    if (g_num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_num_sms <= 0) return CTRLORA_ERR_CUDA;
    }
    const int sms = g_sm_limit > 0 && g_sm_limit < g_num_sms ? g_sm_limit : g_num_sms;
    const int m_tiles = p.tiles_w * p.tiles_h * p.tiles_b;
    const int k_iters = p.taps * p.kchunks + p.kchunks2;
    // ---- pick the N tile (wgmma N = 32, 64 or 128 output columns; GEGLU tiles carry value + gate) and the K split with
    // a per-tile cycle model: a k-step costs max(MMA = BN cycles for 128 x BN x 64 at the dense fp16 rate of one SM,
    // operand bytes / 64 B/clk from L2); a launch costs waves x (k-steps + epilogue).
    int bn_out = a->block_n, splits = a->split_k > 0 ? a->split_k : 1;
    const int max_out = p.geglu ? GEMM_MAX_BN / 2 : GEMM_MAX_BN;
    if (bn_out <= 0) {
        double best_cost = -1;
        for (int cand = max_out; cand >= 32; cand /= 2) {
            if (a->seg_width > 0 && a->seg_width % cand != 0) continue;
            const int bnt = p.geglu ? 2 * cand : cand;
            const int nt = (p.N + cand - 1) / cand;
            const long tiles_mn = (long)m_tiles * nt;
            const double waste = (double)nt * cand / p.N;  // columns computed beyond N
            const int S = a->split_k > 0 ? a->split_k : 1;  // only an explicit request splits K
            const int kps = (k_iters + S - 1) / S;
            const int s_eff = (k_iters + kps - 1) / kps;
            const long tiles = tiles_mn * s_eff;
            const long waves = (tiles + sms - 1) / sms;
            const double t_mma = kps * (double)bnt;
            const double t_load = kps * (double)(GEMM_A_BYTES + bnt * 128) / 64.0;
            double t_tile = (t_mma > t_load ? t_mma : t_load) + 600.0 + cand * 8.0;
            if (s_eff > 1) t_tile += bnt * 12.0;
            const double cost = waves * t_tile * (0.5 + 0.5 * waste);
            if (best_cost < 0 || cost < best_cost) { best_cost = cost; bn_out = cand; splits = s_eff; }
        }
        if (bn_out <= 0) return CTRLORA_ERR_ARG;  // no tile width divides seg_width
    }
    if (bn_out != 32 && bn_out != 64 && bn_out != 128) return CTRLORA_ERR_ARG;
    if (bn_out > max_out) return CTRLORA_ERR_ARG;
    if (a->seg_width > 0 && a->seg_width % bn_out != 0) return CTRLORA_ERR_ARG;
    p.BN = p.geglu ? 2 * bn_out : bn_out;
    p.n_tiles = (p.N + bn_out - 1) / bn_out;
    p.kiters_per_split = (k_iters + splits - 1) / splits;
    p.splits = (k_iters + p.kiters_per_split - 1) / p.kiters_per_split;
    if (p.splits > 1) {
        const long long tiles_mn = (long long)m_tiles * p.n_tiles;
        if (!a->splitk_ws || !a->splitk_counters || tiles_mn * p.splits * GEMM_BM * p.BN * 4 > a->splitk_ws_bytes ||
            tiles_mn > a->splitk_counters_len)
            return CTRLORA_ERR_ARG;
        p.ws = a->splitk_ws;
        p.counters = a->splitk_counters;
    }
    p.stage_bytes = GEMM_A_BYTES + ((p.BN * 128 + 1023) / 1024) * 1024;
    p.stages = GEMM_SMEM_DATA / p.stage_bytes;
    if (p.stages > GEMM_MAX_STAGES) p.stages = GEMM_MAX_STAGES;
    for (int i = 0; i < 3; ++i) { p.out[i] = a->out[i]; p.transposed[i] = a->transposed[i]; }
    p.seg_width = a->seg_width;
    p.ldc = a->ldc; p.out_f32 = a->out_f32;
    p.bias = a->bias; p.rowbias = a->rowbias;
    p.rows_per_img = a->rows_per_img > 0 ? a->rows_per_img : p.W * p.H;
    p.residual = reinterpret_cast<const __half*>(a->residual); p.ldr = a->ldr;
    p.residual_f32 = a->residual_f32;
    p.rowbias_ld = a->rowbias_ld > 0 ? a->rowbias_ld : a->n;
    p.out_scale = a->out_scale;
    p.head_dim = a->head_dim; p.tok_pad = a->tok_pad;
    p.dup_out = reinterpret_cast<__half*>(a->dup_out); p.dup_ld = a->dup_ld;

    CUtensorMap tmA, tmB, tmA2, tmB2;
    {
        uint64_t dims[4] = {(uint64_t)a->a_c, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.Bn};
        uint64_t str[3] = {(uint64_t)a->a_ld * 2, (uint64_t)a->a_ld * 2 * p.W, (uint64_t)a->a_ld * 2 * p.W * p.H};
        uint32_t box[4] = {GEMM_BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.nb};
        int rc = make_tmap_f16(&tmA, a->a, 4, dims, str, box);
        if (rc) return rc;
        const uint64_t rows = p.geglu ? 2ull * p.N : (uint64_t)p.N;
        uint64_t wd[3] = {(uint64_t)a->a_c, (uint64_t)p.taps, rows};
        uint64_t ws[2] = {(uint64_t)a->a_c * 2, (uint64_t)a->a_c * 2 * p.taps};
        uint32_t wb[3] = {GEMM_BK, 1, (uint32_t)bn_out};
        rc = make_tmap_f16(&tmB, a->w, 3, wd, ws, wb);
        if (rc) return rc;
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
        uint32_t wb[3] = {GEMM_BK, 1, (uint32_t)bn_out};
        rc = make_tmap_f16(&tmB2, a->w2, 3, wd, ws, wb);
        if (rc) return rc;
    } else {
        tmA2 = tmA;
        tmB2 = tmB;
    }
    if (!g_attr_set) {
        if (!set_smem_attr<false, 32>() || !set_smem_attr<false, 64>() || !set_smem_attr<false, 128>() ||
            !set_smem_attr<true, 64>() || !set_smem_attr<true, 128>())
            return CTRLORA_ERR_CUDA;
        g_attr_set = true;
    }
    const dim3 grid((unsigned)((long long)m_tiles * p.n_tiles * p.splits));
    cudaError_t lrc;
    if (p.geglu) lrc = p.BN == 64 ? launch_gemm<true, 64>(grid, stream, tmA, tmB, tmA2, tmB2, p)
                                  : launch_gemm<true, 128>(grid, stream, tmA, tmB, tmA2, tmB2, p);
    else lrc = p.BN == 32 ? launch_gemm<false, 32>(grid, stream, tmA, tmB, tmA2, tmB2, p)
             : p.BN == 64 ? launch_gemm<false, 64>(grid, stream, tmA, tmB, tmA2, tmB2, p)
                          : launch_gemm<false, 128>(grid, stream, tmA, tmB, tmA2, tmB2, p);
    if (lrc != cudaSuccess) return CTRLORA_ERR_CUDA;
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}

// The tile-size model of ctrlora_gemm_f16 plans with at most `limit` SMs (0 = all).  A communication kernel that runs
// next to the backward (the overlapped gradient all-reduce) owns a few SMs.  The limit is read at launch time, i.e. it
// is baked into a CUDA graph at capture.
extern "C" int ctrlora_set_sm_limit(int limit) {
    if (limit < 0) return CTRLORA_ERR_ARG;
    g_sm_limit = limit;
    return CTRLORA_OK;
}
