// Weight-gradient GEMM ("TN"): C[P, Q] = sum_m A[m, P] * B[m, Q]   (fp16 operands, fp32 result)
// for the trainable set of the CtrLoRA finetune (reference optimizer filter cldm/cldm_ctrlora_finetune.py:88-100):
//   LoRA   dUp   = dY^T (X Down^T),  dDown = (dY Up)^T X      (factored: no dense dW is ever formed)
//   zero-conv dW = dY^T H            (1x1 convs, cldm/cldm.py:281-282)
// Both operands are row-major over the token dimension m, i.e. "MN-major" for the tensor core: TMA boxes of
// [64 tokens][64 features] (128-byte rows, SWIZZLE_128B) are consumed by wgmma with both operands transposed.
// The token dimension is split across CTAs; every CTA parks its fp32 partial tile in a workspace slice and a second
// kernel sums the slices in a fixed order (deterministic; no atomics).
#include "common.cuh"
#include "ctrlora_b200.h"
#include "wgmma.cuh"

namespace ctrl {

int make_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box);

constexpr int WG_BK = 64;          // tokens per pipeline stage
constexpr int WG_STAGES = 8;       // upper bound; the launcher fits as many as 192 KiB allow
constexpr int WG_THREADS = 384;    // warpgroup 0: TMA producer (one thread), warpgroups 1-2: wgmma, 64 rows of P each
constexpr int WG_CONSUMERS = 256;
constexpr int WG_A_BYTES = 2 * WG_BK * 128;  // two 64-feature atoms of the 128-row P tile
constexpr int WG_SMEM_DATA = 192 * 1024;

struct WgradParams {
    int P, Q, M;
    int q_tile;        // 64 or 128 (the wgmma N)
    int q_atoms;       // q_tile / 64
    int p_tiles, q_tiles, splits;
    int kiters_per_split;
    int stage_bytes, stages;
    float* ws;         // [splits][Q_pad / 4][P_pad][4] fp32, P_pad = p_tiles*128, Q_pad = q_tiles*q_tile
    // direct mode (splits == 1: enough output tiles to fill the machine, e.g. the dense conv gradients of pretraining):
    // the epilogue applies alpha / beta itself and writes the result row-major -- no workspace round trip, no reduce kernel
    int direct;
    float* out;
    long long ldo;
    float alpha, beta;
};

template <int QT>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ WgradParams p) {
    pdl_launch_dependents();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.stages * p.stage_bytes);
    uint64_t* full = bars;
    uint64_t* empty = bars + WG_STAGES;
    const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int i = 0; i < p.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], WG_CONSUMERS); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    const int pt = static_cast<int>(blockIdx.x) % p.p_tiles, qt = static_cast<int>(blockIdx.x) / p.p_tiles;
    const int k_total = (p.M + WG_BK - 1) / WG_BK;
    const int it0 = static_cast<int>(blockIdx.y) * p.kiters_per_split, it1 = min(k_total, it0 + p.kiters_per_split);
    const int nit = it1 - it0;
    if (warp < 4) {
        if (warp == 0 && elect_one()) {
            for (int j = 0; j < nit; ++j) {
                const int s = j % p.stages, tok = (it0 + j) * WG_BK;
                mbar_wait_nocall(&empty[s], ((j / p.stages) & 1) ^ 1);
                uint8_t* dst = smem + s * p.stage_bytes;
                mbar_expect_tx(&full[s], WG_A_BYTES + p.q_atoms * WG_BK * 128);
                tma_load_2d(dst, &tmA, &full[s], pt * 128, tok);
                tma_load_2d(dst + WG_BK * 128, &tmA, &full[s], pt * 128 + 64, tok);
                for (int a = 0; a < p.q_atoms; ++a)
                    tma_load_2d(dst + WG_A_BYTES + a * WG_BK * 128, &tmB, &full[s], qt * QT + 64 * a, tok);
            }
        }
        return;
    }
    const int ct = threadIdx.x - 128, wg = ct >> 7;
    float acc[QT / 2];
#pragma unroll
    for (int i = 0; i < QT / 2; ++i) acc[i] = 0.f;
    const uint32_t smem0 = smem_u32(smem);
    for (int j = 0; j < nit; ++j) {
        const int s = j % p.stages;
        mbar_wait_nocall(&full[s], (j / p.stages) & 1);
        const uint32_t a_base = smem0 + s * p.stage_bytes + wg * WG_BK * 128;
        const uint32_t b_base = smem0 + s * p.stage_bytes + WG_A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < WG_BK / 16; ++k)  // both operands MN-major: a k16 step is 16 token rows = 2048 B
            WgmmaSS<QT, 1, 1>::mma(acc, wgmma_desc_mnmajor(a_base + 2048 * k, WG_BK * 128),
                                   wgmma_desc_mnmajor(b_base + 2048 * k, WG_BK * 128), (j | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (j > 0) mbar_arrive(&empty[(j - 1) % p.stages]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs<QT / 2>(acc);
    const int r0 = pt * 128 + wg * 64 + ((ct & 127) >> 5) * 16 + (lane >> 2), cq = qt * QT + 2 * (lane & 3);
    const long long P_pad = static_cast<long long>(p.p_tiles) * 128;
    const long long slice = P_pad * p.q_tiles * p.q_tile;
#pragma unroll
    for (int i = 0; i < QT / 8; ++i) {
        const int q = cq + 8 * i;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            const float x = acc[4 * i + 2 * h], y = acc[4 * i + 2 * h + 1];
            if (p.direct) {
                if (r >= p.P || q >= p.Q) continue;
                float* o = p.out + r * p.ldo + q;
                if (p.beta != 0.f) { o[0] = p.alpha * x + p.beta * o[0]; o[1] = p.alpha * y + p.beta * o[1]; }
                else { o[0] = p.alpha * x; o[1] = p.alpha * y; }
            } else {
                *reinterpret_cast<float2*>(p.ws + blockIdx.y * slice + ((static_cast<long long>(q >> 2)) * P_pad + r) * 4 + (q & 3)) =
                    make_float2(x, y);
            }
        }
    }
}

// out[p, q] = alpha * sum_s ws[s][p][q] + beta * out[p, q]   (fixed summation order)
// block = 32 rows x 32 columns: the slices are read rows-fastest (512 contiguous bytes per warp, the layout the GEMM
// epilogue wrote), transposed through shared memory, and `out` is read/written as 128-byte row segments.
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ out, int P, int Q, int P_pad, int Q_pad,
                    int splits, long long ldo, float alpha, float beta) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float4 tile[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int r0 = blockIdx.x * 32, c4_0 = blockIdx.y * 8;
    const int q4s = Q >> 2;  // Q is a multiple of 8
    {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        const int pr = r0 + tx, q4 = c4_0 + ty;
        if (pr < P && q4 < q4s) {
            const long long slice = static_cast<long long>(P_pad) * Q_pad;
            const float* src = ws + (static_cast<long long>(q4) * P_pad + pr) * 4;
            for (int s = 0; s < splits; ++s) {
                const float4 v = *reinterpret_cast<const float4*>(src + s * slice);
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
        }
        tile[ty][tx] = acc;
    }
    __syncthreads();
    const int row = threadIdx.x >> 3, c4 = threadIdx.x & 7;
    const int pr = r0 + row, q4 = c4_0 + c4;
    if (pr >= P || q4 >= q4s) return;
    float4 acc = tile[c4][row];
    float* o = out + pr * ldo + 4 * q4;
    if (beta != 0.f) { acc.x = alpha * acc.x + beta * o[0]; acc.y = alpha * acc.y + beta * o[1]; acc.z = alpha * acc.z + beta * o[2]; acc.w = alpha * acc.w + beta * o[3]; }
    else { acc.x *= alpha; acc.y *= alpha; acc.z *= alpha; acc.w *= alpha; }
    o[0] = acc.x; o[1] = acc.y; o[2] = acc.z; o[3] = acc.w;
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_wgrad_tn_f16(const void* a, long long lda, const void* b, long long ldb, int m, int p_dim, int q_dim,
                                    float* out, long long ldo, float alpha, float beta, float* ws, long long ws_bytes,
                                    void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || !b || !out || !ws || p_dim % 8 || q_dim % 8 || lda % 8 || ldb % 8 || m <= 0) return CTRLORA_ERR_ARG;
    WgradParams p;
    memset(&p, 0, sizeof(p));
    p.P = p_dim; p.Q = q_dim; p.M = m;
    p.q_tile = q_dim > 64 ? 128 : 64;
    p.q_atoms = p.q_tile / 64;
    p.p_tiles = (p_dim + 127) / 128;
    p.q_tiles = (q_dim + p.q_tile - 1) / p.q_tile;
    const int k_total = (m + WG_BK - 1) / WG_BK;
    int sms = 132;
    {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    // enough token splits to fill the machine once, at least 8 k-iterations each, within the workspace
    int splits = (sms + p.p_tiles * p.q_tiles - 1) / (p.p_tiles * p.q_tiles);  // one wave: half the workspace traffic of two
    if (splits > k_total / 8) splits = k_total / 8;
    if (splits < 1) splits = 1;
    const long long slice = static_cast<long long>(p.p_tiles) * 128 * p.q_tiles * p.q_tile * 4;
    if (splits > 1) {
        if (slice > ws_bytes) splits = 1;  // does not fit the workspace: single split, written directly
        else if (splits * slice > ws_bytes) splits = static_cast<int>(ws_bytes / slice);
    }
    p.kiters_per_split = (k_total + splits - 1) / splits;
    p.splits = (k_total + p.kiters_per_split - 1) / p.kiters_per_split;
    p.direct = (p.splits == 1 && ldo % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) ? 1 : 0;
    p.out = out; p.ldo = ldo; p.alpha = alpha; p.beta = beta;
    if (!p.direct && p.splits * slice > ws_bytes) return CTRLORA_ERR_ARG;
    p.stage_bytes = WG_A_BYTES + p.q_atoms * WG_BK * 128;
    p.ws = ws;
    CUtensorMap tmA, tmB;
    {
        uint64_t dims[2] = {(uint64_t)p_dim, (uint64_t)m};
        uint64_t str[1] = {(uint64_t)lda * 2};
        uint32_t box[2] = {64, WG_BK};
        int rc = make_tmap_f16(&tmA, a, 2, dims, str, box);
        if (rc) return rc;
        uint64_t dimsb[2] = {(uint64_t)q_dim, (uint64_t)m};
        uint64_t strb[1] = {(uint64_t)ldb * 2};
        rc = make_tmap_f16(&tmB, b, 2, dimsb, strb, box);
        if (rc) return rc;
    }
    p.stages = WG_SMEM_DATA / p.stage_bytes;
    if (p.stages > WG_STAGES) p.stages = WG_STAGES;
    const int smem_bytes = p.stages * p.stage_bytes + 1024 + 256;
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(wgrad_tn_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM_DATA + 1280) != cudaSuccess ||
            cudaFuncSetAttribute(wgrad_tn_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM_DATA + 1280) != cudaSuccess)
            return CTRLORA_ERR_CUDA;
        attr = true;
    }
    const dim3 grid(p.p_tiles * p.q_tiles, p.splits);
    const cudaError_t lrc = p.q_tile == 64 ? launch_pdl(wgrad_tn_kernel<64>, grid, dim3(WG_THREADS), (size_t)smem_bytes, stream, tmA, tmB, p)
                                           : launch_pdl(wgrad_tn_kernel<128>, grid, dim3(WG_THREADS), (size_t)smem_bytes, stream, tmA, tmB, p);
    if (lrc != cudaSuccess) return CTRLORA_ERR_CUDA;
    if (p.direct) return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
    if (launch_pdl(wgrad_reduce_kernel, dim3((unsigned)((p_dim + 31) / 32), (unsigned)((q_dim / 4 + 7) / 8)), dim3(256), (size_t)0, stream,
                   (const float*)ws, out, p_dim, q_dim, p.p_tiles * 128, p.q_tiles * p.q_tile, p.splits, ldo, alpha, beta) !=
        cudaSuccess)
        return CTRLORA_ERR_CUDA;
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}
