// The M-LSD line detector's own kernel (reference: annotator/mlsd/utils.py deccode_output_score_and_ptss with ksize 3
// and topk_n 200, as pred_lines calls it).  The MobileNetV2 backbone and the decoder run on the existing GEMM, tap
// gather, depthwise conv and upsample entry points; what is left is the line decode: per image the centre map's
// sigmoid, the 3 x 3 peak mask, the 200 largest peaks and, for each of them, its displacements and segment length.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

constexpr int kTopK = CTRLORA_MLSD_TOPK;
constexpr int kSelectThreads = 1024;
constexpr int kSelectWarps = kSelectThreads / 32;

__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

// score[b, y, x] = heat * (heat == max of heat over the 3 x 3 window), heat = sigmoid(centre); the window skips pixels
// outside the map (max_pool2d's -inf padding).  One thread per pixel.
__global__ void __launch_bounds__(256)
mlsd_score_kernel(const float* __restrict__ tp, int ld, int c_center, long long items, int h, int w,
                  float* __restrict__ score) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int x = static_cast<int>(i % w);
        const int y = static_cast<int>((i / w) % h);
        const float* img = tp + (i - (long long)y * w - x) * ld + c_center;
        const float heat = sigmoidf(img[((long long)y * w + x) * ld]);
        float m = heat;
        for (int dy = -1; dy <= 1; ++dy) {
            const int yy = y + dy;
            if (yy < 0 || yy >= h) continue;
            for (int dx = -1; dx <= 1; ++dx) {
                const int xx = x + dx;
                if (xx < 0 || xx >= w) continue;
                m = fmaxf(m, sigmoidf(img[((long long)yy * w + xx) * ld]));
            }
        }
        score[i] = heat == m ? heat : 0.f;
    }
}

// One CTA per image.  The scores are >= 0, so their fp32 bits order as unsigned integers.  A radix select over four
// 8-bit digits (most significant first) finds T, the bits of the kTopK-th largest score, and how many of the scores
// equal to T are taken; each digit's histogram is counted per warp (one lane per distinct digit adds the lanes that
// share it), so no atomics are used.  An ordered compaction then gathers the scores above T and the first scores equal
// to T in index order, and a rank sort orders them by score (descending), then index (ascending).
__global__ void __launch_bounds__(kSelectThreads, 1)
mlsd_select_kernel(const float* __restrict__ tp, int ld, int c_disp, const float* __restrict__ score, int n,
                   int* __restrict__ out_idx, float* __restrict__ out_val) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ int hist[kSelectWarps][256];
    __shared__ int total[256];
    __shared__ int warp_cnt[2][kSelectWarps];
    __shared__ unsigned int s_prefix;
    __shared__ int s_k;
    __shared__ int cand_idx[kTopK];
    __shared__ float cand_val[kTopK];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int* bits = reinterpret_cast<const unsigned int*>(score) + (long long)blockIdx.x * n;
    if (tid == 0) { s_prefix = 0; s_k = kTopK; }
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int j = tid; j < kSelectWarps * 256; j += kSelectThreads) (&hist[0][0])[j] = 0;
        __syncthreads();
        const unsigned int prefix = s_prefix;
        const unsigned int hi_mask = shift == 24 ? 0u : ~0u << (shift + 8);
        for (int base = 0; base < n; base += kSelectThreads) {
            const int i = base + tid;
            int key = -1;
            if (i < n) {
                const unsigned int u = __ldg(bits + i);
                if ((u & hi_mask) == prefix) key = static_cast<int>((u >> shift) & 255u);
            }
            const unsigned int peers = __match_any_sync(0xffffffffu, key);
            if (key >= 0 && lane == __ffs(peers) - 1) hist[warp][key] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();
        if (tid < 256) {
            int s = 0;
            for (int q = 0; q < kSelectWarps; ++q) s += hist[q][tid];
            total[tid] = s;
        }
        __syncthreads();
        if (warp == 0) {
            // lane l holds digits 255 - 8 l .. 248 - 8 l (descending); an inclusive scan from the top finds the digit
            // at which the count of larger-or-equal scores first reaches k
            const int k = s_k;
            int c[8], local = 0;
#pragma unroll
            for (int e = 0; e < 8; ++e) { c[e] = total[255 - 8 * lane - e]; local += c[e]; }
            int incl = local;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            const int excl = incl - local;
            if (excl < k && incl >= k) {
                int above = excl, e = 0;
                while (above + c[e] < k) above += c[e++];
                s_prefix = prefix | (static_cast<unsigned int>(255 - 8 * lane - e) << shift);
                s_k = k - above;
            }
        }
        __syncthreads();
    }
    const unsigned int T = s_prefix;
    const int take_eq = s_k;               // scores equal to T that are taken: the first take_eq of them by index
    const int n_gt = kTopK - take_eq;      // scores above T: all taken
    int gt_base = 0, eq_base = 0;
    const unsigned int lt_mask = (1u << lane) - 1u;
    for (int base = 0; base < n; base += kSelectThreads) {
        const int i = base + tid;
        const unsigned int u = i < n ? __ldg(bits + i) : 0u;
        const bool gt = i < n && u > T, eq = i < n && u == T;
        const unsigned int bg = __ballot_sync(0xffffffffu, gt), be = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) { warp_cnt[0][warp] = __popc(bg); warp_cnt[1][warp] = __popc(be); }
        __syncthreads();
        int pg = 0, pe = 0, tg = 0, te = 0;
        for (int q = 0; q < kSelectWarps; ++q) {
            if (q == warp) { pg = tg; pe = te; }
            tg += warp_cnt[0][q];
            te += warp_cnt[1][q];
        }
        if (gt) {
            const int pos = gt_base + pg + __popc(bg & lt_mask);
            cand_idx[pos] = i;
            cand_val[pos] = __uint_as_float(u);
        }
        if (eq) {
            const int pos = eq_base + pe + __popc(be & lt_mask);
            if (pos < take_eq) {
                cand_idx[n_gt + pos] = i;
                cand_val[n_gt + pos] = __uint_as_float(u);
            }
        }
        gt_base += tg;
        eq_base += te;
        __syncthreads();  // warp_cnt is rewritten by the next chunk
    }
    __syncthreads();
    if (tid < kTopK) {
        const float v = cand_val[tid];
        const int idx = cand_idx[tid];
        int rank = 0;
        for (int j = 0; j < kTopK; ++j) {
            const float vj = cand_val[j];
            rank += vj > v || (vj == v && cand_idx[j] < idx);
        }
        const float* d = tp + ((long long)blockIdx.x * n + idx) * ld + c_disp;
        const float d0 = d[0], d1 = d[1], d2 = d[2], d3 = d[3];
        // numpy: sqrt(sum((start - end) ** 2)) over the two coordinates, each step rounded to fp32
        const float ex = __fsub_rn(d0, d2), ey = __fsub_rn(d1, d3);
        const float dist = __fsqrt_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)));
        const long long o = (long long)blockIdx.x * kTopK + rank;
        out_idx[o] = idx;
        float* ov = out_val + o * 6;
        ov[0] = v; ov[1] = dist; ov[2] = d0; ov[3] = d1; ov[4] = d2; ov[5] = d3;
    }
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_mlsd_decode(const float* tp, int ld, int c_center, int c_disp, int batch, int h, int w,
                                   float* score_ws, int* out_idx, float* out_val, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!tp || !score_ws || !out_idx || !out_val || batch < 0 || h < 1 || w < 1 || (long long)h * w < kTopK ||
        (long long)h * w > 0x7fffffffLL - kSelectThreads || c_center < 0 || c_center >= ld || c_disp < 0 ||
        c_disp + 4 > ld)
        return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    const long long items = (long long)batch * h * w;
    int rc = launched(launch_pdl(mlsd_score_kernel, dim3(grid_blocks(items, 256, 8192)), dim3(256), (size_t)0, stream, tp,
                                 ld, c_center, items, h, w, score_ws));
    if (rc) return rc;
    return launched(launch_pdl(mlsd_select_kernel, dim3(batch), dim3(kSelectThreads), (size_t)0, stream, tp, ld, c_disp,
                               (const float*)score_ws, h * w, out_idx, out_val));
}
