// The HED annotator's own kernels (reference: annotator/hed/__init__.py, ControlNetHED_Apache2 and HEDdetector): the
// side projection of each block (1x1 conv C -> 1) fused with the 2x2 max-pool that feeds the next block, and the
// detector's host post-process (bilinear resize of the five side maps, mean, sigmoid, safe_step, uint8) for all five
// maps in one pass.  Every 3x3 conv + ReLU of the network is one ctrlora_gemm_f16 launch with relu = 1.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

// ------------------------------------------------------------------------------------------ side projection + pool
// One group of G = min(C / 8, 32) lanes per 2x2 quad of pixels (y = 2 qy + dy, x = 2 qx + dx); lane l of a group owns the
// 8-channel vectors l, l + G, ... (NV of them) of every pixel of its quad and reads each with one 16-byte load.  Side:
// the lane's products summed in channel order, then a fixed xor tree across the group, then the bias.  Pool: the max
// of the quad's four vectors, stored only for the quads that lie wholly inside the image (max_pool2d floors odd sizes).
template <int NV>
__global__ void __launch_bounds__(256)
hed_side_pool_kernel(const __half* __restrict__ x, const float* __restrict__ wt, const float* __restrict__ bias,
                     float* __restrict__ side, __half* __restrict__ pooled, int h, int w, int channels, long long quads,
                     int qh, int qw) {
    pdl_launch_dependents();
    pdl_wait();
    const int G = channels / (8 * NV);  // lanes per quad: 8, 16 or 32
    const int lane = threadIdx.x & 31, gl = lane % G, per_warp = 32 / G;
    float wr[NV][8];
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) wr[k][e] = __ldg(wt + (gl + k * G) * 8 + e);
    const float b0 = __ldg(bias);
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    const int ph = h >> 1, pw = w >> 1;
    for (long long base = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * per_warp; base < quads;
         base += warps * per_warp) {
        const long long q = base + lane / G;  // warp-uniform loop: every lane takes part in the shuffles below
        const bool valid = q < quads;
        const int qx = valid ? static_cast<int>(q % qw) : 0;
        const long long t = valid ? q / qw : 0;
        const int qy = static_cast<int>(t % qh), b = static_cast<int>(t / qh);
        float acc[4];
        __half2 mx[NV][4];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int y = 2 * qy + (p >> 1), xx = 2 * qx + (p & 1);
            const bool in = valid && y < h && xx < w;
            const __half* px = x + (((long long)b * h + y) * w + xx) * channels;
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < NV; ++k) {
                uint4 u = make_uint4(0, 0, 0, 0);
                if (in) u = *reinterpret_cast<const uint4*>(px + (gl + k * G) * 8);
                const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(hh[e]);
                    s = fmaf(wr[k][2 * e], f.x, s);
                    s = fmaf(wr[k][2 * e + 1], f.y, s);
                    mx[k][e] = p == 0 ? hh[e] : __hmax2(mx[k][e], hh[e]);
                }
            }
            acc[p] = s;
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            if (o >= G) break;
#pragma unroll
            for (int p = 0; p < 4; ++p) acc[p] += __shfl_xor_sync(0xffffffffu, acc[p], o);
        }
        if (!valid) continue;
        if (gl == 0) {
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                const int y = 2 * qy + (p >> 1), xx = 2 * qx + (p & 1);
                if (y < h && xx < w) side[((long long)b * h + y) * w + xx] = acc[p] + b0;
            }
        }
        if (pooled && qy < ph && qx < pw) {
            __half* po = pooled + (((long long)b * ph + qy) * pw + qx) * channels;
#pragma unroll
            for (int k = 0; k < NV; ++k)
                *reinterpret_cast<uint4*>(po + (gl + k * G) * 8) = *reinterpret_cast<const uint4*>(mx[k]);
        }
    }
}

// ------------------------------------------------------------------------------------------ detector post-process
struct HedFuseMaps {
    const float* side[5];        // fp32 [batch, h_l, w_l]
    int h[5], w[5];
    const int* idx[5];           // levels 1..4: source row of each output row [H], then source column of each column [W]
    const float* frac[5];        // the matching fractional weights
};

// cv2.resize(INTER_LINEAR) of one level at output (y, x) from its tables: the horizontal pass on the two source rows,
// then the vertical one, as cv2's HResizeLinear / VResizeLinear order them
__device__ __forceinline__ float hed_resize_at(const HedFuseMaps& m, int l, const float* s, int y, int x, int H) {
    const int* ri = m.idx[l];
    const float* rf = m.frac[l];
    const int r0 = __ldg(ri + y), c0 = __ldg(ri + H + x);
    const float fy = __ldg(rf + y), fx = __ldg(rf + H + x);
    const int r1 = min(r0 + 1, m.h[l] - 1), c1 = min(c0 + 1, m.w[l] - 1);
    const float* s0 = s + (long long)r0 * m.w[l];
    const float* s1 = s + (long long)r1 * m.w[l];
    const float ax = 1.f - fx, ay = 1.f - fy;
    const float t0 = __fadd_rn(__fmul_rn(__ldg(s0 + c0), ax), __fmul_rn(__ldg(s0 + c1), fx));
    const float t1 = __fadd_rn(__fmul_rn(__ldg(s1 + c0), ax), __fmul_rn(__ldg(s1 + c1), fx));
    return __fadd_rn(__fmul_rn(t0, ay), __fmul_rn(t1, fy));
}

// One thread per output pixel: mean = ((((e1 + e2) + e3) + e4) + e5) / 5 in fp32 (numpy's float32 mean over 5), then the
// float64 sigmoid, the optional safe_step (fp32 * 3, int32 truncation, / 2) and (uint8)clip(edge * 255, 0, 255).
__global__ void __launch_bounds__(256)
hed_fuse_kernel(const __grid_constant__ HedFuseMaps m, float* __restrict__ mean, unsigned char* __restrict__ u8, int batch,
                int H, int W, int safe) {
    pdl_launch_dependents();
    pdl_wait();
    const long long n = (long long)batch * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int x = static_cast<int>(i % W);
        const long long t = i / W;
        const int y = static_cast<int>(t % H), b = static_cast<int>(t / H);
        float s = __ldg(m.side[0] + i);  // level 0 has the output's size: cv2.resize is a copy
#pragma unroll
        for (int l = 1; l < 5; ++l)
            s = __fadd_rn(s, hed_resize_at(m, l, m.side[l] + (long long)b * m.h[l] * m.w[l], y, x, H));
        const float mu = __fdiv_rn(s, 5.f);
        mean[i] = mu;
        double e = 1.0 / (1.0 + exp(-static_cast<double>(mu)));
        if (safe) e = static_cast<double>(static_cast<float>(static_cast<int>(__fmul_rn(static_cast<float>(e), 3.f)))) / 2.0;
        u8[i] = static_cast<unsigned char>(fmin(fmax(e * 255.0, 0.0), 255.0));
    }
}

static int launched_hed(cudaError_t e) {
    if (e != cudaSuccess) return CTRLORA_ERR_CUDA;
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}

static unsigned grid_hed(long long items, int per_block) {
    const long long blocks = (items + per_block - 1) / per_block;
    return static_cast<unsigned>(blocks > 8192 ? 8192 : (blocks < 1 ? 1 : blocks));
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_hed_side_pool_f16(const void* x, const float* weight, const float* bias, float* side, void* pooled,
                                         int batch, int h, int w, int channels, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !weight || !bias || !side || batch < 0 || h < 1 || w < 1 ||
        (channels != 64 && channels != 128 && channels != 256 && channels != 512) ||
        (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(pooled) & 15))
        return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    const int qh = (h + 1) / 2, qw = (w + 1) / 2;
    const long long quads = (long long)batch * qh * qw;
    const int nv = channels == 512 ? 2 : 1;
    const int per_block = 8 * (32 / (channels / (8 * nv)));  // quads of one 256-thread block
    const __half* xh = static_cast<const __half*>(x);
    __half* ph = static_cast<__half*>(pooled);
    const dim3 grid(grid_hed(quads, per_block));
    if (nv == 2)
        return launched_hed(launch_pdl(hed_side_pool_kernel<2>, grid, dim3(256), (size_t)0, stream, xh, weight, bias, side,
                                       ph, h, w, channels, quads, qh, qw));
    return launched_hed(launch_pdl(hed_side_pool_kernel<1>, grid, dim3(256), (size_t)0, stream, xh, weight, bias, side, ph,
                                   h, w, channels, quads, qh, qw));
}

extern "C" int ctrlora_hed_fuse(const float* const* sides, const int* side_hw, const int* const* idx,
                                const float* const* frac, float* mean, unsigned char* out_u8, int batch, int h, int w,
                                int safe, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!sides || !side_hw || !idx || !frac || !mean || !out_u8 || batch < 0 || h < 1 || w < 1) return CTRLORA_ERR_ARG;
    HedFuseMaps m;
    memset(&m, 0, sizeof(m));
    for (int l = 0; l < 5; ++l) {
        m.side[l] = sides[l];
        m.h[l] = side_hw[2 * l];
        m.w[l] = side_hw[2 * l + 1];
        if (!m.side[l] || m.h[l] < 1 || m.w[l] < 1) return CTRLORA_ERR_ARG;
        if (l == 0) {
            if (m.h[0] != h || m.w[0] != w) return CTRLORA_ERR_ARG;
            continue;
        }
        m.idx[l] = idx[l];
        m.frac[l] = frac[l];
        if (!m.idx[l] || !m.frac[l]) return CTRLORA_ERR_ARG;
    }
    const long long n = (long long)batch * h * w;
    if (n == 0) return CTRLORA_OK;
    return launched_hed(launch_pdl(hed_fuse_kernel, dim3(grid_hed(n, 256)), dim3(256), (size_t)0, stream, m, mean, out_u8,
                                   batch, h, w, safe));
}
