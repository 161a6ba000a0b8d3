// The MiDaS DPT-Large annotator's own kernels (reference: annotator/midas/__init__.py MidasDetector, midas/vit.py and
// midas/blocks.py).  The ViT, the readout projections, the 1x1 / 3x3 / stride-2 convs and every RCU conv run on the
// existing GEMM, patch-gather, embedding, LayerNorm, attention and GELU entry points; what is left is here:
// - the depth-to-space + bias step that follows a kernel = stride ConvTranspose2d computed as one GEMM;
// - s = a (+ b), relu(s) in one pass: the RCU's input ReLU and the fusion block's skip sum, which the implicit GEMM
//   cannot apply on load (it reads A by TMA);
// - the bilinear x2 upsample with align_corners = True of FeatureFusionBlock_custom and the head's Interpolate (also
//   M-LSD's BlockTypeA, which writes it into a channel slice);
// - the head's last Conv2d(32 -> 1, 1) + bias + ReLU, writing the fp32 depth;
// - MidasDetector's post-process: the min / max normalisation and uint8 depth map, and cv2.Sobel's normal map.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

static bool misaligned(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }

// ------------------------------------------------------------------------------------------ depth to space + bias
// dst[b, y * s + ky, x * s + kx, c] = fp16(src[b, y, x, (ky * s + kx) * C + c] + bias[c]).  One thread per 4 channels.
__global__ void __launch_bounds__(256)
depth_to_space_kernel(const float* __restrict__ src, const float* __restrict__ bias, __half* __restrict__ dst,
                      long long items, int h, int w, int channels, int s) {
    pdl_launch_dependents();
    pdl_wait();
    const int c4 = channels >> 2;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int c = static_cast<int>(i % c4) * 4;
        long long r = i / c4;
        const int ox = static_cast<int>(r % (w * s));
        r /= (w * s);
        const int oy = static_cast<int>(r % (h * s));
        const long long b = r / (h * s);
        const int y = oy / s, ky = oy % s, x = ox / s, kx = ox % s;
        const float4 v = *reinterpret_cast<const float4*>(
            src + ((b * h + y) * w + x) * (long long)(s * s * channels) + (ky * s + kx) * channels + c);
        const float4 bb = *reinterpret_cast<const float4*>(bias + c);
        uint2 o;
        o.x = pack_half2(v.x + bb.x, v.y + bb.y);
        o.y = pack_half2(v.z + bb.z, v.w + bb.w);
        *reinterpret_cast<uint2*>(dst + i * 4) = o;
    }
}

// ------------------------------------------------------------------------------------------ sum + ReLU
// s = fp16(a + b) (b NULL: s = a), r = max(s, 0); either output may be NULL.  8 halves per thread.
__global__ void __launch_bounds__(256)
add_relu_kernel(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ sum,
                __half* __restrict__ relu, long long vecs) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < vecs; v += (long long)gridDim.x * blockDim.x) {
        uint4 ua = reinterpret_cast<const uint4*>(a)[v];
        __half2* ha = reinterpret_cast<__half2*>(&ua);
        if (b) {
            uint4 ub = reinterpret_cast<const uint4*>(b)[v];
            const __half2* hb = reinterpret_cast<const __half2*>(&ub);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 fa = __half22float2(ha[e]), fb = __half22float2(hb[e]);
                ha[e] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
            }
            if (sum) reinterpret_cast<uint4*>(sum)[v] = ua;
        }
        if (relu) {
            const __half2 zero = __float2half2_rn(0.f);
#pragma unroll
            for (int e = 0; e < 4; ++e) ha[e] = __hmax2(ha[e], zero);
            reinterpret_cast<uint4*>(relu)[v] = ua;
        }
    }
}

// ------------------------------------------------------------------------------------------ bilinear x2
// F.interpolate(scale_factor=2, mode="bilinear", align_corners=True) on fp16 [B, h, w, C], fp32 weights and sums as
// torch's CUDA kernel forms them: source index = ((in - 1) / (out - 1)) * dst, lambda = index - floor.  src and dst
// pixel strides src_ld, dst_ld (halves), so either may be a channel slice of a wider buffer.
__global__ void __launch_bounds__(256)
upsample_bilinear2x_kernel(const __half* __restrict__ src, int src_ld, __half* __restrict__ dst, int dst_ld,
                           long long items, int h, int w, int channels) {
    pdl_launch_dependents();
    pdl_wait();
    const int c8 = channels >> 3, oh = 2 * h, ow = 2 * w;
    const float sh = static_cast<float>(h - 1) / static_cast<float>(oh - 1);
    const float sw = static_cast<float>(w - 1) / static_cast<float>(ow - 1);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int c = static_cast<int>(i % c8) * 8;
        long long r = i / c8;
        const int ox = static_cast<int>(r % ow);
        r /= ow;
        const int oy = static_cast<int>(r % oh);
        const long long b = r / oh;
        const float fy = sh * oy, fx = sw * ox;
        const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
        const int y1 = y0 + (y0 < h - 1), x1 = x0 + (x0 < w - 1);
        const float ly1 = fy - y0, ly0 = 1.f - ly1, lx1 = fx - x0, lx0 = 1.f - lx1;
        const __half* base = src + b * h * (long long)w * src_ld + c;
        uint4 q[4];
        q[0] = *reinterpret_cast<const uint4*>(base + ((long long)y0 * w + x0) * src_ld);
        q[1] = *reinterpret_cast<const uint4*>(base + ((long long)y0 * w + x1) * src_ld);
        q[2] = *reinterpret_cast<const uint4*>(base + ((long long)y1 * w + x0) * src_ld);
        q[3] = *reinterpret_cast<const uint4*>(base + ((long long)y1 * w + x1) * src_ld);
        const __half2* h00 = reinterpret_cast<const __half2*>(&q[0]);
        const __half2* h01 = reinterpret_cast<const __half2*>(&q[1]);
        const __half2* h10 = reinterpret_cast<const __half2*>(&q[2]);
        const __half2* h11 = reinterpret_cast<const __half2*>(&q[3]);
        uint4 o;
        __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 a = __half22float2(h00[e]), bq = __half22float2(h01[e]);
            const float2 cq = __half22float2(h10[e]), d = __half22float2(h11[e]);
            const float vx = ly0 * (lx0 * a.x + lx1 * bq.x) + ly1 * (lx0 * cq.x + lx1 * d.x);
            const float vy = ly0 * (lx0 * a.y + lx1 * bq.y) + ly1 * (lx0 * cq.y + lx1 * d.y);
            ho[e] = __floats2half2_rn(vx, vy);
        }
        *reinterpret_cast<uint4*>(dst + ((b * oh + oy) * (long long)ow + ox) * dst_ld + c) = o;
    }
}

// ------------------------------------------------------------------------------------------ head output
// out[p] = max(bias + sum_c weight[c] * x[p, c], 0): Conv2d(C -> 1, 1) + ReLU, fp32 sums in channel order.
constexpr int kHeadMaxC = 64;

__global__ void __launch_bounds__(256)
midas_head_out_kernel(const __half* __restrict__ x, const float* __restrict__ weight, const float* __restrict__ bias,
                      float* __restrict__ out, long long pixels, int channels) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float ws[kHeadMaxC];
    if (threadIdx.x < channels) ws[threadIdx.x] = weight[threadIdx.x];
    __syncthreads();
    const float b0 = bias[0];
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < pixels; p += (long long)gridDim.x * blockDim.x) {
        const uint4* row = reinterpret_cast<const uint4*>(x + p * channels);
        float acc = 0.f;
        for (int v = 0; v < channels / 8; ++v) {
            const uint4 u = row[v];
            const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(hh[e]);
                acc = fmaf(ws[v * 8 + 2 * e], f.x, acc);
                acc = fmaf(ws[v * 8 + 2 * e + 1], f.y, acc);
            }
        }
        out[p] = fmaxf(acc + b0, 0.f);
    }
}

// ------------------------------------------------------------------------------------------ detector post-process
// Per image: the min and the max of the depth (exact in any order, so the result does not depend on the reduction's
// shape).  One block per image.
__global__ void __launch_bounds__(1024)
midas_minmax_kernel(const float* __restrict__ depth, float* __restrict__ minmax, long long hw) {
    pdl_launch_dependents();
    pdl_wait();
    const float* d = depth + blockIdx.x * hw;
    float mn = INFINITY, mx = -INFINITY;
    for (long long i = threadIdx.x; i < hw; i += blockDim.x) {
        const float v = d[i];
        mn = fminf(mn, v);
        mx = fmaxf(mx, v);
    }
    for (int o = 16; o; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    __shared__ float smn[32], smx[32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { smn[warp] = mn; smx[warp] = mx; }
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
        mn = lane < nw ? smn[lane] : INFINITY;
        mx = lane < nw ? smx[lane] : -INFINITY;
        for (int o = 16; o; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if (lane == 0) { minmax[2 * blockIdx.x] = mn; minmax[2 * blockIdx.x + 1] = mx; }
    }
}

__device__ __forceinline__ unsigned char to_u8(float v) {
    // numpy's .clip(0, 255).astype(np.uint8): clamp, then truncate toward zero
    return static_cast<unsigned char>(static_cast<int>(fminf(fmaxf(v, 0.f), 255.f)));
}

// MidasDetector.__call__ after the network, restated in fp32 with every product and sum rounded on its own (no FMA
// contraction), as numpy and cv2 compute them:
//   depth_pt = (d - min) / (max - min);  depth_u8 = u8(depth_pt * 255)
//   x, y = cv2.Sobel(d, CV_32F, 1, 0 / 0, 1, ksize=3) with BORDER_REFLECT_101: the [-1, 0, 1] difference along the
//          derivative's axis and the [1, 2, 1] smoothing across it, both on the raw depth
//   x = y = 0 where depth_pt < bg_th;  n = sqrt((x^2 + y^2) + a^2);  normal_u8 = u8([x, y, a] / n * 127.5 + 127.5)
__global__ void __launch_bounds__(256)
midas_maps_kernel(const float* __restrict__ depth, const float* __restrict__ minmax, unsigned char* __restrict__ depth_u8,
                  unsigned char* __restrict__ normal_u8, long long items, int h, int w, float a, float bg_th) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int x = static_cast<int>(i % w);
        const int y = static_cast<int>((i / w) % h);
        const long long b = i / ((long long)h * w);
        const float* d = depth + b * h * (long long)w;
        const float mn = minmax[2 * b], range = __fsub_rn(minmax[2 * b + 1], mn);
        const float dn = __fdiv_rn(__fsub_rn(d[(long long)y * w + x], mn), range);
        depth_u8[i] = to_u8(__fmul_rn(dn, 255.f));
        const int xm = reflect101(x - 1, w), xp = reflect101(x + 1, w);
        const int ym = reflect101(y - 1, h), yp = reflect101(y + 1, h);
        const float* r0 = d + (long long)ym * w;
        const float* r1 = d + (long long)y * w;
        const float* r2 = d + (long long)yp * w;
        // x: per row the difference, then (R0 + R2) + 2 R1 down the column
        const float dx0 = __fsub_rn(r0[xp], r0[xm]), dx1 = __fsub_rn(r1[xp], r1[xm]), dx2 = __fsub_rn(r2[xp], r2[xm]);
        float gx = __fadd_rn(__fadd_rn(dx0, dx2), __fmul_rn(dx1, 2.f));
        // y: per row (L + R) + 2 C, then the difference down the column
        const float s0 = __fadd_rn(__fadd_rn(r0[xm], r0[xp]), __fmul_rn(r0[x], 2.f));
        const float s2 = __fadd_rn(__fadd_rn(r2[xm], r2[xp]), __fmul_rn(r2[x], 2.f));
        float gy = __fsub_rn(s2, s0);
        if (dn < bg_th) gx = gy = 0.f;
        const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(a, a));
        const float n = __fsqrt_rn(n2);
        unsigned char* o = normal_u8 + i * 3;
        o[0] = to_u8(__fadd_rn(__fmul_rn(__fdiv_rn(gx, n), 127.5f), 127.5f));
        o[1] = to_u8(__fadd_rn(__fmul_rn(__fdiv_rn(gy, n), 127.5f), 127.5f));
        o[2] = to_u8(__fadd_rn(__fmul_rn(__fdiv_rn(a, n), 127.5f), 127.5f));
    }
}

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_depth_to_space_bias(const float* src, const float* bias, void* dst, int batch, int h, int w,
                                           int channels, int s, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!src || !bias || !dst || batch < 0 || h < 1 || w < 1 || channels < 4 || channels % 4 || s < 1 || s > 8 ||
        misaligned(src, 16) || misaligned(bias, 16) || misaligned(dst, 8))
        return CTRLORA_ERR_ARG;
    const long long items = (long long)batch * h * s * w * s * (channels / 4);
    if (items == 0) return CTRLORA_OK;
    return launched(launch_pdl(depth_to_space_kernel, dim3(grid_blocks(items, 256, 8192)), dim3(256), (size_t)0, stream, src, bias,
                                     static_cast<__half*>(dst), items, h, w, channels, s));
}

extern "C" int ctrlora_add_relu_f16(const void* a, const void* b, void* sum, void* relu, long long n, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || (!sum && !relu) || (sum && !b) || n < 0 || n % 8 || misaligned(a, 16) || misaligned(b, 16) ||
        misaligned(sum, 16) || misaligned(relu, 16))
        return CTRLORA_ERR_ARG;
    const long long vecs = n / 8;
    if (vecs == 0) return CTRLORA_OK;
    return launched(launch_pdl(add_relu_kernel, dim3(grid_blocks(vecs, 256, 8192)), dim3(256), (size_t)0, stream,
                                     static_cast<const __half*>(a), static_cast<const __half*>(b), static_cast<__half*>(sum),
                                     static_cast<__half*>(relu), vecs));
}

extern "C" int ctrlora_upsample_bilinear2x_ld_f16(const void* src, int src_ld, void* dst, int dst_ld, int batch, int h,
                                                  int w, int channels, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!src || !dst || batch < 0 || h < 1 || w < 1 || channels < 8 || channels % 8 || src_ld < channels ||
        dst_ld < channels || src_ld % 8 || dst_ld % 8 || misaligned(src, 16) || misaligned(dst, 16))
        return CTRLORA_ERR_ARG;
    const long long items = (long long)batch * 2 * h * 2 * w * (channels / 8);
    if (items == 0) return CTRLORA_OK;
    return launched(launch_pdl(upsample_bilinear2x_kernel, dim3(grid_blocks(items, 256, 8192)), dim3(256), (size_t)0, stream,
                                     static_cast<const __half*>(src), src_ld, static_cast<__half*>(dst), dst_ld, items, h,
                                     w, channels));
}

extern "C" int ctrlora_upsample_bilinear2x_f16(const void* src, void* dst, int batch, int h, int w, int channels,
                                               void* stream_) {
    return ctrlora_upsample_bilinear2x_ld_f16(src, channels, dst, channels, batch, h, w, channels, stream_);
}

extern "C" int ctrlora_midas_head_out_f16(const void* x, const float* weight, const float* bias, float* out,
                                          long long pixels, int channels, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !weight || !bias || !out || pixels < 0 || channels < 8 || channels % 8 || channels > kHeadMaxC ||
        misaligned(x, 16))
        return CTRLORA_ERR_ARG;
    if (pixels == 0) return CTRLORA_OK;
    return launched(launch_pdl(midas_head_out_kernel, dim3(grid_blocks(pixels, 256, 8192)), dim3(256), (size_t)0, stream,
                                     static_cast<const __half*>(x), weight, bias, out, pixels, channels));
}

extern "C" int ctrlora_midas_maps(const float* depth, float* minmax, unsigned char* depth_u8, unsigned char* normal_u8,
                                  int batch, int h, int w, float a, float bg_th, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!depth || !minmax || !depth_u8 || !normal_u8 || batch < 0 || h < 2 || w < 2 || batch > 65535)
        return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    const long long hw = (long long)h * w;
    const int rc = launched(launch_pdl(midas_minmax_kernel, dim3(batch), dim3(1024), (size_t)0, stream, depth, minmax,
                                             hw));
    if (rc) return rc;
    return launched(launch_pdl(midas_maps_kernel, dim3(grid_blocks(batch * hw, 256, 8192)), dim3(256), (size_t)0, stream, depth,
                                     (const float*)minmax, depth_u8, normal_u8, batch * hw, h, w, a, bg_th));
}
