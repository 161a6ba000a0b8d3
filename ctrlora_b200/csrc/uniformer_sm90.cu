// The UniFormer-S + UPerNet segmentation annotator's own kernels (reference: annotator/uniformer, mmseg's
// EncoderDecoder with the UniFormer backbone and UPerHead).  The patch embeds, every 1x1 and 3x3 conv, the linears,
// the attention, LayerNorm and GELU run on the existing entry points; what is left is here:
// - the depthwise k x k conv (k = 3, 5) with bias and an optional residual: CBlock's and SABlock's pos_embed
//   (x + dw3x3(x) in one launch) and CBlock's dw5x5 `attn`; its stride-2 (TFLite padding) and ReLU / ReLU6 variants
//   serve M-LSD's MobileNetV2 (annotator/mlsd/models/mbv2_mlsd_large.py);
// - the bilinear resize with align_corners = False between any two sizes, optionally accumulating into its destination
//   and writing a channel slice of a wider pixel-major buffer: the PPM and FPN resizes and the top-down adds;
// - the adaptive average pool of the PPM, every pool size in one launch;
// - the segmentation output: the two logit resizes, the argmax over the classes and the palette lookup, per pixel.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

static bool misaligned_u(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }

// torch's F.interpolate(size=..., mode="bilinear", align_corners=False) source rule along one axis (upsample_bilinear2d
// with no scale_factor): scale = in / out in fp32, r = max(scale * (dst + 0.5) - 0.5, 0), i0 = floor(r),
// i1 = i0 + (i0 < in - 1), l1 = r - i0, l0 = 1 - l1.
struct Lerp {
    int i0, i1;
    float l0, l1;
};

__device__ __forceinline__ Lerp lerp_src(int dst, float scale, int in) {
    const float r = fmaxf(__fsub_rn(__fmul_rn(scale, static_cast<float>(dst) + 0.5f), 0.5f), 0.f);
    Lerp l;
    l.i0 = min(static_cast<int>(r), in - 1);
    l.i1 = l.i0 + (l.i0 < in - 1);
    l.l1 = fminf(fmaxf(r - static_cast<float>(l.i0), 0.f), 1.f);
    l.l0 = 1.f - l.l1;
    return l;
}

__device__ __forceinline__ void load8(const __half* p, float* v) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        v[2 * e] = f.x;
        v[2 * e + 1] = f.y;
    }
}

__device__ __forceinline__ void store8(__half* p, const float* v) {
    uint4 o;
    o.x = pack_half2(v[0], v[1]);
    o.y = pack_half2(v[2], v[3]);
    o.z = pack_half2(v[4], v[5]);
    o.w = pack_half2(v[6], v[7]);
    *reinterpret_cast<uint4*>(p) = o;
}

// ------------------------------------------------------------------------------------------ depthwise conv
// out[b, y, x, c] = fp16(act((residual[b, y, x, c]) + bias[c] + sum_{ky, kx} weight[ky * K + kx, c] * in[b, S y + ky - P,
// S x + kx - P, c])), zero outside; fp32 sums in tap order.  S = 1: P = K / 2, the output is hi x wi; S = 2: P = 0 (the
// TFLite padding: F.pad(x, (0, 1, 0, 1)) then a padding-0 conv), the output is floor(hi / 2) x floor(wi / 2).  ACT 0
// none, 1 ReLU, 2 ReLU6.  One thread per output pixel and 8 channels.
template <int K, int S, int ACT>
__global__ void __launch_bounds__(256)
dwconv_kernel(const __half* __restrict__ x, const float* __restrict__ weight, const float* __restrict__ bias,
              const __half* __restrict__ residual, __half* __restrict__ out, long long items, int hi, int wi, int h, int w,
              int channels) {
    pdl_launch_dependents();
    pdl_wait();
    const int c8 = channels >> 3;
    constexpr int R = S == 1 ? K / 2 : 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int c = static_cast<int>(i % c8) * 8;
        long long r = i / c8;
        const int px = static_cast<int>(r % w);
        r /= w;
        const int py = static_cast<int>(r % h);
        const long long b = r / h;
        const __half* img = x + b * hi * (long long)wi * channels + c;
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
        for (int ky = 0; ky < K; ++ky) {
            const int iy = S * py + ky - R;
            if (iy < 0 || iy >= hi) continue;
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
                const int ix = S * px + kx - R;
                if (ix < 0 || ix >= wi) continue;
                float v[8];
                load8(img + ((long long)iy * wi + ix) * channels, v);
                const float4 w0 = *reinterpret_cast<const float4*>(weight + (ky * K + kx) * channels + c);
                const float4 w1 = *reinterpret_cast<const float4*>(weight + (ky * K + kx) * channels + c + 4);
                acc[0] = fmaf(w0.x, v[0], acc[0]);
                acc[1] = fmaf(w0.y, v[1], acc[1]);
                acc[2] = fmaf(w0.z, v[2], acc[2]);
                acc[3] = fmaf(w0.w, v[3], acc[3]);
                acc[4] = fmaf(w1.x, v[4], acc[4]);
                acc[5] = fmaf(w1.y, v[5], acc[5]);
                acc[6] = fmaf(w1.z, v[6], acc[6]);
                acc[7] = fmaf(w1.w, v[7], acc[7]);
            }
        }
        const float4 b0 = *reinterpret_cast<const float4*>(bias + c);
        const float4 b1 = *reinterpret_cast<const float4*>(bias + c + 4);
        acc[0] += b0.x; acc[1] += b0.y; acc[2] += b0.z; acc[3] += b0.w;
        acc[4] += b1.x; acc[5] += b1.y; acc[6] += b1.z; acc[7] += b1.w;
        if (residual) {
            float res[8];
            load8(residual + i * 8, res);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] += res[e];
        }
        if (ACT) {
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = ACT == 2 ? fminf(fmaxf(acc[e], 0.f), 6.f) : fmaxf(acc[e], 0.f);
        }
        store8(out + i * 8, acc);
    }
}

// ------------------------------------------------------------------------------------------ bilinear resize
// dst[b, oy, ox, c] (+)= bilinear(src) at torch's align_corners=False source point, fp32 weights and sums:
// l0y * (l0x * s00 + l1x * s01) + l1y * (l0x * s10 + l1x * s11), then + dst (accumulate) and one fp16 rounding.
// src pixel stride src_ld, dst pixel stride dst_ld (halves).  One thread per output pixel and 8 channels.
__global__ void __launch_bounds__(256)
resize_bilinear_kernel(const __half* __restrict__ src, int src_ld, __half* dst, int dst_ld, long long items, int hi,
                       int wi, int ho, int wo, int channels, float sh, float sw, int accumulate) {
    pdl_launch_dependents();
    pdl_wait();
    const int c8 = channels >> 3;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int c = static_cast<int>(i % c8) * 8;
        long long r = i / c8;
        const int ox = static_cast<int>(r % wo);
        r /= wo;
        const int oy = static_cast<int>(r % ho);
        const long long b = r / ho;
        const Lerp ly = lerp_src(oy, sh, hi), lx = lerp_src(ox, sw, wi);
        const __half* base = src + b * hi * (long long)wi * src_ld + c;
        float v00[8], v01[8], v10[8], v11[8], o[8];
        load8(base + ((long long)ly.i0 * wi + lx.i0) * src_ld, v00);
        load8(base + ((long long)ly.i0 * wi + lx.i1) * src_ld, v01);
        load8(base + ((long long)ly.i1 * wi + lx.i0) * src_ld, v10);
        load8(base + ((long long)ly.i1 * wi + lx.i1) * src_ld, v11);
#pragma unroll
        for (int e = 0; e < 8; ++e)
            o[e] = ly.l0 * (lx.l0 * v00[e] + lx.l1 * v01[e]) + ly.l1 * (lx.l0 * v10[e] + lx.l1 * v11[e]);
        __half* d = dst + ((b * ho + oy) * (long long)wo + ox) * dst_ld + c;
        if (accumulate) {
            float prev[8];
            load8(d, prev);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] += prev[e];
        }
        store8(d, o);
    }
}

// ------------------------------------------------------------------------------------------ adaptive average pool
// For each pool size s of `sizes`: dst rows [first_s + (b * s + i) * s + j] = fp16(mean of src over rows
// floor(i h / s) .. ceil((i + 1) h / s) - 1 and the same for columns), torch's AdaptiveAvgPool2d bins; fp32 sums in
// row-major order.  first_s = batch * (sum of the squares of the sizes before s).  dst rows are `channels` wide.
constexpr int kMaxPools = 4;

struct PoolSizes {
    int n;
    int s[kMaxPools];
};

__global__ void __launch_bounds__(256)
adaptive_avg_pool_kernel(const __half* __restrict__ src, int src_ld, __half* __restrict__ dst, long long items, int h,
                         int w, int channels, int batch, PoolSizes sizes) {
    pdl_launch_dependents();
    pdl_wait();
    const int c8 = channels >> 3;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int c = static_cast<int>(i % c8) * 8;
        long long row = i / c8;
        // which pool size the row belongs to
        int s = 0;
        long long rel = row;
#pragma unroll
        for (int k = 0; k < kMaxPools; ++k) {
            if (k == sizes.n) break;
            s = sizes.s[k];
            const long long rows_k = (long long)batch * s * s;
            if (rel < rows_k) break;
            rel -= rows_k;
        }
        const int j = static_cast<int>(rel % s);
        const int ii = static_cast<int>((rel / s) % s);
        const long long b = rel / ((long long)s * s);
        const int y0 = (ii * h) / s, y1 = ((ii + 1) * h + s - 1) / s;
        const int x0 = (j * w) / s, x1 = ((j + 1) * w + s - 1) / s;
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
        const __half* img = src + b * h * (long long)w * src_ld + c;
        for (int y = y0; y < y1; ++y)
            for (int x = x0; x < x1; ++x) {
                float v[8];
                load8(img + ((long long)y * w + x) * src_ld, v);
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] += v[e];
            }
        const float inv = 1.f / static_cast<float>((y1 - y0) * (x1 - x0));
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] *= inv;
        store8(dst + row * channels + c, acc);
    }
}

// ------------------------------------------------------------------------------------------ segmentation output
// Per output pixel (oy, ox) of [ho, wo]: the logits resized [h4, w4] -> [hn, wn] (first step) and then [hn, wn] ->
// [ho, wo] (second step), both by lerp_src, the first step evaluated at the (up to) four network-size points the second
// step reads, so the network-size logits are never stored; then the first class with the largest value, and
// palette[label] as RGB.  fp32 throughout; logits fp32 [batch, h4, w4, ld] with ld % 4 == 0.
__device__ __forceinline__ float4 lerp4(const float4& a, const float4& b, float la, float lb) {
    return make_float4(la * a.x + lb * b.x, la * a.y + lb * b.y, la * a.z + lb * b.z, la * a.w + lb * b.w);
}

__global__ void __launch_bounds__(256)
seg_output_kernel(const float* __restrict__ logits, int ld, int classes, int h4, int w4, int hn, int wn, int ho, int wo,
                  long long items, const unsigned char* __restrict__ palette, unsigned char* __restrict__ rgb,
                  int* __restrict__ labels) {
    pdl_launch_dependents();
    pdl_wait();
    const float s1h = static_cast<float>(h4) / static_cast<float>(hn), s1w = static_cast<float>(w4) / static_cast<float>(wn);
    const float s2h = static_cast<float>(hn) / static_cast<float>(ho), s2w = static_cast<float>(wn) / static_cast<float>(wo);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        const int ox = static_cast<int>(i % wo);
        const int oy = static_cast<int>((i / wo) % ho);
        const long long b = i / ((long long)ho * wo);
        const Lerp Y = lerp_src(oy, s2h, hn), X = lerp_src(ox, s2w, wn);
        // the first step at network rows Y.i0, Y.i1 and columns X.i0, X.i1
        const Lerp ya = lerp_src(Y.i0, s1h, h4), yb = lerp_src(Y.i1, s1h, h4);
        const Lerp xa = lerp_src(X.i0, s1w, w4), xb = lerp_src(X.i1, s1w, w4);
        const float* img = logits + b * h4 * (long long)w4 * ld;
        const float* ra0 = img + (long long)ya.i0 * w4 * ld;
        const float* ra1 = img + (long long)ya.i1 * w4 * ld;
        const float* rb0 = img + (long long)yb.i0 * w4 * ld;
        const float* rb1 = img + (long long)yb.i1 * w4 * ld;
        const int ca0 = xa.i0 * ld, ca1 = xa.i1 * ld, cb0 = xb.i0 * ld, cb1 = xb.i1 * ld;
        float best = -INFINITY;
        int label = 0;
        for (int c = 0; c < classes; c += 4) {
            // point (row r, column q) of the first step: lr0 * (lq0 * L[r0, q0] + lq1 * L[r0, q1]) + lr1 * (...)
            auto point = [&](const float* r0, const float* r1, const Lerp& lr, int q0, int q1, const Lerp& lq) {
                const float4 a = lerp4(*reinterpret_cast<const float4*>(r0 + q0 + c),
                                       *reinterpret_cast<const float4*>(r0 + q1 + c), lq.l0, lq.l1);
                const float4 d = lerp4(*reinterpret_cast<const float4*>(r1 + q0 + c),
                                       *reinterpret_cast<const float4*>(r1 + q1 + c), lq.l0, lq.l1);
                return lerp4(a, d, lr.l0, lr.l1);
            };
            const float4 p00 = point(ra0, ra1, ya, ca0, ca1, xa), p01 = point(ra0, ra1, ya, cb0, cb1, xb);
            const float4 p10 = point(rb0, rb1, yb, ca0, ca1, xa), p11 = point(rb0, rb1, yb, cb0, cb1, xb);
            const float4 v = lerp4(lerp4(p00, p01, X.l0, X.l1), lerp4(p10, p11, X.l0, X.l1), Y.l0, Y.l1);
            const float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (c + e < classes && vs[e] > best) {
                    best = vs[e];
                    label = c + e;
                }
        }
        rgb[i * 3] = palette[label * 3];
        rgb[i * 3 + 1] = palette[label * 3 + 1];
        rgb[i * 3 + 2] = palette[label * 3 + 2];
        if (labels) labels[i] = label;
    }
}

}  // namespace ctrl

using namespace ctrl;

template <int S>
static int launch_dwconv3(int act, dim3 grid, cudaStream_t stream, const __half* x, const float* weight, const float* bias,
                          const __half* residual, __half* out, long long items, int hi, int wi, int h, int w,
                          int channels) {
    if (act == 0)
        return launched(launch_pdl(dwconv_kernel<3, S, 0>, grid, dim3(256), (size_t)0, stream, x, weight, bias, residual,
                                   out, items, hi, wi, h, w, channels));
    if (act == 1)
        return launched(launch_pdl(dwconv_kernel<3, S, 1>, grid, dim3(256), (size_t)0, stream, x, weight, bias, residual,
                                   out, items, hi, wi, h, w, channels));
    return launched(launch_pdl(dwconv_kernel<3, S, 2>, grid, dim3(256), (size_t)0, stream, x, weight, bias, residual, out,
                               items, hi, wi, h, w, channels));
}

extern "C" int ctrlora_dwconv_act_f16(const void* x, const float* weight, const float* bias, const void* residual,
                                      void* out, int batch, int h, int w, int channels, int k, int stride, int act,
                                      void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    // k = 5 (UniFormer's CBlock attn) runs at stride 1 without activation only
    if (!x || !weight || !bias || !out || batch < 0 || h < 1 || w < 1 || channels < 8 || channels % 8 ||
        (k != 3 && k != 5) || (stride != 1 && stride != 2) || act < 0 || act > 2 || (k == 5 && (stride != 1 || act)) ||
        misaligned_u(x, 16) || misaligned_u(weight, 16) || misaligned_u(bias, 16) || misaligned_u(residual, 16) ||
        misaligned_u(out, 16) || out == x)
        return CTRLORA_ERR_ARG;
    const int ho = h / stride, wo = w / stride;
    const long long items = (long long)batch * ho * wo * (channels / 8);
    if (items == 0) return CTRLORA_OK;
    const dim3 grid(grid_blocks(items, 256, 8192));
    const __half* xs = static_cast<const __half*>(x);
    const __half* rs = static_cast<const __half*>(residual);
    __half* o = static_cast<__half*>(out);
    if (k == 5)
        return launched(launch_pdl(dwconv_kernel<5, 1, 0>, grid, dim3(256), (size_t)0, stream, xs, weight, bias, rs, o,
                                   items, h, w, ho, wo, channels));
    if (stride == 1) return launch_dwconv3<1>(act, grid, stream, xs, weight, bias, rs, o, items, h, w, ho, wo, channels);
    return launch_dwconv3<2>(act, grid, stream, xs, weight, bias, rs, o, items, h, w, ho, wo, channels);
}

extern "C" int ctrlora_dwconv_f16(const void* x, const float* weight, const float* bias, const void* residual, void* out,
                                  int batch, int h, int w, int channels, int k, void* stream_) {
    return ctrlora_dwconv_act_f16(x, weight, bias, residual, out, batch, h, w, channels, k, 1, 0, stream_);
}

extern "C" int ctrlora_resize_bilinear_f16(const void* src, int src_ld, void* dst, int dst_ld, int batch, int hi, int wi,
                                           int ho, int wo, int channels, int accumulate, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!src || !dst || batch < 0 || hi < 1 || wi < 1 || ho < 1 || wo < 1 || channels < 8 || channels % 8 ||
        src_ld < channels || dst_ld < channels || src_ld % 8 || dst_ld % 8 || misaligned_u(src, 16) ||
        misaligned_u(dst, 16))
        return CTRLORA_ERR_ARG;
    const long long items = (long long)batch * ho * wo * (channels / 8);
    if (items == 0) return CTRLORA_OK;
    const float sh = static_cast<float>(hi) / static_cast<float>(ho), sw = static_cast<float>(wi) / static_cast<float>(wo);
    return launched(launch_pdl(resize_bilinear_kernel, dim3(grid_blocks(items, 256, 8192)), dim3(256), (size_t)0, stream,
                               static_cast<const __half*>(src), src_ld, static_cast<__half*>(dst), dst_ld, items, hi, wi,
                               ho, wo, channels, sh, sw, accumulate ? 1 : 0));
}

extern "C" int ctrlora_adaptive_avg_pool_f16(const void* src, int src_ld, void* dst, int batch, int h, int w, int channels,
                                             const int* sizes, int n_sizes, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!src || !dst || !sizes || batch < 0 || h < 1 || w < 1 || channels < 8 || channels % 8 || src_ld < channels ||
        src_ld % 8 || n_sizes < 1 || n_sizes > kMaxPools || misaligned_u(src, 16) || misaligned_u(dst, 16))
        return CTRLORA_ERR_ARG;
    PoolSizes ps{};
    ps.n = n_sizes;
    long long rows = 0;
    for (int k = 0; k < n_sizes; ++k) {
        if (sizes[k] < 1) return CTRLORA_ERR_ARG;
        ps.s[k] = sizes[k];
        rows += (long long)batch * sizes[k] * sizes[k];
    }
    const long long items = rows * (channels / 8);
    if (items == 0) return CTRLORA_OK;
    return launched(launch_pdl(adaptive_avg_pool_kernel, dim3(grid_blocks(items, 256, 8192)), dim3(256), (size_t)0, stream,
                               static_cast<const __half*>(src), src_ld, static_cast<__half*>(dst), items, h, w, channels,
                               batch, ps));
}

extern "C" int ctrlora_seg_output(const float* logits, int ld, int classes, int batch, int h4, int w4, int hn, int wn,
                                  int ho, int wo, const unsigned char* palette, unsigned char* rgb, int* labels,
                                  void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!logits || !palette || !rgb || classes < 1 || ld < (classes + 3) / 4 * 4 || ld % 4 || batch < 0 || h4 < 1 ||
        w4 < 1 || hn < 1 || wn < 1 || ho < 1 || wo < 1 || misaligned_u(logits, 16))
        return CTRLORA_ERR_ARG;
    const long long items = (long long)batch * ho * wo;
    if (items == 0) return CTRLORA_OK;
    return launched(launch_pdl(seg_output_kernel, dim3(grid_blocks(items, 256, 8192)), dim3(256), (size_t)0, stream, logits,
                               ld, classes, h4, w4, hn, wn, ho, wo, items, palette, rgb, labels));
}
