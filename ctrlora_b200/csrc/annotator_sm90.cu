// The line-art annotator's own kernels (reference: annotator/lineart/__init__.py, informative-drawings'
// Generator(3, 1, 3)): a tap gather that turns its reflection-padded 7x7 and 3x3 convs and the sub-pixel phases of its
// stride-2 transposed convs into plain ctrlora_gemm_f16 launches, InstanceNorm2d (+ ReLU, + the residual block's add)
// with fixed-order statistics, and the 64 -> 1 output conv fused with the sigmoid and the uint8 quantisation.  The stride-2
// convs reuse ctrlora_im2col_s2_pad_f16; every GEMM is ctrlora_gemm_f16.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

constexpr int kMaxTaps = 64;
struct TapList {
    signed char dy[kMaxTaps], dx[kMaxTaps];
};

// ------------------------------------------------------------------------------------------ tap gather
// dst[b, y, x, t * C + c] = act(src[b, Y(s y + dy_t), X(s x + dx_t), c]) for output pixels (y, x) of [b, h / s, w / s]
// (h, w: the source's size, s: stride 1 or 2), Y / X reflecting or (zero) masking outside the image; columns
// >= taps * C are zero.  act: 0 none, 1 ReLU, 2 LeakyReLU(0.2), in fp32 before the fp16 rounding.  Each thread writes
// 8 columns.  VEC: fp16 pixel-major source with C % 8 == 0, one 16-byte load per thread; otherwise element by element
// from fp16 pixel-major (F32 = false) or fp32 NCHW (F32 = true).
__device__ __forceinline__ float gather_act(float v, int act) {
    return act == 1 ? fmaxf(v, 0.f) : (act == 2 && v < 0.f ? v * 0.2f : v);
}

template <bool VEC, bool F32>
__global__ void __launch_bounds__(256)
tap_gather_kernel(const void* __restrict__ src_, long long ld, __half* __restrict__ dst, int vecs, int h, int w,
                  int channels, const __grid_constant__ TapList taps, int n_taps, int reflect, int k_pad, int stride,
                  int act) {
    // taps is read in place from the parameter bank (__grid_constant__): a by-value copy indexed at run time would be
    // spilled to local memory by every thread; indices are 32-bit (the launch checks vecs < 2^31)
    pdl_launch_dependents();
    pdl_wait();
    const int vecs_per_row = k_pad >> 3, k = n_taps * channels;
    const int ho = h / stride, wo = w / stride;
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < vecs; v += gridDim.x * blockDim.x) {
        const int row = v / vecs_per_row;
        const int col0 = (v - row * vecs_per_row) * 8;
        const int by = row / wo, x = (row - by * wo) * stride;
        const int b = by / ho, y = (by - b * ho) * stride;
        if (VEC) {
            uint4 val = make_uint4(0, 0, 0, 0);
            if (col0 < k) {
                const int t = col0 / channels, c = col0 - t * channels;
                int yy = y + taps.dy[t], xx = x + taps.dx[t];
                bool in = true;
                if (reflect) { yy = reflect101(yy, h); xx = reflect101(xx, w); }
                else in = yy >= 0 && yy < h && xx >= 0 && xx < w;
                if (in) {
                    const __half* s = static_cast<const __half*>(src_) + (((long long)b * h + yy) * w + xx) * ld + c;
                    val = *reinterpret_cast<const uint4*>(s);
                    if (act) {
                        __half2* hv = reinterpret_cast<__half2*>(&val);
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 f = __half22float2(hv[e]);
                            hv[e] = __floats2half2_rn(gather_act(f.x, act), gather_act(f.y, act));
                        }
                    }
                }
            }
            reinterpret_cast<uint4*>(dst)[v] = val;
        } else {
            __align__(16) __half o[8];
            int t = col0 / channels, c = col0 - t * channels;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                float val = 0.f;
                if (t < n_taps) {
                    int yy = y + taps.dy[t], xx = x + taps.dx[t];
                    bool in = true;
                    if (reflect) { yy = reflect101(yy, h); xx = reflect101(xx, w); }
                    else in = yy >= 0 && yy < h && xx >= 0 && xx < w;
                    if (in) {
                        if (F32)
                            val = static_cast<const float*>(src_)[(((long long)b * channels + c) * h + yy) * w + xx];
                        else
                            val = __half2float(static_cast<const __half*>(src_)[(((long long)b * h + yy) * w + xx) * ld + c]);
                        val = gather_act(val, act);
                    }
                }
                o[e] = __float2half_rn(val);
                if (++c == channels) { c = 0; ++t; }
            }
            reinterpret_cast<uint4*>(dst)[v] = *reinterpret_cast<const uint4*>(o);
        }
    }
}

// ------------------------------------------------------------------------------------------ instance norm
// Logical row r of image b (r < rows = HW, or 4 HW for the phases of a stride-2 transposed conv) and where it lives.
// phases: x is [4, B, H, W, C] (phase p = 2 py + px, a [B, H, W, C] GEMM output each), y is [B, 2H, 2W, C] with
// y[b, 2m + py, 2n + px] <- x[p, b, m, n].
__device__ __forceinline__ long long norm_src_row(int b, long long r, int batch, long long hw, int phases) {
    if (!phases) return b * hw + r;
    const unsigned p = static_cast<unsigned>(r) / static_cast<unsigned>(hw);  // r < 4 hw < 2^32 (checked at launch)
    return ((long long)p * batch + b) * hw + (r - p * hw);
}
__device__ __forceinline__ long long norm_dst_row(int b, long long r, long long hw, int w, int phases) {
    if (!phases) return b * hw + r;
    const unsigned p = static_cast<unsigned>(r) / static_cast<unsigned>(hw), pix = static_cast<unsigned>(r - p * hw);
    const unsigned m = pix / static_cast<unsigned>(w), n = pix - m * static_cast<unsigned>(w);
    return (b * 4 * hw) + (2 * m + (p >> 1)) * (2LL * w) + 2 * n + (p & 1);
}

// Per (image, chunk of rows, channel) partial sums of (x - x[row 0]) and its square, stored [image, channel, chunk]:
// thread t owns the 8 channels of vector t % (C / 8) and rows t / (C / 8), + lanes, ... of the chunk; the lanes are then
// summed in lane order (at 512 channels, lanes = 4 and each thread sums two channels).  The shift by the image's first row keeps the one-pass variance accurate when |mean| >> std.
// Fixed partition, fixed order, no atomics.
__global__ void __launch_bounds__(256)
inorm_partial_kernel(const __half* __restrict__ x, float2* __restrict__ part, int batch, long long hw, int channels,
                     int phases, long long rows, long long chunk_rows, int chunks) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float2 red[256][8];
    const int b = blockIdx.y, ck = blockIdx.x;
    const int cv = channels >> 3, lanes = 256 / cv;
    const int vec = threadIdx.x % cv, lane = threadIdx.x / cv;
    float k[8], s[8], q[8];
    {
        const uint4 u = reinterpret_cast<const uint4*>(x + norm_src_row(b, 0, batch, hw, phases) * channels)[vec];
        const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(hh[e]);
            k[2 * e] = f.x; k[2 * e + 1] = f.y;
        }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    const long long r0 = ck * chunk_rows, r1 = r0 + chunk_rows < rows ? r0 + chunk_rows : rows;
#pragma unroll 4
    for (long long r = r0 + lane; r < r1; r += lanes) {
        const uint4 u = reinterpret_cast<const uint4*>(x + norm_src_row(b, r, batch, hw, phases) * channels)[vec];
        const __half2* hh = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(hh[e]);
            const float d0 = f.x - k[2 * e], d1 = f.y - k[2 * e + 1];
            s[2 * e] += d0; s[2 * e + 1] += d1;
            q[2 * e] = fmaf(d0, d0, q[2 * e]); q[2 * e + 1] = fmaf(d1, d1, q[2 * e + 1]);
        }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) red[threadIdx.x][e] = make_float2(s[e], q[e]);
    __syncthreads();
    for (int c = threadIdx.x; c < channels; c += 256) {
        const int v = c >> 3, e = c & 7;
        float2 acc = red[v][e];
        for (int l = 1; l < lanes; ++l) {
            const float2 p = red[l * cv + v][e];
            acc.x += p.x; acc.y += p.y;
        }
        part[((long long)b * channels + c) * chunks + ck] = acc;
    }
}

// stats[b, c] = (mean, 1 / sqrt(biased var + eps)): one warp per (image, channel); lane l sums chunks l, l + 32, ...
// in order, then a fixed xor tree across the lanes
__global__ void __launch_bounds__(256)
inorm_finalize_kernel(const __half* __restrict__ x, const float2* __restrict__ part, float2* __restrict__ stats, int batch,
                      long long hw, int channels, int phases, long long rows, int chunks, float eps) {
    pdl_launch_dependents();
    pdl_wait();
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= batch * channels) return;
    const int b = i / channels, c = i % channels;
    const float2* p = part + (long long)i * chunks;
    float s = 0.f, q = 0.f;
#pragma unroll 4
    for (int ck = lane; ck < chunks; ck += 32) {
        const float2 v = p[ck];
        s += v.x; q += v.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (lane) return;
    const float n = static_cast<float>(rows);
    const float ms = s / n;
    const float var = fmaxf(q / n - ms * ms, 0.f);
    const float k = __half2float(x[norm_src_row(b, 0, batch, hw, phases) * channels + c]);
    stats[i] = make_float2(k + ms, 1.f / sqrtf(var + eps));
}

// y = relu?((x - mean) * rstd) + residual?, 8 channels per thread, fp32 math, one fp16 rounding
__global__ void __launch_bounds__(256)
inorm_apply_kernel(const __half* __restrict__ x, const __half* __restrict__ res, __half* __restrict__ y,
                   const float2* __restrict__ stats, int batch, long long hw, int w, int channels, int phases, long long rows,
                   int relu) {
    pdl_launch_dependents();
    pdl_wait();
    const int cv = channels >> 3;
    const long long vecs = (long long)batch * rows * cv;
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < vecs; v += (long long)gridDim.x * blockDim.x) {
        const int c0 = static_cast<int>(v % cv) * 8;
        const long long br = v / cv;
        const int b = static_cast<int>(br / rows);
        const long long r = br % rows;
        const uint4 xi = *reinterpret_cast<const uint4*>(x + norm_src_row(b, r, batch, hw, phases) * channels + c0);
        const long long drow = norm_dst_row(b, r, hw, w, phases) * channels + c0;
        uint4 ri = make_uint4(0, 0, 0, 0);
        if (res) ri = *reinterpret_cast<const uint4*>(res + drow);
        const __half2* xh = reinterpret_cast<const __half2*>(&xi);
        const __half2* rh = reinterpret_cast<const __half2*>(&ri);
        const float2* st = stats + (long long)b * channels + c0;
        uint4 out;
        __half2* oh = reinterpret_cast<__half2*>(&out);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(xh[e]);
            const float2 m0 = st[2 * e], m1 = st[2 * e + 1];
            float a = (f.x - m0.x) * m0.y, c = (f.y - m1.x) * m1.y;
            if (relu) { a = fmaxf(a, 0.f); c = fmaxf(c, 0.f); }
            if (res) {
                const float2 rr = __half22float2(rh[e]);
                a += rr.x; c += rr.y;
            }
            oh[e] = __floats2half2_rn(a, c);
        }
        *reinterpret_cast<uint4*>(y + drow) = out;
    }
}

// ------------------------------------------------------------------------------------------ output conv
// ReflectionPad2d(3) + Conv2d(C -> 1, 7) + Sigmoid on the CUDA cores: a 16 x 16 block of outputs per CTA, one per thread;
// the 22 x 22 input window is staged channel-pair-planar in shared memory 16 channels at a time (consecutive threads read
// consecutive words), the chunk's weights alongside.  fp32 accumulation; u8 = (uint8)clip(sigmoid * 255, 0, 255), the
// fp32 multiply and the truncation of numpy's `(line * 255.0).clip(0, 255).astype(np.uint8)`.
constexpr int kOT = 16, kOK = 7, kOP = 3, kOW = kOT + kOK - 1, kOC = 16;
__global__ void __launch_bounds__(256)
lineart_out_kernel(const __half* __restrict__ x, const float* __restrict__ wt, const float* __restrict__ bias,
                   float* __restrict__ out, unsigned char* __restrict__ out_u8, int h, int w, int channels) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ __half2 tile[kOC / 2][kOW][kOW];
    __shared__ float wsm[kOK * kOK][kOC];
    const int b = blockIdx.z, ty = threadIdx.x / kOT, tx = threadIdx.x % kOT;
    const int y0 = blockIdx.y * kOT, x0 = blockIdx.x * kOT;
    const __half* xb = x + (long long)b * h * w * channels;
    float acc = 0.f;
    for (int c0 = 0; c0 < channels; c0 += kOC) {
        __syncthreads();
        for (int i = threadIdx.x; i < kOW * kOW * (kOC / 2); i += 256) {
            const int cp = i % (kOC / 2), px = (i / (kOC / 2)) % kOW, py = i / (kOC / 2 * kOW);
            const int yy = reflect101(min(y0 + py - kOP, h - 1 + kOP), h), xx = reflect101(min(x0 + px - kOP, w - 1 + kOP), w);
            tile[cp][py][px] = reinterpret_cast<const __half2*>(xb + ((long long)yy * w + xx) * channels + c0)[cp];
        }
        for (int i = threadIdx.x; i < kOK * kOK * kOC; i += 256) wsm[i / kOC][i % kOC] = wt[(i / kOC) * channels + c0 + i % kOC];
        __syncthreads();
#pragma unroll 1
        for (int ky = 0; ky < kOK; ++ky) {
#pragma unroll
            for (int kx = 0; kx < kOK; ++kx) {
                const float* wk = wsm[ky * kOK + kx];
#pragma unroll
                for (int cp = 0; cp < kOC / 2; ++cp) {
                    const float2 v = __half22float2(tile[cp][ty + ky][tx + kx]);
                    acc = fmaf(v.x, wk[2 * cp], acc);
                    acc = fmaf(v.y, wk[2 * cp + 1], acc);
                }
            }
        }
    }
    const int oy = y0 + ty, ox = x0 + tx;
    if (oy >= h || ox >= w) return;
    const float s = 1.f / (1.f + expf(-(acc + bias[0])));
    const long long o = ((long long)b * h + oy) * w + ox;
    out[o] = s;
    if (out_u8) {
        const float q = fminf(fmaxf(s * 255.f, 0.f), 255.f);
        out_u8[o] = static_cast<unsigned char>(q);
    }
}

// ------------------------------------------------------------------------------------------ anime output conv
// Anime2Sketch's outermost up path: ReLU over the two halves [skip | up] (each fp16 [B, h, w, half], half = C / 2),
// ConvTranspose2d(C -> 1, 4, stride 2, padding 1) + bias, tanh, then * scale + shift as two fp32 roundings (the
// detector's `* 127.5 + 127.5`).  Output pixel (2m + py, 2n + px) reads input rows m + dy through kernel rows ky for the
// (dy, ky) of kAnimeRows[py] (oy = 2 iy - 1 + ky), the same for columns: 4 taps x C channels.  A CTA computes 16 x 16
// outputs, one per thread, from a 10 x 10 input window staged channel-pair-planar in shared memory (ReLU applied, zero
// outside the image); the weights sit channel-major [C][16] so the four phases of a warp read four banks.
constexpr int kAT = 16, kAW = kAT / 2 + 2, kAMaxC = 128;
__global__ void __launch_bounds__(256)
lineart_anime_out_kernel(const __half* __restrict__ skip, const __half* __restrict__ up, const float* __restrict__ wt,
                         const float* __restrict__ bias, float* __restrict__ out, int h, int w, int channels, float scale,
                         float shift) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ __half2 tile[kAMaxC / 2][kAW][kAW];
    __shared__ float wsm[kAMaxC * 16];
    const int b = blockIdx.z, ty = threadIdx.x / kAT, tx = threadIdx.x % kAT;
    const int pairs = channels / 2, half = channels / 2, hp = half / 2;  // channel pairs in all, channels and pairs per half
    const int m0 = blockIdx.y * (kAT / 2) - 1, n0 = blockIdx.x * (kAT / 2) - 1;  // input origin of the window
    for (int i = threadIdx.x; i < kAW * kAW * pairs; i += 256) {
        const int cp = i % pairs, px = (i / pairs) % kAW, py = i / (pairs * kAW);
        const int yy = m0 + py, xx = n0 + px;
        __half2 v = __floats2half2_rn(0.f, 0.f);
        if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
            const __half* src = cp < hp ? skip : up;
            v = reinterpret_cast<const __half2*>(src + (((long long)b * h + yy) * w + xx) * half)[cp < hp ? cp : cp - hp];
            v = __hmax2(v, __floats2half2_rn(0.f, 0.f));
        }
        tile[cp][py][px] = v;
    }
    for (int i = threadIdx.x; i < channels * 16; i += 256) wsm[i] = wt[i];
    __syncthreads();
    const int py = ty & 1, px = tx & 1;
    // window coordinates of input row m (= ty / 2 + 1) and column n; tap a of phase py: (dy, ky)
    const int wy = (ty >> 1) + 1, wx = (tx >> 1) + 1;
    const int dy0 = py ? 1 : 0, ky0 = py ? 0 : 1, dy1 = py ? 0 : -1, ky1 = py ? 2 : 3;
    const int dx0 = px ? 1 : 0, kx0 = px ? 0 : 1, dx1 = px ? 0 : -1, kx1 = px ? 2 : 3;
    float acc = 0.f;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
        const int dy = a ? dy1 : dy0, ky = a ? ky1 : ky0;
#pragma unroll
        for (int bb = 0; bb < 2; ++bb) {
            const int dx = bb ? dx1 : dx0, kx = bb ? kx1 : kx0;
            const float* wk = wsm + ky * 4 + kx;
#pragma unroll 8
            for (int cp = 0; cp < pairs; ++cp) {
                const float2 v = __half22float2(tile[cp][wy + dy][wx + dx]);
                acc = fmaf(v.x, wk[(2 * cp) * 16], acc);
                acc = fmaf(v.y, wk[(2 * cp + 1) * 16], acc);
            }
        }
    }
    const int oy = blockIdx.y * kAT + ty, ox = blockIdx.x * kAT + tx;
    if (oy >= 2 * h || ox >= 2 * w) return;
    const float t = tanhf(acc + bias[0]);
    out[((long long)b * 2 * h + oy) * (2LL * w) + ox] = __fadd_rn(__fmul_rn(t, scale), shift);
}

// rows per statistics chunk: at most 1024 chunks per image, at least 64 rows each (a function of the image alone, so a
// batch of B gives each image the statistics a batch of 1 gives it)
constexpr int kNormMaxChunks = 1024;
static long long inorm_chunk_rows(long long rows) {
    long long c = (rows + kNormMaxChunks - 1) / kNormMaxChunks;
    return c < 64 ? 64 : c;
}

}  // namespace ctrl

using namespace ctrl;

static int tap_gather_launch(const void* src, int src_f32_nchw, long long ld, void* dst, int batch, int h, int w,
                             int channels, const int* taps, int n_taps, int reflect, int k_pad, int stride, int act,
                             void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!src || !dst || !taps || batch < 0 || h < 1 || w < 1 || channels < 1 || n_taps < 1 || n_taps > kMaxTaps ||
        k_pad % 8 || k_pad < n_taps * channels || (!src_f32_nchw && ld < channels) || (stride != 1 && stride != 2) ||
        h % stride || w % stride || act < 0 || act > 2)
        return CTRLORA_ERR_ARG;
    TapList tl;
    memset(&tl, 0, sizeof(tl));
    for (int t = 0; t < n_taps; ++t) {
        const int dy = taps[2 * t], dx = taps[2 * t + 1];
        // reflection needs |offset| < size (nn.ReflectionPad2d's pad < H, W); masked offsets only have to fit the list
        if (reflect ? (dy <= -h || dy >= h || dx <= -w || dx >= w) : (dy < -127 || dy > 127 || dx < -127 || dx > 127))
            return CTRLORA_ERR_ARG;
        tl.dy[t] = static_cast<signed char>(dy);
        tl.dx[t] = static_cast<signed char>(dx);
    }
    const long long vecs = (long long)batch * (h / stride) * (w / stride) * (k_pad / 8);
    if (vecs == 0) return CTRLORA_OK;
    if (vecs >= (1LL << 31)) return CTRLORA_ERR_UNSUPPORTED;
    __half* d = static_cast<__half*>(dst);
    const bool vec = !src_f32_nchw && channels % 8 == 0 && ld % 8 == 0 && !(reinterpret_cast<uintptr_t>(src) & 15);
    if (vec)
        return launched(launch_pdl(tap_gather_kernel<true, false>, dim3(grid_blocks(vecs, 256, 8192)), dim3(256), (size_t)0, stream,
                                         src, ld, d, (int)vecs, h, w, channels, tl, n_taps, reflect, k_pad, stride, act));
    if (src_f32_nchw)
        return launched(launch_pdl(tap_gather_kernel<false, true>, dim3(grid_blocks(vecs, 256, 8192)), dim3(256), (size_t)0, stream,
                                         src, ld, d, (int)vecs, h, w, channels, tl, n_taps, reflect, k_pad, stride, act));
    return launched(launch_pdl(tap_gather_kernel<false, false>, dim3(grid_blocks(vecs, 256, 8192)), dim3(256), (size_t)0, stream,
                                     src, ld, d, (int)vecs, h, w, channels, tl, n_taps, reflect, k_pad, stride, act));
}

extern "C" int ctrlora_tap_gather_f16(const void* src, int src_f32_nchw, long long ld, void* dst, int batch, int h, int w,
                                      int channels, const int* taps, int n_taps, int reflect, int k_pad, void* stream_) {
    return tap_gather_launch(src, src_f32_nchw, ld, dst, batch, h, w, channels, taps, n_taps, reflect, k_pad, 1, 0, stream_);
}

extern "C" int ctrlora_tap_gather_act_f16(const void* src, int src_f32_nchw, long long ld, void* dst, int batch, int h,
                                          int w, int channels, const int* taps, int n_taps, int reflect, int k_pad,
                                          int stride, int act, void* stream_) {
    return tap_gather_launch(src, src_f32_nchw, ld, dst, batch, h, w, channels, taps, n_taps, reflect, k_pad, stride, act,
                             stream_);
}

extern "C" int ctrlora_instance_norm_f16(const void* x, const void* residual, void* y, float* ws, long long ws_floats,
                                         int batch, int h, int w, int channels, int phases, int relu, float eps,
                                         void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !y || !ws || batch < 0 || h < 1 || w < 1 || channels < 64 || channels % 64 || 512 % channels ||
        (phases != 0 && phases != 1) || ws_floats < 2LL * batch * channels * (kNormMaxChunks + 1) ||
        (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15) ||
        (reinterpret_cast<uintptr_t>(residual) & 15) || (reinterpret_cast<uintptr_t>(ws) & 7))
        return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    const long long hw = (long long)h * w, rows = hw * (phases ? 4 : 1);
    if (rows >= (1LL << 32)) return CTRLORA_ERR_UNSUPPORTED;
    const long long chunk_rows = inorm_chunk_rows(rows);
    const int chunks = static_cast<int>((rows + chunk_rows - 1) / chunk_rows);
    float2* part = reinterpret_cast<float2*>(ws);
    float2* stats = part + (long long)batch * chunks * channels;
    const __half* xh = static_cast<const __half*>(x);
    int rc = launched(launch_pdl(inorm_partial_kernel, dim3(chunks, batch), dim3(256), (size_t)0, stream, xh, part,
                                       batch, hw, channels, phases, rows, chunk_rows, chunks));
    if (rc) return rc;
    rc = launched(launch_pdl(inorm_finalize_kernel, dim3((batch * channels + 7) / 8), dim3(256), (size_t)0, stream,
                                   xh, (const float2*)part, stats, batch, hw, channels, phases, rows, chunks, eps));
    if (rc) return rc;
    return launched(launch_pdl(inorm_apply_kernel, dim3(grid_blocks((long long)batch * rows * (channels / 8), 256, 8192)), dim3(256),
                                     (size_t)0, stream, xh, static_cast<const __half*>(residual), static_cast<__half*>(y),
                                     (const float2*)stats, batch, hw, w, channels, phases, rows, relu));
}

extern "C" int ctrlora_lineart_out_f16(const void* x, const float* weight, const float* bias, float* out,
                                       unsigned char* out_u8, int batch, int h, int w, int channels, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !weight || !bias || !out || batch < 0 || h <= kOP || w <= kOP || channels < kOC || channels % kOC ||
        (reinterpret_cast<uintptr_t>(x) & 3))
        return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    if (batch > 65535) return CTRLORA_ERR_UNSUPPORTED;
    const dim3 grid((w + kOT - 1) / kOT, (h + kOT - 1) / kOT, batch);
    return launched(launch_pdl(lineart_out_kernel, grid, dim3(256), (size_t)0, stream, static_cast<const __half*>(x),
                                     weight, bias, out, out_u8, h, w, channels));
}

extern "C" int ctrlora_lineart_anime_out_f16(const void* skip, const void* up, const float* weight, const float* bias,
                                             float* out, int batch, int h, int w, int channels, float scale, float shift,
                                             void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!skip || !up || !weight || !bias || !out || batch < 0 || h < 1 || w < 1 || channels < 4 || channels % 4 ||
        channels > kAMaxC || (reinterpret_cast<uintptr_t>(skip) & 3) || (reinterpret_cast<uintptr_t>(up) & 3))
        return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    if (batch > 65535) return CTRLORA_ERR_UNSUPPORTED;
    const dim3 grid((2 * w + kAT - 1) / kAT, (2 * h + kAT - 1) / kAT, batch);
    return launched(launch_pdl(lineart_anime_out_kernel, grid, dim3(256), (size_t)0, stream,
                                     static_cast<const __half*>(skip), static_cast<const __half*>(up), weight, bias, out, h,
                                     w, channels, scale, shift));
}
