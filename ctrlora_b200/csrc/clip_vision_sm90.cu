// The IP-Adapter image encoder's own kernels (reference: app/gradio_ctrlora_style_transfer.py:385-409, which runs
// transformers' CLIPVisionModelWithProjection, and the ViT-H text tower's exact GELU): the patch gather that turns
// CLIPVisionEmbeddings.patch_embedding (Conv2d, kernel = stride = patch, no bias) into one ctrlora_gemm_f16, the
// class + position embedding assembly of the fp32 residual stream, and exact-erf GELU in place on fc1's fp16 output.
// Everything else of the encoder (q|k|v, attention, out_proj, the MLP, the LayerNorms, the projections) reuses the
// existing entry points.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

// ------------------------------------------------------------------------------------------ patch gather
// out[b * P + py * gw + px, c * p * p + kh * p + kw] = pixels[b, c, py * p + kh, px * p + kw]   (pixels [B, C, img_h, img_w],
// grid gh x gw, P = gh * gw; rows and columns beyond p * gh, p * gw are never read), the Conv2d weight's (c, kh, kw)
// order; columns in [channels * p * p, k_pad) are zero.  Each thread writes 8 columns.
template <typename T>
__global__ void __launch_bounds__(256)
patch_gather_kernel(const T* __restrict__ pix, __half* __restrict__ out, long long vecs, int channels, int img_h, int img_w,
                    int grid_h, int grid_w, int patch, int k_pad) {
    pdl_launch_dependents();
    pdl_wait();
    const int per_img = grid_h * grid_w, pp = patch * patch, k = channels * pp;
    const int vecs_per_row = k_pad >> 3;
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < vecs; v += (long long)gridDim.x * blockDim.x) {
        const long long row = v / vecs_per_row;
        const int col0 = static_cast<int>(v % vecs_per_row) * 8;
        const int b = static_cast<int>(row / per_img), p = static_cast<int>(row % per_img);
        const int y0 = (p / grid_w) * patch, x0 = (p % grid_w) * patch;
        __align__(16) __half h[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int col = col0 + e;
            float val = 0.f;
            if (col < k) {
                const int c = col / pp, r = col % pp;
                const long long idx = ((static_cast<long long>(b) * channels + c) * img_h + y0 + r / patch) * img_w + x0 + r % patch;
                val = static_cast<float>(pix[idx]);
            }
            h[e] = __float2half_rn(val);
        }
        reinterpret_cast<uint4*>(out)[v] = *reinterpret_cast<const uint4*>(h);
    }
}

// ------------------------------------------------------------------------------------------ embedding assembly
// out[b * (P + 1) + t, :] = (t == 0 ? class_embedding : patch_out[b * P + t - 1, :]) + position_embedding[t, :]
// (CLIPVisionEmbeddings: cat([class_embeds, patch_embeds]) + position_embedding, one rounded fp32 add).  One warp per row.
__global__ void __launch_bounds__(256)
vision_embed_kernel(const float* __restrict__ patch_out, long long ldp, const float* __restrict__ cls,
                    const float* __restrict__ pos, float* __restrict__ out, int rows, int patches, int cols) {
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const int b = row / (patches + 1), t = row % (patches + 1);
    const float* src = t == 0 ? cls : patch_out + (static_cast<long long>(b) * patches + t - 1) * ldp;
    const float* pe = pos + static_cast<long long>(t) * cols;
    for (int c = lane * 4; c < cols; c += 128) {
        const float4 a = *reinterpret_cast<const float4*>(src + c), p = *reinterpret_cast<const float4*>(pe + c);
        *reinterpret_cast<float4*>(out + static_cast<long long>(row) * cols + c) =
            make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
    }
}

// ------------------------------------------------------------------------------------------ exact GELU
// 0.5 x (1 + erf(x / sqrt 2)) in fp32 (gelu_erf_f), in place on fp16: transformers' GELUActivation, hidden_act "gelu"
__global__ void __launch_bounds__(256) gelu_erf_kernel(__half* __restrict__ x, long long vecs) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < vecs; v += (long long)gridDim.x * blockDim.x) {
        uint4 u = reinterpret_cast<uint4*>(x)[v];
        __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h[e]);
            h[e] = __floats2half2_rn(gelu_erf_f(f.x), gelu_erf_f(f.y));
        }
        reinterpret_cast<uint4*>(x)[v] = u;
    }
}

}  // namespace ctrl

using namespace ctrl;

static int patch_gather_launch(const void* pixels, int pixels_f32, void* out, int batch, int channels, int img_h, int img_w,
                               int patch, int k_pad, cudaStream_t stream) {
    if (!pixels || !out || batch < 0 || channels < 1 || patch < 1 || img_h < patch || img_w < patch ||
        k_pad < channels * patch * patch || k_pad % 8)
        return CTRLORA_ERR_ARG;
    const int grid_h = img_h / patch, grid_w = img_w / patch;
    const long long rows = static_cast<long long>(batch) * grid_h * grid_w, vecs = rows * (k_pad / 8);
    if (vecs == 0) return CTRLORA_OK;
    __half* o = static_cast<__half*>(out);
    if (pixels_f32)
        return launched(launch_pdl(patch_gather_kernel<float>, dim3(grid_blocks(vecs, 256, 4096)), dim3(256), (size_t)0, stream,
                                          static_cast<const float*>(pixels), o, vecs, channels, img_h, img_w, grid_h, grid_w,
                                          patch, k_pad));
    return launched(launch_pdl(patch_gather_kernel<__half>, dim3(grid_blocks(vecs, 256, 4096)), dim3(256), (size_t)0, stream,
                                      static_cast<const __half*>(pixels), o, vecs, channels, img_h, img_w, grid_h, grid_w,
                                      patch, k_pad));
}

extern "C" int ctrlora_clip_patch_gather(const void* pixels, int pixels_f32, void* out, int batch, int channels, int image,
                                         int patch, int k_pad, void* stream_) {
    if (patch < 1 || image % patch) return CTRLORA_ERR_ARG;
    return patch_gather_launch(pixels, pixels_f32, out, batch, channels, image, image, patch, k_pad,
                               reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int ctrlora_patch_gather_hw(const void* pixels, int pixels_f32, void* out, int batch, int channels, int h, int w,
                                       int patch, int k_pad, void* stream_) {
    return patch_gather_launch(pixels, pixels_f32, out, batch, channels, h, w, patch, k_pad,
                               reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int ctrlora_clip_vision_embed(const float* patch_out, long long ldp, const float* class_embedding,
                                         const float* position_embedding, float* out, int batch, int patches, int cols,
                                         void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!patch_out || !class_embedding || !position_embedding || !out || batch < 0 || patches < 1 || cols < 4 || cols % 4 ||
        ldp < cols || ldp % 4)
        return CTRLORA_ERR_ARG;
    const int rows = batch * (patches + 1);
    if (rows == 0) return CTRLORA_OK;
    return launched(launch_pdl(vision_embed_kernel, dim3((rows + 7) / 8), dim3(256), (size_t)0, stream, patch_out, ldp,
                                      class_embedding, position_embedding, out, rows, patches, cols));
}

extern "C" int ctrlora_gelu_f16(void* x, long long n, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || n < 0 || n % 8) return CTRLORA_ERR_ARG;
    const long long vecs = n / 8;
    if (vecs == 0) return CTRLORA_OK;
    return launched(launch_pdl(gelu_erf_kernel, dim3(grid_blocks(vecs, 256, 4096)), dim3(256), (size_t)0, stream,
                                      static_cast<__half*>(x), vecs));
}
