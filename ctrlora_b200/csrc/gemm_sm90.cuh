// Kernel-side parameter block of the wgmma implicit-GEMM kernel (see gemm_sm90.cu).
#pragma once
#include "common.cuh"

namespace ctrl {

constexpr int GEMM_BM = 128;            // two consumer warpgroups x wgmma M = 64
constexpr int GEMM_BK = 64;             // 64 fp16 = 128 B = one SWIZZLE_128B row
constexpr int GEMM_MAX_BN = 320;        // N of one tile (GEGLU: value half + gate half); 160 accumulators per thread.
                                        // A 320-column tile is two m64n160 MMAs and two 160-row B boxes (TMA boxes
                                        // are at most 256 rows); every UNet width is a multiple of 320
constexpr int GEMM_MAX_STAGES = 8;
constexpr int GEMM_A_BYTES = GEMM_BM * GEMM_BK * 2;   // 16 KiB
constexpr int GEMM_THREADS = 384;       // warpgroup 0: TMA producer (one thread), warpgroups 1-2: wgmma + epilogue
constexpr int GEMM_CONSUMERS = 256;
constexpr int GEMM_PRODUCER_REGS = 40;  // setmaxnreg split: 128 * 40 + 256 * 232 <= 64 K registers
constexpr int GEMM_CONSUMER_REGS = 232;
// Shared memory: [epilogue slots][operand ring][barriers].  The host divides GEMM_SMEM_DATA between the two per tile
// width (GemmKParams::epi_slots, stages).
constexpr int GEMM_SMEM_DATA = 225 * 1024;
constexpr int GEMM_EPI_COLS = 64;                     // row-per-thread epilogue: 64 rows x 64 fp32 columns per warpgroup
constexpr int GEMM_EPI_BYTES = 2 * 64 * GEMM_EPI_COLS * 4;  // 32 KiB, 16-byte chunks XOR-swizzled by row
// TMA epilogue: a slot holds one slab of the output tile, 128 rows x 64 (or 32) fp16 columns in the layout of a
// SWIZZLE_128B (SWIZZLE_64B) box.  The residual slab is loaded into it, the result is written over it and stored from it.
constexpr int GEMM_MAX_SLOTS = 8;
constexpr int GEMM_SMEM_BYTES = GEMM_SMEM_DATA + 1024 /*align slack*/ + 512 /*barriers*/;

struct GemmKParams {
    // tile geometry over the (B, H, W) pixel grid; a plain [M, K] matrix is B=1, H=1, W=M
    int W, H, Bn;
    int bw, bh, nb;                 // TMA box of one 128-row tile: nb * bh * bw == 128
    int tiles_w, tiles_h, tiles_b;  // ceil-div of the dims above by the box
    int N;                          // output columns
    int BN;                         // wgmma N of one tile (GEGLU: value half + gate half)
    int n_tiles;
    int taps, kw, pad;              // filter taps (1 or 9), filter width, zero padding
    int kchunks;                    // ceil(Cin / 64) per tap
    int kchunks2;                   // extra 1x1 segment from the second operand pair (0 = none)
    int geglu;                      // 1: weights are [2N, K]; out = value * gelu(gate)
    int stages, stage_bytes;        // TMA ring: stage = A tile (16 KiB) + B tile (BN * 128 B, 1 KiB aligned); 3 at BN 320
    int epi_slots;                  // epilogue slots in front of the ring (GEMM_EPI_BYTES or more)
    int tma_tiles;                  // whole tiles [0, tma_tiles) run the TMA epilogue, every later unit the row-per-thread one
    // persistent schedule: work unit u < tiles_whole is output tile u over the whole K range; the units after it are
    // the remaining tiles split `splits` ways along K (partial sums meet in `ws`, fp32; the self-cleaning counter of
    // the tile picks the last-arriving CTA, which sums the slices in slice order and runs the epilogue)
    int units, tiles_whole;
    int splits, kiters_per_split;
    float* ws;
    unsigned int* counters;
    // epilogue
    void* out[3];
    int seg_width;                  // 0: single output; else column n goes to out[n / seg_width]
    int transposed[3];              // store segment as [img, head, d, tok_pad] (V^T for attention)
    int ldc;
    int out_f32;
    const float* bias;              // [N] (GEGLU: [2N])
    const float* rowbias;           // [images, rowbias_ld]  per-image additive term (time embedding)
    int rows_per_img;
    int rowbias_ld;
    int residual_f32;
    const __half* residual;         // [M, ldr]
    int ldr;
    float out_scale;
    int head_dim, tok_pad;
    __half* dup_out;               // transposed segments are ALSO stored row-major here (training keeps natural V)
    int dup_ld;
    // grouped launch: tiles of images >= group_b (0 = off) take the second weight maps, bias_g[1] and rowbias_g[1]
    // (rows from image img - rb_img_off); [0] are bias and rowbias, and so are [1] when the launch is not grouped.
    // Indexed in parameter space, so that the 320-column tiles hold no extra pointer in registers.
    int group_b;
    int rb_img_off;
    const float* bias_g[2];
    const float* rowbias_g[2];
    int relu;                       // 1: max(v, 0), 2: min(max(v, 0), 6) last; 3: max(v, 0) before the residual
};

}  // namespace ctrl
