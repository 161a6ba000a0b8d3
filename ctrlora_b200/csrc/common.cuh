// Shared device helpers for the sm_90a kernels: mbarrier, TMA (cp.async.bulk.tensor), wgmma operand descriptors.
// Everything here is inline PTX for sm_90a; there is no fallback for other architectures.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define CTRLORA_OK 0
#define CTRLORA_ERR_ARG 1
#define CTRLORA_ERR_CUDA 2
#define CTRLORA_ERR_TMAP 3
#define CTRLORA_ERR_UNSUPPORTED 4

namespace ctrl {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must trap (clean launch failure) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) {  // ~2 s at 2 GHz
            printf("ctrlora: mbarrier wait timeout block %d thread %d\n", blockIdx.x, threadIdx.x);
            __trap();
        }
    }
}

// Bounded wait without a function call: ptxas serialises every wgmma of a kernel whose in-flight MMAs could cross a
// call (the printf above), so the wgmma kernels use this form.  A protocol bug still traps instead of hanging.
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity))
        if (clock64() - t0 > 4000000000LL) __trap();
}
// Warp-specialised register split (all four warps of a warpgroup execute the same instruction)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
        "[%2];" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---------------------------------------------------------------- wgmma shared-memory operand descriptors
// Operand tiles are what a TMA box with CU_TENSOR_MAP_SWIZZLE_128B produces: rows of 128 bytes (64 fp16), 8-row
// groups of 1024 B, the 16-byte chunks of row r XOR-permuted by (r & 7).  Tile bases must be 1024-byte aligned.
// K-major (contraction dimension contiguous): SBO = 1024 between 8-row groups, LBO unused; a k16 step is +32 B.
__device__ __forceinline__ uint64_t wgmma_desc_kmajor(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;  // SWIZZLE_128B
    return d;
}
// MN-major (the M / N dimension contiguous, e.g. a [tokens][features] tile contracted over tokens): 64-element atoms
// `lbo_bytes` apart along M / N, 8-row groups 1024 B apart along K; a k16 step is +2048 B.
__device__ __forceinline__ uint64_t wgmma_desc_mnmajor(uint32_t smem_addr, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= static_cast<uint64_t>(1024 >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ float max3f(float a, float b, float c) {
    float r;
    asm("max.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
    return r;
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// Every hot kernel starts with launch_dependents (the next kernel in the stream may begin its prologue: barrier init,
// descriptor prefetch) and executes wait before its first global-memory access.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// cluster launch that also chains programmatically (PDL) onto its predecessor in the stream
template <typename... KArgs>
inline cudaError_t launch_cluster_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                      unsigned cluster_x, KArgs... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cluster_x;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    const char* e = getenv("CTRLORA_PDL");
    cfg.numAttrs = (e && e[0] == '0') ? 1 : 2;
    void* ptrs[] = {(void*)&args...};
    return cudaLaunchKernelExC(&cfg, reinterpret_cast<const void*>(kernel), ptrs);
}

template <typename... KArgs>
inline cudaError_t launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                  unsigned cluster_x, KArgs... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cluster_x;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    void* ptrs[] = {(void*)&args...};
    return cudaLaunchKernelExC(&cfg, reinterpret_cast<const void*>(kernel), ptrs);
}

template <typename... KArgs>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              KArgs... args) {
    static int use_pdl = -1;
    if (use_pdl < 0) {
        const char* e = getenv("CTRLORA_PDL");
        use_pdl = (e && e[0] == '0') ? 0 : 1;
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = use_pdl ? 1 : 0;
    void* ptrs[] = {(void*)&args...};
    return cudaLaunchKernelExC(&cfg, reinterpret_cast<const void*>(kernel), ptrs);
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// sigmoid / SiLU on raw ex2 / rcp (the __expf / __fdividef intrinsics add range-fixup FSETP / FMUL / FSEL sequences:
// ncu counted 38 instructions per GEGLU output element with them, see profiles/README.md)
__device__ __forceinline__ float sigmoid_f(float x) { return fast_rcp(1.0f + fast_exp2(-1.4426950408889634f * x)); }
__device__ __forceinline__ float silu_f(float x) { return x * sigmoid_f(x); }
// exact-erf GELU (F.gelu default).  erf via Abramowitz-Stegun 7.1.26 (|abs err| < 1.5e-7, far below fp16 rounding).
// erf_as(x) for the backward; gelu_erf_f is the fused forward form:
//   gelu(x) = max(x, 0) - |x|/2 * w(|x|),  w(a) = poly(t) * t * exp(-a^2/2),  t = 1 / (1 + p a / sqrt 2)
// with the 1/sqrt(2) and log2(e) factors folded into the constants: 2 MUFU + 13 FMA-pipe instructions, no selects.
__device__ __forceinline__ float erf_as(float x) {
    const float ax = fabsf(x);
    const float t = fast_rcp(fmaf(0.3275911f, ax, 1.0f));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float y = 1.0f - poly * t * fast_exp2(-1.4426950408889634f * ax * ax);
    return copysignf(y, x);
}
__device__ __forceinline__ float gelu_erf_f(float x) {
    const float z = x * 0.84932180028801904f;            // x / sqrt(2) * sqrt(log2 e)
    const float e = fast_exp2(-z * z);                    // exp(-x^2 / 2)
    const float t = fast_rcp(fmaf(0.27273706287f, fabsf(z), 1.0f));  // 1 / (1 + 0.3275911 |x| / sqrt 2)
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float w = poly * t * e;                         // 1 - erf(|x| / sqrt 2)
    return fmaf(-0.5f * fabsf(x), w, fmaxf(x, 0.0f));
}

}  // namespace ctrl

// ---------------------------------------------------------------- clusters
namespace ctrl {
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// ---------------------------------------------------------------- raw shared-address variants for single-thread hot loops
// (the generic->shared conversion and pointer arithmetic are hoisted out of the loop by the caller)
__device__ __forceinline__ bool mbar_try_wait_a(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
static __device__ __noinline__ void mbar_wait_slow_a(uint32_t bar, uint32_t parity) {
    long long t0 = clock64();
    while (!mbar_try_wait_a(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) {
            printf("ctrlora: mbarrier wait timeout block %d thread %d\n", blockIdx.x, threadIdx.x);
            __trap();
        }
    }
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait_a(bar, parity)) return;
    if (mbar_try_wait_a(bar, parity)) return;
    mbar_wait_slow_a(bar, parity);
}
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// (elect_one above) lets the compiler keep the surrounding loop in warp-uniform control flow so that TMA operands live
// in uniform registers; a `lane == 0` branch costs an ELECT + R2UR waterfall per instruction.
__device__ __forceinline__ int uniform_warp_idx() { return __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0); }
// ---------------------------------------------------------------- TMA stores (shared -> global, bulk async-group completion)
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups may still be READING shared memory
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// Spin on mbarrier.test_wait (no hardware suspend): lowest wake-up latency, for waits that sit on a per-tile critical chain.
__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    uint32_t ok;
    long long t0 = 0;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(a), "r"(parity)
            : "memory");
        if (!ok) {
            if (t0 == 0) t0 = clock64();
            else if (clock64() - t0 > 4000000000LL) { printf("ctrlora: mbarrier spin timeout block %d thread %d\n", blockIdx.x, threadIdx.x); __trap(); }
        }
    } while (!ok);
}
// ---------------------------------------------------------------- explicit shared-space 16-byte accesses
// Pointers derived from the aligned dynamic-smem base are generic to the compiler (LD.E / ST.E through the LSU's global
// path, "lg throttle" stalls in the row-math loops); these take a 32-bit shared address and emit LDS / STS.
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ float4 lds128f(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts32f(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
// exp2 on the FMA pipe (Cody-Waite split + degree-3 minimax on [-0.5, 0.5], max relative error 1.1e-4: below fp16's
// half-ulp). The softmax / backward row math is MUFU-bound (16 ex2 per clock per SM); evaluating every fourth
// exponential this way moves a quarter of that load to the otherwise idle FMA pipe (the FlashAttention-4 trick).
__device__ __forceinline__ float exp2_poly3(float x) {
    x = fmaxf(x, -126.0f);
    const float t = x + 12582912.0f;  // 1.5 * 2^23: round(x) lands in the low mantissa bits
    const float f = x - (t - 12582912.0f);
    float p = fmaf(0.05459282f, f, 0.24221784f);
    p = fmaf(p, f, 0.6933686f);
    p = fmaf(p, f, 1.0f);
    return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
// degree 4: max relative error 2.7e-6 in fp32 Horner form (ex2.approx itself: 2.4e-7; fp16 rounding of P: 4.9e-4)
__device__ __forceinline__ float exp2_poly4(float x) {
    x = fmaxf(x, -126.0f);
    const float t = x + 12582912.0f;
    const float f = x - (t - 12582912.0f);
    float p = fmaf(0.009570102f, f, 0.05591786f);
    p = fmaf(p, f, 0.24024744f);
    p = fmaf(p, f, 0.6931218f);
    p = fmaf(p, f, 0.99999928f);
    return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
// nn.ReflectionPad2d's and cv2's BORDER_REFLECT_101 index map: the border pixel is not repeated (needs |offset| < n)
__device__ __forceinline__ int reflect101(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// ---------------------------------------------------------------- host-side launch helpers
// an entry point's status after a launch: the launch's own error, else any error pending from earlier work
inline int launched(cudaError_t e) {
    if (e != cudaSuccess) return CTRLORA_ERR_CUDA;
    return cudaGetLastError() == cudaSuccess ? CTRLORA_OK : CTRLORA_ERR_CUDA;
}
// blocks of a grid-stride kernel over `items` at `per_block` per block, clamped to [1, cap]
inline unsigned grid_blocks(long long items, int per_block, long long cap) {
    const long long blocks = (items + per_block - 1) / per_block;
    return static_cast<unsigned>(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}
}  // namespace ctrl
