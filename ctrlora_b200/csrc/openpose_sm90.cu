// The OpenPose body estimator's post-process (reference: annotator/openpose/body.py, Body.__call__ :40-138) on the
// device.  The network's stride-8 maps are resampled to the image size through host-built per-axis tables (the two
// cv2.resize calls of the reference composed into one banded matrix per axis), the 18 part heatmaps are smoothed with
// scipy's gaussian_filter(sigma = 3) in float64, their peaks are compacted in (part, y, x) order by a prefix sum, and
// every candidate limb (part A peak, part B peak) is scored against the two PAF channels of its limb in float64.  Only
// the peaks and the per-pair scores and flags go back to the host, which does the greedy matching and the assembly.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

constexpr int kPeakThreads = 256;
constexpr int kPeakPerThread = 8;
constexpr int kPeakChunk = kPeakThreads * kPeakPerThread;  // map elements per block of the peak count / write passes
constexpr int kSmoothMaxRadius = 16;
constexpr int kMaxLimbs = 32;
constexpr int kLimbSamples = 10;  // mid_num

struct ResampleTabs {
    const int* y_start;   // [H]: first source row of output row y
    const double* y_w;    // [H, ty]: weights of source rows y_start[y] ... y_start[y] + ty - 1
    const int* x_start;   // [W]
    const double* x_w;    // [W, tx]
    int ty, tx;
};

// The resampled value of channel c at output pixel (y, x): sum_i wy_i * (sum_j wx_j * m[y0 + i, x0 + j, c]) in float64,
// rounded once to fp32 (the reference's maps are cv2's float32 output).  m: fp32 pixel-major [h8, w8, ld].
__device__ __forceinline__ float resample_at(const float* __restrict__ m, int ld, int w8, int c, const ResampleTabs& t,
                                             int y, int x) {
    const int y0 = __ldg(t.y_start + y), x0 = __ldg(t.x_start + x);
    const double* wy = t.y_w + (long long)y * t.ty;
    const double* wx = t.x_w + (long long)x * t.tx;
    double acc = 0.0;
    for (int i = 0; i < t.ty; ++i) {
        const float* row = m + ((long long)(y0 + i) * w8 + x0) * ld + c;
        double r = 0.0;
        for (int j = 0; j < t.tx; ++j) r = fma(__ldg(wx + j), static_cast<double>(__ldg(row + (long long)j * ld)), r);
        acc = fma(__ldg(wy + i), r, acc);
    }
    return static_cast<float>(acc);
}

// out[c, y, x] for c < channels: the heatmaps the peak search reads, fp32 [channels, H, W]
__global__ void __launch_bounds__(256)
openpose_resample_kernel(const float* __restrict__ m, int ld, int w8, int channels, const ResampleTabs t,
                         float* __restrict__ out, int H, int W) {
    const long long n = (long long)channels * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int x = static_cast<int>(i % W);
        const long long r = i / W;
        const int y = static_cast<int>(r % H), c = static_cast<int>(r / H);
        out[i] = resample_at(m, ld, w8, c, t, y, x);
    }
}

// scipy.ndimage's 'reflect' extension (d c b a | a b c d | d c b a), repeated for lines shorter than the filter
__device__ __forceinline__ int reflect_index(int i, int n) {
    const int period = 2 * n;
    i %= period;
    if (i < 0) i += period;
    return i < n ? i : period - 1 - i;
}

struct SmoothWeights {
    double w[kSmoothMaxRadius + 1];  // w[0]: centre tap, w[j]: the taps at -j and +j
    int radius;
};

// One pass of gaussian_filter's separable correlation (scipy's correlate1d for a symmetric kernel): along the rows
// (ROWS, axis 0) or the columns (axis 1) of `maps` H x W maps, out = in[0] * w0, then += (in[-j] + in[+j]) * w_j for
// j = radius ... 1, each operation rounded in float64 as scipy's C loop does.
template <typename T, bool ROWS>
__global__ void __launch_bounds__(256)
openpose_smooth_kernel(const T* __restrict__ in, double* __restrict__ out, int maps, int H, int W,
                       const __grid_constant__ SmoothWeights g) {
    const long long n = (long long)maps * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int x = static_cast<int>(i % W);
        const long long r = i / W;
        const int y = static_cast<int>(r % H);
        const T* base = in + (r / H) * H * W;
        auto at = [&](int d) -> double {
            return ROWS ? static_cast<double>(base[(long long)reflect_index(y + d, H) * W + x])
                        : static_cast<double>(base[(long long)y * W + reflect_index(x + d, W)]);
        };
        double o = __dmul_rn(at(0), g.w[0]);
        for (int j = g.radius; j >= 1; --j) o = __dadd_rn(o, __dmul_rn(__dadd_rn(at(-j), at(j)), g.w[j]));
        out[i] = o;
    }
}

// body.py :87-95: >= each of the four neighbours (zero outside the map) and > thre
__device__ __forceinline__ bool is_peak(const double* __restrict__ s, int H, int W, int y, int x, double thre) {
    const double v = s[(long long)y * W + x];
    const double up = y > 0 ? s[(long long)(y - 1) * W + x] : 0.0;
    const double dn = y < H - 1 ? s[(long long)(y + 1) * W + x] : 0.0;
    const double lf = x > 0 ? s[(long long)y * W + x - 1] : 0.0;
    const double rt = x < W - 1 ? s[(long long)y * W + x + 1] : 0.0;
    return v >= up && v >= dn && v >= lf && v >= rt && v > thre;
}

// The peak flags of a thread's kPeakPerThread consecutive elements (element e = (part * H + y) * W + x) as a bit mask
__device__ __forceinline__ unsigned peak_bits(const double* __restrict__ s, long long n, int H, int W, long long e0,
                                              double thre) {
    unsigned bits = 0;
    for (int k = 0; k < kPeakPerThread; ++k) {
        const long long e = e0 + k;
        if (e >= n) break;
        const int x = static_cast<int>(e % W);
        const long long r = e / W;
        const int y = static_cast<int>(r % H);
        if (is_peak(s + (r / H) * H * W, H, W, y, x, thre)) bits |= 1u << k;
    }
    return bits;
}

// Exclusive block-wide prefix sum of v over kPeakThreads threads (warp shuffles, then the warp totals); total: the sum
__device__ __forceinline__ int block_exclusive_scan(int v, int* total) {
    __shared__ int warp_sums[kPeakThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    int before = 0, all = 0;
#pragma unroll
    for (int k = 0; k < kPeakThreads / 32; ++k) {
        if (k < wid) before += warp_sums[k];
        all += warp_sums[k];
    }
    __syncthreads();  // warp_sums is reused by the next call
    *total = all;
    return before + incl - v;
}

__global__ void __launch_bounds__(kPeakThreads)
openpose_peak_count_kernel(const double* __restrict__ s, long long n, int H, int W, double thre, int* __restrict__ counts) {
    const long long e0 = (long long)blockIdx.x * kPeakChunk + (long long)threadIdx.x * kPeakPerThread;
    int total;
    block_exclusive_scan(__popc(peak_bits(s, n, H, W, e0, thre)), &total);
    if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// One block: counts[0 .. blocks) -> their exclusive prefix sum in place, the grand total in counts[blocks]
__global__ void __launch_bounds__(kPeakThreads) openpose_peak_scan_kernel(int* __restrict__ counts, int blocks) {
    int carry = 0;
    for (int base = 0; base < blocks; base += kPeakThreads) {
        const int i = base + threadIdx.x;
        const int v = i < blocks ? counts[i] : 0;
        int total;
        const int ex = block_exclusive_scan(v, &total);
        if (i < blocks) counts[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) counts[blocks] = carry;
}

// Each peak at its global id: offsets[block] + the block-local rank.  x, y, part; score = the unsmoothed heatmap.
__global__ void __launch_bounds__(kPeakThreads)
openpose_peak_write_kernel(const double* __restrict__ s, const float* __restrict__ heat, long long n, int H, int W,
                           double thre, const int* __restrict__ offsets, int* __restrict__ px, int* __restrict__ py,
                           int* __restrict__ part, float* __restrict__ score, int capacity) {
    const long long e0 = (long long)blockIdx.x * kPeakChunk + (long long)threadIdx.x * kPeakPerThread;
    const unsigned bits = peak_bits(s, n, H, W, e0, thre);
    int total;
    int id = offsets[blockIdx.x] + block_exclusive_scan(__popc(bits), &total);
    for (int k = 0; k < kPeakPerThread; ++k) {
        if (!(bits & (1u << k))) continue;
        if (id < capacity) {
            const long long e = e0 + k;
            const long long r = e / W;
            px[id] = static_cast<int>(e % W);
            py[id] = static_cast<int>(r % H);
            part[id] = static_cast<int>(r / H);
            score[id] = heat[e];
        }
        ++id;
    }
}

struct LimbTable {
    // per limb: first pair index, first peak of part A, peaks of A, first peak of part B, peaks of B, PAF channel of
    // the x component, PAF channel of the y component
    int d[kMaxLimbs][7];
    int n;
};

// body.py :107-131 for one (limb, i, j) pair, in float64 with every operation rounded as numpy rounds it
__global__ void __launch_bounds__(256)
openpose_limb_kernel(const float* __restrict__ paf, int ld, int w8, const ResampleTabs t, const int* __restrict__ px,
                     const int* __restrict__ py, const __grid_constant__ LimbTable L, long long pairs, int img_h,
                     double thre, double* __restrict__ score, unsigned char* __restrict__ ok) {
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < pairs; q += (long long)gridDim.x * blockDim.x) {
        int k = 0;
        while (k + 1 < L.n && L.d[k + 1][0] <= q) ++k;
        const int* d = L.d[k];
        const int r = static_cast<int>(q - d[0]);
        const int a = d[1] + r / d[4], b = d[3] + r % d[4];
        const int ax = px[a], ay = py[a], bx = px[b], by = py[b];
        const double dx = static_cast<double>(bx - ax), dy = static_cast<double>(by - ay);
        double norm = sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
        norm = fmax(0.001, norm);
        const double ux = __ddiv_rn(dx, norm), uy = __ddiv_rn(dy, norm);
        // np.linspace(start, stop, 10): I * ((stop - start) / 9) + start, the last point exactly stop
        const double sx = __ddiv_rn(dx, 9.0), sy = __ddiv_rn(dy, 9.0);
        double sum = 0.0;
        int above = 0;
        for (int I = 0; I < kLimbSamples; ++I) {
            const double fx = I == kLimbSamples - 1 ? static_cast<double>(bx) : __dadd_rn(__dmul_rn(I, sx), ax);
            const double fy = I == kLimbSamples - 1 ? static_cast<double>(by) : __dadd_rn(__dmul_rn(I, sy), ay);
            const int ix = static_cast<int>(rint(fx)), iy = static_cast<int>(rint(fy));  // round half to even
            const double vx = resample_at(paf, ld, w8, d[5], t, iy, ix);
            const double vy = resample_at(paf, ld, w8, d[6], t, iy, ix);
            const double sm = __dadd_rn(__dmul_rn(vx, ux), __dmul_rn(vy, uy));
            sum = __dadd_rn(sum, sm);
            above += sm > thre;
        }
        const double prior = fmin(__dsub_rn(__ddiv_rn(__dmul_rn(0.5, static_cast<double>(img_h)), norm), 1.0), 0.0);
        const double sc = __dadd_rn(__ddiv_rn(sum, static_cast<double>(kLimbSamples)), prior);
        score[q] = sc;
        ok[q] = above > 0.8 * kLimbSamples && sc > 0.0;
    }
}

static bool tabs_ok(const ResampleTabs& t) { return t.y_start && t.y_w && t.x_start && t.x_w && t.ty >= 1 && t.tx >= 1; }

}  // namespace ctrl

using namespace ctrl;

extern "C" int ctrlora_openpose_resample(const float* maps, int map_ld, int h8, int w8, int channels, const int* y_start,
                                         const double* y_w, int ty, const int* x_start, const double* x_w, int tx,
                                         float* out, int h, int w, void* stream_) {
    if (!maps || !out || channels < 1 || channels > map_ld || h8 < 1 || w8 < 1 || h < 1 || w < 1 || ty > h8 || tx > w8)
        return CTRLORA_ERR_ARG;
    const ResampleTabs t{y_start, y_w, x_start, x_w, ty, tx};
    if (!tabs_ok(t)) return CTRLORA_ERR_ARG;
    const long long n = (long long)channels * h * w;
    openpose_resample_kernel<<<grid_blocks(n, 256, 8192), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(maps, map_ld, w8,
                                                                                                      channels, t, out, h, w);
    return launched(cudaSuccess);
}

extern "C" int ctrlora_openpose_smooth(const float* in, double* tmp, double* out, int maps, int h, int w,
                                       const double* weights, int radius, void* stream_) {
    if (!in || !tmp || !out || !weights || maps < 0 || h < 1 || w < 1 || radius < 0 || radius > kSmoothMaxRadius)
        return CTRLORA_ERR_ARG;
    SmoothWeights g;
    memset(&g, 0, sizeof(g));
    for (int j = 0; j <= radius; ++j) g.w[j] = weights[j];
    g.radius = radius;
    const long long n = (long long)maps * h * w;
    if (n == 0) return CTRLORA_OK;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    openpose_smooth_kernel<float, true><<<grid_blocks(n, 256, 8192), 256, 0, stream>>>(in, tmp, maps, h, w, g);
    openpose_smooth_kernel<double, false><<<grid_blocks(n, 256, 8192), 256, 0, stream>>>(tmp, out, maps, h, w, g);
    return launched(cudaSuccess);
}

extern "C" int ctrlora_openpose_peaks(const double* smoothed, const float* heat, int maps, int h, int w, double thre,
                                      int* ws, long long ws_ints, int* px, int* py, int* part, float* score, int capacity,
                                      void* stream_) {
    if (!smoothed || !heat || !ws || maps < 1 || h < 1 || w < 1 || capacity < 0 ||
        (capacity > 0 && (!px || !py || !part || !score)))
        return CTRLORA_ERR_ARG;
    const long long n = (long long)maps * h * w;
    const long long blocks = (n + kPeakChunk - 1) / kPeakChunk;
    if (blocks + 1 > ws_ints || blocks > 0x7fffffffLL) return CTRLORA_ERR_ARG;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const unsigned nb = static_cast<unsigned>(blocks);
    openpose_peak_count_kernel<<<nb, kPeakThreads, 0, stream>>>(smoothed, n, h, w, thre, ws);
    openpose_peak_scan_kernel<<<1, kPeakThreads, 0, stream>>>(ws, static_cast<int>(blocks));
    openpose_peak_write_kernel<<<nb, kPeakThreads, 0, stream>>>(smoothed, heat, n, h, w, thre, ws, px, py, part, score,
                                                                capacity);
    return launched(cudaSuccess);
}

extern "C" int ctrlora_openpose_limbs(const float* paf, int paf_ld, int h8, int w8, const int* y_start, const double* y_w,
                                      int ty, const int* x_start, const double* x_w, int tx, const int* px, const int* py,
                                      const int* limbs, int n_limbs, long long pairs, int img_h, double thre,
                                      double* score, unsigned char* ok, void* stream_) {
    const ResampleTabs t{y_start, y_w, x_start, x_w, ty, tx};
    if (!paf || !limbs || n_limbs < 1 || n_limbs > kMaxLimbs || pairs < 0 || img_h < 1 || ty > h8 || tx > w8 ||
        !tabs_ok(t))
        return CTRLORA_ERR_ARG;
    if (pairs == 0) return CTRLORA_OK;
    if (!px || !py || !score || !ok) return CTRLORA_ERR_ARG;
    LimbTable L;
    memset(&L, 0, sizeof(L));
    L.n = n_limbs;
    long long next = 0;
    for (int k = 0; k < n_limbs; ++k) {
        for (int e = 0; e < 7; ++e) L.d[k][e] = limbs[7 * k + e];
        // pair ranges follow each other in limb order; every limb holds nA * nB >= 1 pairs and PAF channels < paf_ld
        if (L.d[k][0] != next || L.d[k][2] < 1 || L.d[k][4] < 1 || L.d[k][5] < 0 || L.d[k][5] >= paf_ld ||
            L.d[k][6] < 0 || L.d[k][6] >= paf_ld)
            return CTRLORA_ERR_ARG;
        next += (long long)L.d[k][2] * L.d[k][4];
    }
    if (next != pairs) return CTRLORA_ERR_ARG;
    openpose_limb_kernel<<<grid_blocks(pairs, 256, 8192), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
        paf, paf_ld, w8, t, px, py, L, pairs, img_h, thre, score, ok);
    return launched(cudaSuccess);
}
