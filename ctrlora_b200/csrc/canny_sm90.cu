// The Canny edge detector (reference: annotator/canny/__init__.py, one call of cv2.Canny(img, low, high) with the
// 3 x 3 aperture and the L1 magnitude).  Two entry points: the classification (gradient, non-maximum suppression and
// the two thresholds) in one tiled kernel, and the hysteresis as connected-component labelling by union-find over the
// candidates in four launches, whatever the image holds.  Integer arithmetic throughout, so the result is cv2's bit for
// bit; the hysteresis output is the union of the 8-connected candidate components that hold a strong pixel, which does
// not depend on the order the atomics link the components in.
#include "common.cuh"
#include "ctrlora_b200.h"

namespace ctrl {

// classify: a kTileW x kTileH output tile per CTA
constexpr int kTileW = 32, kTileH = 16;
constexpr int kClassifyThreads = 256;
constexpr int kPxW = kTileW + 4, kPxH = kTileH + 4;    // uint8 pixels: the tile and a 2-pixel halo, border clamped
constexpr int kMW = kTileW + 2, kMH = kTileH + 2;      // selected magnitudes: the tile and a 1-pixel halo
constexpr int kTg22 = 13573;                           // floor(tan(22.5 deg) * 2^15 + 0.5)

// hysteresis: one pixel per thread, a kLabW x kLabH tile per CTA
constexpr int kLabW = 32, kLabH = 16;
constexpr int kLabThreads = kLabW * kLabH;
constexpr int kStrong = static_cast<int>(0x80000000u);   // a root's label carries this bit when a member is strong
constexpr int kIndex = 0x7fffffff;

// Per pixel of the tile: the 3 x 3 Sobel dx, dy of each channel with the border replicated, m = |dx| + |dy|, the
// channel with the largest m (a later channel wins only when strictly greater); the direction from |dx|, |dy| in
// 2^15 fixed point; the asymmetric non-maximum suppression against magnitudes that are 0 outside the image; then
// class 1 (candidate) when kept and m > lo, 2 (strong) when also m > hi, else 0.
__global__ void __launch_bounds__(kClassifyThreads)
canny_classify_kernel(const unsigned char* __restrict__ img, long long ld, int h, int w, int lo, int hi,
                      unsigned char* __restrict__ cls) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ unsigned char s_px[kPxH][kPxW * 3];
    __shared__ int s_m[kMH][kMW];
    __shared__ short s_dx[kTileH][kTileW], s_dy[kTileH][kTileW];
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH, b = blockIdx.z;
    const unsigned char* src = img + (long long)b * h * ld;
    for (int i = tid; i < kPxH * kPxW * 3; i += kClassifyThreads) {
        const int r = i / (kPxW * 3), c = i - r * (kPxW * 3);
        const int px = c / 3, ch = c - px * 3;
        const int gy = min(max(y0 - 2 + r, 0), h - 1), gx = min(max(x0 - 2 + px, 0), w - 1);
        s_px[r][c] = src[gy * ld + gx * 3 + ch];
    }
    __syncthreads();
    for (int i = tid; i < kMH * kMW; i += kClassifyThreads) {
        const int r = i / kMW, c = i - r * kMW;        // magnitude position (y0 - 1 + r, x0 - 1 + c)
        const int gy = y0 - 1 + r, gx = x0 - 1 + c;
        int best = 0, bdx = 0, bdy = 0;
        if (gy >= 0 && gy < h && gx >= 0 && gx < w) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                // pixel (gy + dy, gx + dx) sits at s_px[r + 1 + dy][(c + 1 + dx) * 3 + ch]
                const unsigned char* up = &s_px[r][c * 3 + ch];
                const unsigned char* mid = &s_px[r + 1][c * 3 + ch];
                const unsigned char* dn = &s_px[r + 2][c * 3 + ch];
                const int dx = (up[6] + 2 * mid[6] + dn[6]) - (up[0] + 2 * mid[0] + dn[0]);
                const int dy = (dn[0] + 2 * dn[3] + dn[6]) - (up[0] + 2 * up[3] + up[6]);
                const int m = abs(dx) + abs(dy);
                if (ch == 0 || m > best) { best = m; bdx = dx; bdy = dy; }
            }
        }
        s_m[r][c] = best;
        if (r >= 1 && r <= kTileH && c >= 1 && c <= kTileW) {
            s_dx[r - 1][c - 1] = static_cast<short>(bdx);
            s_dy[r - 1][c - 1] = static_cast<short>(bdy);
        }
    }
    __syncthreads();
    for (int i = tid; i < kTileH * kTileW; i += kClassifyThreads) {
        const int ty = i / kTileW, tx = i - ty * kTileW;
        const int gy = y0 + ty, gx = x0 + tx;
        if (gy >= h || gx >= w) continue;
        const int r = ty + 1, c = tx + 1;
        const int m = s_m[r][c];
        unsigned char k = 0;
        if (m > lo) {
            const int dx = s_dx[ty][tx], dy = s_dy[ty][tx];
            const int ax = abs(dx), ay = abs(dy) << 15;
            const int tg22x = ax * kTg22;
            bool keep;
            if (ay < tg22x) {
                keep = m > s_m[r][c - 1] && m >= s_m[r][c + 1];
            } else if (ay > tg22x + (ax << 16)) {
                keep = m > s_m[r - 1][c] && m >= s_m[r + 1][c];
            } else if ((dx ^ dy) < 0) {
                keep = m > s_m[r - 1][c + 1] && m > s_m[r + 1][c - 1];
            } else {
                keep = m > s_m[r - 1][c - 1] && m > s_m[r + 1][c + 1];
            }
            if (keep) k = m > hi ? 2 : 1;
        }
        cls[((long long)b * h + gy) * w + gx] = k;
    }
}

// The root of x: labels only ever point to a smaller index, and a root's label is its own index (its kStrong bit set
// once a strong member has been found).  volatile: other CTAs link roots while this one walks.
__device__ __forceinline__ int find_root(const int* lab, int x) {
    const volatile int* l = lab;
    int p = l[x] & kIndex;
    while (p != x) {
        x = p;
        p = l[x] & kIndex;
    }
    return x;
}

// Link the trees of a and b: the larger root is pointed at the smaller one by atomicMin; when another thread has
// linked that root first, retry from where it now points (Playne and Hawick's lock-free union).
__device__ __forceinline__ void unite(int* lab, int a, int b) {
    for (;;) {
        a = find_root(lab, a);
        b = find_root(lab, b);
        if (a == b) return;
        if (a > b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(&lab[b], a);
        if (old == b) return;
        b = old;
    }
}

__device__ __forceinline__ int find_local(const int* s, int x) {
    const volatile int* l = s;
    int p = l[x];
    while (p != x) {
        x = p;
        p = l[x];
    }
    return x;
}

__device__ __forceinline__ void unite_local(int* s, int a, int b) {
    for (;;) {
        a = find_local(s, a);
        b = find_local(s, b);
        if (a == b) return;
        if (a > b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(&s[b], a);
        if (old == b) return;
        b = old;
    }
}

// Launch 1: union-find inside the tile in shared memory (each candidate with its candidate neighbours left, up-left,
// up and up-right that lie in the tile), flattened, then written as global labels: the local root's flat index.  The
// local order (row-major in the tile) follows the global one, so every label points to a smaller-or-equal index.
__global__ void __launch_bounds__(kLabThreads)
canny_label_local_kernel(const unsigned char* __restrict__ cls, int h, int w, int* __restrict__ lab) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ int s[kLabThreads];
    __shared__ unsigned char s_c[kLabH][kLabW];
    const int tx = threadIdx.x, ty = threadIdx.y, t = ty * kLabW + tx;
    const int gx = blockIdx.x * kLabW + tx, gy = blockIdx.y * kLabH + ty;
    const bool in = gx < w && gy < h;
    const long long g = ((long long)blockIdx.z * h + gy) * w + gx;
    const bool cand = in && cls[g] != 0;
    s_c[ty][tx] = cand;
    s[t] = t;
    __syncthreads();
    if (cand) {
        if (tx > 0 && s_c[ty][tx - 1]) unite_local(s, t, t - 1);
        if (ty > 0) {
            if (tx > 0 && s_c[ty - 1][tx - 1]) unite_local(s, t, t - kLabW - 1);
            if (s_c[ty - 1][tx]) unite_local(s, t, t - kLabW);
            if (tx + 1 < kLabW && s_c[ty - 1][tx + 1]) unite_local(s, t, t - kLabW + 1);
        }
    }
    __syncthreads();
    if (!in) return;
    const int r = find_local(s, t);
    const int rx = r % kLabW, ry = r / kLabW;
    lab[g] = static_cast<int>(g - (long long)(ty - ry) * w - (tx - rx));
}

// Launch 2: the pairs that cross tile borders.  A pixel on its tile's left column, top row or right column unites with
// each of its candidate neighbours left, up-left, up and up-right that lies in another tile; together with launch 1
// that covers every 8-connected pair once, the diagonal ones through tile corners included.
__global__ void __launch_bounds__(kLabThreads)
canny_label_border_kernel(const unsigned char* __restrict__ cls, int h, int w, int* __restrict__ lab) {
    pdl_launch_dependents();
    pdl_wait();
    const int tx = threadIdx.x, ty = threadIdx.y;
    if (tx != 0 && ty != 0 && tx != kLabW - 1) return;
    const int gx = blockIdx.x * kLabW + tx, gy = blockIdx.y * kLabH + ty;
    if (gx >= w || gy >= h) return;
    const long long base = (long long)blockIdx.z * h * w;
    const int p = static_cast<int>(base + (long long)gy * w + gx);
    if (!cls[p]) return;
    // neighbour (gy + dy, gx + dx) is in another tile when it leaves this tile's columns or rows
    const int dxs[4] = {-1, -1, 0, 1}, dys[4] = {0, -1, -1, -1};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int nx = gx + dxs[k], ny = gy + dys[k];
        if (nx < 0 || nx >= w || ny < 0) continue;
        if (tx + dxs[k] >= 0 && tx + dxs[k] < kLabW && ty + dys[k] >= 0) continue;  // same tile: launch 1's pair
        const int q = static_cast<int>(base + (long long)ny * w + nx);
        if (cls[q]) unite(lab, p, q);
    }
}

// Launch 3: every candidate's label becomes its root's index, and the root of each strong pixel gets kStrong.  A root
// keeps its own label (only the flag is ORed into it), so walks from other threads still end there.
__global__ void __launch_bounds__(256)
canny_label_flatten_kernel(const unsigned char* __restrict__ cls, long long n, int* __restrict__ lab) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned char c = cls[i];
        if (!c) continue;
        const int x = static_cast<int>(i);
        const int r = find_root(lab, x);
        if (r != x) lab[x] = r;
        if (c == 2) atomicOr(&lab[r], kStrong);
    }
}

// Launch 4: 255 at every candidate whose root carries kStrong, 0 elsewhere.
__global__ void __launch_bounds__(256)
canny_label_output_kernel(const unsigned char* __restrict__ cls, const int* __restrict__ lab, long long n,
                          unsigned char* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        unsigned char v = 0;
        if (cls[i]) v = lab[lab[i] & kIndex] < 0 ? 255 : 0;
        out[i] = v;
    }
}

}  // namespace ctrl

using namespace ctrl;

static bool canny_dims_ok(int batch, int h, int w) {
    return batch >= 0 && h >= 1 && w >= 1 && batch <= 65535 && (long long)batch * h * w < 0x80000000LL;
}

extern "C" int ctrlora_canny_classify(const unsigned char* img, long long ld, int batch, int h, int w, int lo, int hi,
                                      unsigned char* cls, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!img || !cls || !canny_dims_ok(batch, h, w) || ld < 3LL * w || lo > hi) return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    const dim3 grid((w + kTileW - 1) / kTileW, (h + kTileH - 1) / kTileH, batch);
    if (grid.y > 65535) return CTRLORA_ERR_ARG;
    return launched(launch_pdl(canny_classify_kernel, grid, dim3(kClassifyThreads), (size_t)0, stream, img, ld, h, w,
                               lo, hi, cls));
}

extern "C" int ctrlora_canny_hysteresis(const unsigned char* cls, int batch, int h, int w, int* labels_ws,
                                        unsigned char* out, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!cls || !labels_ws || !out || !canny_dims_ok(batch, h, w)) return CTRLORA_ERR_ARG;
    if (batch == 0) return CTRLORA_OK;
    const dim3 grid((w + kLabW - 1) / kLabW, (h + kLabH - 1) / kLabH, batch), block(kLabW, kLabH);
    if (grid.y > 65535) return CTRLORA_ERR_ARG;
    const long long n = (long long)batch * h * w;
    int rc = launched(launch_pdl(canny_label_local_kernel, grid, block, (size_t)0, stream, cls, h, w, labels_ws));
    if (rc) return rc;
    rc = launched(launch_pdl(canny_label_border_kernel, grid, block, (size_t)0, stream, cls, h, w, labels_ws));
    if (rc) return rc;
    const dim3 flat(grid_blocks(n, 256, 8192));
    rc = launched(launch_pdl(canny_label_flatten_kernel, flat, dim3(256), (size_t)0, stream, cls, n, labels_ws));
    if (rc) return rc;
    return launched(launch_pdl(canny_label_output_kernel, flat, dim3(256), (size_t)0, stream, cls,
                               (const int*)labels_ws, n, out));
}
