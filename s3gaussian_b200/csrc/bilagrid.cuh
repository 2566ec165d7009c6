// bilagrid.cuh - per-image bilateral-grid colour correction (Wang et al., "Bilateral Guided Radiance Field
// Processing", SIGGRAPH 2024), restating gsplat's lib_bilagrid:
//   slice()                 -> bilagrid_slice_forward_kernel, and its autograd backward -> bilagrid_gather_kernel +
//                              bilagrid_sum_kernel;
//   total_variation_loss()  -> bilagrid_tv_forward_kernel + bilagrid_tv_reduce_kernel, bilagrid_tv_backward_kernel.
// Grids are [N, 12, L, GY, GX] float32; channel c is entry (c / 4, c % 4) of a 3x4 affine colour matrix.  Images are
// [B, 3, H, W].  No float atomics: every sum is taken in a fixed order, so each result repeats bit for bit.
#pragma once
#include <cstdint>

namespace s3g {

constexpr int BG_MAX_IDS = 512;         // image ids per launch (kernel-parameter array); larger batches loop
constexpr int BG_THREADS = 256;         // slice forward
constexpr int BG_GATHER_THREADS = 128;  // grid-gradient gather: one private accumulator column per thread
constexpr int BG_LEVEL_CHUNK = 8;       // luminance levels one gather CTA accumulates (shared: 8*12*129*4 B)
constexpr int BG_PIX_PER_CTA = 4096;    // pixels of a cell's support one gather CTA walks
constexpr int BG_TV_THREADS = 256;
constexpr int BG_TV_BLOCKS = 1024;      // fixed, so the TV partition (and its rounding) does not depend on the device

struct BgIds { int id[BG_MAX_IDS]; };

struct BgShape {
    int L, GY, GX, H, W;
};

// one coordinate of grid_sample(align_corners=True, padding_mode="border"): clamp to [0, size-1], floor corner i0 and
// the fraction f; corner i0 + 1 (weight f) exists when i0 + 1 < size
struct BgAxis { int i0; float f; };
__device__ __forceinline__ BgAxis bg_axis(float v, int size) {
    v = fminf(fmaxf(v, 0.f), (float)(size - 1));
    BgAxis a;
    a.i0 = min((int)floorf(v), size - 1);
    a.f = v - (float)a.i0;
    return a;
}

// the pixel-centre coordinates and the luminance guide of pixel (i, j) with colour (r, g, b); zraw is unclamped
struct BgCoord { BgAxis x, y, z; float zraw; };
__device__ __forceinline__ BgCoord bg_coord(const BgShape& s, int i, int j, float r, float g, float b) {
    BgCoord c;
    c.x = bg_axis(((float)j + 0.5f) / (float)s.W * (float)(s.GX - 1), s.GX);
    c.y = bg_axis(((float)i + 0.5f) / (float)s.H * (float)(s.GY - 1), s.GY);
    c.zraw = (0.299f * r + 0.587f * g + 0.114f * b) * (float)(s.L - 1);
    c.z = bg_axis(c.zraw, s.L);
    return c;
}

// trilinear A[12] of one grid at c, and (want_dz) dA/dz: the difference of the two z-planes' bilinear values
template <bool want_dz>
__device__ __forceinline__ void bg_sample(const float* __restrict__ grid, const BgShape& s, const BgCoord& c,
                                          float A[12], float dAdz[12]) {
    const int x1 = min(c.x.i0 + 1, s.GX - 1), y1 = min(c.y.i0 + 1, s.GY - 1), z1 = min(c.z.i0 + 1, s.L - 1);
    const int plane = s.GY * s.GX, cs = s.L * plane;
    const int o00 = c.y.i0 * s.GX + c.x.i0, o01 = c.y.i0 * s.GX + x1, o10 = y1 * s.GX + c.x.i0, o11 = y1 * s.GX + x1;
    const float w00 = (1.f - c.y.f) * (1.f - c.x.f), w01 = (1.f - c.y.f) * c.x.f;
    const float w10 = c.y.f * (1.f - c.x.f), w11 = c.y.f * c.x.f;
    const int za = c.z.i0 * plane, zb = z1 * plane;
#pragma unroll
    for (int ch = 0; ch < 12; ++ch) {
        const float* g = grid + ch * cs;
        const float a = w00 * __ldg(g + za + o00) + w01 * __ldg(g + za + o01) + w10 * __ldg(g + za + o10) +
                        w11 * __ldg(g + za + o11);
        const float b = w00 * __ldg(g + zb + o00) + w01 * __ldg(g + zb + o01) + w10 * __ldg(g + zb + o10) +
                        w11 * __ldg(g + zb + o11);
        A[ch] = (1.f - c.z.f) * a + c.z.f * b;
        if (want_dz) dAdz[ch] = b - a;
    }
}

// ---- slice forward: one thread per pixel, blockIdx.y the image ---------------------------------------------------
__global__ void __launch_bounds__(BG_THREADS)
bilagrid_slice_forward_kernel(BgShape s, const float* __restrict__ grids, const BgIds ids,
                              const float* __restrict__ rgb, float* __restrict__ out) {
    const int HW = s.H * s.W;
    const int p = blockIdx.x * BG_THREADS + threadIdx.x;
    if (p >= HW) return;
    const int b = blockIdx.y;
    const size_t base = (size_t)b * 3 * HW + p;
    const float r = __ldg(rgb + base), g = __ldg(rgb + base + HW), bl = __ldg(rgb + base + 2 * HW);
    const int i = p / s.W, j = p - i * s.W;
    const BgCoord c = bg_coord(s, i, j, r, g, bl);
    float A[12], unused[12];
    bg_sample<false>(grids + (size_t)ids.id[b] * 12 * s.L * s.GY * s.GX, s, c, A, unused);
    out[base] = A[0] * r + A[1] * g + A[2] * bl + A[3];
    out[base + HW] = A[4] * r + A[5] * g + A[6] * bl + A[7];
    out[base + 2 * HW] = A[8] * r + A[9] * g + A[10] * bl + A[11];
}

// ---- slice backward --------------------------------------------------------------------------------------------------
// The grid gradient of cell (l, gy, gx) sums w(l, gy, gx; pixel) * dA(pixel) over the pixels whose trilinear stencil
// reaches it, dA = grad_out (x) [r, g, b, 1].  Only the pixels whose x lies in (gx - 1, gx + 1) and whose y lies in
// (gy - 1, gy + 1) can: the cell column's support, a rectangle.  One CTA takes one column, one slice `split` of its
// support rectangle (BG_PIX_PER_CTA pixels in row-major order) and one chunk of BG_LEVEL_CHUNK luminance levels.
// Each thread adds its pixels' contributions into its own shared-memory column of [levels][12] accumulators; the
// columns are then summed in thread order and written as one partial per (column, split).  bilagrid_sum_kernel adds
// the partials in split order.  The order of every addition is fixed by the shapes alone.
// grad_rgb is computed by the CTA of the pixel's home column (x.i0, y.i0) in level chunk 0: every pixel has exactly
// one.  It is A[:, :3]^T grad_out plus the luminance-guide term (dL/dz) (L - 1) (0.299, 0.587, 0.114), the latter 0
// where zraw <= 0 or zraw >= L - 1 (torch's border rule).
struct BgGather {
    int splits, chunk;       // support slices per column, pixels per slice
    int nzc;                 // level chunks
};

__device__ __forceinline__ void bg_support(int g, int size, int extent, int& lo, int& hi) {
    if (size == 1) { lo = 0; hi = extent - 1; return; }
    // pixel centres p with (p + 0.5) (size - 1) / extent in (g - 1, g + 1), widened by one pixel each side; the
    // weight test in the loop is exact
    const double k = (double)extent / (double)(size - 1);
    lo = max(0, (int)floor((g - 1) * k - 0.5) - 1);
    hi = min(extent - 1, (int)ceil((g + 1) * k - 0.5) + 1);
}

__device__ __forceinline__ float bg_weight(const BgAxis& a, int g) {
    return (a.i0 == g ? 1.f - a.f : 0.f) + (a.i0 + 1 == g ? a.f : 0.f);
}

__global__ void __launch_bounds__(BG_GATHER_THREADS)
bilagrid_gather_kernel(BgShape s, BgGather q, const float* __restrict__ grids, const BgIds ids,
                       const float* __restrict__ rgb, const float* __restrict__ grad_out, float* __restrict__ grad_rgb,
                       float* __restrict__ partial) {
    extern __shared__ float acc[];          // [lc * 12][BG_GATHER_THREADS + 1]
    constexpr int T = BG_GATHER_THREADS, STRIDE = T + 1;
    const int col = blockIdx.x / q.splits, split = blockIdx.x - col * q.splits;
    const int gy = col / s.GX, gx = col - gy * s.GX;
    const int b = blockIdx.y / q.nzc, zc = blockIdx.y - b * q.nzc;
    const int l_lo = zc * BG_LEVEL_CHUNK, lc = min(BG_LEVEL_CHUNK, s.L - l_lo);
    const int tid = threadIdx.x;
    for (int o = 0; o < lc * 12; ++o) acc[o * STRIDE + tid] = 0.f;

    int jlo, jhi, ilo, ihi;
    bg_support(gx, s.GX, s.W, jlo, jhi);
    bg_support(gy, s.GY, s.H, ilo, ihi);
    const int nx = jhi - jlo + 1, n = nx * (ihi - ilo + 1);
    const int k0 = split * q.chunk, k1 = min(n, k0 + q.chunk);
    const int HW = s.H * s.W;
    const float* grid = grids + (size_t)ids.id[b] * 12 * s.L * s.GY * s.GX;
    for (int k = k0 + tid; k < k1; k += T) {
        const int i = ilo + k / nx, j = jlo + k % nx;
        const size_t base = (size_t)b * 3 * HW + (size_t)i * s.W + j;
        const float r = __ldg(rgb + base), g = __ldg(rgb + base + HW), bl = __ldg(rgb + base + 2 * HW);
        const float go0 = __ldg(grad_out + base), go1 = __ldg(grad_out + base + HW), go2 = __ldg(grad_out + base + 2 * HW);
        const BgCoord c = bg_coord(s, i, j, r, g, bl);
        const float go[3] = {go0, go1, go2}, aug[4] = {r, g, bl, 1.f};
        if (grad_rgb && zc == 0 && c.x.i0 == gx && c.y.i0 == gy) {
            float A[12], dAdz[12];
            bg_sample<true>(grid, s, c, A, dAdz);
            float dz = 0.f;
#pragma unroll
            for (int ch = 0; ch < 12; ++ch) dz += go[ch >> 2] * aug[ch & 3] * dAdz[ch];
            dz = (c.zraw > 0.f && c.zraw < (float)(s.L - 1)) ? dz * (float)(s.L - 1) : 0.f;
#pragma unroll
            for (int m = 0; m < 3; ++m) {
                const float coef = m == 0 ? 0.299f : (m == 1 ? 0.587f : 0.114f);
                grad_rgb[base + (size_t)m * HW] = A[m] * go0 + A[4 + m] * go1 + A[8 + m] * go2 + dz * coef;
            }
        }
        const float wxy = bg_weight(c.x, gx) * bg_weight(c.y, gy);
        if (wxy == 0.f) continue;
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int l = c.z.i0 + t - l_lo;
            if (l < 0 || l >= lc || c.z.i0 + t >= s.L) continue;
            const float w = wxy * (t == 0 ? 1.f - c.z.f : c.z.f);
            float* a = acc + l * 12 * STRIDE + tid;
#pragma unroll
            for (int ch = 0; ch < 12; ++ch) a[ch * STRIDE] += w * (go[ch >> 2] * aug[ch & 3]);
        }
    }
    __syncthreads();
    float* out = partial + ((((size_t)blockIdx.y * s.GY * s.GX) + col) * q.splits + split) * (BG_LEVEL_CHUNK * 12);
    for (int o = tid; o < lc * 12; o += T) {
        const float* a = acc + o * STRIDE;
        float sum = 0.f;
        for (int t = 0; t < T; ++t) sum += a[t];
        out[o] = sum;
    }
}

// grad_grids[ids[b], ch, l, gy, gx] = sum over splits (in order) of the partials; one thread per written element
__global__ void bilagrid_sum_kernel(BgShape s, BgGather q, int B, const BgIds ids, const float* __restrict__ partial,
                                    float* __restrict__ grad_grids) {
    const int plane = s.GY * s.GX, cs = s.L * plane;
    const long long total = (long long)B * 12 * cs;
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int b = (int)(e / (12 * cs));
    const int r = (int)(e - (long long)b * 12 * cs);
    const int ch = r / cs, l = (r - ch * cs) / plane, col = r - ch * cs - l * plane;
    const int zc = l / BG_LEVEL_CHUNK, ll = l - zc * BG_LEVEL_CHUNK;
    const float* p = partial + (((size_t)(b * q.nzc + zc) * plane + col) * q.splits) * (BG_LEVEL_CHUNK * 12) + ll * 12 + ch;
    float sum = 0.f;
    for (int k = 0; k < q.splits; ++k) sum += p[(size_t)k * BG_LEVEL_CHUNK * 12];
    grad_grids[(size_t)ids.id[b] * 12 * cs + r] = sum;
}

// ---- total variation -------------------------------------------------------------------------------------------------
// tv = (1/N) sum_axes sum (g[+1 along the axis] - g)^2 / count_axis; inv[a] = 1 / count_axis, 0 for an axis of size 1.
struct BgTv {
    long long n;             // N * 12 * L * GY * GX
    int L, GY, GX;
    double inv[3];           // x, y, z (level)
    double invN;
};

__global__ void __launch_bounds__(BG_TV_THREADS)
bilagrid_tv_forward_kernel(BgTv t, const float* __restrict__ g, double* __restrict__ partial) {
    __shared__ double red[BG_TV_THREADS / 32];
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (long long e = (long long)blockIdx.x * BG_TV_THREADS + threadIdx.x; e < t.n; e += (long long)gridDim.x * BG_TV_THREADS) {
        const int x = (int)(e % t.GX), y = (int)((e / t.GX) % t.GY), l = (int)((e / ((long long)t.GX * t.GY)) % t.L);
        const float v = g[e];
        if (x + 1 < t.GX) { const float d = g[e + 1] - v; sx += (double)(d * d); }
        if (y + 1 < t.GY) { const float d = g[e + t.GX] - v; sy += (double)(d * d); }
        if (l + 1 < t.L) { const float d = g[e + (long long)t.GX * t.GY] - v; sz += (double)(d * d); }
    }
    double v = sx * t.inv[0] + sy * t.inv[1] + sz * t.inv[2];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double sum = 0.0;
        for (int w = 0; w < BG_TV_THREADS / 32; ++w) sum += red[w];
        partial[blockIdx.x] = sum;
    }
}

__global__ void bilagrid_tv_reduce_kernel(int nblocks, double invN, const double* __restrict__ partial,
                                          float* __restrict__ loss) {
    __shared__ double red[32];
    double v = 0.0;
    for (int k = threadIdx.x; k < nblocks; k += blockDim.x) v += partial[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double sum = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) sum += red[w];
        loss[0] = (float)(sum * invN);
    }
}

// grad[e] = gscale / N * sum_axes 2 inv_axis ((g[e] - g[e-1]) [e has a predecessor] - (g[e+1] - g[e]) [a successor])
__global__ void __launch_bounds__(BG_TV_THREADS)
bilagrid_tv_backward_kernel(BgTv t, const float* __restrict__ g, const float* __restrict__ gscale,
                            float* __restrict__ grad) {
    const long long e = (long long)blockIdx.x * BG_TV_THREADS + threadIdx.x;
    if (e >= t.n) return;
    const int x = (int)(e % t.GX), y = (int)((e / t.GX) % t.GY), l = (int)((e / ((long long)t.GX * t.GY)) % t.L);
    const float v = g[e];
    const long long step[3] = {1, t.GX, (long long)t.GX * t.GY};
    const int pos[3] = {x, y, l}, size[3] = {t.GX, t.GY, t.L};
    float sum = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        float d = 0.f;
        if (pos[a] > 0) d += v - g[e - step[a]];
        if (pos[a] + 1 < size[a]) d -= g[e + step[a]] - v;
        sum += (float)(2.0 * t.inv[a]) * d;
    }
    grad[e] = __ldg(gscale) * (float)t.invN * sum;
}

}  // namespace s3g
