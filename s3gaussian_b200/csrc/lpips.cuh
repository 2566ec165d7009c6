// lpips.cuh - LPIPS v0.1 with the AlexNet backbone (lpipsPyTorch/modules/{lpips,networks,utils}.py) on the device.
//
// Convolutions are implicit GEMMs on the Hopper warpgroup tensor cores, in the decoder's arithmetic (deform_tc.cuh):
// 3xTF32 (hi*hi + hi*lo + lo*hi) with fp32 accumulators.
//   M = output pixels of every image of the call (the N images of x, then the N of y), N = output channels,
//   K = kh * kw * Cin.  CTA = 128 threads = one warpgroup = a 128-pixel x 64-channel output tile (two M = 64 halves of
//   wgmma m64n64k8); thread r gathers the im2col row of pixel r.  K runs in chunks of 32: the chunk's A (128 x 32) and
//   B (64 x 32) hi/lo operands sit in shared memory in the canonical K-major layout (umma.cuh); two stages, so the
//   gather of chunk c + 1 runs while the wgmmas of chunk c do.  Bias and ReLU are applied in the epilogue.
//   * Layer 1 reads the caller's [N,3,H,W] images and z-scores them in its gather, (v - shift) / scale with a true
//     division, so the zero padding lands on the z-scored tensor; its K order is PyTorch's (c, ky, kx), 363 padded
//     to 384.
//   * Layers 2-5 read internal channels-last (HWC) activations; K order (ky, kx, c), so a 32-wide chunk is 32
//     consecutive channels of one input pixel (every Cin is a multiple of 32): eight 16-byte loads, or zeros in the
//     padding.
// Weights are prepared once per model (lpips_prep_kernel): each layer becomes [Cout / 64][Kpad / 32] tiles of
// 64 x 32 canonical hi | lo (tf32 round-to-nearest split), 16 KB each, copied per chunk with cp.async.
// Max-pool (3/2, no padding, floor) is a channels-last kernel of its own.
// Taps: one warp per pixel pair normalises both feature vectors over channels, weighs the squared difference with
// the lin weights and sums it; blocks write double partials, and one fixed-order double reduction writes each
// layer's mean over its grid (summed over the images) and the total.  No atomics: two calls are bitwise equal.
// The weight preparation and the convolution tile take the backbone as a table (LpAlex here, LpVgg in lpips_vgg.cuh);
// the tap and reduction kernels are the same for every backbone.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "umma.cuh"

namespace s3g {

constexpr int LP_LAYERS = 5;                             // taps (every LPIPS backbone here has five)
constexpr int LP_BM = 128, LP_BK = 32;
constexpr int LP_THREADS = 128;
constexpr int LP_A_FLOATS = LP_BM * LP_BK;               // one operand part (hi or lo) of A
// BN = output channels of a CTA's tile, chosen per convolution by the network's table
__host__ __device__ constexpr int lp_tile_floats(int BN) { return 2 * BN * LP_BK; }   // a prepared weight tile: hi | lo
__host__ __device__ constexpr int lp_stage_floats(int BN) { return 2 * LP_A_FLOATS + lp_tile_floats(BN); }
// two stages: 96 KB at BN = 64 (two CTAs per SM), 128 KB at BN = 128 (one)
__host__ __device__ constexpr int lp_smem_bytes(int BN) { return 2 * lp_stage_floats(BN) * 4; }
constexpr int LP_TAP_WARPS = 8, LP_TAP_PIX = 8;          // tap kernel: 8 warps x 8 pixels per block

// A backbone is a table of its convolutions, taken as a template argument by the weight preparation and the
// convolution tile: input and output channels, kernel size, stride, padding and the tile's BN of convolution l.
// AlexNet: `features` convolutions 0, 3, 6, 8, 10 (VGG16: lpips_vgg.cuh)
struct LpAlex {
    static constexpr int CONVS = 5;
    __host__ __device__ static constexpr int cin(int l) { return l == 0 ? 3 : l == 1 ? 64 : l == 2 ? 192 : l == 3 ? 384 : 256; }
    __host__ __device__ static constexpr int cout(int l) { return l == 0 ? 64 : l == 1 ? 192 : l == 2 ? 384 : 256; }
    __host__ __device__ static constexpr int ks(int l) { return l == 0 ? 11 : l == 1 ? 5 : 3; }
    __host__ __device__ static constexpr int stride(int l) { return l == 0 ? 4 : 1; }
    __host__ __device__ static constexpr int pad(int l) { return l <= 1 ? 2 : 1; }
    __host__ __device__ static constexpr int bn(int) { return 64; }
};

template <class Net> __host__ __device__ constexpr int lp_k(int l) { return Net::ks(l) * Net::ks(l) * Net::cin(l); }
template <class Net> __host__ __device__ constexpr int lp_kpad(int l) { return (lp_k<Net>(l) + LP_BK - 1) / LP_BK * LP_BK; }
// floats of convolution l's prepared weights: [Cout / BN][Kpad / 32] tiles
template <class Net> __host__ __device__ constexpr int lp_prep_floats(int l) { return 2 * Net::cout(l) * lp_kpad<Net>(l); }

// hi = x as is (the tensor core reads its tf32 bits), lo = the truncated remainder (deform.cuh's split_tf32)
__device__ __forceinline__ void lp_split(float x, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(x);
    lo = __float_as_uint(x - __uint_as_float(hi & 0xffffe000u));
}

// ---- weight preparation ------------------------------------------------------------------------------------------
template <class Net>
struct LpPrepArgs {
    const float* w[Net::CONVS];   // [Cout][Cin][k][k], PyTorch layout
    float* dst[Net::CONVS];       // lp_prep_floats<Net>(l) floats of prepared tiles
};
// blockIdx.y = layer; element (co, k) of the padded [Cout][Kpad] matrix in the kernel's K order
template <class Net>
__global__ void __launch_bounds__(256) lpips_prep_kernel(const __grid_constant__ LpPrepArgs<Net> p) {
    const int l = blockIdx.y;
    const int Cin = Net::cin(l), KS = Net::ks(l), K = lp_k<Net>(l), KP = lp_kpad<Net>(l), KC = KP / LP_BK;
    const int BN = Net::bn(l);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Net::cout(l) * KP; e += gridDim.x * blockDim.x) {
        const int co = e / KP, k = e - co * KP;
        float v = 0.f;
        if (k < K) {
            int src = k;                                  // layer 1: (c, ky, kx) is PyTorch's own order
            if (l > 0) {                                  // (ky, kx, c) -> (c, ky, kx)
                const int tap = k / Cin, c = k - tap * Cin;
                src = c * KS * KS + tap;
            }
            v = __ldg(p.w[l] + (size_t)co * K + src);
        }
        uint32_t hi, lo;
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(v));
        const float r = v - __uint_as_float(hi);
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
        float* t = p.dst[l] + (size_t)((co / BN) * KC + k / LP_BK) * lp_tile_floats(BN);
        const int ci = umma::canon_idx(co % BN, k % LP_BK, LP_BK);
        t[ci] = __uint_as_float(hi);
        t[BN * LP_BK + ci] = __uint_as_float(lo);
    }
}

// Dgrad weights of AlexNet's convolutions 1..4 (blockIdx.y + 1): B'[ci][k'] with k' = (ky', kx', co) is
// w[co][ci][KS-1-ky'][KS-1-kx'], the flipped, transposed kernel, as [Cin / 64][KS*KS*Cout / 32] hi | lo tiles
// (lpips_dgrad_kernel's K order: 32 consecutive output channels of one tap per chunk).  Layer 0's dgrad runs on the
// CUDA cores from the PyTorch layout (lpips_dgrad0_kernel).
__global__ void __launch_bounds__(256) lpips_prep_dgrad_kernel(const __grid_constant__ LpPrepArgs<LpAlex> p) {
    constexpr int BN = 64;
    const int l = blockIdx.y + 1;
    const int Cin = LpAlex::cin(l), Cout = LpAlex::cout(l), KS = LpAlex::ks(l), K = KS * KS * Cout, KC = K / LP_BK;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Cin * K; e += gridDim.x * blockDim.x) {
        const int ci = e / K, k = e - ci * K;
        const int tap = k / Cout, co = k - tap * Cout;
        const int ky = KS - 1 - tap / KS, kx = KS - 1 - tap % KS;
        const float v = __ldg(p.w[l] + (((size_t)co * Cin + ci) * KS + ky) * KS + kx);
        uint32_t hi, lo;
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(v));
        const float r = v - __uint_as_float(hi);
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
        float* t = p.dst[l] + (size_t)((ci / BN) * KC + k / LP_BK) * lp_tile_floats(BN);
        const int idx = umma::canon_idx(ci % BN, k % LP_BK, LP_BK);
        t[idx] = __uint_as_float(hi);
        t[BN * LP_BK + idx] = __uint_as_float(lo);
    }
}

// ---- convolution -------------------------------------------------------------------------------------------------
struct LpConvArgs {
    const float* in;        // layers 2-5: [2N][H][W][Cin] channels-last
    const float* x;         // layer 1: images 0..N-1, [N][3][H][W]
    const float* y;         // layer 1: images N..2N-1
    int N;                  // images per input (layer 1)
    int H, W;               // input size
    int Ho, Wo;             // output size
    int M;                  // 2N * Ho * Wo
    const float* wprep;     // this layer's prepared tiles
    const float* bias;      // [Cout]
    float* out;             // [2N][Ho][Wo][Cout] channels-last, ReLU applied
};

__device__ __forceinline__ void lp_cp16(float* sdst, const float* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(umma::smem_u32(sdst)), "l"(gsrc) : "memory");
}

// One 128 x BN output tile of Net's convolution L (DG = false), or of the input gradient of convolution L >= 1
// (DG = true).  The dgrad of a stride-1 "same" convolution is itself one: input dY [NI][H][W][Cout], output dX
// [NI][H][W][Cin], the same KS and PAD, the kernel flipped and transposed (lpips_prep_dgrad_kernel), no bias and no
// ReLU.
template <class Net, int L, bool DG>
__device__ __forceinline__ void lp_conv_tile(const LpConvArgs& a) {
    static_assert(!DG || (L > 0 && Net::stride(L) == 1 && 2 * Net::pad(L) == Net::ks(L) - 1), "dgrad: stride-1 same conv");
    constexpr int Cin = DG ? Net::cout(L) : Net::cin(L), Cout = DG ? Net::cin(L) : Net::cout(L);
    constexpr int KS = Net::ks(L), S = Net::stride(L), PAD = Net::pad(L);
    constexpr int K = KS * KS * Cin, KC = (K + LP_BK - 1) / LP_BK;
    constexpr int BN = Net::bn(L), B_FLOATS = BN * LP_BK, TILE_FLOATS = lp_tile_floats(BN), STAGE_FLOATS = lp_stage_floats(BN);
    static_assert(Cout % BN == 0 && (L == 0 || Cin % LP_BK == 0), "tile shape");
    constexpr uint32_t SBO = (LP_BK / 4) * 128u, MHALF = 8u * SBO;
    extern __shared__ __align__(128) float s_lp[];
    const int tid = threadIdx.x;
    const int m = blockIdx.x * LP_BM + tid;
    const bool valid = m < a.M;
    const int hw = a.Ho * a.Wo;
    const int img = valid ? m / hw : 0;
    const int pix = valid ? m - img * hw : 0;
    const int oy = pix / a.Wo, ox = pix - oy * a.Wo;
    const int iy0 = oy * S - PAD, ix0 = ox * S - PAD;
    const float* wtiles = a.wprep + (size_t)blockIdx.y * KC * TILE_FLOATS;
    const float* src = nullptr;     // layer 1: channel 0 of this pixel's image
    if constexpr (!DG && L == 0) src = (img < a.N ? a.x + (size_t)img * 3 * a.H * a.W : a.y + (size_t)(img - a.N) * 3 * a.H * a.W);

    // this thread's 32 A values of chunk c (zero outside the image, past K and past M)
    float v[LP_BK];
    auto gather = [&](int c) {
        const int k0 = c * LP_BK;
        if constexpr (!DG && L == 0) {
#pragma unroll
            for (int j = 0; j < LP_BK; ++j) {
                const int k = k0 + j;
                const int ch = k / (KS * KS), t = k - ch * (KS * KS), ky = t / KS, kx = t - ky * KS;
                const int iy = iy0 + ky, ix = ix0 + kx;
                // the float32 buffers of networks.py:41-44
                const float shift = ch == 0 ? -.030f : ch == 1 ? -.088f : -.188f;
                const float scale = ch == 0 ? .458f : ch == 1 ? .448f : .450f;
                float z = 0.f;
                if (valid && k < K && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W)
                    z = __fdiv_rn(__fsub_rn(__ldg(src + ((size_t)ch * a.H + iy) * a.W + ix), shift), scale);
                v[j] = z;
            }
        } else {
            const int tap = k0 / Cin, c0 = k0 - tap * Cin, ky = tap / KS, kx = tap - ky * KS;
            const int iy = iy0 + ky, ix = ix0 + kx;
            const bool in = valid && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
            const float4* p = reinterpret_cast<const float4*>(a.in + (((size_t)img * a.H + (in ? iy : 0)) * a.W + (in ? ix : 0)) * Cin + c0);
#pragma unroll
            for (int j = 0; j < LP_BK / 4; ++j) {
                const float4 q = in ? __ldg(p + j) : make_float4(0.f, 0.f, 0.f, 0.f);
                v[4 * j] = q.x; v[4 * j + 1] = q.y; v[4 * j + 2] = q.z; v[4 * j + 3] = q.w;
            }
        }
    };
    // A values -> hi/lo operand tiles of `stage`; the chunk's weight tile -> the stage's B by cp.async
    auto stage_in = [&](int c, int stage) {
        float* st = s_lp + stage * STAGE_FLOATS;
        const float* wt = wtiles + (size_t)c * TILE_FLOATS;
#pragma unroll
        for (int j = 0; j < TILE_FLOATS / 4 / LP_THREADS; ++j)
            lp_cp16(st + 2 * LP_A_FLOATS + 4 * (tid + j * LP_THREADS), wt + 4 * (tid + j * LP_THREADS));
        asm volatile("cp.async.commit_group;" ::: "memory");
#pragma unroll
        for (int j = 0; j < LP_BK; j += 4) {
            uint32_t h[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) lp_split(v[j + i], h[i], lo[i]);
            const int ci = umma::canon_idx(tid, j, LP_BK);
            *reinterpret_cast<uint4*>(st + ci) = make_uint4(h[0], h[1], h[2], h[3]);
            *reinterpret_cast<uint4*>(st + LP_A_FLOATS + ci) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
    };

    float acc[2][BN / 2];
    gather(0);
    stage_in(0, 0);
    for (int c = 0; c < KC; ++c) {
        asm volatile("cp.async.wait_all;" ::: "memory");
        umma::fence_async_smem();
        __syncthreads();
        const float* st = s_lp + (c & 1) * STAGE_FLOATS;
        const uint32_t a_hi = umma::smem_u32(st), a_lo = a_hi + LP_A_FLOATS * 4u;
        const uint32_t b_hi = a_hi + 2u * LP_A_FLOATS * 4u, b_lo = b_hi + B_FLOATS * 4u;
        umma::fence_regs(acc[0]); umma::fence_regs(acc[1]);
        umma::wgmma_fence();
#pragma unroll
        for (int k0 = 0; k0 < LP_BK; k0 += 8) {
            const uint32_t off = (uint32_t)(k0 / 4) * 128u;
            const uint64_t dbh = umma::make_smem_desc(b_hi + off, 128, SBO), dbl = umma::make_smem_desc(b_lo + off, 128, SBO);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint64_t dah = umma::make_smem_desc(a_hi + h * MHALF + off, 128, SBO);
                const uint64_t dal = umma::make_smem_desc(a_lo + h * MHALF + off, 128, SBO);
                umma::wgmma_tf32<BN>(acc[h], dal, dbh, c > 0 || k0 > 0);
                umma::wgmma_tf32<BN>(acc[h], dah, dbl, true);
                umma::wgmma_tf32<BN>(acc[h], dah, dbh, true);
            }
        }
        umma::wgmma_commit();
        // the other stage was last read by chunk c - 1's wgmmas, complete since that iteration's wait
        if (c + 1 < KC) {
            gather(c + 1);
            stage_in(c + 1, (c + 1) & 1);
        }
        umma::wgmma_wait_all();
        umma::fence_regs(acc[0]); umma::fence_regs(acc[1]);
    }
    // epilogue: + bias, ReLU (forward only), channels-last store (fragment layout, umma.cuh)
    const int n0 = blockIdx.y * BN;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int i = 0; i < BN / 2; i += 2) {
            const int row = blockIdx.x * LP_BM + 64 * h + umma::frag_row(i);
            const int col = n0 + umma::frag_col(i);
            if (row < a.M) {
                float2 o = make_float2(acc[h][i], acc[h][i + 1]);
                if constexpr (!DG) {
                    const float b0 = __ldg(a.bias + col), b1 = __ldg(a.bias + col + 1);
                    o = make_float2(fmaxf(o.x + b0, 0.f), fmaxf(o.y + b1, 0.f));
                }
                *reinterpret_cast<float2*>(a.out + (size_t)row * Cout + col) = o;
            }
        }
    }
}

template <int L>
__global__ void __launch_bounds__(LP_THREADS, 2) lpips_conv_kernel(const __grid_constant__ LpConvArgs a) {
    lp_conv_tile<LpAlex, L, false>(a);
}

// dX of convolution L (1..4) from dY; a.in = dY, a.out = dX, a.M = images * H * W, a.wprep = the dgrad tiles
template <int L>
__global__ void __launch_bounds__(LP_THREADS, 2) lpips_dgrad_kernel(const __grid_constant__ LpConvArgs a) {
    lp_conv_tile<LpAlex, L, true>(a);
}

// ---- max-pool 3/2, no padding, floor mode, channels-last [NI][H][W][C] -> [NI][Ho][Wo][C] ---------------------------
__global__ void __launch_bounds__(256) lpips_maxpool_kernel(int total4, int C4, int H, int W, int Ho, int Wo,
                                                            const float4* __restrict__ in, float4* __restrict__ out) {
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total4; e += gridDim.x * blockDim.x) {
        const int c = e % C4;
        int r = e / C4;
        const int ox = r % Wo;
        r /= Wo;
        const int oy = r % Ho, n = r / Ho;
        const float4* p = in + (((size_t)n * H + 2 * oy) * W + 2 * ox) * C4 + c;
        float4 m = __ldg(p);
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const float4 q = __ldg(p + ((size_t)dy * W + dx) * C4);
                m.x = fmaxf(m.x, q.x); m.y = fmaxf(m.y, q.y); m.z = fmaxf(m.z, q.z); m.w = fmaxf(m.w, q.w);
            }
        out[e] = m;
    }
}

// ---- taps --------------------------------------------------------------------------------------------------------
// pixel p < P = N * Hl * Wl of feature map f [2N][Hl][Wl][C]: x's features at row p, y's at row P + p.
// d(p) = sum_c w_c (fx_c / (|fx| + 1e-10) - fy_c / (|fy| + 1e-10))^2; partial[block] = sum of its pixels' d.
template <int C>
__global__ void __launch_bounds__(32 * LP_TAP_WARPS) lpips_tap_kernel(int P, const float* __restrict__ f,
                                                                       const float* __restrict__ lin,
                                                                       double* __restrict__ partial) {
    constexpr int PER = C / 32;
    __shared__ double s_w[LP_TAP_WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float w[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) w[i] = __ldg(lin + lane + 32 * i);
    double wsum = 0.0;
    for (int j = 0; j < LP_TAP_PIX; ++j) {
        const int p = (blockIdx.x * LP_TAP_WARPS + warp) * LP_TAP_PIX + j;
        if (p >= P) break;
        const float* fx = f + (size_t)p * C;
        const float* fy = f + ((size_t)P + p) * C;
        float xv[PER], yv[PER], sx = 0.f, sy = 0.f;
#pragma unroll
        for (int i = 0; i < PER; ++i) {
            xv[i] = __ldg(fx + lane + 32 * i);
            yv[i] = __ldg(fy + lane + 32 * i);
            sx = fmaf(xv[i], xv[i], sx);
            sy = fmaf(yv[i], yv[i], sy);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sx += __shfl_xor_sync(0xffffffffu, sx, o);
            sy += __shfl_xor_sync(0xffffffffu, sy, o);
        }
        const float nx = sqrtf(sx) + 1e-10f, ny = sqrtf(sy) + 1e-10f;
        float d = 0.f;
#pragma unroll
        for (int i = 0; i < PER; ++i) {
            const float t = __fdiv_rn(xv[i], nx) - __fdiv_rn(yv[i], ny);
            d = fmaf(w[i], t * t, d);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        wsum += (double)d;
    }
    if (lane == 0) s_w[warp] = wsum;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
#pragma unroll
        for (int i = 0; i < LP_TAP_WARPS; ++i) s += s_w[i];
        partial[blockIdx.x] = s;
    }
}

struct LpReduceArgs {
    const double* partial[LP_LAYERS];
    int blocks[LP_LAYERS];
    double pixels[LP_LAYERS];     // Hl * Wl: the layer's mean is over its own grid
    double* out;                  // [6]
};
// one block: out[l] = sum of layer l's partials / pixels[l] in a fixed order, out[5] = out[0] + ... + out[4]
__global__ void __launch_bounds__(256) lpips_reduce_kernel(const __grid_constant__ LpReduceArgs r) {
    __shared__ double red[256];
    double total = 0.0;
    for (int l = 0; l < LP_LAYERS; ++l) {
        double s = 0.0;
        for (int i = threadIdx.x; i < r.blocks[l]; i += 256) s += r.partial[l][i];
        red[threadIdx.x] = s;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            const double m = red[0] / r.pixels[l];
            r.out[l] = m;
            total += m;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) r.out[LP_LAYERS] = total;
}

// ==== backward ====================================================================================================
// The gradients of the images that need one: NB = N (x's or y's) or 2N (x's then y's) rows of every buffer, at image
// i0 = 0 or N of the forward's 2N.  From the top: tap 5 -> dgrad 5 -> tap 4 -> dgrad 4 -> tap 3 -> dgrad 3 -> pool 2
// -> tap 2 -> dgrad 2 -> pool 1 -> tap 1 -> layer-1 dgrad into the caller's CHW images.

// Tap l's gradient, added to the gradient g already there (unless `accumulate` is 0) and masked by the ReLU:
// g <- (f > 0) ? g + d tap / d f : 0, in place, channels-last rows.  One warp per pixel pair p < P = N * Hl * Wl, as
// the forward tap.  With a = f / D, D = |f| + 1e-10 and G = gout[l] + gout[5]:
//   u = G * 2 * lin * (a_x - a_y) / (Hl * Wl)   (-u on the y side),   d/df = u / D - f (u.f) / (|f| D^2)
// A zero feature vector gets 0 (its whole row is masked; torch's threshold_backward zeroes the reference's 0/0).
// x's row p is row p of g when wx; y's row p is row (wx ? P : 0) + p when wy.  f holds all 2N images.
template <int C>
__global__ void __launch_bounds__(32 * LP_TAP_WARPS) lpips_tap_bwd_kernel(int P, int layer, double pixels, int wx, int wy,
                                                                          int accumulate, const float* __restrict__ f,
                                                                          const float* __restrict__ lin,
                                                                          const double* __restrict__ gout,
                                                                          float* __restrict__ g) {
    constexpr int PER = C / 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float coef = (float)((__ldg(gout + layer) + __ldg(gout + LP_LAYERS)) * 2.0 / pixels);
    float w[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) w[i] = __ldg(lin + lane + 32 * i);
    for (int j = 0; j < LP_TAP_PIX; ++j) {
        const int p = (blockIdx.x * LP_TAP_WARPS + warp) * LP_TAP_PIX + j;
        if (p >= P) break;
        const float* fx = f + (size_t)p * C;
        const float* fy = f + ((size_t)P + p) * C;
        float xv[PER], yv[PER], u[PER], sx = 0.f, sy = 0.f;
#pragma unroll
        for (int i = 0; i < PER; ++i) {
            xv[i] = __ldg(fx + lane + 32 * i);
            yv[i] = __ldg(fy + lane + 32 * i);
            sx = fmaf(xv[i], xv[i], sx);
            sy = fmaf(yv[i], yv[i], sy);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sx += __shfl_xor_sync(0xffffffffu, sx, o);
            sy += __shfl_xor_sync(0xffffffffu, sy, o);
        }
        const float ax = sqrtf(sx), ay = sqrtf(sy), nx = ax + 1e-10f, ny = ay + 1e-10f;
#pragma unroll
        for (int i = 0; i < PER; ++i) u[i] = coef * w[i] * (__fdiv_rn(xv[i], nx) - __fdiv_rn(yv[i], ny));
#pragma unroll
        for (int side = 0; side < 2; ++side) {
            if (side == 0 ? !wx : !wy) continue;
            const float* fv = side == 0 ? xv : yv;
            const float norm = side == 0 ? ax : ay, D = side == 0 ? nx : ny, sgn = side == 0 ? 1.f : -1.f;
            float dot = 0.f;
#pragma unroll
            for (int i = 0; i < PER; ++i) dot = fmaf(u[i], fv[i], dot);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
            // (u.f) / |f| / D / D one division at a time: |f| D^2 underflows for tiny non-zero features
            const float k = norm > 0.f ? __fdiv_rn(__fdiv_rn(__fdiv_rn(dot, norm), D), D) : 0.f;
            float* gr = g + ((size_t)(side == 0 ? 0 : (wx ? P : 0)) + p) * C;
#pragma unroll
            for (int i = 0; i < PER; ++i) {
                const float d = sgn * (__fdiv_rn(u[i], D) - fv[i] * k);
                const float v = accumulate ? gr[lane + 32 * i] + d : d;
                gr[lane + 32 * i] = fv[i] > 0.f ? v : 0.f;
            }
        }
    }
}

// Max-pool 3/2 backward as a gather over the conv output grid [NB][H][W][C] (float4 units): each element sums dout
// over the (at most 2 x 2) windows containing it in which it is the argmax, recomputed from the saved conv output
// `in` with torch's rule (the first maximum in row-major order wins ties).  No atomics.
__global__ void __launch_bounds__(256) lpips_maxpool_bwd_kernel(int total4, int C4, int H, int W, int Ho, int Wo,
                                                                const float4* __restrict__ in,
                                                                const float4* __restrict__ dout,
                                                                float4* __restrict__ din) {
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total4; e += gridDim.x * blockDim.x) {
        const int c = e % C4;
        int r = e / C4;
        const int ix = r % W;
        r /= W;
        const int iy = r % H, n = r / H;
        const int oy0 = iy < 2 ? 0 : (iy - 1) / 2, oy1 = min(iy / 2, Ho - 1);
        const int ox0 = ix < 2 ? 0 : (ix - 1) / 2, ox1 = min(ix / 2, Wo - 1);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int oy = oy0; oy <= oy1; ++oy)
            for (int ox = ox0; ox <= ox1; ++ox) {
                const float4* p = in + (((size_t)n * H + 2 * oy) * W + 2 * ox) * C4 + c;
                float4 m = __ldg(p);
                int4 am = make_int4(0, 0, 0, 0);
#pragma unroll
                for (int t = 1; t < 9; ++t) {
                    const float4 q = __ldg(p + ((size_t)(t / 3) * W + t % 3) * C4);
                    if (q.x > m.x) { m.x = q.x; am.x = t; }
                    if (q.y > m.y) { m.y = q.y; am.y = t; }
                    if (q.z > m.z) { m.z = q.z; am.z = t; }
                    if (q.w > m.w) { m.w = q.w; am.w = t; }
                }
                const int self = (iy - 2 * oy) * 3 + (ix - 2 * ox);
                const float4 d = __ldg(dout + (((size_t)n * Ho + oy) * Wo + ox) * C4 + c);
                if (am.x == self) acc.x += d.x;
                if (am.y == self) acc.y += d.y;
                if (am.z == self) acc.z += d.z;
                if (am.w == self) acc.w += d.w;
            }
        din[e] = acc;
    }
}

// Layer-1 dgrad (11x11, stride 4, pad 2, Cin 3) on the CUDA cores in fp32: three output channels would fill a
// 64-wide tensor-core tile to 5%.  dz[c][iy][ix] = sum over the <= 3 x 3 (ky, kx) with ky = iy + 2 (mod 4), oy =
// (iy + 2 - ky) / 4, and likewise in x, of sum_co dY[oy][ox][co] w[co][c][ky][kx]; the image gradient is dz / scale,
// a true division like the forward's z-score.  Each block takes one phase (iy mod 4, ix mod 4) of one image, so its
// threads share the same taps, whose weights it stages in shared memory; a 32 x 8 block covers 128 x 32 pixels.
constexpr int LP_D0_TX = 32, LP_D0_TY = 8;
struct LpDgrad0Args {
    const float* dy;       // [NB][Ho][Wo][64], the gradient of conv 1's pre-ReLU output
    const float* w;        // [64][3][11][11]
    float* first;          // images 0..N-1 of dy: [N][3][H][W]
    float* second;         // images N..NB-1 (NB = 2N)
    int N, H, W, Ho, Wo, tiles_x, tiles_y;
};
__global__ void __launch_bounds__(LP_D0_TX * LP_D0_TY) lpips_dgrad0_kernel(const __grid_constant__ LpDgrad0Args a) {
    constexpr int KS = 11, S = 4, PAD = 2, CO = 64;
    __shared__ float4 s_w[3][3][CO];
    int b = blockIdx.x;
    const int tx = b % a.tiles_x; b /= a.tiles_x;
    const int ty = b % a.tiles_y; b /= a.tiles_y;
    const int phase = b % (S * S), n = b / (S * S);
    const int py = phase / S, px = phase % S;
    const int ry = (py + PAD) % S, rx = (px + PAD) % S;   // ky = ry + 4 i, kx = rx + 4 j
    for (int e = threadIdx.y * LP_D0_TX + threadIdx.x; e < 9 * CO; e += LP_D0_TX * LP_D0_TY) {
        const int co = e % CO, t = e / CO, ky = ry + S * (t / 3), kx = rx + S * (t % 3);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ky < KS && kx < KS) {
            const float* wp = a.w + ((size_t)co * 3 * KS + ky) * KS + kx;
            v = make_float4(__ldg(wp), __ldg(wp + KS * KS), __ldg(wp + 2 * KS * KS), 0.f);
        }
        s_w[t / 3][t % 3][co] = v;
    }
    __syncthreads();
    const int iy = S * (ty * LP_D0_TY + threadIdx.y) + py, ix = S * (tx * LP_D0_TX + threadIdx.x) + px;
    if (iy >= a.H || ix >= a.W) return;
    float ax = 0.f, ay = 0.f, az = 0.f;
    for (int i = 0; i < 3; ++i) {
        const int ky = ry + S * i, ny = iy + PAD - ky;
        if (ky >= KS || ny < 0) continue;
        const int oy = ny / S;
        if (oy >= a.Ho) continue;
        for (int j = 0; j < 3; ++j) {
            const int kx = rx + S * j, nx = ix + PAD - kx;
            if (kx >= KS || nx < 0) continue;
            const int ox = nx / S;
            if (ox >= a.Wo) continue;
            const float4* g = reinterpret_cast<const float4*>(a.dy + (((size_t)n * a.Ho + oy) * a.Wo + ox) * CO);
#pragma unroll 4
            for (int c4 = 0; c4 < CO / 4; ++c4) {
                const float4 d = __ldg(g + c4);
                const float4 w0 = s_w[i][j][4 * c4], w1 = s_w[i][j][4 * c4 + 1];
                const float4 w2 = s_w[i][j][4 * c4 + 2], w3 = s_w[i][j][4 * c4 + 3];
                ax = fmaf(d.x, w0.x, ax); ay = fmaf(d.x, w0.y, ay); az = fmaf(d.x, w0.z, az);
                ax = fmaf(d.y, w1.x, ax); ay = fmaf(d.y, w1.y, ay); az = fmaf(d.y, w1.z, az);
                ax = fmaf(d.z, w2.x, ax); ay = fmaf(d.z, w2.y, ay); az = fmaf(d.z, w2.z, az);
                ax = fmaf(d.w, w3.x, ax); ay = fmaf(d.w, w3.y, ay); az = fmaf(d.w, w3.z, az);
            }
        }
    }
    float* out = n < a.N ? a.first + (size_t)n * 3 * a.H * a.W : a.second + (size_t)(n - a.N) * 3 * a.H * a.W;
    const size_t hw = (size_t)a.H * a.W, o = (size_t)iy * a.W + ix;
    // the float32 scale of networks.py:44 (lpips_conv_kernel<0>'s gather)
    out[o] = __fdiv_rn(ax, .458f);
    out[hw + o] = __fdiv_rn(ay, .448f);
    out[2 * hw + o] = __fdiv_rn(az, .450f);
}

}  // namespace s3g
