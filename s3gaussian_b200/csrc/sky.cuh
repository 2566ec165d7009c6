// sky.cuh - the sky model (EmerNeRF's sky head: a direction MLP behind the Gaussians) on the tensor cores.
//
// Per pixel: the world-space ray direction v, its sinusoidal encoding enc (E = 33), h1 = relu(W0 enc + b0),
// h2 = relu(W1 [h1, enc] + b1), sky = sigmoid(W2 h2 + b2); the width Wd is 64, 128, 192 or 256.  Every dense layer of
// width Wd runs as 3xTF32 mma.sync (hi*hi + hi*lo + lo*hi, fp32 accumulate), the same arithmetic as deform.cuh; the
// 3-wide output layer runs on the CUDA cores in fp32.  Both biases of the wide layers ride on a constant-1 column of
// the encoding (enc is padded to 40 columns: 33 features, a 1, six 0s), so every wide product is a plain GEMM.
//
// forward  sky_forward_kernel (one warp = 32 pixels as two m16 tiles, 4 warps per CTA)
//   * W1's hi/lo parts (Wd = 256: 606 KB) do not fit in shared memory, so the A operand comes from registers and the
//     B operand is read from L1/L2: sky_prep_forward_kernel splits the live W0 | b0 and W1 | b1 into tf32 hi/lo parts
//     on every call and stores them in the order of the B fragments (one 16-byte load per lane per 3 MMAs);
//   * the layer-1 output tile h1[:, 8s, 8s + 8) leaves its accumulators (C fragment) and is the A fragment of
//     layer 2's k-step s directly: the k order inside the step is permuted (physical column t holds logical column
//     2t, t + 4 holds 2t + 1) and the B fragments are prepared with the same permutation.  h1 never leaves the
//     registers;
//   * layer 2's outputs are produced in column chunks (all Wd columns up to Wd = 128, 64 columns above: 128 and 64
//     accumulators per lane), each followed by its share of the output layer, so h2 never leaves the registers
//     either.  Above Wd = 128 layer 1 is recomputed for every chunk (+31 % MACs at Wd = 256); chunks of 128 columns
//     need more than 255 registers and spill;
//   * nothing per pixel but the 3 x H x W output is written to global memory.
//
// backward  recompute, in chunks of SKY_CHUNK pixels, into the workspace (pixel-major, fp32):
//   X1 [p][Wd + 40] = [h1 | enc | 1 | 0]   (sky_encode_kernel, then layer 1 through sky_gemm_kernel)
//   H2 [p][Wd + 8]  = [h2 | 1 | 0]          (layer 2 through sky_gemm_kernel)
//   DZ [p][8], D2 [p][Wd]                  (sky_head_kernel: one warp per pixel, output layer, sigmoid, dL/dz and
//                                           dL/d(pre-activation of h2))
//   D1 [p][Wd] = (D2 W1[:, :Wd]) * (h1 > 0) (sky_gemm_kernel)
//   then the weight gradients, contracted over pixels with split-K: [dW1 | db1] = D2^T X1, [dW0 | db0] = D1^T X1[:, Wd:],
//   [dW2 | db2] = DZ^T H2, split over pixels so that every product fills the GPU (api_sky.cu: split_for); each split is
//   one CTA's fixed pixel range, written as a partial; sky_reduce_kernel adds the
//   partials in split order and the chunks in chunk order.  No atomics: two calls give bitwise equal gradients.
//   Memory: (4 Wd + 56) floats per pixel of a chunk (at most SKY_CHUNK pixels) plus the partials; none of it lives
//   past the call.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "deform.cuh"   // split_tf32, mma_tf32

namespace s3g {

constexpr int SKY_E = 33;              // encoding features
constexpr int SKY_EP = 40;             // encoding + the constant-1 bias column + zero padding
constexpr int SKY_ONE = 33;            // column of the 1 inside the padded encoding
constexpr int SKY_CHUNK = 65536;       // pixels per backward chunk
constexpr int SKY_FWD_WARPS = 4;

struct SkyNet {
    int wd;
    const float *w0, *b0, *w1, *b1, *w2, *b2;
};

struct SkyCam {
    int H, W;
    const float* c2w;         // DEVICE [4][4]
    const float* intrinsic;   // DEVICE [3][3]
};

// the padded encoding of pixel `pix` (row-major), e[0..39]: v, sin(v s), sin(v s + pi/2) for s = 1, 2, 4, 8, 16 laid
// out scale-major, then 1, then zeros.  float32 throughout, as torch computes it; accurate sinf.
__device__ __forceinline__ void sky_encode(const SkyCam& cam, int pix, float (&e)[SKY_EP]) {
    const float fx = __ldg(cam.intrinsic + 0), cx = __ldg(cam.intrinsic + 2);
    const float fy = __ldg(cam.intrinsic + 4), cy = __ldg(cam.intrinsic + 5);
    const int y = pix / cam.W, x = pix - y * cam.W;
    const float u0 = ((float)x - cx + 0.5f) / fx, u1 = ((float)y - cy + 0.5f) / fy;
    float d[3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
        d[i] = __fadd_rn(__fadd_rn(__fmul_rn(u0, __ldg(cam.c2w + 4 * i)), __fmul_rn(u1, __ldg(cam.c2w + 4 * i + 1))),
                         __ldg(cam.c2w + 4 * i + 2));
    const float n = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
    const float den = n + 1e-8f;
#pragma unroll
    for (int i = 0; i < 3; ++i) e[i] = d[i] / den;
#pragma unroll
    for (int s = 0; s < 5; ++s)
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float xb = e[i] * (float)(1 << s);
            e[3 + 3 * s + i] = sinf(xb);
            e[18 + 3 * s + i] = sinf(xb + 1.57079637f);
        }
    e[SKY_ONE] = 1.f;
#pragma unroll
    for (int k = SKY_ONE + 1; k < SKY_EP; ++k) e[k] = 0.f;
}

__device__ __forceinline__ float sky_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }

// ---- forward ----------------------------------------------------------------------------------------------------
// Prepared B fragments: block (n, q) of 32 lanes x float4 (b0 hi, b1 hi, b0 lo, b1 lo), lane = 4 g + t:
//   layer 1 (W0 | b0, K = 40):         n < Wd/8, q < 5;           b0 = W0p[8n + g][8q + t],  b1 = W0p[8n + g][8q + t + 4]
//   layer 2 (W1 | b1, K = Wd + 40):    n < Wd/8, q < Wd/8 + 5;    q < Wd/8 (the h1 part, permuted k):
//                                      b0 = W1p[8n + g][8q + 2t], b1 = W1p[8n + g][8q + 2t + 1]; else as layer 1
// W0p / W1p: the weights with the bias in the column of the encoding's 1 and zeros in the padding.
__device__ __forceinline__ float sky_w0p(const SkyNet& n, int row, int k) {
    return k < SKY_E ? __ldg(n.w0 + row * SKY_E + k) : k == SKY_ONE ? __ldg(n.b0 + row) : 0.f;
}
__device__ __forceinline__ float sky_w1p(const SkyNet& n, int row, int k) {
    const int K = n.wd + SKY_E;
    return k < K ? __ldg(n.w1 + (size_t)row * K + k) : k == n.wd + SKY_ONE ? __ldg(n.b1 + row) : 0.f;
}

__global__ void __launch_bounds__(256) sky_prep_forward_kernel(SkyNet net, float4* __restrict__ f0, float4* __restrict__ f1) {
    const int NT = net.wd / 8, Q1 = NT + SKY_EP / 8;
    const int n0 = NT * 5 * 32, n1 = NT * Q1 * 32;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n0 + n1; e += gridDim.x * blockDim.x) {
        const bool l1 = e < n0;
        const int i = l1 ? e : e - n0, lane = i & 31, blk = i >> 5, g = lane >> 2, t = lane & 3;
        const int Q = l1 ? 5 : Q1, n = blk / Q, q = blk - n * Q;
        float v0, v1;
        if (l1) {
            v0 = sky_w0p(net, 8 * n + g, 8 * q + t);
            v1 = sky_w0p(net, 8 * n + g, 8 * q + t + 4);
        } else if (q < NT) {
            v0 = sky_w1p(net, 8 * n + g, 8 * q + 2 * t);
            v1 = sky_w1p(net, 8 * n + g, 8 * q + 2 * t + 1);
        } else {
            v0 = sky_w1p(net, 8 * n + g, 8 * q + t);
            v1 = sky_w1p(net, 8 * n + g, 8 * q + t + 4);
        }
        uint32_t h0, lo0, h1, lo1;
        split_tf32(v0, h0, lo0);
        split_tf32(v1, h1, lo1);
        (l1 ? f0 : f1)[i] = make_float4(__uint_as_float(h0), __uint_as_float(h1), __uint_as_float(lo0), __uint_as_float(lo1));
    }
}

__device__ __forceinline__ void sky_mma3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], float4 b) {
    const uint32_t bh[2] = {__float_as_uint(b.x), __float_as_uint(b.y)};
    const uint32_t bl[2] = {__float_as_uint(b.z), __float_as_uint(b.w)};
    mma_tf32(d, al, bh);
    mma_tf32(d, ah, bl);
    mma_tf32(d, ah, bh);
}

// this lane's A fragment (standard k order) of k-step q of the encoding, m-tile mt, split into hi / lo
__device__ __forceinline__ void sky_enc_frag(const float* sE, int mt, int q, uint32_t (&ah)[4], uint32_t (&al)[4]) {
    const int g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
    const float* r0 = sE + (16 * mt + g) * (SKY_EP + 1);
    const float* r1 = r0 + 8 * (SKY_EP + 1);
    split_tf32(r0[8 * q + t], ah[0], al[0]);
    split_tf32(r1[8 * q + t], ah[1], al[1]);
    split_tf32(r0[8 * q + t + 4], ah[2], al[2]);
    split_tf32(r1[8 * q + t + 4], ah[3], al[3]);
}

template <int WD>
__global__ void __launch_bounds__(32 * SKY_FWD_WARPS) sky_forward_kernel(SkyNet net, SkyCam cam, const float4* __restrict__ f0,
                                                                      const float4* __restrict__ f1, float* __restrict__ out) {
    constexpr int NT = WD / 8, Q1 = NT + SKY_EP / 8;
    constexpr int NC = WD <= 128 ? WD : 64, CT = NC / 8;   // layer-2 column chunk and its n-tiles
    __shared__ float sEnc[SKY_FWD_WARPS][32 * (SKY_EP + 1)];
    __shared__ float sZ[SKY_FWD_WARPS][12 * 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int HW = cam.H * cam.W;
    const int p0 = (blockIdx.x * SKY_FWD_WARPS + warp) * 32;
    if (p0 >= HW) return;
    float* sE = sEnc[warp];
    {
        float e[SKY_EP];
        sky_encode(cam, min(p0 + lane, HW - 1), e);
#pragma unroll
        for (int k = 0; k < SKY_EP; ++k) sE[lane * (SKY_EP + 1) + k] = e[k];
    }
    __syncwarp();

    // [m-tile][row g / g + 8][channel]: this lane's partial sums of the output layer, kept in shared memory between the
    // column chunks so that they do not hold registers through the MMA loops
    float* zs = sZ[warp] + lane;
#pragma unroll
    for (int i = 0; i < 12; ++i) zs[32 * i] = 0.f;
    for (int c0 = 0; c0 < WD; c0 += NC) {
        float acc[2][CT][4] = {};
        for (int s = 0; s < NT; ++s) {
            // layer 1, output columns [8s, 8s + 8)
            float h[2][4] = {};
#pragma unroll
            for (int q = 0; q < 5; ++q) {
                const float4 b = __ldg(f0 + (s * 5 + q) * 32 + lane);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    uint32_t ah[4], al[4];
                    sky_enc_frag(sE, mt, q, ah, al);
                    sky_mma3(h[mt], ah, al, b);
                }
            }
            // relu; C fragment (g, 2t) (g, 2t+1) (g+8, 2t) (g+8, 2t+1) -> permuted A fragment of layer 2's k-step s
            uint32_t ah[2][4], al[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                split_tf32(fmaxf(h[mt][0], 0.f), ah[mt][0], al[mt][0]);
                split_tf32(fmaxf(h[mt][2], 0.f), ah[mt][1], al[mt][1]);
                split_tf32(fmaxf(h[mt][1], 0.f), ah[mt][2], al[mt][2]);
                split_tf32(fmaxf(h[mt][3], 0.f), ah[mt][3], al[mt][3]);
            }
#pragma unroll
            for (int j = 0; j < CT; ++j) {
                const float4 b = __ldg(f1 + ((c0 / 8 + j) * Q1 + s) * 32 + lane);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) sky_mma3(acc[mt][j], ah[mt], al[mt], b);
            }
        }
        // layer 2, the skip part [enc | 1 | 0] (k-steps NT .. NT + 4, standard k order; carries b1)
#pragma unroll
        for (int q = 0; q < 5; ++q) {
            uint32_t ah[2][4], al[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) sky_enc_frag(sE, mt, q, ah[mt], al[mt]);
#pragma unroll
            for (int j = 0; j < CT; ++j) {
                const float4 b = __ldg(f1 + ((c0 / 8 + j) * Q1 + NT + q) * 32 + lane);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) sky_mma3(acc[mt][j], ah[mt], al[mt], b);
            }
        }
        // relu, then this chunk's share of the output layer (fp32, fixed order)
        float z[2][2][3];
#pragma unroll
        for (int i = 0; i < 12; ++i) (&z[0][0][0])[i] = zs[32 * i];
#pragma unroll
        for (int j = 0; j < CT; ++j) {
            const int col = c0 + 8 * j + 2 * t;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float w0 = __ldg(net.w2 + c * WD + col), w1 = __ldg(net.w2 + c * WD + col + 1);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    z[mt][0][c] = fmaf(w0, fmaxf(acc[mt][j][0], 0.f), z[mt][0][c]);
                    z[mt][0][c] = fmaf(w1, fmaxf(acc[mt][j][1], 0.f), z[mt][0][c]);
                    z[mt][1][c] = fmaf(w0, fmaxf(acc[mt][j][2], 0.f), z[mt][1][c]);
                    z[mt][1][c] = fmaf(w1, fmaxf(acc[mt][j][3], 0.f), z[mt][1][c]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 12; ++i) zs[32 * i] = (&z[0][0][0])[i];
    }
    float z[2][2][3];
#pragma unroll
    for (int i = 0; i < 12; ++i) (&z[0][0][0])[i] = zs[32 * i];
    // the four lanes t of a row hold its partial sums: add them in a fixed tree, + b2, sigmoid
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float v = z[mt][r][c];
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                z[mt][r][c] = v;
            }
    if (t == 0) {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int p = p0 + 16 * mt + 8 * r + g;
                if (p < HW)
#pragma unroll
                    for (int c = 0; c < 3; ++c) out[(size_t)c * HW + p] = sky_sigmoid(z[mt][r][c] + __ldg(net.b2 + c));
            }
    }
}

// ---- backward ---------------------------------------------------------------------------------------------------
// Padded weights (fp32, rebuilt from the live parameters on every call):
//   W0p [Wd][40] = [W0 | b0 | 0],  W1p [Wd][Wd + 40] = [W1 | b1 | 0],  W2p [8][Wd + 8] = [W2 | b2 | 0; 0]
__global__ void sky_prep_backward_kernel(SkyNet net, float* __restrict__ w0p, float* __restrict__ w1p, float* __restrict__ w2p) {
    const int wd = net.wd, K1 = wd + SKY_EP, K2 = wd + 8;
    const int n0 = wd * SKY_EP, n1 = wd * K1, n2 = 8 * K2;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n0 + n1 + n2; e += gridDim.x * blockDim.x) {
        if (e < n0) {
            w0p[e] = sky_w0p(net, e / SKY_EP, e % SKY_EP);
        } else if (e < n0 + n1) {
            const int i = e - n0;
            w1p[i] = sky_w1p(net, i / K1, i % K1);
        } else {
            const int i = e - n0 - n1, c = i / K2, k = i % K2;
            w2p[i] = c >= 3 ? 0.f : k < wd ? __ldg(net.w2 + c * wd + k) : k == wd ? __ldg(net.b2 + c) : 0.f;
        }
    }
}

// X1[p][Wd ..] = the padded encoding, H2[p][Wd ..] = [1, 0 x 7] for the np pixels of the chunk starting at pix0
__global__ void sky_encode_kernel(SkyCam cam, int wd, int pix0, int np, float* __restrict__ x1, float* __restrict__ h2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= np) return;
    float e[SKY_EP];
    sky_encode(cam, pix0 + i, e);
    float4* dx = reinterpret_cast<float4*>(x1 + (size_t)i * (wd + SKY_EP) + wd);
#pragma unroll
    for (int k = 0; k < SKY_EP / 4; ++k) dx[k] = make_float4(e[4 * k], e[4 * k + 1], e[4 * k + 2], e[4 * k + 3]);
    float4* dh = reinterpret_cast<float4*>(h2 + (size_t)i * (wd + 8) + wd);
    dh[0] = make_float4(1.f, 0.f, 0.f, 0.f);
    dh[1] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// C[m][n] (op)= sum over k in this CTA's range of A(m, k) B(k, n), 3xTF32 mma.sync, 64 x 64 CTA tiles, k-steps of 16.
//   A(m, k) = A_KMAJ ? A[m lda + k] : A[k lda + m];   B(k, n) = B_KMAJ ? B[n ldb + k] : B[k ldb + n]
// SPLIT: blockIdx.z takes k range [z kper, (z + 1) kper) and writes its own partial C + z cstride.
enum { SKY_EPI_STORE = 0, SKY_EPI_RELU = 1, SKY_EPI_MASK = 2 };
struct SkyGemm {
    int M, N, K;
    const float* A; int lda;
    const float* B; int ldb;
    float* C; int ldc; size_t cstride;
    int kper;
    const float* mask; int ldm;   // SKY_EPI_MASK: C *= (mask[m ldm + n] > 0)
};
constexpr int SKY_GB = 64, SKY_GK = 16, SKY_GPAD = 8;

template <bool A_KMAJ, bool B_KMAJ, int EPI>
__global__ void __launch_bounds__(128, 2) sky_gemm_kernel(const SkyGemm a) {
    __shared__ float sA[SKY_GK][SKY_GB + SKY_GPAD], sB[SKY_GK][SKY_GB + SKY_GPAD];
    const int m0 = blockIdx.x * SKY_GB, n0 = blockIdx.y * SKY_GB;
    const int kb = blockIdx.z * a.kper, ke = min(a.K, kb + a.kper);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
    float acc[2][4][4] = {};
    for (int k0 = kb; k0 < ke; k0 += SKY_GK) {
        // 64 x 16 elements of each operand, 8 per thread
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const int e = threadIdx.x + 128 * r;
            int mm, kk;
            if (A_KMAJ) { mm = e >> 4; kk = e & 15; } else { kk = e >> 6; mm = e & 63; }
            const int gm = m0 + mm, gk = k0 + kk;
            sA[kk][mm] = (gm < a.M && gk < ke) ? (A_KMAJ ? a.A[(size_t)gm * a.lda + gk] : a.A[(size_t)gk * a.lda + gm]) : 0.f;
            int nn;
            if (B_KMAJ) { nn = e >> 4; kk = e & 15; } else { kk = e >> 6; nn = e & 63; }
            const int gn = n0 + nn, gk2 = k0 + kk;
            sB[kk][nn] = (gn < a.N && gk2 < ke) ? (B_KMAJ ? a.B[(size_t)gn * a.ldb + gk2] : a.B[(size_t)gk2 * a.ldb + gn]) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int ks = 0; ks < SKY_GK; ks += 8) {
            uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const int m = wm + 16 * mt + g;
                split_tf32(sA[ks + t][m], ah[mt][0], al[mt][0]);
                split_tf32(sA[ks + t][m + 8], ah[mt][1], al[mt][1]);
                split_tf32(sA[ks + t + 4][m], ah[mt][2], al[mt][2]);
                split_tf32(sA[ks + t + 4][m + 8], ah[mt][3], al[mt][3]);
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int n = wn + 8 * nt + g;
                split_tf32(sB[ks + t][n], bh[nt][0], bl[nt][0]);
                split_tf32(sB[ks + t + 4][n], bh[nt][1], bl[nt][1]);
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    mma_tf32(acc[mt][nt], al[mt], bh[nt]);
                    mma_tf32(acc[mt][nt], ah[mt], bl[nt]);
                    mma_tf32(acc[mt][nt], ah[mt], bh[nt]);
                }
        }
        __syncthreads();
    }
    float* C = a.C + blockIdx.z * a.cstride;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int m = m0 + wm + 16 * mt + g + 8 * (i >> 1), n = n0 + wn + 8 * nt + 2 * t + (i & 1);
                if (m >= a.M || n >= a.N) continue;
                float v = acc[mt][nt][i];
                if (EPI == SKY_EPI_RELU) v = fmaxf(v, 0.f);
                if (EPI == SKY_EPI_MASK) v = a.mask[(size_t)m * a.ldm + n] > 0.f ? v : 0.f;
                C[(size_t)m * a.ldc + n] = v;
            }
}

// one warp per pixel: z = W2p H2[p] (b2 through the 1 column), sky = sigmoid(z), dz = dL/dsky sky (1 - sky);
// DZ[p] = [dz, 0 x 5]; D2[p][j] = (sum_c W2[c][j] dz_c) (h2_j > 0)
__global__ void __launch_bounds__(256) sky_head_kernel(int wd, int HW, int pix0, int np, const float* __restrict__ w2p,
                                                       const float* __restrict__ h2, const float* __restrict__ gsky,
                                                       float* __restrict__ dz, float* __restrict__ d2) {
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= np) return;
    const int K2 = wd + 8;
    const float* h = h2 + (size_t)i * K2;
    float z[3] = {0.f, 0.f, 0.f};
    for (int k = lane; k < K2; k += 32) {
        const float v = h[k];
#pragma unroll
        for (int c = 0; c < 3; ++c) z[c] = fmaf(__ldg(w2p + c * K2 + k), v, z[c]);
    }
    float d[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float v = z[c];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        const float s = sky_sigmoid(v);
        d[c] = gsky[(size_t)c * HW + pix0 + i] * s * (1.f - s);
    }
    if (lane < 8) dz[(size_t)i * 8 + lane] = lane < 3 ? d[lane] : 0.f;
    for (int k = lane; k < wd; k += 32) {
        const float gh = __ldg(w2p + k) * d[0] + __ldg(w2p + K2 + k) * d[1] + __ldg(w2p + 2 * K2 + k) * d[2];
        d2[(size_t)i * wd + k] = h[k] > 0.f ? gh : 0.f;
    }
}

// acc[i] = (first ? 0 : acc[i]) + sum over s < S of part[s n + i], in split order
__global__ void sky_reduce_kernel(int n, int S, const float* __restrict__ part, float* __restrict__ acc, int first) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float v = first ? 0.f : acc[i];
    for (int s = 0; s < S; ++s) v += part[(size_t)s * n + i];
    acc[i] = v;
}

// the accumulated [dW | db] blocks -> the caller's gradient tensors
struct SkyGrads {
    float *w0, *b0, *w1, *b1, *w2, *b2;
};
__global__ void sky_scatter_kernel(int wd, const float* __restrict__ g0, const float* __restrict__ g1,
                                   const float* __restrict__ g2, SkyGrads o) {
    const int K1 = wd + SKY_EP, K2 = wd + 8;
    const int n0 = wd * SKY_EP, n1 = wd * K1, n2 = 3 * K2;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n0 + n1 + n2; e += gridDim.x * blockDim.x) {
        if (e < n0) {
            const int r = e / SKY_EP, k = e % SKY_EP;
            if (k < SKY_E) o.w0[r * SKY_E + k] = g0[e];
            else if (k == SKY_ONE) o.b0[r] = g0[e];
        } else if (e < n0 + n1) {
            const int i = e - n0, r = i / K1, k = i % K1;
            if (k < wd + SKY_E) o.w1[(size_t)r * (wd + SKY_E) + k] = g1[i];
            else if (k == wd + SKY_ONE) o.b1[r] = g1[i];
        } else {
            const int i = e - n0 - n1, c = i / K2, k = i % K2;
            if (k < wd) o.w2[c * wd + k] = g2[i];
            else if (k == wd) o.b2[c] = g2[i];
        }
    }
}

}  // namespace s3g
