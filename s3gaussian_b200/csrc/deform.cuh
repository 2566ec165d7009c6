// deform.cuh - HexPlane sample + multi-head deformation decoder + render() front-end,
// fused, forward and backward, for sm_90a.
//
// Replaces ~150 PyTorch launches per render (24 F.grid_sample, 14 Linear/ReLU, poc_fre,
// exp/normalize/sigmoid, eval_sh; scene/hexplane.py:73-106, scene/deformation.py:78-166,
// gaussian_renderer/__init__.py:99-117) with two kernels each way:
//
//   forward   hexplane_sample_kernel      four Gaussians per warp, lane = (Gaussian, channel quad): every bilinear
//                                         corner of the channels-last planes is one LDG.128; the six plane samples
//                                         of a level are multiplied in registers -> features [P][32L]
//             deform_forward_tc_kernel    (deform_tc.cuh) the dense layers on wgmma, 3xTF32 (hi*hi + hi*lo +
//                                         lo*hi, fp32 accumulate: 1e-4-relative parity with PyTorch fp32 rules out
//                                         plain TF32 / BF16, ~1e-3), xyz+dx, exp / normalize / sigmoid, SH->RGB with
//                                         the undeformed view direction fused into the epilogues
//   backward  deform_backward_kernel      mma.sync 3xTF32, tiles of 64 Gaussians: the hidden activations come from
//                                         what the wgmma forward kept;
//                                         push-back through the heads, Linear gradients into per-CTA partial buffers
//                                         (deform_reduce_kernel sums them), dL/d(features) [P][32L]
//             hexplane_scatter_kernel     plane gradients with 128-bit REDs (time planes: per-texel sums +
//                                         hexplane_time_rows_kernel), d(xyz) through the bilinear weights
#pragma once
#include "../../include/s3g_b200.h"
#include "common.cuh"

namespace s3g {

constexpr int DT = 64;            // Gaussians per tile
constexpr int DTHREADS = 512;        // 16 warps: the tile kernels run one CTA per SM (shared memory), so the
                                     // only latency hiding is warps within the CTA
constexpr int HWID = 64;          // hidden width (net_width)
constexpr int HS = HWID + 4;      // smem row stride of 64-wide tiles (== 4 mod 32: conflict-free fragments)
constexpr int FD = 32;            // features per plane

struct Head2 {                    // Sequential(ReLU, Linear(64,64), ReLU, Linear(64,k))
    const float *w1, *b1, *w2, *b2;
};
struct DNet {                     // device-side view of s3g_deform_net
    int L;
    int reso[S3G_MAX_LEVELS][4];
    const float* planes[S3G_MAX_LEVELS][6];
    float aabb0[3], inv_span2[3];     // p_hat = (p - aabb0) * inv_span2 - 1 ; inv_span2 = 2/(aabb1-aabb0)
    const float *w_feat, *b_feat;
    Head2 pos, scl, rot, opa, shs;
    const float *w_d0, *b_d0, *w_d2, *b_d2, *w_d4, *b_d4;
};
// ids of the Linear layers (deform_host.cuh: DeformLayer describes each), plus TL_FEATB: the second K-half of the
// feature layer in the wgmma forward's weight table (deform_tc.cuh: TcTable)
enum { TL_FEAT = 0, TL_POS1, TL_POS2, TL_SCL1, TL_SCL2, TL_ROT1, TL_ROT2, TL_OPA1, TL_OPA2, TL_SHS1, TL_SHS2,
       TL_D0, TL_D2, TL_D4, TL_FEATB, TL_COUNT };

// plane k samples coordinates (a,b): (0,1),(0,2),(0,3),(1,2),(1,3),(2,3) - compile-time so that
// unrolled loops index register arrays statically
__host__ __device__ constexpr int comb_a(int k) { return k < 3 ? 0 : (k < 5 ? 1 : 2); }
__host__ __device__ constexpr int comb_b(int k) { return k == 0 ? 1 : (k == 1 ? 2 : (k == 2 ? 3 : (k == 3 ? 2 : 3))); }

// ---- 3xTF32 tensor-core tile product ----------------------------------------
// x = hi + lo with hi, lo representable in tf32.  The tensor cores read sign, exponent and the top 10
// mantissa bits of a tf32 operand and ignore the rest (truncation), so hi is x itself and lo the exact
// remainder x - trunc(x), passed as is (its own truncation error is <= 2^-20 |x|).  Two instructions instead of
// two round-to-nearest conversions (cvt.rna.tf32.f32) per element, in the backward decoder's innermost loops.
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(x);
    lo = __float_as_uint(x - __uint_as_float(hi & 0xffffe000u));
}
// round-to-nearest variant for data that is split once and reused (weights of the wgmma path)
__device__ __forceinline__ void split_tf32_rna(float x, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
    const float r = x - __uint_as_float(hi);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
        "{%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// The three products of NT output tiles.  The two small cross terms accumulate in `ds`, the hi*hi term in `d` (summed by
// the caller at the end): 2 NT independent HMMA chains per warp instead of NT, and dependent HMMAs are 2 NT
// instructions apart, which hides the tensor pipe's result latency.
template <int NT>
__device__ __forceinline__ void mma3_multi(float (&d)[NT][4], float (&ds)[NT][4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                           const uint32_t (&bh)[NT][2], const uint32_t (&bl)[NT][2]) {
#pragma unroll
    for (int j = 0; j < NT; ++j) mma_tf32(ds[j], al, bh[j]);
#pragma unroll
    for (int j = 0; j < NT; ++j) mma_tf32(d[j], ah, bh[j]);
#pragma unroll
    for (int j = 0; j < NT; ++j) mma_tf32(ds[j], ah, bl[j]);
}
template <int NT>
__device__ __forceinline__ void mma3_fold(float (&d)[NT][4], const float (&ds)[NT][4]) {
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) d[j][i] += ds[j][i];
}

// ---- double-buffered weight staging -------------------------------------------------
// Every dense layer of a tile reads its weight matrix from shared memory.  Staging it at the
// top of the layer exposes one L2 round trip per layer (10-20 layers per tile, more than
// the MMA time); instead the NEXT layer's weights are fetched with cp.async into the
// other buffer while the current layer computes.  The per-tile sequence of weights is fixed, so
// the host passes it in (WSeq) and the pipe walks it cyclically.
struct WSeq {
    const float* W[28];
    short N[28], K[28];
    int count;
};
__device__ __forceinline__ void cp_async16_w(void* smem, const void* gmem) {
    uint32_t sa = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem) : "memory");
}
struct WPipe {
    // NB: no dynamically indexed member arrays - `buf[cur]` put the whole struct into local memory, with local loads
    // at the head of every product
    float *b0, *b1;
    int cur, wi, count;
    const WSeq* seq;     // shared-memory copy (a dynamically indexed kernel parameter is a long-scoreboard load)
    // descriptor of layer wi + 1, read one product ahead of its use so that acquire() never waits on it
    const float* nW;
    int nK, nN;
    bool nNew;           // layer wi + 1 uses other weights than layer wi
    __device__ __forceinline__ void prefetch(const float* Wg, int K, int N, float* dst) const {
        const int WS = K + 4, k4n = K >> 2;
        const bool pow2 = (k4n & (k4n - 1)) == 0;     // K = 64, 128, 256: a shift instead of an integer division
        const int sh = __ffs(k4n) - 1;
        for (int e = threadIdx.x; e < N * k4n; e += DTHREADS) {
            const int n = pow2 ? (e >> sh) : e / k4n, k4 = e - n * k4n;
            cp_async16_w(dst + n * WS + 4 * k4, Wg + (size_t)n * K + 4 * k4);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    __device__ __forceinline__ void load_next() {
        const int nxt = (wi + 1 == count) ? 0 : wi + 1;
        nW = seq->W[nxt]; nK = seq->K[nxt]; nN = seq->N[nxt];
        nNew = nW != seq->W[wi];
    }
    // kernel prologue: copies the sequence to shared memory, fetches layer 0 and ends with a barrier
    __device__ __forceinline__ void start(const WSeq& src, WSeq* s_seq, float* b0_, float* b1_) {
        for (int i = threadIdx.x; i < (int)(sizeof(WSeq) / 4); i += DTHREADS)
            reinterpret_cast<uint32_t*>(s_seq)[i] = reinterpret_cast<const uint32_t*>(&src)[i];
        __syncthreads();
        seq = s_seq; b0 = b0_; b1 = b1_;
        cur = 0; wi = 0; count = s_seq->count;
        prefetch(s_seq->W[0], s_seq->K[0], s_seq->N[0], b0);
        load_next();
        release();
        __syncthreads();
    }
    // Weights of layer `wi` are in the returned buffer (the previous product's release() + barrier made them
    // visible); the next layer's start flowing into the other buffer, which nobody reads any more since that
    // same barrier.  No barrier of its own: one per product instead of two.
    __device__ __forceinline__ float* acquire() {
        float* mine = cur ? b1 : b0;
        if (nNew) {
            prefetch(nW, nK, nN, cur ? b0 : b1);
            cur ^= 1;
        }
        wi = (wi + 1 == count) ? 0 : wi + 1;
        load_next();
        return mine;
    }
    // end of a product, immediately before its closing __syncthreads(): this thread's share of the next
    // layer's weights has landed
    __device__ __forceinline__ void release() const { asm volatile("cp.async.wait_all;" ::: "memory"); }
};

// out[g][n] = sum_k in[g][k] * W[n][k] + b[n],  g < 64, n < N (N = 64 or 48).
// 16 warps: (warp & 3) picks 16 rows, (warp >> 2) picks 16 of the columns (N = 48: the last group idles).
// sIn / sOut / sW are distinct smem regions; ends with a __syncthreads().
template <int K, int N>
__device__ __forceinline__ void tile_linear(const float* sIn, int inStride, WPipe& pipe,
                                            const float* __restrict__ bg, float* sOut, int outStride) {
    constexpr int WS = K + 4;
    constexpr int NTW = 2;               // n-tiles (of 8) per warp
    static_assert(N % 16 == 0 && N <= 64, "tile_linear: N in {16, 32, 48, 64}");
    const float* sW = pipe.acquire();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int r0 = (warp & 3) * 16;
    const int c0 = (warp >> 2) * 16;
    const bool active = c0 < N;
    float acc[NTW][4], accs[NTW][4];
#pragma unroll
    for (int j = 0; j < NTW; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[j][i] = accs[j][i] = 0.f;
    const float* rowA = sIn + (r0 + g) * inStride + t;
    const float* rowB = sIn + (r0 + g + 8) * inStride + t;
    float bias[NTW][2];                  // fetched before the k loop so the epilogue does not wait on L2
#pragma unroll
    for (int j = 0; j < NTW; ++j) {
        const int col = c0 + 8 * j + 2 * t;
        bias[j][0] = active ? __ldg(bg + col) : 0.f;
        bias[j][1] = active ? __ldg(bg + col + 1) : 0.f;
    }
#pragma unroll 4
    for (int k0 = 0; active && k0 < K; k0 += 8) {
        float a[4] = {rowA[k0], rowB[k0], rowA[k0 + 4], rowB[k0 + 4]};
        uint32_t ah[4], al[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) split_tf32(a[i], ah[i], al[i]);
        uint32_t bh[NTW][2], bl[NTW][2];
#pragma unroll
        for (int j = 0; j < NTW; ++j) {
            const float* wr = sW + (c0 + 8 * j + g) * WS + k0 + t;
            split_tf32(wr[0], bh[j][0], bl[j][0]);
            split_tf32(wr[4], bh[j][1], bl[j][1]);
        }
        mma3_multi<NTW>(acc, accs, ah, al, bh, bl);
    }
    mma3_fold<NTW>(acc, accs);
#pragma unroll
    for (int j = 0; j < NTW; ++j) {
        if (!active) break;
        const int col = c0 + 8 * j + 2 * t;
        const float b0 = bias[j][0], b1 = bias[j][1];
        float v0 = acc[j][0] + b0, v1 = acc[j][1] + b1, v2 = acc[j][2] + b0, v3 = acc[j][3] + b1;
        sOut[(r0 + g) * outStride + col] = v0;
        sOut[(r0 + g) * outStride + col + 1] = v1;
        sOut[(r0 + g + 8) * outStride + col] = v2;
        sOut[(r0 + g + 8) * outStride + col + 1] = v3;
    }
    pipe.release();
    __syncthreads();
}

// Tiny output layers (k <= 4): out[g][o] = sum_j in[g][j] * W[o][j] + b[o]; thread = (g, o).
__device__ __forceinline__ void tile_small_out(const float* sIn, int inStride, const float* __restrict__ Wg,
                                               const float* __restrict__ bg, int k, float* sOut,
                                               int outStride, int outCol) {
    const int g = threadIdx.x >> 2, o = threadIdx.x & 3;
    if (o < k && g < DT) {
        const float* in = sIn + g * inStride;
        const float* w = Wg + o * HWID;
        float s = 0.f;
#pragma unroll 16
        for (int j = 0; j < HWID; ++j) s = fmaf(in[j], __ldg(w + j), s);
        sOut[g * outStride + outCol + o] = s + __ldg(bg + o);
    }
}

// ---- HexPlane sampling -------------------------------------------------------
// torch grid_sample(bilinear, align_corners=True, padding_mode='border') separates per axis:
// ix = clamp((x+1)/2*(R-1), 0, R-1), i0 = floor(ix), f = ix - i0, neighbours i0 and i0+1 with
// weights (1-f) and f.  When i0+1 falls outside, f is exactly 0, so the neighbour index is
// clamped instead of predicated (its weight is 0).  One AxisTap per (level, axis) is shared by
// the three planes that use the axis - the per-plane work is 2 IMADs, 4 loads, 8 multiplies.
struct AxisTap {
    int i0, i1;          // texel indices (i1 clamped to R-1)
    float f, omf;        // fractional part and 1 - f
    float g;             // d(ix)/d(p_hat): (R-1)/2 inside, 0 where border-clamped
};
__device__ __forceinline__ AxisTap axis_tap(float x, int R) {
    AxisTap t;
    const float m = (float)(R - 1);
    float ix = ((x + 1.f) * 0.5f) * m;
    t.g = (ix <= 0.f || ix >= m) ? 0.f : 0.5f * m;     // clip_coordinates_set_grad
    ix = fminf(fmaxf(ix, 0.f), m);
    const float i0f = floorf(ix);
    t.i0 = (int)i0f;
    t.i1 = min(t.i0 + 1, R - 1);
    t.f = ix - i0f;
    t.omf = 1.f - t.f;
    return t;
}

// ---- lane layout of the two plane kernels ------------------------------------------------
// A warp works on FOUR Gaussians at a time: lane = (Gaussian sub = lane >> 3, channel quad q = lane & 7).  One
// bilinear corner of the channels-last planes is one LDG.128 / RED.128 per lane, 8 lanes = the corner's 128-byte line.
// Axis taps, texel offsets and bilinear weights are per Gaussian, so with one channel per lane (round 1) all 32 lanes
// of a warp computed the same ones; with four channels per lane that overhead is amortised over 4x the data and
// the load / RED instruction count drops 4x (both kernels are bound by instruction issue).
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void red4(float* p, float a, float b, float c, float d) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d)
                 : "memory");
}
// bilinear sample of four channels; the expression tree is the one-channel version's, per component
__device__ __forceinline__ void bilerp4(const AxisTap& X, const AxisTap& Y, const float4 (&v)[4], float (&s)[4]) {
    const float w00 = X.omf * Y.omf, w01 = X.f * Y.omf, w10 = X.omf * Y.f, w11 = X.f * Y.f;
    s[0] = w00 * v[0].x + w01 * v[1].x + w10 * v[2].x + w11 * v[3].x;
    s[1] = w00 * v[0].y + w01 * v[1].y + w10 * v[2].y + w11 * v[3].y;
    s[2] = w00 * v[0].z + w01 * v[1].z + w10 * v[2].z + w11 * v[3].z;
    s[3] = w00 * v[0].w + w01 * v[1].w + w10 * v[2].w + w11 * v[3].w;
}

// SH basis (utils/sh_utils.py:57-112) for unit direction (x,y,z); returns count
__device__ __forceinline__ int sh_basis16(int deg, float x, float y, float z, float* b) {
    b[0] = 0.28209479177387814f;
    if (deg < 1) return 1;
    const float C1 = 0.4886025119029199f;
    b[1] = -C1 * y; b[2] = C1 * z; b[3] = -C1 * x;
    if (deg < 2) return 4;
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    b[4] = 1.0925484305920792f * xy; b[5] = -1.0925484305920792f * yz;
    b[6] = 0.31539156525252005f * (2.f * zz - xx - yy);
    b[7] = -1.0925484305920792f * xz; b[8] = 0.5462742152960396f * (xx - yy);
    if (deg < 3) return 9;
    b[9] = -0.5900435899266435f * y * (3.f * xx - yy);
    b[10] = 2.890611442640554f * xy * z;
    b[11] = -0.4570457994644658f * y * (4.f * zz - xx - yy);
    b[12] = 0.3731763325901154f * z * (2.f * zz - 3.f * xx - 3.f * yy);
    b[13] = -0.4570457994644658f * x * (4.f * zz - xx - yy);
    b[14] = 1.445305721320277f * z * (xx - yy);
    b[15] = -0.5900435899266435f * x * (xx - 3.f * yy);
    return 16;
}

// ---- stage 1: HexPlane sampling, one warp per Gaussian, high occupancy ---------------
// The gather (12 KB of texels per Gaussian, L2-resident planes) is latency-bound unless many
// warps keep loads in flight, which the shared-memory-heavy decoder CTAs cannot; it is its own
// kernel and hands the [P][32L] features over through HBM (1 GB at 2M Gaussians).
struct SampleArgs {
    DNet net;
    int P;
    const float* xyz;
    float time;
    float* features;
};
template <int LT>
__global__ void __launch_bounds__(256, 3) hexplane_sample_kernel(SampleArgs a) {
    const DNet& n = a.net;
    const int lane = threadIdx.x & 31, sub = lane >> 3, q4 = (lane & 7) * 4;
    const int wpb = blockDim.x >> 5;
    const int L = LT > 0 ? LT : n.L;
    const int FL = FD * L;
    // Every block walks ONE contiguous run of Gaussians (its warps interleaved inside it): with the model kept in
    // a spatially coherent order (GaussianModel.spatial_sort, Morton curve) a block keeps revisiting the same few
    // texel lines while they are still in its SM's L1; in arbitrary order the assignment makes no difference.
    const int chunk = (a.P + gridDim.x - 1) / gridDim.x;
    const int g_begin = blockIdx.x * chunk, g_end = min(a.P, g_begin + chunk);
    for (int gb = g_begin + 4 * (threadIdx.x >> 5); gb < g_end; gb += 4 * wpb) {
        const int gi = gb + sub;
        const bool valid = gi < g_end;
        const int gc = valid ? gi : g_end - 1;        // tail lanes repeat the last Gaussian and store nothing
        float ph[4];
#pragma unroll
        for (int c = 0; c < 3; ++c) ph[c] = (__ldg(a.xyz + (size_t)gc * 3 + c) - n.aabb0[c]) * n.inv_span2[c] - 1.0f;
        ph[3] = a.time;
#pragma unroll
        for (int l = 0; l < (LT > 0 ? LT : S3G_MAX_LEVELS); ++l) {
            if (LT == 0 && l >= L) break;
            AxisTap ax[4];
#pragma unroll
            for (int d = 0; d < 4; ++d) ax[d] = axis_tap(ph[d], n.reso[l][d]);
            float f[4] = {1.f, 1.f, 1.f, 1.f};
#pragma unroll
            for (int h = 0; h < 2; ++h) {        // three planes = twelve 16-byte loads per lane in flight
                float4 v[3][4];
#pragma unroll
                for (int kk = 0; kk < 3; ++kk) {
                    const int k = 3 * h + kk, ca = comb_a(k), cb = comb_b(k);
                    const int W = n.reso[l][ca];
                    const float* pl = n.planes[l][k] + q4;
                    // unsigned 32-bit texel offsets (planes are < 2^32 floats): one IMAD.WIDE.U32 per address
                    const int r0 = ax[cb].i0 * W, r1 = ax[cb].i1 * W;
                    v[kk][0] = ldg4(pl + (uint32_t)(r0 + ax[ca].i0) * FD);
                    v[kk][1] = ldg4(pl + (uint32_t)(r0 + ax[ca].i1) * FD);
                    v[kk][2] = ldg4(pl + (uint32_t)(r1 + ax[ca].i0) * FD);
                    v[kk][3] = ldg4(pl + (uint32_t)(r1 + ax[ca].i1) * FD);
                }
#pragma unroll
                for (int kk = 0; kk < 3; ++kk) {
                    const int k = 3 * h + kk;
                    float sv[4];
                    bilerp4(ax[comb_a(k)], ax[comb_b(k)], v[kk], sv);
#pragma unroll
                    for (int c = 0; c < 4; ++c) f[c] = (k == 0) ? sv[c] : f[c] * sv[c];   // interp_space = 1 * s0 * s1 * ... (hexplane.py:87-96)
                }
            }
            if (valid) *reinterpret_cast<float4*>(a.features + (size_t)gi * FL + l * FD + q4) = make_float4(f[0], f[1], f[2], f[3]);
        }
    }
}

// store a [64][32L] tile of per-Gaussian rows from smem rows of stride FS to global memory
__device__ __forceinline__ void tile_rows_store(float* __restrict__ gdst, int g0, int P, int FL, const float* sSrc, int FS) {
    const int n4 = FL / 4;
    for (int i = threadIdx.x; i < DT * n4; i += DTHREADS) {
        const int g = i / n4, c4 = i - g * n4;
        if (g0 + g < P)
            *(reinterpret_cast<float4*>(gdst + (size_t)(g0 + g) * FL) + c4) = *reinterpret_cast<const float4*>(sSrc + g * FS + 4 * c4);
    }
}

// =============================================================================
// Backward
// =============================================================================

// out[g][k] (op)= ( sum_n in[g][n] * W[n][k] ) (* [mask[g][k] > 0]),  W is the PyTorch [N][K] weight,
// i.e. the transposed product used to push deltas back through a Linear.
enum { TL_ASSIGN = 0, TL_ASSIGN_MASK = 1, TL_ACCUM = 2, TL_ACCUM_MASK = 3 };
template <int K, int N, int MODE>
__device__ __forceinline__ void tile_linear_T(const float* sIn, int inStride, WPipe& pipe, float* sOut,
                                              int outStride, const float* sMask, int maskStride) {
    constexpr int WS = K + 4;
    constexpr int NTW = K / 32;          // output n-tiles (of 8) per warp: 4 column groups of K/4
    static_assert(K % 32 == 0, "tile_linear_T: K must be a multiple of 32");
    const float* sW = pipe.acquire();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int r0 = (warp & 3) * 16;
    const int c0 = (warp >> 2) * (K / 4);
    float acc[NTW][4], accs[NTW][4];
#pragma unroll
    for (int j = 0; j < NTW; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[j][i] = accs[j][i] = 0.f;
    // The contraction index of an MMA can be permuted freely as long as A and B agree: fragment slots (t, t+4)
    // take the physical indices (2t, 2t+1).  The weight reads W[n0+2t(+1)][c+g] then fall on banks 8t+g (+4)
    // (row stride == 4 mod 32): conflict-free, where the natural slots gave 4t+g, two-way conflicts.
    const float* rowA = sIn + (r0 + g) * inStride + 2 * t;
    const float* rowB = sIn + (r0 + g + 8) * inStride + 2 * t;
#pragma unroll 2
    for (int n0 = 0; n0 < N; n0 += 8) {
        const float2 ra = *reinterpret_cast<const float2*>(rowA + n0), rb = *reinterpret_cast<const float2*>(rowB + n0);
        const float a[4] = {ra.x, rb.x, ra.y, rb.y};
        uint32_t ah[4], al[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) split_tf32(a[i], ah[i], al[i]);
        uint32_t bh[NTW][2], bl[NTW][2];
#pragma unroll
        for (int j = 0; j < NTW; ++j) {
            const float* wr = sW + (n0 + 2 * t) * WS + c0 + 8 * j + g;
            split_tf32(wr[0], bh[j][0], bl[j][0]);
            split_tf32(wr[WS], bh[j][1], bl[j][1]);
        }
        mma3_multi<NTW>(acc, accs, ah, al, bh, bl);
    }
    mma3_fold<NTW>(acc, accs);
#pragma unroll
    for (int j = 0; j < NTW; ++j) {
        const int col = c0 + 8 * j + 2 * t;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + g + 8 * h;
            float v0 = acc[j][2 * h], v1 = acc[j][2 * h + 1];
            if (MODE == TL_ASSIGN_MASK || MODE == TL_ACCUM_MASK) {
                if (!(sMask[row * maskStride + col] > 0.f)) v0 = 0.f;
                if (!(sMask[row * maskStride + col + 1] > 0.f)) v1 = 0.f;
            }
            float* o = sOut + row * outStride + col;
            if (MODE == TL_ACCUM || MODE == TL_ACCUM_MASK) { o[0] += v0; o[1] += v1; }
            else { o[0] = v0; o[1] = v1; }
        }
    }
    pipe.release();
    __syncthreads();
}

// gW[m][n] += sum_g delta[g][m] * act(actv[g][n])   (Linear weight gradient of one tile)
// gb[m]    += sum_g delta[g][m]
template <int M, int NIN, bool RELU_ACT>
__device__ __forceinline__ void dw_accum(const float* sDelta, int dStride, const float* sAct, int aStride,
                                         float* __restrict__ gW, float* __restrict__ gb) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    constexpr int TN = NIN / 8;
    constexpr int NT = 2;                        // n-tiles per work item: the delta fragment is split once for both
    static_assert(TN % NT == 0, "dw_accum: NIN must be a multiple of 16");
    constexpr int ITEMS = (M / 16) * (TN / NT);
    for (int item = warp; item < ITEMS; item += DTHREADS / 32) {
        const int m0 = (item / (TN / NT)) * 16, n0 = (item % (TN / NT)) * (8 * NT);
        float acc[NT][4], accs[NT][4];
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[j][i] = accs[j][i] = 0.f;
#pragma unroll 2
        for (int k0 = 0; k0 < DT; k0 += 8) {
            // A[m][k] = delta[k][m]; contraction slots (t, t+4) -> rows (2t, 2t+1) of the tile: banks 8t+g for
            // every row stride == 4 (mod 32) or == 20 (mod 32) used here, conflict-free (see tile_linear_T)
            const float* dr = sDelta + (k0 + 2 * t) * dStride + m0 + g;
            const float a[4] = {dr[0], dr[8], dr[dStride], dr[dStride + 8]};
            uint32_t ah[4], al[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) split_tf32(a[i], ah[i], al[i]);
            uint32_t bh[NT][2], bl[NT][2];
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                const float* ar = sAct + (k0 + 2 * t) * aStride + n0 + 8 * j + g;
                float b[2] = {ar[0], ar[aStride]};
                if (RELU_ACT) { b[0] = fmaxf(b[0], 0.f); b[1] = fmaxf(b[1], 0.f); }
                split_tf32(b[0], bh[j][0], bl[j][0]);
                split_tf32(b[1], bh[j][1], bl[j][1]);
            }
            mma3_multi<NT>(acc, accs, ah, al, bh, bl);
        }
        mma3_fold<NT>(acc, accs);
        // fire-and-forget REDs on the CTA-private partial buffer: a load-add-store would expose
        // one L2 round trip per output tile
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            float* p0 = gW + (size_t)(m0 + g) * NIN + n0 + 8 * j + 2 * t;
            float* p1 = gW + (size_t)(m0 + g + 8) * NIN + n0 + 8 * j + 2 * t;
            atomicAdd(p0, acc[j][0]); atomicAdd(p0 + 1, acc[j][1]);
            atomicAdd(p1, acc[j][2]); atomicAdd(p1 + 1, acc[j][3]);
        }
    }
    if (threadIdx.x < M) {
        float sacc = 0.f;
        for (int k = 0; k < DT; ++k) sacc += sDelta[k * dStride + threadIdx.x];
        atomicAdd(gb + threadIdx.x, sacc);
    }
}

// small output layer (k <= 4 outputs): weight/bias gradients and delta push-back, SIMT.
//   gW2[o][j] += sum_g dout[g][o] * act[g][j];  gb2[o] += sum_g dout[g][o]
//   D[g][j] = (sum_o dout[g][o] * W2[o][j]) * [act[g][j] > 0]
__device__ __forceinline__ void small_head_backward(const float* sDout, int k, const float* sAct, int aStride,
                                                    const float* __restrict__ W2, float* __restrict__ gW2,
                                                    float* __restrict__ gb2, float* sD, int dStride,
                                                    bool wait_async = false) {
    const int tid = threadIdx.x;
    {   // weight grads: thread -> (o, j)
        const int o = tid >> 6, j = tid & 63;
        if (o < k) {
            float sacc = 0.f;
            for (int g = 0; g < DT; ++g) sacc = fmaf(sDout[g * 4 + o], sAct[g * aStride + j], sacc);
            atomicAdd(gW2 + o * HWID + j, sacc);
        }
        if (tid < k) {
            float sb = 0.f;
            for (int g = 0; g < DT; ++g) sb += sDout[g * 4 + tid];
            atomicAdd(gb2 + tid, sb);
        }
    }
    for (int e = tid; e < DT * HWID; e += DTHREADS) {
        const int g = e >> 6, j = e & 63;
        float v = 0.f;
        for (int o = 0; o < k; ++o) v = fmaf(sDout[g * 4 + o], __ldg(W2 + o * HWID + j), v);
        sD[g * dStride + j] = sAct[g * aStride + j] > 0.f ? v : 0.f;
    }
    if (wait_async) asm volatile("cp.async.wait_all;" ::: "memory");    // tiles requested before the call are visible after it
    __syncthreads();
}

struct GradOff {     // offsets (in floats) of every Linear gradient inside one CTA's partial buffer; -1 = disabled
    int w_feat, b_feat;
    int pos[4], scl[4], rot[4], opa[4], shs[4];     // w1, b1, w2, b2
    int d0w, d0b, d2w, d2b, d4w, d4b;
    int total;
};

struct DeformBwdArgs {
    DNet net;
    int P;
    const float *xyz, *scales, *rot, *opacity, *shs, *campos;
    float time;
    int sh_degree;
    const float *g_means, *g_scales, *g_rot, *g_opacity, *g_colors, *g_dx, *g_dshs, *g_feat;
    float *d_xyz, *d_scales, *d_rot, *d_opacity, *d_shs;
    float* gplanes[S3G_MAX_LEVELS][6];
    float* partial;      // [gridDim.x][off.total]
    const float* features;   // [P][32L] from the forward
    const float* acts;       // hidden activations kept by the wgmma forward (layout: DeformTcArgs::acts)
    int act_slot[8];         // slot of h, pos, scl, rot, opa, shs, d0, d2 (deform_host.cuh: act_slots), -1 = absent
    size_t act_stride;       // floats per slot = ceil(P / 128) * 128 * 64
    float* dfeatures;        // [P][32L] dL/d(features), consumed by hexplane_scatter_kernel
    GradOff off;
    WSeq wseq;
};

struct DeformBwdSmem {
    float *X, *F, *H, *DH, *A, *B, *D1, *D2, *Dout, *W, *G;
    __device__ DeformBwdSmem(float* base, int L) {
        const int FS = FD * L + 4;
        const int AB = (FS > 2 * HS ? FS : 2 * HS);
        X = base;                      // [64][4]
        F = X + DT * 4;                // [64][FS]
        H = F + DT * FS;               // [64][HS]
        DH = H + DT * HS;
        A = DH + DT * HS;              // A and B are contiguous: DF [64][FS] aliases them at the end
        B = A + DT * HS;
        D1 = A + DT * AB;
        D2 = D1 + DT * HS;
        Dout = D2 + DT * HS;           // [64][52]
        W = Dout + DT * 52;            // 2 x [64][max(FS,HS)] (double-buffered weight staging)
        G = W + 2 * HWID * (FS > HS ? FS : HS);   // [64][16] per-Gaussian scalars (small deltas)
    }
    __host__ __device__ static size_t floats(int L) {
        const int FS = FD * L + 4;
        const int AB = (FS > 2 * HS ? FS : 2 * HS);
        return (size_t)DT * 4 + DT * FS + 2 * DT * HS + DT * AB + 2 * DT * HS + DT * 52 + 2 * HWID * (FS > HS ? FS : HS) + DT * 16;
    }
};

__device__ __forceinline__ float ldz(const float* p, size_t i) { return p ? p[i] : 0.f; }

// [64][FL] rows of a per-Gaussian array -> smem rows of stride FS with cp.async (rows past P are zero-filled);
// completion: the caller's cp.async.wait_all (WPipe::release) + barrier
__device__ __forceinline__ void tile_rows_async(const float* __restrict__ gsrc, int g0, int P, int FL, float* sDst, int FS) {
    const int n4 = FL >> 2;
    for (int i = threadIdx.x; i < DT * n4; i += DTHREADS) {
        const int g = i / n4, c4 = i - g * n4;
        const bool ok = g0 + g < P;
        const float* src = gsrc + (size_t)(ok ? g0 + g : 0) * FL + 4 * c4;
        const uint32_t sa = (uint32_t)__cvta_generic_to_shared(sDst + g * FS + 4 * c4);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(sa), "l"(src), "r"(ok ? 16 : 0) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

// One 64-row half of a kept 128 x 64 operand tile (deform_tc.cuh) -> smem rows of stride FS.  The tile is stored in the
// tensor core's K-major core-matrix order: 16-byte piece i of the half holds columns 4*((i >> 3) & 15) .. +3 of row
// 8 * (i >> 7) + (i & 7).  The 16 KB are contiguous in global memory, so the copy is fully coalesced.
__device__ __forceinline__ void tile_canon_async(const float* __restrict__ half, float* sDst, int FS) {
    for (int i = threadIdx.x; i < DT * 16; i += DTHREADS) {
        const int r = ((i >> 7) << 3) + (i & 7), kq = (i >> 3) & 15;
        cp_async16_w(sDst + r * FS + 4 * kq, half + 4 * i);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

template <int KF>   // KF = 32*L
__device__ __forceinline__ void feat_layers_bwd(const DeformBwdSmem& sm, const DNet& n, float* part, const GradOff& off,
                                                int FS, WPipe& pipe) {
    // dW0 += DH^T F ; db0 ; DF = DH W0  (DF aliases A|B)
    dw_accum<64, KF, false>(sm.DH, HS, sm.F, FS, part + off.w_feat, part + off.b_feat);
    __syncthreads();
    tile_linear_T<KF, 64, TL_ASSIGN>(sm.DH, HS, pipe, sm.A, FS, nullptr, 0);
}

// One of the scales, rotation and opacity heads (k = 3, 4, 1 outputs) in deform_backward_kernel.  When the head is on,
// fetch() starts the next kept activation, and the head's outputs are recomputed into G[11..11+k) from its kept hidden
// layer Ab; act_bwd(on) writes the activation backward to Dout and to the d_* output; then, when the head is on, its
// two layers' gradients go into the partial buffer (GradOff row o) and the delta is pushed back into DH.
template <class Fetch, class ActBwd>
__device__ __forceinline__ void small_head_bwd(int k, const Head2& h, const int (&o)[4], float* Ab, Fetch fetch,
                                               ActBwd act_bwd, const DeformBwdSmem& sm, float* part, WPipe& pipe) {
    const bool on = h.w1 != nullptr;
    if (on) {
        fetch();
        tile_small_out(Ab, HS, h.w2, h.b2, k, sm.G, 16, 11);
        __syncthreads();
    }
    act_bwd(on);
    __syncthreads();
    if (on) {
        small_head_backward(sm.Dout, k, Ab, HS, h.w2, part + o[2], part + o[3], sm.D1, HS);
        dw_accum<64, 64, true>(sm.D1, HS, sm.H, HS, part + o[0], part + o[1]);
        tile_linear_T<64, 64, TL_ACCUM_MASK>(sm.D1, HS, pipe, sm.DH, HS, sm.H, HS);
    }
}

// The hidden activations (h and every head's hidden layer) are read from the buffer the wgmma forward filled, so a
// tile runs only the push-back products and the SH output layer; the stored tiles arrive by cp.async one head ahead
// of their use, alternating between the two activation buffers.
template <int LT>
__global__ void __launch_bounds__(DTHREADS, 1) deform_backward_kernel(const __grid_constant__ DeformBwdArgs a) {
    extern __shared__ __align__(16) float s_dyn[];
    const DNet& n = a.net;
    const int L = n.L;
    const int FS = FD * L + 4;
    DeformBwdSmem sm(s_dyn, L);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ntiles = (a.P + DT - 1) / DT;
    float* part = a.partial + (size_t)blockIdx.x * a.off.total;
    for (int i = tid; i < a.off.total; i += DTHREADS) part[i] = 0.f;
    __shared__ WSeq s_seq;
    WPipe pipe;
    pipe.start(a.wseq, &s_seq, sm.W, sm.W + HWID * (FS > HS ? FS : HS));
    __syncthreads();
    // which of the two activation buffers each stored tile lands in (consecutive enabled kinds alternate)
    const bool on_pos = n.pos.w1, on_scl = n.scl.w1, on_rot = n.rot.w1, on_opa = n.opa.w1, on_shs = n.shs.w1, on_d = n.w_d0;
    // The dino head needs its second hidden layer first, so that one travels a head ahead and takes the next
    // buffer in turn; the first hidden layer follows at the start of the head into the buffer the previous head used.
    float* abuf[8];
    {
        int j = 0;
        const bool en[6] = {false, on_pos, on_scl, on_rot, on_opa, on_shs};
#pragma unroll
        for (int k = 0; k < 6; ++k) { abuf[k] = (j & 1) ? sm.B : sm.A; if (en[k]) ++j; }
        abuf[7] = (j & 1) ? sm.B : sm.A;
        abuf[6] = (j & 1) ? sm.A : sm.B;
    }
#define S3G_FETCH_ACT(KIND) tile_canon_async(a.acts + (size_t)a.act_slot[KIND] * a.act_stride + (size_t)g0 * 64, abuf[KIND], HS)
    // start the load of the first enabled activation kind after `kind` (a compile-time constant at every call)
    auto fetch_after = [&](int kind, int g0) {
        if (kind < 1 && on_pos) S3G_FETCH_ACT(1);
        else if (kind < 2 && on_scl) S3G_FETCH_ACT(2);
        else if (kind < 3 && on_rot) S3G_FETCH_ACT(3);
        else if (kind < 4 && on_opa) S3G_FETCH_ACT(4);
        else if (kind < 5 && on_shs) S3G_FETCH_ACT(5);
        else if (kind < 6 && on_d) S3G_FETCH_ACT(7);
    };

    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int g0 = tile * DT;
        // ---- h, the features (for the last product pair) and the first head's hidden layer: stored by the forward.
        // The copies fly while the tile's scalars are set up; one barrier (after G below) covers all of it.
        tile_canon_async(a.acts + (size_t)a.act_slot[0] * a.act_stride + (size_t)g0 * 64, sm.H, HS);
        fetch_after(0, g0);
        tile_rows_async(a.features, g0, a.P, FD * L, sm.F, FS);     // last group: only the final product pair reads it
        if (tid < DT * 3) {
            const int g = tid / 3, c = tid - 3 * g;
            sm.X[g * 4 + c] = (g0 + g < a.P) ? a.xyz[(size_t)(g0 + g) * 3 + c] : 0.f;
        }
        for (int i = tid; i < DT * HS; i += DTHREADS) sm.DH[i] = 0.f;

        // ---- per-Gaussian activation backward -> small deltas in G[g][0..10] ----
        //  G: [0..2] d(dx) , [3..5] d(ds), [6..9] d(dr), [10] d(do)
        if (tid < DT) {
            const int g = tid, gi = g0 + g;
            float* G = sm.G + g * 16;
#pragma unroll
            for (int i = 0; i < 16; ++i) G[i] = 0.f;
            if (gi < a.P) {
#pragma unroll
                for (int c = 0; c < 3; ++c) G[c] = ldz(a.g_means, (size_t)gi * 3 + c) + ldz(a.g_dx, (size_t)gi * 3 + c);
            }
        }
        asm volatile("cp.async.wait_group 1;" ::: "memory");      // everything but the features
        __syncthreads();
        // scales / rotation / opacity need their head outputs first (when the heads are on), so
        // the forward of those heads is recomputed into S-like columns of G[11..15] lazily below.

        // ---- pos head ------------------------------------------------------------
        if (n.pos.w1) {
            float* Ab = abuf[1];
            fetch_after(1, g0);
            if (tid < DT * 4) sm.Dout[tid] = sm.G[(tid >> 2) * 16 + (tid & 3)] * ((tid & 3) < 3 ? 1.f : 0.f);
            __syncthreads();
            small_head_backward(sm.Dout, 3, Ab, HS, n.pos.w2, part + a.off.pos[2], part + a.off.pos[3], sm.D1, HS);
            dw_accum<64, 64, true>(sm.D1, HS, sm.H, HS, part + a.off.pos[0], part + a.off.pos[1]);
            tile_linear_T<64, 64, TL_ACCUM_MASK>(sm.D1, HS, pipe, sm.DH, HS, sm.H, HS);
        }
        small_head_bwd(3, n.scl, a.off.scl, abuf[2], [&] { fetch_after(2, g0); }, [&](bool on) {      // scales_act = exp(scales + ds)
            if (tid < DT * 4) {
                const int g = tid >> 2, c = tid & 3, gi = g0 + g;
                float d = 0.f;
                if (c < 3 && gi < a.P) {
                    const float sfin = a.scales[(size_t)gi * 3 + c] + (on ? sm.G[g * 16 + 11 + c] : 0.f);
                    d = ldz(a.g_scales, (size_t)gi * 3 + c) * expf(sfin);
                    a.d_scales[(size_t)gi * 3 + c] = d;
                }
                sm.Dout[tid] = d;
            }
        }, sm, part, pipe);
        small_head_bwd(4, n.rot, a.off.rot, abuf[3], [&] { fetch_after(3, g0); }, [&](bool on) {      // rot_act = normalize(rot + dr)
            if (tid < DT) {
                const int g = tid, gi = g0 + g;
                float dq[4] = {0.f, 0.f, 0.f, 0.f};
                if (gi < a.P) {
                    float q[4], gq[4], nn = 0.f, dot = 0.f;
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        q[i] = a.rot[(size_t)gi * 4 + i] + (on ? sm.G[g * 16 + 11 + i] : 0.f);
                        gq[i] = ldz(a.g_rot, (size_t)gi * 4 + i);
                        nn += q[i] * q[i];
                    }
                    const float nrm = sqrtf(nn);
                    if (nrm > 1e-12f) {          // F.normalize: x / max(|x|, eps)
                        const float inv = 1.f / nrm;
#pragma unroll
                        for (int i = 0; i < 4; ++i) dot += q[i] * inv * gq[i];
#pragma unroll
                        for (int i = 0; i < 4; ++i) dq[i] = (gq[i] - q[i] * inv * dot) * inv;
                    } else {
#pragma unroll
                        for (int i = 0; i < 4; ++i) dq[i] = gq[i] * 1e12f;
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i) a.d_rot[(size_t)gi * 4 + i] = dq[i];
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) sm.Dout[g * 4 + i] = dq[i];
            }
        }, sm, part, pipe);
        small_head_bwd(1, n.opa, a.off.opa, abuf[4], [&] { fetch_after(4, g0); }, [&](bool on) {      // opacity_act = sigmoid(opacity + do)
            if (tid < DT * 4) {
                const int g = tid >> 2, c = tid & 3, gi = g0 + g;
                float d = 0.f;
                if (c == 0 && gi < a.P) {
                    const float o = a.opacity[gi] + (on ? sm.G[g * 16 + 11] : 0.f);
                    const float sg = 1.0f / (1.0f + expf(-o));
                    d = ldz(a.g_opacity, gi) * sg * (1.f - sg);
                    a.d_opacity[gi] = d;
                }
                sm.Dout[tid] = d;
            }
        }, sm, part, pipe);
        // ---- shs head + SH->RGB backward ---------------------------------------------
        {
            const bool on = n.shs.w1 != nullptr;
            // the tile's [64][48] rows of shs and g_dshs are contiguous in global memory; they are fetched here, two
            // products ahead of their use (read at the point of use, their latency is exposed)
            constexpr int SPT = DT * 48 / DTHREADS;
            float pre_shs[SPT], pre_gd[SPT];
            {
                const size_t base = (size_t)g0 * 48, lim = (size_t)a.P * 48;
#pragma unroll
                for (int i = 0; i < SPT; ++i) {
                    const size_t idx = base + tid + i * DTHREADS;
                    pre_shs[i] = idx < lim ? __ldg(a.shs + idx) : 0.f;
                    pre_gd[i] = (a.g_dshs && idx < lim) ? __ldg(a.g_dshs + idx) : 0.f;
                }
            }
            float* Ab = abuf[5];
            if (on) {
                fetch_after(5, g0);
                tile_linear<64, 48>(Ab, HS, pipe, n.shs.b2, sm.Dout, 52);   // dshs
            } else {
                for (int i = tid; i < DT * 52; i += DTHREADS) sm.Dout[i] = 0.f;
                __syncthreads();
            }
            // shs_final = shs + dshs (in place)
#pragma unroll
            for (int i = 0; i < SPT; ++i) {
                const int e = tid + i * DTHREADS, g = e / 48, j = e - 48 * g;
                if (g0 + g < a.P) sm.Dout[g * 52 + j] += pre_shs[i];
            }
            __syncthreads();
            // per (Gaussian, colour channel) - four lanes per Gaussian, the fourth idles: colour clamp mask,
            // dL/dshs_final = basis (x) g_col, dL/d(dir) -> d_xyz part (into G[11..13]).  (One thread per Gaussian left
            // 14 of the 16 warps waiting at the next barrier for the longest scalar stretch of the tile.)
            if (tid < DT * 4) {
                const int g = tid >> 2, c = tid & 3, gi = g0 + g;
                const bool live = gi < a.P;
                float bs[16];
                float grc = 0.f;
                int nb = 0;
                float dd[3] = {0.f, 0.f, 0.f};      // this channel's share of dL/d(dir)
                float vx = 0.f, vy = 0.f, vz = 0.f, s2 = 1.f;
                float* sf = sm.Dout + g * 52;
                if (live) {
                    vx = sm.X[g * 4 + 0] - a.campos[0]; vy = sm.X[g * 4 + 1] - a.campos[1]; vz = sm.X[g * 4 + 2] - a.campos[2];
                    s2 = vx * vx + vy * vy + vz * vz;
                    const float inv = 1.0f / sqrtf(s2);
                    const float x = vx * inv, y = vy * inv, z = vz * inv;
                    nb = sh_basis16(a.sh_degree, x, y, z, bs);
                    if (c < 3) {
                        float r = 0.f;
                        for (int k = 0; k < nb; ++k) r = fmaf(bs[k], sf[3 * k + c], r);
                        grc = (r + 0.5f > 0.0f) ? ldz(a.g_colors, (size_t)gi * 3 + c) : 0.f;   // clamp_min(.,0)
                        if (a.sh_degree > 0) {
                            const float C1 = 0.4886025119029199f;
                            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
#define SHF(i) sf[3 * (i) + c]
                            float dx_ = -C1 * SHF(3), dy_ = -C1 * SHF(1), dz_ = C1 * SHF(2);
                            if (a.sh_degree > 1) {
                                dx_ += 1.0925484305920792f * y * SHF(4) + 0.31539156525252005f * -2.f * x * SHF(6) +
                                       -1.0925484305920792f * z * SHF(7) + 0.5462742152960396f * 2.f * x * SHF(8);
                                dy_ += 1.0925484305920792f * x * SHF(4) + -1.0925484305920792f * z * SHF(5) +
                                       0.31539156525252005f * -2.f * y * SHF(6) + 0.5462742152960396f * -2.f * y * SHF(8);
                                dz_ += -1.0925484305920792f * y * SHF(5) + 0.31539156525252005f * 4.f * z * SHF(6) +
                                       -1.0925484305920792f * x * SHF(7);
                            }
                            if (a.sh_degree > 2) {
                                dx_ += -0.5900435899266435f * SHF(9) * 6.f * xy + 2.890611442640554f * SHF(10) * yz +
                                       -0.4570457994644658f * SHF(11) * -2.f * xy + 0.3731763325901154f * SHF(12) * -6.f * xz +
                                       -0.4570457994644658f * SHF(13) * (-3.f * xx + 4.f * zz - yy) +
                                       1.445305721320277f * SHF(14) * 2.f * xz + -0.5900435899266435f * SHF(15) * 3.f * (xx - yy);
                                dy_ += -0.5900435899266435f * SHF(9) * 3.f * (xx - yy) + 2.890611442640554f * SHF(10) * xz +
                                       -0.4570457994644658f * SHF(11) * (-3.f * yy + 4.f * zz - xx) +
                                       0.3731763325901154f * SHF(12) * -6.f * yz + -0.4570457994644658f * SHF(13) * -2.f * xy +
                                       1.445305721320277f * SHF(14) * -2.f * yz + -0.5900435899266435f * SHF(15) * -6.f * xy;
                                dz_ += 2.890611442640554f * SHF(10) * xy + -0.4570457994644658f * SHF(11) * 8.f * yz +
                                       0.3731763325901154f * SHF(12) * 3.f * (2.f * zz - xx - yy) +
                                       -0.4570457994644658f * SHF(13) * 8.f * xz + 1.445305721320277f * SHF(14) * (xx - yy);
                            }
#undef SHF
                            dd[0] = dx_ * grc; dd[1] = dy_ * grc; dd[2] = dz_ * grc;
                        }
                    }
                }
                // (c0 + c1) + (c2 + 0): the order the one-thread version summed the channels in
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    dd[i] += __shfl_xor_sync(0xffffffffu, dd[i], 1);
                    dd[i] += __shfl_xor_sync(0xffffffffu, dd[i], 2);
                }
                if (c == 0) {
                    float dxyz[3] = {0.f, 0.f, 0.f};
                    if (live && a.sh_degree > 0) {       // through dir = v / |v|
                        const float inv32 = 1.0f / sqrtf(s2 * s2 * s2);
                        const float dot = vx * dd[0] + vy * dd[1] + vz * dd[2];
                        dxyz[0] = (s2 * dd[0] - vx * dot) * inv32;
                        dxyz[1] = (s2 * dd[1] - vy * dot) * inv32;
                        dxyz[2] = (s2 * dd[2] - vz * dot) * inv32;
                    }
                    sm.G[g * 16 + 11] = dxyz[0]; sm.G[g * 16 + 12] = dxyz[1]; sm.G[g * 16 + 13] = dxyz[2];
                }
                // overwrite this channel's third of the row with dL/dshs_final (every lane of the group has read its
                // coefficients above: the shuffles are a convergence point of the warp)
                if (c < 3) {
                    for (int k = 0; k < 16; ++k) sf[3 * k + c] = (k < nb ? bs[k] : 0.f) * grc;
                }
            }
            __syncthreads();
            // d_shs (param) = dL/dshs_final ; delta of the head output = that + g_dshs
#pragma unroll
            for (int i = 0; i < SPT; ++i) {
                const int e = tid + i * DTHREADS, g = e / 48, j = e - 48 * g;
                if (g0 + g < a.P) {
                    const float v = sm.Dout[g * 52 + j];
                    a.d_shs[(size_t)(g0 + g) * 48 + j] = v;
                    sm.Dout[g * 52 + j] = v + pre_gd[i];
                } else {
                    sm.Dout[g * 52 + j] = 0.f;
                }
            }
            __syncthreads();
            if (on) {
                dw_accum<48, 64, false>(sm.Dout, 52, Ab, HS, part + a.off.shs[2], part + a.off.shs[3]);
                tile_linear_T<64, 48, TL_ASSIGN_MASK>(sm.Dout, 52, pipe, sm.D1, HS, Ab, HS);
                dw_accum<64, 64, true>(sm.D1, HS, sm.H, HS, part + a.off.shs[0], part + a.off.shs[1]);
                tile_linear_T<64, 64, TL_ACCUM_MASK>(sm.D1, HS, pipe, sm.DH, HS, sm.H, HS);
            }
        }
        // ---- dino head ------------------------------------------------------------------
        if (n.w_d0) {
            float* Ad = abuf[6];
            float* Bd = abuf[7];
            S3G_FETCH_ACT(6);      // d2's layer arrived during the previous head; d0's (needed later) goes where that head's tile was
            if (tid < DT * 4) {
                const int g = tid >> 2, c = tid & 3, gi = g0 + g;
                sm.Dout[tid] = (c < 3 && gi < a.P) ? ldz(a.g_feat, (size_t)gi * 3 + c) : 0.f;
            }
            __syncthreads();
            small_head_backward(sm.Dout, 3, Bd, HS, n.w_d4, part + a.off.d4w, part + a.off.d4b, sm.D2, HS, true);
            dw_accum<64, 64, false>(sm.D2, HS, Ad, HS, part + a.off.d2w, part + a.off.d2b);
            tile_linear_T<64, 64, TL_ASSIGN_MASK>(sm.D2, HS, pipe, sm.D1, HS, Ad, HS);
            dw_accum<64, 64, false>(sm.D1, HS, sm.H, HS, part + a.off.d0w, part + a.off.d0b);
            tile_linear_T<64, 64, TL_ACCUM>(sm.D1, HS, pipe, sm.DH, HS, nullptr, 0);
        }
        __syncthreads();
        // ---- feature layer ---------------------------------------------------------------
        if (LT == 4 || L == 4) feat_layers_bwd<128>(sm, n, part, a.off, FS, pipe);
        else if (L == 1) feat_layers_bwd<32>(sm, n, part, a.off, FS, pipe);
        else if (L == 2) feat_layers_bwd<64>(sm, n, part, a.off, FS, pipe);
        else if (L == 3) feat_layers_bwd<96>(sm, n, part, a.off, FS, pipe);
        // DF now lives in sm.A with row stride FS: hand it to the scatter kernel, and write the
        // part of d_xyz that does not go through the planes (identity path + SH view direction)
        tile_rows_store(a.dfeatures, g0, a.P, FD * L, sm.A, FS);
        if (tid < DT * 3) {
            const int g = tid / 3, c = tid - 3 * g, gi = g0 + g;
            if (gi < a.P) a.d_xyz[(size_t)gi * 3 + c] = ldz(a.g_means, (size_t)gi * 3 + c) + sm.G[g * 16 + 11 + c];
        }
        __syncthreads();
    }
}

#undef S3G_FETCH_ACT

// ---- plane-gradient scatter + d(xyz) through the bilinear weights --------------------
// One warp per Gaussian, lane = channel: every tap is one 128-byte-wide RED.
struct ScatterArgs {
    DNet net;
    int P;
    const float* xyz;
    float time;
    const float* dfeatures;               // [P][32L]
    float* gplanes[S3G_MAX_LEVELS][6];
    float* d_xyz;                          // [P,3], += grid path
    // Every Gaussian of a call has the same time coordinate, so on the three planes with a time axis (k = 2, 4, 5)
    // all of them hit the same two texel rows with the same two row weights.  Their gradients are accumulated per
    // spatial texel in tacc[level][axis] ([reso][32], zeroed by the host) - two REDs instead of four - and
    // hexplane_time_rows_kernel spreads the sums over the two rows afterwards: 72 instead of 96 REDs per Gaussian.
    float* tacc[S3G_MAX_LEVELS][3];
};
// (two resident blocks per SM: the kernel is bound by L2 atomic / load throughput rather than by occupancy, and
// capping the registers for a third block measured slower on an earlier GPU)
template <int LT>
__global__ void __launch_bounds__(256, 2) hexplane_scatter_kernel(ScatterArgs a) {
    const DNet& n = a.net;
    const int L = LT > 0 ? LT : n.L;
    const int lane = threadIdx.x & 31, sub = lane >> 3, q = lane & 7, q4 = q * 4;   // see "lane layout" above
    const int wpb = blockDim.x >> 5;
    const int FL = FD * L;
    const int chunk = (a.P + gridDim.x - 1) / gridDim.x;      // contiguous run per block, see hexplane_sample_kernel
    const int g_begin = blockIdx.x * chunk, g_end = min(a.P, g_begin + chunk);
    for (int gb = g_begin + 4 * (threadIdx.x >> 5); gb < g_end; gb += 4 * wpb) {
        const int gi = gb + sub;
        const bool valid = gi < g_end;
        const int gc = valid ? gi : g_end - 1;
        float ph[4];
#pragma unroll
        for (int c = 0; c < 3; ++c) ph[c] = (__ldg(a.xyz + (size_t)gc * 3 + c) - n.aabb0[c]) * n.inv_span2[c] - 1.0f;
        ph[3] = a.time;
        float dph[3] = {0.f, 0.f, 0.f};    // this lane's share of dL/dp_hat
#pragma unroll
        for (int l = 0; l < (LT > 0 ? LT : S3G_MAX_LEVELS); ++l) {
            if (LT == 0 && l >= L) break;
            AxisTap ax[4];
#pragma unroll
            for (int d = 0; d < 4; ++d) ax[d] = axis_tap(ph[d], n.reso[l][d]);
            float df[4] = {0.f, 0.f, 0.f, 0.f};
            if (valid) {
                const float4 t = ldg4(a.dfeatures + (size_t)gi * FL + l * FD + q4);
                df[0] = t.x; df[1] = t.y; df[2] = t.z; df[3] = t.w;
            }
            // pass 1 (k ascending): texel offsets and the prefix products pre[k] = s_0 * ... * s_{k-1}
            uint32_t o00[6], o01[6], o10[6], o11[6];      // unsigned 32-bit texel offsets: one IMAD.WIDE.U32 per address
            float pre[6][4];
            {
                float run[4] = {1.f, 1.f, 1.f, 1.f};
#pragma unroll
                for (int k = 0; k < 6; ++k) {
                    const int ca = comb_a(k), cb = comb_b(k);
                    const int W = n.reso[l][ca];
                    const float* pl = n.planes[l][k] + q4;
                    const int r0 = ax[cb].i0 * W, r1 = ax[cb].i1 * W;
                    o00[k] = (uint32_t)(r0 + ax[ca].i0) * FD; o01[k] = (uint32_t)(r0 + ax[ca].i1) * FD;
                    o10[k] = (uint32_t)(r1 + ax[ca].i0) * FD; o11[k] = (uint32_t)(r1 + ax[ca].i1) * FD;
                    const float4 v[4] = {ldg4(pl + o00[k]), ldg4(pl + o01[k]), ldg4(pl + o10[k]), ldg4(pl + o11[k])};
                    float sv[4];
                    bilerp4(ax[ca], ax[cb], v, sv);
#pragma unroll
                    for (int c = 0; c < 4; ++c) { pre[k][c] = run[c]; run[c] *= sv[c]; }
                }
            }
            // pass 2 (k descending, running suffix product): ds_k = df * prod_{j != k} s_j.  The corner values are
            // read again (L1 hits) instead of being kept: 96 registers per level would not fit.
            float suf[4] = {1.f, 1.f, 1.f, 1.f};
#pragma unroll
            for (int k = 5; k >= 0; --k) {
                const int ca = comb_a(k), cb = comb_b(k);
                const AxisTap& X = ax[ca];
                const AxisTap& Y = ax[cb];
                const float* pl = n.planes[l][k] + q4;
                const float4 v[4] = {ldg4(pl + o00[k]), ldg4(pl + o01[k]), ldg4(pl + o10[k]), ldg4(pl + o11[k])};
                float sv[4], ds[4];
                bilerp4(X, Y, v, sv);
#pragma unroll
                for (int c = 0; c < 4; ++c) { ds[c] = df[c] * pre[k][c] * suf[c]; suf[c] *= sv[c]; }
                // a border-clamped neighbour carries weight exactly 0 and aliases a valid texel: adding
                // 0.0 leaves it unchanged, so the four REDs are unconditional (no branches in the loop)
                if (valid) {
                    float* gp = a.gplanes[l][k] + q4;
                    float wx0[4], wx1[4];
#pragma unroll
                    for (int c = 0; c < 4; ++c) { wx0[c] = X.omf * ds[c]; wx1[c] = X.f * ds[c]; }
                    if (cb == 3) {      // time plane: per-texel sums, the row weights are applied once afterwards
                        float* tp = a.tacc[l][ca] + q4;
                        red4(tp + (uint32_t)X.i0 * FD, wx0[0], wx0[1], wx0[2], wx0[3]);
                        red4(tp + (uint32_t)X.i1 * FD, wx1[0], wx1[1], wx1[2], wx1[3]);
                    } else {
                    red4(gp + o00[k], wx0[0] * Y.omf, wx0[1] * Y.omf, wx0[2] * Y.omf, wx0[3] * Y.omf);
                    red4(gp + o01[k], wx1[0] * Y.omf, wx1[1] * Y.omf, wx1[2] * Y.omf, wx1[3] * Y.omf);
                    red4(gp + o10[k], wx0[0] * Y.f, wx0[1] * Y.f, wx0[2] * Y.f, wx0[3] * Y.f);
                    red4(gp + o11[k], wx1[0] * Y.f, wx1[1] * Y.f, wx1[2] * Y.f, wx1[3] * Y.f);
                    }
                }
                // d(sample)/d(ix), d(sample)/d(iy)
                const float vv[4][4] = {{v[0].x, v[0].y, v[0].z, v[0].w}, {v[1].x, v[1].y, v[1].z, v[1].w},
                                        {v[2].x, v[2].y, v[2].z, v[2].w}, {v[3].x, v[3].y, v[3].z, v[3].w}};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float dsx = (vv[1][c] - vv[0][c]) * Y.omf + (vv[3][c] - vv[2][c]) * Y.f;
                    const float dsy = (vv[2][c] - vv[0][c]) * X.omf + (vv[3][c] - vv[1][c]) * X.f;
                    if (ca < 3) dph[ca] += ds[c] * dsx * X.g;
                    if (cb < 3) dph[cb] += ds[c] * dsy * Y.g;
                }
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) dph[c] += __shfl_xor_sync(0xffffffffu, dph[c], o);   // the Gaussian's 8 lanes
        }
        if (valid && q < 3) {
            const float d = q == 0 ? dph[0] : (q == 1 ? dph[1] : dph[2]);
            a.d_xyz[(size_t)gi * 3 + q] += d * n.inv_span2[q];
        }
    }
}

// gplane[l][k][t0][ix] += (1 - f_t) * tacc[l][axis][ix],  gplane[l][k][t1][ix] += f_t * tacc[l][axis][ix]  for the three
// planes with a time axis; runs after the scatter kernel on the same stream (no other writer of these planes then).
struct TimeRowsArgs {
    DNet net;
    float time;
    float* gplanes[S3G_MAX_LEVELS][6];
    const float* tacc[S3G_MAX_LEVELS][3];
};
static __global__ void __launch_bounds__(256) hexplane_time_rows_kernel(TimeRowsArgs a) {
    const int l = blockIdx.z, axis = blockIdx.y;
    const int k = axis == 0 ? 2 : (axis == 1 ? 4 : 5);
    const int W = a.net.reso[l][axis];
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= W * FD) return;
    const AxisTap T = axis_tap(a.time, a.net.reso[l][3]);
    const float v = a.tacc[l][axis][e];
    float* gp = a.gplanes[l][k];
    // a border-clamped second row has weight exactly 0 and aliases the first: adding 0.0 leaves it unchanged
    gp[(size_t)T.i0 * W * FD + e] += T.omf * v;
    gp[(size_t)T.i1 * W * FD + e] += T.f * v;
}

// sum the per-CTA partial Linear gradients: one thread per gradient element
struct ReduceSeg { float* dst; int off; int count; };
struct ReduceArgs { ReduceSeg seg[32]; int nseg; const float* partial; int stride; int nparts; };
static __global__ void __launch_bounds__(256) deform_reduce_kernel(ReduceArgs r) {
    const ReduceSeg sg = r.seg[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sg.count) return;
    const float* p = r.partial + sg.off + i;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    int q = 0;
    for (; q + 4 <= r.nparts; q += 4) {      // four independent loads in flight
        s0 += p[(size_t)q * r.stride];
        s1 += p[(size_t)(q + 1) * r.stride];
        s2 += p[(size_t)(q + 2) * r.stride];
        s3 += p[(size_t)(q + 3) * r.stride];
    }
    for (; q < r.nparts; ++q) s0 += p[(size_t)q * r.stride];
    sg.dst[i] = (s0 + s1) + (s2 + s3);
}

}  // namespace s3g
