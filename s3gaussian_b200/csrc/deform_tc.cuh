// deform_tc.cuh - the deformation decoder (forward) on the Hopper warpgroup tensor cores (wgmma).
//
// Same 3xTF32 arithmetic as the backward decoder of deform.cuh (hi*hi + hi*lo + lo*hi, fp32
// accumulate) but the dense layers are wgmma.mma_async instructions reading both operands from
// shared memory instead of warp-level mma.sync:
//
//   CTA = 128 threads = one warpgroup = one tile of 128 Gaussians; thread r owns Gaussian r.
//   * activations are split into tf32 hi/lo parts by their owner thread and stored to shared
//     memory in the canonical K-major core-matrix layout the wgmma descriptors address;
//   * each layer's pre-split weights arrive with ONE bulk async copy (TMA, cp.async.bulk ->
//     mbarrier complete_tx) that overlaps the previous layer's epilogue;
//   * the warpgroup issues the K/8 x 3 x 2 (two M = 64 halves) wgmmas of a layer, fp32 accumulators in registers;
//   * the accumulators (fragment layout, umma.cuh) go through a shared-memory staging tile that reuses the lo
//     operand buffer, so that the epilogue again runs on the thread's own row: bias, ReLU, split, store
//     - the per-Gaussian outputs (xyz+dx, exp/normalize/sigmoid, SH->RGB) are finished in the same registers;
//   * no operand tile is wider than 64 columns (the feature layer runs as two K-halves accumulated in registers),
//     so a CTA needs 96 KB of shared memory: two CTAs per SM hide each other's MMA and barrier latency;
//   * for training, every hidden layer's operand tile is also copied to global memory by one bulk async copy
//     (DeformTcArgs::acts) - the backward kernel reads those instead of recomputing the layers.
#pragma once
#include "deform.cuh"
#include "umma.cuh"

namespace s3g {

constexpr int TCM = 128;          // Gaussians per tile = two wgmma M = 64 halves

// prepared-weight table, indexed by the layer ids TL_* (deform.cuh)
// (TL_FEAT / TL_FEATB: the feature layer is run as two K-halves, columns [0,64) and [64,32L) of its weight, so that no
//  operand tile is wider than 64 columns: 96 KB of shared memory per CTA instead of 192 KB, two CTAs per SM)
struct TcTable {
    int off[TL_COUNT];     // float offset of the layer's [hi | lo] block in the prepared buffer, -1 = absent
    int npad[TL_COUNT];    // rows padded to a multiple of 16
    int k[TL_COUNT];
    int total;
};

// W [N][K] (PyTorch layout) -> canonical K-major tiles of its tf32 hi and lo parts, rows >= N zero.
// One launch for all layers: blockIdx.y = layer.
struct TcPrepArgs {
    const float* W[TL_COUNT];   // first element of the (sub-)matrix
    int n[TL_COUNT];
    int ld[TL_COUNT];           // row stride of the source matrix (= its full K)
    TcTable tab;
    float* dst;
};
__global__ void __launch_bounds__(256) tc_prep_weights_kernel(const __grid_constant__ TcPrepArgs p) {
    const int l = blockIdx.y;
    if (p.tab.off[l] < 0) return;
    const int K = p.tab.k[l], NP = p.tab.npad[l], N = p.n[l];
    float* dst = p.dst + p.tab.off[l];
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < NP * K; e += gridDim.x * blockDim.x) {
        const int n = e / K, k = e - n * K;
        const float v = n < N ? __ldg(p.W[l] + (size_t)n * p.ld[l] + k) : 0.f;
        uint32_t hi, lo;
        split_tf32_rna(v, hi, lo);
        const int ci = umma::canon_idx(n, k, K);
        dst[ci] = __uint_as_float(hi);
        dst[NP * K + ci] = __uint_as_float(lo);
    }
}

struct DeformTcArgs {
    DNet net;
    int P;
    const float *xyz, *scales, *rot, *opacity, *shs, *campos;
    int sh_degree;
    float *o_means, *o_scales, *o_rot, *o_opacity, *o_colors, *o_dx, *o_dshs, *o_feat;
    const float* features;     // [P][32L]
    const float* wprep;        // prepared weights (TcTable offsets)
    TcTable tab;
    // Hidden activations kept for the backward (or NULL): [slot][tile][128 x 64 operand tile], i.e. every stored tile
    // is the shared-memory image of the K-major operand it was for the next layer, written by ONE bulk async copy
    // (cp.async.bulk shared -> global) issued next to that layer's MMAs - no per-thread stores.  The hi operand
    // holds the fp32 value itself (the tensor core ignores the low mantissa bits), so the copy is exact.
    float* acts;
    int act_slot[8];           // slot of H, pos, scl, rot, opa, shs, d0, d2 (deform_host.cuh: act_slots), -1 = absent
    size_t act_stride;         // floats per slot = ceil(P / 128) * 128 * 64
};

struct TcCtx {
    float *op_hi, *op_lo, *w_sm;
    float* stage;    // [128][64] layer outputs, row r at r * 64, columns XOR-swizzled (tc_stage_idx); aliases op_lo
    uint64_t* w_bar;
    uint32_t wph;
    const float* wprep;
    const TcTable* tab;
    int loaded;      // layer whose weights are in (or on their way to) w_sm
};

__device__ __forceinline__ void tc_fetch_weights(TcCtx& c, int layer) {   // thread 0 only
    const uint32_t bytes = (uint32_t)(2 * c.tab->npad[layer] * c.tab->k[layer]) * 4u;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(umma::smem_u32(c.w_bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(umma::smem_u32(c.w_sm)), "l"(c.wprep + c.tab->off[layer]), "r"(bytes), "r"(umma::smem_u32(c.w_bar)) : "memory");
}

// staging index of (row, col): the XOR key is a bijection of row % 32, so the owner-row reads of a warp hit 32 banks
__device__ __forceinline__ int tc_stage_idx(int row, int col) {
    return row * 64 + (col ^ (((row & 7) << 2) | ((row >> 3) & 3)));
}

// All 128 threads.  The operand for `layer` has just been written to op_hi/op_lo by its owners.
// Runs the layer (N = its padded output width) into the accumulators `acc` (two M = 64 halves, fragment layout)
// and returns when they are complete and the operand buffers are free again; meanwhile the weights of
// `next_layer` (or -1) start streaming into the weight buffer.
// `keep` (or NULL): global destination of this layer's hi operand tile (128 x K floats), see DeformTcArgs::acts.
template <int N, int K>
__device__ __forceinline__ void tc_mma(TcCtx& c, int layer, int next_layer, float* keep, float (&acc)[2][N / 2], bool accumulate) {
    umma::fence_async_smem();
    __syncthreads();
    if (threadIdx.x == 0 && keep) {
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     ::"l"(keep), "r"(umma::smem_u32(c.op_hi)), "r"((uint32_t)(TCM * K) * 4u) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    umma::mbar_wait(c.w_bar, c.wph);
    constexpr uint32_t sbo = (uint32_t)(K / 4) * 128u, mhalf = 8u * sbo;
    const uint32_t a_hi = umma::smem_u32(c.op_hi), a_lo = umma::smem_u32(c.op_lo);
    const uint32_t b_hi = umma::smem_u32(c.w_sm), b_lo = b_hi + (uint32_t)(N * K) * 4u;
    umma::fence_regs(acc[0]); umma::fence_regs(acc[1]);
    umma::wgmma_fence();
#pragma unroll
    for (int k0 = 0; k0 < K; k0 += 8) {
        const uint32_t off = (uint32_t)(k0 / 4) * 128u;
        const uint64_t dbh = umma::make_smem_desc(b_hi + off, 128, sbo), dbl = umma::make_smem_desc(b_lo + off, 128, sbo);
#pragma unroll
        for (int m = 0; m < 2; ++m) {
            const uint64_t dah = umma::make_smem_desc(a_hi + m * mhalf + off, 128, sbo);
            const uint64_t dal = umma::make_smem_desc(a_lo + m * mhalf + off, 128, sbo);
            umma::wgmma_tf32<N>(acc[m], dal, dbh, accumulate || k0 > 0);
            umma::wgmma_tf32<N>(acc[m], dah, dbl, true);
            umma::wgmma_tf32<N>(acc[m], dah, dbh, true);
        }
    }
    umma::wgmma_commit();
    umma::wgmma_wait_all();
    umma::fence_regs(acc[0]); umma::fence_regs(acc[1]);
    // the operand buffer is rewritten after the barrier: the copy must have read it by then (it runs while the
    // MMAs do, so this wait is normally already satisfied)
    if (threadIdx.x == 0 && keep) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    __syncthreads();
    c.wph ^= 1;
    if (threadIdx.x == 0 && next_layer >= 0) tc_fetch_weights(c, next_layer);
}

// accumulators -> staging tile, readable by every owner thread when this returns
template <int N>
__device__ __forceinline__ void tc_stage(TcCtx& c, const float (&acc)[2][N / 2]) {
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) c.stage[tc_stage_idx(64 * m + umma::frag_row(i), umma::frag_col(i))] = acc[m][i];
    __syncthreads();
}

// one layer with K = 64 inputs: MMAs, then its outputs staged for the owner threads
template <int N>
__device__ __forceinline__ void tc_run_layer(TcCtx& c, int layer, int next_layer, float* keep = nullptr) {
    float acc[2][N / 2];
    tc_mma<N, 64>(c, layer, next_layer, keep, acc, false);
    tc_stage<N>(c, acc);
}

// the staging tile aliases op_lo: every owner has to be done reading it before operands are written again
__device__ __forceinline__ void tc_operand_begin() { __syncthreads(); }

// owner thread stores 4 consecutive activations (k..k+3, k % 4 == 0) of its row as hi and lo parts
__device__ __forceinline__ void tc_store4(TcCtx& c, int row, int k, int K, float v0, float v1, float v2, float v3) {
    uint32_t h[4], l[4];
    split_tf32(v0, h[0], l[0]); split_tf32(v1, h[1], l[1]); split_tf32(v2, h[2], l[2]); split_tf32(v3, h[3], l[3]);
    const int ci = umma::canon_idx(row, k, K);
    *reinterpret_cast<uint4*>(c.op_hi + ci) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(c.op_lo + ci) = make_uint4(l[0], l[1], l[2], l[3]);
}
template <bool RELU>
__device__ __forceinline__ void tc_store_row64(TcCtx& c, int row, const float (&v)[64]) {
    tc_operand_begin();
#pragma unroll
    for (int k = 0; k < 64; k += 4) {
        float a0 = v[k], a1 = v[k + 1], a2 = v[k + 2], a3 = v[k + 3];
        if (RELU) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); a2 = fmaxf(a2, 0.f); a3 = fmaxf(a3, 0.f); }
        tc_store4(c, row, k, 64, a0, a1, a2, a3);
    }
}
// this thread's row of a 64-wide layer output: staging -> registers, + bias
__device__ __forceinline__ void tc_load_row64(const TcCtx& c, const float* sBias, float (&v)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) v[i] = c.stage[tc_stage_idx(threadIdx.x, i)] + sBias[i];
}
// 32 consecutive output columns [col0, col0 + 32) of this thread's row
__device__ __forceinline__ void tc_load32(const TcCtx& c, int col0, float (&v)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = c.stage[tc_stage_idx(threadIdx.x, col0 + i)];
}

// two-layer head on relu(h) (or raw h): returns the first 32 output columns (+bias) of the last layer
template <bool RELU_IN>
__device__ __forceinline__ void tc_head2(TcCtx& c, int row, const float (&h)[64], int l1, int l2, const float* sB1, int next,
                                         float (&out)[32], float* keep_h, float* keep_a) {
    tc_store_row64<RELU_IN>(c, row, h);
    tc_run_layer<64>(c, l1, l2, keep_h);
    float a[64];
    tc_load_row64(c, sB1, a);
    tc_store_row64<true>(c, row, a);
    tc_run_layer<16>(c, l2, next, keep_a);
    tc_load32(c, 0, out);
}

__global__ void __launch_bounds__(TCM, 2) deform_forward_tc_kernel(const __grid_constant__ DeformTcArgs a) {
    extern __shared__ __align__(128) float s_dyn[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ float s_bias[14 * 64];       // every bias, 64 floats per layer slot
    const DNet& n = a.net;
    const int L = n.L, KF = FD * L;
    const int tid = threadIdx.x;
    TcCtx c;
    c.op_hi = s_dyn;                        // [128][64] canonical
    c.op_lo = s_dyn + TCM * 64;
    c.w_sm = s_dyn + 2 * TCM * 64;          // [hi | lo], up to 2 x 64 x 64
    c.stage = c.op_lo;
    c.w_bar = &s_bar;
    c.wph = 0;
    c.wprep = a.wprep; c.tab = &a.tab;

    // biases -> smem (zero where a layer is absent or padded)
    for (int i = tid; i < 14 * 64; i += TCM) s_bias[i] = 0.f;
    __syncthreads();
    {
        const float* bp[14] = {n.b_feat, n.pos.b1, n.pos.b2, n.scl.b1, n.scl.b2, n.rot.b1, n.rot.b2, n.opa.b1, n.opa.b2,
                               n.shs.b1, n.shs.b2, n.b_d0, n.b_d2, n.b_d4};
        const int bn[14] = {64, 64, 3, 64, 3, 64, 4, 64, 1, 64, 48, 64, 64, 3};
#pragma unroll
        for (int l = 0; l < 14; ++l)
            if (bp[l] && tid < bn[l]) s_bias[l * 64 + tid] = bp[l][tid];
    }
    if (tid == 0) umma::mbar_init(&s_bar, 1);
    __syncthreads();
    if (tid == 0) tc_fetch_weights(c, TL_FEAT);

    const int ntiles = (a.P + TCM - 1) / TCM;
    // order of the optional heads (what follows what) for weight prefetching
    const bool on_pos = n.pos.w1, on_scl = n.scl.w1, on_rot = n.rot.w1, on_opa = n.opa.w1, on_shs = n.shs.w1, on_d = n.w_d0;
    // heads run in the order pos, scl, rot, opa, dino, shs (shs last: h is dead by then)
    const int after_d = on_shs ? TL_SHS1 : TL_FEAT;
    const int after_opa = on_d ? TL_D0 : after_d;
    const int after_rot = on_opa ? TL_OPA1 : after_opa;
    const int after_scl = on_rot ? TL_ROT1 : after_rot;
    const int after_pos = on_scl ? TL_SCL1 : after_scl;
    const int first_after_feat = on_pos ? TL_POS1 : after_pos;
    const int after_shs = TL_FEAT;

    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int gi = tile * TCM + tid;
        const bool valid = gi < a.P;
        // ---- features -> operand, in two K-halves (columns [0,64) and [64,32L)); each half is 16 x 16 B loads in
        //      flight per thread, the second half's are issued before the first half's MMAs are waited for
        {
            const float4* fr = reinterpret_cast<const float4*>(a.features + (size_t)(valid ? gi : 0) * KF);
            const int KA = KF < 64 ? KF : 64, KB = KF - KA;
            float4 v[16];
#pragma unroll
            for (int j = 0; j < 16; ++j)
                v[j] = (valid && 4 * j < KA) ? __ldg(fr + j) : make_float4(0.f, 0.f, 0.f, 0.f);
            tc_operand_begin();
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (4 * j < KA) tc_store4(c, tid, 4 * j, KA, v[j].x, v[j].y, v[j].z, v[j].w);
            if (KB > 0) {
#pragma unroll
                for (int j = 0; j < 16; ++j)
                    v[j] = (valid && 4 * j < KB) ? __ldg(fr + 16 + j) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            float acc[2][32];
            const int nf = KB > 0 ? TL_FEATB : first_after_feat;
            if (KA == 64) tc_mma<64, 64>(c, TL_FEAT, nf, nullptr, acc, false);
            else tc_mma<64, 32>(c, TL_FEAT, nf, nullptr, acc, false);
            if (KB > 0) {     // tc_mma returned after a barrier: the operand buffers are free
#pragma unroll
                for (int j = 0; j < 16; ++j)
                    if (4 * j < KB) tc_store4(c, tid, 4 * j, KB, v[j].x, v[j].y, v[j].z, v[j].w);
                if (KB == 64) tc_mma<64, 64>(c, TL_FEATB, first_after_feat, nullptr, acc, true);
                else tc_mma<64, 32>(c, TL_FEATB, first_after_feat, nullptr, acc, true);
            }
            tc_stage<64>(c, acc);
        }
        float h[64];
        tc_load_row64(c, s_bias + TL_FEAT * 64, h);
        // where this tile's kept activations go; h is kept raw when the dino head (the one consumer of raw h) is on,
        // else as the relu(h) operand of the first enabled head (mask and products of the backward only need that)
        auto keep = [&](int kind) -> float* {
            return (a.acts && a.act_slot[kind] >= 0) ? a.acts + (size_t)a.act_slot[kind] * a.act_stride + (size_t)tile * (TCM * 64) : nullptr;
        };
        float* keep_h = on_d ? nullptr : keep(0);      // handed to the first relu head that runs, then cleared

        float dxv[3] = {0.f, 0.f, 0.f}, dsv[3] = {0.f, 0.f, 0.f}, drv[4] = {0.f, 0.f, 0.f, 0.f}, dov = 0.f, featv[3] = {0.f, 0.f, 0.f};
        float o32[32];
        if (on_pos) {
            tc_head2<true>(c, tid, h, TL_POS1, TL_POS2, s_bias + TL_POS1 * 64, after_pos, o32, keep_h, keep(1));
            keep_h = nullptr;
#pragma unroll
            for (int i = 0; i < 3; ++i) dxv[i] = o32[i] + s_bias[TL_POS2 * 64 + i];
        }
        if (on_scl) {
            tc_head2<true>(c, tid, h, TL_SCL1, TL_SCL2, s_bias + TL_SCL1 * 64, after_scl, o32, keep_h, keep(2));
            keep_h = nullptr;
#pragma unroll
            for (int i = 0; i < 3; ++i) dsv[i] = o32[i] + s_bias[TL_SCL2 * 64 + i];
        }
        if (on_rot) {
            tc_head2<true>(c, tid, h, TL_ROT1, TL_ROT2, s_bias + TL_ROT1 * 64, after_rot, o32, keep_h, keep(3));
            keep_h = nullptr;
#pragma unroll
            for (int i = 0; i < 4; ++i) drv[i] = o32[i] + s_bias[TL_ROT2 * 64 + i];
        }
        if (on_opa) {
            tc_head2<true>(c, tid, h, TL_OPA1, TL_OPA2, s_bias + TL_OPA1 * 64, after_opa, o32, keep_h, keep(4));
            keep_h = nullptr;
            dov = o32[0] + s_bias[TL_OPA2 * 64];
        }
        // ---- dino head (no leading ReLU) -----------------------------------------------------------
        if (on_d) {
            tc_store_row64<false>(c, tid, h);
            tc_run_layer<64>(c, TL_D0, TL_D2, keep(0));
            float av[64];
            tc_load_row64(c, s_bias + TL_D0 * 64, av);
            tc_store_row64<true>(c, tid, av);
            tc_run_layer<64>(c, TL_D2, TL_D4, keep(6));
            tc_load_row64(c, s_bias + TL_D2 * 64, av);
            tc_store_row64<true>(c, tid, av);
            tc_run_layer<16>(c, TL_D4, after_d, keep(7));
            tc_load32(c, 0, o32);
#pragma unroll
            for (int i = 0; i < 3; ++i) featv[i] = o32[i] + s_bias[TL_D4 * 64 + i];
        }
        // ---- SH head + colours ------------------------------------------------------------------
        float rgb[3] = {0.f, 0.f, 0.f};
        float bs[16];
        int nb = 0;
        float px = 0.f, py = 0.f, pz = 0.f;
        if (valid) {
            px = a.xyz[(size_t)gi * 3]; py = a.xyz[(size_t)gi * 3 + 1]; pz = a.xyz[(size_t)gi * 3 + 2];
            const float vx = px - a.campos[0], vy = py - a.campos[1], vz = pz - a.campos[2];
            const float inv = 1.0f / sqrtf(vx * vx + vy * vy + vz * vz);
            nb = sh_basis16(a.sh_degree, vx * inv, vy * inv, vz * inv, bs);
        }
        // this Gaussian's SH coefficients: issued here, consumed after the two SH layers
        float4 shs4[12];
        {
            const float4* sr = reinterpret_cast<const float4*>(a.shs + (size_t)(valid ? gi : 0) * 48);
#pragma unroll
            for (int j = 0; j < 12; ++j) shs4[j] = valid ? __ldg(sr + j) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (on_shs) {
            tc_store_row64<true>(c, tid, h);
            tc_run_layer<64>(c, TL_SHS1, TL_SHS2, keep_h);
            keep_h = nullptr;
            float av[64];
            tc_load_row64(c, s_bias + TL_SHS1 * 64, av);
            tc_store_row64<true>(c, tid, av);
            tc_run_layer<48>(c, TL_SHS2, after_shs, keep(5));
        }
        {   // dshs (the 48 staged columns) in two halves: out, shs + dshs, colour accumulation
            float* dshs_row = a.o_dshs ? a.o_dshs + (size_t)(valid ? gi : 0) * 48 : nullptr;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                float t[32];
                if (on_shs) {
                    if (half == 0) tc_load32(c, 0, t);
                    else {
#pragma unroll
                        for (int i = 0; i < 16; ++i) t[i] = c.stage[tc_stage_idx(tid, 32 + i)];
                    }
                }
                const int cnt = half == 0 ? 32 : 16;
#pragma unroll
                for (int j4 = 0; j4 < cnt; j4 += 4) {
                    const int j = 32 * half + j4;
                    float d[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) d[i] = on_shs ? t[j4 + i] + s_bias[TL_SHS2 * 64 + j + i] : 0.f;
                    if (valid) {
                        if (dshs_row) *reinterpret_cast<float4*>(dshs_row + j) = make_float4(d[0], d[1], d[2], d[3]);
                        const float4 s4 = shs4[j >> 2];
                        const float sf[4] = {s4.x + d[0], s4.y + d[1], s4.z + d[2], s4.w + d[3]};
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int idx = j + i, kk = idx / 3, ch = idx - 3 * kk;
                            if (kk < nb) rgb[ch] = fmaf(bs[kk], sf[i], rgb[ch]);
                        }
                    }
                }
            }
        }
        // ---- per-Gaussian outputs ------------------------------------------------------------------
        if (valid) {
            a.o_means[(size_t)gi * 3 + 0] = px + dxv[0];
            a.o_means[(size_t)gi * 3 + 1] = py + dxv[1];
            a.o_means[(size_t)gi * 3 + 2] = pz + dxv[2];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                if (a.o_dx) a.o_dx[(size_t)gi * 3 + i] = dxv[i];
                if (a.o_feat) a.o_feat[(size_t)gi * 3 + i] = featv[i];
                a.o_scales[(size_t)gi * 3 + i] = expf(a.scales[(size_t)gi * 3 + i] + dsv[i]);
                a.o_colors[(size_t)gi * 3 + i] = fmaxf(rgb[i] + 0.5f, 0.0f);
            }
            float q[4], nn = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) { q[i] = a.rot[(size_t)gi * 4 + i] + drv[i]; nn += q[i] * q[i]; }
            const float invn = 1.0f / fmaxf(sqrtf(nn), 1e-12f);
#pragma unroll
            for (int i = 0; i < 4; ++i) a.o_rot[(size_t)gi * 4 + i] = q[i] * invn;
            a.o_opacity[gi] = 1.0f / (1.0f + expf(-(a.opacity[gi] + dov)));
        }
    }
    // drain: the weights requested for a tile that never comes must land before the CTA exits
    if (tid == 0) umma::mbar_wait(c.w_bar, c.wph);
}

}  // namespace s3g
