// mcmc.cuh - 3DGS-MCMC's relocation and position noise (include/s3g_b200.h, "MCMC densification").
//
//   mcmc_relocate_kernel: blockIdx.y == 0 gives each pair j one thread that relocates row dst[j] (a copy of src[j]
//                         the caller made) and writes the result to dst[j] and src[j]; blockIdx.y == 1 + t zeroes
//                         descriptor t's rows at dst[j] (and at src[j] for the Adam moments).
//   mcmc_noise_kernel:    one thread per Gaussian, xyz += step * gate(o) * R diag(s^2) R^T eps.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace s3g {

constexpr int MCMC_BLOCK = 256;
constexpr int MCMC_N_MAX = 51;                           // 3DGS-MCMC's n_max: the ratio is clamped to it
constexpr double MCMC_O_MAX = 1.0 - 1.0 / 8388608.0;    // 1 - 2^-23, the largest opacity stored
constexpr int MCMC_MAX_ZERO = 32;

struct McmcZeroRows {
    float* rows;                      // [rows, row_floats], zeroed at dst[j]
    int row_floats;
    int at_src;                       // 1: at src[j] as well (the Adam moments)
};

struct McmcRelocArgs {
    McmcZeroRows t[MCMC_MAX_ZERO];
    int n;
    const long long* src;
    const long long* dst;
    const int* ratio;
    float min_opacity;
    float* opacity;                   // raw (logit) [rows,1]
    float* scaling;                   // raw (log) [rows,3]
};

// log(1 + e^x) without overflow
__device__ __forceinline__ double mcmc_softplus(double x) { return x > 0.0 ? x + log1p(exp(-x)) : log1p(exp(x)); }

// The relocation of one row with raw opacity x, in double (the alternating sum cancels badly in float32 at large N):
//   o = sigmoid(x), o' = 1 - (1 - o)^(1/N), D = sum_{i=1..N} sum_{k=0..i-1} C(i-1,k) (-1)^k o'^(k+1) / sqrt(k+1).
// Summing over i first (sum_{i=k+1..N} C(i-1,k) = C(N,k+1)) gives D = sum_{m=1..N} C(N,m) (-1)^(m-1) o'^m / sqrt(m),
// one loop of N terms with exact int64 binomials.  -log(1 - o) = softplus(x) keeps o near 1 accurate:
//   o' = -expm1(-softplus(x) / N), logit(o') = log(o') + softplus(x) / N.
// Writes the raw opacity (logit of o' clamped to [min_opacity, 1 - 2^-23]) and the log-scale offset log(o / D).
// N = 1 is the identity exactly: the raw values are kept unless the clamp applies.
__device__ __forceinline__ void mcmc_relocate_row(float x, int ratio, float min_opacity, float* x_out,
                                                  double* dlog_s) {
    const int N = min(max(ratio, 1), MCMC_N_MAX);
    const double lo = (double)min_opacity;
    const double sp = mcmc_softplus((double)x);
    const double o = exp(-mcmc_softplus(-(double)x));
    if (N == 1) {
        *dlog_s = 0.0;
        *x_out = o < lo ? (float)(log(lo) - log1p(-lo))
                        : o > MCMC_O_MAX ? (float)(log(MCMC_O_MAX) - log1p(-MCMC_O_MAX)) : x;
        return;
    }
    const double t = sp / N;
    const double op = -expm1(-t);
    double D = 0.0, p = 1.0;
    long long c = 1;                  // C(N, m)
    for (int m = 1; m <= N; ++m) {
        c = c * (N - m + 1) / m;
        p *= op;
        const double term = (double)c * p * rsqrt((double)m);
        D += (m & 1) ? term : -term;
    }
    *dlog_s = log(o / D);
    double logit;
    if (op < lo) logit = log(lo) - log1p(-lo);
    else if (op > MCMC_O_MAX) logit = log(MCMC_O_MAX) - log1p(-MCMC_O_MAX);
    else logit = log(op) + t;
    *x_out = (float)logit;
}

__global__ void __launch_bounds__(MCMC_BLOCK) mcmc_relocate_kernel(const __grid_constant__ McmcRelocArgs a) {
    if (blockIdx.y == 0) {
        const int j = blockIdx.x * MCMC_BLOCK + threadIdx.x;
        if (j >= a.n) return;
        const long long d = a.dst[j], s = a.src[j];
        float x;
        double dlog;
        mcmc_relocate_row(a.opacity[d], a.ratio[j], a.min_opacity, &x, &dlog);
        float ls[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) ls[k] = (float)((double)a.scaling[3 * d + k] + dlog);
        // dst rows (dead or appended) and src rows (alive) are disjoint, so no thread reads a row another writes; a row
        // drawn several times gets the same values from each of its writers
        a.opacity[d] = x;
        a.opacity[s] = x;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            a.scaling[3 * d + k] = ls[k];
            a.scaling[3 * s + k] = ls[k];
        }
        return;
    }
    const McmcZeroRows& t = a.t[blockIdx.y - 1];
    const long long total = (long long)a.n * t.row_floats;
    for (long long e = (long long)blockIdx.x * MCMC_BLOCK + threadIdx.x; e < total;
         e += (long long)gridDim.x * MCMC_BLOCK) {
        const long long j = e / t.row_floats;
        const int c = (int)(e - j * t.row_floats);
        t.rows[a.dst[j] * t.row_floats + c] = 0.f;
        if (t.at_src) t.rows[a.src[j] * t.row_floats + c] = 0.f;
    }
}

// 3DGS-MCMC's noise: gate = 1 / (1 + exp(-100 ((1 - o) - 0.995))), Sigma = R diag(s^2) R^T (R of the normalised
// quaternion, as build_rotation), xyz += step * gate * Sigma eps with step = xyz_lr * noise_lr.  The gate is formed in
// double: 100 (1 - o) amplifies a float32 rounding of 1 - o to ~2e-5 of the gate.  Sigma eps = R (s^2 * (R^T eps)).
__global__ void __launch_bounds__(MCMC_BLOCK)
mcmc_noise_kernel(int P, float* __restrict__ xyz, const float* __restrict__ scaling, const float* __restrict__ rotation,
                  const float* __restrict__ opacity, const float* __restrict__ eps, float step) {
    const int i = blockIdx.x * MCMC_BLOCK + threadIdx.x;
    if (i >= P) return;
    const double one_minus_o = 1.0 / (1.0 + exp((double)opacity[i]));
    const float gate = (float)(1.0 / (1.0 + exp(-100.0 * (one_minus_o - 0.995))));
    const float qw = rotation[4 * i + 0], qx = rotation[4 * i + 1], qy = rotation[4 * i + 2], qz = rotation[4 * i + 3];
    const float inv = 1.f / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
    const float w = qw * inv, x = qx * inv, y = qy * inv, z = qz * inv;
    const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - w * z), 2.f * (x * z + w * y)},
                           {2.f * (x * y + w * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - w * x)},
                           {2.f * (x * z - w * y), 2.f * (y * z + w * x), 1.f - 2.f * (x * x + y * y)}};
    const float e0 = eps[3 * i + 0], e1 = eps[3 * i + 1], e2 = eps[3 * i + 2];
    float u[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float s2 = expf(2.f * scaling[3 * i + k]);
        u[k] = s2 * (R[0][k] * e0 + R[1][k] * e1 + R[2][k] * e2);
    }
    const float g = step * gate;
#pragma unroll
    for (int r = 0; r < 3; ++r) xyz[3 * i + r] += g * (R[r][0] * u[0] + R[r][1] * u[1] + R[r][2] * u[2]);
}

}  // namespace s3g
