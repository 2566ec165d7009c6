// api_mcmc.cu - extern "C" entry points of the MCMC densification (see include/s3g_b200.h).
#include <algorithm>
#include <climits>
#include <cstdint>

#include "api_common.cuh"
#include "mcmc.cuh"

using namespace s3g;

namespace {
inline int fail(int code, const char* what) { return s3g::api_fail(code, what); }
}  // namespace

extern "C" {

int s3g_mcmc_relocate(int n, const int64_t* src, const int64_t* dst, const int32_t* ratio, float min_opacity,
                      float* opacity, float* scaling, int n_zero, const s3g_row_tensor* zero, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (n < 0) return fail(S3G_ERR_ARG, "mcmc_relocate: n < 0");
    if (n_zero < 0 || n_zero > MCMC_MAX_ZERO) return fail(S3G_ERR_ARG, "mcmc_relocate: 0..32 zero descriptors expected");
    if (n_zero > 0 && !zero) return fail(S3G_ERR_ARG, "mcmc_relocate: null descriptor array");
    if (n == 0) return S3G_OK;
    if (!src || !dst || !ratio || !opacity || !scaling) return fail(S3G_ERR_ARG, "mcmc_relocate: null pointer");
    if (!(min_opacity > 0.f && min_opacity < 1.f)) return fail(S3G_ERR_ARG, "mcmc_relocate: min_opacity outside (0, 1)");
    McmcRelocArgs a;
    a.n = n;
    a.src = reinterpret_cast<const long long*>(src);
    a.dst = reinterpret_cast<const long long*>(dst);
    a.ratio = ratio;
    a.min_opacity = min_opacity;
    a.opacity = opacity;
    a.scaling = scaling;
    long long most = n;
    for (int i = 0; i < n_zero; ++i) {
        const s3g_row_tensor& t = zero[i];
        if (!t.dst || t.row_floats <= 0) return fail(S3G_ERR_ARG, "mcmc_relocate: null dst or row_floats <= 0");
        a.t[i] = McmcZeroRows{t.dst, t.row_floats, t.zero_new};
        most = std::max(most, (long long)n * t.row_floats);
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long want = (most + MCMC_BLOCK - 1) / MCMC_BLOCK;
    const int gx = (int)std::max<long long>(std::min<long long>(want, (long long)sms * 8), (n + MCMC_BLOCK - 1) / MCMC_BLOCK);
    mcmc_relocate_kernel<<<dim3(gx, 1 + n_zero), MCMC_BLOCK, 0, stream>>>(a);
    S3G_CUDA(cudaGetLastError(), "mcmc_relocate launch");
    return S3G_OK;
}

int s3g_mcmc_noise(int P, float* xyz, const float* scaling, const float* rotation, const float* opacity,
                   const float* eps, float step, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "mcmc_noise: P < 0");
    if (P == 0) return S3G_OK;
    if (P > INT_MAX / 4) return fail(S3G_ERR_ARG, "mcmc_noise: P too large for 32-bit element indices");
    if (!xyz || !scaling || !rotation || !opacity || !eps) return fail(S3G_ERR_ARG, "mcmc_noise: null pointer");
    mcmc_noise_kernel<<<(P + MCMC_BLOCK - 1) / MCMC_BLOCK, MCMC_BLOCK, 0, stream>>>(P, xyz, scaling, rotation, opacity,
                                                                                   eps, step);
    S3G_CUDA(cudaGetLastError(), "mcmc_noise launch");
    return S3G_OK;
}

}  // extern "C"
