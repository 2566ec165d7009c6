// api_eval.cu - extern "C" entry points of the evaluation metrics (include/s3g_b200.h, csrc/eval_metrics.cuh).
#include <cstdint>

#include "api_common.cuh"
#include "eval_metrics.cuh"

using namespace s3g;

namespace {
inline int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return s3g::api_fail(code, what, e); }

dim3 eval_grid(int C, int H, int W) { return dim3((W + EV_T - 1) / EV_T, (H + EV_T - 1) / EV_T, C); }
}  // namespace

extern "C" {

size_t s3g_eval_metrics_workspace_bytes(int C, int H, int W) {
    if (C <= 0 || H <= 0 || W <= 0) return 0;
    const dim3 g = eval_grid(C, H, W);
    return 256 + sizeof(float) * EV_PARTS * (size_t)g.x * g.y * g.z;
}

int s3g_eval_metrics(int C, int H, int W, const float* image, const float* gt, const uint8_t* mask, double* out,
                     void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (C < 1 || C > 4) return fail(S3G_ERR_ARG, "eval_metrics: 1 <= C <= 4 channels expected");
    if (H < 7 || W < 7) return fail(S3G_ERR_ARG, "eval_metrics: image sides must be >= 7 (the SSIM window)");
    if ((int64_t)H * W >= (1ll << 31) / C) return fail(S3G_ERR_ARG, "eval_metrics: image too large");
    if (!image || !gt || !out || !workspace) return fail(S3G_ERR_ARG, "eval_metrics: null image/gt/out/workspace");
    const dim3 g = eval_grid(C, H, W);
    float* partial = reinterpret_cast<float*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    eval_metrics_kernel<<<g, EV_THREADS, 0, stream>>>(H, W, image, gt, mask, partial);
    S3G_CUDA(cudaGetLastError(), "eval_metrics launch");
    eval_reduce_kernel<<<C, 256, 0, stream>>>((int)(g.x * g.y), partial, out);
    S3G_CUDA(cudaGetLastError(), "eval_reduce launch");
    return S3G_OK;
}

}  // extern "C"
