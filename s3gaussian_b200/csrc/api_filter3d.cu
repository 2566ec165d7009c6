// api_filter3d.cu - extern "C" entry points of the 3-D smoothing filter (see include/s3g_b200.h).
#include <climits>
#include <cstdint>

#include "api_common.cuh"
#include "filter3d.cuh"

using namespace s3g;

namespace {
inline int fail(int code, const char* what) { return s3g::api_fail(code, what); }
inline int blocks(int P) { return (P + F3D_BLOCK - 1) / F3D_BLOCK; }
}  // namespace

extern "C" {

size_t s3g_filter3d_compute_workspace_bytes(int P) { return P > 0 ? 16 : 0; }

int s3g_filter3d_compute(int P, const float* xyz, int C, const float* viewmatrices, const float* cams,
                         float* filter_3d, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "filter3d_compute: P < 0");
    if (P == 0) return S3G_OK;
    if (C < 1) return fail(S3G_ERR_ARG, "filter3d_compute: C < 1");
    if (P > INT_MAX / 3 || C > INT_MAX / 16)
        return fail(S3G_ERR_ARG, "filter3d_compute: P or C too large for 32-bit element indices");
    if (!xyz || !viewmatrices || !cams || !filter_3d || !workspace)
        return fail(S3G_ERR_ARG, "filter3d_compute: null pointer");
    if (reinterpret_cast<uintptr_t>(workspace) % 16 != 0)
        return fail(S3G_ERR_ARG, "filter3d_compute: workspace not 16-byte aligned");
    uint32_t* ws = static_cast<uint32_t*>(workspace);
    S3G_CUDA(cudaMemsetAsync(ws, 0, sizeof(uint32_t), stream), "filter3d_compute memset");
    filter3d_depth_kernel<<<blocks(P), F3D_BLOCK, 0, stream>>>(P, xyz, C, viewmatrices, cams, filter_3d, ws);
    filter3d_fill_kernel<<<blocks(P), F3D_BLOCK, 0, stream>>>(P, filter_3d, ws);
    S3G_CUDA(cudaGetLastError(), "filter3d_compute launch");
    return S3G_OK;
}

int s3g_filter3d_apply_forward(int P, const float* scales, const float* opacity, const float* filter_3d,
                               float* out_scales, float* out_opacity, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "filter3d_apply_forward: P < 0");
    if (P == 0) return S3G_OK;
    if (P > INT_MAX / 3) return fail(S3G_ERR_ARG, "filter3d_apply_forward: P too large for 32-bit element indices");
    if (!scales || !opacity || !filter_3d || !out_scales || !out_opacity)
        return fail(S3G_ERR_ARG, "filter3d_apply_forward: null pointer");
    filter3d_apply_forward_kernel<<<blocks(P), F3D_BLOCK, 0, stream>>>(P, scales, opacity, filter_3d, out_scales,
                                                                       out_opacity);
    S3G_CUDA(cudaGetLastError(), "filter3d_apply_forward launch");
    return S3G_OK;
}

int s3g_filter3d_apply_backward(int P, const float* scales, const float* opacity, const float* filter_3d,
                                const float* g_out_scales, const float* g_out_opacity, float* g_scales,
                                float* g_opacity, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "filter3d_apply_backward: P < 0");
    if (P == 0) return S3G_OK;
    if (P > INT_MAX / 3) return fail(S3G_ERR_ARG, "filter3d_apply_backward: P too large for 32-bit element indices");
    if (!scales || !opacity || !filter_3d || !g_out_scales || !g_out_opacity || !g_scales || !g_opacity)
        return fail(S3G_ERR_ARG, "filter3d_apply_backward: null pointer");
    filter3d_apply_backward_kernel<<<blocks(P), F3D_BLOCK, 0, stream>>>(P, scales, opacity, filter_3d, g_out_scales,
                                                                        g_out_opacity, g_scales, g_opacity);
    S3G_CUDA(cudaGetLastError(), "filter3d_apply_backward launch");
    return S3G_OK;
}

}  // extern "C"
