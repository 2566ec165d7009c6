// api_bilagrid.cu - extern "C" entry points of the bilateral-grid colour correction (see include/s3g_b200.h).
#include <algorithm>
#include <climits>
#include <cstdint>
#include <vector>

#include "api_common.cuh"
#include "bilagrid.cuh"

using namespace s3g;

namespace {
inline int fail(int code, const char* what) { return s3g::api_fail(code, what); }

int check_grid(int N, int L, int GY, int GX) {
    if (N <= 0 || L <= 0 || GY <= 0 || GX <= 0) return fail(S3G_ERR_ARG, "bilagrid: a grid size <= 0");
    if ((long long)N * 12 * L * GY * GX > INT_MAX)
        return fail(S3G_ERR_ARG, "bilagrid: N * 12 * L * GY * GX too large for 32-bit element indices");
    return S3G_OK;
}

int check_slice(int N, int L, int GY, int GX, const float* grids, int B, int H, int W, const int32_t* ids,
                const float* rgb) {
    if (int rc = check_grid(N, L, GY, GX)) return rc;
    if (B <= 0 || H <= 0 || W <= 0) return fail(S3G_ERR_ARG, "bilagrid_slice: an image size <= 0");
    if (3LL * H * W > INT_MAX) return fail(S3G_ERR_ARG, "bilagrid_slice: 3 * H * W too large for 32-bit pixel indices");
    if (!grids || !ids || !rgb) return fail(S3G_ERR_ARG, "bilagrid_slice: null pointer");
    std::vector<int32_t> sorted(ids, ids + B);
    std::sort(sorted.begin(), sorted.end());
    if (sorted.front() < 0 || sorted.back() >= N) return fail(S3G_ERR_ARG, "bilagrid_slice: an image id outside [0, N)");
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
        return fail(S3G_ERR_ARG, "bilagrid_slice: duplicate image ids");
    return S3G_OK;
}

BgIds chunk_ids(const int32_t* ids, int b0, int nb) {
    BgIds c;
    for (int k = 0; k < nb; ++k) c.id[k] = ids[b0 + k];
    return c;
}

// the support of a cell column along one axis, at most: the pixel centres within one cell on either side, plus the
// one-pixel margin bg_support adds on each side
long long support_extent(int size, int extent) {
    if (size == 1) return extent;
    return std::min<long long>(extent, (long long)(2.0 * extent / (size - 1)) + 6);
}

BgGather gather_plan(int L, int GY, int GX, int H, int W) {
    BgGather q;
    const long long n = support_extent(GX, W) * support_extent(GY, H);
    q.splits = (int)std::max<long long>(1, (n + BG_PIX_PER_CTA - 1) / BG_PIX_PER_CTA);
    q.chunk = (int)((n + q.splits - 1) / q.splits);
    q.nzc = (L + BG_LEVEL_CHUNK - 1) / BG_LEVEL_CHUNK;
    return q;
}
}  // namespace

extern "C" {

int s3g_bilagrid_slice_forward(int N, int L, int GY, int GX, const float* grids, int B, int H, int W,
                               const int32_t* image_ids, const float* rgb, float* out, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = check_slice(N, L, GY, GX, grids, B, H, W, image_ids, rgb)) return rc;
    if (!out) return fail(S3G_ERR_ARG, "bilagrid_slice_forward: null pointer");
    const BgShape s{L, GY, GX, H, W};
    const int HW = H * W;
    for (int b0 = 0; b0 < B; b0 += BG_MAX_IDS) {
        const int nb = std::min(BG_MAX_IDS, B - b0);
        const size_t off = (size_t)b0 * 3 * HW;
        bilagrid_slice_forward_kernel<<<dim3((HW + BG_THREADS - 1) / BG_THREADS, nb), BG_THREADS, 0, stream>>>(
            s, grids, chunk_ids(image_ids, b0, nb), rgb + off, out + off);
        S3G_CUDA(cudaGetLastError(), "bilagrid_slice_forward launch");
    }
    return S3G_OK;
}

size_t s3g_bilagrid_slice_backward_workspace_bytes(int N, int L, int GY, int GX, int B, int H, int W) {
    if (N <= 0 || L <= 0 || GY <= 0 || GX <= 0 || B <= 0 || H <= 0 || W <= 0) return 0;
    const BgGather q = gather_plan(L, GY, GX, H, W);
    return sizeof(float) * (size_t)std::min(B, BG_MAX_IDS) * q.nzc * GY * GX * q.splits * BG_LEVEL_CHUNK * 12;
}

int s3g_bilagrid_slice_backward(int N, int L, int GY, int GX, const float* grids, int B, int H, int W,
                                const int32_t* image_ids, const float* rgb, const float* grad_out, float* grad_rgb,
                                float* grad_grids, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = check_slice(N, L, GY, GX, grids, B, H, W, image_ids, rgb)) return rc;
    if (!grad_out || !grad_grids || !workspace) return fail(S3G_ERR_ARG, "bilagrid_slice_backward: null pointer");
    if (reinterpret_cast<uintptr_t>(workspace) % 16 != 0)
        return fail(S3G_ERR_ARG, "bilagrid_slice_backward: workspace not 16-byte aligned");
    const BgGather q = gather_plan(L, GY, GX, H, W);
    const int nbmax = std::min(B, BG_MAX_IDS);
    if ((long long)GY * GX * q.splits > INT_MAX || (long long)nbmax * q.nzc > 65535)
        return fail(S3G_ERR_ARG, "bilagrid_slice_backward: grid too large for one launch");
    const BgShape s{L, GY, GX, H, W};
    const int HW = H * W;
    const size_t smem = sizeof(float) * std::min(L, BG_LEVEL_CHUNK) * 12 * (BG_GATHER_THREADS + 1);
    S3G_CUDA(cudaFuncSetAttribute(bilagrid_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
             "bilagrid_gather smem attribute");
    float* partial = static_cast<float*>(workspace);
    const long long per_image = 12LL * L * GY * GX;
    for (int b0 = 0; b0 < B; b0 += BG_MAX_IDS) {
        const int nb = std::min(BG_MAX_IDS, B - b0);
        const size_t off = (size_t)b0 * 3 * HW;
        const BgIds ids = chunk_ids(image_ids, b0, nb);
        bilagrid_gather_kernel<<<dim3(GY * GX * q.splits, nb * q.nzc), BG_GATHER_THREADS, smem, stream>>>(
            s, q, grids, ids, rgb + off, grad_out + off, grad_rgb ? grad_rgb + off : nullptr, partial);
        S3G_CUDA(cudaGetLastError(), "bilagrid_gather launch");
        const long long total = nb * per_image;
        bilagrid_sum_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(s, q, nb, ids, partial, grad_grids);
        S3G_CUDA(cudaGetLastError(), "bilagrid_sum launch");
    }
    return S3G_OK;
}

namespace {
BgTv tv_plan(int N, int L, int GY, int GX) {
    BgTv t;
    t.n = (long long)N * 12 * L * GY * GX;
    t.L = L; t.GY = GY; t.GX = GX;
    // gsplat divides each axis' sum by the element count of the shifted grid without the batch dimension (at least 1)
    const double per = 12.0 * L * GY * GX;
    t.inv[0] = GX > 1 ? 1.0 / (per / GX * (GX - 1)) : 0.0;
    t.inv[1] = GY > 1 ? 1.0 / (per / GY * (GY - 1)) : 0.0;
    t.inv[2] = L > 1 ? 1.0 / (per / L * (L - 1)) : 0.0;
    t.invN = 1.0 / N;
    return t;
}
int tv_blocks(long long n) { return (int)std::min<long long>(BG_TV_BLOCKS, (n + BG_TV_THREADS - 1) / BG_TV_THREADS); }
}  // namespace

size_t s3g_bilagrid_tv_workspace_bytes(int N, int L, int GY, int GX) {
    if (N <= 0 || L <= 0 || GY <= 0 || GX <= 0) return 0;
    return sizeof(double) * (size_t)tv_blocks((long long)N * 12 * L * GY * GX);
}

int s3g_bilagrid_tv_forward(int N, int L, int GY, int GX, const float* grids, float* loss, void* workspace,
                            void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = check_grid(N, L, GY, GX)) return rc;
    if (!grids || !loss || !workspace) return fail(S3G_ERR_ARG, "bilagrid_tv_forward: null pointer");
    if (reinterpret_cast<uintptr_t>(workspace) % 8 != 0)
        return fail(S3G_ERR_ARG, "bilagrid_tv_forward: workspace not 8-byte aligned");
    const BgTv t = tv_plan(N, L, GY, GX);
    const int nb = tv_blocks(t.n);
    double* partial = static_cast<double*>(workspace);
    bilagrid_tv_forward_kernel<<<nb, BG_TV_THREADS, 0, stream>>>(t, grids, partial);
    S3G_CUDA(cudaGetLastError(), "bilagrid_tv_forward launch");
    bilagrid_tv_reduce_kernel<<<1, 1024, 0, stream>>>(nb, t.invN, partial, loss);
    S3G_CUDA(cudaGetLastError(), "bilagrid_tv_reduce launch");
    return S3G_OK;
}

int s3g_bilagrid_tv_backward(int N, int L, int GY, int GX, const float* grids, const float* gscale, float* grad,
                             void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = check_grid(N, L, GY, GX)) return rc;
    if (!grids || !gscale || !grad) return fail(S3G_ERR_ARG, "bilagrid_tv_backward: null pointer");
    const BgTv t = tv_plan(N, L, GY, GX);
    bilagrid_tv_backward_kernel<<<(unsigned)((t.n + BG_TV_THREADS - 1) / BG_TV_THREADS), BG_TV_THREADS, 0, stream>>>(
        t, grids, gscale, grad);
    S3G_CUDA(cudaGetLastError(), "bilagrid_tv_backward launch");
    return S3G_OK;
}

}  // extern "C"
