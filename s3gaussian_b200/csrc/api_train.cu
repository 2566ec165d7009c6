// api_train.cu - extern "C" entry points of the training-step kernels (see include/s3g_b200.h).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>

#include "api_common.cuh"
#include "train_step.cuh"

using namespace s3g;

namespace {
inline int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return s3g::api_fail(code, what, e); }
}  // namespace

extern "C" {

// ---- training-step kernels (train_step.cuh) --------------------------------------------------
int s3g_adam_step(int n, const s3g_adam_tensor* tensors, double beta1, double beta2, double eps, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (n < 0 || (n > 0 && !tensors)) return fail(S3G_ERR_ARG, "adam_step: bad tensor table");
    AdamArgs a;
    a.w1 = (float)(1.0 - beta1);
    a.beta2 = (float)beta2;
    a.omb2 = (float)(1.0 - beta2);
    a.eps = (float)eps;
    int i = 0;
    while (i < n) {
        a.count = 0;
        int blocks = 0;
        for (; i < n && a.count < ADAM_MAX_TENSORS; ++i) {
            const s3g_adam_tensor& t = tensors[i];
            if (t.numel == 0) continue;
            if (t.numel < 0 || !t.param || !t.grad || !t.exp_avg || !t.exp_avg_sq || t.step < 1)
                return fail(S3G_ERR_ARG, "adam_step: null pointer, negative numel or step < 1");
            const long long nb = (t.numel + ADAM_CHUNK - 1) / ADAM_CHUNK;
            if (nb + blocks > 0x7fffffffLL) return fail(S3G_ERR_ARG, "adam_step: tensor too large");
            AdamTensor& d = a.t[a.count];
            d.p = t.param; d.g = t.grad; d.m = t.exp_avg; d.v = t.exp_avg_sq; d.n = t.numel;
            const double bc1 = 1.0 - std::pow(beta1, (double)t.step);
            const double bc2 = 1.0 - std::pow(beta2, (double)t.step);
            d.step_size = (float)(t.lr / bc1);
            d.bc2_sqrt = (float)std::sqrt(bc2);
            a.block_start[a.count] = blocks;
            blocks += (int)nb;
            ++a.count;
        }
        a.block_start[a.count] = blocks;
        if (blocks > 0) {
            adam_multi_tensor_kernel<<<blocks, ADAM_THREADS, 0, stream>>>(a);
            S3G_CUDA(cudaGetLastError(), "adam_step launch");
        }
    }
    return S3G_OK;
}

int s3g_adam_step_selective(int n, const s3g_adam_tensor* tensors, const int32_t* row_width, int64_t rows,
                            const uint8_t* visible, double beta1, double beta2, double eps, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (n < 0 || (n > 0 && (!tensors || !row_width))) return fail(S3G_ERR_ARG, "adam_step_selective: bad tensor table");
    if (rows < 0) return fail(S3G_ERR_ARG, "adam_step_selective: rows < 0");
    // every argument is checked before the first launch, so an error leaves every tensor as it was
    long long total_blocks = 0;
    for (int i = 0; i < n; ++i) {
        const s3g_adam_tensor& t = tensors[i];
        const int w = row_width[i];
        if (w < 0) return fail(S3G_ERR_ARG, "adam_step_selective: row_width < 0");
        if (t.numel < 0) return fail(S3G_ERR_ARG, "adam_step_selective: negative numel");
        if (w > 0 && (t.numel % w != 0 || t.numel / w != rows))
            return fail(S3G_ERR_ARG, "adam_step_selective: a masked tensor needs numel == rows * row_width");
        if (t.numel == 0) continue;
        if (!t.param || !t.grad || !t.exp_avg || !t.exp_avg_sq || t.step < 1)
            return fail(S3G_ERR_ARG, "adam_step_selective: null pointer or step < 1");
        if (w > 0 && !visible) return fail(S3G_ERR_ARG, "adam_step_selective: null visible");
        if (w > 0 && t.numel > 0x7fffffffLL)
            return fail(S3G_ERR_ARG, "adam_step_selective: a masked tensor must have fewer than 2^31 elements");
        total_blocks += (t.numel + ADAM_CHUNK - 1) / ADAM_CHUNK;
        if (total_blocks > 0x7fffffffLL) return fail(S3G_ERR_ARG, "adam_step_selective: tensors too large");
    }
    AdamSelectiveArgs a;
    a.w1 = (float)(1.0 - beta1);
    a.beta2 = (float)beta2;
    a.omb2 = (float)(1.0 - beta2);
    a.eps = (float)eps;
    a.visible = visible;
    int i = 0;
    while (i < n) {
        a.count = 0;
        int blocks = 0;
        for (; i < n && a.count < ADAM_MAX_TENSORS; ++i) {
            const s3g_adam_tensor& t = tensors[i];
            if (t.numel == 0) continue;
            AdamTensor& d = a.t[a.count];
            d.p = t.param; d.g = t.grad; d.m = t.exp_avg; d.v = t.exp_avg_sq; d.n = t.numel;
            const double bc1 = 1.0 - std::pow(beta1, (double)t.step);
            const double bc2 = 1.0 - std::pow(beta2, (double)t.step);
            d.step_size = (float)(t.lr / bc1);
            d.bc2_sqrt = (float)std::sqrt(bc2);
            a.row_width[a.count] = (unsigned)row_width[i];
            a.block_start[a.count] = blocks;
            blocks += (int)((t.numel + ADAM_CHUNK - 1) / ADAM_CHUNK);
            ++a.count;
        }
        a.block_start[a.count] = blocks;
        if (blocks > 0) {
            adam_selective_kernel<<<blocks, ADAM_THREADS, 0, stream>>>(a);
            S3G_CUDA(cudaGetLastError(), "adam_step_selective launch");
        }
    }
    return S3G_OK;
}

int s3g_densify_stats(int P,const float* viewspace_grad, const int* radii, float* xyz_gradient_accum,
                      float* denom, float* max_radii2D, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "densify_stats: P < 0");
    if (P == 0) return S3G_OK;
    if (!viewspace_grad || !radii || !xyz_gradient_accum || !denom || !max_radii2D)
        return fail(S3G_ERR_ARG, "densify_stats: null pointer");
    densify_stats_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, viewspace_grad, radii, xyz_gradient_accum, denom, max_radii2D);
    S3G_CUDA(cudaGetLastError(), "densify_stats launch");
    return S3G_OK;
}

int s3g_densify_stats_abs(int P, const float* viewspace_grad, const float* viewspace_absgrad, const int* radii,
                          float* xyz_gradient_accum, float* xyz_gradient_accum_abs, float* denom, float* max_radii2D,
                          void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "densify_stats_abs: P < 0");
    if (P == 0) return S3G_OK;
    if (!viewspace_grad || !viewspace_absgrad || !radii || !xyz_gradient_accum || !xyz_gradient_accum_abs || !denom ||
        !max_radii2D)
        return fail(S3G_ERR_ARG, "densify_stats_abs: null pointer");
    densify_stats_abs_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, viewspace_grad, viewspace_absgrad, radii,
                                                                  xyz_gradient_accum, xyz_gradient_accum_abs, denom,
                                                                  max_radii2D);
    S3G_CUDA(cudaGetLastError(), "densify_stats_abs launch");
    return S3G_OK;
}

namespace {
constexpr int kDepthBlocks = 592;    // 4 per SM
struct LossPlan {
    size_t map_floats, img_blocks;
    dim3 grid;
};
LossPlan loss_plan(int B, int C, int H, int W) {
    LossPlan p;
    p.map_floats = (size_t)B * C * H * W;
    p.grid = dim3((W + LOSS_T - 1) / LOSS_T, (H + LOSS_T - 1) / LOSS_T, B * C);
    p.img_blocks = (size_t)p.grid.x * p.grid.y * p.grid.z;
    return p;
}
}  // namespace

size_t s3g_image_loss_workspace_bytes(int B, int C, int H, int W) {
    if (B <= 0 || C < 0 || H <= 0 || W <= 0) return 0;
    const LossPlan p = loss_plan(B, C, H, W);
    return 256 + sizeof(float) * (3 * p.map_floats + 2 * p.img_blocks + 2 * kDepthBlocks);
}

namespace {
struct LossBufs { float *m0, *m1, *m2, *part_img, *part_dep; };
LossBufs loss_bufs(const LossPlan& p, const void* workspace) {
    LossBufs b;
    float* ws = reinterpret_cast<float*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    b.m0 = ws; b.m1 = b.m0 + p.map_floats; b.m2 = b.m1 + p.map_floats;
    b.part_img = b.m2 + p.map_floats; b.part_dep = b.part_img + 2 * p.img_blocks;
    return b;
}
LossWin loss_window() {
    // gaussian(11, 1.5) of loss_utils.py:56-58: float32 exp values normalised by their float32 sum
    LossWin win;
    float g[11], s = 0.f;
    for (int x = 0; x < 11; ++x) g[x] = (float)std::exp(-(double)((x - 5) * (x - 5)) / (2.0 * 1.5 * 1.5));
    for (int x = 0; x < 11; ++x) s += g[x];
    for (int x = 0; x < 11; ++x) win.w[x] = g[x] / s;
    return win;
}
int loss_check(int B, int C, int H, int W, const void* image, const void* gt, const void* depth, const void* gt_depth) {
    if (B <= 0 || C < 0 || H <= 0 || W <= 0) return fail(S3G_ERR_ARG, "image_loss: empty image");
    if ((long long)B * C > 65535) return fail(S3G_ERR_ARG, "image_loss: too many image planes");
    if (C > 0 && (!image || !gt)) return fail(S3G_ERR_ARG, "image_loss: null image pointer");
    if (C == 0 && !depth) return fail(S3G_ERR_ARG, "image_loss: neither image nor depth");
    if ((depth == nullptr) != (gt_depth == nullptr)) return fail(S3G_ERR_ARG, "image_loss: depth and gt_depth go together");
    return S3G_OK;
}
}  // namespace

int s3g_image_loss_forward(int B, int C, int H, int W, const float* image, const float* gt_image, const float* depth,
                           const float* gt_depth, float max_depth, double* sums, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = loss_check(B, C, H, W, image, gt_image, depth, gt_depth)) return rc;
    if (!sums || !workspace) return fail(S3G_ERR_ARG, "image_loss_forward: null sums/workspace");
    const LossPlan p = loss_plan(B, C, H, W);
    const LossBufs b = loss_bufs(p, workspace);
    if (C > 0) {
        loss_stats_kernel<<<p.grid, LOSS_THREADS, 0, stream>>>(H, W, image, gt_image, loss_window(), b.m0, b.m1, b.m2, b.part_img);
        S3G_CUDA(cudaGetLastError(), "loss_stats launch");
    }
    int ndep = 0;
    if (depth) {
        ndep = kDepthBlocks;
        loss_depth_stats_kernel<<<kDepthBlocks, LOSS_THREADS, 0, stream>>>((size_t)B * H * W, depth, gt_depth, max_depth, b.part_dep);
        S3G_CUDA(cudaGetLastError(), "loss_depth_stats launch");
    }
    loss_reduce_kernel<<<1, 256, 0, stream>>>((int)p.img_blocks, b.part_img, ndep, b.part_dep, sums);
    S3G_CUDA(cudaGetLastError(), "loss_reduce launch");
    return S3G_OK;
}

// ---- the same terms without SSIM (lambda_dssim == 0) ---------------------------------------------------------
int s3g_image_l1_depth_forward(int B, int C, int H, int W, const float* image, const float* gt_image, const float* depth,
                               const float* gt_depth, float max_depth, double* sums, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = loss_check(B, C, H, W, image, gt_image, depth, gt_depth)) return rc;
    if (!sums || !workspace) return fail(S3G_ERR_ARG, "image_l1_depth_forward: null sums/workspace");
    float* ws = reinterpret_cast<float*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    float* part_img = ws;
    float* part_dep = ws + 2 * kDepthBlocks;
    int nimg = 0, ndep = 0;
    if (C > 0) {
        nimg = kDepthBlocks;
        loss_l1_stats_kernel<<<kDepthBlocks, LOSS_THREADS, 0, stream>>>((size_t)B * C * H * W, image, gt_image, part_img);
        S3G_CUDA(cudaGetLastError(), "loss_l1_stats launch");
    }
    if (depth) {
        ndep = kDepthBlocks;
        loss_depth_stats_kernel<<<kDepthBlocks, LOSS_THREADS, 0, stream>>>((size_t)B * H * W, depth, gt_depth, max_depth, part_dep);
        S3G_CUDA(cudaGetLastError(), "loss_depth_stats launch");
    }
    loss_reduce_kernel<<<1, 256, 0, stream>>>(nimg, part_img, ndep, part_dep, sums);
    S3G_CUDA(cudaGetLastError(), "loss_reduce launch");
    return S3G_OK;
}

int s3g_image_l1_depth_backward(int B, int C, int H, int W, const float* image, const float* gt_image, const float* depth,
                                const float* gt_depth, float max_depth, const float* weights, const double* sums,
                                float* g_image, float* g_depth, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = loss_check(B, C, H, W, image, gt_image, depth, gt_depth)) return rc;
    if (!weights || !sums || (C > 0 && !g_image) || (depth && !g_depth))
        return fail(S3G_ERR_ARG, "image_l1_depth_backward: null pointer");
    if (C > 0) {
        const size_t n = (size_t)B * C * H * W;
        loss_l1_grad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(n, image, gt_image, weights, 1.0f / (float)n, g_image);
        S3G_CUDA(cudaGetLastError(), "loss_l1_grad launch");
    }
    if (depth) {
        const size_t nd = (size_t)B * H * W;
        loss_depth_grad_kernel<<<(unsigned)((nd + 255) / 256), 256, 0, stream>>>(nd, depth, gt_depth, max_depth, weights, sums, g_depth);
        S3G_CUDA(cudaGetLastError(), "loss_depth_grad launch");
    }
    return S3G_OK;
}

int s3g_image_loss_backward(int B, int C, int H, int W, const float* image, const float* gt_image, const float* depth,
                            const float* gt_depth, float max_depth, const float* weights, const double* sums,
                            const void* workspace, float* g_image, float* g_depth, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = loss_check(B, C, H, W, image, gt_image, depth, gt_depth)) return rc;
    if (!weights || !sums || !workspace || (C > 0 && !g_image) || (depth && !g_depth))
        return fail(S3G_ERR_ARG, "image_loss_backward: null pointer");
    const LossPlan p = loss_plan(B, C, H, W);
    const LossBufs b = loss_bufs(p, workspace);
    if (C > 0) {
        loss_grad_kernel<<<p.grid, LOSS_THREADS, 0, stream>>>(H, W, image, gt_image, loss_window(), b.m0, b.m1, b.m2, weights,
                                                             1.0f / (float)p.map_floats, g_image);
        S3G_CUDA(cudaGetLastError(), "loss_grad launch");
    }
    if (depth) {
        const size_t nd = (size_t)B * H * W;
        loss_depth_grad_kernel<<<(unsigned)((nd + 255) / 256), 256, 0, stream>>>(nd, depth, gt_depth, max_depth, weights, sums, g_depth);
        S3G_CUDA(cudaGetLastError(), "loss_depth_grad launch");
    }
    return S3G_OK;
}

// ---- HexPlane regularisers -------------------------------------------------------------------
namespace {
int reg_table(int n, const s3g_plane_desc* planes, bool need_grad, RegArgs& a) {
    if (n <= 0 || n > REG_MAX_PLANES || !planes) return fail(S3G_ERR_ARG, "plane_reg: 1..48 planes expected");
    int blocks = 0;
    a.count = n;
    for (int i = 0; i < n; ++i) {
        const s3g_plane_desc& d = planes[i];
        if (!d.plane || (need_grad && !d.grad)) return fail(S3G_ERR_ARG, "plane_reg: null plane / grad pointer");
        if (d.H < 3 || d.W < 1 || d.C < 4 || d.C % 4) return fail(S3G_ERR_ARG, "plane_reg: need H >= 3, W >= 1, C % 4 == 0");
        // the kernels read planes and write gradients as float4
        if ((reinterpret_cast<uintptr_t>(d.plane) | (need_grad ? reinterpret_cast<uintptr_t>(d.grad) : 0)) & 15)
            return fail(S3G_ERR_ARG, "plane_reg: plane / grad pointers must be 16-byte aligned");
        RegPlane& p = a.p[i];
        p.t = d.plane; p.g = d.grad; p.H = d.H; p.W = d.W; p.C = d.C;
        p.k_smooth = (float)((double)d.w_smooth / ((double)d.C * (d.H - 2) * d.W));
        p.k_l1 = (float)((double)d.w_l1 / ((double)d.C * d.H * d.W));
        const long long n4 = (long long)d.H * d.W * d.C / 4;
        a.block_start[i] = blocks;
        const long long nb = (n4 + REG_CHUNK4 - 1) / REG_CHUNK4;
        if (blocks + nb > 0x7fffffffLL) return fail(S3G_ERR_ARG, "plane_reg: planes too large");
        blocks += (int)nb;
    }
    a.block_start[n] = blocks;
    return blocks;
}
}  // namespace

size_t s3g_plane_reg_workspace_bytes(int n, const s3g_plane_desc* planes) {
    RegArgs a;
    const int blocks = reg_table(n, planes, false, a);
    return blocks < 0 ? 0 : 256 + sizeof(double) * (size_t)blocks;
}

int s3g_plane_reg_forward(int n, const s3g_plane_desc* planes, double* total, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    RegArgs a;
    const int blocks = reg_table(n, planes, false, a);
    if (blocks < 0) return blocks;
    if (!total || !workspace) return fail(S3G_ERR_ARG, "plane_reg_forward: null total/workspace");
    double* partial = reinterpret_cast<double*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    plane_reg_forward_kernel<<<blocks, REG_THREADS, 0, stream>>>(a, partial);
    S3G_CUDA(cudaGetLastError(), "plane_reg_forward launch");
    plane_reg_reduce_kernel<<<1, 256, 0, stream>>>(blocks, partial, total);
    S3G_CUDA(cudaGetLastError(), "plane_reg_reduce launch");
    return S3G_OK;
}

int s3g_plane_reg_backward(int n, const s3g_plane_desc* planes, const float* gscale, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    RegArgs a;
    const int blocks = reg_table(n, planes, true, a);
    if (blocks < 0) return blocks;
    if (!gscale) return fail(S3G_ERR_ARG, "plane_reg_backward: null gscale");
    plane_reg_backward_kernel<<<blocks, REG_THREADS, 0, stream>>>(a, gscale);
    S3G_CUDA(cudaGetLastError(), "plane_reg_backward launch");
    return S3G_OK;
}

// ---- densify / prune row gather ----------------------------------------------------------------
int s3g_gather_rows(int n, const s3g_row_tensor* tensors, int64_t n_out, int64_t n_kept, const int64_t* src_index,
                    void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (n <= 0 || n > ROWS_MAX_TENSORS || !tensors) return fail(S3G_ERR_ARG, "gather_rows: 1..32 tensors expected");
    if (n_out < 0 || n_kept < 0 || n_kept > n_out) return fail(S3G_ERR_ARG, "gather_rows: need 0 <= n_kept <= n_out");
    if (n_out == 0) return S3G_OK;
    if (!src_index) return fail(S3G_ERR_ARG, "gather_rows: null src_index");
    RowArgs a;
    a.count = n; a.n_out = n_out; a.n_kept = n_kept;
    a.src_index = reinterpret_cast<const long long*>(src_index);
    long long most = 0;
    for (int i = 0; i < n; ++i) {
        const s3g_row_tensor& t = tensors[i];
        if (!t.src || !t.dst || t.row_floats <= 0) return fail(S3G_ERR_ARG, "gather_rows: null pointer or row_floats <= 0");
        a.t[i] = RowTensor{t.src, t.dst, t.row_floats, t.zero_new};
        most = std::max(most, (long long)n_out * t.row_floats);
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long want = (most + 255) / 256;
    const int gx = (int)std::min<long long>(want, (long long)sms * 8);
    gather_rows_kernel<<<dim3(gx, n), 256, 0, stream>>>(a);
    S3G_CUDA(cudaGetLastError(), "gather_rows launch");
    return S3G_OK;
}

}  // extern "C"
