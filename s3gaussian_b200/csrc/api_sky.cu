// api_sky.cu - extern "C" entry points of the sky model (see include/s3g_b200.h and sky.cuh).
#include <algorithm>
#include <climits>
#include <cstdint>

#include "api_common.cuh"
#include "sky.cuh"

using namespace s3g;

namespace {
inline int fail(int code, const char* what) { return s3g::api_fail(code, what); }

bool width_ok(int w) { return w >= 64 && w <= 256 && w % 64 == 0; }

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// split-K count of a weight-gradient product [M x N] over np pixels: enough CTAs for two per SM (132 SMs), each with at
// least 256 pixels; a function of the shapes only, so the partition (and the summation order) never changes.  It does
// not decrease with np, so the chunk size bounds the partials.
int split_for(int M, int N, int np) {
    const int tiles = ((M + SKY_GB - 1) / SKY_GB) * ((N + SKY_GB - 1) / SKY_GB);
    return std::max(1, std::min((264 + tiles - 1) / tiles, np / 256));
}

// float counts of the workspace regions
struct SkyLayout {
    int wd, chunk;
    size_t f0, f1;                       // forward: prepared B fragments (floats)
    size_t w0p, w1p, w2p;                // backward: padded weights
    size_t x1, h2, dz, d2, d1;           // backward: one chunk's activations
    size_t g0, g1, g2;                   // backward: accumulated [dW | db] blocks
    int s0, s1, s2;                      // backward: split-K counts at a full chunk
    size_t fwd_bytes() const { return align256(f0 * 4) + align256(f1 * 4); }
    size_t part() const { return s0 * g0 + s1 * g1 + s2 * g2; }
    size_t bwd_bytes() const {
        size_t b = 0;
        for (size_t n : {w0p, w1p, w2p, x1, h2, dz, d2, d1, g0, g1, g2}) b += align256(n * 4);
        return b + align256(part() * 4);
    }
};

SkyLayout layout(int wd, int H, int W) {
    SkyLayout l;
    l.wd = wd;
    l.chunk = (int)std::min<long long>((long long)H * W, SKY_CHUNK);
    const size_t NT = wd / 8, C = l.chunk;
    l.f0 = NT * 5 * 32 * 4;
    l.f1 = NT * (NT + SKY_EP / 8) * 32 * 4;
    l.w0p = (size_t)wd * SKY_EP;
    l.w1p = (size_t)wd * (wd + SKY_EP);
    l.w2p = 8 * (size_t)(wd + 8);
    l.x1 = C * (wd + SKY_EP);
    l.h2 = C * (wd + 8);
    l.dz = C * 8;
    l.d2 = C * wd;
    l.d1 = C * wd;
    l.g0 = l.w0p;
    l.g1 = l.w1p;
    l.g2 = l.w2p;
    l.s0 = split_for(wd, SKY_EP, l.chunk);
    l.s1 = split_for(wd, wd + SKY_EP, l.chunk);
    l.s2 = split_for(8, wd + 8, l.chunk);
    return l;
}

int check_common(const s3g_sky_net* net, int H, int W, const float* c2w, const float* intrinsic, const void* ws,
                 const char* who) {
    if (!net) return fail(S3G_ERR_ARG, who);
    if (!width_ok(net->width)) return fail(S3G_ERR_ARG, "sky: width must be a multiple of 64 in [64, 256]");
    if (H < 1 || W < 1) return fail(S3G_ERR_ARG, "sky: H and W must be >= 1");
    if (3LL * H * W > INT_MAX) return fail(S3G_ERR_ARG, "sky: 3 * H * W too large for 32-bit pixel indices");
    if (!net->w0 || !net->b0 || !net->w1 || !net->b1 || !net->w2 || !net->b2 || !c2w || !intrinsic)
        return fail(S3G_ERR_ARG, "sky: null pointer");
    if (!ws) return fail(S3G_ERR_ARG, "sky: null workspace");
    if (reinterpret_cast<uintptr_t>(ws) % 16 != 0) return fail(S3G_ERR_ARG, "sky: workspace not 16-byte aligned");
    return S3G_OK;
}

SkyNet to_net(const s3g_sky_net* n) { return SkyNet{n->width, n->w0, n->b0, n->w1, n->b1, n->w2, n->b2}; }

template <bool AK, bool BK, int EPI>
int gemm(const SkyGemm& g, int splits, cudaStream_t stream, const char* what) {
    const dim3 grid((g.M + SKY_GB - 1) / SKY_GB, (g.N + SKY_GB - 1) / SKY_GB, splits);
    sky_gemm_kernel<AK, BK, EPI><<<grid, 128, 0, stream>>>(g);
    S3G_CUDA(cudaGetLastError(), what);
    return S3G_OK;
}
}  // namespace

extern "C" {

size_t s3g_sky_workspace_bytes(int width, int H, int W) {
    if (!width_ok(width) || H < 1 || W < 1 || 3LL * H * W > INT_MAX) return 0;
    const SkyLayout l = layout(width, H, W);
    return std::max(l.fwd_bytes(), l.bwd_bytes());
}

int s3g_sky_forward(const s3g_sky_net* net, int H, int W, const float* c2w, const float* intrinsic, float* out_sky,
                    void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = check_common(net, H, W, c2w, intrinsic, workspace, "sky_forward: null net")) return rc;
    if (!out_sky) return fail(S3G_ERR_ARG, "sky_forward: null pointer");
    const SkyLayout l = layout(net->width, H, W);
    float4* f0 = static_cast<float4*>(workspace);
    float4* f1 = reinterpret_cast<float4*>(static_cast<char*>(workspace) + align256(l.f0 * 4));
    const SkyNet n = to_net(net);
    sky_prep_forward_kernel<<<(unsigned)((l.f0 + l.f1) / 4 + 255) / 256, 256, 0, stream>>>(n, f0, f1);
    S3G_CUDA(cudaGetLastError(), "sky_prep_forward launch");
    const SkyCam cam{H, W, c2w, intrinsic};
    const int px_per_cta = 32 * SKY_FWD_WARPS;
    const unsigned grid = (unsigned)(((long long)H * W + px_per_cta - 1) / px_per_cta);
    switch (net->width) {
        case 64: sky_forward_kernel<64><<<grid, px_per_cta, 0, stream>>>(n, cam, f0, f1, out_sky); break;
        case 128: sky_forward_kernel<128><<<grid, px_per_cta, 0, stream>>>(n, cam, f0, f1, out_sky); break;
        case 192: sky_forward_kernel<192><<<grid, px_per_cta, 0, stream>>>(n, cam, f0, f1, out_sky); break;
        default: sky_forward_kernel<256><<<grid, px_per_cta, 0, stream>>>(n, cam, f0, f1, out_sky); break;
    }
    S3G_CUDA(cudaGetLastError(), "sky_forward launch");
    return S3G_OK;
}

int s3g_sky_backward(const s3g_sky_net* net, int H, int W, const float* c2w, const float* intrinsic,
                     const float* dL_dsky, const s3g_sky_net_grads* grads, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (int rc = check_common(net, H, W, c2w, intrinsic, workspace, "sky_backward: null net")) return rc;
    if (!dL_dsky || !grads || !grads->w0 || !grads->b0 || !grads->w1 || !grads->b1 || !grads->w2 || !grads->b2)
        return fail(S3G_ERR_ARG, "sky_backward: null pointer");
    const int wd = net->width, HW = H * W;
    const SkyLayout l = layout(wd, H, W);
    char* p = static_cast<char*>(workspace);
    auto take = [&](size_t n) { float* r = reinterpret_cast<float*>(p); p += align256(n * 4); return r; };
    float *w0p = take(l.w0p), *w1p = take(l.w1p), *w2p = take(l.w2p);
    float *x1 = take(l.x1), *h2 = take(l.h2), *dz = take(l.dz), *d2 = take(l.d2), *d1 = take(l.d1);
    float *g0 = take(l.g0), *g1 = take(l.g1), *g2 = take(l.g2);
    float* part = take(l.part());
    const SkyNet n = to_net(net);
    const size_t nprep = l.w0p + l.w1p + l.w2p;
    sky_prep_backward_kernel<<<(unsigned)((nprep + 255) / 256), 256, 0, stream>>>(n, w0p, w1p, w2p);
    S3G_CUDA(cudaGetLastError(), "sky_prep_backward launch");
    const SkyCam cam{H, W, c2w, intrinsic};
    const int K1 = wd + SKY_EP, K2 = wd + 8;
    for (int pix0 = 0, chunk = 0; pix0 < HW; pix0 += l.chunk, ++chunk) {
        const int np = std::min(l.chunk, HW - pix0);
        sky_encode_kernel<<<(np + 127) / 128, 128, 0, stream>>>(cam, wd, pix0, np, x1, h2);
        S3G_CUDA(cudaGetLastError(), "sky_encode launch");
        // h1 = relu([enc | 1] W0p^T) into X1[:, :Wd]; h2 = relu(X1 W1p^T) into H2[:, :Wd]
        SkyGemm q{np, wd, SKY_EP, x1 + wd, K1, w0p, SKY_EP, x1, K1, 0, SKY_EP, nullptr, 0};
        if (int rc = gemm<true, true, SKY_EPI_RELU>(q, 1, stream, "sky_gemm layer 1 launch")) return rc;
        q = SkyGemm{np, wd, K1, x1, K1, w1p, K1, h2, K2, 0, K1, nullptr, 0};
        if (int rc = gemm<true, true, SKY_EPI_RELU>(q, 1, stream, "sky_gemm layer 2 launch")) return rc;
        sky_head_kernel<<<(np + 7) / 8, 256, 0, stream>>>(wd, HW, pix0, np, w2p, h2, dL_dsky, dz, d2);
        S3G_CUDA(cudaGetLastError(), "sky_head launch");
        // dL/d(pre-activation of h1) = (D2 W1[:, :Wd]) (h1 > 0)
        q = SkyGemm{np, wd, wd, d2, wd, w1p, K1, d1, wd, 0, wd, x1, K1};
        if (int rc = gemm<true, false, SKY_EPI_MASK>(q, 1, stream, "sky_gemm dh1 launch")) return rc;
        // weight gradients over the chunk's pixels: a fixed split of the pixels, one partial per split
        float *p1 = part, *p0 = part + (size_t)l.s1 * l.g1, *p2 = p0 + (size_t)l.s0 * l.g0;
        const struct { int M, N; const float* a; int lda; const float* b; int ldb; float *part, *acc; size_t n; } wg[3] = {
            {wd, K1, d2, wd, x1, K1, p1, g1, l.g1}, {wd, SKY_EP, d1, wd, x1 + wd, K1, p0, g0, l.g0},
            {8, K2, dz, 8, h2, K2, p2, g2, l.g2}};
        for (const auto& r : wg) {
            const int want = split_for(r.M, r.N, np);
            const int kper = ((np + want - 1) / want + SKY_GK - 1) / SKY_GK * SKY_GK;
            const int S = (np + kper - 1) / kper;
            q = SkyGemm{r.M, r.N, np, r.a, r.lda, r.b, r.ldb, r.part, r.N, r.n, kper, nullptr, 0};
            if (int rc = gemm<false, false, SKY_EPI_STORE>(q, S, stream, "sky_gemm weight-gradient launch")) return rc;
            sky_reduce_kernel<<<(unsigned)((r.n + 255) / 256), 256, 0, stream>>>((int)r.n, S, r.part, r.acc, chunk == 0);
            S3G_CUDA(cudaGetLastError(), "sky_reduce launch");
        }
    }
    const SkyGrads o{grads->w0, grads->b0, grads->w1, grads->b1, grads->w2, grads->b2};
    sky_scatter_kernel<<<(unsigned)((l.g0 + l.g1 + 3 * (size_t)K2 + 255) / 256), 256, 0, stream>>>(wd, g0, g1, g2, o);
    S3G_CUDA(cudaGetLastError(), "sky_scatter launch");
    return S3G_OK;
}

}  // extern "C"
