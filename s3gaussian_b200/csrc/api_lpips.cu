// api_lpips.cu - extern "C" entry points of LPIPS v0.1, AlexNet and VGG16 backbones (include/s3g_b200.h,
// csrc/lpips.cuh, csrc/lpips_vgg.cuh).
#include <algorithm>
#include <cstdint>

#include "api_common.cuh"
#include "common.cuh"
#include "lpips_vgg.cuh"

using namespace s3g;

namespace {
inline int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return s3g::api_fail(code, what, e); }

// float offsets inside the prepared buffer: the five layers' weight tiles, then every bias, then every lin weight
struct LpPrepared {
    size_t tiles[LP_LAYERS], bias[LP_LAYERS], lin[LP_LAYERS], total;
    LpPrepared() {
        size_t o = 0;
        for (int l = 0; l < LP_LAYERS; ++l) { tiles[l] = o; o += (size_t)lp_prep_floats<LpAlex>(l); }
        for (int l = 0; l < LP_LAYERS; ++l) { bias[l] = o; o += LpAlex::cout(l); }
        for (int l = 0; l < LP_LAYERS; ++l) { lin[l] = o; o += LpAlex::cout(l); }
        total = o;
    }
};

// the activations of one call: conv output l (channels-last, 2N images), max-pools after conv 1 and 2, tap partials
struct LpShapes {
    int64_t h[LP_LAYERS], w[LP_LAYERS];   // conv output sizes (the tap grids)
    int64_t ph[2], pw[2];                  // max-pool output sizes
    int64_t conv_elems[LP_LAYERS], pool_elems[2];
    int64_t tap_blocks[LP_LAYERS];
    size_t conv_off[LP_LAYERS], pool_off[2], part_off[LP_LAYERS], bytes;
    LpShapes(int N, int H, int W) {
        const int64_t NI = 2 * (int64_t)N;
        int64_t ih = H, iw = W;
        size_t o = 0;
        auto take = [&](int64_t bytes_) { const size_t at = o; o += ((size_t)bytes_ + 255) & ~(size_t)255; return at; };
        for (int l = 0; l < LP_LAYERS; ++l) {
            h[l] = (ih + 2 * LpAlex::pad(l) - LpAlex::ks(l)) / LpAlex::stride(l) + 1;
            w[l] = (iw + 2 * LpAlex::pad(l) - LpAlex::ks(l)) / LpAlex::stride(l) + 1;
            conv_elems[l] = NI * h[l] * w[l] * LpAlex::cout(l);
            conv_off[l] = take(conv_elems[l] * 4);
            ih = h[l]; iw = w[l];
            if (l < 2) {
                ph[l] = (ih - 3) / 2 + 1; pw[l] = (iw - 3) / 2 + 1;
                pool_elems[l] = NI * ph[l] * pw[l] * LpAlex::cout(l);
                pool_off[l] = take(pool_elems[l] * 4);
                ih = ph[l]; iw = pw[l];
            }
        }
        for (int l = 0; l < LP_LAYERS; ++l) {
            tap_blocks[l] = div_up64((int64_t)N * h[l] * w[l], LP_TAP_WARPS * LP_TAP_PIX);
            part_off[l] = take(tap_blocks[l] * 8);
        }
        bytes = o + 256;   // + alignment of the base
    }
    bool fits_int32() const {
        for (int l = 0; l < LP_LAYERS; ++l) if (conv_elems[l] >= INT32_MAX) return false;
        return true;   // the pools are smaller than the convolutions they follow
    }
};

bool args_ok(int N, int H, int W) {
    return N >= 1 && H >= 31 && W >= 31 && (int64_t)N * 3 * H * W < INT32_MAX && LpShapes(N, H, W).fits_int32();
}

// float offsets inside the backward's prepared buffer: conv 1's weights as given ([64][3][11][11], read by the CUDA
// core dgrad), then the dgrad tiles of convolutions 2-5
struct LpPreparedBwd {
    size_t w0, tiles[LP_LAYERS], total;
    LpPreparedBwd() {
        size_t o = 0;
        w0 = o; o += (size_t)LpAlex::cout(0) * lp_k<LpAlex>(0);
        tiles[0] = 0;
        for (int l = 1; l < LP_LAYERS; ++l) { tiles[l] = o; o += (size_t)lp_prep_floats<LpAlex>(l); }
        total = o;
    }
};

// The backward's two ping-pong gradient buffers, sized for all 2N images.  Going down, A holds the gradients at
// conv 5, 3 and 2's outputs and at conv 1's, B those at conv 4's output and at the two max-pool outputs.
struct LpBwdShapes {
    size_t a_off, b_off, bytes;
    explicit LpBwdShapes(const LpShapes& s) {
        const int64_t a = std::max({s.conv_elems[4], s.conv_elems[2], s.conv_elems[1], s.conv_elems[0]});
        const int64_t b = std::max({s.conv_elems[3], s.pool_elems[1], s.pool_elems[0]});
        a_off = 0;
        b_off = ((size_t)a * 4 + 255) & ~(size_t)255;
        bytes = b_off + (((size_t)b * 4 + 255) & ~(size_t)255) + 256;   // + alignment of the base
    }
};

template <int L>
int launch_dgrad(const LpConvArgs& a, cudaStream_t stream) {
    S3G_CUDA(cudaFuncSetAttribute(lpips_dgrad_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, lp_smem_bytes(LpAlex::bn(L))),
             "lpips dgrad smem attribute");
    const dim3 grid((unsigned)div_up64(a.M, LP_BM), LpAlex::cin(L) / LpAlex::bn(L));
    lpips_dgrad_kernel<L><<<grid, LP_THREADS, lp_smem_bytes(LpAlex::bn(L)), stream>>>(a);
    S3G_CUDA(cudaGetLastError(), "lpips dgrad launch");
    return S3G_OK;
}

template <int C>
int launch_tap_bwd(int P, int layer, double pixels, int wx, int wy, int accumulate, const float* f, const float* lin,
                   const double* gout, float* g, cudaStream_t stream) {
    const int64_t blocks = div_up64(P, LP_TAP_WARPS * LP_TAP_PIX);
    lpips_tap_bwd_kernel<C><<<(unsigned)blocks, 32 * LP_TAP_WARPS, 0, stream>>>(P, layer, pixels, wx, wy, accumulate, f,
                                                                               lin, gout, g);
    S3G_CUDA(cudaGetLastError(), "lpips tap backward launch");
    return S3G_OK;
}

int tap_bwd(int l, int P, double pixels, int wx, int wy, int accumulate, const float* f, const float* lin,
            const double* gout, float* g, cudaStream_t stream) {
    switch (LpAlex::cout(l)) {
        case 64: return launch_tap_bwd<64>(P, l, pixels, wx, wy, accumulate, f, lin, gout, g, stream);
        case 192: return launch_tap_bwd<192>(P, l, pixels, wx, wy, accumulate, f, lin, gout, g, stream);
        case 384: return launch_tap_bwd<384>(P, l, pixels, wx, wy, accumulate, f, lin, gout, g, stream);
        default: return launch_tap_bwd<256>(P, l, pixels, wx, wy, accumulate, f, lin, gout, g, stream);
    }
}

bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

template <int L>
int launch_conv(const LpConvArgs& a, cudaStream_t stream) {
    S3G_CUDA(cudaFuncSetAttribute(lpips_conv_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, lp_smem_bytes(LpAlex::bn(L))),
             "lpips conv smem attribute");
    const dim3 grid((unsigned)div_up64(a.M, LP_BM), LpAlex::cout(L) / LpAlex::bn(L));
    lpips_conv_kernel<L><<<grid, LP_THREADS, lp_smem_bytes(LpAlex::bn(L)), stream>>>(a);
    S3G_CUDA(cudaGetLastError(), "lpips conv launch");
    return S3G_OK;
}

template <int C>
int launch_tap(int P, int64_t blocks, const float* f, const float* lin, double* partial, cudaStream_t stream) {
    lpips_tap_kernel<C><<<(unsigned)blocks, 32 * LP_TAP_WARPS, 0, stream>>>(P, f, lin, partial);
    S3G_CUDA(cudaGetLastError(), "lpips tap launch");
    return S3G_OK;
}

// the tap of a feature map with C channels (AlexNet's and VGG16's tap widths)
int tap_fwd(int C, int P, int64_t blocks, const float* f, const float* lin, double* partial, cudaStream_t stream) {
    switch (C) {
        case 64: return launch_tap<64>(P, blocks, f, lin, partial, stream);
        case 128: return launch_tap<128>(P, blocks, f, lin, partial, stream);
        case 192: return launch_tap<192>(P, blocks, f, lin, partial, stream);
        case 256: return launch_tap<256>(P, blocks, f, lin, partial, stream);
        case 384: return launch_tap<384>(P, blocks, f, lin, partial, stream);
        case 512: return launch_tap<512>(P, blocks, f, lin, partial, stream);
        default: return fail(S3G_ERR_ARG, "lpips tap: unsupported channel count");
    }
}

// ---- VGG16 (lpips_vgg.cuh) -----------------------------------------------------------------------------------------
constexpr int VGG_MIN_SIDE = 16;   // below it the fourth max-pool's output is empty

// float offsets inside the VGG prepared buffer: the thirteen convolutions' weight tiles, every bias, the five lin weights
struct LpVggPrepared {
    size_t tiles[LpVgg::CONVS], bias[LpVgg::CONVS], lin[LP_LAYERS], total;
    LpVggPrepared() {
        size_t o = 0;
        for (int l = 0; l < LpVgg::CONVS; ++l) { tiles[l] = o; o += (size_t)lp_prep_floats<LpVgg>(l); }
        for (int l = 0; l < LpVgg::CONVS; ++l) { bias[l] = o; o += LpVgg::cout(l); }
        for (int g = 0; g < LP_LAYERS; ++g) { lin[g] = o; o += LpVgg::cout(LpVgg::last(g)); }
        total = o;
    }
};

// One call's workspace: two activation buffers the layers ping-pong between, each as large as a group-1 convolution's
// output (the largest tensor: every max-pool quarters the pixels and the channels at most double), and the taps'
// partial sums.  Group g works on an (H >> g) x (W >> g) grid.
struct LpVggShapes {
    int64_t h[LP_LAYERS], w[LP_LAYERS], act_elems, tap_blocks[LP_LAYERS];
    size_t act_off[2], part_off[LP_LAYERS], bytes;
    LpVggShapes(int N, int H, int W) {
        size_t o = 0;
        auto take = [&](int64_t bytes_) { const size_t at = o; o += ((size_t)bytes_ + 255) & ~(size_t)255; return at; };
        act_elems = 2 * (int64_t)N * H * W * LpVgg::cout(0);
        for (int i = 0; i < 2; ++i) act_off[i] = take(act_elems * 4);
        for (int g = 0; g < LP_LAYERS; ++g) {
            h[g] = H >> g; w[g] = W >> g;
            tap_blocks[g] = div_up64((int64_t)N * h[g] * w[g], LP_TAP_WARPS * LP_TAP_PIX);
            part_off[g] = take(tap_blocks[g] * 8);
        }
        bytes = o + 256;   // + alignment of the base
    }
};

bool vgg_args_ok(int N, int H, int W) {
    return N >= 1 && H >= VGG_MIN_SIDE && W >= VGG_MIN_SIDE && 2 * (int64_t)N * H * W * LpVgg::cout(0) < INT32_MAX;
}

template <int L>
int launch_vgg_conv(const LpConvArgs& a, cudaStream_t stream) {
    constexpr int BN = LpVgg::bn(L);
    S3G_CUDA(cudaFuncSetAttribute(lpips_vgg_conv_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, lp_smem_bytes(BN)),
             "lpips vgg conv smem attribute");
    const dim3 grid((unsigned)div_up64(a.M, LP_BM), LpVgg::cout(L) / BN);
    lpips_vgg_conv_kernel<L><<<grid, LP_THREADS, lp_smem_bytes(BN), stream>>>(a);
    S3G_CUDA(cudaGetLastError(), "lpips vgg conv launch");
    return S3G_OK;
}

// convolutions of one shape share a kernel: 5, 6 are 256 -> 256, 8..12 are 512 -> 512
int vgg_conv(int l, const LpConvArgs& a, cudaStream_t stream) {
    switch (l) {
        case 0: return launch_vgg_conv<0>(a, stream);
        case 1: return launch_vgg_conv<1>(a, stream);
        case 2: return launch_vgg_conv<2>(a, stream);
        case 3: return launch_vgg_conv<3>(a, stream);
        case 4: return launch_vgg_conv<4>(a, stream);
        case 5: case 6: return launch_vgg_conv<5>(a, stream);
        case 7: return launch_vgg_conv<7>(a, stream);
        default: return launch_vgg_conv<8>(a, stream);
    }
}
}  // namespace

extern "C" {

size_t s3g_lpips_alex_prepared_bytes(void) { return LpPrepared().total * sizeof(float); }

int s3g_lpips_alex_prepare(const s3g_lpips_alex_weights* wts, void* prepared, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (!wts || !prepared) return fail(S3G_ERR_ARG, "lpips_alex_prepare: null weights/prepared");
    for (int l = 0; l < LP_LAYERS; ++l)
        if (!wts->conv_w[l] || !wts->conv_b[l] || !wts->lin_w[l])
            return fail(S3G_ERR_ARG, "lpips_alex_prepare: null weight pointer");
    if ((reinterpret_cast<uintptr_t>(prepared) & 15) != 0)
        return fail(S3G_ERR_ARG, "lpips_alex_prepare: prepared must be 16-byte aligned");
    const LpPrepared lay;
    float* dst = static_cast<float*>(prepared);
    LpPrepArgs<LpAlex> p;
    for (int l = 0; l < LP_LAYERS; ++l) {
        p.w[l] = wts->conv_w[l];
        p.dst[l] = dst + lay.tiles[l];
        S3G_CUDA(cudaMemcpyAsync(dst + lay.bias[l], wts->conv_b[l], LpAlex::cout(l) * sizeof(float), cudaMemcpyDeviceToDevice,
                                 stream), "lpips_alex_prepare bias copy");
        S3G_CUDA(cudaMemcpyAsync(dst + lay.lin[l], wts->lin_w[l], LpAlex::cout(l) * sizeof(float), cudaMemcpyDeviceToDevice,
                                 stream), "lpips_alex_prepare lin copy");
    }
    lpips_prep_kernel<LpAlex><<<dim3(256, LP_LAYERS), 256, 0, stream>>>(p);
    S3G_CUDA(cudaGetLastError(), "lpips_prep launch");
    return S3G_OK;
}

size_t s3g_lpips_alex_workspace_bytes(int N, int H, int W) {
    if (!args_ok(N, H, W)) return 0;
    return LpShapes(N, H, W).bytes;
}

int s3g_lpips_alex(int N, int H, int W, const float* x, const float* y, const void* prepared, double* out,
                   void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (N < 1) return fail(S3G_ERR_ARG, "lpips_alex: N >= 1 images expected");
    if (H < 31 || W < 31) return fail(S3G_ERR_ARG, "lpips_alex: image sides must be >= 31 (AlexNet's second max-pool)");
    if (!args_ok(N, H, W)) return fail(S3G_ERR_ARG, "lpips_alex: images too large for 32-bit indices");
    if (!x || !y || !prepared || !out || !workspace) return fail(S3G_ERR_ARG, "lpips_alex: null x/y/prepared/out/workspace");
    if ((reinterpret_cast<uintptr_t>(prepared) & 15) != 0) return fail(S3G_ERR_ARG, "lpips_alex: unaligned prepared");
    const LpShapes s(N, H, W);
    const LpPrepared lay;
    const float* wp = static_cast<const float*>(prepared);
    char* base = reinterpret_cast<char*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    auto buf = [&](size_t off) { return reinterpret_cast<float*>(base + off); };

    // conv l reads the pool after conv 1 and 2, the previous conv after that
    const float* in = nullptr;
    int ih = H, iw = W;
    for (int l = 0; l < LP_LAYERS; ++l) {
        LpConvArgs a;
        a.in = in; a.x = x; a.y = y; a.N = N; a.H = ih; a.W = iw;
        a.Ho = (int)s.h[l]; a.Wo = (int)s.w[l];
        a.M = 2 * N * a.Ho * a.Wo;
        a.wprep = wp + lay.tiles[l];
        a.bias = wp + lay.bias[l];
        a.out = buf(s.conv_off[l]);
        int rc = S3G_OK;
        switch (l) {
            case 0: rc = launch_conv<0>(a, stream); break;
            case 1: rc = launch_conv<1>(a, stream); break;
            case 2: rc = launch_conv<2>(a, stream); break;
            case 3: rc = launch_conv<3>(a, stream); break;
            default: rc = launch_conv<4>(a, stream); break;
        }
        if (rc != S3G_OK) return rc;
        in = a.out; ih = a.Ho; iw = a.Wo;
        if (l < 2) {
            const int C4 = LpAlex::cout(l) / 4;
            const int total4 = (int)(s.pool_elems[l] / 4);
            const int grid = (int)std::min<int64_t>(div_up64(total4, 256), (int64_t)device_sm_count() * 16);
            float* po = buf(s.pool_off[l]);
            lpips_maxpool_kernel<<<grid, 256, 0, stream>>>(total4, C4, ih, iw, (int)s.ph[l], (int)s.pw[l],
                                                           reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(po));
            S3G_CUDA(cudaGetLastError(), "lpips maxpool launch");
            in = po; ih = (int)s.ph[l]; iw = (int)s.pw[l];
        }
    }
    LpReduceArgs r;
    for (int l = 0; l < LP_LAYERS; ++l) {
        const int P = (int)(N * s.h[l] * s.w[l]);
        const float* f = buf(s.conv_off[l]);
        const float* lin = wp + lay.lin[l];
        double* part = reinterpret_cast<double*>(base + s.part_off[l]);
        const int rc = tap_fwd(LpAlex::cout(l), P, s.tap_blocks[l], f, lin, part, stream);
        if (rc != S3G_OK) return rc;
        r.partial[l] = part;
        r.blocks[l] = (int)s.tap_blocks[l];
        r.pixels[l] = (double)(s.h[l] * s.w[l]);
    }
    r.out = out;
    lpips_reduce_kernel<<<1, 256, 0, stream>>>(r);
    S3G_CUDA(cudaGetLastError(), "lpips reduce launch");
    return S3G_OK;
}

size_t s3g_lpips_alex_backward_prepared_bytes(void) { return LpPreparedBwd().total * sizeof(float); }

int s3g_lpips_alex_backward_prepare(const s3g_lpips_alex_weights* wts, void* prepared_bwd, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (!wts || !prepared_bwd) return fail(S3G_ERR_ARG, "lpips_alex_backward_prepare: null weights/prepared_bwd");
    for (int l = 0; l < LP_LAYERS; ++l)
        if (!wts->conv_w[l]) return fail(S3G_ERR_ARG, "lpips_alex_backward_prepare: null convolution weight pointer");
    if (!aligned(prepared_bwd, 16))
        return fail(S3G_ERR_ARG, "lpips_alex_backward_prepare: prepared_bwd must be 16-byte aligned");
    const LpPreparedBwd lay;
    float* dst = static_cast<float*>(prepared_bwd);
    S3G_CUDA(cudaMemcpyAsync(dst + lay.w0, wts->conv_w[0], (size_t)LpAlex::cout(0) * lp_k<LpAlex>(0) * sizeof(float),
                             cudaMemcpyDeviceToDevice, stream), "lpips_alex_backward_prepare conv 1 copy");
    LpPrepArgs<LpAlex> p{};
    for (int l = 1; l < LP_LAYERS; ++l) {
        p.w[l] = wts->conv_w[l];
        p.dst[l] = dst + lay.tiles[l];
    }
    lpips_prep_dgrad_kernel<<<dim3(256, LP_LAYERS - 1), 256, 0, stream>>>(p);
    S3G_CUDA(cudaGetLastError(), "lpips_prep_dgrad launch");
    return S3G_OK;
}

size_t s3g_lpips_alex_backward_workspace_bytes(int N, int H, int W) {
    if (!args_ok(N, H, W)) return 0;
    return LpBwdShapes(LpShapes(N, H, W)).bytes;
}

int s3g_lpips_alex_backward(int N, int H, int W, const void* prepared, const void* prepared_bwd,
                            const void* fwd_workspace, const double* grad_out, float* grad_x, float* grad_y,
                            void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (N < 1) return fail(S3G_ERR_ARG, "lpips_alex_backward: N >= 1 images expected");
    if (H < 31 || W < 31) return fail(S3G_ERR_ARG, "lpips_alex_backward: image sides must be >= 31");
    if (!args_ok(N, H, W)) return fail(S3G_ERR_ARG, "lpips_alex_backward: images too large for 32-bit indices");
    if (!prepared || !prepared_bwd || !fwd_workspace || !grad_out || !workspace)
        return fail(S3G_ERR_ARG, "lpips_alex_backward: null prepared/prepared_bwd/fwd_workspace/grad_out/workspace");
    if (!grad_x && !grad_y) return fail(S3G_ERR_ARG, "lpips_alex_backward: neither grad_x nor grad_y requested");
    if (!aligned(prepared, 16) || !aligned(prepared_bwd, 16) || !aligned(grad_out, 8) || !aligned(grad_x, 4) ||
        !aligned(grad_y, 4))
        return fail(S3G_ERR_ARG, "lpips_alex_backward: unaligned prepared/prepared_bwd (16), grad_out (8) or grad (4)");
    const LpShapes s(N, H, W);
    const LpBwdShapes bs(s);
    const LpPrepared lay;
    const LpPreparedBwd blay;
    const float* wp = static_cast<const float*>(prepared);
    const float* wb = static_cast<const float*>(prepared_bwd);
    // the forward's layout (s3g_lpips_alex): same base rounding, same offsets
    const char* fbase = reinterpret_cast<const char*>(((uintptr_t)fwd_workspace + 255) & ~(uintptr_t)255);
    auto saved = [&](size_t off) { return reinterpret_cast<const float*>(fbase + off); };
    char* base = reinterpret_cast<char*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    float* ga = reinterpret_cast<float*>(base + bs.a_off);
    float* gb = reinterpret_cast<float*>(base + bs.b_off);

    const int wx = grad_x != nullptr, wy = grad_y != nullptr;
    const int NB = (wx + wy) * N;          // images with a gradient: rows of every buffer below
    const int64_t i0 = wx ? 0 : N;          // ... starting at this image of the forward's 2N
    auto tap = [&](int l, int accumulate, float* g) {
        return tap_bwd(l, (int)(N * s.h[l] * s.w[l]), (double)(s.h[l] * s.w[l]), wx, wy, accumulate,
                       saved(s.conv_off[l]), wp + lay.lin[l], grad_out, g, stream);
    };
    auto dgrad = [&](int l, const float* dy, float* dx) {
        LpConvArgs a{};
        a.in = dy; a.N = NB; a.H = a.Ho = (int)s.h[l]; a.W = a.Wo = (int)s.w[l];
        a.M = NB * a.Ho * a.Wo;
        a.wprep = wb + blay.tiles[l];
        a.out = dx;
        switch (l) {
            case 1: return launch_dgrad<1>(a, stream);
            case 2: return launch_dgrad<2>(a, stream);
            case 3: return launch_dgrad<3>(a, stream);
            default: return launch_dgrad<4>(a, stream);
        }
    };
    // gradient at pool p's output (dout) -> gradient at conv p's output (din), argmaxes from the saved conv output
    auto pool = [&](int p, const float* dout, float* din) {
        const int C4 = LpAlex::cout(p) / 4;
        const int64_t total4 = (int64_t)NB * s.h[p] * s.w[p] * C4;
        const int grid = (int)std::min<int64_t>(div_up64(total4, 256), (int64_t)device_sm_count() * 16);
        const float* in = saved(s.conv_off[p]) + i0 * s.h[p] * s.w[p] * LpAlex::cout(p);
        lpips_maxpool_bwd_kernel<<<grid, 256, 0, stream>>>((int)total4, C4, (int)s.h[p], (int)s.w[p], (int)s.ph[p],
                                                            (int)s.pw[p], reinterpret_cast<const float4*>(in),
                                                            reinterpret_cast<const float4*>(dout),
                                                            reinterpret_cast<float4*>(din));
        S3G_CUDA(cudaGetLastError(), "lpips maxpool backward launch");
        return S3G_OK;
    };
    int rc;
    if ((rc = tap(4, 0, ga)) != S3G_OK) return rc;
    if ((rc = dgrad(4, ga, gb)) != S3G_OK) return rc;
    if ((rc = tap(3, 1, gb)) != S3G_OK) return rc;
    if ((rc = dgrad(3, gb, ga)) != S3G_OK) return rc;
    if ((rc = tap(2, 1, ga)) != S3G_OK) return rc;
    if ((rc = dgrad(2, ga, gb)) != S3G_OK) return rc;
    if ((rc = pool(1, gb, ga)) != S3G_OK) return rc;
    if ((rc = tap(1, 1, ga)) != S3G_OK) return rc;
    if ((rc = dgrad(1, ga, gb)) != S3G_OK) return rc;
    if ((rc = pool(0, gb, ga)) != S3G_OK) return rc;
    if ((rc = tap(0, 1, ga)) != S3G_OK) return rc;

    LpDgrad0Args d{};
    d.dy = ga; d.w = wb + blay.w0;
    d.first = wx ? grad_x : grad_y; d.second = grad_y;
    d.N = N; d.H = H; d.W = W; d.Ho = (int)s.h[0]; d.Wo = (int)s.w[0];
    d.tiles_x = (int)div_up64(div_up64(W, 4), LP_D0_TX);
    d.tiles_y = (int)div_up64(div_up64(H, 4), LP_D0_TY);
    const int64_t blocks = (int64_t)NB * 16 * d.tiles_x * d.tiles_y;
    lpips_dgrad0_kernel<<<(unsigned)blocks, dim3(LP_D0_TX, LP_D0_TY), 0, stream>>>(d);
    S3G_CUDA(cudaGetLastError(), "lpips dgrad0 launch");
    return S3G_OK;
}

size_t s3g_lpips_vgg_prepared_bytes(void) { return LpVggPrepared().total * sizeof(float); }

int s3g_lpips_vgg_prepare(const s3g_lpips_vgg_weights* wts, void* prepared, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (!wts || !prepared) return fail(S3G_ERR_ARG, "lpips_vgg_prepare: null weights/prepared");
    for (int l = 0; l < LpVgg::CONVS; ++l)
        if (!wts->conv_w[l] || !wts->conv_b[l]) return fail(S3G_ERR_ARG, "lpips_vgg_prepare: null weight pointer");
    for (int g = 0; g < LP_LAYERS; ++g)
        if (!wts->lin_w[g]) return fail(S3G_ERR_ARG, "lpips_vgg_prepare: null lin weight pointer");
    if (!aligned(prepared, 16)) return fail(S3G_ERR_ARG, "lpips_vgg_prepare: prepared must be 16-byte aligned");
    const LpVggPrepared lay;
    float* dst = static_cast<float*>(prepared);
    LpPrepArgs<LpVgg> p;
    for (int l = 0; l < LpVgg::CONVS; ++l) {
        p.w[l] = wts->conv_w[l];
        p.dst[l] = dst + lay.tiles[l];
        S3G_CUDA(cudaMemcpyAsync(dst + lay.bias[l], wts->conv_b[l], LpVgg::cout(l) * sizeof(float),
                                 cudaMemcpyDeviceToDevice, stream), "lpips_vgg_prepare bias copy");
    }
    for (int g = 0; g < LP_LAYERS; ++g)
        S3G_CUDA(cudaMemcpyAsync(dst + lay.lin[g], wts->lin_w[g], LpVgg::cout(LpVgg::last(g)) * sizeof(float),
                                 cudaMemcpyDeviceToDevice, stream), "lpips_vgg_prepare lin copy");
    lpips_prep_kernel<LpVgg><<<dim3(256, LpVgg::CONVS), 256, 0, stream>>>(p);
    S3G_CUDA(cudaGetLastError(), "lpips_prep launch");
    return S3G_OK;
}

size_t s3g_lpips_vgg_workspace_bytes(int N, int H, int W) {
    if (!vgg_args_ok(N, H, W)) return 0;
    return LpVggShapes(N, H, W).bytes;
}

int s3g_lpips_vgg(int N, int H, int W, const float* x, const float* y, const void* prepared, double* out,
                  void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (N < 1) return fail(S3G_ERR_ARG, "lpips_vgg: N >= 1 images expected");
    if (H < VGG_MIN_SIDE || W < VGG_MIN_SIDE)
        return fail(S3G_ERR_ARG, "lpips_vgg: image sides must be >= 16 (VGG16's fourth max-pool)");
    if (!vgg_args_ok(N, H, W)) return fail(S3G_ERR_ARG, "lpips_vgg: images too large for 32-bit indices");
    if (!x || !y || !prepared || !out || !workspace) return fail(S3G_ERR_ARG, "lpips_vgg: null x/y/prepared/out/workspace");
    if (!aligned(prepared, 16)) return fail(S3G_ERR_ARG, "lpips_vgg: unaligned prepared");
    const LpVggShapes s(N, H, W);
    const LpVggPrepared lay;
    const float* wp = static_cast<const float*>(prepared);
    char* base = reinterpret_cast<char*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    float* act[2] = {reinterpret_cast<float*>(base + s.act_off[0]), reinterpret_cast<float*>(base + s.act_off[1])};

    // every kernel reads one activation buffer and writes the other
    LpReduceArgs r;
    const float* in = nullptr;
    int o = 0, g = 0;
    for (int l = 0; l < LpVgg::CONVS; ++l) {
        const int gh = (int)s.h[g], gw = (int)s.w[g];
        LpConvArgs a;
        a.in = in; a.x = x; a.y = y; a.N = N; a.H = a.Ho = gh; a.W = a.Wo = gw;
        a.M = 2 * N * gh * gw;
        a.wprep = wp + lay.tiles[l];
        a.bias = wp + lay.bias[l];
        a.out = act[o];
        int rc = vgg_conv(l, a, stream);
        if (rc != S3G_OK) return rc;
        in = a.out; o ^= 1;
        if (l != LpVgg::last(g)) continue;
        const int C = LpVgg::cout(l);
        double* part = reinterpret_cast<double*>(base + s.part_off[g]);
        rc = tap_fwd(C, N * gh * gw, s.tap_blocks[g], in, wp + lay.lin[g], part, stream);
        if (rc != S3G_OK) return rc;
        r.partial[g] = part;
        r.blocks[g] = (int)s.tap_blocks[g];
        r.pixels[g] = (double)(s.h[g] * s.w[g]);
        if (++g == LP_LAYERS) break;
        const int ph = (int)s.h[g], pw = (int)s.w[g];
        const int total4 = 2 * N * ph * pw * (C / 4);
        const int grid = (int)std::min<int64_t>(div_up64(total4, 256), (int64_t)device_sm_count() * 16);
        lpips_maxpool2_kernel<<<grid, 256, 0, stream>>>(total4, C / 4, gh, gw, ph, pw, reinterpret_cast<const float4*>(in),
                                                        reinterpret_cast<float4*>(act[o]));
        S3G_CUDA(cudaGetLastError(), "lpips vgg maxpool launch");
        in = act[o]; o ^= 1;
    }
    r.out = out;
    lpips_reduce_kernel<<<1, 256, 0, stream>>>(r);
    S3G_CUDA(cudaGetLastError(), "lpips reduce launch");
    return S3G_OK;
}

}  // extern "C"
