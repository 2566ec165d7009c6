// api.cu - extern "C" entry points of libs3g_b200.so (see include/s3g_b200.h).
//
// Host orchestration of the forward / backward passes; mirrors the control flow
// of CudaRasterizer::Rasterizer::{markVisible,forward,backward}
// (DGR/cuda_rasterizer/rasterizer_impl.cu:141-153,198-339,343-444) behind a flat
// C ABI.  No torch, no CPU fallback: every path ends in a kernel launch on the
// caller's stream or in an error code.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <string>

#include "api_common.cuh"
#include "binning.cuh"
#include "common.cuh"
#include "composite.cuh"
#include "preprocess.cuh"
#define S3G_SCAN_IMPL
#include "radix_sort.cuh"

using namespace s3g;

namespace {
thread_local std::string g_last_error;

inline int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return s3g::api_fail(code, what, e); }


// debug mode: synchronise + check after every stage (CHECK_CUDA, auxiliary.h:166-173)
#define S3G_STAGE(what)                                                            \
    do {                                                                           \
        cudaError_t e__ = cudaGetLastError();                                      \
        if (e__ == cudaSuccess && debug) e__ = cudaStreamSynchronize(stream);      \
        if (e__ != cudaSuccess) return fail(S3G_ERR_CUDA, what, e__);              \
    } while (0)

// ---- optional per-stage timing -------------------------------------------
constexpr int kMaxStages = 12;
struct StageTimer {
    bool on = false;
    int n[2] = {0, 0};
    cudaEvent_t ev[2][kMaxStages + 1] = {};
    const char* names[2][kMaxStages] = {};
    void mark(int which, cudaStream_t s, const char* name_of_stage_that_starts) {
        if (!on) return;
        int i = n[which];
        if (i > kMaxStages) return;
        if (!ev[which][i]) cudaEventCreate(&ev[which][i]);
        cudaEventRecord(ev[which][i], s);
        if (name_of_stage_that_starts && i < kMaxStages) names[which][i] = name_of_stage_that_starts;
        n[which] = i + 1;
    }
    void begin(int which) { n[which] = 0; }
};
StageTimer g_timer;
#define S3G_MARK(which, name) g_timer.mark(which, stream, name)

// ---- the instance count as the host sees it ---------------------------------
// Two words of mapped pinned memory per (thread, device): the scan kernel's last block stores {count, sequence}
// there (st.volatile + __threadfence_system); the host polls the sequence word.  last_capacity is the binning
// capacity (in instances) this thread requested on that device the last time.
struct HostCount {
    volatile uint64_t* host = nullptr;
    volatile uint64_t* dev = nullptr;
    uint64_t seq = 0;
    int64_t last_capacity = 0;
    int scan_resident_blocks = 0;
};
HostCount* host_count() {
    static thread_local HostCount table[64];
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) return nullptr;
    HostCount* h = &table[d];
    if (!h->host) {
        void* p = nullptr;
        if (cudaHostAlloc(&p, 2 * sizeof(uint64_t), cudaHostAllocMapped) != cudaSuccess) return nullptr;
        void* dp = nullptr;
        if (cudaHostGetDevicePointer(&dp, p, 0) != cudaSuccess) return nullptr;
        h->host = static_cast<volatile uint64_t*>(p);
        h->dev = static_cast<volatile uint64_t*>(dp);
        h->host[0] = 0;
        h->host[1] = 0;
    }
    return h;
}
// Spin until the scan of call `seq` has published its total.  The stream is queried now and then so that a
// faulted or finished-without-publishing stream ends the wait with an error instead of a hang.
int wait_host_count(HostCount* hc, uint64_t seq, cudaStream_t stream, int64_t* out) {
    for (uint64_t spins = 0;; ++spins) {
        if (hc->host[1] == seq) break;
        if ((spins & 0x3fff) == 0x3fff) {
            cudaError_t q = cudaStreamQuery(stream);
            if (q != cudaSuccess && q != cudaErrorNotReady) return fail(S3G_ERR_CUDA, "num_rendered wait", q);
            if (q == cudaSuccess && hc->host[1] != seq)
                return fail(S3G_ERR_STATE, "num_rendered wait: stream drained without publishing the count");
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    __sync_synchronize();
    *out = (int64_t)hc->host[0];
    return S3G_OK;
}

// number of key bits that cover every tile id (getHigherMsb, rasterizer_impl.cu:35-50)
int tile_key_bits(uint32_t tiles) {
    int b = 0;
    while (b < 32 && (tiles >> b) != 0) ++b;
    return b < 1 ? 1 : b;
}
}  // namespace
namespace s3g {
int api_fail(int code, const char* what, cudaError_t e) {
    g_last_error = what;
    if (e != cudaSuccess) {
        g_last_error += ": ";
        g_last_error += cudaGetErrorString(e);
    }
    return code;
}
}  // namespace s3g

extern "C" {

int s3g_abi_version(void) { return S3G_ABI_VERSION; }
const char* s3g_last_error(void) { return g_last_error.c_str(); }
const char* s3g_build_arch(void) { return "sm_90a"; }

int s3g_profile_enable(int on) {
    g_timer.on = on != 0;
    return S3G_OK;
}
int s3g_profile_read(int which, float* ms, int capacity) {
    if (which < 0 || which > 1 || !ms) return fail(S3G_ERR_ARG, "profile_read: bad argument");
    int stages = g_timer.n[which] - 1;
    if (stages < 0) stages = 0;
    if (stages > capacity) stages = capacity;
    for (int i = 0; i < stages; ++i) {
        cudaError_t e = cudaEventSynchronize(g_timer.ev[which][i + 1]);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms[i], g_timer.ev[which][i], g_timer.ev[which][i + 1]);
        if (e != cudaSuccess) return fail(S3G_ERR_CUDA, "profile_read", e);
    }
    return stages;
}
const char* s3g_profile_stage_name(int which, int index) {
    if (which < 0 || which > 1 || index < 0 || index >= kMaxStages || !g_timer.names[which][index]) return "";
    return g_timer.names[which][index];
}

size_t s3g_geom_bytes(int64_t P) {
    size_t t = 0;
    GeomState::carve(nullptr, P, &t);
    return t;
}
size_t s3g_binning_bytes(int64_t R) {
    size_t t = 0;
    BinningState::carve(nullptr, R, &t);
    return t;
}
size_t s3g_image_bytes(int width, int height) {
    size_t t = 0;
    ImageState::carve(nullptr, width, height, &t);
    return t;
}
size_t s3g_sort_temp_bytes(int64_t n) {
    // look-back state + the two ping-pong arrays
    size_t m = (size_t)(n > 0 ? n : 1);
    return SortTemp::bytes(n) + 2 * (m * sizeof(uint32_t) + 128);
}

int s3g_state_field(int buffer, const char* name, int64_t P, int64_t R, int width, int height,
                    size_t* offset, size_t* elem_bytes, size_t* count) {
    if (!name || !offset || !elem_bytes || !count) return fail(S3G_ERR_ARG, "state_field: null argument");
    // carve on a fake 128-aligned base so that pointers are offsets + base
    char* base = reinterpret_cast<char*>((uintptr_t)1 << 40);
    auto set = [&](const void* p, size_t eb, size_t n) {
        *offset = (size_t)(reinterpret_cast<const char*>(p) - base);
        *elem_bytes = eb;
        *count = n;
        return S3G_OK;
    };
    const std::string f(name);
    if (buffer == 0) {
        GeomState g = GeomState::carve(base, P);
        if (f == "xyAB") return set(g.xyAB, 16, P);
        if (f == "Cod") return set(g.Cod, 16, P);
        if (f == "rgb") return set(g.rgb, 16, P);
        if (f == "depth_key") return set(g.depth_key, 4, P);
        if (f == "tiles_touched") return set(g.tiles_touched, 4, P);
        if (f == "rect") return set(g.rect, 8, P);
        if (f == "clamped") return set(g.clamped, 1, P);
        if (f == "order") return set(g.order_a, 4, P);
        if (f == "offsets") return set(g.offsets, 4, P);
        if (f == "grad_rec") return set(g.grad_rec, 4, (size_t)P * GRAD_REC);
    } else if (buffer == 1) {
        BinningState b = BinningState::carve(base, R);
        if (f == "point_list") return set(b.point_list, 4, R);   // first field: independent of the capacity
    } else if (buffer == 2) {
        ImageState s = ImageState::carve(base, width, height);
        TileGrid tg = tile_grid(width, height);
        if (f == "final_T") return set(s.final_T, 4, (size_t)width * height);
        if (f == "n_contrib") return set(s.n_contrib, 4, (size_t)width * height);
        if (f == "ranges") return set(s.ranges, 8, (size_t)tg.count());
    }
    return fail(S3G_ERR_ARG, "state_field: unknown buffer/field");
}

int s3g_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "mark_visible: P < 0");
    if (P == 0) return S3G_OK;
    if (!means3D || !viewmatrix || !projmatrix || !present)
        return fail(S3G_ERR_ARG, "mark_visible: null pointer");
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, viewmatrix, projmatrix,
                                                             present);
    S3G_CUDA(cudaGetLastError(), "mark_visible launch");
    return S3G_OK;
}

int s3g_sort_pairs_u32(int64_t n, uint32_t* keys_in, uint32_t* vals_in, uint32_t* keys_out,
                       uint32_t* vals_out, int begin_bit, int end_bit, void* temp, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (n < 0 || n >= (1ll << 30)) return fail(S3G_ERR_ARG, "sort: n out of range");
    if (begin_bit < 0 || end_bit > 32 || end_bit <= begin_bit)
        return fail(S3G_ERR_ARG, "sort: bad bit range");
    if (n == 0) return S3G_OK;
    // scratch ping-pong lives in temp after the SortTemp block
    Carver c(static_cast<char*>(temp));
    SortTemp st = SortTemp::carve(c, n);
    uint32_t* kt = c.take<uint32_t>((size_t)n);
    uint32_t* vt = c.take<uint32_t>((size_t)n);
    S3G_CUDA(radix_sort_pairs((uint32_t)n, keys_in, vals_in, kt, vt, keys_out, vals_out, begin_bit,
                              end_bit, st, stream),
             "radix sort");
    return S3G_OK;
}

}  // extern "C"

namespace {
int64_t forward_impl(s3g_alloc_fn geom_alloc, void* geom_user, s3g_alloc_fn binning_alloc,
                              void* binning_user, s3g_alloc_fn image_alloc, void* image_user, int P,
                              int D, int M, const float* background, int width, int height,
                              const float* means3D, const float* shs, const float* colors_precomp,
                              const float* opacities, const float* scales, float scale_modifier,
                              const float* rotations, const float* cov3D_precomp,
                              const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                              float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                              float* out_depth, int* radii, int debug, void* stream_,
                              const float* colors_aux, float* out_aux, const uint8_t* group = nullptr,
                              float* out_color_d = nullptr, float* out_depth_d = nullptr,
                              float* out_color_s = nullptr, float* out_depth_s = nullptr) {
    (void)prefiltered;   // the reference only uses it for a device-side trap (auxiliary.h:156-160)
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0 || width <= 0 || height <= 0) return fail(S3G_ERR_ARG, "forward: bad sizes");
    if (!geom_alloc || !binning_alloc || !image_alloc) return fail(S3G_ERR_ARG, "forward: null allocator");
    if (!out_color || !out_depth || !background) return fail(S3G_ERR_ARG, "forward: null output/background");
    const size_t HW = (size_t)width * height;
    if ((colors_aux != nullptr) != (out_aux != nullptr))
        return fail(S3G_ERR_ARG, "forward: colors_aux and out_color_aux go together");
    const bool split = out_color_d != nullptr;
    if (split && colors_aux) return fail(S3G_ERR_ARG, "forward: the split and aux forwards do not combine");
    if (P == 0) {   // rasterize_points.cu:82: outputs stay zero-filled
        if (split) {
            S3G_CUDA(cudaMemsetAsync(out_color_d, 0, 3 * HW * sizeof(float), stream), "memset color_d");
            S3G_CUDA(cudaMemsetAsync(out_depth_d, 0, HW * sizeof(float), stream), "memset depth_d");
            S3G_CUDA(cudaMemsetAsync(out_color_s, 0, 3 * HW * sizeof(float), stream), "memset color_s");
            S3G_CUDA(cudaMemsetAsync(out_depth_s, 0, HW * sizeof(float), stream), "memset depth_s");
        }
        if (out_aux) S3G_CUDA(cudaMemsetAsync(out_aux, 0, 3 * HW * sizeof(float), stream), "memset aux");
        S3G_CUDA(cudaMemsetAsync(out_color, 0, 3 * HW * sizeof(float), stream), "memset color");
        S3G_CUDA(cudaMemsetAsync(out_depth, 0, HW * sizeof(float), stream), "memset depth");
        return 0;
    }
    if (!means3D || !opacities || !viewmatrix || !projmatrix)
        return fail(S3G_ERR_ARG, "forward: null input");
    if (!colors_precomp && !shs)
        return fail(S3G_ERR_ARG, "forward: need SHs or precomputed colours");
    if (!colors_precomp && !cam_pos) return fail(S3G_ERR_ARG, "forward: SH path needs cam_pos");
    if (!cov3D_precomp && (!scales || !rotations))
        return fail(S3G_ERR_ARG, "forward: need scales+rotations or precomputed cov3D");
    if (!colors_precomp && (D < 0 || D > 3 || M < (D + 1) * (D + 1)))
        return fail(S3G_ERR_ARG, "forward: SH degree/coefficient count mismatch");
    if ((int64_t)P >= (1ll << 30)) return fail(S3G_ERR_ARG, "forward: P too large");

    const TileGrid tg = tile_grid(width, height);
    if (tg.x > 65535 || tg.y > 65535) return fail(S3G_ERR_ARG, "forward: image too large");

    char* gptr = geom_alloc(geom_user, s3g_geom_bytes(P));
    if (!gptr) return fail(S3G_ERR_ALLOC, "forward: geometry allocator returned NULL");
    GeomState geom = GeomState::carve(gptr, P);
    char* iptr = image_alloc(image_user, s3g_image_bytes(width, height));
    if (!iptr) return fail(S3G_ERR_ALLOC, "forward: image allocator returned NULL");
    ImageState img = ImageState::carve(iptr, width, height);
    if (!radii) radii = geom.internal_radii;

    // ---- per-Gaussian preprocess -----------------------------------------
    PreFwdArgs pa;
    pa.P = P; pa.D = D; pa.M = M;
    pa.means3D = means3D; pa.scales = scales; pa.scale_modifier = scale_modifier;
    pa.rotations = rotations; pa.opacities = opacities; pa.shs = shs;
    pa.cov3D_precomp = cov3D_precomp; pa.colors_precomp = colors_precomp;
    pa.view = viewmatrix; pa.proj = projmatrix; pa.campos = cam_pos;
    pa.W = width; pa.H = height;
    pa.tan_fovx = tan_fovx; pa.tan_fovy = tan_fovy;
    pa.focal_y = height / (2.0f * tan_fovy);   // rasterizer_impl.cu:223-224
    pa.focal_x = width / (2.0f * tan_fovx);
    pa.radii = radii; pa.xyAB = geom.xyAB; pa.Cod = geom.Cod; pa.rgb = geom.rgb;
    pa.colors_aux = colors_aux; pa.aux = geom.aux;
    pa.depth_key = geom.depth_key; pa.tiles_touched = geom.tiles_touched; pa.rect = geom.rect;
    pa.clamped = geom.clamped; pa.order = geom.order_a;
    pa.grid_x = tg.x; pa.grid_y = tg.y;
    // scan_misc[4]: dynamic-Gaussian count of a split forward (zeroed with the scan state below)
    pa.group = split ? group : nullptr;
    pa.group_count = split ? geom.scan_misc + 4 : nullptr;
    g_timer.begin(0);
    // one memset for everything the chained scan and the depth sort expect zeroed (look-back words, tickets,
    // digit histograms)
    S3G_CUDA(cudaMemsetAsync(geom.scan_status, 0, geom.zero_bytes, stream), "memset scan/sort state");
    S3G_MARK(0, "preprocess_forward");
    {
        const bool use_sh = colors_precomp == nullptr;
        const size_t smem = use_sh ? (size_t)(PRE_THREADS / 32) * 32 * row_stride(3 * M) * sizeof(float) : 0;
        if (smem > 200 * 1024) return fail(S3G_ERR_ARG, "forward: too many SH coefficients");
        const int grid = (P + PRE_THREADS - 1) / PRE_THREADS;
        if (use_sh && M == 16) {
            preprocess_forward_kernel<16><<<grid, PRE_THREADS, smem, stream>>>(pa);
        } else {
            if (smem > 48 * 1024)
                S3G_CUDA(cudaFuncSetAttribute(preprocess_forward_kernel<0>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                         "smem attribute");
            preprocess_forward_kernel<0><<<grid, PRE_THREADS, smem, stream>>>(pa);
        }
    }
    S3G_STAGE("preprocess_forward");
    S3G_MARK(0, "depth_sort");

    // ---- depth digits of the LSD sort, over Gaussians --------------------
    S3G_CUDA(radix_sort_pairs((uint32_t)P, geom.depth_key, geom.order_a, geom.key_b, geom.order_b,
                              nullptr, geom.order_a, 0, 32, geom.sort, stream, nullptr, /*hist_ready=*/false,
                              /*prepared=*/true),
             "depth sort");
    S3G_STAGE("depth sort");

    S3G_MARK(0, "scan");
    // ---- offsets in depth order + total ----------------------------------
    // The total (num_rendered, rasterizer_impl.cu:281-282) stays on the device for the binning kernels and is
    // ALSO stored by the scan's last block into mapped pinned memory: the host reads it without a copy, an event or
    // a stream synchronisation, after the rest of the forward has been enqueued.
    HostCount* hc = host_count();
    if (!hc) return fail(S3G_ERR_CUDA, "forward: pinned count buffer");
    const uint64_t seq = ++hc->seq;
    {
        const uint32_t nblk = (uint32_t)div_up64(P, SCAN_TILE);
        if (hc->scan_resident_blocks == 0) {        // once per (thread, device): how many scan blocks fit at the same time
            int per_sm = 0, sms = 0, dev = 0;
            S3G_CUDA(cudaGetDevice(&dev), "cudaGetDevice");
            S3G_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev), "SM count");
            S3G_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, scan_tiles_kernel, SCAN_THREADS, 0), "occupancy");
            hc->scan_resident_blocks = std::max(1, per_sm * sms);
        }
        // (a concurrent kernel on another stream can only delay residency: its slots free up when it ends, and a
        //  grid that fits is never waiting on a block that cannot eventually be placed)
        const int use_tickets = (int64_t)nblk > hc->scan_resident_blocks ? 1 : 0;
        scan_tiles_kernel<<<nblk, SCAN_THREADS, 0, stream>>>(geom.order_a, geom.tiles_touched,
                                                             (uint32_t)P, geom.offsets,
                                                             geom.scan_status, geom.scan_misc, hc->dev, seq,
                                                             use_tickets);
        S3G_STAGE("scan");
    }
    const uint32_t* n_dev = geom.scan_misc + 2;     // low word of the u64 total (checked < 2^30 below)

    // Capacity of the binning arena: what this thread asked for last time (the arena only grows).  The first call
    // has nothing to go by and waits for the count; later calls enqueue everything against the remembered capacity
    // and verify afterwards - the GPU never waits for the host.
    int64_t cap = hc->last_capacity;
    int64_t R = -1;
    if (cap <= 0) {
        int rc = wait_host_count(hc, seq, stream, &R);
        if (rc != S3G_OK) return rc;
        if (R >= (1ll << 30)) return fail(S3G_ERR_ARG, "forward: more than 2^30 tile instances");
        cap = R + R / 8 + 1;
    }
    const uint32_t n_tiles = (uint32_t)tg.count();
    const int tile_bits = tile_key_bits(n_tiles);
    for (int attempt = 0;; ++attempt) {
        char* bptr = binning_alloc(binning_user, s3g_binning_bytes(cap));
        if (!bptr) return fail(S3G_ERR_ALLOC, "forward: binning allocator returned NULL");
        hc->last_capacity = cap;
        BinningState bin = BinningState::carve(bptr, cap);

        S3G_MARK(0, "emit");
        S3G_CUDA(cudaMemsetAsync(img.tile_hist, 0, (size_t)n_tiles * sizeof(uint32_t), stream), "memset tile_hist");
        S3G_CUDA(radix_sort_prepare(bin.sort, stream), "memset tile sort state");
        {
            const size_t hist_smem = (size_t)n_tiles * sizeof(uint32_t);
            const int blocks_needed = (P + 255) / 256;
            if (hist_smem <= 64 * 1024) {
                if (hist_smem > 48 * 1024)
                    S3G_CUDA(cudaFuncSetAttribute(emit_instances_kernel<true>,
                                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hist_smem),
                             "emit smem attribute");
                // two 512-thread blocks per SM: the private histogram is zeroed and flushed once per block
                const int grid = std::min((P + 511) / 512, device_sm_count() * 2);
                emit_instances_kernel<true><<<grid, 512, hist_smem, stream>>>(
                    (uint32_t)P, geom.order_a, geom.offsets, geom.tiles_touched, geom.rect, tg.x, n_tiles,
                    (uint32_t)cap, bin.tile_a, bin.idx_a, img.tile_hist);
            } else {
                emit_instances_kernel<false><<<blocks_needed, 256, 0, stream>>>(
                    (uint32_t)P, geom.order_a, geom.offsets, geom.tiles_touched, geom.rect, tg.x, n_tiles,
                    (uint32_t)cap, bin.tile_a, bin.idx_a, img.tile_hist);
            }
        }
        S3G_STAGE("emit");
        S3G_MARK(0, "tile_offsets");
        {
            const int npass = (tile_bits + RADIX_BITS - 1) / RADIX_BITS;
            tile_offsets_kernel<<<1, 1024, 0, stream>>>(n_tiles, img.tile_hist, img.ranges, npass, tile_bits,
                                                        bin.sort.hist, n_dev, (uint32_t)cap);
        }
        S3G_STAGE("tile offsets");
        S3G_MARK(0, "tile_sort");
        S3G_CUDA(radix_sort_pairs((uint32_t)cap, bin.tile_a, bin.idx_a, bin.tile_b, bin.idx_b, nullptr,
                                  bin.point_list, 0, tile_bits, bin.sort, stream, n_dev, /*hist_ready=*/true),
                 "tile sort");
        S3G_STAGE("tile sort");

        S3G_MARK(0, "render_forward");
        RenderFwdArgs ra;
        ra.ranges = img.ranges; ra.point_list = bin.point_list; ra.W = width; ra.H = height;
        ra.xyAB = geom.xyAB; ra.Cod = geom.Cod; ra.rgb = geom.rgb; ra.bg = background;
        ra.final_T = img.final_T; ra.n_contrib = img.n_contrib;
        ra.out_color = out_color; ra.out_depth = out_depth;
        ra.aux = geom.aux; ra.out_aux = out_aux;
        if (split) {
            RenderSplitArgs sa;
            sa.f = ra;
            sa.out_color_d = out_color_d; sa.out_depth_d = out_depth_d;
            sa.out_color_s = out_color_s; sa.out_depth_s = out_depth_s;
            sa.group_count = geom.scan_misc + 4; sa.P = (uint32_t)P;
            render_forward_split_kernel<<<dim3(tg.x, tg.y), TILE_PIX, 0, stream>>>(sa);
        } else if (colors_aux) render_forward_kernel<true><<<dim3(tg.x, tg.y), TILE_PIX, 0, stream>>>(ra);
        else render_forward_kernel<false><<<dim3(tg.x, tg.y), TILE_PIX, 0, stream>>>(ra);
        S3G_STAGE("render_forward");
        S3G_MARK(0, nullptr);

        if (R < 0) {
            int rc = wait_host_count(hc, seq, stream, &R);
            if (rc != S3G_OK) return rc;
            if (R >= (1ll << 30)) return fail(S3G_ERR_ARG, "forward: more than 2^30 tile instances");
        }
        if (R <= cap) break;
        // the count outgrew the remembered capacity: every write above was clamped to `cap`, nothing is lost
        // but this attempt's tail; grow the arena and run the tail again
        if (attempt > 0) return fail(S3G_ERR_STATE, "forward: binning capacity still too small after growing");
        cap = R + R / 8 + 1;
        g_timer.begin(0);   // stage timers describe the attempt that counts
        S3G_MARK(0, "retry");
    }
    return R;
}

int backward_impl(int P, int D, int M, int64_t R, const float* background, int width,
                           int height, const float* means3D, const float* shs,
                           const float* colors_precomp, const float* scales, float scale_modifier,
                           const float* rotations, const float* cov3D_precomp,
                           const float* viewmatrix, const float* projmatrix, const float* campos,
                           float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                           char* binning_buffer, char* image_buffer, const float* dL_dpix,
                           const float* dL_dpix_depth, float* dL_dmean2D, float* dL_dconic,
                           float* dL_dopacity, float* dL_dcolor, float* dL_ddepth, float* dL_dmean3D,
                           float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                           int debug, void* stream_, const float* dL_dpix_aux, float* dL_dcolor_aux,
                           const s3g_peer_sink* sink = nullptr) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0 || width <= 0 || height <= 0 || R < 0) return fail(S3G_ERR_ARG, "backward: bad sizes");
    if (P == 0) return S3G_OK;   // rasterize_points.cu:165
    if (!geom_buffer || !image_buffer || (R > 0 && !binning_buffer))
        return fail(S3G_ERR_STATE, "backward: missing state buffer");
    if (!means3D || !viewmatrix || !projmatrix || !background || !dL_dpix || !dL_dpix_depth)
        return fail(S3G_ERR_ARG, "backward: null input");
    if (!sink && (!dL_dmean2D || !dL_dopacity || !dL_dcolor || !dL_dmean3D || !dL_dcov3D || !dL_dscale || !dL_drot))
        return fail(S3G_ERR_ARG, "backward: null gradient output");
    if (sink) {
        if (!dL_dmean2D || !dL_dcolor) return fail(S3G_ERR_ARG, "backward_dp: dL_dmean2D / dL_dcolor stay local and must be given");
        if (cov3D_precomp) return fail(S3G_ERR_ARG, "backward_dp: precomputed 3-D covariances are not exchanged");
        if (sink->world < 2 || sink->world > 16 || sink->rank < 0 || sink->rank >= sink->world || sink->chunk <= 0 ||
            (sink->chunk & 3) || sink->off_means3D < 0 || sink->off_opacities < 0 || sink->off_scales < 0 ||
            sink->off_rotations < 0 || (colors_precomp == nullptr && (sink->off_shs < 0 || (sink->off_shs & 3))))
            return fail(S3G_ERR_ARG, "backward_dp: bad peer sink (world, rank, chunk % 4, offsets, off_shs % 4)");
        for (int p = 0; p < sink->world; ++p)
            if (!sink->stage[p]) return fail(S3G_ERR_ARG, "backward_dp: null staging pointer");
    }
    if ((dL_dpix_aux != nullptr) != (dL_dcolor_aux != nullptr))
        return fail(S3G_ERR_ARG, "backward: dL_dpix_aux and dL_dcolor_aux go together");
    const bool use_aux = dL_dpix_aux != nullptr;
    const bool use_sh = (colors_precomp == nullptr);
    if (use_sh && (!shs || (!dL_dsh && !sink) || !campos)) return fail(S3G_ERR_ARG, "backward: SH path needs shs, dL_dsh, campos");
    if (!cov3D_precomp && (!scales || !rotations))
        return fail(S3G_ERR_ARG, "backward: need scales+rotations or precomputed cov3D");

    GeomState geom = GeomState::carve(geom_buffer, P);
    BinningState bin = BinningState::carve(binning_buffer, R);
    ImageState img = ImageState::carve(image_buffer, width, height);
    if (!radii) radii = geom.internal_radii;
    const TileGrid tg = tile_grid(width, height);

    g_timer.begin(1);
    S3G_MARK(1, "zero_grad_rec");
    S3G_CUDA(cudaMemsetAsync(geom.grad_rec, 0, (size_t)P * GRAD_REC * sizeof(float), stream),
             "memset grad_rec");
    S3G_MARK(1, "render_backward");
    if (R > 0) {
        RenderBwdArgs ra;
        ra.ranges = img.ranges; ra.point_list = bin.point_list; ra.W = width; ra.H = height;
        ra.bg = background; ra.xyAB = geom.xyAB; ra.Cod = geom.Cod; ra.rgb = geom.rgb;
        ra.final_T = img.final_T; ra.n_contrib = img.n_contrib;
        ra.dL_dpix = dL_dpix; ra.dL_dpix_depth = dL_dpix_depth; ra.grad_rec = geom.grad_rec;
        ra.aux = geom.aux; ra.dL_dpix_aux = dL_dpix_aux;
        // > 48 KB of dynamic shared memory needs the opt-in, once per device
        static unsigned long long attr_done = 0;
        int devid = 0;
        S3G_CUDA(cudaGetDevice(&devid), "cudaGetDevice");
        if (devid >= 64 || !((attr_done >> devid) & 1ull)) {
            S3G_CUDA(cudaFuncSetAttribute(render_backward_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)sizeof(RenderBwdSmem<false>)),
                     "render_backward smem attribute");
            S3G_CUDA(cudaFuncSetAttribute(render_backward_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)sizeof(RenderBwdSmem<true>)),
                     "render_backward smem attribute");
            if (devid < 64) attr_done |= 1ull << devid;
        }
        if (use_aux)
            render_backward_kernel<true><<<dim3(tg.x, tg.y), TILE_PIX, sizeof(RenderBwdSmem<true>), stream>>>(ra);
        else
            render_backward_kernel<false><<<dim3(tg.x, tg.y), TILE_PIX, sizeof(RenderBwdSmem<false>), stream>>>(ra);
        S3G_STAGE("render_backward");
    }

    S3G_MARK(1, "preprocess_backward");
    PreBwdArgs pb;
    pb.P = P; pb.D = D; pb.M = use_sh ? M : 0;
    pb.means3D = means3D; pb.radii = radii;
    pb.shs = use_sh ? shs : nullptr;   // backward.cu:406
    pb.clamped = geom.clamped;
    pb.scales = cov3D_precomp ? nullptr : scales;   // backward.cu:410 (the reference keys on scales)
    pb.rotations = rotations; pb.scale_modifier = scale_modifier;
    pb.cov3D_precomp = cov3D_precomp;
    pb.view = viewmatrix; pb.proj = projmatrix; pb.campos = campos;
    pb.focal_y = height / (2.0f * tan_fovy);
    pb.focal_x = width / (2.0f * tan_fovx);
    pb.tan_fovx = tan_fovx; pb.tan_fovy = tan_fovy;
    pb.grad_rec = geom.grad_rec;
    pb.dL_dmean2D = dL_dmean2D; pb.dL_dconic = dL_dconic; pb.dL_dopacity = dL_dopacity;
    pb.dL_dcolor = dL_dcolor; pb.dL_dcolor_aux = dL_dcolor_aux; pb.dL_ddepth = dL_ddepth; pb.dL_dmean3D = dL_dmean3D;
    pb.dL_dcov3D = dL_dcov3D; pb.dL_dsh = use_sh ? dL_dsh : nullptr;
    pb.dL_dscale = dL_dscale; pb.dL_drot = dL_drot;
    if (sink) {
        for (int p = 0; p < 16; ++p) pb.sink.stage[p] = p < sink->world ? static_cast<float*>(sink->stage[p]) : nullptr;
        pb.sink.world = sink->world; pb.sink.rank = sink->rank; pb.sink.chunk = sink->chunk;
        pb.sink.off_mean3D = sink->off_means3D; pb.sink.off_sh = sink->off_shs; pb.sink.off_opacity = sink->off_opacities;
        pb.sink.off_scale = sink->off_scales; pb.sink.off_rot = sink->off_rotations;
    }
    {
        const size_t smem = use_sh ? (size_t)(PRE_THREADS / 32) * 32 * row_stride(3 * M) * sizeof(float) : 0;
        if (smem > 200 * 1024) return fail(S3G_ERR_ARG, "backward: too many SH coefficients");
        const int grid = (P + PRE_THREADS - 1) / PRE_THREADS;
        if (sink) {
            if (use_sh && M == 16) {
                preprocess_backward_kernel<16, true><<<grid, PRE_THREADS, smem, stream>>>(pb);
            } else {
                if (smem > 48 * 1024)
                    S3G_CUDA(cudaFuncSetAttribute(preprocess_backward_kernel<0, true>,
                                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                             "smem attribute");
                preprocess_backward_kernel<0, true><<<grid, PRE_THREADS, smem, stream>>>(pb);
            }
        } else if (use_sh && M == 16) {
            preprocess_backward_kernel<16><<<grid, PRE_THREADS, smem, stream>>>(pb);
        } else {
            if (smem > 48 * 1024)
                S3G_CUDA(cudaFuncSetAttribute(preprocess_backward_kernel<0>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                         "smem attribute");
            preprocess_backward_kernel<0><<<grid, PRE_THREADS, smem, stream>>>(pb);
        }
    }
    S3G_STAGE("preprocess_backward");
    S3G_MARK(1, nullptr);
    return S3G_OK;
}
}  // namespace

extern "C" {

int64_t s3g_rasterize_forward(s3g_alloc_fn geom_alloc, void* geom_user, s3g_alloc_fn binning_alloc,
                              void* binning_user, s3g_alloc_fn image_alloc, void* image_user, int P,
                              int D, int M, const float* background, int width, int height,
                              const float* means3D, const float* shs, const float* colors_precomp,
                              const float* opacities, const float* scales, float scale_modifier,
                              const float* rotations, const float* cov3D_precomp,
                              const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                              float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                              float* out_depth, int* radii, int debug, void* stream) {
    return forward_impl(geom_alloc, geom_user, binning_alloc, binning_user, image_alloc, image_user, P, D, M, background,
                        width, height, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations,
                        cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered, out_color,
                        out_depth, radii, debug, stream, nullptr, nullptr);
}

int64_t s3g_rasterize_forward_aux(s3g_alloc_fn geom_alloc, void* geom_user, s3g_alloc_fn binning_alloc,
                                  void* binning_user, s3g_alloc_fn image_alloc, void* image_user, int P,
                                  int D, int M, const float* background, int width, int height,
                                  const float* means3D, const float* shs, const float* colors_precomp,
                                  const float* opacities, const float* scales, float scale_modifier,
                                  const float* rotations, const float* cov3D_precomp,
                                  const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                  float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                                  float* out_depth, int* radii, int debug, void* stream,
                                  const float* colors_aux, float* out_color_aux) {
    if (!colors_aux || !out_color_aux) return fail(S3G_ERR_ARG, "forward_aux: null aux colours / aux image");
    return forward_impl(geom_alloc, geom_user, binning_alloc, binning_user, image_alloc, image_user, P, D, M, background,
                        width, height, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations,
                        cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered, out_color,
                        out_depth, radii, debug, stream, colors_aux, out_color_aux);
}

int64_t s3g_rasterize_forward_split(s3g_alloc_fn geom_alloc, void* geom_user, s3g_alloc_fn binning_alloc,
                                    void* binning_user, s3g_alloc_fn image_alloc, void* image_user, int P,
                                    int D, int M, const float* background, int width, int height,
                                    const float* means3D, const float* shs, const float* colors_precomp,
                                    const float* opacities, const float* scales, float scale_modifier,
                                    const float* rotations, const float* cov3D_precomp,
                                    const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                    float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                                    float* out_depth, int* radii, int debug, void* stream,
                                    const uint8_t* group, float* out_color_d, float* out_depth_d,
                                    float* out_color_s, float* out_depth_s) {
    if (!out_color_d || !out_depth_d || !out_color_s || !out_depth_s)
        return fail(S3G_ERR_ARG, "forward_split: null dynamic/static output");
    if (P > 0 && !group) return fail(S3G_ERR_ARG, "forward_split: null group");
    return forward_impl(geom_alloc, geom_user, binning_alloc, binning_user, image_alloc, image_user, P, D, M, background,
                        width, height, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations,
                        cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered, out_color,
                        out_depth, radii, debug, stream, nullptr, nullptr, group, out_color_d, out_depth_d,
                        out_color_s, out_depth_s);
}

int s3g_rasterize_backward(int P, int D, int M, int64_t R, const float* background, int width,
                           int height, const float* means3D, const float* shs,
                           const float* colors_precomp, const float* scales, float scale_modifier,
                           const float* rotations, const float* cov3D_precomp,
                           const float* viewmatrix, const float* projmatrix, const float* campos,
                           float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                           char* binning_buffer, char* image_buffer, const float* dL_dpix,
                           const float* dL_dpix_depth, float* dL_dmean2D, float* dL_dconic,
                           float* dL_dopacity, float* dL_dcolor, float* dL_ddepth, float* dL_dmean3D,
                           float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                           int debug, void* stream) {
    return backward_impl(P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales, scale_modifier,
                         rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer,
                         binning_buffer, image_buffer, dL_dpix, dL_dpix_depth, dL_dmean2D, dL_dconic, dL_dopacity,
                         dL_dcolor, dL_ddepth, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, debug, stream, nullptr,
                         nullptr);
}

int s3g_rasterize_backward_dp(int P, int D, int M, int64_t R, const float* background, int width,
                              int height, const float* means3D, const float* shs,
                              const float* colors_precomp, const float* scales, float scale_modifier,
                              const float* rotations, const float* cov3D_precomp,
                              const float* viewmatrix, const float* projmatrix, const float* campos,
                              float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                              char* binning_buffer, char* image_buffer, const float* dL_dpix,
                              const float* dL_dpix_depth, float* dL_dmean2D, float* dL_dconic,
                              float* dL_dopacity, float* dL_dcolor, float* dL_ddepth, float* dL_dmean3D,
                              float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                              int debug, void* stream, const s3g_peer_sink* sink) {
    if (!sink) return fail(S3G_ERR_ARG, "backward_dp: null sink");
    return backward_impl(P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales, scale_modifier,
                         rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer,
                         binning_buffer, image_buffer, dL_dpix, dL_dpix_depth, dL_dmean2D, dL_dconic, dL_dopacity,
                         dL_dcolor, dL_ddepth, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, debug, stream, nullptr,
                         nullptr, sink);
}

int s3g_rasterize_backward_aux(int P, int D, int M, int64_t R, const float* background, int width,
                               int height, const float* means3D, const float* shs,
                               const float* colors_precomp, const float* scales, float scale_modifier,
                               const float* rotations, const float* cov3D_precomp,
                               const float* viewmatrix, const float* projmatrix, const float* campos,
                               float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                               char* binning_buffer, char* image_buffer, const float* dL_dpix,
                               const float* dL_dpix_depth, float* dL_dmean2D, float* dL_dconic,
                               float* dL_dopacity, float* dL_dcolor, float* dL_ddepth, float* dL_dmean3D,
                               float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                               int debug, void* stream, const float* dL_dpix_aux, float* dL_dcolor_aux) {
    if (!dL_dpix_aux || !dL_dcolor_aux) return fail(S3G_ERR_ARG, "backward_aux: null aux gradients");
    return backward_impl(P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales, scale_modifier,
                         rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer,
                         binning_buffer, image_buffer, dL_dpix, dL_dpix_depth, dL_dmean2D, dL_dconic, dL_dopacity,
                         dL_dcolor, dL_ddepth, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, debug, stream,
                         dL_dpix_aux, dL_dcolor_aux);
}

}  // extern "C"
