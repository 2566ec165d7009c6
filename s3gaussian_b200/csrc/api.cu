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
#include <mutex>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "api_common.cuh"
#include "binning.cuh"
#include "camera_grad.cuh"
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

// Launch a per-Gaussian kernel that stages each warp's SH rows (3 * M floats per Gaussian) in dynamic shared memory
// when use_sh: k16 for rows of 16 coefficients, whose length it knows at compile time, k0 for any other M or no SH.
template <class Args>
int launch_sh_rows(void (*k16)(Args), void (*k0)(Args), const Args& args, int grid, int threads, int M, bool use_sh,
                   const char* what, cudaStream_t stream) {
    const size_t smem = use_sh ? (size_t)threads * row_stride(3 * M) * sizeof(float) : 0;
    if (smem > 200 * 1024) return fail(S3G_ERR_ARG, (std::string(what) + ": too many SH coefficients").c_str());
    if (use_sh && M == 16) {
        k16<<<grid, threads, smem, stream>>>(args);
        return S3G_OK;
    }
    if (smem > 48 * 1024)
        S3G_CUDA(cudaFuncSetAttribute(k0, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "smem attribute");
    k0<<<grid, threads, smem, stream>>>(args);
    return S3G_OK;
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
        if (f == "median_contrib") return set(s.median_contrib, 4, (size_t)width * height);
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
// Image buffers whose last forward kept the median state (OpacityOut::median_contrib), with the image size: the
// backward checks a median gradient against it on the host, before any launch.  Every forward on a buffer updates
// its entry; the oldest entries go beyond kMedianStates.
constexpr size_t kMedianStates = 1024;
struct MedianState {
    const char* image;
    int width, height;
};
std::mutex g_median_mu;
std::vector<MedianState> g_median_states;

void note_median_state(const char* image, int width, int height, bool kept) {
    std::lock_guard<std::mutex> lock(g_median_mu);
    auto& v = g_median_states;
    for (size_t i = 0; i < v.size(); ++i)
        if (v[i].image == image) {
            v.erase(v.begin() + i);
            break;
        }
    if (!kept) return;
    if (v.size() == kMedianStates) v.erase(v.begin());
    v.push_back({image, width, height});
}
bool has_median_state(const char* image, int width, int height) {
    std::lock_guard<std::mutex> lock(g_median_mu);
    for (const MedianState& m : g_median_states)
        if (m.image == image) return m.width == width && m.height == height;
    return false;
}

// Geometry buffers whose last forward was antialiased (s3g_rasterize_forward_antialiased): the backward and the camera
// pass apply that forward's chain rule, chosen on the host before any launch.  Every forward on a buffer updates its
// entry.  Unlike the median record this one has no cap: a forgotten entry would silently give the plain gradients.
// It holds one pointer per distinct buffer address an antialiased forward has used and no later forward has reused.
std::mutex g_aa_mu;
std::unordered_set<const char*> g_aa_states;

void note_aa_state(const char* geom, bool antialiased) {
    std::lock_guard<std::mutex> lock(g_aa_mu);
    if (antialiased) g_aa_states.insert(geom);
    else g_aa_states.erase(geom);
}
bool has_aa_state(const char* geom) {
    if (!geom) return false;
    std::lock_guard<std::mutex> lock(g_aa_mu);
    return g_aa_states.count(geom) != 0;
}

// Geometry buffers whose last forward went through a lens (s3g_rasterize_forward_lens), with that lens: the backward
// applies its chain rule, chosen on the host before any launch.  Every forward on a buffer updates its entry; no cap,
// for the reason of the antialiasing record.
std::mutex g_lens_mu;
std::unordered_map<const char*, LensParams> g_lens_states;

void note_lens_state(const char* geom, const LensParams* lens) {
    std::lock_guard<std::mutex> lock(g_lens_mu);
    if (lens) g_lens_states[geom] = *lens;
    else g_lens_states.erase(geom);
}
bool lens_state(const char* geom, LensParams* out) {
    if (!geom) return false;
    std::lock_guard<std::mutex> lock(g_lens_mu);
    auto it = g_lens_states.find(geom);
    if (it == g_lens_states.end()) return false;
    if (out) *out = it->second;
    return true;
}

// s*: the smallest positive root of 1 + 3 k1 s + 5 k2 s^2 + 7 k3 s^3 = d(r rho(r^2))/dr, in double, or +inf.  The
// polynomial is monotone between its critical points; the first interval whose end is not positive holds the root,
// found by bisection.
double lens_max_radius2(double k1, double k2, double k3) {
    const double c[4] = {1.0, 3.0 * k1, 5.0 * k2, 7.0 * k3};
    auto p = [&](double s) { return c[0] + s * (c[1] + s * (c[2] + s * c[3])); };
    int deg = 3;
    while (deg > 0 && c[deg] == 0.0) --deg;
    if (deg == 0) return INFINITY;
    double bound = 0.0;   // Cauchy: every root has |s| < 1 + max |c_i / c_deg|
    for (int i = 0; i < deg; ++i) bound = std::max(bound, std::fabs(c[i] / c[deg]));
    bound += 1.0;
    // positive roots of p' = c1 + 2 c2 s + 3 c3 s^2, ascending
    std::vector<double> ends;
    const double qa = 3.0 * c[3], qb = 2.0 * c[2], qc = c[1];
    if (qa != 0.0) {
        const double disc = qb * qb - 4.0 * qa * qc;
        if (disc >= 0.0) {
            const double r = std::sqrt(disc);
            const double q = -0.5 * (qb + (qb >= 0.0 ? r : -r));
            if (q != 0.0) {
                ends.push_back(q / qa);
                ends.push_back(qc / q);
            } else {
                ends.push_back(0.0);
            }
        }
    } else if (qb != 0.0) {
        ends.push_back(-qc / qb);
    }
    std::sort(ends.begin(), ends.end());
    std::vector<double> pts = {0.0};
    for (double e : ends)
        if (e > 0.0 && e < bound) pts.push_back(e);
    pts.push_back(bound);
    for (size_t i = 0; i + 1 < pts.size(); ++i) {
        double lo = pts[i], hi = pts[i + 1];
        if (p(hi) > 0.0) continue;   // p(lo) > 0 here: no root yet
        for (int it = 0; it < 400 && lo < hi; ++it) {
            const double mid = 0.5 * (lo + hi);
            if (mid <= lo || mid >= hi) break;
            if (p(mid) > 0.0) lo = mid;
            else hi = mid;
        }
        return hi;
    }
    return INFINITY;
}

// The kernels' LensParams of a lens and an image size; S3G_ERR_ARG for a lens s3g_rasterize_forward_lens rejects.
int lens_params(const s3g_raster_lens* l, int width, int height, LensParams* out) {
    if (!l) return fail(S3G_ERR_ARG, "forward_lens: null lens");
    if (!(std::isfinite(l->fx) && l->fx > 0.f && std::isfinite(l->fy) && l->fy > 0.f))
        return fail(S3G_ERR_ARG, "forward_lens: fx and fy must be finite and positive");
    for (float v : {l->cx, l->cy, l->k1, l->k2, l->p1, l->p2, l->k3})
        if (!std::isfinite(v)) return fail(S3G_ERR_ARG, "forward_lens: cx, cy and the distortion coefficients must be finite");
    LensParams& L = *out;
    L.fx = l->fx; L.fy = l->fy; L.cx = l->cx; L.cy = l->cy;
    L.k1 = l->k1; L.k2 = l->k2; L.p1 = l->p1; L.p2 = l->p2; L.k3 = l->k3;
    L.max_r2 = (float)lens_max_radius2(l->k1, l->k2, l->k3);
    L.xlo = (float)(-1.3 * (double)l->cx / l->fx);
    L.xhi = (float)(1.3 * ((double)width - l->cx) / l->fx);
    L.ylo = (float)(-1.3 * (double)l->cy / l->fy);
    L.yhi = (float)(1.3 * ((double)height - l->cy) / l->fy);
    L.ndc_x = 2.f / (float)width;
    L.ndc_y = 2.f / (float)height;
    return S3G_OK;
}

// one forward composite walk; the plain walks take the RenderFwdArgs part of ra, and an opacity walk is launched when
// opa is given
template <int NA, bool SPLIT>
void launch_render_forward(const RenderSplitArgs& ra, const AuxSet& a1, const OpacityOut* opa, dim3 grid,
                           cudaStream_t stream) {
    if (opa) render_forward_opacity_kernel<NA, SPLIT><<<grid, TILE_PIX, 0, stream>>>(ra, a1, *opa);
    else render_forward_kernel<NA, SPLIT><<<grid, TILE_PIX, 0, stream>>>(ra, a1);
}

// o: the opacity outputs (s3g_rasterize_forward_opacity), or NULL for the plain forward.  aa: antialiased
// lens: the lens forward's parameters (s3g_rasterize_forward_lens), or NULL
int64_t forward_impl(const s3g_raster_scene& s, const s3g_raster_forward_args& f, const s3g_raster_opacity_args* o,
                     bool aa, cudaStream_t stream, const LensParams* lens = nullptr) {
    const int P = s.P, width = s.width, height = s.height, debug = s.debug;
    if (P < 0 || width <= 0 || height <= 0) return fail(S3G_ERR_ARG, "forward: bad sizes");
    if (!f.geom_alloc || !f.binning_alloc || !f.image_alloc) return fail(S3G_ERR_ARG, "forward: null allocator");
    if (!f.out_color || !f.out_depth || !s.background) return fail(S3G_ERR_ARG, "forward: null output/background");
    const size_t HW = (size_t)width * height;
    if ((f.colors_aux != nullptr) != (f.out_color_aux != nullptr))
        return fail(S3G_ERR_ARG, "forward: colors_aux and out_color_aux go together");
    const int n_group_out = (f.out_color_d != nullptr) + (f.out_depth_d != nullptr) + (f.out_color_s != nullptr) +
                            (f.out_depth_s != nullptr);
    if (n_group_out != 0 && n_group_out != 4)
        return fail(S3G_ERR_ARG, "forward_eval: the four dynamic/static outputs are all given or all NULL");
    if (n_group_out == 0 && f.group) return fail(S3G_ERR_ARG, "forward_eval: group without dynamic/static outputs");
    if (n_group_out == 4 && P > 0 && !f.group) return fail(S3G_ERR_ARG, "forward_eval: null group");
    if (f.n_flow < 0 || f.n_flow > 2) return fail(S3G_ERR_ARG, "forward_eval: n_flow must be 0, 1 or 2");
    for (int k = 0; k < 2; ++k) {
        if (k >= f.n_flow) {
            if (f.flow_colors[k] || f.out_flow[k])
                return fail(S3G_ERR_ARG, "forward_eval: flow pointers beyond n_flow must be NULL");
            continue;
        }
        if (!f.out_flow[k] || (P > 0 && !f.flow_colors[k]))
            return fail(S3G_ERR_ARG, "forward_eval: null flow colours / flow image");
        if ((reinterpret_cast<uintptr_t>(f.flow_colors[k]) & 15) != 0)
            return fail(S3G_ERR_ARG, "forward_eval: flow colours must be 16-byte aligned [P,4] float arrays");
    }
    const bool split = n_group_out == 4;
    if (split && f.colors_aux) return fail(S3G_ERR_ARG, "forward: the split and aux forwards do not combine");
    // the composite writes the first flow set through the aux slot
    if (f.n_flow > 0 && f.colors_aux) return fail(S3G_ERR_ARG, "forward: colors_aux and flow colours do not combine");
    const s3g_raster_opacity_args no_opa = {};
    const s3g_raster_opacity_args& op = o ? *o : no_opa;
    if (op.dL_dpix_alpha || op.dL_dpix_median)
        return fail(S3G_ERR_ARG, "forward_opacity: dL_dpix_alpha / dL_dpix_median are backward inputs");
    if ((op.out_alpha_d != nullptr) != (op.out_alpha_s != nullptr))
        return fail(S3G_ERR_ARG, "forward_opacity: out_alpha_d and out_alpha_s go together");
    if (op.out_alpha_d && !split)
        return fail(S3G_ERR_ARG, "forward_opacity: out_alpha_d / out_alpha_s need the decomposition (group)");
    const bool use_opa = op.out_alpha || op.out_median_depth || op.out_alpha_d;
    // the median positions are kept where a backward may follow: not after the decomposition or a flow set
    const bool keep_median = op.out_median_depth && !split && f.n_flow == 0;
    if (P == 0) {   // rasterize_points.cu:82: outputs stay zero-filled
        for (float* a : {op.out_alpha, op.out_median_depth, op.out_alpha_d, op.out_alpha_s})
            if (a) S3G_CUDA(cudaMemsetAsync(a, 0, HW * sizeof(float), stream), "memset opacity image");
        if (split) {
            S3G_CUDA(cudaMemsetAsync(f.out_color_d, 0, 3 * HW * sizeof(float), stream), "memset color_d");
            S3G_CUDA(cudaMemsetAsync(f.out_depth_d, 0, HW * sizeof(float), stream), "memset depth_d");
            S3G_CUDA(cudaMemsetAsync(f.out_color_s, 0, 3 * HW * sizeof(float), stream), "memset color_s");
            S3G_CUDA(cudaMemsetAsync(f.out_depth_s, 0, HW * sizeof(float), stream), "memset depth_s");
        }
        if (f.out_color_aux)
            S3G_CUDA(cudaMemsetAsync(f.out_color_aux, 0, 3 * HW * sizeof(float), stream), "memset aux");
        for (float* o : f.out_flow)
            if (o) S3G_CUDA(cudaMemsetAsync(o, 0, 3 * HW * sizeof(float), stream), "memset flow");
        S3G_CUDA(cudaMemsetAsync(f.out_color, 0, 3 * HW * sizeof(float), stream), "memset color");
        S3G_CUDA(cudaMemsetAsync(f.out_depth, 0, HW * sizeof(float), stream), "memset depth");
        return 0;
    }
    if (!s.means3D || !s.opacities || !s.viewmatrix || !s.projmatrix)
        return fail(S3G_ERR_ARG, "forward: null input");
    if (!s.colors_precomp && !s.shs)
        return fail(S3G_ERR_ARG, "forward: need SHs or precomputed colours");
    if (!s.colors_precomp && !s.cam_pos) return fail(S3G_ERR_ARG, "forward: SH path needs cam_pos");
    if (!s.cov3D_precomp && (!s.scales || !s.rotations))
        return fail(S3G_ERR_ARG, "forward: need scales+rotations or precomputed cov3D");
    if (!s.colors_precomp && (s.D < 0 || s.D > 3 || s.M < (s.D + 1) * (s.D + 1)))
        return fail(S3G_ERR_ARG, "forward: SH degree/coefficient count mismatch");
    if ((int64_t)P >= (1ll << 30)) return fail(S3G_ERR_ARG, "forward: P too large");

    const TileGrid tg = tile_grid(width, height);
    if (tg.x > 65535 || tg.y > 65535) return fail(S3G_ERR_ARG, "forward: image too large");

    char* gptr = f.geom_alloc(f.geom_user, s3g_geom_bytes(P));
    if (!gptr) return fail(S3G_ERR_ALLOC, "forward: geometry allocator returned NULL");
    GeomState geom = GeomState::carve(gptr, P);
    note_aa_state(gptr, aa);
    note_lens_state(gptr, lens);
    char* iptr = f.image_alloc(f.image_user, s3g_image_bytes(width, height));
    if (!iptr) return fail(S3G_ERR_ALLOC, "forward: image allocator returned NULL");
    ImageState img = ImageState::carve(iptr, width, height);
    note_median_state(iptr, width, height, keep_median);
    int* radii = f.radii ? f.radii : geom.internal_radii;

    // ---- per-Gaussian preprocess -----------------------------------------
    PreFwdArgs pa;
    pa.P = P; pa.D = s.D; pa.M = s.M;
    pa.means3D = s.means3D; pa.scales = s.scales; pa.scale_modifier = s.scale_modifier;
    pa.rotations = s.rotations; pa.opacities = s.opacities; pa.shs = s.shs;
    pa.cov3D_precomp = s.cov3D_precomp; pa.colors_precomp = s.colors_precomp;
    pa.view = s.viewmatrix; pa.proj = s.projmatrix; pa.campos = s.cam_pos;
    pa.W = width; pa.H = height;
    pa.tan_fovx = s.tan_fovx; pa.tan_fovy = s.tan_fovy;
    pa.focal_y = height / (2.0f * s.tan_fovy);   // rasterizer_impl.cu:223-224
    pa.focal_x = width / (2.0f * s.tan_fovx);
    pa.radii = radii; pa.xyAB = geom.xyAB; pa.Cod = geom.Cod; pa.rgb = geom.rgb;
    pa.colors_aux = f.colors_aux; pa.aux = geom.aux;
    pa.depth_key = geom.depth_key; pa.tiles_touched = geom.tiles_touched; pa.rect = geom.rect;
    pa.clamped = geom.clamped; pa.order = geom.order_a;
    pa.grid_x = tg.x; pa.grid_y = tg.y;
    // scan_misc[4]: dynamic-Gaussian count of a split forward (zeroed with the scan state below)
    pa.group = split ? f.group : nullptr;
    pa.group_count = split ? geom.scan_misc + 4 : nullptr;
    g_timer.begin(0);
    // one memset for everything the chained scan and the depth sort expect zeroed (look-back words, tickets,
    // digit histograms)
    S3G_CUDA(cudaMemsetAsync(geom.scan_status, 0, geom.zero_bytes, stream), "memset scan/sort state");
    S3G_MARK(0, "preprocess_forward");
    {
        const int grid = (P + PRE_THREADS - 1) / PRE_THREADS;
        const bool use_sh = s.colors_precomp == nullptr;
        int rc;
        if (lens) {
            PreFwdLensArgs pl;
            static_cast<PreFwdArgs&>(pl) = pa;
            pl.lens = *lens;
            rc = aa ? launch_sh_rows(preprocess_forward_lens_kernel<16, true>, preprocess_forward_lens_kernel<0, true>,
                                     pl, grid, PRE_THREADS, s.M, use_sh, "forward", stream)
                    : launch_sh_rows(preprocess_forward_lens_kernel<16, false>,
                                     preprocess_forward_lens_kernel<0, false>, pl, grid, PRE_THREADS, s.M, use_sh,
                                     "forward", stream);
        } else {
            rc = aa ? launch_sh_rows(preprocess_forward_kernel<16, true>, preprocess_forward_kernel<0, true>, pa,
                                     grid, PRE_THREADS, s.M, use_sh, "forward", stream)
                    : launch_sh_rows(preprocess_forward_kernel<16>, preprocess_forward_kernel<0>, pa, grid,
                                     PRE_THREADS, s.M, use_sh, "forward", stream);
        }
        if (rc != S3G_OK) return rc;
    }
    S3G_STAGE("preprocess_forward");
    S3G_MARK(0, "depth_sort");

    // ---- depth digits of the LSD sort, over Gaussians --------------------
    // The offsets are first written by the scan below, so until then their buffer is the sort's second key scratch
    // and depth_key keeps every Gaussian's key (what s3g_state_field exports under that name).
    S3G_CUDA(radix_sort_pairs((uint32_t)P, geom.depth_key, geom.order_a, geom.key_b, geom.order_b,
                              nullptr, geom.order_a, 0, 32, geom.sort, stream, nullptr, /*hist_ready=*/false,
                              /*prepared=*/true, /*keys_spare=*/geom.offsets),
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
        char* bptr = f.binning_alloc(f.binning_user, s3g_binning_bytes(cap));
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
        RenderSplitArgs ra = {};
        ra.ranges = img.ranges; ra.point_list = bin.point_list; ra.W = width; ra.H = height;
        ra.xyAB = geom.xyAB; ra.Cod = geom.Cod; ra.rgb = geom.rgb; ra.bg = s.background;
        ra.final_T = img.final_T; ra.n_contrib = img.n_contrib;
        ra.out_color = f.out_color; ra.out_depth = f.out_depth;
        ra.aux = geom.aux; ra.out_aux = f.out_color_aux;
        // flow colour sets are gathered from the caller's [P,4] arrays directly (no copy into geom.aux)
        AuxSet a1 = {reinterpret_cast<const float4*>(f.flow_colors[1]), f.out_flow[1]};
        if (f.n_flow > 0) { ra.aux = reinterpret_cast<const float4*>(f.flow_colors[0]); ra.out_aux = f.out_flow[0]; }
        ra.out_color_d = f.out_color_d; ra.out_depth_d = f.out_depth_d;
        ra.out_color_s = f.out_color_s; ra.out_depth_s = f.out_depth_s;
        ra.group_count = geom.scan_misc + 4; ra.P = (uint32_t)P;
        const int na = f.n_flow == 2 ? 2 : (f.colors_aux || f.n_flow == 1) ? 1 : 0;   // extra colour sets
        const dim3 grid(tg.x, tg.y);
        const OpacityOut oo = {op.out_alpha, op.out_median_depth, op.out_alpha_d, op.out_alpha_s,
                               keep_median ? img.median_contrib : nullptr};
        const OpacityOut* opa = use_opa ? &oo : nullptr;
        if (split) {
            if (na == 2) launch_render_forward<2, true>(ra, a1, opa, grid, stream);
            else if (na == 1) launch_render_forward<1, true>(ra, a1, opa, grid, stream);
            else launch_render_forward<0, true>(ra, a1, opa, grid, stream);
        } else if (na == 2) launch_render_forward<2, false>(ra, a1, opa, grid, stream);
        else if (na == 1) launch_render_forward<1, false>(ra, a1, opa, grid, stream);
        else launch_render_forward<0, false>(ra, a1, opa, grid, stream);
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

// one backward composite walk (the default walk takes the RenderBwdArgs part of ra); > 48 KB of dynamic shared memory
// needs the opt-in, once per (kernel, device)
template <bool AUX, bool DET, bool OPA, bool ABS>
int launch_render_backward(const RenderBwdDetArgs& ra, const TileGrid& tg, cudaStream_t stream) {
    static unsigned long long attr_done = 0;
    int devid = 0;
    S3G_CUDA(cudaGetDevice(&devid), "cudaGetDevice");
    if (devid >= 64 || !((attr_done >> devid) & 1ull)) {
        S3G_CUDA(cudaFuncSetAttribute(render_backward_kernel<AUX, DET, OPA, ABS>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sizeof(RenderBwdSmem<AUX, DET, OPA, ABS>)),
                 DET ? "render_backward_det smem attribute" : "render_backward smem attribute");
        if (devid < 64) attr_done |= 1ull << devid;
    }
    render_backward_kernel<AUX, DET, OPA, ABS>
        <<<dim3(tg.x, tg.y), TILE_PIX, sizeof(RenderBwdSmem<AUX, DET, OPA, ABS>), stream>>>(ra);
    return S3G_OK;
}
template <bool DET, bool ABS>
int launch_render_backward(bool aux, bool opa, const RenderBwdDetArgs& ra, const TileGrid& tg, cudaStream_t stream) {
    if (opa) return aux ? launch_render_backward<true, DET, true, ABS>(ra, tg, stream)
                        : launch_render_backward<false, DET, true, ABS>(ra, tg, stream);
    return aux ? launch_render_backward<true, DET, false, ABS>(ra, tg, stream)
               : launch_render_backward<false, DET, false, ABS>(ra, tg, stream);
}
template <bool DET>
int launch_render_backward(bool aux, bool opa, bool abs, const RenderBwdDetArgs& ra, const TileGrid& tg,
                           cudaStream_t stream) {
    return abs ? launch_render_backward<DET, true>(aux, opa, ra, tg, stream)
               : launch_render_backward<DET, false>(aux, opa, ra, tg, stream);
}

// det: the deterministic destination of the backward composite walk (composite.cuh) with det_ws as its workspace,
// instead of the REDs into grad_rec; everything else, validation included, is shared.
// o: the opacity-image gradients (the *_opacity entry points), or NULL.
// absgrad: the absolute screen-space gradients as well (s3g_rasterize_backward_absgrad), written to dL_dmean2D_abs
int backward_impl(const s3g_raster_scene& s, const s3g_raster_backward_args& b, const s3g_raster_opacity_args* o,
                  cudaStream_t stream, bool det, void* det_ws, bool absgrad = false, float* dL_dmean2D_abs = nullptr) {
    const int P = s.P, width = s.width, height = s.height, debug = s.debug;
    const s3g_peer_sink* sink = b.sink;
    if (P < 0 || width <= 0 || height <= 0 || b.R < 0) return fail(S3G_ERR_ARG, "backward: bad sizes");
    if (P == 0) return S3G_OK;   // rasterize_points.cu:165
    if (absgrad && !dL_dmean2D_abs) return fail(S3G_ERR_ARG, "backward_absgrad: null dL_dmean2D_abs");
    if (!b.geom_buffer || !b.image_buffer || (b.R > 0 && !b.binning_buffer))
        return fail(S3G_ERR_STATE, "backward: missing state buffer");
    if (!s.means3D || !s.viewmatrix || !s.projmatrix || !s.background || !b.dL_dpix || !b.dL_dpix_depth)
        return fail(S3G_ERR_ARG, "backward: null input");
    if (!sink && (!b.dL_dmean2D || !b.dL_dopacity || !b.dL_dcolor || !b.dL_dmean3D || !b.dL_dcov3D || !b.dL_dscale ||
                  !b.dL_drot))
        return fail(S3G_ERR_ARG, "backward: null gradient output");
    if (!sink && (reinterpret_cast<uintptr_t>(b.dL_drot) & 15))
        return fail(S3G_ERR_ARG, "backward: dL_drot must be 16-byte aligned (its [P,4] rows are stored 16 bytes at a time)");
    if (sink) {
        if (!b.dL_dmean2D || !b.dL_dcolor) return fail(S3G_ERR_ARG, "backward_dp: dL_dmean2D / dL_dcolor stay local and must be given");
        if (s.cov3D_precomp) return fail(S3G_ERR_ARG, "backward_dp: precomputed 3-D covariances are not exchanged");
        if (sink->world < 2 || sink->world > 16 || sink->rank < 0 || sink->rank >= sink->world || sink->chunk <= 0 ||
            (sink->chunk & 3) || sink->off_means3D < 0 || sink->off_opacities < 0 || sink->off_scales < 0 ||
            sink->off_rotations < 0 || (s.colors_precomp == nullptr && (sink->off_shs < 0 || (sink->off_shs & 3))))
            return fail(S3G_ERR_ARG, "backward_dp: bad peer sink (world, rank, chunk % 4, offsets, off_shs % 4)");
        for (int p = 0; p < sink->world; ++p)
            if (!sink->stage[p]) return fail(S3G_ERR_ARG, "backward_dp: null staging pointer");
    }
    const bool aa = has_aa_state(b.geom_buffer);
    if (sink && aa)
        return fail(S3G_ERR_ARG, "backward_dp: the fused gradient exchange does not take an antialiased forward's "
                                 "gradients");
    LensParams lens;
    const bool use_lens = lens_state(b.geom_buffer, &lens);
    if (sink && use_lens)
        return fail(S3G_ERR_ARG, "backward_dp: the fused gradient exchange does not take a lens forward's gradients");
    if ((b.dL_dpix_aux != nullptr) != (b.dL_dcolor_aux != nullptr))
        return fail(S3G_ERR_ARG, "backward: dL_dpix_aux and dL_dcolor_aux go together");
    const bool use_aux = b.dL_dpix_aux != nullptr;
    if (sink && use_aux) return fail(S3G_ERR_ARG, "backward: a peer sink and the aux gradients do not combine");
    const bool use_sh = (s.colors_precomp == nullptr);
    if (use_sh && (!s.shs || (!b.dL_dsh && !sink) || !s.cam_pos)) return fail(S3G_ERR_ARG, "backward: SH path needs shs, dL_dsh, campos");
    if (!s.cov3D_precomp && (!s.scales || !s.rotations))
        return fail(S3G_ERR_ARG, "backward: need scales+rotations or precomputed cov3D");
    if (det && sink) return fail(S3G_ERR_ARG, "backward_deterministic: the fused gradient exchange is not deterministic");
    if (det && b.R > 0 && (!det_ws || (reinterpret_cast<uintptr_t>(det_ws) & 15)))
        return fail(S3G_ERR_ARG, "backward_deterministic: workspace must be non-NULL and 16-byte aligned");
    const s3g_raster_opacity_args no_opa = {};
    const s3g_raster_opacity_args& op = o ? *o : no_opa;
    if (op.out_alpha_d || op.out_alpha_s)
        return fail(S3G_ERR_ARG, "backward_opacity: the decomposition (out_alpha_d / out_alpha_s) is forward only");
    if (op.out_alpha || op.out_median_depth)
        return fail(S3G_ERR_ARG, "backward_opacity: out_alpha / out_median_depth are forward outputs");
    const bool use_opa = op.dL_dpix_alpha || op.dL_dpix_median;
    if (sink && use_opa)
        return fail(S3G_ERR_ARG, "backward_opacity: a peer sink and the opacity-image gradients do not combine");
    if (op.dL_dpix_median && !has_median_state(b.image_buffer, width, height))
        return fail(S3G_ERR_ARG, "backward_opacity: dL_dpix_median needs a forward that kept the median state "
                                 "(s3g_rasterize_forward_opacity with out_median_depth, no decomposition or flow set)");

    GeomState geom = GeomState::carve(b.geom_buffer, P);
    BinningState bin = BinningState::carve(b.binning_buffer, b.R);
    ImageState img = ImageState::carve(b.image_buffer, width, height);
    const int* radii = b.radii ? b.radii : geom.internal_radii;
    const TileGrid tg = tile_grid(width, height);

    g_timer.begin(1);
    const bool det_walk = det && b.R > 0;
    RenderBwdDetArgs ra = {};
    ra.ranges = img.ranges; ra.point_list = bin.point_list; ra.W = width; ra.H = height;
    ra.bg = s.background; ra.xyAB = geom.xyAB; ra.Cod = geom.Cod; ra.rgb = geom.rgb;
    ra.final_T = img.final_T; ra.n_contrib = img.n_contrib;
    ra.dL_dpix = b.dL_dpix; ra.dL_dpix_depth = b.dL_dpix_depth; ra.grad_rec = geom.grad_rec;
    ra.aux = geom.aux; ra.dL_dpix_aux = b.dL_dpix_aux;
    ra.dL_dpix_alpha = op.dL_dpix_alpha; ra.dL_dpix_median = op.dL_dpix_median; ra.median_contrib = img.median_contrib;
    if (det_walk) {
        // every grad_rec row is written by the gather: no memset
        float4* records = static_cast<float4*>(det_ws);
        uint32_t* base = reinterpret_cast<uint32_t*>(static_cast<char*>(det_ws) + det_records_bytes(b.R));
        ra.rect = geom.rect; ra.base = base; ra.records = records;
        S3G_MARK(1, "det_base");
        det_base_kernel<<<(P + 255) / 256, 256, 0, stream>>>((uint32_t)P, geom.order_a, geom.offsets, base);
        S3G_STAGE("det_base");
        S3G_MARK(1, "render_backward_det");
        const int rc = launch_render_backward<true>(use_aux, use_opa, absgrad, ra, tg, stream);
        if (rc != S3G_OK) return rc;
        S3G_STAGE("render_backward_det");
        S3G_MARK(1, "grad_rec_gather");
        grad_rec_gather_kernel<<<(unsigned)div_up64((int64_t)P * 4, 256), 256, 0, stream>>>(
            (uint32_t)P, (use_aux || absgrad) ? 4 : 3, geom.tiles_touched, base, records, reinterpret_cast<float4*>(geom.grad_rec));
        S3G_STAGE("grad_rec_gather");
    } else {
        S3G_MARK(1, "zero_grad_rec");
        S3G_CUDA(cudaMemsetAsync(geom.grad_rec, 0, (size_t)P * GRAD_REC * sizeof(float), stream),
                 "memset grad_rec");
        S3G_MARK(1, "render_backward");
        if (b.R > 0) {
            const int rc = launch_render_backward<false>(use_aux, use_opa, absgrad, ra, tg, stream);
            if (rc != S3G_OK) return rc;
            S3G_STAGE("render_backward");
        }
    }

    S3G_MARK(1, "preprocess_backward");
    PreBwdArgs pb;
    pb.P = P; pb.D = s.D; pb.M = use_sh ? s.M : 0;
    pb.means3D = s.means3D; pb.radii = radii;
    pb.shs = use_sh ? s.shs : nullptr;   // backward.cu:406
    pb.clamped = geom.clamped;
    pb.scales = s.cov3D_precomp ? nullptr : s.scales;   // backward.cu:410 (the reference keys on scales)
    pb.rotations = s.rotations; pb.scale_modifier = s.scale_modifier;
    pb.cov3D_precomp = s.cov3D_precomp;
    pb.view = s.viewmatrix; pb.proj = s.projmatrix; pb.campos = s.cam_pos;
    pb.focal_y = height / (2.0f * s.tan_fovy);
    pb.focal_x = width / (2.0f * s.tan_fovx);
    pb.tan_fovx = s.tan_fovx; pb.tan_fovy = s.tan_fovy;
    pb.grad_rec = geom.grad_rec;
    pb.dL_dmean2D = b.dL_dmean2D; pb.dL_dconic = b.dL_dconic; pb.dL_dopacity = b.dL_dopacity;
    pb.dL_dcolor = b.dL_dcolor; pb.dL_dcolor_aux = b.dL_dcolor_aux; pb.dL_ddepth = b.dL_ddepth; pb.dL_dmean3D = b.dL_dmean3D;
    pb.dL_dcov3D = b.dL_dcov3D; pb.dL_dsh = use_sh ? b.dL_dsh : nullptr;
    pb.dL_dscale = b.dL_dscale; pb.dL_drot = b.dL_drot;
    pb.Cod = geom.Cod;
    if (sink) {
        for (int p = 0; p < 16; ++p) pb.sink.stage[p] = p < sink->world ? static_cast<float*>(sink->stage[p]) : nullptr;
        pb.sink.world = sink->world; pb.sink.rank = sink->rank; pb.sink.chunk = sink->chunk;
        pb.sink.off_mean3D = sink->off_means3D; pb.sink.off_sh = sink->off_shs; pb.sink.off_opacity = sink->off_opacities;
        pb.sink.off_scale = sink->off_scales; pb.sink.off_rot = sink->off_rotations;
    }
    {
        const int grid = (P + PRE_THREADS - 1) / PRE_THREADS;
        PreBwdLensArgs pbl;
        if (use_lens) {
            static_cast<PreBwdArgs&>(pbl) = pb;
            pbl.lens = lens;
        }
        const int rc = use_lens ? (aa ? launch_sh_rows(preprocess_backward_lens_kernel<16, true>,
                                                       preprocess_backward_lens_kernel<0, true>, pbl, grid,
                                                       PRE_THREADS, s.M, use_sh, "backward", stream)
                                      : launch_sh_rows(preprocess_backward_lens_kernel<16, false>,
                                                       preprocess_backward_lens_kernel<0, false>, pbl, grid,
                                                       PRE_THREADS, s.M, use_sh, "backward", stream))
                       : sink ? launch_sh_rows(preprocess_backward_kernel<16, true>, preprocess_backward_kernel<0, true>,
                                             pb, grid, PRE_THREADS, s.M, use_sh, "backward", stream)
                       : aa ? launch_sh_rows(preprocess_backward_kernel<16, false, true>,
                                             preprocess_backward_kernel<0, false, true>, pb, grid, PRE_THREADS, s.M,
                                             use_sh, "backward", stream)
                            : launch_sh_rows(preprocess_backward_kernel<16>, preprocess_backward_kernel<0>, pb, grid,
                                             PRE_THREADS, s.M, use_sh, "backward", stream);
        if (rc != S3G_OK) return rc;
    }
    S3G_STAGE("preprocess_backward");
    if (absgrad) {
        S3G_MARK(1, "absgrad_export");
        absgrad_export_kernel<<<(P + 255) / 256, 256, 0, stream>>>((uint32_t)P, radii, geom.grad_rec,
                                                                   dL_dmean2D_abs);
        S3G_STAGE("absgrad_export");
    }
    S3G_MARK(1, nullptr);
    return S3G_OK;
}
}  // namespace

extern "C" {

int64_t s3g_rasterize_forward(const s3g_raster_scene* scene, const s3g_raster_forward_args* fwd, void* stream) {
    if (!scene || !fwd) return fail(S3G_ERR_ARG, "forward: null scene / forward arguments");
    return forward_impl(*scene, *fwd, nullptr, false, static_cast<cudaStream_t>(stream));
}

int64_t s3g_rasterize_forward_opacity(const s3g_raster_scene* scene, const s3g_raster_forward_args* fwd,
                                      const s3g_raster_opacity_args* opa, void* stream) {
    if (!scene || !fwd) return fail(S3G_ERR_ARG, "forward_opacity: null scene / forward arguments");
    return forward_impl(*scene, *fwd, opa, false, static_cast<cudaStream_t>(stream));
}

int64_t s3g_rasterize_forward_antialiased(const s3g_raster_scene* scene, const s3g_raster_forward_args* fwd,
                                          const s3g_raster_opacity_args* opa, void* stream) {
    if (!scene || !fwd) return fail(S3G_ERR_ARG, "forward_antialiased: null scene / forward arguments");
    return forward_impl(*scene, *fwd, opa, true, static_cast<cudaStream_t>(stream));
}

int64_t s3g_rasterize_forward_lens(const s3g_raster_scene* scene, const s3g_raster_forward_args* fwd,
                                   const s3g_raster_opacity_args* opa, int antialiased, const s3g_raster_lens* lens,
                                   void* stream) {
    if (!scene || !fwd) return fail(S3G_ERR_ARG, "forward_lens: null scene / forward arguments");
    LensParams L;
    const int rc = lens_params(lens, scene->width, scene->height, &L);
    if (rc != S3G_OK) return rc;
    return forward_impl(*scene, *fwd, opa, antialiased != 0, static_cast<cudaStream_t>(stream), &L);
}

double s3g_lens_max_radius2(const s3g_raster_lens* lens) {
    if (!lens) return NAN;
    return lens_max_radius2(lens->k1, lens->k2, lens->k3);
}

int s3g_rasterize_backward(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd, void* stream) {
    if (!scene || !bwd) return fail(S3G_ERR_ARG, "backward: null scene / backward arguments");
    return backward_impl(*scene, *bwd, nullptr, static_cast<cudaStream_t>(stream), false, nullptr);
}

int s3g_rasterize_backward_opacity(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                   const s3g_raster_opacity_args* opa, void* stream) {
    if (!scene || !bwd) return fail(S3G_ERR_ARG, "backward_opacity: null scene / backward arguments");
    return backward_impl(*scene, *bwd, opa, static_cast<cudaStream_t>(stream), false, nullptr);
}

size_t s3g_rasterize_backward_deterministic_workspace_bytes(int P, int64_t R, int width, int height) {
    if (P < 0 || R < 0 || R >= (1ll << 30) || width <= 0 || height <= 0) return 0;
    return det_records_bytes(R) + (size_t)P * sizeof(uint32_t);
}

int s3g_rasterize_backward_deterministic(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                         void* workspace, void* stream) {
    if (!scene || !bwd) return fail(S3G_ERR_ARG, "backward_deterministic: null scene / backward arguments");
    return backward_impl(*scene, *bwd, nullptr, static_cast<cudaStream_t>(stream), true, workspace);
}

int s3g_rasterize_backward_deterministic_opacity(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                                 const s3g_raster_opacity_args* opa, void* workspace, void* stream) {
    if (!scene || !bwd) return fail(S3G_ERR_ARG, "backward_deterministic_opacity: null scene / backward arguments");
    return backward_impl(*scene, *bwd, opa, static_cast<cudaStream_t>(stream), true, workspace);
}

int s3g_rasterize_backward_absgrad(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                   const s3g_raster_opacity_args* opa, float* dL_dmean2D_abs, int deterministic,
                                   void* workspace, void* stream) {
    if (!scene || !bwd) return fail(S3G_ERR_ARG, "backward_absgrad: null scene / backward arguments");
    return backward_impl(*scene, *bwd, opa, static_cast<cudaStream_t>(stream), deterministic != 0, workspace, true,
                         dL_dmean2D_abs);
}

size_t s3g_rasterize_camera_backward_workspace_bytes(int P) {
    if (P <= 0) return 0;
    return (size_t)camera_grad_blocks(P) * CAM_NCOMP * sizeof(double);
}

int s3g_rasterize_camera_backward(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                  const s3g_raster_camera_grads* out, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (!scene || !bwd || !out) return fail(S3G_ERR_ARG, "camera_backward: null scene / backward arguments / outputs");
    const s3g_raster_scene& s = *scene;
    const s3g_raster_backward_args& b = *bwd;
    const int P = s.P, debug = s.debug;
    if (!b.dL_dconic || !b.dL_ddepth)
        return fail(S3G_ERR_ARG, "camera_backward: the backward must have exported dL_dconic and dL_ddepth");
    if (!out->dL_dviewmatrix && !out->dL_dprojmatrix && !out->dL_dcampos)
        return fail(S3G_ERR_ARG, "camera_backward: no output asked for");
    if (lens_state(b.geom_buffer, nullptr))
        return fail(S3G_ERR_ARG, "camera_backward: camera gradients after a lens forward are not implemented");
    if (P < 0 || s.width <= 0 || s.height <= 0) return fail(S3G_ERR_ARG, "camera_backward: bad sizes");
    if (P > 0 && (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 15)))
        return fail(S3G_ERR_ARG, "camera_backward: workspace must be non-NULL and 16-byte aligned");
    if (P == 0) {   // nothing is rendered: the gradients are zero
        if (out->dL_dviewmatrix) S3G_CUDA(cudaMemsetAsync(out->dL_dviewmatrix, 0, 16 * sizeof(float), stream), "memset");
        if (out->dL_dprojmatrix) S3G_CUDA(cudaMemsetAsync(out->dL_dprojmatrix, 0, 16 * sizeof(float), stream), "memset");
        if (out->dL_dcampos) S3G_CUDA(cudaMemsetAsync(out->dL_dcampos, 0, 3 * sizeof(float), stream), "memset");
        return S3G_OK;
    }
    if (!s.means3D || !s.viewmatrix || !s.projmatrix || !b.dL_dmean2D)
        return fail(S3G_ERR_ARG, "camera_backward: null input");
    if (!s.cov3D_precomp && (!s.scales || !s.rotations))
        return fail(S3G_ERR_ARG, "camera_backward: need scales+rotations or precomputed cov3D");
    if (!b.radii && !b.geom_buffer) return fail(S3G_ERR_STATE, "camera_backward: missing state buffer");
    // campos enters through the SH colours only: with precomputed colours its gradient is zero
    const bool campos = out->dL_dcampos && !s.colors_precomp;
    if (campos) {
        if (!s.shs || !s.cam_pos || !b.dL_dcolor) return fail(S3G_ERR_ARG, "camera_backward: SH path needs shs, campos, dL_dcolor");
        if (!b.geom_buffer) return fail(S3G_ERR_STATE, "camera_backward: missing state buffer");
        if (s.D < 0 || s.D > 3 || s.M < (s.D + 1) * (s.D + 1))
            return fail(S3G_ERR_ARG, "camera_backward: SH degree/coefficient count mismatch");
    }
    const GeomState geom = GeomState::carve(b.geom_buffer, P);
    CamBwdArgs ca;
    ca.P = P; ca.D = s.D; ca.M = campos ? s.M : 0;
    ca.means3D = s.means3D; ca.radii = b.radii ? b.radii : geom.internal_radii;
    ca.shs = campos ? s.shs : nullptr; ca.clamped = campos ? geom.clamped : nullptr;
    ca.scales = s.cov3D_precomp ? nullptr : s.scales; ca.rotations = s.rotations; ca.scale_modifier = s.scale_modifier;
    ca.cov3D_precomp = s.cov3D_precomp;
    ca.view = s.viewmatrix; ca.proj = s.projmatrix; ca.campos = campos ? s.cam_pos : nullptr;
    ca.focal_y = s.height / (2.0f * s.tan_fovy);
    ca.focal_x = s.width / (2.0f * s.tan_fovx);
    ca.tan_fovx = s.tan_fovx; ca.tan_fovy = s.tan_fovy;
    ca.dL_dmean2D = b.dL_dmean2D; ca.dL_dconic = b.dL_dconic; ca.dL_ddepth = b.dL_ddepth; ca.dL_dcolor = b.dL_dcolor;
    ca.partial = static_cast<double*>(workspace);
    ca.nblocks = camera_grad_blocks(P);
    // after an antialiased forward: the opacity factor's term, from the records that forward and the backward left
    const bool aa = has_aa_state(b.geom_buffer);
    ca.grad_rec = geom.grad_rec; ca.Cod = geom.Cod;
    if (campos) {
        const int rc = aa ? launch_sh_rows(camera_grad_partial_kernel<16, true, true>,
                                           camera_grad_partial_kernel<0, true, true>, ca, ca.nblocks, CAM_THREADS,
                                           s.M, true, "camera_backward", stream)
                          : launch_sh_rows(camera_grad_partial_kernel<16, true>, camera_grad_partial_kernel<0, true>,
                                           ca, ca.nblocks, CAM_THREADS, s.M, true, "camera_backward", stream);
        if (rc != S3G_OK) return rc;
    } else if (aa) {
        camera_grad_partial_kernel<0, false, true><<<ca.nblocks, CAM_THREADS, 0, stream>>>(ca);
    } else {
        camera_grad_partial_kernel<0, false><<<ca.nblocks, CAM_THREADS, 0, stream>>>(ca);
    }
    S3G_STAGE("camera_grad_partial");
    camera_grad_finish_kernel<<<1, 32 * CAM_NCOMP, 0, stream>>>(ca.partial, ca.nblocks, out->dL_dviewmatrix,
                                                                  out->dL_dprojmatrix, out->dL_dcampos);
    S3G_STAGE("camera_grad_finish");
    return S3G_OK;
}

}  // extern "C"
