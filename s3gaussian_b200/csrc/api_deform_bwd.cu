// api_deform_bwd.cu - extern "C" entry points of the fused HexPlane + decoder stage, backward (see include/s3g_b200.h).
#include <cstdlib>
#include "deform_host.cuh"

using namespace s3g;

namespace {
// layout of one CTA's partial-gradient buffer
int make_offsets(const DNet& d, GradOff& o) {
    int t = 0;
    auto take = [&](int n) { int r = t; t += (n + 3) & ~3; return r; };
    for (int id = 0; id < TL_LAYERS; ++id) {
        const bool on = layer_on(d, id);
        grad_off(o, kLayers[id].ow) = on ? take(kLayers[id].n * layer_k(id, d.L)) : -1;
        grad_off(o, kLayers[id].ob) = on ? take(kLayers[id].n) : -1;
    }
    o.total = t;
    return t;
}
int bwd_grid(int ntiles) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return ntiles < sms ? ntiles : sms;
}
constexpr int kMaxBwdGrid = 256;
// per-texel accumulators of the time planes (ScatterArgs::tacc): [level][axis][reso][32] floats
size_t tacc_floats(const DNet& d) {
    size_t t = 0;
    for (int l = 0; l < d.L; ++l)
        for (int ax = 0; ax < 3; ++ax) t += (size_t)d.reso[l][ax] * FD;
    return t;
}

}  // namespace

extern "C" {

size_t s3g_deform_saved_bytes(const s3g_deform_net* net, int P) {
    DNet d;
    if (to_dnet(net, d) != S3G_OK || P <= 0) return 0;
    int slot[ACT_KINDS];
    return (size_t)act_slots(d, slot) * ((size_t)((P + 127) / 128) * 128 * 64) * sizeof(float);
}

size_t s3g_deform_workspace_bytes(const s3g_deform_net* net, int P) {
    DNet d;
    if (to_dnet(net, d) != S3G_OK) return 0;
    GradOff o;
    make_offsets(d, o);
    // per-CTA partial Linear gradients + dL/d(features) [P][32L]
    // + the time planes' per-texel accumulators
    return (size_t)kMaxBwdGrid * o.total * sizeof(float) + 512 + (size_t)(P > 0 ? P : 0) * FD * d.L * sizeof(float) + 256 +
           tacc_floats(d) * sizeof(float) + 256;
}

int s3g_deform_backward_saved(const s3g_deform_net* net, int P, const float* xyz, const float* scales,
                              const float* rotations, const float* opacity, const float* shs, float time,
                              const float* campos, int sh_degree, const float* features, const float* acts,
                              const float* g_means3D, const float* g_scales_act, const float* g_rot_act, const float* g_opacity_act,
                              const float* g_colors, const float* g_dx, const float* g_dshs, const float* g_feat,
                              float* d_xyz, float* d_scales, float* d_rotations, float* d_opacity, float* d_shs,
                              const s3g_deform_net_grads* grads, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "deform_backward: P < 0");
    DeformBwdArgs a;
    int rc = to_dnet(net, a.net);
    if (rc != S3G_OK) return rc;
    if (!grads || !workspace) return fail(S3G_ERR_ARG, "deform_backward: null grads/workspace");
    if (P > 0 && (!xyz || !scales || !rotations || !opacity || !shs || !campos || !features))
        return fail(S3G_ERR_ARG, "deform_backward: null input");
    if (P > 0 && !acts)
        return fail(S3G_ERR_ARG, "deform_backward: null acts (the hidden activations s3g_deform_forward_save keeps)");
    if (P > 0 && (!d_xyz || !d_scales || !d_rotations || !d_opacity || !d_shs))
        return fail(S3G_ERR_ARG, "deform_backward: null output");
    if (sh_degree < 0 || sh_degree > 3) return fail(S3G_ERR_ARG, "deform_backward: sh_degree must be 0..3");
    const DNet& d = a.net;
    a.P = P; a.xyz = xyz; a.scales = scales; a.rot = rotations; a.opacity = opacity; a.shs = shs;
    a.campos = campos; a.time = time; a.sh_degree = sh_degree;
    a.g_means = g_means3D; a.g_scales = g_scales_act; a.g_rot = g_rot_act; a.g_opacity = g_opacity_act;
    a.g_colors = g_colors; a.g_dx = g_dx; a.g_dshs = g_dshs; a.g_feat = g_feat;
    a.d_xyz = d_xyz; a.d_scales = d_scales; a.d_rot = d_rotations; a.d_opacity = d_opacity; a.d_shs = d_shs;
    for (int l = 0; l < d.L; ++l)
        for (int k = 0; k < 6; ++k) {
            a.gplanes[l][k] = grads->planes[l][k];
            if (!a.gplanes[l][k]) return fail(S3G_ERR_ARG, "deform_backward: null plane gradient");
        }
    make_offsets(d, a.off);
    act_slots(d, a.act_slot);
    a.acts = acts;
    a.act_stride = (size_t)((P + 127) / 128) * 128 * 64;
    build_wseq(d, a.wseq);
    a.partial = reinterpret_cast<float*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    a.features = features;
    a.dfeatures = a.partial + (size_t)kMaxBwdGrid * a.off.total;
    const int ntiles = (P + DT - 1) / DT;
    int grid = bwd_grid(ntiles);
    if (grid > kMaxBwdGrid) grid = kMaxBwdGrid;
    // destination table of the reduction
    ReduceArgs r;
    r.nseg = 0; r.partial = a.partial; r.stride = a.off.total; r.nparts = grid > 0 ? grid : 0;
    auto seg = [&](float* dst, int off, int count) -> bool {
        if (off < 0) return true;
        if (!dst) return false;
        r.seg[r.nseg++] = ReduceSeg{dst, off, count};
        return true;
    };
    bool ok = true;
    for (int id = 0; id < TL_LAYERS && ok; ++id) {
        const DeformLayer& l = kLayers[id];
        ok = seg(grads->*l.gw, grad_off(a.off, l.ow), l.n * layer_k(id, d.L)) && seg(grads->*l.gb, grad_off(a.off, l.ob), l.n);
    }
    if (!ok) return fail(S3G_ERR_ARG, "deform_backward: null Linear gradient for an enabled layer");
    if (P > 0) {
        const size_t smem = DeformBwdSmem::floats(d.L) * sizeof(float);
        if (smem > 227 * 1024) return fail(S3G_ERR_UNSUPPORTED, "deform_backward: too many levels for shared memory");
        auto launch = [&](auto kernel) -> int {
            S3G_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "deform bwd smem attr");
            kernel<<<grid, DTHREADS, smem, stream>>>(a);
            return S3G_OK;
        };
        rc = d.L == 4 ? launch(deform_backward_kernel<4>) : launch(deform_backward_kernel<0>);
        if (rc != S3G_OK) return rc;
        S3G_CUDA(cudaGetLastError(), "deform_backward launch");
        ScatterArgs sc;
        sc.net = a.net; sc.P = P; sc.xyz = xyz; sc.time = time; sc.dfeatures = a.dfeatures; sc.d_xyz = d_xyz;
        for (int l = 0; l < S3G_MAX_LEVELS; ++l)
            for (int k = 0; k < 6; ++k) sc.gplanes[l][k] = l < d.L ? a.gplanes[l][k] : nullptr;
        TimeRowsArgs tr;
        tr.net = a.net; tr.time = time;
        {
            float* tacc = reinterpret_cast<float*>(((uintptr_t)(a.dfeatures + (size_t)P * FD * d.L) + 255) & ~(uintptr_t)255);
            S3G_CUDA(cudaMemsetAsync(tacc, 0, tacc_floats(d) * sizeof(float), stream), "deform bwd memset (time-plane sums)");
            int maxw = 1;
            for (int l = 0; l < S3G_MAX_LEVELS; ++l)
                for (int ax = 0; ax < 3; ++ax) {
                    sc.tacc[l][ax] = l < d.L ? tacc : nullptr;
                    tr.tacc[l][ax] = sc.tacc[l][ax];
                    if (l < d.L) { tacc += (size_t)d.reso[l][ax] * FD; maxw = std::max(maxw, d.reso[l][ax]); }
                }
            for (int l = 0; l < S3G_MAX_LEVELS; ++l)
                for (int k = 0; k < 6; ++k) tr.gplanes[l][k] = sc.gplanes[l][k];
            int dev = 0, sms = 132;
            cudaGetDevice(&dev);
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            const int blocks = std::min((P + 7) / 8, sms * 8);
            if (d.L == 4) hexplane_scatter_kernel<4><<<blocks, 256, 0, stream>>>(sc);
            else hexplane_scatter_kernel<0><<<blocks, 256, 0, stream>>>(sc);
            S3G_CUDA(cudaGetLastError(), "hexplane_scatter launch");
            hexplane_time_rows_kernel<<<dim3((maxw * FD + 255) / 256, 3, d.L), 256, 0, stream>>>(tr);
            S3G_CUDA(cudaGetLastError(), "hexplane_time_rows launch");
        }
    }
    {
        int maxc = 1;
        for (int i = 0; i < r.nseg; ++i) maxc = std::max(maxc, r.seg[i].count);
        deform_reduce_kernel<<<dim3((maxc + 255) / 256, r.nseg), 256, 0, stream>>>(r);
    }
    S3G_CUDA(cudaGetLastError(), "deform_reduce launch");
    return S3G_OK;
}

}  // extern "C"
