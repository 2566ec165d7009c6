// api_deform.cu - extern "C" entry points of the fused HexPlane + decoder stage, forward (see include/s3g_b200.h).
#include "deform_host.cuh"
#include "deform_tc.cuh"

using namespace s3g;

namespace {
// prepared-weight table of the wgmma decoder
void build_tc_table(const DNet& d, TcTable& t, TcPrepArgs* prep) {
    int off = 0;
    auto put = [&](int id, const float* W, int N, int K, int ld) {
        if (!W || K <= 0) { t.off[id] = -1; t.npad[id] = 0; t.k[id] = 0; if (prep) { prep->W[id] = nullptr; prep->n[id] = 0; prep->ld[id] = 0; } return; }
        const int np = (N + 15) & ~15;
        t.off[id] = off; t.npad[id] = np; t.k[id] = K;
        off += 2 * np * K;
        if (prep) { prep->W[id] = W; prep->n[id] = N; prep->ld[id] = ld; }
    };
    for (int id = 0; id < TL_LAYERS; ++id) {
        const float* W = layer_on(d, id) ? layer_w(d, id) : nullptr;
        const int N = kLayers[id].n, K = layer_k(id, d.L);
        if (id == TL_FEAT) {    // the feature layer as two K-halves (deform_tc.cuh: TL_FEAT / TL_FEATB)
            const int KA = K < 64 ? K : 64;
            put(TL_FEAT, W, N, KA, K);
            put(TL_FEATB, W + KA, N, K - KA, K);
        } else {
            put(id, W, N, K, K);
        }
    }
    t.total = off;
}
int deform_grid(int ntiles, int ctas_per_sm = 1) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int g = sms * ctas_per_sm;      // persistent CTAs, as many as are resident at once
    return ntiles < g ? ntiles : g;
}
}  // namespace

extern "C" {

int s3g_deform_forward_save(const s3g_deform_net* net, int P, const float* xyz, const float* scales,
                            const float* rotations, const float* opacity, const float* shs, float time,
                            const float* campos, int sh_degree, float* means3D, float* scales_act,
                            float* rot_act, float* opacity_act, float* colors, float* dx, float* dshs,
                            float* feat, float* features, float* acts, void* workspace, void* stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P < 0) return fail(S3G_ERR_ARG, "deform_forward: P < 0");
    if (P == 0) return S3G_OK;
    struct { DNet net; } a;
    int rc = to_dnet(net, a.net);
    if (rc != S3G_OK) return rc;
    if (!xyz || !scales || !rotations || !opacity || !shs || !campos)
        return fail(S3G_ERR_ARG, "deform_forward: null input");
    if (!means3D || !scales_act || !rot_act || !opacity_act || !colors || !features)
        return fail(S3G_ERR_ARG, "deform_forward: null output");
    if (sh_degree < 0 || sh_degree > 3) return fail(S3G_ERR_ARG, "deform_forward: sh_degree must be 0..3");
    {
        SampleArgs sa;
        sa.net = a.net; sa.P = P; sa.xyz = xyz; sa.time = time; sa.features = features;
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        const int blocks = std::min((P + 7) / 8, sms * 12);
        if (a.net.L == 4) hexplane_sample_kernel<4><<<blocks, 256, 0, stream>>>(sa);
        else hexplane_sample_kernel<0><<<blocks, 256, 0, stream>>>(sa);
        S3G_CUDA(cudaGetLastError(), "hexplane_sample launch");
    }
    {
        // ---- decoder on the warpgroup tensor cores (wgmma) ------------------------------------------
        if (!workspace) return fail(S3G_ERR_ARG, "deform_forward: null workspace");
        DeformTcArgs t;
        t.net = a.net; t.P = P; t.xyz = xyz; t.scales = scales; t.rot = rotations; t.opacity = opacity; t.shs = shs;
        t.campos = campos; t.sh_degree = sh_degree;
        t.o_means = means3D; t.o_scales = scales_act; t.o_rot = rot_act; t.o_opacity = opacity_act; t.o_colors = colors;
        t.o_dx = dx; t.o_dshs = dshs; t.o_feat = feat; t.features = features;
        t.acts = acts;
        t.act_stride = (size_t)((P + 127) / 128) * 128 * 64;
        act_slots(a.net, t.act_slot);
        TcPrepArgs pp;
        build_tc_table(a.net, t.tab, &pp);
        pp.tab = t.tab;
        pp.dst = reinterpret_cast<float*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
        t.wprep = pp.dst;
        tc_prep_weights_kernel<<<dim3(8, TL_COUNT), 256, 0, stream>>>(pp);
        S3G_CUDA(cudaGetLastError(), "tc_prep_weights launch");
        // operands [128][64] hi + lo (lo doubles as the output staging tile), weights [64][64] hi + lo: 96 KB, two CTAs per SM
        const size_t smem = (size_t)(2 * TCM * 64 + 2 * 64 * 64) * sizeof(float);
        S3G_CUDA(cudaFuncSetAttribute(deform_forward_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "deform tc smem attr");
        const int ntiles = (P + TCM - 1) / TCM;
        deform_forward_tc_kernel<<<deform_grid(ntiles, 2), TCM, smem, stream>>>(t);
    }
    S3G_CUDA(cudaGetLastError(), "deform_forward launch");
    return S3G_OK;
}


size_t s3g_deform_forward_workspace_bytes(const s3g_deform_net* net) {
    DNet d;
    if (to_dnet(net, d) != S3G_OK) return 0;
    TcTable t;
    build_tc_table(d, t, nullptr);
    return (size_t)t.total * sizeof(float) + 512;
}

}  // extern "C"
