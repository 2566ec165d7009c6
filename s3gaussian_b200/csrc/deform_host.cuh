// deform_host.cuh - host-side helpers shared by the forward and backward translation units of the fused
// HexPlane + decoder stage (api_deform.cu, api_deform_bwd.cu).
#pragma once
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>

#include "api_common.cuh"
#include "common.cuh"
#include "deform.cuh"

namespace s3g {
inline int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return api_fail(code, what, e); }

inline int to_dnet(const s3g_deform_net* n, DNet& d) {
    if (!n) return fail(S3G_ERR_ARG, "deform: null net");
    if (n->feat_dim != FD) return fail(S3G_ERR_UNSUPPORTED, "deform: output_coordinate_dim must be 32");
    if (n->width != HWID) return fail(S3G_ERR_UNSUPPORTED, "deform: net_width must be 64");
    // (8 levels were accepted up to round 2 but could never launch: 64-row tiles of 256 features need 235 KB of
    //  shared memory.  The reference's own configs use 4: multires [1,2,4,8], arguments/__init__.py:215.)
    if (n->num_levels < 1 || n->num_levels > 4)
        return fail(S3G_ERR_UNSUPPORTED, "deform: number of HexPlane levels (len(multires)) must be 1..4");
    d.L = n->num_levels;
    for (int l = 0; l < d.L; ++l) {
        for (int c = 0; c < 4; ++c) {
            d.reso[l][c] = n->reso[l][c];
            if (d.reso[l][c] < 2) return fail(S3G_ERR_ARG, "deform: plane resolution < 2");
        }
        for (int k = 0; k < 6; ++k) {
            d.planes[l][k] = n->planes[l][k];
            if (!d.planes[l][k]) return fail(S3G_ERR_ARG, "deform: null plane");
        }
    }
    for (int c = 0; c < 3; ++c) {
        d.aabb0[c] = n->aabb[c];
        d.inv_span2[c] = 2.0f / (n->aabb[3 + c] - n->aabb[c]);   // hexplane.py:19-20
    }
    if (!n->w_feat || !n->b_feat) return fail(S3G_ERR_ARG, "deform: null feature_out");
    d.w_feat = n->w_feat; d.b_feat = n->b_feat;
    d.pos = {n->w_pos1, n->b_pos1, n->w_pos2, n->b_pos2};
    d.scl = {n->w_scl1, n->b_scl1, n->w_scl2, n->b_scl2};
    d.rot = {n->w_rot1, n->b_rot1, n->w_rot2, n->b_rot2};
    d.opa = {n->w_opa1, n->b_opa1, n->w_opa2, n->b_opa2};
    d.shs = {n->w_shs1, n->b_shs1, n->w_shs2, n->b_shs2};
    d.w_d0 = n->w_dino0; d.b_d0 = n->b_dino0; d.w_d2 = n->w_dino2; d.b_d2 = n->b_dino2;
    d.w_d4 = n->w_dino4; d.b_d4 = n->b_dino4;
    const Head2* hs[5] = {&d.pos, &d.scl, &d.rot, &d.opa, &d.shs};
    for (const Head2* h : hs)
        if (h->w1 && !(h->b1 && h->w2 && h->b2)) return fail(S3G_ERR_ARG, "deform: incomplete head");
    if (d.w_d0 && !(d.b_d0 && d.w_d2 && d.b_d2 && d.w_d4 && d.b_d4))
        return fail(S3G_ERR_ARG, "deform: incomplete dino head");
    return S3G_OK;
}
// weight matrices in the order one backward tile consumes them (see WPipe).  The backward reads the hidden
// activations the forward stored, so only the push-back products (and the 48-wide SH output layer, whose result is
// not stored) use weights.
inline void build_wseq(const DNet& d, WSeq& q) {
    q.count = 0;
    auto add = [&](const float* W, int N, int K) { q.W[q.count] = W; q.N[q.count] = (short)N; q.K[q.count] = (short)K; ++q.count; };
    const Head2* small[4] = {&d.pos, &d.scl, &d.rot, &d.opa};
    for (const Head2* h : small)
        if (h->w1) add(h->w1, 64, 64);
    if (d.shs.w1) { add(d.shs.w2, 48, 64); add(d.shs.w2, 48, 64); add(d.shs.w1, 64, 64); }
    if (d.w_d0) { add(d.w_d2, 64, 64); add(d.w_d0, 64, 64); }
    add(d.w_feat, 64, FD * d.L);
}

// Hidden activations the wgmma forward can keep for the backward: [slot][P][64] floats, one slot per enabled
// kind in this order.  Returns the slot count and fills slot[kind] (-1 = absent).
enum { AK_H = 0, AK_POS, AK_SCL, AK_ROT, AK_OPA, AK_SHS, AK_D0, AK_D2, AK_COUNT };
inline int act_slots(const DNet& d, int (&slot)[AK_COUNT]) {
    for (int i = 0; i < AK_COUNT; ++i) slot[i] = -1;
    int n = 0;
    slot[AK_H] = n++;
    if (d.pos.w1) slot[AK_POS] = n++;
    if (d.scl.w1) slot[AK_SCL] = n++;
    if (d.rot.w1) slot[AK_ROT] = n++;
    if (d.opa.w1) slot[AK_OPA] = n++;
    if (d.shs.w1) slot[AK_SHS] = n++;
    if (d.w_d0) { slot[AK_D0] = n++; slot[AK_D2] = n++; }
    return n;
}

}  // namespace s3g
