// deform_host.cuh - host-side helpers shared by the forward and backward translation units of the fused
// HexPlane + decoder stage (api_deform.cu, api_deform_bwd.cu).
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <initializer_list>

#include "api_common.cuh"
#include "common.cuh"
#include "deform.cuh"

namespace s3g {
inline int fail(int code, const char* what, cudaError_t e = cudaSuccess) { return api_fail(code, what, e); }

// The decoder's Linear layers, one row per TL_* id: where the layer's weight [n][k] and bias [n] pointers sit in
// s3g_deform_net, s3g_deform_net_grads and DNet, where GradOff keeps the offsets of their gradients, the output
// width n, and the head the layer belongs to, as the id of that head's first layer (a head is on when that layer's
// weight is set).  The input width k is 64, or 32 L for feature_out (layer_k).
struct DeformLayer {
    int id;
    const float* s3g_deform_net::*w;
    const float* s3g_deform_net::*b;
    float* s3g_deform_net_grads::*gw;
    float* s3g_deform_net_grads::*gb;
    // byte offsets: a pointer-to-member cannot name a Head2 field of DNet or an array element of GradOff
    size_t dw, db;       // offsetof(DNet, ...)
    size_t ow, ob;       // offsetof(GradOff, ...)
    int n;
    int head;
};
#define S3G_LAYER(id, f, dw, db, ow, ob, n, head)                                                                     \
    DeformLayer{id, &s3g_deform_net::w_##f, &s3g_deform_net::b_##f, &s3g_deform_net_grads::w_##f,                    \
                &s3g_deform_net_grads::b_##f, offsetof(DNet, dw), offsetof(DNet, db), offsetof(GradOff, ow),         \
                offsetof(GradOff, ob), n, head}
constexpr int TL_LAYERS = TL_FEATB;
constexpr DeformLayer kLayers[TL_LAYERS] = {
    S3G_LAYER(TL_FEAT, feat, w_feat, b_feat, w_feat, b_feat, 64, TL_FEAT),
    S3G_LAYER(TL_POS1, pos1, pos.w1, pos.b1, pos[0], pos[1], 64, TL_POS1),
    S3G_LAYER(TL_POS2, pos2, pos.w2, pos.b2, pos[2], pos[3], 3, TL_POS1),
    S3G_LAYER(TL_SCL1, scl1, scl.w1, scl.b1, scl[0], scl[1], 64, TL_SCL1),
    S3G_LAYER(TL_SCL2, scl2, scl.w2, scl.b2, scl[2], scl[3], 3, TL_SCL1),
    S3G_LAYER(TL_ROT1, rot1, rot.w1, rot.b1, rot[0], rot[1], 64, TL_ROT1),
    S3G_LAYER(TL_ROT2, rot2, rot.w2, rot.b2, rot[2], rot[3], 4, TL_ROT1),
    S3G_LAYER(TL_OPA1, opa1, opa.w1, opa.b1, opa[0], opa[1], 64, TL_OPA1),
    S3G_LAYER(TL_OPA2, opa2, opa.w2, opa.b2, opa[2], opa[3], 1, TL_OPA1),
    S3G_LAYER(TL_SHS1, shs1, shs.w1, shs.b1, shs[0], shs[1], 64, TL_SHS1),
    S3G_LAYER(TL_SHS2, shs2, shs.w2, shs.b2, shs[2], shs[3], 48, TL_SHS1),
    S3G_LAYER(TL_D0, dino0, w_d0, b_d0, d0w, d0b, 64, TL_D0),
    S3G_LAYER(TL_D2, dino2, w_d2, b_d2, d2w, d2b, 64, TL_D0),
    S3G_LAYER(TL_D4, dino4, w_d4, b_d4, d4w, d4b, 3, TL_D0),
};
#undef S3G_LAYER
constexpr bool rows_in_id_order() {
    for (int i = 0; i < TL_LAYERS; ++i)
        if (kLayers[i].id != i) return false;
    return true;
}
static_assert(rows_in_id_order(), "kLayers: row i describes layer i");

// a layer's pointer in DNet, or its gradient offset in GradOff, at a byte offset from the table
inline const float*& dnet_ptr(DNet& d, size_t off) { return *reinterpret_cast<const float**>(reinterpret_cast<char*>(&d) + off); }
inline const float* dnet_ptr(const DNet& d, size_t off) {
    return *reinterpret_cast<const float* const*>(reinterpret_cast<const char*>(&d) + off);
}
inline int& grad_off(GradOff& o, size_t off) { return *reinterpret_cast<int*>(reinterpret_cast<char*>(&o) + off); }

inline const float* layer_w(const DNet& d, int id) { return dnet_ptr(d, kLayers[id].dw); }
inline bool layer_on(const DNet& d, int id) { return layer_w(d, kLayers[id].head) != nullptr; }
inline int layer_k(int id, int L) { return id == TL_FEAT ? FD * L : HWID; }

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
    for (const DeformLayer& l : kLayers) {
        if (n->*kLayers[l.head].w && !(n->*l.w && n->*l.b))
            return fail(S3G_ERR_ARG, l.head == TL_D0 ? "deform: incomplete dino head" : "deform: incomplete head");
        dnet_ptr(d, l.dw) = n->*l.w;
        dnet_ptr(d, l.db) = n->*l.b;
    }
    return S3G_OK;
}

// weight matrices in the order one backward tile consumes them (see WPipe).  The backward reads the hidden
// activations the forward stored, so only the push-back products (and the 48-wide SH output layer, whose result is
// not stored) use weights.
inline void build_wseq(const DNet& d, WSeq& q) {
    q.count = 0;
    auto add = [&](int id) {
        q.W[q.count] = layer_w(d, id); q.N[q.count] = (short)kLayers[id].n; q.K[q.count] = (short)layer_k(id, d.L);
        ++q.count;
    };
    for (int id : {TL_POS1, TL_SCL1, TL_ROT1, TL_OPA1})
        if (layer_on(d, id)) add(id);
    if (layer_on(d, TL_SHS1)) { add(TL_SHS2); add(TL_SHS2); add(TL_SHS1); }
    if (layer_on(d, TL_D0)) { add(TL_D2); add(TL_D0); }
    add(TL_FEAT);
}

// Hidden activations the wgmma forward can keep for the backward: [slot][P][64] floats, one slot per enabled kind.
// Kind 0 is h; kinds 1..7 are the inputs of the layers that are not the first of their head, in TL_* order: the
// hidden layer of the pos, scl, rot, opa and shs heads, then the dino head's two.  Returns the slot count and fills
// slot[kind] (-1 = absent).
constexpr int ACT_KINDS = 8;      // DeformTcArgs::act_slot, DeformBwdArgs::act_slot
static_assert([] { int c = 1; for (const DeformLayer& l : kLayers) c += l.head != l.id; return c; }() == ACT_KINDS,
              "one kept activation kind per layer that is not the first of its head, plus h");
inline int act_slots(const DNet& d, int (&slot)[ACT_KINDS]) {
    int kind = 0, n = 0;
    slot[kind++] = n++;     // h
    for (int id = 0; id < TL_LAYERS; ++id)
        if (kLayers[id].head != id) slot[kind++] = layer_on(d, id) ? n++ : -1;
    return n;
}

}  // namespace s3g
