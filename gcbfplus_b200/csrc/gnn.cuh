// gnn.cuh -- device functions of the non-GEMM GNN kernels (edge features, segment softmax + aggregation) that gnn.cu's
// kernels share with the train step and the persistent rollout kernel, and the workspace layouts shared by forward /
// backward.
//
// Replaces gcbfplus/nn/gnn.py:44-75 (GNNLayer message/aggregate/update), nn/mlp.py:6-30,
// algo/module/cbf.py:12-21, algo/module/policy.py:63-73, and the edge-feature part of
// env/double_integrator.py:223-264 / 275-286 (edge_blocks / add_edge_feats) and twins.
#pragma once
#include "common.cuh"

namespace gcbf {

constexpr int FEAT_LD = 8;  // per-edge feature row stride (ed <= 6)

// Saved activations of one network forward (float offsets into the workspace).
struct GnnWs {
    int64_t feat, x1, x2, msg, g1, g2, att, ag, v1, v2, v3, h1, h2, total;
};
inline GnnWs make_ws(int64_t cap, int64_t A) {
    GnnWs w;
    WsSlots S{8};   // 32-byte slots: 256-bit epilogue stores
    w.feat = S.take(cap * FEAT_LD);
    w.x1 = S.take(cap * 256);
    w.x2 = S.take(cap * 256);
    w.msg = S.take(cap * 128);
    w.g1 = S.take(cap * 128);
    w.g2 = S.take(cap * 128);
    w.att = S.take(cap);
    w.ag = S.take(A * 128);
    w.v1 = S.take(A * 256);
    w.v2 = S.take(A * 256);
    w.v3 = S.take(A * 128);
    w.h1 = S.take(A * 256);
    w.h2 = S.take(A * 256);
    w.total = S.off;
    return w;
}

// Folded inference weights (gcbf_prepare_infer, gnn.cu): float offsets inside the blob.
struct InferLayout {
    int w23, b23, a23, c23, uh, buh, ho, bho;          // folded fp32 weights (the gradient of the folded train step uses
                                                       // the same offsets: [0, t_w23) floats)
    int t_w23, t_a1, t_u1, t_uh;                       // transposed tf32 planes: hi at t_x, lo at t_x + size
    int q_u12, b_u12;                                  // U2 U3 and bu2 U3 + bu3 (needed to un-fold the gradient of uh)
    int p_w23, p_a1, p_u1, p_uh;                       // straight tf32 planes (backward-data operands): hi, lo at + size
    int total;
};
inline InferLayout make_infer_layout(int out_dim) {
    InferLayout I;
    WsSlots S{4};
    I.w23 = S.take(256 * 128);
    I.b23 = S.take(128);
    I.a23 = S.take(128);
    I.c23 = S.take(4);
    I.uh = S.take(256 * 256);
    I.buh = S.take(256);
    I.ho = S.take(256 * out_dim);
    I.bho = S.take(4);
    I.t_w23 = S.take(2 * 128 * 256);
    I.t_a1 = S.take(2 * 128 * 128);
    I.t_u1 = S.take(2 * 256 * 128);
    I.t_uh = S.take(2 * 256 * 256);
    I.q_u12 = S.take(256 * 128);
    I.b_u12 = S.take(128);
    I.p_w23 = S.take(2 * 256 * 128);
    I.p_a1 = S.take(2 * 128 * 128);
    I.p_u1 = S.take(2 * 128 * 256);
    I.p_uh = S.take(2 * 256 * 256);
    I.total = S.off;
    return I;
}

// edge_state (dubins_car.py:260-264: (x, y, v cos th, v sin th); identity otherwise)
template <int KIND>
__device__ __forceinline__ void edge_state_dev(const float* s, float* es) {
    constexpr int SD = EnvTraits<KIND>::SD;
    if (KIND == GCBF_ENV_DUBINS_CAR) {
        es[0] = s[0];
        es[1] = s[1];
        es[2] = s[3] * cosf(s[2]);
        es[3] = s[3] * sinf(s[2]);
    } else {
#pragma unroll
        for (int c = 0; c < SD; ++c) es[c] = s[c];
    }
}

// ds = des (d edge_state / d s): the DubinsCar (x, y, v cos th, v sin th) Jacobian, the identity otherwise
template <int KIND>
__device__ __forceinline__ void edge_state_vjp_dev(const float* s, const float* des, float* ds) {
    constexpr int SD = EnvTraits<KIND>::SD;
    if (KIND == GCBF_ENV_DUBINS_CAR) {
        const float c = cosf(s[2]), sn = sinf(s[2]);
        ds[0] = des[0];
        ds[1] = des[1];
        ds[2] = des[2] * (-s[3] * sn) + des[3] * (s[3] * c);
        ds[3] = des[2] * c + des[3] * sn;
    } else {
#pragma unroll
        for (int c = 0; c < SD; ++c) ds[c] = des[c];
    }
}

// Sender edge-state for an edge code (see gcbf_b200.h): agent / goal / hit node.
template <int KIND>
__device__ __forceinline__ void sender_state_dev(int code, int a, int R, const float* agent, const float* goal,
                                                 const float* hits, float* es) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, PD = T::PD, ED = T::ED;
    if (code >= 0) {
        edge_state_dev<KIND>(agent + (size_t)code * SD, es);
    } else if (code == -1) {
        edge_state_dev<KIND>(goal + (size_t)a * SD, es);
    } else {
        const int k = min(-2 - code, R - 1);
        const float* h = hits + ((size_t)a * R + k) * PD;
#pragma unroll
        for (int c = 0; c < ED; ++c) es[c] = (c < PD) ? h[c] : 0.f;
    }
}

// feat = es(recv) - es(send), position part norm-clipped when `clip`
// (double_integrator.py:239-244 / 279-284).  Returns the clip coefficient and raw norm.
template <int KIND>
__device__ __forceinline__ void edge_feat_dev(const float* er, const float* es, bool clip, float rc, float* feat,
                                              float* coef_out, float* nrm_out) {
    using T = EnvTraits<KIND>;
    constexpr int PD = T::PD, ED = T::ED;
    // explicit fused multiply-adds: the same bits whether the translation unit is compiled with -fmad=true (gnn.cu,
    // train.cu) or -fmad=false (rollout_persist.cu, which shares this function with the bit-exact geometry code)
    float sq = 0.f;
#pragma unroll
    for (int c = 0; c < ED; ++c) {
        feat[c] = er[c] - es[c];
        if (c < PD) sq = (c == 0) ? feat[c] * feat[c] : fmaf(feat[c], feat[c], sq);
    }
    float coef = 1.f;
    const float nrm = sqrtf(1e-6f + sq);
    if (clip && nrm > rc) coef = rc / fmaxf(nrm, rc);
    if (clip) {
#pragma unroll
        for (int c = 0; c < PD; ++c) feat[c] *= coef;
    }
    *coef_out = coef;
    *nrm_out = nrm;
}

// ---- segment softmax of given gate logits + weighted aggregation (gnn.py:64-72) for one receiver, one warp: the
// receiver's edge rows are [rs, rs + rd) of ATT (logits) and MSG ([.][128] messages); returns this lane's 4 columns
// of AG.  Shared by attn_aggregate_kernel (inference) and the persistent rollout kernel.
__device__ __forceinline__ float4 aggregate_logits(int rs, int rd, const float* ATT, const float* MSG, int lane) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rd <= 4) {
        // fast path (typical degree: goal + 0..3 neighbours / hits): every logit and message row is requested before
        // anything is consumed, so the warp waits for ONE round trip to L2 instead of three
        float lg[4];
        float4 mv[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int e = rs + min(q, max(rd - 1, 0));
            lg[q] = (q < rd) ? ATT[e] : -INFINITY;
            mv[q] = (q < rd) ? *reinterpret_cast<const float4*>(MSG + (size_t)e * 128 + lane * 4)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float mx = -INFINITY;
#pragma unroll
        for (int q = 0; q < 4; ++q) mx = fmaxf(mx, lg[q]);      // same left-to-right order as the general path
        float den = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (q < rd) den += expf(lg[q] - mx);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (q < rd) {
                const float att = expf(lg[q] - mx) / den;
                acc.x = fmaf(att, mv[q].x, acc.x);
                acc.y = fmaf(att, mv[q].y, acc.y);
                acc.z = fmaf(att, mv[q].z, acc.z);
                acc.w = fmaf(att, mv[q].w, acc.w);
            }
        }
        return acc;
    }
    float mx = -INFINITY;
    for (int e = rs; e < rs + rd; ++e) mx = fmaxf(mx, ATT[e]);
    float den = 0.f;
    for (int e = rs; e < rs + rd; ++e) den += expf(ATT[e] - mx);
    for (int e = rs; e < rs + rd; ++e) {
        const float att = expf(ATT[e] - mx) / den;
        const float4 m = *reinterpret_cast<const float4*>(MSG + (size_t)e * 128 + lane * 4);
        acc.x = fmaf(att, m.x, acc.x);
        acc.y = fmaf(att, m.y, acc.y);
        acc.z = fmaf(att, m.z, acc.z);
        acc.w = fmaf(att, m.w, acc.w);
    }
    return acc;
}

}  // namespace gcbf
