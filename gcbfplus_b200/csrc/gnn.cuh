// gnn.cuh -- non-GEMM kernels of the GNN (edge features + first message layer, attention
// softmax + aggregation, output head) and the workspace layout shared by forward / backward.
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

// ---- edge features + message layer 1: X1 = relu(feat @ W1[:ed] + W1[ed + sender_type] + W1[ed+3+2] + b1)
// one warp per edge (grid-stride); lane owns 8 output columns.
template <int KIND>
__global__ void __launch_bounds__(256)
edge_l1_kernel(const gcbf_env_desc d, const float* __restrict__ W1, const float* __restrict__ b1,
               const float* __restrict__ agent, const float* __restrict__ goal, const float* __restrict__ hits,
               const int32_t* __restrict__ edge_recv, const int32_t* __restrict__ edge_src,
               const int32_t* __restrict__ counters, const int clip_all, float* __restrict__ feat_out,
               float* __restrict__ X1) {
    using T = EnvTraits<KIND>;
    constexpr int ED = T::ED, SD = T::SD;
    __shared__ __align__(16) float sW[ED][256];
    __shared__ __align__(16) float sB[3][256];  // [hit, goal, agent] sender one-hot rows + receiver row + bias
    for (int i = threadIdx.x; i < ED * 256; i += blockDim.x) sW[i / 256][i % 256] = W1[i];
    for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) {
        const int t = i / 256, c = i % 256;
        sB[t][c] = W1[(ED + t) * 256 + c] + W1[(ED + 3 + 2) * 256 + c] + b1[c];
    }
    __syncthreads();
    const int nE = min(counters[0], d.edge_cap);
    const int A = d.n_graphs * d.n_agents;
    const int lane = threadIdx.x & 31;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    for (int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < nE; e += warps_total) {
        const int a = min(max(edge_recv[e], 0), A - 1);
        int code = edge_src[e];
        code = min(code, A - 1);
        float er[ED], es[ED], f[ED], coef, nrm;
        edge_state_dev<KIND>(agent + (size_t)a * SD, er);
        sender_state_dev<KIND>(code, a, d.n_hits, agent, goal, hits, es);
        edge_feat_dev<KIND>(er, es, clip_all || code == -1, d.comm_radius, f, &coef, &nrm);
        const int t = (code >= 0) ? 2 : ((code == -1) ? 1 : 0);
        if (lane < ED) feat_out[(size_t)e * FEAT_LD + lane] = f[lane];
        float y[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) y[j] = sB[t][lane * 8 + j];
#pragma unroll
        for (int c = 0; c < ED; ++c) {
#pragma unroll
            for (int j = 0; j < 8; ++j) y[j] = fmaf(f[c], sW[c][lane * 8 + j], y[j]);
        }
        float4* dst = reinterpret_cast<float4*>(X1 + (size_t)e * 256 + lane * 8);
        dst[0] = make_float4(fmaxf(y[0], 0.f), fmaxf(y[1], 0.f), fmaxf(y[2], 0.f), fmaxf(y[3], 0.f));
        dst[1] = make_float4(fmaxf(y[4], 0.f), fmaxf(y[5], 0.f), fmaxf(y[6], 0.f), fmaxf(y[7], 0.f));
    }
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

// ---- gate logit + segment softmax + weighted aggregation (gnn.py:64-72); warp per receiver.
// gate = G2 @ a3 + ba3 ; att = softmax over the receiver's edges ; AG[a] = sum att * MSG.
static __global__ void __launch_bounds__(256)
attn_aggregate_kernel(const int A, const int edge_cap, const float* __restrict__ G2, const float* __restrict__ MSG,
                      const float* __restrict__ a3, const float* __restrict__ ba3,
                      const int32_t* __restrict__ row_start, const int32_t* __restrict__ row_deg,
                      float* __restrict__ ATT, float* __restrict__ AG, int32_t* __restrict__ zero_counter = nullptr) {
    // G2 == nullptr (inference): ATT already holds the gate logits (written by tc::edge_chain_kernel) and is
    // left as it is.  Otherwise (training) the gate logits are computed here and ATT receives the attention weights
    // that the backward pass reads.
    // zero_counter (rollout step): edge counter of the NEXT graph, cleared here so that no memset node sits in the
    // per-step kernel chain (the graph build two kernels later accumulates into it)
    if (zero_counter && blockIdx.x == 0 && threadIdx.x == 0) zero_counter[0] = 0;
    const int lane = threadIdx.x & 31;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    const float4 w = G2 ? *reinterpret_cast<const float4*>(a3 + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float bias = G2 ? ba3[0] : 0.f;
    for (int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; a < A; a += warps_total) {
        const int rs = row_start[a];
        int rd = row_deg[a];
        if (rs < 0 || rs + rd > edge_cap) rd = 0;
        if (!G2) {
            *reinterpret_cast<float4*>(AG + (size_t)a * 128 + lane * 4) = aggregate_logits(rs, rd, ATT, MSG, lane);
            continue;
        }
        if (rd <= 4) {
            // training fast path: the gate rows and the message rows of all (<= 4) edges are requested up front and the
            // 4 dot products are reduced together; same arithmetic order as the general path below
            float sg[4];
            float4 mv[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int e = rs + min(q, max(rd - 1, 0));
                const bool on = q < rd;
                const float4 g = on ? *reinterpret_cast<const float4*>(G2 + (size_t)e * 128 + lane * 4)
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
                mv[q] = on ? *reinterpret_cast<const float4*>(MSG + (size_t)e * 128 + lane * 4)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
                sg[q] = g.x * w.x + g.y * w.y + g.z * w.z + g.w * w.w;
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1)
#pragma unroll
                for (int q = 0; q < 4; ++q) sg[q] += __shfl_xor_sync(0xffffffffu, sg[q], off);
            float mx = -INFINITY;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                sg[q] = (q < rd) ? sg[q] + bias : -INFINITY;
                mx = fmaxf(mx, sg[q]);
            }
            float den = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (q < rd) den += expf(sg[q] - mx);
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (q < rd) {
                    const float att = expf(sg[q] - mx) / den;
                    acc.x = fmaf(att, mv[q].x, acc.x);
                    acc.y = fmaf(att, mv[q].y, acc.y);
                    acc.z = fmaf(att, mv[q].z, acc.z);
                    acc.w = fmaf(att, mv[q].w, acc.w);
                    if (lane == 0) ATT[rs + q] = att;
                }
            }
            *reinterpret_cast<float4*>(AG + (size_t)a * 128 + lane * 4) = acc;
            continue;
        }
        float mx = -INFINITY;
        for (int e = rs; e < rs + rd; ++e) {
            const float4 g = *reinterpret_cast<const float4*>(G2 + (size_t)e * 128 + lane * 4);
            float s = g.x * w.x + g.y * w.y + g.z * w.z + g.w * w.w;
            s = warp_sum(s) + bias;
            if (lane == 0) ATT[e] = s;
            mx = fmaxf(mx, s);
        }
        __syncwarp();
        float den = 0.f;
        for (int e = rs; e < rs + rd; ++e) den += expf(ATT[e] - mx);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int e = rs; e < rs + rd; ++e) {
            const float att = expf(ATT[e] - mx) / den;
            const float4 m = *reinterpret_cast<const float4*>(MSG + (size_t)e * 128 + lane * 4);
            acc.x = fmaf(att, m.x, acc.x);
            acc.y = fmaf(att, m.y, acc.y);
            acc.z = fmaf(att, m.z, acc.z);
            acc.w = fmaf(att, m.w, acc.w);
            __syncwarp();
            if (lane == 0) ATT[e] = att;
        }
        *reinterpret_cast<float4*>(AG + (size_t)a * 128 + lane * 4) = acc;
    }
}

// ---- output layer pre-activations z[a][0..3] = H @ W[256, nout] (no bias / tanh): SIMT-path producer of the
// policy tail's input (the tensor-core path gets it from the EPI_RELU_DOTN epilogue).  Warp per agent.
static __global__ void __launch_bounds__(256)
head_z_kernel(const int A, const int nout, const float* __restrict__ H, const float* __restrict__ W,
              float* __restrict__ z) {
    const int lane = threadIdx.x & 31;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    for (int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; a < A; a += warps_total) {
        const float4 h0 = *reinterpret_cast<const float4*>(H + (size_t)a * 256 + lane * 8);
        const float4 h1 = *reinterpret_cast<const float4*>(H + (size_t)a * 256 + lane * 8 + 4);
        const float hv[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
        float out[4] = {0.f, 0.f, 0.f, 0.f};
        for (int j = 0; j < nout; ++j) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) s = fmaf(hv[k], W[(lane * 8 + k) * nout + j], s);
            out[j] = warp_sum(s);
        }
        if (lane == 0) *reinterpret_cast<float4*>(z + (size_t)a * 4) = make_float4(out[0], out[1], out[2], out[3]);
    }
}

// ---- output head: out = tanh(H2 @ W[256, nout] + b); warp per agent.
static __global__ void __launch_bounds__(256)
head_out_kernel(const int A, const int nout, const float* __restrict__ H2, const float* __restrict__ W,
                const float* __restrict__ b, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    float wl[8][4];
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) wl[k][j] = (j < nout) ? W[(lane * 8 + k) * nout + j] : 0.f;
    // four agents per iteration: all eight row loads are in flight before the first reduction (latency-bound loop)
    for (int a0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; a0 < A; a0 += 4 * warps_total) {
        float4 hq[4][2];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int a = min(a0 + q * warps_total, A - 1);
            hq[q][0] = *reinterpret_cast<const float4*>(H2 + (size_t)a * 256 + lane * 8);
            hq[q][1] = *reinterpret_cast<const float4*>(H2 + (size_t)a * 256 + lane * 8 + 4);
        }
        float sv[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float hv[8] = {hq[q][0].x, hq[q][0].y, hq[q][0].z, hq[q][0].w, hq[q][1].x, hq[q][1].y, hq[q][1].z, hq[q][1].w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float s = 0.f;
#pragma unroll
                for (int k = 0; k < 8; ++k) s = fmaf(hv[k], wl[k][j], s);
                sv[q][j] = s;
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1)
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int j = 0; j < 4; ++j) sv[q][j] += __shfl_xor_sync(0xffffffffu, sv[q][j], off);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int a = a0 + q * warps_total;
            if (a < A && lane < nout) {
                float s = sv[q][0];
                if (lane == 1) s = sv[q][1];
                if (lane == 2) s = sv[q][2];
                if (lane == 3) s = sv[q][3];
                out[(size_t)a * nout + lane] = tanhf(s + b[lane]);
            }
        }
    }
}

}  // namespace gcbf
