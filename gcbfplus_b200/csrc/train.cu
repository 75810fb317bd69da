// train.cu -- the GCBF+ train step: three GNN forwards with saved activations, the four
// losses, hand-written backward (dW via split-M GEMMs, dX through the edge features, the Euler
// step and the action clip back into the actor), global-norm clip + AdamW + apply_if_finite,
// and the target-network polyak update.  Every sum that spans CTAs is taken in a fixed order (per-CTA partials in the
// workspace, then partial_sum_kernel; per-edge input gradients gathered per agent), so the step is bit-identical from
// run to run for the same inputs on the same GPU model.  On the tensor-core path the step runs on the folded
// network (gnn_backward_folded / unfold_jobs below: 4 GEMMs per pass and direction instead of
// 9-10, same gradient); the strict-fp32 SIMT path runs the layer-by-layer step.
//
// Replaces gcbfplus/algo/gcbf_plus.py:354-447 (update_inner / get_loss / value_and_grad),
// trainer/utils.py:62-75 (compute_norm_and_clip), optax.adamw + optax.apply_if_finite
// (gcbf_plus.py:109-110,127-128) and gcbf_plus.py:188-191 (update_tgt).
#include "gemm.cuh"
#include "gemm_tc.cuh"
#include "geometry_dev.cuh"
#include "gnn.cuh"
#include "translayout.cuh"
#include "smalljobs.cuh"
#include "internal.cuh"

namespace gcbf {

// ------------------------------------------------------------------------------------ act + dynamics (forward)
// a = 2 pi + u_ref ; u = clip_action(a) ; x' = agent_step_euler(x, u)   (gcbf_plus.py:386-391)
template <int KIND>
__global__ void act_dyn_kernel(const gcbf_env_desc d, const float* __restrict__ agent, const float* __restrict__ goal,
                               const float* __restrict__ pi, float* __restrict__ action, float* __restrict__ xnext) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= d.n_graphs * d.n_agents) return;
    float x[SD], gl[SD], ur[NU], act[NU], xn[SD];
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        x[c] = agent[(size_t)a * SD + c];
        gl[c] = goal[(size_t)a * SD + c];
    }
    u_ref_dev<KIND>(d, x, gl, ur);
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        act[c] = 2.f * pi[(size_t)a * NU + c] + ur[c];
        action[(size_t)a * NU + c] = act[c];
    }
    step_agent<KIND>(d, x, gl, act, ur, true, xn);
#pragma unroll
    for (int c = 0; c < SD; ++c) xnext[(size_t)a * SD + c] = xn[c];
}

// ------------------------------------------------------------------------------------ losses (gcbf_plus.py:362-431)
// stats (local numerators): 0 sum relu(h+eps)[unsafe]  1 sum relu(-h+eps)[safe]  2 sum max_val_h_dot
// 3 sum ||a-u_qp||^2  4 #(h<0 & unsafe)  5 #(h>0 & safe)  6 #(h_dot + alpha h > 0)  7 n_unsafe  8 n_safe  9 n_agents
// denoms (global): 0 n_unsafe  1 n_safe  2 n_agents
struct TrainHP {
    float alpha, eps, c_action, c_unsafe, c_safe, c_hdot, dt_inv;
};

template <int NU>
__global__ void __launch_bounds__(256)
loss_kernel(const int A, const TrainHP hp, const float* __restrict__ h, const float* __restrict__ h_next,
            const uint8_t* __restrict__ safe_m, const uint8_t* __restrict__ unsafe_m, const float* __restrict__ action,
            const float* __restrict__ u_qp, const float* __restrict__ denoms, float* __restrict__ dh,
            float* __restrict__ dh_next, float* __restrict__ da, float* __restrict__ labelled,
            float* __restrict__ part) {
    // part[blockIdx.x][10]: this CTA's stats, reduced in CTA order by partial_sum_kernel
    __shared__ float red[10][8];
    float loc[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) loc[i] = 0.f;
    const float inv_unsafe = 1.f / (denoms[0] + 1e-6f);
    const float inv_safe = 1.f / (denoms[1] + 1e-6f);
    const float inv_n = 1.f / denoms[2];
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < A; a += gridDim.x * blockDim.x) {
        const float hv = h[a], hn = h_next[a];
        const bool us = unsafe_m[a] != 0, sf = safe_m[a] != 0;
        const bool lab = us || sf;
        float g = 0.f;
        if (us) {
            const float v = hv + hp.eps;
            if (v > 0.f) { loc[0] += v; g += hp.c_unsafe * inv_unsafe; }
            if (hv < 0.f) loc[4] += 1.f;
            loc[7] += 1.f;
        }
        if (sf) {
            const float v = -hv + hp.eps;
            if (v > 0.f) { loc[1] += v; g -= hp.c_safe * inv_safe; }
            if (hv > 0.f) loc[5] += 1.f;
            loc[8] += 1.f;
        }
        const float h_dot = (hn - hv) * hp.dt_inv;
        const float v = -h_dot - hp.alpha * hv + hp.eps;
        float gn = 0.f;
        if (v > 0.f) {
            loc[2] += v;
            const float w = hp.c_hdot * inv_n;
            gn = -hp.dt_inv * w;                                  // d/dh'
            g += (lab ? (hp.dt_inv - hp.alpha) : (-hp.alpha)) * w;  // d/dh (h inside h_dot detached if unlabelled)
        }
        if (h_dot + hp.alpha * hv > 0.f) loc[6] += 1.f;
        loc[9] += 1.f;
        dh[a] = g;
        dh_next[a] = gn;
        labelled[a] = lab ? 1.f : 0.f;
        float sq = 0.f;
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            const float df = action[(size_t)a * NU + c] - u_qp[(size_t)a * NU + c];
            sq += df * df;
            da[(size_t)a * NU + c] = hp.c_action * 2.f * df * inv_n;
        }
        loc[3] += sq;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const float s = warp_sum(loc[i]);
        if (lane == 0) red[i][warp] = s;
    }
    __syncthreads();
    if (threadIdx.x < 10) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += red[threadIdx.x][w];
        part[blockIdx.x * 10 + threadIdx.x] = s;
    }
}

// counts of the label masks (denominators; all-reduced across ranks by the host).  The atomics add integer-valued
// floats, which is exact -- hence order-independent -- while the counts stay below 2^24 agents per minibatch.
__global__ void mask_count_kernel(const int A, const uint8_t* __restrict__ safe_m, const uint8_t* __restrict__ unsafe_m,
                                  float* __restrict__ denoms) {
    float us = 0.f, sf = 0.f;
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < A; a += gridDim.x * blockDim.x) {
        us += unsafe_m[a] ? 1.f : 0.f;
        sf += safe_m[a] ? 1.f : 0.f;
    }
    us = warp_sum(us);
    sf = warp_sum(sf);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(denoms + 0, us);
        atomicAdd(denoms + 1, sf);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(denoms + 2, (float)A);
}

// ------------------------------------------------------------------------------------ backward: output head
// out = tanh(z), z = H2 @ W + b.  dz = d_out (1 - out^2); dW += H2^T (w dz); db += sum w dz; dH2 = dz W^T.
__global__ void __launch_bounds__(256)
head_out_bwd_kernel(const int A, const int nout, const float* __restrict__ H2, const float* __restrict__ W,
                    const float* __restrict__ out, const float* __restrict__ d_out, const float* __restrict__ roww,
                    float* __restrict__ dH2, float* __restrict__ part, const int mask_relu) {
    // mask_relu (folded train step): H2 is the ReLU output feeding the folded output layer; dH2 is masked by H2 > 0 here
    // part (nullptr: data-only backward): part[blockIdx.x][257 nout] = this CTA's [dW (256 x nout) | db (nout)]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    float wacc[8][4], bacc[4];
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) wacc[k][j] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) bacc[j] = 0.f;
    float wl[8][4];
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) wl[k][j] = (j < nout) ? W[(lane * 8 + k) * nout + j] : 0.f;
    // two agents per iteration: every load of both rows is issued before the first use (the loop is latency-bound)
    for (int a0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; a0 < A; a0 += 2 * warps_total) {
        const int a1 = a0 + warps_total;
        const bool two = a1 < A;
        const int a1c = two ? a1 : a0;
        float4 hq[2][2];
        hq[0][0] = *reinterpret_cast<const float4*>(H2 + (size_t)a0 * 256 + lane * 8);
        hq[0][1] = *reinterpret_cast<const float4*>(H2 + (size_t)a0 * 256 + lane * 8 + 4);
        hq[1][0] = *reinterpret_cast<const float4*>(H2 + (size_t)a1c * 256 + lane * 8);
        hq[1][1] = *reinterpret_cast<const float4*>(H2 + (size_t)a1c * 256 + lane * 8 + 4);
        float rwq[2], dzq[2][4];
        rwq[0] = roww ? roww[a0] : 1.f;
        rwq[1] = roww ? roww[a1c] : 1.f;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int a = q ? a1c : a0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j < nout) {
                    const float o = out[(size_t)a * nout + j];
                    dzq[q][j] = d_out[(size_t)a * nout + j] * (1.f - o * o);
                } else {
                    dzq[q][j] = 0.f;
                }
            }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            if (q == 1 && !two) break;
            const int a = q ? a1 : a0;
            const float hv[8] = {hq[q][0].x, hq[q][0].y, hq[q][0].z, hq[q][0].w, hq[q][1].x, hq[q][1].y, hq[q][1].z, hq[q][1].w};
            const float rw = rwq[q];
            float dh[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                float s = 0.f;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    s = fmaf(dzq[q][j], wl[k][j], s);
                    wacc[k][j] = fmaf(hv[k], rw * dzq[q][j], wacc[k][j]);
                }
                dh[k] = (mask_relu && !(hv[k] > 0.f)) ? 0.f : s;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) bacc[j] += rw * dzq[q][j];
            float4* dst = reinterpret_cast<float4*>(dH2 + (size_t)a * 256 + lane * 8);
            dst[0] = make_float4(dh[0], dh[1], dh[2], dh[3]);
            dst[1] = make_float4(dh[4], dh[5], dh[6], dh[7]);
        }
    }
    if (!part) return;   // data-only backward (QP labels): no parameter gradient
    // one slot per warp, summed over the 8 warps in warp order
    __shared__ float s_w[8][256 * 4 + 4];    // [warp][k][j][lane]: the 32 lanes of a warp hit 32 different banks
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (j < nout) s_w[warp][(k * 4 + j) * 32 + lane] = wacc[k][j];
    if (lane == 0)      // bacc is warp-uniform (every lane sees the same dz)
        for (int j = 0; j < nout; ++j) s_w[warp][1024 + j] = bacc[j];
    __syncthreads();
    float* dst = part + (size_t)blockIdx.x * 257 * nout;
    for (int i = threadIdx.x; i < 257 * nout; i += blockDim.x) {
        int idx;
        if (i < 256 * nout) {
            const int row = i / nout, j = i % nout;      // W row = lane * 8 + k
            idx = ((row & 7) * 4 + j) * 32 + (row >> 3);
        } else {
            idx = 1024 + i - 256 * nout;
        }
        float v = 0.f;
        for (int w = 0; w < 8; ++w) v += s_w[w][idx];
        dst[i] = v;
    }
}

// ------------------------------------------------------------------------------------ backward: attention + aggregation
// AG[a] = sum_e att_e MSG_e, att = softmax(gate), gate_e = G2_e . a3 + ba3.
// dMSG_e = att_e dAG ; datt_e = dAG . MSG_e ; dgate_e = att_e (datt_e - sum att datt) ;
// dG2_e = dgate_e a3 ; da3 += w sum dgate_e G2_e ; dba3 += w sum dgate_e.
__global__ void __launch_bounds__(256)
attn_aggregate_bwd_kernel(const int A, const int edge_cap, const float* __restrict__ dAG, const float* __restrict__ MSG,
                          const float* __restrict__ G2, const float* __restrict__ ATT, const float* __restrict__ a3,
                          const int32_t* __restrict__ row_start, const int32_t* __restrict__ row_deg,
                          const float* __restrict__ roww, float* __restrict__ dMSG, float* __restrict__ dG2,
                          float* __restrict__ part, const int mask_relu) {
    // mask_relu (folded train step): G2 is the ReLU output of the gate's first layer and a3 the folded gate vector;
    // dG2 is masked by G2 > 0 here
    // part (nullptr: data-only backward): part[blockIdx.x][129] = this CTA's [da3 (128) | dba3]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    const float4 w3 = *reinterpret_cast<const float4*>(a3 + lane * 4);
    float4 acc3 = make_float4(0.f, 0.f, 0.f, 0.f);
    float accb = 0.f;
    for (int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; a < A; a += warps_total) {
        const int rs = row_start[a];
        int rd = row_deg[a];
        if (rs < 0 || rs + rd > edge_cap) rd = 0;
        const float4 dag = *reinterpret_cast<const float4*>(dAG + (size_t)a * 128 + lane * 4);
        const float rw = roww ? roww[a] : 1.f;
        float dot_sum = 0.f;
        if (rd <= 4) {
            // the common case (goal row + a few neighbours): MSG is read once, the 4 dot products are reduced together
            float p[4], at[4];
            float4 g[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int e = rs + min(q, max(rd - 1, 0));
                const bool on = q < rd;
                const float4 m = on ? *reinterpret_cast<const float4*>(MSG + (size_t)e * 128 + lane * 4)
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
                g[q] = on ? *reinterpret_cast<const float4*>(G2 + (size_t)e * 128 + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                at[q] = on ? ATT[e] : 0.f;
                p[q] = dag.x * m.x + dag.y * m.y + dag.z * m.z + dag.w * m.w;
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1)
#pragma unroll
                for (int q = 0; q < 4; ++q) p[q] += __shfl_xor_sync(0xffffffffu, p[q], off);
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (q < rd) dot_sum = fmaf(at[q], p[q], dot_sum);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (q < rd) {
                    const int e = rs + q;
                    const float att = at[q];
                    const float dgate = att * (p[q] - dot_sum);
                    *reinterpret_cast<float4*>(dMSG + (size_t)e * 128 + lane * 4) =
                        make_float4(att * dag.x, att * dag.y, att * dag.z, att * dag.w);
                    float4 dg = make_float4(dgate * w3.x, dgate * w3.y, dgate * w3.z, dgate * w3.w);
                    if (mask_relu) {
                        dg.x = g[q].x > 0.f ? dg.x : 0.f; dg.y = g[q].y > 0.f ? dg.y : 0.f;
                        dg.z = g[q].z > 0.f ? dg.z : 0.f; dg.w = g[q].w > 0.f ? dg.w : 0.f;
                    }
                    *reinterpret_cast<float4*>(dG2 + (size_t)e * 128 + lane * 4) = dg;
                    const float wd = rw * dgate;
                    acc3.x = fmaf(wd, g[q].x, acc3.x);
                    acc3.y = fmaf(wd, g[q].y, acc3.y);
                    acc3.z = fmaf(wd, g[q].z, acc3.z);
                    acc3.w = fmaf(wd, g[q].w, acc3.w);
                    accb += wd;
                }
            }
            continue;
        }
        for (int e = rs; e < rs + rd; ++e) {
            const float4 m = *reinterpret_cast<const float4*>(MSG + (size_t)e * 128 + lane * 4);
            const float datt = warp_sum(dag.x * m.x + dag.y * m.y + dag.z * m.z + dag.w * m.w);
            dot_sum = fmaf(ATT[e], datt, dot_sum);
        }
        for (int e = rs; e < rs + rd; ++e) {
            const float att = ATT[e];
            const float4 m = *reinterpret_cast<const float4*>(MSG + (size_t)e * 128 + lane * 4);
            const float datt = warp_sum(dag.x * m.x + dag.y * m.y + dag.z * m.z + dag.w * m.w);
            const float dgate = att * (datt - dot_sum);
            *reinterpret_cast<float4*>(dMSG + (size_t)e * 128 + lane * 4) =
                make_float4(att * dag.x, att * dag.y, att * dag.z, att * dag.w);
            const float4 g = *reinterpret_cast<const float4*>(G2 + (size_t)e * 128 + lane * 4);
            float4 dg = make_float4(dgate * w3.x, dgate * w3.y, dgate * w3.z, dgate * w3.w);
            if (mask_relu) {
                dg.x = g.x > 0.f ? dg.x : 0.f; dg.y = g.y > 0.f ? dg.y : 0.f;
                dg.z = g.z > 0.f ? dg.z : 0.f; dg.w = g.w > 0.f ? dg.w : 0.f;
            }
            *reinterpret_cast<float4*>(dG2 + (size_t)e * 128 + lane * 4) = dg;
            const float wd = rw * dgate;
            acc3.x = fmaf(wd, g.x, acc3.x);
            acc3.y = fmaf(wd, g.y, acc3.y);
            acc3.z = fmaf(wd, g.z, acc3.z);
            acc3.w = fmaf(wd, g.w, acc3.w);
            accb += wd;
        }
    }
    if (!part) return;  // data-only backward
    __shared__ float s_a[8][132];                 // [warp][component][lane]: conflict-free; summed in warp order
    s_a[warp][0 * 32 + lane] = acc3.x;
    s_a[warp][1 * 32 + lane] = acc3.y;
    s_a[warp][2 * 32 + lane] = acc3.z;
    s_a[warp][3 * 32 + lane] = acc3.w;
    accb = warp_sum(accb);
    if (lane == 0) s_a[warp][128] = accb;
    __syncthreads();
    if (threadIdx.x < 129) {
        const int idx = threadIdx.x < 128 ? (threadIdx.x & 3) * 32 + (threadIdx.x >> 2) : 128;
        float v = 0.f;
        for (int w = 0; w < 8; ++w) v += s_a[w][idx];
        part[(size_t)blockIdx.x * 129 + threadIdx.x] = v;
    }
}

// ------------------------------------------------------------------------------------ backward: edge layer 1
// dY = dX1pre [nE,256] (already masked by X1 > 0).  dW1[:ed] += feat^T (w dY); dW1[ed+t] += sum_{type t} w dY;
// dW1[ed+5] += sum w dY; db1 += sum w dY.  Thread = output column; CTA = strided chunk of edges.
// part[blockIdx.x][(ED + 4) x 256]: this CTA's rows 0 .. ED+2 of dW1 and the all-edge sum (dW1[ED+5] and db1).
__host__ __device__ constexpr int edge_l1_part_floats(int ed) { return (ed + 4) * 256; }
template <int ED>
__global__ void __launch_bounds__(256)
edge_l1_bwd_w_kernel(const int edge_cap, const int n_agents_total, const int32_t* __restrict__ counters,
                     const float* __restrict__ dY, const float* __restrict__ feat,
                     const int32_t* __restrict__ edge_src, const int32_t* __restrict__ edge_recv,
                     const float* __restrict__ roww, float* __restrict__ part) {
    // chunks of 64 edges: the per-edge metadata (features, sender type, row weight) is staged in shared memory so that the
    // dY loads of a chunk are independent of it and 8 of them are in flight per thread
    constexpr int CH = 64;
    __shared__ float s_feat[CH][ED];
    __shared__ float s_w[CH];
    __shared__ int s_t[CH];
    const int nE = min(counters[0], edge_cap);
    const int c = threadIdx.x;
    float accw[ED], acct[3], accall = 0.f;
#pragma unroll
    for (int i = 0; i < ED; ++i) accw[i] = 0.f;
    acct[0] = acct[1] = acct[2] = 0.f;
    const int n_chunks = (nE + CH - 1) / CH;
    for (int ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
        const int e0 = ch * CH;
        const int n = min(CH, nE - e0);
        __syncthreads();
        if (c < CH) {
            float w = 0.f;
            int t = 0;
            if (c < n) {
                w = roww ? roww[min(max(edge_recv[e0 + c], 0), n_agents_total - 1)] : 1.f;
                const int code = edge_src[e0 + c];
                t = (code >= 0) ? 2 : ((code == -1) ? 1 : 0);
            }
            s_w[c] = w;
            s_t[c] = t;
        }
        for (int i = c; i < CH * ED; i += 256) {
            const int r = i / ED, k = i % ED;
            s_feat[r][k] = (r < n) ? feat[(size_t)(e0 + r) * FEAT_LD + k] : 0.f;
        }
        __syncthreads();
        for (int r0 = 0; r0 < n; r0 += 8) {
            float g[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) g[q] = (r0 + q < n) ? dY[(size_t)(e0 + r0 + q) * 256 + c] : 0.f;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int r = r0 + q;       // rows >= n carry w = 0 and g = 0
                const float gg = s_w[r & (CH - 1)] * g[q];
                const int t = s_t[r & (CH - 1)];
#pragma unroll
                for (int i = 0; i < ED; ++i) accw[i] = fmaf(s_feat[r & (CH - 1)][i], gg, accw[i]);
                acct[0] += (t == 0) ? gg : 0.f;
                acct[1] += (t == 1) ? gg : 0.f;
                acct[2] += (t == 2) ? gg : 0.f;
                accall += gg;
            }
        }
    }
    float* dst = part + (size_t)blockIdx.x * edge_l1_part_floats(ED);
#pragma unroll
    for (int i = 0; i < ED; ++i) dst[i * 256 + c] = accw[i];
#pragma unroll
    for (int t = 0; t < 3; ++t) dst[(ED + t) * 256 + c] = acct[t];
    dst[(ED + 3) * 256 + c] = accall;
}

// dfeat = dY @ W1[:ed]^T through the norm-clip, per edge: je[e][:ED] = d out[recv] / d feat_e (edge-state space).
// The QP labels use it as the Jacobian block; the train step gathers it per agent (edge_grad_gather_kernel).
// One warp per edge.
template <int KIND>
__global__ void __launch_bounds__(256)
edge_l1_bwd_x_kernel(const gcbf_env_desc d, const float* __restrict__ W1, const float* __restrict__ dY,
                     const float* __restrict__ agent, const float* __restrict__ goal, const float* __restrict__ hits,
                     const int32_t* __restrict__ edge_recv, const int32_t* __restrict__ edge_src,
                     const int32_t* __restrict__ counters, const int clip_all, float* __restrict__ je) {
    using T = EnvTraits<KIND>;
    constexpr int ED = T::ED, SD = T::SD, PD = T::PD;
    __shared__ __align__(16) float sW[ED][256];
    for (int i = threadIdx.x; i < ED * 256; i += blockDim.x) sW[i / 256][i % 256] = W1[i];
    __syncthreads();
    const int nE = min(counters[0], d.edge_cap);
    const int A = d.n_graphs * d.n_agents;
    const int lane = threadIdx.x & 31;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    for (int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < nE; e += warps_total) {
        const float4 g0 = *reinterpret_cast<const float4*>(dY + (size_t)e * 256 + lane * 8);
        const float4 g1 = *reinterpret_cast<const float4*>(dY + (size_t)e * 256 + lane * 8 + 4);
        const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        float df[ED];
#pragma unroll
        for (int c = 0; c < ED; ++c) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) s = fmaf(gv[j], sW[c][lane * 8 + j], s);
            df[c] = warp_sum(s);
        }
        if (lane == 0) {
            const int a = min(max(edge_recv[e], 0), A - 1);
            int code = min(edge_src[e], A - 1);
            float er[ED], es[ED], f[ED], coef, nrm;
            edge_state_dev<KIND>(agent + (size_t)a * SD, er);
            sender_state_dev<KIND>(code, a, d.n_hits, agent, goal, hits, es);
            const bool clip = clip_all || code == -1;
            edge_feat_dev<KIND>(er, es, clip, d.comm_radius, f, &coef, &nrm);
            if (clip && coef != 1.f) {
                // feat_p = coef * dlt_p, coef = rc / n: d dlt_q = coef (df_q - dlt_q (sum_p df_p dlt_p) / n^2)
                float dotp = 0.f;
#pragma unroll
                for (int p = 0; p < PD; ++p) dotp += df[p] * (er[p] - es[p]);
                const float inv_n2 = 1.f / (nrm * nrm);
#pragma unroll
                for (int p = 0; p < PD; ++p) df[p] = coef * (df[p] - (er[p] - es[p]) * dotp * inv_n2);
            }
#pragma unroll
            for (int c = 0; c < ED; ++c) je[(size_t)e * 8 + c] = df[c];
        }
    }
}

// d_es[a] = sum_{e in row a} je[e] - sum_{e : sender(e) = a} je[e]: feat_e = es(recv) - es(sender).  The edges sent by
// agent a are the mirrors of a's agent edges -- edge a -> j lies in row j, since the radius graph is symmetric -- so
// every agent reads its own row and its neighbours' rows, in row order, and writes its gradient once.
template <int ED>
__global__ void __launch_bounds__(128)
edge_grad_gather_kernel(const int A, const int edge_cap, const int32_t* __restrict__ row_start,
                        const int32_t* __restrict__ row_deg, const int32_t* __restrict__ edge_src,
                        const float* __restrict__ je, float* __restrict__ d_es) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A) return;
    float s[ED];
#pragma unroll
    for (int c = 0; c < ED; ++c) s[c] = 0.f;
    const int rs = row_start[a];
    int rd = row_deg[a];
    if (rs < 0 || rs + rd > edge_cap) rd = 0;
    for (int e = rs; e < rs + rd; ++e)
#pragma unroll
        for (int c = 0; c < ED; ++c) s[c] += je[(size_t)e * 8 + c];
    for (int e = rs; e < rs + rd; ++e) {
        const int j = edge_src[e];
        if (j < 0 || j >= A) continue;
        const int rs2 = row_start[j];
        int rd2 = row_deg[j];
        if (rs2 < 0 || rs2 + rd2 > edge_cap) rd2 = 0;
        for (int e2 = rs2; e2 < rs2 + rd2; ++e2) {
            if (edge_src[e2] == a) {
#pragma unroll
                for (int c = 0; c < ED; ++c) s[c] -= je[(size_t)e2 * 8 + c];
                break;
            }
        }
    }
#pragma unroll
    for (int c = 0; c < ED; ++c) d_es[(size_t)a * ED + c] = s[c];
}

// d_es (edge-state grads of x') -> d a.   x' = clip_state(x + xdot(x, u) dt), u = clip_action(a)
// (gcbf_plus.py:386-391; double_integrator.py:128-143,340-354 and twins): the chain edge state -> state ->
// clip_state -> Euler -> clip_action of agent `a`, shared by the train step and the policy refinement.
template <int KIND>
__device__ __forceinline__ void dyn_chain_dev(const gcbf_env_desc& d, const float* agent, const float* goal,
                                              const float* action, const float* xnext, const float* d_es, const int a,
                                              float* g) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU, ED = T::ED;
    float dx[SD], xn[SD], de[ED];
#pragma unroll
    for (int c = 0; c < ED; ++c) de[c] = d_es[(size_t)a * ED + c];
#pragma unroll
    for (int c = 0; c < SD; ++c) xn[c] = xnext[(size_t)a * SD + c];
    if (KIND == GCBF_ENV_DUBINS_CAR) {  // es = (x, y, v cos th, v sin th)
        const float th = xn[2], v = xn[3];
        dx[0] = de[0];
        dx[1] = de[1];
        dx[2] = de[2] * (-v * sinf(th)) + de[3] * (v * cosf(th));
        dx[3] = de[2] * cosf(th) + de[3] * sinf(th);
    } else {
#pragma unroll
        for (int c = 0; c < SD; ++c) dx[c] = de[c];
    }
    // clip_state: zero gradient on clipped velocity components
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        const bool limited = (KIND == GCBF_ENV_DOUBLE_INTEGRATOR && c >= 2) || (KIND == GCBF_ENV_DUBINS_CAR && c == 3) ||
                             (KIND == GCBF_ENV_LINEAR_DRONE && c >= 3);
        if (limited && !(xn[c] > -d.v_lim && xn[c] < d.v_lim)) dx[c] = 0.f;
    }
    float du[NU];
    if (KIND == GCBF_ENV_SINGLE_INTEGRATOR) {
        du[0] = dx[0] * d.dt;
        du[1] = dx[1] * d.dt;
    } else if (KIND == GCBF_ENV_DOUBLE_INTEGRATOR) {
        du[0] = dx[2] * d.dt / d.mass;
        du[1] = dx[3] * d.dt / d.mass;
    } else if (KIND == GCBF_ENV_DUBINS_CAR) {
        const float ddx = agent[(size_t)a * SD + 0] - goal[(size_t)a * SD + 0];
        const float ddy = agent[(size_t)a * SD + 1] - goal[(size_t)a * SD + 1];
        const float keep = (sqrtf(ddx * ddx + ddy * ddy) < d.half_r) ? 0.f : 1.f;
        du[0] = dx[2] * 20.f * d.dt * keep;
        du[1] = dx[3] * d.dt * keep;
    } else {
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < SD; ++r) s += dx[r] * d.B[r * NU + c];
            du[c] = s * d.dt;
        }
    }
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        const float act = action[(size_t)a * NU + c];
        g[c] = (act > -d.u_lim && act < d.u_lim) ? du[c] : 0.f;  // clip_action
    }
}

// train step: a = 2 pi + u_ref, so d_pi = 2 (da_dyn + da_direct).
template <int KIND>
__global__ void dyn_bwd_kernel(const gcbf_env_desc d, const float* __restrict__ agent, const float* __restrict__ goal,
                               const float* __restrict__ action, const float* __restrict__ xnext,
                               const float* __restrict__ d_es, const float* __restrict__ da_direct,
                               float* __restrict__ d_pi) {
    constexpr int NU = EnvTraits<KIND>::NU;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= d.n_graphs * d.n_agents) return;
    float g[NU];
    dyn_chain_dev<KIND>(d, agent, goal, action, xnext, d_es, a, g);
#pragma unroll
    for (int c = 0; c < NU; ++c) d_pi[(size_t)a * NU + c] = 2.f * (g[c] + da_direct[(size_t)a * NU + c]);
}

// ------------------------------------------------------------------------------------ one network backward
// Built by aggregate initialisation, in this order.
struct BwdArgs {
    const gcbf_env_desc* d;
    GraphRefs g;           // the graph of the forward pass
    float* gw;             // gradient workspace (make_ws layout)
    float* part;           // PART_FLOATS: per-CTA partials of the weight-gradient reductions (when G is set)
    int use_tc;            // 1: backward-data GEMMs on the wgmma path
    int out_dim;
    const float* P;        // parameters
    const float* PT;       // backward-data B operands (prepare_bwd_operands)
    const float* fw;       // forward workspace (saved activations)
    const float* out;      // network output (tanh applied) [A, out_dim]
    const float* d_out;    // upstream gradient wrt the output [A, out_dim]
    const float* roww;     // optional per-agent weights applied to every dW / db contribution
    float* G;              // parameter gradient (accumulated); nullptr: data-only backward
    int clip_all;
    float* d_es;           // optional [A, ED] (written): gradient wrt the agents' edge states, gathered from `je`
    float* je;             // [cap, 8] when d_es is wanted or the per-edge blocks are the result: d out[recv] / d feat_e
    const int32_t* agent_rows = nullptr;   // optional device row count of the agent-row GEMMs (default: every agent)
};

// Backward-data B operands of a one-layer network: the straight tf32 planes (build_planes) on the tensor-core path,
// W^T (TransLayout) on the SIMT path.
static int32_t prepare_bwd_operands(int ed, int out_dim, int use_tc, const float* P, float* PT, cudaStream_t st) {
    if (use_tc) return build_planes(ed, out_dim, 1, P, PT, st);
    const ParamLayout L = make_layout(ed, out_dim);
    return build_transposes(L, make_trans_layout(L), P, PT, st);
}

// ---- the parameter-gradient kernels followed by the ordered sum of their per-CTA partials
static int grid_for_part(int grid, int64_t part_floats) {
    return min(grid, (int)(PART_FLOATS / part_floats));
}

// output layer: dW, db (nullptr: data-only) and dH2
static int32_t head_out_bwd(const BwdArgs& b, int grid, const float* H2, const float* W, float* dH2, float* dW, float* db,
                            int mask_relu, cudaStream_t st) {
    const int A = b.d->n_graphs * b.d->n_agents, no = b.out_dim;
    grid = grid_for_part(grid, 257 * no);
    head_out_bwd_kernel<<<grid, 256, 0, st>>>(A, no, H2, W, b.out, b.d_out, b.roww, dH2, dW ? b.part : nullptr, mask_relu);
    count_launch();
    if (int32_t rc = check_launch("head_out_bwd_kernel")) return rc;
    if (!dW) return 0;
    return launch_partial_sum(b.part, 257 * no, grid, PartSegs().add(dW, 256 * no).add(db, no), st);
}

// attention + aggregation: dMSG, dG2 and (da3 != nullptr) the gate vector's gradient da3, dba3
static int32_t attn_aggregate_bwd(const BwdArgs& b, int grid, const float* dAG, const float* MSG, const float* G2,
                                  const float* ATT, const float* a3, float* dMSG, float* dG2, float* da3, float* dba3,
                                  int mask_relu, cudaStream_t st) {
    const int A = b.d->n_graphs * b.d->n_agents;
    grid = grid_for_part(grid, 129);
    attn_aggregate_bwd_kernel<<<grid, 256, 0, st>>>(A, b.d->edge_cap, dAG, MSG, G2, ATT, a3, b.g.row_start,
                                                    b.g.row_deg, b.roww, dMSG, dG2, da3 ? b.part : nullptr, mask_relu);
    count_launch();
    if (int32_t rc = check_launch("attn_aggregate_bwd_kernel")) return rc;
    if (!da3) return 0;
    return launch_partial_sum(b.part, 129, grid, PartSegs().add(da3, 128).add(dba3, 1), st);
}

// edge layer 1: dW1 / db1 (wgrad) from the saved features, and the per-edge input gradient je, gathered into d_es
static int32_t edge_l1_bwd(const BwdArgs& b, const ParamLayout& L, const float* dY, const float* feat, bool wgrad,
                           cudaStream_t st) {
    const gcbf_env_desc* d = b.d;
    const int ed = env_ed(d->env_kind), cap = d->edge_cap, A = d->n_graphs * d->n_agents, nsm = sm_count();
    if (wgrad) {
        float* dW1 = b.G + L.w[L_MSG0];
        const int grid = grid_for_part(min(max(cap / 64, 1), 4 * nsm), edge_l1_part_floats(ed));   // chunks of 64 edges
        switch (ed) {
            case 2: edge_l1_bwd_w_kernel<2><<<grid, 256, 0, st>>>(cap, A, b.g.counters, dY, feat, b.g.edge_src, b.g.edge_recv, b.roww, b.part); break;
            case 4: edge_l1_bwd_w_kernel<4><<<grid, 256, 0, st>>>(cap, A, b.g.counters, dY, feat, b.g.edge_src, b.g.edge_recv, b.roww, b.part); break;
            default: edge_l1_bwd_w_kernel<6><<<grid, 256, 0, st>>>(cap, A, b.g.counters, dY, feat, b.g.edge_src, b.g.edge_recv, b.roww, b.part); break;
        }
        count_launch();
        if (int32_t rc = check_launch("edge_l1_bwd_w_kernel")) return rc;
        if (int32_t rc = launch_partial_sum(b.part, edge_l1_part_floats(ed), grid,
                                            PartSegs().add(dW1, (ed + 3) * 256).add(dW1 + (ed + 5) * 256, 256, b.G + L.b[L_MSG0]),
                                            st))
            return rc;
    }
    if (!b.je) return 0;
    const int grid = min((cap + 7) / 8, 4 * nsm);
    GCBF_DISPATCH_ENV(d->env_kind, {
        edge_l1_bwd_x_kernel<KIND><<<grid, 256, 0, st>>>(*d, b.P + L.w[L_MSG0], dY, b.g.agent, b.g.goal, b.g.hits,
                                                         b.g.edge_recv, b.g.edge_src, b.g.counters, b.clip_all, b.je);
    });
    count_launch();
    if (int32_t rc = check_launch("edge_l1_bwd_x_kernel")) return rc;
    if (!b.d_es) return 0;
    switch (ed) {
        case 2: edge_grad_gather_kernel<2><<<(A + 127) / 128, 128, 0, st>>>(A, cap, b.g.row_start, b.g.row_deg, b.g.edge_src, b.je, b.d_es); break;
        case 4: edge_grad_gather_kernel<4><<<(A + 127) / 128, 128, 0, st>>>(A, cap, b.g.row_start, b.g.row_deg, b.g.edge_src, b.je, b.d_es); break;
        default: edge_grad_gather_kernel<6><<<(A + 127) / 128, 128, 0, st>>>(A, cap, b.g.row_start, b.g.row_deg, b.g.edge_src, b.je, b.d_es); break;
    }
    count_launch();
    return check_launch("edge_grad_gather_kernel");
}

// dW += X^T (w dY) and db (+ db2) += sum_m w dY: the SIMT split-M kernel followed by column-sum launches.  Only
// the SIMT train step computes weight gradients layer by layer; the folded step has its own (gnn_backward_folded).
static int32_t dense_bwd_weight(const BwdArgs& b, const float* X, int ldx, const float* dY, float* C, float* db,
                                float* db2, const int32_t* row2agent, RowCount rc, int K1, int N, int A,
                                cudaStream_t st) {
    if (int32_t r = launch_gemm_tn(X, ldx, dY, C, b.roww, row2agent, rc, K1, N, A, st, b.part)) return r;
    return launch_colsum(dY, db, b.roww, row2agent, rc, N, A, st, b.part, db2);
}

// dX = epi(dY @ W_i^T) (+= if accum) with the B operand at b.PT + boff[li].  Tensor core: the straight tf32 planes of
// W_i (PlaneLayout.s, W itself is the K-major operand); SIMT: W_i^T (TransLayout).
static int32_t dense_bwd_data(const BwdArgs& b, const ParamLayout& L, const int* boff, int li, int epi, bool accum,
                              const float* dY, float* dX, const float* aux, RowCount rc, cudaStream_t st) {
    const int N = (li == L_UPD0) ? 128 : L.in[li];
    const int K = L.out[li];
    const float* B = b.PT + boff[li];
    if (b.use_tc) return tc::launch_gemm_tc(epi, accum, dY, B, B + K * N, nullptr, nullptr, dX, aux, rc, K, N, st);
    return launch_gemm_nn(epi, accum, dY, B, nullptr, nullptr, dX, aux, rc, K, N, st);
}

static int32_t gnn_backward_impl(const BwdArgs& b, cudaStream_t st) {
    const gcbf_env_desc* d = b.d;
    const int ed = env_ed(d->env_kind);
    const ParamLayout L = make_layout(ed, b.out_dim);
    const TransLayout TL = make_trans_layout(L);
    const PlaneLayout Q = make_plane_layout(make_deep_layout(ed, b.out_dim, 1), ed);
    const int* boff = b.use_tc ? Q.s : TL.w;
    const int A = d->n_graphs * d->n_agents, cap = d->edge_cap;
    const GnnWs W = make_ws(cap, A);
    const RowCount re{b.g.counters, 0, cap};
    const RowCount ra{b.agent_rows, A, A};
    const int nsm = sm_count();
    const float* fw = b.fw;
    float* gw = b.gw;
    int32_t rc;
    const bool wgrad = b.G != nullptr;   // false: data-only backward (d network / d inputs), used by the QP labels
    float* const Gz = b.G;
#define RC(x) do { if ((rc = (x))) return rc; } while (0)
#define WG(x) do { if (wgrad) RC(x); } while (0)
    // ---- output layer
    RC(head_out_bwd(b, min((A + 7) / 8, 2 * nsm), fw + W.h2, b.P + L.w[L_OUT], gw + W.h2,
                    wgrad ? Gz + L.w[L_OUT] : nullptr, wgrad ? Gz + L.b[L_OUT] : nullptr, 0, st));
    // ---- head MLP
    WG(dense_bwd_weight(b, fw + W.h1, 256, gw + W.h2, b.G + L.w[L_HEAD1], b.G + L.b[L_HEAD1], nullptr, nullptr, ra, 256, 256, A, st));
    RC(dense_bwd_data(b, L, boff, L_HEAD1, EPI_RELU_MASK, false, gw + W.h2, gw + W.h1, fw + W.h1, ra, st));
    WG(dense_bwd_weight(b, fw + W.v3, 128, gw + W.h1, b.G + L.w[L_HEAD0], b.G + L.b[L_HEAD0], nullptr, nullptr, ra, 128, 256, A, st));
    RC(dense_bwd_data(b, L, boff, L_HEAD0, EPI_NONE, false, gw + W.h1, gw + W.v3, nullptr, ra, st));
    // ---- update MLP
    WG(dense_bwd_weight(b, fw + W.v2, 256, gw + W.v3, b.G + L.w[L_UPDOUT], b.G + L.b[L_UPDOUT], nullptr, nullptr, ra, 256, 128, A, st));
    RC(dense_bwd_data(b, L, boff, L_UPDOUT, EPI_NONE, false, gw + W.v3, gw + W.v2, nullptr, ra, st));
    WG(dense_bwd_weight(b, fw + W.v1, 256, gw + W.v2, b.G + L.w[L_UPD1], b.G + L.b[L_UPD1], nullptr, nullptr, ra, 256, 256, A, st));
    RC(dense_bwd_data(b, L, boff, L_UPD1, EPI_RELU_MASK, false, gw + W.v2, gw + W.v1, fw + W.v1, ra, st));
    WG(dense_bwd_weight(b, fw + W.ag, 128, gw + W.v1, b.G + L.w[L_UPD0] + 3 * 256, b.G + L.b[L_UPD0], b.G + L.w[L_UPD0] + 2 * 256, nullptr, ra, 128, 256, A, st));
    RC(dense_bwd_data(b, L, boff, L_UPD0, EPI_NONE, false, gw + W.v1, gw + W.ag, nullptr, ra, st));
    // ---- attention + aggregation
    RC(attn_aggregate_bwd(b, min((A + 7) / 8, 2 * nsm), gw + W.ag, fw + W.msg, fw + W.g2, fw + W.att, b.P + L.w[L_GATE],
                          gw + W.msg, gw + W.g2, wgrad ? Gz + L.w[L_GATE] : nullptr, wgrad ? Gz + L.b[L_GATE] : nullptr, 0,
                          st));
    // ---- gate MLP (edge rows; dW weighted by the receiver's weight)
    WG(dense_bwd_weight(b, fw + W.g1, 128, gw + W.g2, b.G + L.w[L_ATT1], b.G + L.b[L_ATT1], nullptr, b.g.edge_recv, re, 128, 128, A, st));
    RC(dense_bwd_data(b, L, boff, L_ATT1, EPI_RELU_MASK, false, gw + W.g2, gw + W.g1, fw + W.g1, re, st));
    WG(dense_bwd_weight(b, fw + W.msg, 128, gw + W.g1, b.G + L.w[L_ATT0], b.G + L.b[L_ATT0], nullptr, b.g.edge_recv, re, 128, 128, A, st));
    RC(dense_bwd_data(b, L, boff, L_ATT0, EPI_NONE, true, gw + W.g1, gw + W.msg, nullptr, re, st));
    // ---- message MLP
    WG(dense_bwd_weight(b, fw + W.x2, 256, gw + W.msg, b.G + L.w[L_MSGOUT], b.G + L.b[L_MSGOUT], nullptr, b.g.edge_recv, re, 256, 128, A, st));
    RC(dense_bwd_data(b, L, boff, L_MSGOUT, EPI_NONE, false, gw + W.msg, gw + W.x2, nullptr, re, st));
    WG(dense_bwd_weight(b, fw + W.x1, 256, gw + W.x2, b.G + L.w[L_MSG1], b.G + L.b[L_MSG1], nullptr, b.g.edge_recv, re, 256, 256, A, st));
    RC(dense_bwd_data(b, L, boff, L_MSG1, EPI_RELU_MASK, false, gw + W.x2, gw + W.x1, fw + W.x1, re, st));
    // ---- edge layer 1
    RC(edge_l1_bwd(b, L, gw + W.x1, fw + W.feat, wgrad, st));
#undef WG
#undef RC
    return 0;
}

// ------------------------------------------------------------------------------------ folded train step
// Every MLP block ends in two linear layers with no activation between them (mlp.py:23-29, act_final=False), and the
// update block's tail feeds the head's first layer directly.  The forward of the train step therefore runs on the same
// folded weights as the rollout (gcbf_prepare_infer: W23 = W2 W3, a23 = A2 a3, UH = U2 U3 H1, HO = H2 H3) -- 4 GEMMs per
// network instead of 9 -- keeps the ReLU outputs (x1, g1, v1, h1) plus msg / att / ag, and the backward differentiates
// the folded network: 4 weight-gradient GEMMs and 4 data GEMMs per pass instead of 10 + 9.  The gradients of the folded
// weights (accumulated over the passes of a network in `Gf`, InferLayout offsets) are un-folded onto the flax
// parameters at the end by the chain rule of the products (unfold_jobs: two launches of small products for both networks).
// Same function, same gradient; only the rounding differs (~1e-6 relative, like the rollout's folded forward).
static int32_t gnn_backward_folded(const BwdArgs& b, const float* blob, float* Gf, cudaStream_t st) {
    const gcbf_env_desc* d = b.d;
    const int ed = env_ed(d->env_kind);
    const ParamLayout L = make_layout(ed, b.out_dim);
    const InferLayout I = make_infer_layout(b.out_dim);
    const int A = d->n_graphs * d->n_agents, cap = d->edge_cap;
    const GnnWs W = make_ws(cap, A);
    const RowCount re{b.g.counters, 0, cap};
    const RowCount ra{nullptr, A, A};
    const int nsm = sm_count();
    const float* fw = b.fw;
    float* gw = b.gw;
    int32_t rc;
#define RC(x) do { if ((rc = (x))) return rc; } while (0)
    auto data = [&](int epi, bool accum, const float* dY, int p_off, int K, int N, float* dX, const float* aux,
                    RowCount rows) -> int32_t {
        return tc::launch_gemm_tc(epi, accum, dY, blob + p_off, blob + p_off + K * N, nullptr, nullptr, dX, aux, rows, K, N, st);
    };
    // ---- folded output layer: z = h1 HO + bho, out = tanh(z); dh1 masked by h1 > 0
    RC(head_out_bwd(b, min((A + 7) / 8, 2 * nsm), fw + W.h1, blob + I.ho, gw + W.h1, Gf + I.ho, Gf + I.bho, 1, st));
    // ---- h1 = relu(v1 UH + buh)
    RC(tc::launch_gemm_tn_tc(fw + W.v1, 256, gw + W.h1, Gf + I.uh, b.roww, nullptr, ra, 256, 256, A, st, Gf + I.buh, nullptr,
                             b.part));
    RC(data(EPI_RELU_MASK, false, gw + W.h1, I.p_uh, 256, 256, gw + W.v1, fw + W.v1, ra));
    // ---- v1 = relu(ag U1[3:] + U1[2] + bu1)
    RC(tc::launch_gemm_tn_tc(fw + W.ag, 128, gw + W.v1, b.G + L.w[L_UPD0] + 3 * 256, b.roww, nullptr, ra, 128, 256, A, st,
                             b.G + L.b[L_UPD0], b.G + L.w[L_UPD0] + 2 * 256, b.part));
    RC(data(EPI_NONE, false, gw + W.v1, I.p_u1, 256, 128, gw + W.ag, nullptr, ra));
    // ---- attention + aggregation with the folded gate vector (g1 = relu output of the gate's first layer)
    // (latency-bound warp-per-receiver loop: as many warps in flight as fit)
    RC(attn_aggregate_bwd(b, min((A + 7) / 8, 6 * nsm), gw + W.ag, fw + W.msg, fw + W.g1, fw + W.att, blob + I.a23,
                          gw + W.msg, gw + W.g1, Gf + I.a23, Gf + I.c23, 1, st));
    // ---- g1 = relu(msg A1 + ba1)
    RC(tc::launch_gemm_tn_tc(fw + W.msg, 128, gw + W.g1, b.G + L.w[L_ATT0], b.roww, b.g.edge_recv, re, 128, 128, A, st,
                             b.G + L.b[L_ATT0], nullptr, b.part));
    RC(data(EPI_NONE, true, gw + W.g1, I.p_a1, 128, 128, gw + W.msg, nullptr, re));
    // ---- msg = x1 W23 + b23
    RC(tc::launch_gemm_tn_tc(fw + W.x1, 256, gw + W.msg, Gf + I.w23, b.roww, b.g.edge_recv, re, 256, 128, A, st, Gf + I.b23,
                             nullptr, b.part));
    RC(data(EPI_RELU_MASK, false, gw + W.msg, I.p_w23, 128, 256, gw + W.x1, fw + W.x1, re));
    // ---- edge layer 1
    RC(edge_l1_bwd(b, L, gw + W.x1, fw + W.feat, true, st));
#undef RC
    return 0;
}

constexpr int64_t UNFOLD_SCRATCH = 256 * 128 + 128;   // floats of unfold_jobs' `scratch`: T [256, 128] and t [128]

// Chain rule of the folded products: G (flax layout) += d(folded) / d(parameters) applied to Gf.
//   W23 = W2 W3, b23 = b2 W3 + b3          -> dW2 = dW23 W3^T, dW3 = W2^T dW23 + b2 (x) db23, db2 = db23 W3^T, db3 = db23
//   a23 = A2 a3, c23 = ba2 . a3 + ba3      -> dA2 = da23 (x) a3, da3 = A2^T da23 + ba2 dc23, dba2 = a3 dc23, dba3 = dc23
//   UH = U2 U3 H1, buh = (bu2 U3 + bu3) H1 + bh1
//        T = dUH H1^T, t = dbuh H1^T       -> dU2 = T U3^T, dU3 = U2^T T + bu2 (x) t, dH1 = (U2 U3)^T dUH + (bu2 U3 + bu3) (x) dbuh,
//                                             dbu2 = t U3^T, dbu3 = t, dbh1 = dbuh
//   HO = H2 H3, bho = bh2 H3 + bh3         -> dH2 = dHO H3^T, dH3 = H2^T dHO + bh2 (x) dbho, dbh2 = dbho H3^T, dbh3 = dbho
static void unfold_jobs(int ed, int out_dim, const float* P, const float* blob, const float* Gf, float* G, float* scratch,
                        SmallJobList& JT, SmallJobList& J) {
    const ParamLayout L = make_layout(ed, out_dim);
    const InferLayout I = make_infer_layout(out_dim);
    const int no = out_dim;
    float* T = scratch;              // [256, 128]
    float* t = scratch + 256 * 128;  // [128]
    const float* H1 = P + L.w[L_HEAD0];     // [128, 256]
    JT.add(T, 256, 128, 256, Gf + I.uh, 256, 1, H1, 1, 256, nullptr, nullptr, nullptr, false);
    JT.add(t, 1, 128, 256, Gf + I.buh, 0, 1, H1, 1, 256, nullptr, nullptr, nullptr, false);
    const float* W2 = P + L.w[L_MSG1];      // [256, 256]
    const float* W3 = P + L.w[L_MSGOUT];    // [256, 128]
    J.add(G + L.w[L_MSG1], 256, 256, 128, Gf + I.w23, 128, 1, W3, 1, 128, nullptr, nullptr, nullptr, true);
    J.add(G + L.w[L_MSGOUT], 256, 128, 256, W2, 1, 256, Gf + I.w23, 128, 1, P + L.b[L_MSG1], Gf + I.b23, nullptr, true);
    J.add(G + L.b[L_MSG1], 1, 256, 128, Gf + I.b23, 0, 1, W3, 1, 128, nullptr, nullptr, nullptr, true);
    J.add(G + L.b[L_MSGOUT], 1, 128, 0, nullptr, 0, 0, nullptr, 0, 0, nullptr, nullptr, Gf + I.b23, true);
    const float* A2 = P + L.w[L_ATT1];      // [128, 128]
    const float* a3 = P + L.w[L_GATE];      // [128, 1]
    J.add(G + L.w[L_ATT1], 128, 128, 0, nullptr, 0, 0, nullptr, 0, 0, Gf + I.a23, a3, nullptr, true);
    J.add(G + L.w[L_GATE], 128, 1, 128, A2, 1, 128, Gf + I.a23, 1, 0, P + L.b[L_ATT1], Gf + I.c23, nullptr, true);
    J.add(G + L.b[L_ATT1], 1, 128, 0, nullptr, 0, 0, nullptr, 0, 0, Gf + I.c23, a3, nullptr, true);
    J.add(G + L.b[L_GATE], 1, 1, 0, nullptr, 0, 0, nullptr, 0, 0, nullptr, nullptr, Gf + I.c23, true);
    const float* U2 = P + L.w[L_UPD1];      // [256, 256]
    const float* U3 = P + L.w[L_UPDOUT];    // [256, 128]
    J.add(G + L.w[L_UPD1], 256, 256, 128, T, 128, 1, U3, 1, 128, nullptr, nullptr, nullptr, true);
    J.add(G + L.w[L_UPDOUT], 256, 128, 256, U2, 1, 256, T, 128, 1, P + L.b[L_UPD1], t, nullptr, true);
    J.add(G + L.w[L_HEAD0], 128, 256, 256, blob + I.q_u12, 1, 128, Gf + I.uh, 256, 1, blob + I.b_u12, Gf + I.buh, nullptr, true);
    J.add(G + L.b[L_UPD1], 1, 256, 128, t, 0, 1, U3, 1, 128, nullptr, nullptr, nullptr, true);
    J.add(G + L.b[L_UPDOUT], 1, 128, 0, nullptr, 0, 0, nullptr, 0, 0, nullptr, nullptr, t, true);
    J.add(G + L.b[L_HEAD0], 1, 256, 0, nullptr, 0, 0, nullptr, 0, 0, nullptr, nullptr, Gf + I.buh, true);
    const float* H2 = P + L.w[L_HEAD1];     // [256, 256]
    const float* H3 = P + L.w[L_OUT];       // [256, no]
    J.add(G + L.w[L_HEAD1], 256, 256, no, Gf + I.ho, no, 1, H3, 1, no, nullptr, nullptr, nullptr, true);
    J.add(G + L.w[L_OUT], 256, no, 256, H2, 1, 256, Gf + I.ho, no, 1, P + L.b[L_HEAD1], Gf + I.bho, nullptr, true);
    J.add(G + L.b[L_HEAD1], 1, 256, no, Gf + I.bho, 0, 1, H3, 1, no, nullptr, nullptr, nullptr, true);
    J.add(G + L.b[L_OUT], 1, no, 0, nullptr, 0, 0, nullptr, 0, 0, nullptr, nullptr, Gf + I.bho, true);
}

// ------------------------------------------------------------------------------------ optimizer kernels
// deterministic two-stage sum of squares (every rank must derive the SAME clip scale from the
// all-reduced gradient, so no float atomics here): SQN_BLOCKS partials, then an ordered tree.
constexpr int SQN_BLOCKS = 256;
__global__ void __launch_bounds__(256)
sqnorm_partial_kernel(const float* __restrict__ g, const int n, float* __restrict__ partial) {
    __shared__ float sh[2][256];
    float s = 0.f, bad = 0.f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float v = g[i];
        s = fmaf(v, v, s);
        bad += isfinite(v) ? 0.f : 1.f;
    }
    sh[0][threadIdx.x] = s;
    sh[1][threadIdx.x] = bad;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            sh[0][threadIdx.x] += sh[0][threadIdx.x + o];
            sh[1][threadIdx.x] += sh[1][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = sh[0][0];
        partial[SQN_BLOCKS + blockIdx.x] = sh[1][0];
    }
}
__global__ void __launch_bounds__(SQN_BLOCKS)
sqnorm_final_kernel(const float* __restrict__ partial, float* __restrict__ out) {
    __shared__ float sh[2][SQN_BLOCKS];
    sh[0][threadIdx.x] = partial[threadIdx.x];
    sh[1][threadIdx.x] = partial[SQN_BLOCKS + threadIdx.x];
    __syncthreads();
    for (int o = SQN_BLOCKS / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            sh[0][threadIdx.x] += sh[0][threadIdx.x + o];
            sh[1][threadIdx.x] += sh[1][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        out[0] = sh[0][0];
        out[1] = sh[1][0];
    }
}

// compute_norm_and_clip (trainer/utils.py:66-75) + optax.adamw + apply_if_finite.
// norm_info[0] = sum g^2, norm_info[1] = #non-finite; step[0] = optimizer step count (advanced by thread 0).
__global__ void __launch_bounds__(256)
clip_adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                  const int n, const float* __restrict__ norm_info, int32_t* __restrict__ step, const float lr,
                  const float b1, const float b2, const float eps, const float wd, const float max_norm) {
    if (norm_info[1] > 0.f || !isfinite(norm_info[0])) return;  // apply_if_finite: skip, state not advanced
    const int t = step[0] + 1;
    const float gnorm = sqrtf(norm_info[0]);
    const float denom = fmaxf(max_norm, gnorm);
    const float bc1 = 1.f - powf(b1, (float)t), bc2 = 1.f - powf(b2, (float)t);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float gi = (g[i] / denom) * max_norm;
        const float mi = b1 * m[i] + (1.f - b1) * gi;
        const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        const float mhat = mi / bc1, vhat = vi / bc2;
        p[i] = p[i] - lr * (mhat / (sqrtf(vhat) + eps) + wd * p[i]);
    }
}
__global__ void adamw_advance_kernel(const float* __restrict__ norm_info, int32_t* __restrict__ step) {
    if (!(norm_info[1] > 0.f || !isfinite(norm_info[0]))) step[0] += 1;
}

__global__ void polyak_kernel(float* __restrict__ tgt, const float* __restrict__ src, const int n, const float tau) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        tgt[i] = tau * src[i] + (1.f - tau) * tgt[i];
}

}  // namespace gcbf
#include "qp.cuh"
#include "refine.cuh"
namespace gcbf {

// ------------------------------------------------------------------------------------ QP label workspace layout
struct QpWs {
    int64_t ws0, gws, pt_cbf, h, ones, je, qb, qs, qe, ur, qsc, rev, total;
};
static QpWs make_qp_ws(const gcbf_env_desc* d) {
    const int ed = env_ed(d->env_kind);
    const int64_t A = (int64_t)d->n_graphs * d->n_agents, cap = d->edge_cap;
    const GnnWs W = make_ws(d->edge_cap, A);
    QpWs t;
    WsSlots S{8};   // 32-byte slots: 256-bit epilogue stores
    t.ws0 = S.take(W.total);
    t.gws = S.take(W.total);
    t.pt_cbf = S.take(make_plane_layout(make_deep_layout(ed, 1, 1), ed).total);   // also holds the SIMT TransLayout
    t.h = S.take(A);
    t.ones = S.take(A);
    t.je = S.take(cap * 8);
    t.qb = S.take(A);
    t.qs = S.take(A * 4);
    t.qe = S.take(cap * 4);
    t.ur = S.take(A * 4);
    t.qsc = S.take(A);
    t.rev = S.take(cap);
    t.total = S.off;
    return t;
}

__global__ void fill_kernel(float* __restrict__ p, const int n, const float v) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = v;
}

// ------------------------------------------------------------------------------------ train workspace layout
// One parameter region per network, holding what the step of its GEMM path needs: the SIMT step the transposed
// weights (TransLayout, at `pt`), the folded tensor-core step [folded blob (InferLayout) at `pt` | gradient of the
// folded weights at `gf` | un-fold scratch at `scr`].
struct TrainNetWs {
    int64_t pt, gf, scr;
};
struct TrainWs {
    int64_t ws0, ws1, ws2, gws;
    TrainNetWs net_cbf, net_act;
    int64_t h, hn, pi, act, xn, d_es, je, dh, dhn, da, dpi, lab, part, total;
};
static TrainWs make_train_ws(const gcbf_env_desc* d) {
    const int ed = env_ed(d->env_kind), nu = env_nu(d->env_kind), sd = env_sd(d->env_kind);
    const int64_t A = (int64_t)d->n_graphs * d->n_agents;
    const GnnWs W = make_ws(d->edge_cap, A);
    TrainWs t;
    WsSlots S{8};   // 32-byte slots: 256-bit epilogue stores
    auto take_net = [&](int out_dim) {
        const InferLayout I = make_infer_layout(out_dim);
        WsSlots F{8};   // the folded step's region
        F.take(I.total);
        const int64_t gf = F.take(I.t_w23), scr = F.take(UNFOLD_SCRATCH);
        const int64_t simt = make_trans_layout(make_layout(ed, out_dim)).total;
        TrainNetWs n;
        n.pt = S.take(simt > F.off ? simt : F.off);
        n.gf = n.pt + gf;
        n.scr = n.pt + scr;
        return n;
    };
    t.ws0 = S.take(W.total);
    t.ws1 = S.take(W.total);
    t.ws2 = S.take(W.total);
    t.gws = S.take(W.total);
    t.net_cbf = take_net(1);
    t.net_act = take_net(nu);
    t.h = S.take(A);
    t.hn = S.take(A);
    t.pi = S.take(A * nu);
    t.act = S.take(A * nu);
    t.xn = S.take(A * sd);
    t.d_es = S.take(A * ed);
    t.je = S.take((int64_t)d->edge_cap * 8);
    t.dh = S.take(A);
    t.dhn = S.take(A);
    t.da = S.take(A * nu);
    t.dpi = S.take(A * nu);
    t.lab = S.take(A);
    t.part = S.take(PART_FLOATS);
    t.total = S.off;
    return t;
}

}  // namespace gcbf

using namespace gcbf;

extern "C" __attribute__((visibility("default"))) int64_t gcbf_train_workspace_floats(const gcbf_env_desc* desc) {
    return graph_desc_ok(desc) ? make_train_ws(desc).total : -1;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_mask_counts(const uint8_t* safe_mask,
                                                                           const uint8_t* unsafe_mask,
                                                                           int32_t n_agents_total, float* denoms,
                                                                           void* stream) {
    GCBF_REQUIRE(safe_mask && unsafe_mask && denoms && n_agents_total > 0, "gcbf_mask_counts: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(denoms, 0, 4 * sizeof(float), st);
    if (e != cudaSuccess) { set_error("cudaMemsetAsync: %s", cudaGetErrorString(e)); return (int32_t)e; }
    mask_count_kernel<<<min((n_agents_total + 255) / 256, 2 * sm_count()), 256, 0, st>>>(n_agents_total, safe_mask,
                                                                                         unsafe_mask, denoms);
    count_launch();
    return check_launch("mask_count_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_train_step(
    const gcbf_env_desc* desc, const float* hp_host, const float* cbf_params, const float* actor_params,
    const float* agent, const float* goal, const float* hits, const int32_t* row_start, const int32_t* row_deg,
    const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters, const uint8_t* safe_mask,
    const uint8_t* unsafe_mask, const float* u_qp, const float* denoms, float* grad_cbf, float* grad_actor,
    float* stats, float* workspace, int64_t workspace_floats, void* stream) {
    GCBF_REQUIRE(desc && hp_host && cbf_params && actor_params && agent && goal && hits && row_start && row_deg &&
                     edge_recv && edge_src && counters && safe_mask && unsafe_mask && u_qp && denoms && grad_cbf &&
                     grad_actor && stats && workspace, "gcbf_train_step: NULL pointer argument");
    if (int32_t rc = check_graph_desc(desc, "gcbf_train_step")) return rc;
    const TrainWs TW = make_train_ws(desc);
    GCBF_REQUIRE(workspace_floats >= TW.total, "train workspace too small: %lld < %lld floats",
                 (long long)workspace_floats, (long long)TW.total);
    GCBF_REQUIRE(((uintptr_t)workspace & 15) == 0 && ((uintptr_t)cbf_params & 15) == 0 &&
                     ((uintptr_t)actor_params & 15) == 0 && ((uintptr_t)grad_cbf & 15) == 0 &&
                     ((uintptr_t)grad_actor & 15) == 0, "buffers must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const gcbf_env_desc* d = desc;
    const int ed = env_ed(d->env_kind), nu = env_nu(d->env_kind);
    const int A = d->n_graphs * d->n_agents;
    const ParamLayout Lc = make_layout(ed, 1), La = make_layout(ed, nu);
    float* ws = workspace;
    TrainHP hp;
    hp.alpha = hp_host[0];
    hp.eps = hp_host[1];
    hp.c_action = hp_host[2];
    hp.c_unsafe = hp_host[3];
    hp.c_safe = hp_host[4];
    hp.c_hdot = hp_host[5];
    hp.dt_inv = 1.f / d->dt;
    int32_t rc;
#define RC(x) do { if ((rc = (x))) return rc; } while (0)
    cudaError_t e;
    if ((e = cudaMemsetAsync(grad_cbf, 0, sizeof(float) * Lc.total, st)) != cudaSuccess ||
        (e = cudaMemsetAsync(grad_actor, 0, sizeof(float) * La.total, st)) != cudaSuccess ||
        (e = cudaMemsetAsync(stats, 0, sizeof(float) * 16, st)) != cudaSuccess) {
        set_error("cudaMemsetAsync: %s", cudaGetErrorString(e));
        return (int32_t)e;
    }
    // tensor-core path: the folded step; SIMT path: the layer-by-layer step (see TrainWs for the parameter regions)
    const int use_tc = hp_host[6] != 0.f;
    float* blob_c = ws + TW.net_cbf.pt;
    float* blob_a = ws + TW.net_act.pt;
    float* gf_c = ws + TW.net_cbf.gf;
    float* gf_a = ws + TW.net_act.gf;
    if (use_tc) {
        RC(prepare_infer_pair(ed, 1, cbf_params, blob_c, nu, actor_params, blob_a, st));
        if ((e = cudaMemsetAsync(gf_c, 0, sizeof(float) * make_infer_layout(1).t_w23, st)) != cudaSuccess ||
            (e = cudaMemsetAsync(gf_a, 0, sizeof(float) * make_infer_layout(nu).t_w23, st)) != cudaSuccess) {
            set_error("cudaMemsetAsync: %s", cudaGetErrorString(e));
            return (int32_t)e;
        }
    } else {
        RC(prepare_bwd_operands(ed, 1, 0, cbf_params, blob_c, st));
        RC(prepare_bwd_operands(ed, nu, 0, actor_params, blob_a, st));
    }
    // ---- forward: h = cbf(g), pi = actor(g), x' = f(x, clip(2 pi + u_ref)), h' = cbf(g')
    const GraphRefs g{agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters};
    const GraphRefs gn = g.with_agent(ws + TW.xn);
    auto forward = [&](int out_dim, const float* params, const float* blob, const GraphRefs& gr, int clip_all,
                       float* out, float* fws) -> int32_t {
        if (use_tc)
            return gnn_infer_impl(d, out_dim, params, blob, 1, gr, clip_all, out, fws, st, nullptr, nullptr, nullptr,
                                  0xF, 1);
        return gnn_forward(d, out_dim, 1, params, nullptr, gr, clip_all, out, nullptr, fws, st);
    };
    RC(forward(1, cbf_params, blob_c, g, 0, ws + TW.h, ws + TW.ws0));
    RC(forward(nu, actor_params, blob_a, g, 0, ws + TW.pi, ws + TW.ws1));
    GCBF_DISPATCH_ENV(d->env_kind, {
        act_dyn_kernel<KIND><<<(A + 127) / 128, 128, 0, st>>>(*d, agent, goal, ws + TW.pi, ws + TW.act, ws + TW.xn);
    });
    count_launch();
    RC(check_launch("act_dyn_kernel"));
    RC(forward(1, cbf_params, blob_c, gn, 1, ws + TW.hn, ws + TW.ws2));
    // ---- losses and their derivatives wrt h, h', a
    {
        const int grid = min((A + 255) / 256, 2 * sm_count());
        if (nu == 2)
            loss_kernel<2><<<grid, 256, 0, st>>>(A, hp, ws + TW.h, ws + TW.hn, safe_mask, unsafe_mask, ws + TW.act, u_qp,
                                                 denoms, ws + TW.dh, ws + TW.dhn, ws + TW.da, ws + TW.lab, ws + TW.part);
        else
            loss_kernel<3><<<grid, 256, 0, st>>>(A, hp, ws + TW.h, ws + TW.hn, safe_mask, unsafe_mask, ws + TW.act, u_qp,
                                                 denoms, ws + TW.dh, ws + TW.dhn, ws + TW.da, ws + TW.lab, ws + TW.part);
        count_launch();
        RC(check_launch("loss_kernel"));
        RC(launch_partial_sum(ws + TW.part, 10, grid, PartSegs().add(stats, 10), st));
    }
    auto backward = [&](const BwdArgs& b, const float* blob, float* gf) -> int32_t {
        return use_tc ? gnn_backward_folded(b, blob, gf, st) : gnn_backward_impl(b, st);
    };
    float* const gw = ws + TW.gws;
    float* const part = ws + TW.part;
    // ---- backward 1: cbf on g' (dW only from labelled receivers; dX from all) -> d_es
    RC(backward({d, gn, gw, part, use_tc, 1, cbf_params, blob_c, ws + TW.ws2, ws + TW.hn, ws + TW.dhn, ws + TW.lab,
                 grad_cbf, 1, ws + TW.d_es, ws + TW.je}, blob_c, gf_c));
    // ---- through the Euler step / clips into the policy output
    GCBF_DISPATCH_ENV(d->env_kind, {
        dyn_bwd_kernel<KIND><<<(A + 127) / 128, 128, 0, st>>>(*d, agent, goal, ws + TW.act, ws + TW.xn, ws + TW.d_es,
                                                              ws + TW.da, ws + TW.dpi);
    });
    count_launch();
    RC(check_launch("dyn_bwd_kernel"));
    // ---- backward 2: actor on g
    RC(backward({d, g, gw, part, use_tc, nu, actor_params, blob_a, ws + TW.ws1, ws + TW.pi, ws + TW.dpi, nullptr,
                 grad_actor, 0, nullptr, nullptr}, blob_a, gf_a));
    // ---- backward 3: cbf on g
    RC(backward({d, g, gw, part, use_tc, 1, cbf_params, blob_c, ws + TW.ws0, ws + TW.h, ws + TW.dh, nullptr, grad_cbf, 0,
                 nullptr, nullptr}, blob_c, gf_c));
    if (use_tc) {
        SmallJobList JT, JU;      // both networks share the two un-fold launches
        unfold_jobs(ed, 1, cbf_params, blob_c, gf_c, grad_cbf, ws + TW.net_cbf.scr, JT, JU);
        unfold_jobs(ed, nu, actor_params, blob_a, gf_a, grad_actor, ws + TW.net_act.scr, JT, JU);
        RC(JT.launch(st));
        RC(JU.launch(st));
    }
#undef RC
    return 0;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_grad_sqnorm(const float* grad, int32_t n, float* out,
                                                                           void* stream) {
    GCBF_REQUIRE(grad && out && n > 0, "gcbf_grad_sqnorm: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    sqnorm_partial_kernel<<<SQN_BLOCKS, 256, 0, st>>>(grad, n, out + 2);
    count_launch();
    if (int32_t rc = check_launch("sqnorm_partial_kernel")) return rc;
    sqnorm_final_kernel<<<1, SQN_BLOCKS, 0, st>>>(out + 2, out);
    count_launch();
    return check_launch("sqnorm_final_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_clip_adamw(float* params, const float* grad, float* m,
                                                                          float* v, int32_t n,
                                                                          const float* norm_info, int32_t* step,
                                                                          float lr, float b1, float b2, float eps,
                                                                          float wd, float max_norm, void* stream) {
    GCBF_REQUIRE(params && grad && m && v && norm_info && step && n > 0, "gcbf_clip_adamw: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    clip_adamw_kernel<<<min((n + 1023) / 1024, 2 * sm_count()), 256, 0, st>>>(params, grad, m, v, n, norm_info, step, lr,
                                                                             b1, b2, eps, wd, max_norm);
    count_launch();
    if (int32_t rc = check_launch("clip_adamw_kernel")) return rc;
    adamw_advance_kernel<<<1, 1, 0, st>>>(norm_info, step);
    count_launch();
    return check_launch("adamw_advance_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_polyak(float* tgt, const float* src, int32_t n,
                                                                      float tau, void* stream) {
    GCBF_REQUIRE(tgt && src && n > 0, "gcbf_polyak: bad argument");
    polyak_kernel<<<min((n + 1023) / 1024, 2 * sm_count()), 256, 0, (cudaStream_t)stream>>>(tgt, src, n, tau);
    count_launch();
    return check_launch("polyak_kernel");
}

// ------------------------------------------------------------------------------------ QP action labels
extern "C" __attribute__((visibility("default"))) int64_t gcbf_qp_workspace_floats(const gcbf_env_desc* desc) {
    return graph_desc_ok(desc) ? make_qp_ws(desc).total : -1;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_qp_workspace_layout(const gcbf_env_desc* desc,
                                                                                   int64_t* offsets8_host) {
    GCBF_REQUIRE(offsets8_host, "gcbf_qp_workspace_layout: bad argument");
    if (int32_t rc = check_graph_desc(desc, "gcbf_qp_workspace_layout")) return rc;
    const QpWs Q = make_qp_ws(desc);
    const int64_t o[8] = {Q.h, Q.je, Q.qb, Q.qs, Q.qe, Q.ur, Q.qsc, Q.rev};
    for (int i = 0; i < 8; ++i) offsets8_host[i] = o[i];
    return 0;
}

// The QP of the labels with the nominal action u_nom in place of u_ref (u_nom == NULL: u_ref, the labels themselves).
static int32_t qp_solve(const char* name, const gcbf_env_desc* desc, float alpha, int32_t use_tensor_cores,
                        int32_t max_iter, float tol, const float* cbf_params, const float* agent, const float* goal,
                        const float* hits, const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv,
                        const int32_t* edge_src, const int32_t* counters, const float* u_nom, float* u_qp, float* aux,
                        int32_t* iters, float* workspace, int64_t workspace_floats, void* stream) {
    GCBF_REQUIRE(desc && cbf_params && agent && goal && hits && row_start && row_deg && edge_recv && edge_src &&
                     counters && u_qp && workspace, "%s: NULL pointer argument", name);
    if (int32_t rc = check_graph_desc(desc, name)) return rc;
    GCBF_REQUIRE(desc->n_agents <= QP_MAX_AGENTS, "%s: n_agents %d > %d not supported", name, desc->n_agents,
                 QP_MAX_AGENTS);
    GCBF_REQUIRE(max_iter > 0 && tol >= 0.f, "%s: bad solver settings", name);
    const QpWs Q = make_qp_ws(desc);
    GCBF_REQUIRE(workspace_floats >= Q.total, "qp workspace too small: %lld < %lld floats", (long long)workspace_floats,
                 (long long)Q.total);
    GCBF_REQUIRE(((uintptr_t)workspace & 15) == 0 && ((uintptr_t)cbf_params & 15) == 0, "buffers must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const gcbf_env_desc* d = desc;
    const int ed = env_ed(d->env_kind), nu = env_nu(d->env_kind);
    const int A = d->n_graphs * d->n_agents, N = d->n_agents;
    float* ws = workspace;
    const GraphRefs g{agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters};
    int32_t rc;
#define RC(x) do { if ((rc = (x))) return rc; } while (0)
    RC(prepare_bwd_operands(ed, 1, use_tensor_cores, cbf_params, ws + Q.pt_cbf, st));
    // h = cbf(add_edge_feats(graph, x)): every edge feature norm-clipped (gcbf_plus.py:310-316)
    RC(gnn_forward(d, 1, 1, cbf_params, use_tensor_cores ? ws + Q.pt_cbf : nullptr, g, 1, ws + Q.h, nullptr, ws + Q.ws0,
                   st));
    fill_kernel<<<min((A + 255) / 256, 2 * sm_count()), 256, 0, st>>>(ws + Q.ones, A, 1.f);
    count_launch();
    RC(check_launch("fill_kernel"));
    // Jacobian: data-only backward with upstream 1, kept per edge
    RC(gnn_backward_impl({d, g, ws + Q.gws, nullptr, use_tensor_cores, 1, cbf_params, ws + Q.pt_cbf, ws + Q.ws0, ws + Q.h,
                          ws + Q.ones, nullptr, nullptr, 1, nullptr, ws + Q.je}, st));
    int32_t* rev = reinterpret_cast<int32_t*>(ws + Q.rev);
    GCBF_DISPATCH_ENV(d->env_kind, {
        qp_assemble_kernel<KIND><<<(A + 127) / 128, 128, 0, st>>>(*d, alpha, agent, goal, ws + Q.h, ws + Q.je, row_start,
                                                                  row_deg, edge_src, u_nom, ws + Q.qb, ws + Q.qs,
                                                                  ws + Q.qe, ws + Q.ur, ws + Q.qsc, rev);
    });
    count_launch();
    RC(check_launch("qp_assemble_kernel"));
    const int nt = min(1024, (N + 31) / 32 * 32);
    // compacted agent-agent blocks per graph kept in shared memory: N (N - 1) at most, 24 per agent is generous for
    // radius graphs, and whatever fits under the 227 KB limit; denser graphs iterate on the global edge list.
    int nbr_cap = (int)min((int64_t)N * (N - 1), (int64_t)24 * N);
    const size_t smem_base = qp_solve_smem(N, nu, 0), entry = sizeof(int) + 2 * nu * sizeof(float);
    const size_t smem_max = 200 * 1024;
    if (smem_base + (size_t)nbr_cap * entry > smem_max) nbr_cap = (int)((smem_max - smem_base) / entry);
    nbr_cap = max(nbr_cap, 1);
    const size_t smem = qp_solve_smem(N, nu, nbr_cap);
    cudaError_t e;
#define QP_LAUNCH(NUv)                                                                                                  \
    do {                                                                                                                \
        if ((e = cudaFuncSetAttribute(qp_solve_kernel<NUv>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) !=  \
            cudaSuccess) {                                                                                              \
            set_error("cudaFuncSetAttribute(qp_solve_kernel): %s", cudaGetErrorString(e));                              \
            return (int32_t)e;                                                                                          \
        }                                                                                                               \
        qp_solve_kernel<NUv><<<d->n_graphs, nt, smem, st>>>(N, d->edge_cap, nbr_cap, d->u_lim, max_iter, tol, ws + Q.qb,  \
                                                            ws + Q.qs, ws + Q.qe, ws + Q.ur, ws + Q.qsc, rev, row_start, \
                                                            row_deg, edge_src, u_qp, aux, iters);                       \
    } while (0)
    if (nu == 2) QP_LAUNCH(2);
    else QP_LAUNCH(3);
#undef QP_LAUNCH
    count_launch();
    RC(check_launch("qp_solve_kernel"));
#undef RC
    return 0;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_qp_labels(
    const gcbf_env_desc* desc, float alpha, int32_t use_tensor_cores, int32_t max_iter, float tol,
    const float* cbf_params, const float* agent, const float* goal, const float* hits, const int32_t* row_start,
    const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters, float* u_qp,
    float* aux, int32_t* iters, float* workspace, int64_t workspace_floats, void* stream) {
    return qp_solve("gcbf_qp_labels", desc, alpha, use_tensor_cores, max_iter, tol, cbf_params, agent, goal, hits,
                    row_start, row_deg, edge_recv, edge_src, counters, nullptr, u_qp, aux, iters, workspace,
                    workspace_floats, stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_qp_filter(
    const gcbf_env_desc* desc, float alpha, int32_t use_tensor_cores, int32_t max_iter, float tol,
    const float* cbf_params, const float* agent, const float* goal, const float* hits, const int32_t* row_start,
    const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters,
    const float* u_nom, float* u, float* aux, int32_t* iters, float* workspace, int64_t workspace_floats,
    void* stream) {
    return qp_solve("gcbf_qp_filter", desc, alpha, use_tensor_cores, max_iter, tol, cbf_params, agent, goal, hits,
                    row_start, row_deg, edge_recv, edge_src, counters, u_nom, u, aux, iters, workspace,
                    workspace_floats, stream);
}

// ------------------------------------------------------------------------------------ online policy refinement
extern "C" __attribute__((visibility("default"))) int32_t gcbf_refine_prepare(int32_t edge_dim, int32_t use_tensor_cores,
                                                                              const float* cbf_params, float* prepared,
                                                                              void* stream) {
    GCBF_REQUIRE(cbf_params && prepared && (edge_dim == 2 || edge_dim == 4 || edge_dim == 6),
                 "gcbf_refine_prepare: bad argument");
    GCBF_REQUIRE((((uintptr_t)cbf_params | (uintptr_t)prepared) & 15) == 0, "buffers must be 16-byte aligned");
    return prepare_bwd_operands(edge_dim, 1, use_tensor_cores, cbf_params, prepared, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int64_t gcbf_refine_workspace_floats(const gcbf_env_desc* desc) {
    return graph_desc_ok(desc) ? make_refine_ws(desc).total : -1;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_refine_actions(
    const gcbf_env_desc* desc, float alpha, float lr, int32_t max_iter, int32_t use_tensor_cores,
    const float* cbf_params, const float* cbf_prepared, const float* pi, const float* agent, const float* goal,
    const float* hits, const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv,
    const int32_t* edge_src, const int32_t* counters, float* action, float* value, int32_t* iters, float* workspace,
    int64_t workspace_floats, void* stream) {
    GCBF_REQUIRE(desc && cbf_params && cbf_prepared && pi && agent && goal && hits && row_start && row_deg &&
                     edge_recv && edge_src && counters && action && workspace, "gcbf_refine_actions: NULL pointer argument");
    if (int32_t rc = check_graph_desc(desc, "gcbf_refine_actions")) return rc;
    GCBF_REQUIRE(desc->dt > 0.f, "gcbf_refine_actions: bad descriptor (dt %g)", (double)desc->dt);
    GCBF_REQUIRE(max_iter > 0 && isfinite(lr) && isfinite(alpha), "gcbf_refine_actions: bad settings (max_iter %d)",
                 max_iter);
    const RefineWs R = make_refine_ws(desc);
    GCBF_REQUIRE(workspace_floats >= R.total, "refine workspace too small: %lld < %lld floats",
                 (long long)workspace_floats, (long long)R.total);
    GCBF_REQUIRE((((uintptr_t)workspace | (uintptr_t)cbf_params | (uintptr_t)cbf_prepared) & 15) == 0,
                 "buffers must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const gcbf_env_desc* d = desc;
    const int nu = env_nu(d->env_kind);
    const int G = d->n_graphs, N = d->n_agents, A = G * N;
    const int blocks = (A + 127) / 128;
    float* ws = workspace;
    int32_t* active = reinterpret_cast<int32_t*>(ws + R.active);
    int32_t* upd = reinterpret_cast<int32_t*>(ws + R.upd);
    int32_t* rows = reinterpret_cast<int32_t*>(ws + R.rows);
    const float* PT = cbf_prepared;
    int32_t rc;
#define RC(x) do { if ((rc = (x))) return rc; } while (0)
    // g: the graph; gn: its edges over the next states x'; gr: the same with the refinement steps' device edge count
    const GraphRefs g{agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters};
    const GraphRefs gn = g.with_agent(ws + R.xn);
    GraphRefs gr = gn;
    gr.counters = rows;
    auto forward = [&](const GraphRefs& on, int clip_all, const int32_t* arows, float* out) -> int32_t {
        return gnn_forward(d, 1, 1, cbf_params, use_tensor_cores ? PT : nullptr, on, clip_all, out, nullptr, ws + R.fw,
                           st, arows);
    };
    // 1. h = cbf(g) on the graph's own edge features
    RC(forward(g, 0, nullptr, ws + R.h));
    // 2. h(g'(u_ref)), every edge feature recomputed and norm-clipped (forward_graph)
    GCBF_DISPATCH_ENV(d->env_kind, {
        refine_next_state_kernel<KIND><<<blocks, 128, 0, st>>>(*d, nullptr, agent, goal, nullptr, ws + R.ur, ws + R.xn);
    });
    count_launch();
    RC(check_launch("refine_next_state_kernel"));
    RC(forward(gn, 1, nullptr, ws + R.hn));
    // 3. per-agent selection of the starting action; every graph active
    if (nu == 2)
        refine_init_kernel<2><<<blocks, 128, 0, st>>>(G, A, alpha, d->dt, ws + R.h, ws + R.hn, ws + R.ur, pi, counters,
                                                      action, active, rows);
    else
        refine_init_kernel<3><<<blocks, 128, 0, st>>>(G, A, alpha, d->dt, ws + R.h, ws + R.hn, ws + R.ur, pi, counters,
                                                      action, active, rows);
    count_launch();
    RC(check_launch("refine_init_kernel"));
    // 4. the refinement steps: data-only backward of h' into the edge-state gradient of x' (same as the QP labels'
    //    Jacobian pass, gathered per agent), then the chain into the action
    const BwdArgs b{d, gr, ws + R.gw, nullptr, use_tensor_cores, 1, cbf_params, PT, ws + R.fw, ws + R.hn, ws + R.dhn,
                    nullptr, nullptr, 1, ws + R.d_es, ws + R.je, rows + 1};
    for (int it = 0; it < max_iter; ++it) {
        GCBF_DISPATCH_ENV(d->env_kind, {
            refine_next_state_kernel<KIND><<<blocks, 128, 0, st>>>(*d, rows, agent, goal, action, nullptr, ws + R.xn);
        });
        count_launch();
        RC(check_launch("refine_next_state_kernel"));
        RC(forward(gr, 1, rows + 1, ws + R.hn));
        refine_value_kernel<<<G, REFINE_VALUE_THREADS, 0, st>>>(N, env_sd(d->env_kind), alpha, d->dt, it, max_iter,
                                                                ws + R.h, ws + R.hn, ws + R.xn, ws + R.dhn, active,
                                                                upd, value, iters);
        count_launch();
        RC(check_launch("refine_value_kernel"));
        RC(gnn_backward_impl(b, st));
        GCBF_DISPATCH_ENV(d->env_kind, {
            refine_update_kernel<KIND><<<blocks, 128, 0, st>>>(*d, lr, agent, goal, ws + R.xn, ws + R.d_es, active, upd,
                                                               counters, rows, action);
        });
        count_launch();
        RC(check_launch("refine_update_kernel"));
    }
#undef RC
    return 0;
}
