// gnn.cu -- GNN forward for one network (CBF h(x) or policy pi(x)) over a swarm batch.
#include "gemm.cuh"
#include "gemm_tc.cuh"
#include "gnn.cuh"
#include "gemm_tc_prod.cuh"
#include "translayout.cuh"
#include "smalljobs.cuh"
#include "internal.cuh"

using namespace gcbf;

// ---- building blocks exported for unit tests and for bench.py's isolated kernel timing ----
extern "C" __attribute__((visibility("default"))) int32_t gcbf_gemm_nn(int32_t epi, int32_t accum, const float* A,
                                                                       const float* B, const float* bias,
                                                                       const float* bias2, float* C, const float* aux,
                                                                       const int32_t* m_ptr, int32_t m_fixed,
                                                                       int32_t m_cap, int32_t K, int32_t N,
                                                                       void* stream) {
    GCBF_REQUIRE(A && B && C, "gcbf_gemm_nn: NULL pointer");
    GCBF_REQUIRE((epi != EPI_BIAS && epi != EPI_BIAS_RELU) || bias, "gcbf_gemm_nn: bias required");
    GCBF_REQUIRE(epi != EPI_RELU_MASK || aux, "gcbf_gemm_nn: aux required");
    return launch_gemm_nn(epi, accum != 0, A, B, bias, bias2, C, aux, RowCount{m_ptr, m_fixed, m_cap}, K, N,
                          (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_gemm_tn(const float* X, int32_t ldx, const float* dY,
                                                                       float* C, const float* roww,
                                                                       const int32_t* row2agent, const int32_t* m_ptr,
                                                                       int32_t m_fixed, int32_t m_cap, int32_t K1,
                                                                       int32_t N, int32_t n_agents_total, void* stream) {
    GCBF_REQUIRE(X && dY && C, "gcbf_gemm_tn: NULL pointer");
    return launch_gemm_tn(X, ldx, dY, C, roww, row2agent, RowCount{m_ptr, m_fixed, m_cap}, K1, N, n_agents_total,
                          (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_colsum(const float* dY, float* db, const float* roww,
                                                                      const int32_t* row2agent, const int32_t* m_ptr,
                                                                      int32_t m_fixed, int32_t m_cap, int32_t N,
                                                                      int32_t n_agents_total, void* stream) {
    GCBF_REQUIRE(dY && db, "gcbf_colsum: NULL pointer");
    return launch_colsum(dY, db, roww, row2agent, RowCount{m_ptr, m_fixed, m_cap}, N, n_agents_total,
                         (cudaStream_t)stream);
}

// ---- tensor-core (wgmma 3xTF32) variant of gcbf_gemm_nn: C = epi(A[M,K] @ Bt[N,K]^T) ----
extern "C" __attribute__((visibility("default"))) int32_t gcbf_gemm_tc(int32_t epi, int32_t accum, const float* A,
                                                                       const float* Bt_hi, const float* Bt_lo,
                                                                       const float* bias,
                                                                       const float* bias2, float* C, const float* aux,
                                                                       const int32_t* m_ptr, int32_t m_fixed,
                                                                       int32_t m_cap, int32_t K, int32_t N,
                                                                       int32_t ndot, void* stream) {
    GCBF_REQUIRE(A && Bt_hi && Bt_lo && C, "gcbf_gemm_tc: NULL pointer");
    GCBF_REQUIRE(epi != EPI_RELU_DOTN || (bias && aux), "gcbf_gemm_tc: bias and aux required");
    GCBF_REQUIRE(epi != EPI_RELU_DOTN || (ndot >= 1 && ndot <= 4), "gcbf_gemm_tc: ndot must be in [1, 4]");
    GCBF_REQUIRE((epi != EPI_BIAS && epi != EPI_BIAS_RELU) || bias, "gcbf_gemm_tc: bias required");
    GCBF_REQUIRE(epi != EPI_RELU_MASK || aux, "gcbf_gemm_tc: aux required");
    GCBF_REQUIRE((((uintptr_t)A | (uintptr_t)Bt_hi | (uintptr_t)Bt_lo | (uintptr_t)C) & 15) == 0,
                 "gcbf_gemm_tc: 16-byte alignment required");
    return gcbf::tc::launch_gemm_tc(epi, accum != 0, A, Bt_hi, Bt_lo, bias, bias2, C, aux,
                                    RowCount{m_ptr, m_fixed, m_cap}, K, N, (cudaStream_t)stream, ndot);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_split_tf32(const float* in, float* hi, float* lo, int32_t n,
                                                                          void* stream) {
    GCBF_REQUIRE(in && hi && lo && n > 0, "gcbf_split_tf32: bad argument");
    gcbf::tc::split_tf32_kernel<<<min((n + 255) / 256, 4 * sm_count()), 256, 0, (cudaStream_t)stream>>>(in, hi, lo, n);
    count_launch();
    return check_launch("split_tf32_kernel");
}
extern "C" __attribute__((visibility("default"))) int32_t gcbf_gemm_tn_tc(const float* X, int32_t ldx, const float* dY,
                                                                          float* C, const float* roww,
                                                                          const int32_t* row2agent,
                                                                          const int32_t* m_ptr, int32_t m_fixed,
                                                                          int32_t m_cap, int32_t K1, int32_t N,
                                                                          int32_t n_agents_total, float* cs1, float* cs2,
                                                                          void* stream) {
    GCBF_REQUIRE(X && dY && C, "gcbf_gemm_tn_tc: NULL pointer");
    GCBF_REQUIRE(cs1 || !cs2, "gcbf_gemm_tn_tc: cs2 without cs1");
    GCBF_REQUIRE((((uintptr_t)X | (uintptr_t)dY | (uintptr_t)C) & 15) == 0, "gcbf_gemm_tn_tc: 16-byte alignment required");
    return gcbf::tc::launch_gemm_tn_tc(X, ldx, dY, C, roww, row2agent, RowCount{m_ptr, m_fixed, m_cap}, K1, N,
                                       n_agents_total, (cudaStream_t)stream, cs1, cs2);
}

// =====================================================================================================
// Inference path with folded weights.  Every MLP block of the GNN ends in two linear layers with no
// activation in between (act_final=False, gcbfplus/nn/mlp.py:23-29; SURVEY A.3), so for rollouts
//   msg   = relu1 @ (W2 W3) + (b2 W3 + b3)                      256 -> 128
//   gate  = relu(msg A1 + ba1) . (A2 a3) + (ba2 . a3 + ba3)     128 -> 128 -> 1
//   h1    = relu(relu(aggr U1' + bu1') @ (U2 U3 H1) + ((bu2 U3 + bu3) H1 + bh1))   128 -> 256 -> 256
//   out   = tanh(h1 @ (H2 H3) + (bh2 H3 + bh3))                 256 -> nu
// 4 GEMMs + 3 small kernels per forward instead of 9 + 3, 2.4x fewer FLOPs.  The folded weights are
// rebuilt from the training parameters by gcbf_prepare_infer (once per parameter update).
// =====================================================================================================
namespace gcbf {

// Folded weights + operand planes: two dependency waves of small products, then all planes.  The jobs of several
// networks can share the three launches (prepare_infer_pair: both networks of the train step).
static void prepare_infer_jobs(int ed, int out_dim, const float* P, float* blob, SmallJobList& J1, SmallJobList& J2,
                               PlaneJobList& PJ) {
    const ParamLayout L = make_layout(ed, out_dim);
    const InferLayout I = make_infer_layout(out_dim);
    // message tail: W23 = W2 W3, b23 = b2 W3 + b3
    J1.add(blob + I.w23, 256, 128, 256, P + L.w[L_MSG1], 256, 1, P + L.w[L_MSGOUT], 128, 1, nullptr, nullptr, nullptr, false);
    J1.add(blob + I.b23, 1, 128, 256, P + L.b[L_MSG1], 0, 1, P + L.w[L_MSGOUT], 128, 1, nullptr, nullptr, P + L.b[L_MSGOUT], false);
    // gate tail: a23 = A2 a3 ; c = ba2 . a3 + ba3
    J1.add(blob + I.a23, 128, 1, 128, P + L.w[L_ATT1], 128, 1, P + L.w[L_GATE], 1, 1, nullptr, nullptr, nullptr, false);
    J1.add(blob + I.c23, 1, 1, 128, P + L.b[L_ATT1], 0, 1, P + L.w[L_GATE], 1, 1, nullptr, nullptr, P + L.b[L_GATE], false);
    // update tail: Q = U2 U3, b' = bu2 U3 + bu3
    J1.add(blob + I.q_u12, 256, 128, 256, P + L.w[L_UPD1], 256, 1, P + L.w[L_UPDOUT], 128, 1, nullptr, nullptr, nullptr, false);
    J1.add(blob + I.b_u12, 1, 128, 256, P + L.b[L_UPD1], 0, 1, P + L.w[L_UPDOUT], 128, 1, nullptr, nullptr, P + L.b[L_UPDOUT], false);
    // head tail: HO = H2 H3, bho = bh2 H3 + bh3
    J1.add(blob + I.ho, 256, out_dim, 256, P + L.w[L_HEAD1], 256, 1, P + L.w[L_OUT], out_dim, 1, nullptr, nullptr, nullptr, false);
    J1.add(blob + I.bho, 1, out_dim, 256, P + L.b[L_HEAD1], 0, 1, P + L.w[L_OUT], out_dim, 1, nullptr, nullptr, P + L.b[L_OUT], false);
    // update tail folded into the head's first layer: UH = Q H1, buh = b' H1 + bh1
    J2.add(blob + I.uh, 256, 256, 128, blob + I.q_u12, 128, 1, P + L.w[L_HEAD0], 256, 1, nullptr, nullptr, nullptr, false);
    J2.add(blob + I.buh, 1, 256, 128, blob + I.b_u12, 0, 1, P + L.w[L_HEAD0], 256, 1, nullptr, nullptr, P + L.b[L_HEAD0], false);
    // tf32 planes: transposed (forward B operands) and straight (backward-data B operands) of the 4 GEMM weights
    struct { const float* src; int rows, cols, t, p; } T[4] = {
        {blob + I.w23, 256, 128, I.t_w23, I.p_w23}, {P + L.w[L_ATT0], 128, 128, I.t_a1, I.p_a1},
        {P + L.w[L_UPD0] + 3 * 256, 128, 256, I.t_u1, I.p_u1}, {blob + I.uh, 256, 256, I.t_uh, I.p_uh}};
    for (int i = 0; i < 4; ++i) {
        const int n = T[i].rows * T[i].cols;
        PJ.add(T[i].src, T[i].rows, T[i].cols, true, blob + T[i].t, blob + T[i].t + n);
        PJ.add(T[i].src, T[i].rows, T[i].cols, false, blob + T[i].p, blob + T[i].p + n);
    }
}
static int32_t prepare_infer_launch(SmallJobList& J1, SmallJobList& J2, PlaneJobList& PJ, cudaStream_t st) {
    if (int32_t rc = J1.launch(st)) return rc;
    if (int32_t rc = J2.launch(st)) return rc;
    return PJ.launch(st);
}
int32_t prepare_infer_impl(int ed, int out_dim, const float* P, float* blob, cudaStream_t st) {
    SmallJobList J1, J2;
    PlaneJobList PJ;
    prepare_infer_jobs(ed, out_dim, P, blob, J1, J2, PJ);
    return prepare_infer_launch(J1, J2, PJ, st);
}
int32_t prepare_infer_pair(int ed, int out_a, const float* Pa, float* blob_a, int out_b, const float* Pb, float* blob_b,
                           cudaStream_t st) {
    SmallJobList J1, J2;
    PlaneJobList PJ;
    prepare_infer_jobs(ed, out_a, Pa, blob_a, J1, J2, PJ);
    prepare_infer_jobs(ed, out_b, Pb, blob_b, J1, J2, PJ);
    return prepare_infer_launch(J1, J2, PJ, st);
}

int32_t gnn_infer_impl(const gcbf_env_desc* d, int out_dim, const float* P, const float* blob, int use_tc,
                       const GraphRefs& g, int clip_all, float* out, float* ws, cudaStream_t st, float* z_out,
                       int* z_parts, int32_t* zero_counter, int select, int keep_activations) {
    // keep_activations (folded train step): the unfused launch sequence, every layer output left in the workspace
    // (feat, x1, msg, g1, att, ag, v1, h1) for the backward pass; GEMMs still on the tensor-core path when use_tc
    // select (gcbf_rollout_step_select, measurement hook): bit 0 edge message (+ chained gate) kernel, bit 1 attention
    // aggregate, bit 2 update layer, bit 3 folded update/head layer; a cleared bit skips that launch
    // z_out != nullptr (rollout step): instead of `out`, write the output layer's pre-activation partial sums
    // z[part][A][4] (no bias, no tanh) for the policy tail fused into graph_build_kernel
    const int ed = env_ed(d->env_kind);
    const ParamLayout L = make_layout(ed, out_dim);
    const InferLayout I = make_infer_layout(out_dim);
    const int A = d->n_graphs * d->n_agents, cap = d->edge_cap;
    const GnnWs W = make_ws(cap, A);
    const RowCount re{g.counters, 0, cap};
    const RowCount ra{nullptr, A, A};
    const int nsm = sm_count();
    int32_t rc;
    auto gemm = [&](int epi, const float* X, const float* Wf, int t_off, int K, int N, const float* bias,
                    const float* bias2, float* Y, RowCount rows) -> int32_t {
        if (use_tc) return tc::launch_gemm_tc(epi, false, X, blob + t_off, blob + t_off + K * N, bias, bias2, Y, nullptr, rows, K, N, st);
        return launch_gemm_nn(epi, false, X, Wf, bias, bias2, Y, nullptr, rows, K, N, st);
    };
    if (use_tc && !keep_activations) {
        // tensor-core path, 4 launches: {edge features + layer 1 produced in-kernel -> folded message GEMM -> chained
        // gate layer + folded gate vector -> logits}, {softmax + aggregate}, {update layer 1},
        // {update/head folded layer (+ output layer) below}
        if (select & 1) {
            tc::ChainArgs ch;
            ch.bias_g = P + L.b[L_ATT0];
            ch.avec = blob + I.a23;
            ch.cst = blob + I.c23;
            ch.logits = ws + W.att;
            if ((rc = tc::launch_edge_msg(d, P + L.w[L_MSG0], P + L.b[L_MSG0], g, clip_all, blob + I.t_w23,
                                          blob + I.t_w23 + 256 * 128, blob + I.b23, ws + W.msg, st, blob + I.t_a1,
                                          blob + I.t_a1 + 128 * 128, ch))) return rc;
        }
        // (measured: producing the aggregate inside the update GEMM (tc::launch_attn_upd) is slower than the
        //  separate warp-per-receiver kernel + TMA-fed GEMM: 36.6 us vs 13.2 + 11.7 us -- its N-split repeats
        //  the aggregation and the per-thread MSG gathers are latency-bound; the edge producer above is a win)
        if (select & 2) {
            const int grid = min((A + 7) / 8, 8 * nsm);   // 8 x 256 threads per SM: one receiver per warp in flight (latency-bound kernel)
            attn_aggregate_kernel<<<grid, 256, 0, st>>>(A, cap, nullptr, ws + W.msg, blob + I.a23, blob + I.c23,
                                                        g.row_start, g.row_deg, ws + W.att, ws + W.ag, zero_counter);
            count_launch();
            if ((rc = check_launch("attn_aggregate_kernel"))) return rc;
        }
        if ((select & 4) && (rc = gemm(EPI_BIAS_RELU, ws + W.ag, P + L.w[L_UPD0] + 3 * 256, I.t_u1, 128, 256, P + L.b[L_UPD0],
                                       P + L.w[L_UPD0] + 2 * 256, ws + W.v1, ra))) return rc;
    } else {
        {
            const int grid = min((cap + 7) / 8, 4 * nsm);
            GCBF_DISPATCH_ENV(d->env_kind, {
                edge_l1_kernel<KIND><<<grid, 256, 0, st>>>(*d, P + L.w[L_MSG0], P + L.b[L_MSG0], g.agent, g.goal,
                                                           g.hits, g.edge_recv, g.edge_src, g.counters, clip_all,
                                                           ws + W.feat, ws + W.x1);
            });
            count_launch();
            if ((rc = check_launch("edge_l1_kernel"))) return rc;
        }
        if ((rc = gemm(EPI_BIAS, ws + W.x1, blob + I.w23, I.t_w23, 256, 128, blob + I.b23, nullptr, ws + W.msg, re))) return rc;
        if ((rc = gemm(EPI_BIAS_RELU, ws + W.msg, P + L.w[L_ATT0], I.t_a1, 128, 128, P + L.b[L_ATT0], nullptr, ws + W.g1, re))) return rc;
        {
            const int grid = min((A + 7) / 8, 8 * nsm);
            attn_aggregate_kernel<<<grid, 256, 0, st>>>(A, cap, ws + W.g1, ws + W.msg, blob + I.a23, blob + I.c23,
                                                        g.row_start, g.row_deg, ws + W.att, ws + W.ag, zero_counter);
            count_launch();
            if ((rc = check_launch("attn_aggregate_kernel"))) return rc;
        }
        if ((rc = gemm(EPI_BIAS_RELU, ws + W.ag, P + L.w[L_UPD0] + 3 * 256, I.t_u1, 128, 256, P + L.b[L_UPD0],
                       P + L.w[L_UPD0] + 2 * 256, ws + W.v1, ra))) return rc;
    }
    if (z_out != nullptr) {
        if (use_tc) {   // last hidden layer + output layer partial sums in the GEMM epilogue (h1 never leaves the SM)
            *z_parts = 256 / tc::BN;   // one partial sum per 128-wide column tile
            if (!(select & 8)) return 0;
            return tc::launch_gemm_tc(EPI_RELU_DOTN, false, ws + W.v1, blob + I.t_uh, blob + I.t_uh + 256 * 256, blob + I.buh,
                                      nullptr, z_out, blob + I.ho, ra, 256, 256, st, out_dim, z_parts);
        }
        if ((rc = gemm(EPI_BIAS_RELU, ws + W.v1, blob + I.uh, I.t_uh, 256, 256, blob + I.buh, nullptr, ws + W.h1, ra))) return rc;
        const int grid = min((A + 7) / 8, 4 * nsm);
        head_z_kernel<<<grid, 256, 0, st>>>(A, out_dim, ws + W.h1, blob + I.ho, z_out);
        count_launch();
        *z_parts = 1;
        return check_launch("head_z_kernel");
    }
    if ((rc = gemm(EPI_BIAS_RELU, ws + W.v1, blob + I.uh, I.t_uh, 256, 256, blob + I.buh, nullptr, ws + W.h1, ra))) return rc;
    if (out != nullptr) {
        const int grid = min((A + 7) / 8, 4 * nsm);
        head_out_kernel<<<grid, 256, 0, st>>>(A, out_dim, ws + W.h1, blob + I.ho, blob + I.bho, out);
        count_launch();
        if ((rc = check_launch("head_out_kernel"))) return rc;
    }
    return 0;
}

}  // namespace gcbf

extern "C" __attribute__((visibility("default"))) int32_t gcbf_infer_count(int32_t edge_dim, int32_t out_dim) {
    if (edge_dim < 1 || edge_dim > 6 || out_dim < 1 || out_dim > 4) return -1;
    return make_infer_layout(out_dim).total;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_prepare_infer(int32_t edge_dim, int32_t out_dim,
                                                                             const float* params, float* infer_blob,
                                                                             void* stream) {
    GCBF_REQUIRE(edge_dim >= 1 && edge_dim <= 6 && out_dim >= 1 && out_dim <= 4 && params && infer_blob,
                 "gcbf_prepare_infer: bad argument");
    GCBF_REQUIRE((((uintptr_t)params | (uintptr_t)infer_blob) & 15) == 0, "gcbf_prepare_infer: 16-byte alignment required");
    return prepare_infer_impl(edge_dim, out_dim, params, infer_blob, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_gnn_infer(
    const gcbf_env_desc* desc, int32_t net_kind, int32_t out_dim, const float* params, const float* infer_blob,
    int32_t use_tensor_cores, const float* agent, const float* goal, const float* hits, const int32_t* row_start,
    const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters,
    int32_t clip_all, float* out, float* workspace, int64_t workspace_floats, void* stream) {
    GCBF_REQUIRE(desc && params && infer_blob && agent && goal && hits && row_start && row_deg && edge_recv && edge_src &&
                     counters && out && workspace, "gcbf_gnn_infer: NULL pointer argument");
    if (int32_t rc = check_graph_desc(desc, "gcbf_gnn_infer")) return rc;
    GCBF_REQUIRE(net_kind == GCBF_NET_CBF || net_kind == GCBF_NET_ACTOR, "bad net_kind %d", net_kind);
    GCBF_REQUIRE(out_dim >= 1 && out_dim <= 4 && (net_kind != GCBF_NET_CBF || out_dim == 1), "bad out_dim %d", out_dim);
    const int64_t need = make_ws(desc->edge_cap, (int64_t)desc->n_graphs * desc->n_agents).total;
    GCBF_REQUIRE(workspace_floats >= need, "workspace too small: %lld < %lld floats", (long long)workspace_floats,
                 (long long)need);
    GCBF_REQUIRE((((uintptr_t)params | (uintptr_t)workspace | (uintptr_t)infer_blob) & 15) == 0,
                 "params/infer_blob/workspace must be 16-byte aligned");
    const GraphRefs g{agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters};
    return gnn_infer_impl(desc, out_dim, params, infer_blob, use_tensor_cores, g, clip_all, out, workspace,
                          (cudaStream_t)stream);
}

// =====================================================================================================
// Unfolded forward of an n_layers-deep network (gnn.py:78-104; n_layers = 1 is the reference's one-layer GNN): the
// GEMMs read the tf32 planes of PlaneLayout (tensor-core path) or, at n_layers = 1, the parameters themselves
// (strict-fp32 SIMT path).
// Edges and their features are the same in every layer; only the node features change.  Receivers are always agents,
// so goal and hit nodes never receive a message: their layer output is update_l([y_{l-1} | 0]), one constant row per
// layer for "goal" and one for "hit".  They ride along as node rows A and A + 1 of the node-level GEMMs of every layer
// that a later layer reads.
// From layer 1 on, the first message layer W1 = [We; Ws; Wr] is split: pre1_e = feat_e We + S[src_e] + R[recv_e] + b1
// with the node-level products S = y Ws and R = y Wr, so the edge kernel gathers two 256-wide rows instead of running a
// K = ed + 256 GEMM per edge.
// =====================================================================================================
namespace gcbf {

int32_t build_planes(int ed, int out_dim, int n_layers, const float* P, float* PT, cudaStream_t st) {
    const PlaneLayout Q = make_plane_layout(make_deep_layout(ed, out_dim, n_layers), ed);
    PlaneJobList PJ;
    for (int l = 0; l < n_layers; ++l) {
        for (int i = 0; i < 13; ++i) {
            if (Q.t[l][i] < 0) continue;
            const int rows = Q.rows[l][i], cols = Q.cols[l][i], n = rows * cols;
            PJ.add(P + Q.src[l][i], rows, cols, true, PT + Q.t[l][i], PT + Q.t[l][i] + n);
            if (Q.s[i] >= 0) PJ.add(P + Q.src[l][i], rows, cols, false, PT + Q.s[i], PT + Q.s[i] + n);
        }
        if (int32_t rc = PJ.launch(st)) return rc;   // one launch per layer: 18 jobs at n_layers = 1, <= 11 after
    }
    return 0;
}

// Workspace of the unfolded forward: the activations of make_ws (the layout the backward reads) and, at n_layers > 1,
// with A + 2 node rows, plus S | R and the update input [y | ag].
struct DeepWs {
    GnnWs g;
    int64_t s, r, cat, total;
};
static DeepWs make_deep_ws(int64_t cap, int64_t A, int n_layers) {
    DeepWs W;
    const int64_t nodes = n_layers > 1 ? A + 2 : A, node_block = n_layers > 1 ? nodes * 256 : 0;
    WsSlots S{8};
    W.g = make_ws(cap, nodes);
    S.take(W.g.total);
    W.s = S.take(node_block);
    W.r = S.take(node_block);
    W.cat = S.take(node_block);
    W.total = S.off;
    return W;
}

// X1 = relu(feat We + S[sender row] + R[receiver] + b1); warp per edge, lane owns 8 output columns.  The sender row of
// a goal / hit node is the constant row A / A + 1.
template <int ED>
__global__ void __launch_bounds__(256)
edge_deep_kernel(const int A, const int edge_cap, const float* __restrict__ We, const float* __restrict__ b1,
                 const float* __restrict__ feat, const float* __restrict__ S, const float* __restrict__ R,
                 const int32_t* __restrict__ edge_recv, const int32_t* __restrict__ edge_src,
                 const int32_t* __restrict__ counters, float* __restrict__ X1) {
    __shared__ __align__(16) float sW[ED][256];
    __shared__ __align__(16) float sB[256];
    for (int i = threadIdx.x; i < ED * 256; i += blockDim.x) sW[i / 256][i % 256] = We[i];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sB[i] = b1[i];
    __syncthreads();
    const int nE = min(counters[0], edge_cap);
    const int lane = threadIdx.x & 31;
    const int warps_total = (gridDim.x * blockDim.x) >> 5;
    for (int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < nE; e += warps_total) {
        const int a = min(max(edge_recv[e], 0), A - 1);
        const int code = min(edge_src[e], A - 1);
        const int srow = code >= 0 ? code : (code == -1 ? A : A + 1);
        const float4* sp = reinterpret_cast<const float4*>(S + (size_t)srow * 256 + lane * 8);
        const float4* rp = reinterpret_cast<const float4*>(R + (size_t)a * 256 + lane * 8);
        const float4 s0 = sp[0], s1 = sp[1], r0 = rp[0], r1 = rp[1];
        const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        const float rv[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
        float f[ED];
#pragma unroll
        for (int c = 0; c < ED; ++c) f[c] = feat[(size_t)e * FEAT_LD + c];
        float y[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) y[j] = sB[lane * 8 + j] + sv[j] + rv[j];
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

// Rows A (goal, one-hot [0,1,0]) and A + 1 (hit, [1,0,0]) of layer 0's first update layer: relu(U0[type] + bu0), the
// aggregate being zero.
static __global__ void const_rows_l0_kernel(const int A, const float* __restrict__ U0, const float* __restrict__ bu0,
                                            float* __restrict__ V1) {
    for (int i = threadIdx.x; i < 2 * 256; i += blockDim.x) {
        const int r = i / 256, c = i % 256;
        V1[(size_t)(A + r) * 256 + c] = fmaxf(U0[(1 - r) * 256 + c] + bu0[c], 0.f);
    }
}

// CAT[r] = [Y[r] | AG[r]] for the A + 2 node rows; the goal / hit rows (r >= A) take a zero aggregate.
static __global__ void __launch_bounds__(256)
node_concat_kernel(const int A, const float* __restrict__ Y, const float* __restrict__ AG, float* __restrict__ CAT) {
    const int n = (A + 2) * 64;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int r = i >> 6, q = i & 63;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q < 32) v = *reinterpret_cast<const float4*>(Y + (size_t)r * 128 + q * 4);
        else if (r < A) v = *reinterpret_cast<const float4*>(AG + (size_t)r * 128 + (q - 32) * 4);
        *reinterpret_cast<float4*>(CAT + (size_t)r * 256 + q * 4) = v;
    }
}

int32_t gnn_forward(const gcbf_env_desc* d, int out_dim, int n_layers, const float* P, const float* PT,
                    const GraphRefs& g, int clip_all, float* out, float* z_out, float* ws, cudaStream_t st,
                    const int32_t* agent_rows) {
    const int ed = env_ed(d->env_kind);
    const DeepLayout D = make_deep_layout(ed, out_dim, n_layers);
    const PlaneLayout Q = make_plane_layout(D, ed);
    const int A = d->n_graphs * d->n_agents, cap = d->edge_cap;
    const DeepWs DW = make_deep_ws(cap, A, n_layers);
    const GnnWs& W = DW.g;
    const RowCount re{g.counters, 0, cap};
    const RowCount ra{agent_rows, A, A};
    const RowCount ra2{nullptr, A + 2, A + 2};
    const int nsm = sm_count();
    int32_t rc;
    // Y = epi(X W + bias (+ bias2)) with W the weight in slot i of layer l
    auto gemm = [&](int epi, int l, int i, const float* X, const float* bias, const float* bias2, float* Y,
                    RowCount rows) -> int32_t {
        const int K = Q.rows[l][i], N = Q.cols[l][i];
        if (PT)
            return tc::launch_gemm_tc(epi, false, X, PT + Q.t[l][i], PT + Q.t[l][i] + K * N, bias, bias2, Y, nullptr,
                                      rows, K, N, st);
        return launch_gemm_nn(epi, false, X, P + Q.src[l][i], bias, bias2, Y, nullptr, rows, K, N, st);
    };
    for (int l = 0; l < n_layers; ++l) {
        const ParamLayout& L = D.layer[l];
        const bool carry = l + 1 < n_layers;   // a later layer reads the goal / hit rows of this one
        const RowCount rn = carry ? ra2 : ra;
        const int egrid = min((cap + 7) / 8, 4 * nsm);
        if (l == 0) {
            GCBF_DISPATCH_ENV(d->env_kind, {
                edge_l1_kernel<KIND><<<egrid, 256, 0, st>>>(*d, P + L.w[L_MSG0], P + L.b[L_MSG0], g.agent, g.goal,
                                                            g.hits, g.edge_recv, g.edge_src, g.counters, clip_all,
                                                            ws + W.feat, ws + W.x1);
            });
            count_launch();
            if ((rc = check_launch("edge_l1_kernel"))) return rc;
        } else {
            if ((rc = gemm(EPI_NONE, l, L_MSG0, ws + W.v3, nullptr, nullptr, ws + DW.s, ra2))) return rc;
            if ((rc = gemm(EPI_NONE, l, DEEP_WR, ws + W.v3, nullptr, nullptr, ws + DW.r, ra))) return rc;
            GCBF_DISPATCH_ENV(d->env_kind, {
                edge_deep_kernel<EnvTraits<KIND>::ED><<<egrid, 256, 0, st>>>(
                    A, cap, P + L.w[L_MSG0], P + L.b[L_MSG0], ws + W.feat, ws + DW.s, ws + DW.r, g.edge_recv,
                    g.edge_src, g.counters, ws + W.x1);
            });
            count_launch();
            if ((rc = check_launch("edge_deep_kernel"))) return rc;
        }
        if ((rc = gemm(EPI_BIAS, l, L_MSG1, ws + W.x1, P + L.b[L_MSG1], nullptr, ws + W.x2, re))) return rc;
        if ((rc = gemm(EPI_BIAS, l, L_MSGOUT, ws + W.x2, P + L.b[L_MSGOUT], nullptr, ws + W.msg, re))) return rc;
        if ((rc = gemm(EPI_BIAS_RELU, l, L_ATT0, ws + W.msg, P + L.b[L_ATT0], nullptr, ws + W.g1, re))) return rc;
        if ((rc = gemm(EPI_BIAS, l, L_ATT1, ws + W.g1, P + L.b[L_ATT1], nullptr, ws + W.g2, re))) return rc;
        {
            const int grid = min((A + 7) / 8, 4 * nsm);
            attn_aggregate_kernel<<<grid, 256, 0, st>>>(A, cap, ws + W.g2, ws + W.msg, P + L.w[L_GATE], P + L.b[L_GATE],
                                                        g.row_start, g.row_deg, ws + W.att, ws + W.ag);
            count_launch();
            if ((rc = check_launch("attn_aggregate_kernel"))) return rc;
        }
        if (l == 0) {
            // agent one-hot [0,0,1] folded into the bias: row 2 of update/Dense_0
            if ((rc = gemm(EPI_BIAS_RELU, l, L_UPD0, ws + W.ag, P + L.b[L_UPD0], P + L.w[L_UPD0] + 2 * 256, ws + W.v1,
                           ra))) return rc;
            if (carry) {
                const_rows_l0_kernel<<<1, 256, 0, st>>>(A, P + L.w[L_UPD0], P + L.b[L_UPD0], ws + W.v1);
                count_launch();
                if ((rc = check_launch("const_rows_l0_kernel"))) return rc;
            }
        } else {
            node_concat_kernel<<<min((A + 2 + 3) / 4, 4 * nsm), 256, 0, st>>>(A, ws + W.v3, ws + W.ag, ws + DW.cat);
            count_launch();
            if ((rc = check_launch("node_concat_kernel"))) return rc;
            if ((rc = gemm(EPI_BIAS_RELU, l, L_UPD0, ws + DW.cat, P + L.b[L_UPD0], nullptr, ws + W.v1, rn))) return rc;
        }
        if ((rc = gemm(EPI_BIAS, l, L_UPD1, ws + W.v1, P + L.b[L_UPD1], nullptr, ws + W.v2, rn))) return rc;
        if ((rc = gemm(EPI_BIAS, l, L_UPDOUT, ws + W.v2, P + L.b[L_UPDOUT], nullptr, ws + W.v3, rn))) return rc;
    }
    const ParamLayout& L = D.layer[0];
    if ((rc = gemm(EPI_BIAS_RELU, 0, L_HEAD0, ws + W.v3, P + L.b[L_HEAD0], nullptr, ws + W.h1, ra))) return rc;
    if ((rc = gemm(EPI_BIAS, 0, L_HEAD1, ws + W.h1, P + L.b[L_HEAD1], nullptr, ws + W.h2, ra))) return rc;
    const int grid = min((A + 7) / 8, 4 * nsm);
    if (out != nullptr) {
        head_out_kernel<<<grid, 256, 0, st>>>(A, out_dim, ws + W.h2, P + L.w[L_OUT], P + L.b[L_OUT], out);
        count_launch();
        return check_launch("head_out_kernel");
    }
    head_z_kernel<<<grid, 256, 0, st>>>(A, out_dim, ws + W.h2, P + L.w[L_OUT], z_out);
    count_launch();
    return check_launch("head_z_kernel");
}

}  // namespace gcbf

static bool deep_dims_ok(int32_t edge_dim, int32_t out_dim, int32_t n_layers) {
    return edge_dim >= 1 && edge_dim <= 6 && out_dim >= 1 && out_dim <= 4 && n_layers >= 1 &&
           n_layers <= gcbf::GCBF_MAX_LAYERS;
}
static bool ws_dims_ok(const gcbf_env_desc* desc, int32_t n_layers) {
    return graph_sizes_ok(desc) && n_layers >= 1 && n_layers <= gcbf::GCBF_MAX_LAYERS;
}

// Workspace of the rollout step: the forward's (make_deep_ws) and, 16-byte aligned after it, the output layer's
// partial sums z [2][A][4].
struct StepWs {
    int64_t z, total;
};
static StepWs make_step_ws(const gcbf_env_desc* d, int n_layers) {
    const int64_t A = (int64_t)d->n_graphs * d->n_agents, fwd = make_deep_ws(d->edge_cap, A, n_layers).total;
    return {(fwd + 3) & ~(int64_t)3, fwd + 8 * A + 16};
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_params_t_count_l(int32_t edge_dim, int32_t out_dim,
                                                                                int32_t n_layers) {
    if (!deep_dims_ok(edge_dim, out_dim, n_layers)) return -1;
    return make_plane_layout(make_deep_layout(edge_dim, out_dim, n_layers), edge_dim).total;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_prepare_params_l(int32_t edge_dim, int32_t out_dim,
                                                                                int32_t n_layers, const float* params,
                                                                                float* params_t, void* stream) {
    GCBF_REQUIRE(deep_dims_ok(edge_dim, out_dim, n_layers) && params && params_t, "gcbf_prepare_params_l: bad argument");
    GCBF_REQUIRE((((uintptr_t)params | (uintptr_t)params_t) & 15) == 0, "gcbf_prepare_params_l: 16-byte alignment required");
    return build_planes(edge_dim, out_dim, n_layers, params, params_t, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int64_t gcbf_gnn_workspace_floats_l(const gcbf_env_desc* desc,
                                                                                     int32_t out_dim, int32_t n_layers) {
    (void)out_dim;
    if (!ws_dims_ok(desc, n_layers)) return -1;
    return make_deep_ws(desc->edge_cap, (int64_t)desc->n_graphs * desc->n_agents, n_layers).total;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_gnn_forward_l(
    const gcbf_env_desc* desc, int32_t net_kind, int32_t out_dim, int32_t n_layers, const float* params,
    const float* params_t, const float* agent, const float* goal, const float* hits, const int32_t* row_start,
    const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters, int32_t clip_all,
    float* out, float* workspace, int64_t workspace_floats, void* stream) {
    GCBF_REQUIRE(n_layers >= 1 && n_layers <= GCBF_MAX_LAYERS, "gcbf_gnn_forward_l: n_layers %d outside [1, %d]",
                 n_layers, GCBF_MAX_LAYERS);
    GCBF_REQUIRE(desc && params && agent && goal && hits && row_start && row_deg && edge_recv && edge_src && counters &&
                     out && workspace, "gcbf_gnn_forward_l: NULL pointer argument");
    GCBF_REQUIRE(n_layers == 1 || params_t, "gcbf_gnn_forward_l: n_layers > 1 runs on the tensor-core path only "
                                            "(params_t from gcbf_prepare_params_l); the strict-fp32 SIMT path "
                                            "implements n_layers = 1");
    if (int32_t rc = check_graph_desc(desc, "gcbf_gnn_forward_l")) return rc;
    GCBF_REQUIRE(net_kind == GCBF_NET_CBF || net_kind == GCBF_NET_ACTOR, "bad net_kind %d", net_kind);
    GCBF_REQUIRE(out_dim >= 1 && out_dim <= 4 && (net_kind != GCBF_NET_CBF || out_dim == 1), "bad out_dim %d", out_dim);
    const int64_t need = make_deep_ws(desc->edge_cap, (int64_t)desc->n_graphs * desc->n_agents, n_layers).total;
    GCBF_REQUIRE(workspace_floats >= need, "workspace too small: %lld < %lld floats", (long long)workspace_floats,
                 (long long)need);
    GCBF_REQUIRE((((uintptr_t)params | (uintptr_t)params_t | (uintptr_t)workspace) & 15) == 0,
                 "params/params_t/workspace must be 16-byte aligned");
    const GraphRefs g{agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters};
    return gnn_forward(desc, out_dim, n_layers, params, params_t, g, clip_all, out, nullptr, workspace,
                       (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int64_t gcbf_rollout_workspace_floats_l(const gcbf_env_desc* desc,
                                                                                         int32_t n_layers) {
    if (!ws_dims_ok(desc, n_layers)) return -1;
    return make_step_ws(desc, n_layers).total;
}

// ---------------------------------------------------------------------------------------------------
// One closed-loop rollout step in a single call: policy forward -> a = 2 pi + u_ref, clip, Euler, reward / cost terms
// -> LiDAR + neighbour lists of the next state (+ reward / cost reduction).
// n_layers = 1: the folded forward (gnn_infer_impl), 6 launches on the tensor-core path with no memset / copy node in
// between: {edge features + message layer}, {gate layer -> logits}, {segment softmax + aggregate; clears the next edge
// counter}, {update layer}, {folded update/head layer + output layer partial sums}, {policy tail fused into the graph
// build of the next state}.  `select` (gcbf_rollout_step_select) skips launches of that chain.
// n_layers > 1: the unfolded forward (gnn_forward) on the tensor-core path, then the same fused tail and build.
// (Programmatic dependent launch of this chain was built and measured: +1 % (inside a CUDA graph the kernel-to-kernel
//  gap is already ~1 us) and it was NOT safe as written -- a dependent kernel that starts early can keep L1 /
//  read-only-cache lines of buffers its predecessor rewrites (DubinsCar rollouts became non-deterministic with only the
//  edge-message GEMM launched that way).  Removed.)
// ---------------------------------------------------------------------------------------------------
static int32_t rollout_step(
    const char* fn, const gcbf_env_desc* desc, int32_t n_layers, const float* actor_params, const float* infer_blob,
    int32_t use_tensor_cores, const float* agent, const float* goal, const float* obstacles, const float* ray_table,
    const float* hits, const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv,
    const int32_t* edge_src, const int32_t* counters, float* action, float* next_agent, float* next_hits,
    int32_t* next_row_start, int32_t* next_row_deg, int32_t* next_edge_recv, int32_t* next_edge_src,
    int32_t* next_counters, float* reward, float* cost, float* workspace, int64_t workspace_floats, int32_t select,
    void* stream) {
    GCBF_REQUIRE(n_layers >= 1 && n_layers <= GCBF_MAX_LAYERS, "%s: n_layers %d outside [1, %d]", fn, n_layers,
                 GCBF_MAX_LAYERS);
    GCBF_REQUIRE(desc && actor_params && infer_blob && agent && goal && ray_table && hits && row_start && row_deg &&
                     edge_recv && edge_src && counters && action && next_agent && next_hits && next_row_start &&
                     next_row_deg && next_edge_recv && next_edge_src && next_counters && reward && cost && workspace,
                 "%s: NULL pointer argument", fn);
    GCBF_REQUIRE(n_layers == 1 || use_tensor_cores, "%s: n_layers > 1 runs on the tensor-core path only", fn);
    GCBF_REQUIRE(select == GCBF_STEP_ALL || use_tensor_cores, "%s: partial steps need the tensor-core path", fn);
    GCBF_REQUIRE(next_row_start != row_start && next_row_deg != row_deg && next_edge_recv != edge_recv &&
                     next_edge_src != edge_src && next_counters != counters,
                 "%s: the next graph must not alias the current one (double-buffer the edge lists)", fn);
    if (int32_t rc = check_graph_desc(desc, fn)) return rc;
    GCBF_REQUIRE(desc->n_obs == 0 || obstacles, "obstacles is NULL but n_obs > 0");
    const StepWs W = make_step_ws(desc, n_layers);
    GCBF_REQUIRE(workspace_floats >= W.total, "workspace too small: %lld < %lld floats", (long long)workspace_floats,
                 (long long)W.total);
    const uintptr_t planes = n_layers > 1 ? (uintptr_t)actor_params | (uintptr_t)infer_blob : 0;   // PlaneLayout
    GCBF_REQUIRE((((uintptr_t)workspace | planes) & 15) == 0, "%s: actor_params/infer_blob/workspace must be 16-byte "
                                                              "aligned", fn);
    cudaStream_t st = (cudaStream_t)stream;
    const int nu = env_nu(desc->env_kind);
    const GraphRefs g{agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters};
    float* z = workspace + W.z;
    TailArgs tl;
    tl.z = z;
    tl.parts = 1;
    tl.z_cap = desc->n_graphs * desc->n_agents;
    tl.agent_prev = agent;
    tl.goal = goal;
    tl.row_start_prev = row_start;
    tl.row_deg_prev = row_deg;
    tl.edge_src_prev = edge_src;
    tl.action = action;
    tl.next_agent = next_agent;
    int32_t flags = 1;   // cast rays
    if (n_layers == 1) {
        if (int32_t rc = gnn_infer_impl(desc, nu, actor_params, infer_blob, use_tensor_cores, g, 0, nullptr, workspace,
                                        st, z, &tl.parts, next_counters, select & 0xF)) return rc;
        if (!(select & 16)) return 0;
        tl.bHO = infer_blob + make_infer_layout(nu).bho;
        // the attention kernel cleared the next edge counter; a partial step without it lets the build clear it
        if (select & 2) flags |= 4;
    } else {
        if (int32_t rc = gnn_forward(desc, nu, n_layers, actor_params, infer_blob, g, 0, nullptr, z, workspace, st))
            return rc;
        tl.bHO = actor_params + make_deep_layout(env_ed(desc->env_kind), nu, n_layers).layer[0].b[L_OUT];
    }
    return graph_build_impl(desc, nullptr, obstacles, ray_table, next_hits, next_row_start, next_row_deg, next_edge_recv,
                            next_edge_src, next_counters, flags, tl, reward, cost, stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_rollout_step_l(
    const gcbf_env_desc* desc, int32_t n_layers, const float* actor_params, const float* infer_blob,
    int32_t use_tensor_cores, const float* agent, const float* goal, const float* obstacles, const float* ray_table,
    const float* hits, const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv,
    const int32_t* edge_src, const int32_t* counters, float* action, float* next_agent, float* next_hits,
    int32_t* next_row_start, int32_t* next_row_deg, int32_t* next_edge_recv, int32_t* next_edge_src,
    int32_t* next_counters, float* reward, float* cost, float* workspace, int64_t workspace_floats, void* stream) {
    return rollout_step("gcbf_rollout_step_l", desc, n_layers, actor_params, infer_blob, use_tensor_cores, agent, goal,
                        obstacles, ray_table, hits, row_start, row_deg, edge_recv, edge_src, counters, action,
                        next_agent, next_hits, next_row_start, next_row_deg, next_edge_recv, next_edge_src,
                        next_counters, reward, cost, workspace, workspace_floats, GCBF_STEP_ALL, stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_rollout_step_select(
    const gcbf_env_desc* desc, const float* actor_params, const float* infer_blob, int32_t use_tensor_cores,
    const float* agent, const float* goal, const float* obstacles, const float* ray_table, const float* hits,
    const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src,
    const int32_t* counters, float* action, float* next_agent, float* next_hits, int32_t* next_row_start,
    int32_t* next_row_deg, int32_t* next_edge_recv, int32_t* next_edge_src, int32_t* next_counters, float* reward,
    float* cost, float* workspace, int64_t workspace_floats, int32_t select, void* stream) {
    return rollout_step("gcbf_rollout_step_select", desc, 1, actor_params, infer_blob, use_tensor_cores, agent, goal,
                        obstacles, ray_table, hits, row_start, row_deg, edge_recv, edge_src, counters, action,
                        next_agent, next_hits, next_row_start, next_row_deg, next_edge_recv, next_edge_src,
                        next_counters, reward, cost, workspace, workspace_floats, select, stream);
}
