// internal.cuh -- host functions that one translation unit of libgcbf_b200.so defines and another calls.
#pragma once
#include "common.cuh"
#include "gemm.cuh"
#include "translayout.cuh"

namespace gcbf {

// The swarm graph of a batch (gcbf_graph_build's outputs) and the agent and goal states it was built from.
struct GraphRefs {
    const float *agent, *goal, *hits;
    const int32_t *row_start, *row_deg, *edge_recv, *edge_src, *counters;
    GraphRefs with_agent(const float* x) const {   // same edges, other agent states (x' of the train step)
        GraphRefs r = *this;
        r.agent = x;
        return r;
    }
};

// Descriptor of a batch of graphs with edge lists: a known environment and positive sizes.  The layer-aware workspace
// queries do not depend on the environment and check the sizes only.
inline bool graph_sizes_ok(const gcbf_env_desc* d) {
    return d && d->n_graphs > 0 && d->n_agents > 0 && d->edge_cap > 0;
}
inline bool graph_desc_ok(const gcbf_env_desc* d) {
    return graph_sizes_ok(d) && d->env_kind >= 0 && d->env_kind <= 3;
}
inline int32_t check_graph_desc(const gcbf_env_desc* d, const char* fn) {
    GCBF_REQUIRE(d, "%s: desc is NULL", fn);
    GCBF_REQUIRE(graph_desc_ok(d), "%s: bad descriptor (env_kind %d, n_graphs %d, n_agents %d, edge_cap %d)", fn,
                 d->env_kind, d->n_graphs, d->n_agents, d->edge_cap);
    return 0;
}

// dense.cu: dst += the ordered sum of `nparts` per-CTA partials (partial_sum_kernel; see PartSegs).
int32_t launch_partial_sum(const float* part, int64_t stride, int nparts, const PartSegs& segs, cudaStream_t st,
                           const int32_t* m_ptr = nullptr, int m_cap = 0, int rows_per_part = 1);

// dense.cu: the strict-fp32 SIMT GEMMs.  C = epi(A @ B) (+= with accum); C += X^T (w dY); db (and db2) += sum_m w dY.
// `part` (optional, PART_FLOATS): split the rows over many CTAs and add the splits in order; without it one CTA per
// output tile walks all rows.
int32_t launch_gemm_nn(int epi, bool accum, const float* A, const float* B, const float* bias, const float* bias2,
                       float* C, const float* aux, RowCount rc, int K, int N, cudaStream_t st);
int32_t launch_gemm_tn(const float* X, int ldx, const float* dY, float* C, const float* roww, const int32_t* row2agent,
                       RowCount rc, int K1, int N, int n_agents_total, cudaStream_t st, float* part = nullptr);
int32_t launch_colsum(const float* dY, float* db, const float* roww, const int32_t* row2agent, RowCount rc, int N,
                      int n_agents_total, cudaStream_t st, float* part = nullptr, float* db2 = nullptr);

namespace tc {
// dense.cu: the wgmma 3xTF32 GEMMs.  C = epi(A @ Bt^T) with Bt as its tf32 hi / lo planes (EPI_RELU_DOTN: one output
// partial sum per 128-wide column tile, *parts_out of them); C += X^T (w dY) with the column sums cs1 (and cs2) fused.
int32_t launch_gemm_tc(int epi, bool accum, const float* A, const float* Bt_hi, const float* Bt_lo, const float* bias,
                       const float* bias2, float* C, const float* aux, RowCount rc, int K, int N, cudaStream_t st,
                       int ndot = 0, int* parts_out = nullptr);
int32_t launch_gemm_tn_tc(const float* X, int ldx, const float* dY, float* C, const float* roww,
                          const int32_t* row2agent, RowCount rc, int K1, int N, int n_agents_total, cudaStream_t st,
                          float* cs1 = nullptr, float* cs2 = nullptr, float* part = nullptr);
}  // namespace tc

// dense.cu: the transposed GEMM weights of one network (TransLayout) into PT.
int32_t build_transposes(const ParamLayout& L, const TransLayout& T, const float* P, float* PT, cudaStream_t st);

// geometry.cu: LiDAR hits + neighbour lists (gcbf_graph_build).  tail.z != nullptr: the rollout step's policy tail
// runs in the same kernel and the build is of the next state it computes.
int32_t graph_build_impl(const gcbf_env_desc* desc, const float* agent, const float* obstacles, const float* ray_table,
                         float* hits, int32_t* row_start, int32_t* row_deg, int32_t* edge_recv, int32_t* edge_src,
                         int32_t* counters, int32_t flags, const TailArgs& tail, float* reward, float* cost, void* stream);

// gnn.cu: the tf32 planes of an n_layers-deep network (PlaneLayout, translayout.cuh) into PT.
int32_t build_planes(int ed, int out_dim, int n_layers, const float* P, float* PT, cudaStream_t st);

// gnn.cu: unfolded forward of an n_layers-deep network over graph g with every activation left in `ws`.  PT: the
// planes of build_planes (tensor-core GEMMs) or nullptr (strict-fp32 SIMT GEMMs on P, n_layers = 1 only).
// out != nullptr: tanh(head) [A, out_dim]; else z_out [1][A][4] receives the output layer's pre-activations without
// bias.  agent_rows (optional): device row count of the agent-row GEMMs, like g.counters for the edge rows.
int32_t gnn_forward(const gcbf_env_desc* d, int out_dim, int n_layers, const float* P, const float* PT,
                    const GraphRefs& g, int clip_all, float* out, float* z_out, float* ws, cudaStream_t st,
                    const int32_t* agent_rows = nullptr);

// gnn.cu: the folded weights of two networks (gcbf_prepare_infer) in shared launches, and the folded forward.
int32_t prepare_infer_pair(int ed, int out_a, const float* Pa, float* blob_a, int out_b, const float* Pb, float* blob_b,
                           cudaStream_t st);
int32_t gnn_infer_impl(const gcbf_env_desc* d, int out_dim, const float* P, const float* blob, int use_tc,
                       const GraphRefs& g, int clip_all, float* out, float* ws, cudaStream_t st,
                       float* z_out = nullptr, int* z_parts = nullptr, int32_t* zero_counter = nullptr,
                       int select = 0xF, int keep_activations = 0);

// train.cu: a = 2 pi + u_ref and x' = Euler(x, clip_action(a)) per agent (act_dyn_kernel).
int32_t launch_act_dyn(const gcbf_env_desc* d, const float* agent, const float* goal, const float* pi, float* action,
                       float* xnext, cudaStream_t st);

// train.cu: one network's backward of the one-layer unfolded forward (gnn_forward's saved activations).  Built by
// aggregate initialisation, in this order.
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
int32_t gnn_backward_impl(const BwdArgs& b, cudaStream_t st);

// train.cu: the backward-data B operands of a one-layer network: the straight tf32 planes (build_planes) on the
// tensor-core path, W^T (TransLayout) on the SIMT path.
int32_t prepare_bwd_operands(int ed, int out_dim, int use_tc, const float* P, float* PT, cudaStream_t st);

}  // namespace gcbf
