// internal.cuh -- host functions that one translation unit of libgcbf_b200.so defines and another calls.
#pragma once
#include "common.cuh"

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

}  // namespace gcbf
