// internal.cuh -- host functions that one translation unit of libgcbf_b200.so defines and another calls.
#pragma once
#include "common.cuh"

namespace gcbf {

// geometry.cu: LiDAR hits + neighbour lists (gcbf_graph_build).  tail.z != nullptr: the rollout step's policy tail
// runs in the same kernel and the build is of the next state it computes.
int32_t graph_build_impl(const gcbf_env_desc* desc, const float* agent, const float* obstacles, const float* ray_table,
                         float* hits, int32_t* row_start, int32_t* row_deg, int32_t* edge_recv, int32_t* edge_src,
                         int32_t* counters, int32_t flags, const TailArgs& tail, float* reward, float* cost, void* stream);

// gnn.cu: the tf32 planes of an n_layers-deep network (PlaneLayout, translayout.cuh) into PT.
int32_t build_planes(int ed, int out_dim, int n_layers, const float* P, float* PT, cudaStream_t st);

// gnn.cu: unfolded forward of an n_layers-deep network with every activation left in `ws`.  PT: the planes of
// build_planes (tensor-core GEMMs) or nullptr (strict-fp32 SIMT GEMMs on P, n_layers = 1 only).  out != nullptr:
// tanh(head) [A, out_dim]; else z_out [1][A][4] receives the output layer's pre-activations without bias.
// agent_rows (optional): device row count of the agent-row GEMMs, like `counters` for the edge rows.
int32_t gnn_forward(const gcbf_env_desc* d, int out_dim, int n_layers, const float* P, const float* PT,
                    const float* agent, const float* goal, const float* hits, const int32_t* row_start,
                    const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src, const int32_t* counters,
                    int clip_all, float* out, float* z_out, float* ws, cudaStream_t st,
                    const int32_t* agent_rows = nullptr);

// gnn.cu: the folded weights of two networks (gcbf_prepare_infer) in shared launches, and the folded forward.
int32_t prepare_infer_pair(int ed, int out_a, const float* Pa, float* blob_a, int out_b, const float* Pb, float* blob_b,
                           cudaStream_t st);
int32_t gnn_infer_impl(const gcbf_env_desc* d, int out_dim, const float* P, const float* blob, int use_tc,
                       const float* agent, const float* goal, const float* hits, const int32_t* row_start,
                       const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src,
                       const int32_t* counters, int clip_all, float* out, float* ws, cudaStream_t st,
                       float* z_out = nullptr, int* z_parts = nullptr, int32_t* zero_counter = nullptr,
                       int select = 0xF, int keep_activations = 0);

}  // namespace gcbf
