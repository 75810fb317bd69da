// refine.cu -- online policy refinement of GCBF+ (gcbfplus/algo/gcbf.py:161-201) for a batch of G graphs.
// It runs on the train step's pieces (internal.cuh) -- the CBF forward with saved activations (gnn_forward), its
// data-only backward into the per-agent edge-state gradient (gnn_backward_impl with G = nullptr) -- and the chain edge
// state -> state -> clip_state -> Euler -> clip_action (dyn_chain_dev, geometry_dev.cuh).
//
// Per graph, h = cbf(g) is a constant and the action is refined by gradient steps on
//   val(a) = mean_agents relu(-(cbf(forward_graph(g, a)) - h) / dt - alpha h)
// while val > 0 and fewer than max_iter steps were taken; the test reads the value BEFORE the update, so the loop runs
// at least once and the last update is applied even where the new value is 0.  The launch sequence is fixed (no host
// sync, capturable in a CUDA graph): h, h(g'(u_ref)), init, then max_iter times [x' = f(x, a), h' = cbf(g'), value,
// data-only backward, gradient + update].  Early exit: once no graph of the batch is active the device row counts
// `rows` = (edge rows, agent rows) of the GEMMs and edge kernels drop to 0 and the small kernels return on entry.
// Graphs that stopped while others continue still compute; their update is masked.
#include "geometry_dev.cuh"
#include "gnn.cuh"
#include "internal.cuh"

namespace gcbf {

constexpr int32_t REFINE_CAPPED_BIT = 1 << 30;

// relu with JAX's NaN propagation (jnp.maximum(NaN, 0) = NaN)
__device__ __forceinline__ float relu_nan(const float t) { return t > 0.f ? t : (t == t ? 0.f : t); }

// x' = agent_step_euler(x, clip_action(a)) with a = the action (or u_ref, written to `ur`, when action is NULL)
template <int KIND>
__global__ void refine_next_state_kernel(const gcbf_env_desc d, const int32_t* __restrict__ rows,
                                         const float* __restrict__ agent, const float* __restrict__ goal,
                                         const float* __restrict__ action, float* __restrict__ ur,
                                         float* __restrict__ xnext) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU;
    if (rows && rows[1] == 0) return;       // every graph finished
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= d.n_graphs * d.n_agents) return;
    float x[SD], gl[SD], u[NU], act[NU], xn[SD];
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        x[c] = agent[(size_t)a * SD + c];
        gl[c] = goal[(size_t)a * SD + c];
    }
    u_ref_dev<KIND>(d, x, gl, u);
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        act[c] = action ? action[(size_t)a * NU + c] : u[c];
        if (!action) ur[(size_t)a * NU + c] = u[c];
    }
    step_agent<KIND>(d, x, gl, act, u, true, xn);
#pragma unroll
    for (int c = 0; c < SD; ++c) xnext[(size_t)a * SD + c] = xn[c];
}

// a = where(relu(-(h(g'(u_ref)) - h) / dt - alpha h) > 0, 2 pi + u_ref, u_ref) per agent; every graph active; the
// device row counts start at the full graph.
template <int NU>
__global__ void refine_init_kernel(const int G, const int A, const float alpha, const float dt,
                                   const float* __restrict__ h, const float* __restrict__ h_ur,
                                   const float* __restrict__ ur, const float* __restrict__ pi,
                                   const int32_t* __restrict__ counters, float* __restrict__ action,
                                   int32_t* __restrict__ active, int32_t* __restrict__ rows) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a == 0) {
        rows[0] = counters[0];
        rows[1] = A;
    }
    if (a < G) active[a] = 1;
    if (a >= A) return;
    const float v = relu_nan(-((h_ur[a] - h[a]) / dt) - alpha * h[a]);
    const bool nn = v > 0.f;
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        const float u = ur[(size_t)a * NU + c];
        action[(size_t)a * NU + c] = nn ? 2.f * pi[(size_t)a * NU + c] + u : u;
    }
}

// One CTA per graph: val = mean_i relu(term_i), summed in a fixed order (per-thread strided sums, then a fixed tree;
// no atomics), the upstream d val / d h'_i = -1[term_i > 0] / (N dt), and the graph's state: upd = entered this
// iteration active (its update is applied), active = takes part in the next one (val > 0 && it + 1 < max_iter).
constexpr int REFINE_VALUE_THREADS = 256;
__global__ void __launch_bounds__(REFINE_VALUE_THREADS)
refine_value_kernel(const int N, const int SD, const float alpha, const float dt, const int it, const int max_iter,
                    const float* __restrict__ h, const float* __restrict__ hn, const float* __restrict__ xnext,
                    float* __restrict__ dhn,
                    int32_t* __restrict__ active, int32_t* __restrict__ upd, float* __restrict__ value,
                    int32_t* __restrict__ iters) {
    __shared__ float red[REFINE_VALUE_THREADS];
    const int g = blockIdx.x, t = threadIdx.x;
    if (!active[g]) {
        if (t == 0) upd[g] = 0;
        return;
    }
    const float up = -(1.f / (float)N) / dt;
    float s = 0.f;
    for (int i = t; i < N; i += REFINE_VALUE_THREADS) {
        const int a = g * N + i;
        float term = -((hn[a] - h[a]) / dt) - alpha * h[a];
        // a NaN next state (an agent exactly at its goal has a NaN u_ref) makes the reference's h' NaN; the network
        // kernels' ReLU maps NaN pre-activations to 0, so the NaN is carried into the value here
        for (int c = 0; c < SD; ++c) term = isnan(xnext[(size_t)a * SD + c]) ? xnext[(size_t)a * SD + c] : term;
        s += relu_nan(term);
        dhn[a] = term > 0.f ? up : 0.f;
    }
    red[t] = s;
    __syncthreads();
    for (int o = REFINE_VALUE_THREADS / 2; o > 0; o >>= 1) {
        if (t < o) red[t] += red[t + o];
        __syncthreads();
    }
    if (t == 0) {
        const float val = red[0] / (float)N;
        upd[g] = 1;
        active[g] = (val > 0.f && it + 1 < max_iter) ? 1 : 0;
        if (value) value[g] = val;
        if (iters) iters[g] = (it + 1) | ((it + 1 == max_iter && val > 0.f) ? REFINE_CAPPED_BIT : 0);
    }
}

// a -= lr * d val / d a for the agents of the graphs that entered this iteration active (dyn_chain_dev: factor 1, no
// direct term); thread 0 sets the row counts of the next iteration (0 once no graph is active).
template <int KIND>
__global__ void refine_update_kernel(const gcbf_env_desc d, const float lr, const float* __restrict__ agent,
                                     const float* __restrict__ goal, const float* __restrict__ xnext,
                                     const float* __restrict__ d_es, const int32_t* __restrict__ active,
                                     const int32_t* __restrict__ upd, const int32_t* __restrict__ counters,
                                     int32_t* __restrict__ rows, float* action) {
    constexpr int NU = EnvTraits<KIND>::NU;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    const int A = d.n_graphs * d.n_agents;
    if (a == 0) {
        int any = 0;
        for (int g = 0; g < d.n_graphs; ++g) any |= active[g];
        rows[0] = any ? counters[0] : 0;
        rows[1] = any ? A : 0;
    }
    if (a >= A || !upd[a / d.n_agents]) return;
    float g[NU];
    dyn_chain_dev<KIND>(d, agent, goal, action, xnext, d_es, a, g);
#pragma unroll
    for (int c = 0; c < NU; ++c) action[(size_t)a * NU + c] = action[(size_t)a * NU + c] - lr * g[c];
}

// ------------------------------------------------------------------------------------ workspace layout
struct RefineWs {
    int64_t fw, gw, h, hn, dhn, ur, xn, d_es, je, active, upd, rows, total;
};
static RefineWs make_refine_ws(const gcbf_env_desc* d) {
    const int ed = env_ed(d->env_kind), nu = env_nu(d->env_kind), sd = env_sd(d->env_kind);
    const int64_t A = (int64_t)d->n_graphs * d->n_agents, cap = d->edge_cap;
    const GnnWs W = make_ws(d->edge_cap, A);
    RefineWs t;
    WsSlots S{8};   // 32-byte slots
    t.fw = S.take(W.total);
    t.gw = S.take(W.total);
    t.h = S.take(A);
    t.hn = S.take(A);
    t.dhn = S.take(A);
    t.ur = S.take(A * nu);
    t.xn = S.take(A * sd);
    t.d_es = S.take(A * ed);
    t.je = S.take(cap * 8);
    t.active = S.take(d->n_graphs);
    t.upd = S.take(d->n_graphs);
    t.rows = S.take(2);
    t.total = S.off;
    return t;
}

}  // namespace gcbf

using namespace gcbf;

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
