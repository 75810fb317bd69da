// falsify.cu -- the CBF condition of the closed loop and its gradient with respect to the agent states, for a batch of
// G graphs: what GCBFPlus.falsify climbs to find states in the learned safe set from which the policy breaks the
// condition.  Like refine.cu it runs on the train step's pieces (internal.cuh) -- the one-layer forward with saved
// activations (gnn_forward), the data-only backward into the per-agent edge-state gradient (gnn_backward_impl with
// G = nullptr) and act_dyn_kernel (launch_act_dyn) -- plus the state Jacobians of u_ref_dev, euler_dev and
// edge_state_dev.
//
// Per graph, with a = 2 pi(g) + u_ref(x), x' = Euler(x, clip_action(a)) and g' = forward_graph(g, a):
//   term_i = -(h_i(g') - h_i(g)) / dt - alpha h_i(g),   J = max term_i over the agents with h_i(g) >= 0 and a finite term
// (ties: lowest index; worst = -1 and no gradient where no agent qualifies).  d J / d x holds the topology and the
// LiDAR hit points fixed.  The launch sequence is fixed (no host sync, capturable):
//   forwards: cbf(g), actor(g), act_dyn (a, x'), cbf(g')
//   falsify_select_kernel: term, worst, upstream (1/dt - alpha) on h_{i*} and -1/dt on h'_{i*}
//   [grad] data-only backward of cbf(g') -> d_es';  falsify_dyn_kernel -> dpi, d/dx through Euler and u_ref;
//          data-only backwards of actor(g) (upstream dpi) and cbf(g) -> d_es;  falsify_grad_kernel -> grad_x
// Every sum runs in a fixed order (no float atomics): bit-identical from run to run on one GPU model.
#include "geometry_dev.cuh"
#include "gnn.cuh"
#include "internal.cuh"

namespace gcbf {

// One CTA per graph: the terms of its agents and the worst agent, found by per-thread strided scans (ascending
// index, strict >) and a fixed tree that prefers the lower index on ties.  A NaN next state (an agent exactly at its
// goal has a NaN u_ref) makes the agent's term NaN, as in refine_value_kernel.  dh / dhn: the upstream gradients of J
// wrt h and h' (zero but at the worst agent).
constexpr int FALSIFY_SELECT_THREADS = 256;
__global__ void __launch_bounds__(FALSIFY_SELECT_THREADS)
falsify_select_kernel(const int N, const int SD, const float alpha, const float dt, const float* __restrict__ h,
                      const float* __restrict__ hn, const float* __restrict__ xnext, float* __restrict__ term,
                      int32_t* __restrict__ worst, float* __restrict__ dh, float* __restrict__ dhn) {
    __shared__ float s_v[FALSIFY_SELECT_THREADS];
    __shared__ int s_i[FALSIFY_SELECT_THREADS];
    const int g = blockIdx.x, t = threadIdx.x;
    float best = -INFINITY;
    int bi = -1;
    for (int i = t; i < N; i += FALSIFY_SELECT_THREADS) {
        const int a = g * N + i;
        float tm = -((hn[a] - h[a]) / dt) - alpha * h[a];
        for (int c = 0; c < SD; ++c) tm = isnan(xnext[(size_t)a * SD + c]) ? xnext[(size_t)a * SD + c] : tm;
        term[a] = tm;
        dh[a] = 0.f;
        dhn[a] = 0.f;
        if (h[a] >= 0.f && isfinite(tm) && (bi < 0 || tm > best)) {
            best = tm;
            bi = i;
        }
    }
    s_v[t] = best;
    s_i[t] = bi;
    __syncthreads();
    for (int o = FALSIFY_SELECT_THREADS / 2; o > 0; o >>= 1) {
        if (t < o) {
            const int j = s_i[t + o], k = s_i[t];
            if (j >= 0 && (k < 0 || s_v[t + o] > s_v[t] || (s_v[t + o] == s_v[t] && j < k))) {
                s_v[t] = s_v[t + o];
                s_i[t] = j;
            }
        }
        __syncthreads();
    }
    if (t == 0) {
        const int i = s_i[0];
        worst[g] = i;
        if (i >= 0) {
            dh[g * N + i] = 1.f / dt - alpha;
            dhn[g * N + i] = -1.f / dt;
        }
    }
}

// Per agent: d_es' (edge-state gradient at x') -> x' (edge-state Jacobian, velocity clip) -> Euler: the direct part
// dx'/dx and du -> clip_action -> da.  a = 2 pi + u_ref: dpi = 2 da, and da flows into x through u_ref.  gx: the
// gradient of J wrt x through x' and u_ref (NaN for an agent with a NaN u_ref).
template <int KIND>
__global__ void falsify_dyn_kernel(const gcbf_env_desc d, const float* __restrict__ agent,
                                   const float* __restrict__ goal, const float* __restrict__ action,
                                   const float* __restrict__ xnext, const float* __restrict__ d_es,
                                   float* __restrict__ dpi, float* __restrict__ gx) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU, ED = T::ED;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= d.n_graphs * d.n_agents) return;
    float x[SD], gl[SD], xn[SD], de[ED], dxn[SD], dx[SD], du[NU], ur[NU];
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        x[c] = agent[(size_t)a * SD + c];
        gl[c] = goal[(size_t)a * SD + c];
        xn[c] = xnext[(size_t)a * SD + c];
    }
#pragma unroll
    for (int c = 0; c < ED; ++c) de[c] = d_es[(size_t)a * ED + c];
    edge_state_vjp_dev<KIND>(xn, de, dxn);
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        const bool limited = (KIND == GCBF_ENV_DOUBLE_INTEGRATOR && c >= 2) || (KIND == GCBF_ENV_DUBINS_CAR && c == 3) ||
                             (KIND == GCBF_ENV_LINEAR_DRONE && c >= 3);
        if (limited && !(xn[c] > -d.v_lim && xn[c] < d.v_lim)) dxn[c] = 0.f;
    }
    euler_vjp_dev<KIND>(d, x, gl, dxn, dx, du);
    bool nan_ur = false;
    u_ref_dev<KIND>(d, x, gl, ur);
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        const float act = action[(size_t)a * NU + c];
        du[c] = (act > -d.u_lim && act < d.u_lim) ? du[c] : 0.f;
        dpi[(size_t)a * NU + c] = 2.f * du[c];
        nan_ur |= isnan(ur[c]);
    }
    u_ref_vjp_dev<KIND>(d, x, gl, du, dx);
#pragma unroll
    for (int c = 0; c < SD; ++c) gx[(size_t)a * SD + c] = nan_ur ? NAN : dx[c];
}

// grad_x = (d_es of the actor + d_es of the CBF on g) . d edge_state / dx + gx
template <int KIND>
__global__ void falsify_grad_kernel(const gcbf_env_desc d, const float* __restrict__ agent,
                                    const float* __restrict__ des_actor, const float* __restrict__ des_cbf,
                                    const float* __restrict__ gx, float* __restrict__ grad_x) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, ED = T::ED;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= d.n_graphs * d.n_agents) return;
    float x[SD], de[ED], dx[SD];
#pragma unroll
    for (int c = 0; c < SD; ++c) x[c] = agent[(size_t)a * SD + c];
#pragma unroll
    for (int c = 0; c < ED; ++c) de[c] = des_actor[(size_t)a * ED + c] + des_cbf[(size_t)a * ED + c];
    edge_state_vjp_dev<KIND>(x, de, dx);
#pragma unroll
    for (int c = 0; c < SD; ++c) grad_x[(size_t)a * SD + c] = dx[c] + gx[(size_t)a * SD + c];
}

// ------------------------------------------------------------------------------------ workspace layout
// Three forward workspaces (cbf(g), actor(g), cbf(g')): each backward reads its own forward's saved activations.
struct FalsifyWs {
    int64_t fw_h, fw_pi, fw_hn, gw, hn, pi, act, xn, dh, dhn, dpi, gx, des_n, des_a, des_c, je, total;
};
static FalsifyWs make_falsify_ws(const gcbf_env_desc* d) {
    const int ed = env_ed(d->env_kind), nu = env_nu(d->env_kind), sd = env_sd(d->env_kind);
    const int64_t A = (int64_t)d->n_graphs * d->n_agents, cap = d->edge_cap;
    const GnnWs W = make_ws(d->edge_cap, A);
    FalsifyWs t;
    WsSlots S{8};   // 32-byte slots
    t.fw_h = S.take(W.total);
    t.fw_pi = S.take(W.total);
    t.fw_hn = S.take(W.total);
    t.gw = S.take(W.total);
    t.hn = S.take(A);
    t.pi = S.take(A * nu);
    t.act = S.take(A * nu);
    t.xn = S.take(A * sd);
    t.dh = S.take(A);
    t.dhn = S.take(A);
    t.dpi = S.take(A * nu);
    t.gx = S.take(A * sd);
    t.des_n = S.take(A * ed);
    t.des_a = S.take(A * ed);
    t.des_c = S.take(A * ed);
    t.je = S.take(cap * 8);
    t.total = S.off;
    return t;
}

}  // namespace gcbf

using namespace gcbf;

// ------------------------------------------------------------------------------------ CBF condition + state gradient
extern "C" __attribute__((visibility("default"))) int32_t gcbf_cbf_condition_prepare(int32_t edge_dim, int32_t out_dim,
                                                                                     int32_t use_tensor_cores,
                                                                                     const float* params,
                                                                                     float* prepared,
                                                                                     int64_t prepared_floats,
                                                                                     void* stream) {
    GCBF_REQUIRE(params && prepared && (edge_dim == 2 || edge_dim == 4 || edge_dim == 6) && out_dim >= 1 && out_dim <= 3,
                 "gcbf_cbf_condition_prepare: bad argument");
    GCBF_REQUIRE((((uintptr_t)params | (uintptr_t)prepared) & 15) == 0, "buffers must be 16-byte aligned");
    const ParamLayout L = make_layout(edge_dim, out_dim);
    const int64_t need = use_tensor_cores ? make_plane_layout(make_deep_layout(edge_dim, out_dim, 1), edge_dim).total
                                          : make_trans_layout(L).total;
    GCBF_REQUIRE(prepared_floats >= need, "gcbf_cbf_condition_prepare: buffer too small: %lld < %lld floats",
                 (long long)prepared_floats, (long long)need);
    return prepare_bwd_operands(edge_dim, out_dim, use_tensor_cores, params, prepared, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int64_t gcbf_cbf_condition_workspace_floats(const gcbf_env_desc* desc) {
    return graph_desc_ok(desc) ? make_falsify_ws(desc).total : -1;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_cbf_condition(
    const gcbf_env_desc* desc, float alpha, int32_t use_tensor_cores, const float* cbf_params, const float* cbf_planes,
    const float* actor_params, const float* actor_planes, const float* agent, const float* goal, const float* hits,
    const int32_t* row_start, const int32_t* row_deg, const int32_t* edge_recv, const int32_t* edge_src,
    const int32_t* counters, float* h, float* term, int32_t* worst, float* grad_x, float* workspace,
    int64_t workspace_floats, void* stream) {
    GCBF_REQUIRE(desc && cbf_params && cbf_planes && actor_params && actor_planes && agent && goal && hits &&
                     row_start && row_deg && edge_recv && edge_src && counters && h && term && worst && workspace,
                 "gcbf_cbf_condition: NULL pointer argument");
    if (int32_t rc = check_graph_desc(desc, "gcbf_cbf_condition")) return rc;
    GCBF_REQUIRE(desc->dt > 0.f && isfinite(alpha), "gcbf_cbf_condition: bad settings (dt %g, alpha %g)",
                 (double)desc->dt, (double)alpha);
    const FalsifyWs F = make_falsify_ws(desc);
    GCBF_REQUIRE(workspace_floats >= F.total, "cbf condition workspace too small: %lld < %lld floats",
                 (long long)workspace_floats, (long long)F.total);
    GCBF_REQUIRE((((uintptr_t)workspace | (uintptr_t)cbf_params | (uintptr_t)cbf_planes | (uintptr_t)actor_params |
                   (uintptr_t)actor_planes) & 15) == 0, "buffers must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const gcbf_env_desc* d = desc;
    const int nu = env_nu(d->env_kind);
    const int G = d->n_graphs, N = d->n_agents, A = G * N;
    const int blocks = (A + 127) / 128;
    float* ws = workspace;
    int32_t rc;
#define RC(x) do { if ((rc = (x))) return rc; } while (0)
    // g: the graph; gn: its edges over the next states x' (forward_graph: every feature norm-clipped)
    const GraphRefs g{agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters};
    const GraphRefs gn = g.with_agent(ws + F.xn);
    auto forward = [&](int out_dim, const float* P, const float* PT, const GraphRefs& on, int clip_all, float* out,
                       float* fws) -> int32_t {
        return gnn_forward(d, out_dim, 1, P, use_tensor_cores ? PT : nullptr, on, clip_all, out, nullptr, fws, st);
    };
    // 1. forwards: h = cbf(g), pi = actor(g), a = 2 pi + u_ref and x' (act_dyn_kernel), h' = cbf(g')
    RC(forward(1, cbf_params, cbf_planes, g, 0, h, ws + F.fw_h));
    RC(forward(nu, actor_params, actor_planes, g, 0, ws + F.pi, ws + F.fw_pi));
    RC(launch_act_dyn(d, agent, goal, ws + F.pi, ws + F.act, ws + F.xn, st));
    RC(forward(1, cbf_params, cbf_planes, gn, 1, ws + F.hn, ws + F.fw_hn));
    // 2. terms, worst agent per graph, upstream gradients of J wrt h and h'
    falsify_select_kernel<<<G, FALSIFY_SELECT_THREADS, 0, st>>>(N, env_sd(d->env_kind), alpha, d->dt, h, ws + F.hn,
                                                                ws + F.xn, term, worst, ws + F.dh, ws + F.dhn);
    count_launch();
    RC(check_launch("falsify_select_kernel"));
    if (!grad_x) return 0;
    // 3. data-only backward of cbf(g') -> d_es'
    RC(gnn_backward_impl({d, gn, ws + F.gw, nullptr, use_tensor_cores, 1, cbf_params, cbf_planes, ws + F.fw_hn,
                          ws + F.hn, ws + F.dhn, nullptr, nullptr, 1, ws + F.des_n, ws + F.je}, st));
    // 4. through x' = Euler(x, clip_action(2 pi + u_ref(x))): dpi and the direct / u_ref parts of d J / dx
    GCBF_DISPATCH_ENV(d->env_kind, {
        falsify_dyn_kernel<KIND><<<blocks, 128, 0, st>>>(*d, agent, goal, ws + F.act, ws + F.xn, ws + F.des_n,
                                                         ws + F.dpi, ws + F.gx);
    });
    count_launch();
    RC(check_launch("falsify_dyn_kernel"));
    // 5. data-only backwards on g: the actor with upstream dpi, the CBF with upstream dh
    RC(gnn_backward_impl({d, g, ws + F.gw, nullptr, use_tensor_cores, nu, actor_params, actor_planes, ws + F.fw_pi,
                          ws + F.pi, ws + F.dpi, nullptr, nullptr, 0, ws + F.des_a, ws + F.je}, st));
    RC(gnn_backward_impl({d, g, ws + F.gw, nullptr, use_tensor_cores, 1, cbf_params, cbf_planes, ws + F.fw_h, h,
                          ws + F.dh, nullptr, nullptr, 0, ws + F.des_c, ws + F.je}, st));
    // 6. edge-state gradients -> states, plus the Euler / u_ref part
    GCBF_DISPATCH_ENV(d->env_kind, {
        falsify_grad_kernel<KIND><<<blocks, 128, 0, st>>>(*d, agent, ws + F.des_a, ws + F.des_c, ws + F.gx, grad_x);
    });
    count_launch();
    RC(check_launch("falsify_grad_kernel"));
#undef RC
    return 0;
}
