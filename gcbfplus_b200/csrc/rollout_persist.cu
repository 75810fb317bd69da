// rollout_persist.cu -- the whole closed-loop rollout of trainer/utils.py:25-55 as ONE persistent kernel: one
// thread-block CLUSTER per environment, a loop over the T env-steps inside the kernel, cluster barriers where the
// 5-launch path (gcbf_rollout_step_l) has kernel boundaries.
//
// Why: environments are independent graphs, and at BASELINE's configs[2] (16 envs x 512 agents) every kernel of the
// 5-launch env-step is a single wave whose duration is its per-CTA latency chain plus ~4 us of launch / prologue
// (mbarrier init, layer-1 table, tensor-map fetch, obstacle / ray tables).  Here that setup is paid once per ROLLOUT, the 4 kernel boundaries per step become barrier.cluster phases (~0.2 us), and
// an environment's messages / aggregates / hidden rows stay in L2 between phases.
//
// Per env-step (cluster of C CTAs, 512 threads each; per-env receiver-ordered edge lists):
//   E   edge tiles of 128 edges -> CTA (tile % C): edge features + message layer 1 produced in-CTA -> folded message
//       GEMM 256->128 (wgmma 3xTF32, register accumulator) -> chained gate GEMM 128->128 -> logits         [gemm_tc_prod.cuh]
//   A   warp per receiver: segment softmax + weighted aggregate                                             [gnn.cuh aggregate_logits]
//   U1  (agent tile, column half) items: update layer 128->256, bias + one-hot row, ReLU                   [gemm_tc.cuh EPI_BIAS_RELU]
//   U2  same items: folded update/head layer 256->256, ReLU, output-layer partial sums                      [gemm_tc.cuh EPI_RELU_DOTN]
//   G   policy tail (tanh, a = 2 pi + u_ref, clip, Euler; record action / next state / reward / cost terms of the
//       CTA's own agents) + LiDAR + stable top-k + radius neighbour lists of the next state, rows laid out in agent order through a
//       CTA-local prefix sum and a cluster-wide exchange of the CTA totals over distributed shared memory    [geometry_dev.cuh]
// The phases call the device functions the 5-launch kernels call (GEMM main loops and epilogues; aggregate; policy
// tail, LiDAR, neighbour scan and row fill), so the two paths give the same bits (tests/test_gpu_rollout.py).  What
// differs stays here: the edge-row limit of a local group, the row base from the prefix over the cluster, and that
// each CTA records its own agents (the environment's first CTA reduces their reward / cost terms one step later, after
// the environment barrier).  This translation unit is
// compiled with -fmad=false like geometry.cu (the LiDAR / dynamics code must keep one rounding per operation); the
// GEMM-side code uses explicit fmaf wherever the other translation units rely on contraction.
//
// Replaces: gcbfplus/trainer/utils.py:25-55 (rollout scan body), algo/gcbf_plus.py:176-186, env/double_integrator.py:145-198,
// 223-320, env/utils.py:49-131, nn/gnn.py:44-104 -- for the 2-D environments (SingleIntegrator, DoubleIntegrator, DubinsCar)
// with n_agents <= 512; LinearDrone (514 rays, 33 KB of per-warp alpha scratch) stays on the 5-launch path.
#include <stdlib.h>

#include "gemm_tc_prod.cuh"
#include "geometry_dev.cuh"
#include "gnn.cuh"

namespace gcbf {
namespace rp {
using namespace tc;

constexpr int PT = 512;             // threads per CTA
constexpr int PW = PT / 32;         // warps per CTA
constexpr int STG = 65536;          // one pipeline stage: A hi | A lo | B hi | B lo, 16 KB each (BN = 128)
constexpr int MAX_N = 512;
constexpr int MAX_OBS = 32;
constexpr int MAX_APC = 64;         // agents per CTA (MAX_N / 8 CTAs)
constexpr int FILL_NA = 2;          // rows per warp in one pass of the row fill (4 at 128 registers spills in SI)

// barrier indices
// B_MAIN: both consumer warpgroups' main-loop MMAs of an edge tile retired; B_T2F: its chained gate GEMM retired
enum { B_FULL = 0, B_EMPTY = 3, B_B2F = 6, B_B2E = 8, B_MAIN = 10, B_T2F = 11, B_COUNT = 12 };

// Rollout constants staged in shared memory once per rollout (float offsets).  The epilogues and the tail read them
// per element, and every cluster barrier invalidates L1, so from global memory each phase would refetch them from L2.
// NU = 2 in every 2-D environment.
constexpr int PNU = 2;
enum {
    K_B23 = 0,          // [128] message bias (folded W23 layer)
    K_BIAS_G = 128,     // [128] gate hidden-layer bias
    K_AVEC = 256,       // [128] folded gate vector
    K_BU1 = 384,        // [256] update-layer bias
    K_BU1ROW = 640,     // [256] update-layer agent one-hot row
    K_BUH = 896,        // [256] folded update / head bias
    K_HO = 1152,        // [256][NU] folded output layer
    K_BHO = K_HO + 256 * PNU,   // [NU] output bias
    K_CST = K_BHO + PNU,        // [1] folded gate constant
    K_COL_THR = K_CST + 1,      // [1] two_r_sq_thr = sqrt_threshold(two_r)
    K_FLOATS = K_COL_THR + 1
};

struct PArgs {
    gcbf_env_desc d;
    int T, cap_env, C;
    // folded policy weights (gcbf_prepare_infer) and raw layer-1 / bias rows
    const float *W1, *b1, *b23, *bias_g, *avec, *cst, *b_u1, *b_u1row, *buh, *ho, *bho;
    const float *goal, *obstacles, *ray_table;
    float *agent, *hits, *actions, *rewards, *costs;     // trajectory record
    int32_t* counters;                                   // [T + 1][4]
    // per-environment scratch (L2)
    int32_t *row_start, *row_deg, *edge_recv, *edge_src; // [2][...] double-buffered lists
    float *msg, *logit, *ag, *v1, *z;
    float* terms;                                        // [2][A][4] per-agent reward / cost terms, by step parity
    unsigned long long* prof;                            // optional [T + 1][8] %globaltimer stamps of cluster 0 / CTA 0 (ns)
    // 1 when 2r < comm_radius: every agent closer than 2r is in the row, so the cost's collision term comes from the
    // neighbour scan of the graph build (s_col) instead of collides_prev's walk of the previous row
    int col_scan;
    // mode 0: one hardware cluster of C CTAs per environment (every barrier is barrier.cluster).
    // mode 1 ("pairs"): when fewer clusters of C CTAs than environments are resident (BASELINE's config has 16
    // environments of 8 CTAs), the C CTAs of an environment are C/2 hardware clusters of 2.  A pair owns 2 APC consecutive agents, their edge
    // rows (its own segment of the environment's edge lists), their edge tiles and their agent tile: the phases
    // E -> A -> U1 -> U2 and the graph build only need pair barriers (barrier.cluster, DSMEM for the row prefix);
    // the one environment-wide dependency -- the policy tail needs every agent's next state -- is a software barrier
    // (arrival counter in global memory) once per step.
    int soft;                                            // 0 / 1 = mode
    unsigned* gbar;                                      // [E] arrival counters of the environment barrier (zeroed by the launcher)
    // network table (gcbf_rollout_persistent_multi): environment e runs network net_of_env[e] (NULL: network 0), whose
    // raw parameters / folded weights sit p_stride / i_stride floats after the previous network's; the weight-plane maps
    // are 3-D with the network outermost.  counters is [T + 1][n_nets][4].
    const int32_t* net_of_env;
    int64_t p_stride, i_stride;
    int n_nets;
};

__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void cluster_sync_all() {
    __syncwarp();
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// software group barrier (soft mode): bar.sync, then one thread publishes this CTA's writes (gpu-scope fence, cumulative
// over the bar.sync), arrives on the environment's counter and spins with acquire loads until all C CTAs of the group
// have arrived for this generation; its trailing gpu-scope fence invalidates the SM's L1 for the loads that follow
__device__ __forceinline__ void soft_group_sync(unsigned* ctr, unsigned target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(ctr, 1u);
        unsigned v;
        const unsigned long long t0 = global_ns();
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
            if (v < target && global_ns() - t0 > MBAR_TIMEOUT_NS) __trap();   // same wall-time bound as mbar_wait
        } while (v < target);
        __threadfence();
    }
    __syncthreads();
}
__device__ __forceinline__ void fence_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
template <int KIND>
__global__ void __launch_bounds__(PT, 1)
rollout_persist_kernel(const __grid_constant__ PArgs P, const __grid_constant__ CUtensorMap tmW23h,
                       const __grid_constant__ CUtensorMap tmW23l, const __grid_constant__ CUtensorMap tmA1h,
                       const __grid_constant__ CUtensorMap tmA1l, const __grid_constant__ CUtensorMap tmU1h,
                       const __grid_constant__ CUtensorMap tmU1l, const __grid_constant__ CUtensorMap tmUHh,
                       const __grid_constant__ CUtensorMap tmUHl, const __grid_constant__ CUtensorMap tmAG,
                       const __grid_constant__ CUtensorMap tmV1) {
    using TR = EnvTraits<KIND>;
    constexpr int SD = TR::SD, ED = TR::ED, NU = TR::NU, PD = TR::PD;
    static_assert(PD == 2 && NU == PNU, "persistent rollout kernel: 2-D environments");
    constexpr int OBW = 16, OBS2 = OBS2D;
    constexpr int A_BYTES = 16384, B_BYTES = 16384;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align1024(smem_raw);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 3 * STG);
    int* s_tot = reinterpret_cast<int*>(smem + 3 * STG + 256 + 16);       // [8] CTA edge totals of the cluster
    float* sW = reinterpret_cast<float*>(smem + 3 * STG + 512);            // [(ED + 3)][256]
    float* sst = sW + 7 * 256;                                             // [N][SD] states of all agents of the environment
    float* sobs = sst + MAX_N * 4;                                         // [O][24]
    float* stab = sobs + MAX_OBS * OBS2;                                   // [32][2]
    unsigned* sbits = reinterpret_cast<unsigned*>(stab + 64);              // [APC][n_words | 1] neighbour words
    int* s_off = reinterpret_cast<int*>(sbits + 64 * 17);                  // [APC + 1]
    unsigned* s_hb = reinterpret_cast<unsigned*>(s_off + 72);              // [APC]
    float* s_red = reinterpret_cast<float*>(s_hb + 64);                    // [3][PW]
    float* sk = s_red + 3 * PW;                                            // [K_FLOATS] rollout constants
    uint8_t* s_col = reinterpret_cast<uint8_t*>(sk + K_FLOATS);            // [APC] collision flags of the graph built last

    const gcbf_env_desc& d = P.d;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int C = P.C;
    const bool soft = P.soft != 0;
    const int rank = (int)(blockIdx.x % C);          // CTA inside the environment
    const int env = blockIdx.x / C;
    const int L = soft ? 2 : C;                      // CTAs per LOCAL group = hardware cluster size
    const int lrank = rank % L, grp = rank / L;      // (cluster rank, group inside the environment)
    // SYNC_LOCAL: barrier of the hardware cluster (the CTAs that share edge rows / agent tiles).
    // SYNC_ENV(n): all C CTAs of the environment (mode 0: the same cluster barrier; pair mode: software barrier), the
    // n-th environment barrier of the rollout (pair mode: arrival target n * C).  It runs once per env-step.
#define SYNC_LOCAL() cluster_sync_all()
#define SYNC_ENV(n)                                                    \
    do {                                                               \
        if (soft) {                                                    \
            soft_group_sync(P.gbar + env, (n) * (unsigned)C);          \
        } else {                                                       \
            cluster_sync_all();                                        \
        }                                                              \
    } while (0)
    const int N = d.n_agents, E = d.n_graphs, O = d.n_obs, R = d.n_hits, cap = P.cap_env;
    const int A_tot = E * N;
    const int APC = (N + C - 1) / C;                 // agents per CTA
    const int a_lo = min(rank * APC, N), a_hi = min(a_lo + APC, N);
    const int n_words = (N + 31) / 32;
    const size_t env_e0 = (size_t)env * cap;          // first edge slot of this environment
    const int env_a0 = env * N;                       // first global agent id
    const int seg_cap = cap / (C / L);                // edge rows of one local group (mode 0: the whole environment)
    const int seg_off = grp * seg_cap;                // ... and where they start inside the environment's lists
    const int ga_lo = min(grp * L * APC, N), ga_hi = min(ga_lo + L * APC, N);   // agents of my local group
    // this environment's network.  Re-read where it is used (one L1 / L2 hit) rather than kept live across the step
    // loop: the kernel sits at its 128-register limit
    auto net = [&]() { return P.net_of_env != nullptr ? P.net_of_env[env] : 0; };

    // ---------------------------------------------------------------- one-time setup
    if (tid == 0) {
        for (int s = 0; s < 3; ++s) {
            mbar_init(&bars[B_FULL + s], 1);
            mbar_init(&bars[B_EMPTY + s], CONSUMERS);
        }
        for (int i = 0; i < 2; ++i) {
            mbar_init(&bars[B_B2F + i], 1);
            mbar_init(&bars[B_B2E + i], CONSUMERS);
        }
        mbar_init(&bars[B_MAIN], CONSUMERS);
        mbar_init(&bars[B_T2F], CONSUMERS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const int64_t p_off = net() * P.p_stride, i_off = net() * P.i_stride;   // this network's raw / folded weights
    load_l1_table<ED>(sW, P.W1 + p_off, P.b1 + p_off, tid, PT);   // message layer 1: W1[:ED] and the per-sender-type bias table
    auto stage = [&](int off, const float* src, int n) {
        for (int i = tid; i < n; i += PT) sk[off + i] = src[i];
    };
    stage(K_B23, P.b23 + i_off, 128);
    stage(K_BIAS_G, P.bias_g + p_off, 128);
    stage(K_AVEC, P.avec + i_off, 128);
    stage(K_BU1, P.b_u1 + p_off, 256);
    stage(K_BU1ROW, P.b_u1row + p_off, 256);
    stage(K_BUH, P.buh + i_off, 256);
    stage(K_HO, P.ho + i_off, 256 * NU);
    stage(K_BHO, P.bho + i_off, NU);
    stage(K_CST, P.cst + i_off, 1);
    // obstacles of this environment (+ derived far-skip fields) and the ray table stay resident for the whole rollout
    if (O > 0) {
        const float* ob = P.obstacles + (d.obs_per_graph ? (size_t)env * O * OBW : 0);
        for (int i = tid; i < O * OBW; i += PT) sobs[(i / OBW) * OBS2 + (i % OBW)] = ob[i];
    }
    for (int i = tid; i < d.n_rays * PD; i += PT) stab[i] = P.ray_table[i];
    for (int i = tid; i < MAX_APC; i += PT) s_col[i] = 0;
    if (tid == 0) sk[K_COL_THR] = sqrt_threshold(d.two_r);
    __syncthreads();
    derive_far_fields(sobs, O, d.comm_radius, tid, PT);
    uint32_t it = 0;      // k-blocks pushed through the 3-stage ring so far (all roles advance it identically)
    uint32_t ne = 0;      // edge tiles this CTA has processed (chain barriers)
    int M_cur = 0;        // edge rows of my local group's segment in the current graph
    SYNC_LOCAL();
    if (P.prof != nullptr && rank == 0 && tid == 0) P.prof[(size_t)(P.T + 1) * 8 + 2 * env] = gtime();   // cluster start

    // =================================================================================================
    for (int t = -1; t < P.T; ++t) {
        const int b = t & 1;                       // list half holding the graph of state t (t = -1: none)
        const float* agent_t = P.agent + (size_t)max(t, 0) * A_tot * SD;
        const float* hits_t = P.hits + (size_t)max(t, 0) * A_tot * R * PD;
        const int32_t* rs_t = P.row_start + (size_t)b * A_tot;
        const int32_t* rd_t = P.row_deg + (size_t)b * A_tot;
        const int32_t* er_t = P.edge_recv + (size_t)b * E * cap;
        const int32_t* es_t = P.edge_src + (size_t)b * E * cap;
        const bool stamp = P.prof != nullptr && blockIdx.x == 0 && tid == 0;
        unsigned long long* pr = P.prof + (size_t)(t + 1) * 8;
        if (stamp) pr[0] = gtime();
        if (t >= 0) {
            // ============================================================ phase E: edge tiles
            const int n_tiles = (M_cur + BM - 1) / BM;                  // tiles of my group's edge segment
            const int my_tiles = (n_tiles > lrank) ? (n_tiles - lrank + L - 1) / L : 0;
            const size_t seg_e0 = env_e0 + seg_off;                      // first slot of the segment
            if (warp == 0) {
                if (lane == 0) {
                    const int k = net();
                    uint32_t it_l = it, ne_l = ne;
                    for (int tile = lrank; tile < n_tiles; tile += L, ++ne_l) {
                        if (ne_l > 0) mbar_wait(&bars[B_T2F], (ne_l - 1) & 1);
                        for (int kb = 0; kb < 8; ++kb, ++it_l) {
                            const int s = it_l % 3;
                            mbar_wait(&bars[B_EMPTY + s], ((it_l / 3) & 1) ^ 1);
                            uint8_t* st = smem + s * STG;
                            mbar_expect_tx(&bars[B_FULL + s], 2 * B_BYTES);
                            tma_load_3d(st + 2 * A_BYTES, &tmW23h, &bars[B_FULL + s], kb * BK, 0, k);
                            tma_load_3d(st + 2 * A_BYTES + B_BYTES, &tmW23l, &bars[B_FULL + s], kb * BK, 0, k);
                        }
                        mbar_wait(&bars[B_MAIN], ne_l & 1);           // main-loop MMAs retired: stage 2 is free
                        for (int kb2 = 0; kb2 < 4; ++kb2) {
                            const uint32_t j2 = ne_l * 4 + kb2, slot = j2 & 1, use = j2 >> 1;
                            mbar_wait(&bars[B_B2E + slot], (use & 1) ^ 1);
                            uint8_t* sl = smem + 2 * STG + slot * 32768;
                            mbar_expect_tx(&bars[B_B2F + slot], 32768);
                            tma_load_3d(sl, &tmA1h, &bars[B_B2F + slot], kb2 * BK, 0, k);
                            tma_load_3d(sl + 16384, &tmA1l, &bars[B_B2F + slot], kb2 * BK, 0, k);
                        }
                    }
                }
            } else if (warp >= 8) {
                // consumer warpgroups (warps 8..15): PRODUCE the A operand of the tile in registers (each thread the
                // fragment of two edge rows: features + message layer 1, tf32 hi / lo split), issue the MMAs, drain the
                // message tile (global + shared-memory hand-over), run the chained gate GEMM and turn it into the gate
                // logits -- the code of tc::edge_chain_kernel, so the two paths give the same bits
                const int g = (warp - 8) >> 2, wt = tid & 127;
                const int r = 64 * g + frag_row0(wt);          // the thread's fragment rows r, r + 8 of the tile
                const int rs = r + 8 * setup_row(lane);         // ... and the one it sets up (tc::share_rows)
                uint32_t it_l = it, ne_l = ne;
                for (int tile = lrank; tile < n_tiles; tile += L, ++ne_l) {
                    const int ml = tile * BM + rs;
                    const bool row_ok = ml < M_cur;
                    float fs[ED], f[2][ED];
                    int ss = 0, stype[2];
#pragma unroll
                    for (int c = 0; c < ED; ++c) fs[c] = 0.f;
                    if (row_ok) {
                        const int a = min(max(er_t[seg_e0 + ml], env_a0), env_a0 + N - 1);
                        const int code = min(es_t[seg_e0 + ml], env_a0 + N - 1);
                        float er[ED], es[ED], coef, nrm;
                        // agent states come from the CTA's own copy of the environment's states (the values the
                        // record holds; no dependence on another CTA's global stores)
                        edge_state_dev<KIND>(sst + (size_t)(a - env_a0) * SD, er);
                        if (code >= 0) edge_state_dev<KIND>(sst + (size_t)(max(code, env_a0) - env_a0) * SD, es);
                        else sender_state_dev<KIND>(code, a, R, agent_t, P.goal, hits_t, es);
                        edge_feat_dev<KIND>(er, es, code == -1, d.comm_radius, fs, &coef, &nrm);
                        ss = (code >= 0) ? 2 : ((code == -1) ? 1 : 0);
                    }
                    share_rows<ED>(fs, ss, lane, f, stype);
                    const bool ok[2] = {tile * BM + r < M_cur, tile * BM + r + 8 < M_cur};
                    float dacc[64];
                    edge_tile_mainloop<ED>(dacc, smem, &bars[B_FULL], &bars[B_EMPTY], it_l, lane, ok, sW, f, stype);
                    mbar_arrive(&bars[B_MAIN]);
                    bar_consumers();               // both main loops retired: the hand-over may overwrite stages 0-1
                    drain_msg(dacc, smem, g, wt, sk + K_B23, P.msg + (seg_e0 + (size_t)tile * BM) * 128, M_cur - tile * BM);
                    fence_async_smem();
                    bar_wg(g);
                    float d2[64];
#pragma unroll
                    for (int i = 0; i < 64; ++i) d2[i] = 0.f;
                    for (int kb2 = 0; kb2 < 4; ++kb2) {
                        const uint32_t j2 = ne_l * 4 + kb2, slot = j2 & 1, use = j2 >> 1;
                        mbar_wait(&bars[B_B2F + slot], use & 1);
                        wg_fence();
                        chain_kblock(d2, smem, g, kb2, slot);
                        wg_commit();
                        wg_wait<0>();
                        mbar_arrive(&bars[B_B2E + slot]);
                    }
                    float q[2][1];
                    frag_relu_dot<1>(d2, sk + K_BIAS_G, sk + K_AVEC, 1, 1, wt, q);
                    if ((lane & 3) == 0) {
                        const int rr = tile * BM + 64 * g + frag_row0(wt);
                        if (rr < M_cur) P.logit[seg_e0 + rr] = q[0][0] + sk[K_CST];
                        if (rr + 8 < M_cur) P.logit[seg_e0 + rr + 8] = q[1][0] + sk[K_CST];
                    }
                    mbar_arrive(&bars[B_T2F]);
                }
            }
            it += 8u * my_tiles;
            ne += my_tiles;
            SYNC_LOCAL();
            if (stamp) pr[1] = gtime();

            // ============================================================ phase A: segment softmax + aggregate
            for (int il = a_lo + warp; il < a_hi; il += PW) {
                const int a = env_a0 + il;
                const int rs = rs_t[a];
                int rd = rd_t[a];
                if (rs < 0 || rs + rd > cap) rd = 0;
                *reinterpret_cast<float4*>(P.ag + (size_t)a * 128 + lane * 4) =
                    aggregate_logits(rs, rd, P.logit + env_e0, P.msg + env_e0 * 128, lane);
            }
            fence_async_global();          // generic-proxy writes of AG -> TMA (async proxy) reads in phase U1
            SYNC_LOCAL();
            if (stamp) pr[2] = gtime();

            // ============================================================ phases U1 / U2: agent-side GEMMs
            const int n_items = ((ga_hi - ga_lo + BM - 1) / BM) * 2;   // (agent tile of my group, 128-column half)
            const int my_items = (n_items > lrank) ? (n_items - lrank + L - 1) / L : 0;
            float* z_t = P.z + (size_t)(t & 1) * 2 * A_tot * 4;         // output partial sums, double-buffered by step parity
#pragma unroll 1
            for (int ph2 = 0; ph2 < 2; ++ph2) {
                const int nkb = ph2 == 0 ? 4 : 8;                      // K = 128 (update layer) / 256 (folded update/head)
                const CUtensorMap* tmA = ph2 == 0 ? &tmAG : &tmV1;
                const CUtensorMap* tmBh = ph2 == 0 ? &tmU1h : &tmUHh;
                const CUtensorMap* tmBl = ph2 == 0 ? &tmU1l : &tmUHl;
                if (warp == 0) {
                    if (lane == 0) {
                        const int k = net();
                        uint32_t it_l = it;
                        fence_async_global();      // consumer side of the generic-store -> TMA-load hand-over (AG / V1)
                        for (int item = lrank; item < n_items; item += L) {
                            const int m0 = ga_lo + (item >> 1) * BM, nc0 = (item & 1) * 128;
                            for (int kb = 0; kb < nkb; ++kb, ++it_l) {
                                const int s = it_l % 3;
                                mbar_wait(&bars[B_EMPTY + s], ((it_l / 3) & 1) ^ 1);
                                uint8_t* st = smem + s * STG;
                                mbar_expect_tx(&bars[B_FULL + s], A_BYTES + 2 * B_BYTES);
                                tma_load_2d(st, tmA, &bars[B_FULL + s], kb * BK, env_a0 + m0);
                                tma_load_3d(st + 2 * A_BYTES, tmBh, &bars[B_FULL + s], kb * BK, nc0, k);
                                tma_load_3d(st + 2 * A_BYTES + B_BYTES, tmBl, &bars[B_FULL + s], kb * BK, nc0, k);
                            }
                        }
                    }
                } else if (warp >= 8) {
                    // consumer warpgroups: split the TMA-landed A rows, MMAs, epilogue from the accumulator registers
                    // (U1: bias + one-hot row + ReLU -> V1; U2: output-layer partial sums of this column half -> z), the
                    // code and summation order of gemm_tc_kernel's EPI_BIAS_RELU / EPI_RELU_DOTN
                    const int g = (warp - 8) >> 2, wt = tid & 127;
                    uint32_t it_l = it;
                    for (int item = lrank; item < n_items; item += L) {
                        float dacc[64];
                        tma_a_mainloop(dacc, smem, &bars[B_FULL], &bars[B_EMPTY], it_l, nkb, g, wt);
                        const int m0 = ga_lo + (item >> 1) * BM, nc0 = (item & 1) * 128;
                        const int r0 = m0 + 64 * g + frag_row0(wt);     // agent inside the environment
                        if (ph2 == 0) {
#pragma unroll
                            for (int i = 0; i < 64; i += 2) {
                                const int ml = r0 + 8 * ((i >> 1) & 1);
                                if (ml >= ga_hi) continue;
                                const int n = nc0 + frag_col(wt, i);
                                float2 o = make_float2(dacc[i], dacc[i + 1]);
                                const float2 bb = *reinterpret_cast<const float2*>(sk + K_BU1 + n);
                                o.x += bb.x; o.y += bb.y;
                                const float2 b2 = *reinterpret_cast<const float2*>(sk + K_BU1ROW + n);
                                o.x += b2.x; o.y += b2.y;
                                o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f);
                                *reinterpret_cast<float2*>(P.v1 + (size_t)(env_a0 + ml) * 256 + n) = o;
                            }
                        } else {
                            float q[2][4];
                            frag_relu_dot<4>(dacc, sk + K_BUH + nc0, sk + K_HO + nc0 * NU, NU, NU, wt, q);
                            if ((lane & 3) == 0)
#pragma unroll
                                for (int h = 0; h < 2; ++h)
                                    if (r0 + 8 * h < ga_hi)
                                        *reinterpret_cast<float4*>(z_t + ((size_t)(item & 1) * A_tot + env_a0 + r0 + 8 * h) * 4) =
                                            make_float4(q[h][0], q[h][1], q[h][2], q[h][3]);
                        }
                    }
                }
                it += (uint32_t)nkb * my_items;
                if (ph2 == 0) fence_async_global();   // V1 rows (generic stores) -> TMA reads of phase U2
                if (ph2 == 0) SYNC_LOCAL();
                else SYNC_ENV((unsigned)t + 1u);      // the policy tail needs the output sums of EVERY agent
                if (stamp) pr[3 + ph2] = gtime();
            }
        }

        // ================================================================ phase G: tail + graph of state t + 1
        {
            const int tn = t + 1;
            float* agent_n = P.agent + (size_t)tn * A_tot * SD;
            float* hits_n = P.hits + (size_t)tn * A_tot * R * PD;
            const int bn_ = tn & 1;
            int32_t* rs_n = P.row_start + (size_t)bn_ * A_tot;
            int32_t* rd_n = P.row_deg + (size_t)bn_ * A_tot;
            int32_t* er_n = P.edge_recv + (size_t)bn_ * E * cap;
            int32_t* es_n = P.edge_src + (size_t)bn_ * E * cap;
            if (t < 0) {
                for (int i = tid; i < N; i += PT) {
                    const float* a = agent_n + (size_t)(env_a0 + i) * SD;
#pragma unroll
                    for (int c = 0; c < SD; ++c) sst[i * SD + c] = a[c];
                }
            } else {
                // fused policy tail (geometry.cu graph_build_kernel): every CTA recomputes the next state of all N
                // agents into its position table and records its own agents [a_lo, a_hi): action, next state and the
                // per-agent reward / cost terms (terms, by step parity).  The environment's first CTA reduces the terms
                // of step t - 1 in the same loop, with reduce_reward_cost's thread -> agent mapping.
                // Ordering: the owners wrote those terms, and the next states agent_t that collides_prev reads, in
                // phase G of step t - 1 (t = 0: agent_t is the initial state).  The environment barrier at the end of
                // this step's U2 (barrier.cluster release / acquire in mode 0; gpu-scope fences around the arrival
                // counter in pair mode) makes them visible here.  Terms of step t go to the other parity half.  The
                // half read here is rewritten in phase G of step t + 1, after that step's environment barrier, which
                // the first CTA reaches only after this reduce.
                const bool red = rank == 0 && t > 0;
                float acc[3] = {0.f, 0.f, 0.f};
                float* act_t = P.actions + (size_t)t * A_tot * NU;
                float* terms_t = P.terms + (size_t)(t & 1) * A_tot * 4;
                for (int i = tid; i < N; i += PT) {
                    const size_t a = (size_t)env_a0 + i;
                    if (red) {
                        const float4 v = *reinterpret_cast<const float4*>(P.terms + ((size_t)((t - 1) & 1) * A_tot + a) * 4);
                        acc[0] += v.x;
                        acc[1] += v.y;
                        acc[2] += v.z;
                    }
                    const bool own = i >= a_lo && i < a_hi;
                    float zz[4] = {0.f, 0.f, 0.f, 0.f};
                    const float* z_t = P.z + (size_t)(t & 1) * 2 * A_tot * 4;
                    for (int p = 0; p < 2; ++p) {
                        const float4 v = *reinterpret_cast<const float4*>(z_t + ((size_t)p * A_tot + a) * 4);
                        zz[0] += v.x; zz[1] += v.y; zz[2] += v.z; zz[3] += v.w;
                    }
                    float x[SD], gl[SD], ur[NU], act[NU], xn[SD];
#pragma unroll
                    for (int c = 0; c < SD; ++c) {
                        x[c] = sst[i * SD + c];              // state t (== agent_t[a], this CTA's copy)
                        gl[c] = P.goal[a * SD + c];
                    }
                    policy_action<KIND>(d, x, gl, zz, sk + K_BHO, ur, act);
                    if (own)
#pragma unroll
                        for (int c = 0; c < NU; ++c) act_t[a * NU + c] = act[c];
                    const float sq = step_agent<KIND>(d, x, gl, act, ur, true, xn);
#pragma unroll
                    for (int c = 0; c < SD; ++c) sst[i * SD + c] = xn[c];
                    if (own) {
#pragma unroll
                        for (int c = 0; c < SD; ++c) agent_n[a * SD + c] = xn[c];
                        const float nr = sqrtf(sq);
                        // the agent's own row of the graph of state t was filled by this CTA (phase G of step t - 1),
                        // and so was its collision flag, which is cleared here for the next graph
                        const bool col = P.col_scan ? s_col[i - a_lo] != 0
                                                    : collides_prev<PD, SD>(x, rs_t[a], rd_t[a], es_t + env_e0, agent_t, d.two_r);
                        s_col[i - a_lo] = 0;
                        const bool in_obs = O > 0 && inside_any<PD, OBS2>(sobs, O, x, d.radius);
                        *reinterpret_cast<float4*>(terms_t + a * 4) =
                            make_float4(nr * nr, col ? 1.f : 0.f, in_obs ? 1.f : 0.f, 0.f);
                    }
                }
                if (red)
                    reduce_reward_cost<PW>(acc, s_red, N, P.rewards + (size_t)(t - 1) * E + env,
                                           P.costs + (size_t)(t - 1) * E + env);
            }
            __syncthreads();
            if (stamp) pr[5] = gtime();

            // ---- neighbour words (thread per (word, agent)) with the collision flags, and LiDAR + active hit bits (warp
            // per agent) of this CTA's agents.  The words do not depend on the LiDAR, so the two overlap across warps.
            const int n_slots = a_hi - a_lo;
            const int bstride = n_words | 1;
            neighbour_words<PD, SD, true>(d, sst, a_lo, n_slots, sbits, bstride, tid, PT, sk[K_COL_THR], s_col);
            for (int slot = warp; slot < n_slots; slot += PW) {
                const int i = a_lo + slot;
                float p[PD], h[PD];
#pragma unroll
                for (int c = 0; c < PD; ++c) p[c] = sst[i * SD + c];
                float* my_hits = hits_n + ((size_t)env_a0 + i) * R * PD;
                lidar2d_warp(p, stab, sobs, O, d.n_rays, R, lane, my_hits, h[0], h[1]);
                const unsigned hit_bits = active_hit_bits<PD>(d, p, h, lane, true);
                if (lane == 0) s_hb[slot] = hit_bits;
            }
            __syncthreads();
            if (warp == 0) {                     // row degrees 1 + neighbours + active hits, their exclusive prefix (<= 64 rows)
                auto degree = [&](int slot) {
                    if (slot >= n_slots) return 0;
                    int c = 1 + __popc(s_hb[slot]);
                    for (int w = 0; w < n_words; ++w) c += __popc(sbits[slot * bstride + w]);
                    return c;
                };
                int v0 = degree(lane);
                int v1 = degree(lane + 32);
                int inc0 = v0, inc1 = v1;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int n0_ = __shfl_up_sync(0xffffffffu, inc0, o);
                    const int n1_ = __shfl_up_sync(0xffffffffu, inc1, o);
                    if (lane >= o) { inc0 += n0_; inc1 += n1_; }
                }
                const int tot0 = __shfl_sync(0xffffffffu, inc0, 31);
                __syncwarp();
                if (lane == 0) s_off[0] = 0;
                if (lane < APC) s_off[lane + 1] = inc0;
                if (lane + 32 < APC) s_off[lane + 33] = tot0 + inc1;
                __syncwarp();
                const int total = s_off[APC];
                if (lane < L) {                  // my total -> slot [lrank] of every CTA of my hardware cluster (DSMEM)
                    uint32_t ra;
                    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(smem_u32(&s_tot[lrank])), "r"(lane));
                    asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(ra), "r"(total) : "memory");
                }
            }
            SYNC_LOCAL();
            if (stamp) pr[6] = gtime();
            int base = 0, env_total = 0;         // (rows before mine, rows of my local group's segment)
            for (int r2 = 0; r2 < L; ++r2) {
                const int v = s_tot[r2];
                base += (r2 < lrank) ? v : 0;
                env_total += v;
            }
            // ---- fill pass: rows [goal | agents ascending | active hits ascending], agent order inside the environment,
            // FILL_NA agents per warp (slots s0 + PW a; slots past n_slots repeat s0 and write nothing).  An overflowed
            // row is dropped (row degree 0), and so is its collision flag: collides_prev finds no sender in it
            for (int s0 = warp; s0 < n_slots; s0 += PW * FILL_NA) {
                int rbase[FILL_NA], a_id[FILL_NA];
                bool ok[FILL_NA];
                const unsigned* my_bits[FILL_NA];
                unsigned hit_bits[FILL_NA];
#pragma unroll
                for (int a = 0; a < FILL_NA; ++a) {
                    const int slot = s0 + PW * a;
                    const bool in = slot < n_slots;
                    const int sl = in ? slot : s0;
                    a_id[a] = env_a0 + a_lo + sl;
                    const int deg = s_off[sl + 1] - s_off[sl];
                    const bool over = base + s_off[sl] + deg > seg_cap;
                    rbase[a] = seg_off + base + s_off[sl];       // row offset inside the environment's lists
                    ok[a] = in && !over;
                    my_bits[a] = sbits + sl * bstride;
                    hit_bits[a] = s_hb[sl];
                    if (in && lane == 0) {
                        if (over) {
                            atomicOr(&P.counters[((size_t)tn * P.n_nets + net()) * 4 + 1], 1);
                            s_col[sl] = 0;
                        }
                        rs_n[a_id[a]] = over ? 0 : rbase[a];
                        rd_n[a_id[a]] = over ? 0 : deg;
                    }
                }
                fill_row<FILL_NA>(er_n + env_e0, es_n + env_e0, rbase, a_id, ok, env_a0, my_bits, n_words, hit_bits, lane);
            }
            if (lrank == 0 && tid == 0) atomicAdd(&P.counters[((size_t)tn * P.n_nets + net()) * 4 + 0], min(env_total, seg_cap));
            M_cur = min(env_total, seg_cap);
            SYNC_LOCAL();
            if (stamp) pr[7] = gtime();
        }
    }
    // reward / cost of the last step: its owners wrote the terms in the last phase G
    if (P.T > 0) {
        SYNC_ENV((unsigned)P.T + 1u);
        if (rank == 0) {
            const int t = P.T - 1;
            float acc[3] = {0.f, 0.f, 0.f};
            for (int i = tid; i < N; i += PT) {
                const float4 v = *reinterpret_cast<const float4*>(P.terms + ((size_t)(t & 1) * A_tot + env_a0 + i) * 4);
                acc[0] += v.x;
                acc[1] += v.y;
                acc[2] += v.z;
            }
            reduce_reward_cost<PW>(acc, s_red, N, P.rewards + (size_t)t * E + env, P.costs + (size_t)t * E + env);
        }
    }
#undef SYNC_LOCAL
#undef SYNC_ENV
    if (P.prof != nullptr && rank == 0 && tid == 0) P.prof[(size_t)(P.T + 1) * 8 + 2 * env + 1] = gtime();   // cluster end
}

struct WsLayout {
    int64_t msg, logit, ag, v1, z, terms, row_start, row_deg, edge_recv, edge_src, gbar, total;
};
static WsLayout make_ws_layout(int E, int N, int cap_env) {   // (+ 16 (T + 1) floats of phase stamps appended by the caller)
    WsLayout W;
    int64_t o = 0;
    auto take = [&](int64_t n) { int64_t r = o; o += (n + 63) & ~(int64_t)63; return r; };
    const int64_t A = (int64_t)E * N, EC = (int64_t)E * cap_env;
    W.msg = take(EC * 128);
    W.logit = take(EC);
    W.ag = take(A * 128 + 128 * 128);      // + one tile of slack: the last environment's row tile may overhang
    W.v1 = take(A * 256 + 128 * 256);
    W.z = take(2 * 2 * A * 4);             // [step parity][column half][A][4]
    W.terms = take(2 * A * 4);             // [step parity][A][||u - u_ref||^2, collides, inside an obstacle, 0]
    W.row_start = take(2 * A);
    W.row_deg = take(2 * A);
    W.edge_recv = take(2 * EC);
    W.edge_src = take(2 * EC);
    W.gbar = take(E);
    W.total = o;
    return W;
}
static int cluster_size(int N, int cap_env) {
    const int items = ((N + 127) / 128) * 2;
    const int tiles = (min(cap_env, 3 * N) + 127) / 128;      // typical real edge count ~2 N
    int c = 1;
    while (c < 8 && c < max(items, tiles)) c <<= 1;
    return c;
}

}  // namespace rp
}  // namespace gcbf

using namespace gcbf;

extern "C" __attribute__((visibility("default"))) int64_t gcbf_rollout_persistent_workspace_floats(const gcbf_env_desc* desc) {
    if (!desc || desc->edge_cap <= 0 || desc->n_graphs <= 0 || desc->n_agents <= 0) return -1;
    return rp::make_ws_layout(desc->n_graphs, desc->n_agents, desc->edge_cap / desc->n_graphs).total + 64;
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_rollout_persistent_max_clusters(int32_t cluster_size);

// 0: unsupported configuration; 1: supported, but the device cannot keep one cluster per environment resident at the
// same time (environments beyond the resident clusters wait for a free cluster slot and the rollout takes two rounds);
// 2: supported and fully co-resident.
extern "C" __attribute__((visibility("default"))) int32_t gcbf_rollout_persistent_supported(const gcbf_env_desc* desc) {
    if (!desc) return 0;
    const bool ok = desc->env_kind >= 0 && desc->env_kind <= 2 && desc->n_agents >= 1 && desc->n_agents <= rp::MAX_N &&
                    desc->n_obs <= rp::MAX_OBS && desc->n_rays <= 32 && desc->n_hits == desc->n_rays && desc->n_graphs >= 1 &&
                    desc->edge_cap / desc->n_graphs >= desc->n_agents && (desc->obs_per_graph == 1 || desc->n_obs == 0);
    if (!ok) return 0;
    const int C = rp::cluster_size(desc->n_agents, desc->edge_cap / desc->n_graphs);
    static int cached[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};     // occupancy per cluster size (0 = not queried yet)
    if (cached[C] == 0) {
        const int n = gcbf_rollout_persistent_max_clusters(C);
        cached[C] = n > 0 ? n : -1;
    }
    if (cached[C] > 0 && desc->n_graphs <= cached[C]) return 2;          // one hardware cluster per environment, all resident
    if (cached[2] == 0) {
        const int n = gcbf_rollout_persistent_max_clusters(2);
        cached[2] = n > 0 ? n : -1;
    }
    if (C >= 2 && desc->n_graphs * C <= sm_count() && desc->n_graphs * (C / 2) <= cached[2]) return 2;   // pair mode
    return 1;
}

static int persist_smem_bytes() {
    return 3 * rp::STG + 512 + 7 * 256 * 4 + rp::MAX_N * 4 * 4 + rp::MAX_OBS * 24 * 4 + 64 * 4 + 64 * 17 * 4 + 72 * 4 + 64 * 4 +
           3 * rp::PW * 4 + rp::K_FLOATS * 4 + rp::MAX_APC + 1024;
}

/* Co-resident clusters of `cluster_size` CTAs of the persistent rollout kernel on the current device
 * (cudaOccupancyMaxActiveClusters): environments beyond this number wait for a free cluster slot. */
extern "C" __attribute__((visibility("default"))) int32_t gcbf_rollout_persistent_max_clusters(int32_t cluster_size) {
    auto kern = rp::rollout_persist_kernel<GCBF_ENV_DOUBLE_INTEGRATOR>;
    const int smem = persist_smem_bytes();
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return -1;
    if (cluster_size > 8 &&
        cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) return -1;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)(cluster_size * 64), 1, 1);
    cfg.blockDim = dim3(rp::PT, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cluster_size;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    return n;
}

// Per-network strides of the stacked arrays of gcbf_rollout_persistent_multi: the raw-parameter and folded-weight counts
// rounded up to 4 floats (16 bytes: the stride of a TMA map and the alignment every network's block keeps).
static int64_t net_stride(int64_t count) { return (count + 3) & ~(int64_t)3; }

extern "C" __attribute__((visibility("default"))) int32_t gcbf_rollout_persistent_multi_strides(
    int32_t edge_dim, int32_t out_dim, int64_t* param_stride, int64_t* infer_stride) {
    GCBF_REQUIRE(param_stride && infer_stride, "gcbf_rollout_persistent_multi_strides: NULL pointer argument");
    const int32_t pc = gcbf_param_count_l(edge_dim, out_dim, 1), ic = gcbf_infer_count(edge_dim, out_dim);
    GCBF_REQUIRE(pc > 0 && ic > 0, "gcbf_rollout_persistent_multi_strides: bad argument (edge_dim %d, out_dim %d)",
                 edge_dim, out_dim);
    *param_stride = net_stride(pc);
    *infer_stride = net_stride(ic);
    return 0;
}

// The launch behind gcbf_rollout_persistent (n_nets = 1, net_of_env NULL) and gcbf_rollout_persistent_multi.  `rounds`
// (the multi entry point) also launches when the environments' clusters are not all co-resident and pair mode does not
// fit: in mode 0 no cluster ever waits on another, so the clusters beyond the resident ones run in later rounds.
static int32_t persist_launch(const char* who, bool rounds, const gcbf_env_desc* desc, int32_t n_steps, int32_t n_nets,
                              const float* actor_params, const float* infer_blob, const int32_t* net_of_env,
                              const float* goal, const float* obstacles, const float* ray_table, float* agent_rec,
                              float* hits_rec, float* actions_rec, float* rewards, float* costs, int32_t* counters,
                              float* workspace, int64_t workspace_floats, uint64_t* phase_stamps, void* stream) {
    GCBF_REQUIRE(desc && actor_params && infer_blob && goal && ray_table && agent_rec && hits_rec && actions_rec && rewards &&
                     costs && counters && workspace, "%s: NULL pointer argument", who);
    GCBF_REQUIRE(gcbf_rollout_persistent_supported(desc) > 0, "%s: unsupported configuration (2-D envs, "
                 "n_agents <= 512, n_obs <= 32, edge_cap >= n_graphs * n_agents)", who);
    GCBF_REQUIRE(desc->n_obs == 0 || obstacles, "obstacles is NULL but n_obs > 0");
    GCBF_REQUIRE(n_steps >= 0, "n_steps must be >= 0");
    const int E = desc->n_graphs, N = desc->n_agents;
    const int cap_env = desc->edge_cap / E;
    const rp::WsLayout W = rp::make_ws_layout(E, N, cap_env);
    GCBF_REQUIRE(workspace_floats >= W.total, "workspace too small: %lld < %lld floats", (long long)workspace_floats,
                 (long long)W.total);
    GCBF_REQUIRE(((uintptr_t)workspace & 255) == 0 && ((uintptr_t)actor_params & 15) == 0 && ((uintptr_t)infer_blob & 15) == 0,
                 "workspace must be 256-byte aligned, parameters 16-byte aligned");
    const int ed = env_ed(desc->env_kind), nu = env_nu(desc->env_kind);
    const ParamLayout L = make_layout(ed, nu);
    const InferLayout I = make_infer_layout(nu);
    rp::PArgs P;
    memset(&P, 0, sizeof(P));
    P.d = *desc;
    P.T = n_steps;
    P.cap_env = cap_env;
    P.C = rp::cluster_size(N, cap_env);
    P.col_scan = desc->two_r < desc->comm_radius ? 1 : 0;
    P.net_of_env = net_of_env;
    P.n_nets = n_nets;
    P.p_stride = net_stride(gcbf_param_count_l(ed, nu, 1));
    P.i_stride = net_stride(gcbf_infer_count(ed, nu));
    const int max_cl = gcbf_rollout_persistent_max_clusters(P.C);
    // mode 0: one hardware cluster per environment when all of them are resident at once; otherwise mode 1: clusters of 2 + one software barrier per step, when the grid fits on the
    // device (1 CTA / SM).  GCBF_PERSIST_SOFT=1 forces mode 1 (tests).
    static const int force_soft = [] { const char* e = getenv("GCBF_PERSIST_SOFT"); return e ? atoi(e) : -1; }();
    const bool pairs_fit = P.C >= 2 && E * P.C <= sm_count();
    P.soft = (force_soft >= 0) ? (force_soft != 0) : ((E <= max_cl || (rounds && !pairs_fit)) ? 0 : 1);
    GCBF_REQUIRE(!P.soft || pairs_fit, "pair mode needs n_graphs * %d <= %d CTAs", P.C, sm_count());
    GCBF_REQUIRE(P.soft || E <= max_cl || force_soft == 0 || rounds, "more environments (%d) than resident clusters (%d)", E,
                 max_cl);
    P.gbar = reinterpret_cast<unsigned*>(workspace + W.gbar);
    P.W1 = actor_params + L.w[L_MSG0];
    P.b1 = actor_params + L.b[L_MSG0];
    P.b23 = infer_blob + I.b23;
    P.bias_g = actor_params + L.b[L_ATT0];
    P.avec = infer_blob + I.a23;
    P.cst = infer_blob + I.c23;
    P.b_u1 = actor_params + L.b[L_UPD0];
    P.b_u1row = actor_params + L.w[L_UPD0] + 2 * 256;
    P.buh = infer_blob + I.buh;
    P.ho = infer_blob + I.ho;
    P.bho = infer_blob + I.bho;
    P.goal = goal;
    P.obstacles = obstacles;
    P.ray_table = ray_table;
    P.agent = agent_rec;
    P.hits = hits_rec;
    P.actions = actions_rec;
    P.rewards = rewards;
    P.costs = costs;
    P.counters = counters;
    P.prof = reinterpret_cast<unsigned long long*>(phase_stamps);
    P.msg = workspace + W.msg;
    P.logit = workspace + W.logit;
    P.ag = workspace + W.ag;
    P.v1 = workspace + W.v1;
    P.z = workspace + W.z;
    P.terms = workspace + W.terms;
    P.row_start = reinterpret_cast<int32_t*>(workspace + W.row_start);
    P.row_deg = reinterpret_cast<int32_t*>(workspace + W.row_deg);
    P.edge_recv = reinterpret_cast<int32_t*>(workspace + W.edge_recv);
    P.edge_src = reinterpret_cast<int32_t*>(workspace + W.edge_src);
    CUtensorMap tW23h, tW23l, tA1h, tA1l, tU1h, tU1l, tUHh, tUHl, tAG, tV1;
    int32_t rc;
    const int K = n_nets;
    const int64_t S = P.i_stride;
#define RC(x) do { if ((rc = (x))) return rc; } while (0)
    RC(tc::make_map_stack(&tW23h, infer_blob + I.t_w23, 128, 256, 128, K, S));
    RC(tc::make_map_stack(&tW23l, infer_blob + I.t_w23 + 256 * 128, 128, 256, 128, K, S));
    RC(tc::make_map_stack(&tA1h, infer_blob + I.t_a1, 128, 128, 128, K, S));
    RC(tc::make_map_stack(&tA1l, infer_blob + I.t_a1 + 128 * 128, 128, 128, 128, K, S));
    RC(tc::make_map_stack(&tU1h, infer_blob + I.t_u1, 256, 128, 128, K, S));
    RC(tc::make_map_stack(&tU1l, infer_blob + I.t_u1 + 256 * 128, 256, 128, 128, K, S));
    RC(tc::make_map_stack(&tUHh, infer_blob + I.t_uh, 256, 256, 128, K, S));
    RC(tc::make_map_stack(&tUHl, infer_blob + I.t_uh + 256 * 256, 256, 256, 128, K, S));
    RC(tc::make_map(&tAG, P.ag, E * N + 128, 128, 128));
    RC(tc::make_map(&tV1, P.v1, E * N + 128, 256, 128));
#undef RC
    const int smem = persist_smem_bytes();
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)(E * P.C), 1, 1);
    cfg.blockDim = dim3(rp::PT, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)(P.soft ? 2 : P.C);
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    // pair mode spins on a counter the other CTAs of the environment must reach: every CTA has to be resident.  The grid
    // was checked against the SM count (1 CTA / SM) and the cluster-of-2 occupancy above.  A protocol failure ends in a
    // trap, not a hang.
    cudaError_t e = cudaSuccess;
    if (P.soft && (e = cudaMemsetAsync(P.gbar, 0, sizeof(unsigned) * E, (cudaStream_t)stream)) != cudaSuccess) {
        set_error("cudaMemsetAsync: %s", cudaGetErrorString(e));
        return (int32_t)e;
    }
    switch (desc->env_kind) {
#define GCBF_RP_CASE(K)                                                                                               \
    case K: {                                                                                                         \
        auto kern = rp::rollout_persist_kernel<K>;                                                                    \
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);                            \
        if (e == cudaSuccess)                                                                                         \
            e = cudaLaunchKernelEx(&cfg, kern, P, tW23h, tW23l, tA1h, tA1l, tU1h, tU1l, tUHh, tUHl, tAG, tV1);        \
    } break;
        GCBF_RP_CASE(GCBF_ENV_SINGLE_INTEGRATOR)
        GCBF_RP_CASE(GCBF_ENV_DOUBLE_INTEGRATOR)
        GCBF_RP_CASE(GCBF_ENV_DUBINS_CAR)
#undef GCBF_RP_CASE
        default: set_error("%s: bad env_kind", who); return -1;
    }
    if (e != cudaSuccess) {
        set_error("rollout_persist_kernel launch: %s", cudaGetErrorString(e));
        return (int32_t)e;
    }
    count_launch();
    return check_launch("rollout_persist_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_rollout_persistent(
    const gcbf_env_desc* desc, int32_t n_steps, const float* actor_params, const float* infer_blob, const float* goal,
    const float* obstacles, const float* ray_table, float* agent_rec, float* hits_rec, float* actions_rec, float* rewards,
    float* costs, int32_t* counters, float* workspace, int64_t workspace_floats, uint64_t* phase_stamps, void* stream) {
    return persist_launch("gcbf_rollout_persistent", false, desc, n_steps, 1, actor_params, infer_blob, nullptr, goal,
                          obstacles, ray_table, agent_rec, hits_rec, actions_rec, rewards, costs, counters, workspace,
                          workspace_floats, phase_stamps, stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_rollout_persistent_multi(
    const gcbf_env_desc* desc, int32_t n_steps, int32_t n_nets, const float* actor_params, const float* infer_blob,
    const int32_t* net_of_env, const float* goal, const float* obstacles, const float* ray_table, float* agent_rec,
    float* hits_rec, float* actions_rec, float* rewards, float* costs, int32_t* counters, float* workspace,
    int64_t workspace_floats, uint64_t* phase_stamps, void* stream) {
    GCBF_REQUIRE(n_nets >= 1, "gcbf_rollout_persistent_multi: n_nets must be >= 1, got %d", n_nets);
    GCBF_REQUIRE(net_of_env != nullptr, "gcbf_rollout_persistent_multi: net_of_env is NULL");
    GCBF_REQUIRE(((uintptr_t)actor_params & 15) == 0 && ((uintptr_t)infer_blob & 15) == 0 && ((uintptr_t)net_of_env & 3) == 0,
                 "gcbf_rollout_persistent_multi: the stacked actor_params / infer_blob must be 16-byte aligned, "
                 "net_of_env 4-byte aligned");
    return persist_launch("gcbf_rollout_persistent_multi", true, desc, n_steps, n_nets, actor_params, infer_blob,
                          net_of_env, goal, obstacles, ray_table, agent_rec, hits_rec, actions_rec, rewards, costs,
                          counters, workspace, workspace_floats, phase_stamps, stream);
}
