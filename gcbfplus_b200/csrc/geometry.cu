// geometry.cu -- graph build (radius neighbour lists + LiDAR ray cast + top-k), labels and
// the per-agent dynamics step.  Compiled with -fmad=false: every arithmetic step keeps the
// reference's one-rounding-per-op semantics, so index sets / hit ordering / masks are
// bit-exact against the CPU oracle (oracle/geometry.py, oracle/envs.py).
//
// Replaces (reference paths): gcbfplus/env/utils.py:49-131 (get_lidar, raytracing,
// inside_obstacles), env/obstacle.py:53-96 (Rectangle), :234-270 (Sphere),
// env/double_integrator.py:223-264 (edge_blocks), :128-198 (step/cost), :332-338 (u_ref),
// :356-440 (masks) and their SingleIntegrator / DubinsCar / LinearDrone twins,
// algo/gcbf_plus.py:160-186 (safe_mask horizon labelling, act).
#include <math.h>

#include "common.cuh"
#include "geometry_dev.cuh"

namespace gcbf {

// ------------------------------------------------------------------------------------
// graph build: one warp per agent, GB_WARPS agents per CTA, grid = (ceil(N/GB_WARPS), G)
// smem: positions of all N agents of the graph, its obstacles, 3-D alpha scratch.
// ------------------------------------------------------------------------------------
template <int KIND>
__global__ void __launch_bounds__(GB_WARPS * 32)
graph_build_kernel(const gcbf_env_desc d, const float* __restrict__ agent, const float* __restrict__ obstacles,
                   const float* __restrict__ ray_table, float* __restrict__ hits, int32_t* __restrict__ row_start,
                   int32_t* __restrict__ row_deg, int32_t* __restrict__ edge_recv, int32_t* __restrict__ edge_src,
                   int32_t* __restrict__ counters, const int do_cast, const TailArgs tl,
                   float* __restrict__ reward, float* __restrict__ cost, const int rounds) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, PD = T::PD, NU = T::NU;
    constexpr int OBW = (PD == 2) ? 16 : 4;
    extern __shared__ float smem[];
    const int N = d.n_agents, O = d.n_obs, R = d.n_hits;
    constexpr int OBS2 = (PD == 2) ? OBS2D : 4; // 2-D: packed rectangle + the derived fields of derive_far_fields
    float* spos = smem;                         // [N, PD]
    float* sobs = spos + N * PD;                // [O, OBS2]
    float* stab = sobs + O * OBS2;              // [n_rays, PD]
    float* salpha = stab + d.n_rays * PD;       // 3-D only: [GB_WARPS, n_rays]
    const int n_words = (N + 31) / 32;
    unsigned* sbits = reinterpret_cast<unsigned*>(salpha + (PD == 3 ? GB_WARPS * d.n_rays : 0));  // [GB_WARPS, n_words]
    int* stk = reinterpret_cast<int*>(sbits + GB_WARPS * n_words);                                 // 3-D only: [GB_WARPS, 96] top-k scratch
    __shared__ int s_off[GB_WARPS + 1];
    __shared__ int s_base;

    const int g = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (O > 0) {
        const float* ob = obstacles + (d.obs_per_graph ? (size_t)g * O * OBW : 0);
        for (int i = tid; i < O * OBW; i += blockDim.x) sobs[(i / OBW) * OBS2 + (i % OBW)] = ob[i];
    }
    for (int i = tid; i < d.n_rays * PD; i += blockDim.x) stab[i] = ray_table[i];
    if (tl.z == nullptr) {
        for (int i = tid; i < N; i += blockDim.x) {
            const float* a = agent + ((size_t)g * N + i) * SD;
#pragma unroll
            for (int c = 0; c < PD; ++c) spos[i * PD + c] = a[c];
        }
    } else {
        // ---- fused policy tail (rollout step): pi = tanh(sum_parts z + bHO) (policy.py:72), a = 2 pi + u_ref
        // (gcbf_plus.py:182-186), clip_action, agent_step_euler (double_integrator.py:128-143).  Every CTA of graph g
        // recomputes the next state of all N agents (thread per agent, a few hundred instructions) straight into its
        // position table -- that replaces a separate kernel and a round trip through HBM; the graph's first CTA also
        // records actions / next states and reduces the reward / cost terms of the step (double_integrator.py:145-198)
        // in a fixed order.  The cost reads the PREVIOUS edge lists (the new ones are being written by this kernel
        // into the other half of the caller's double buffer).
        __shared__ float s_red[3][GB_WARPS];
        const bool rec = blockIdx.x == 0;
        float acc[3] = {0.f, 0.f, 0.f};
        for (int i = tid; i < N; i += blockDim.x) {
            const size_t a = (size_t)g * N + i;
            float zz[4] = {0.f, 0.f, 0.f, 0.f};
            for (int p = 0; p < tl.parts; ++p) {
                const float4 v = *reinterpret_cast<const float4*>(tl.z + ((size_t)p * tl.z_cap + a) * 4);
                zz[0] += v.x; zz[1] += v.y; zz[2] += v.z; zz[3] += v.w;
            }
            float x[SD], gl[SD], ur[NU], act[NU], xn[SD];
#pragma unroll
            for (int c = 0; c < SD; ++c) {
                x[c] = tl.agent_prev[a * SD + c];
                gl[c] = tl.goal[a * SD + c];
            }
            policy_action<KIND>(d, x, gl, zz, tl.bHO, ur, act);
            if (rec)
#pragma unroll
                for (int c = 0; c < NU; ++c) tl.action[a * NU + c] = act[c];
            const float sq = step_agent<KIND>(d, x, gl, act, ur, true, xn);
#pragma unroll
            for (int c = 0; c < PD; ++c) spos[i * PD + c] = xn[c];
            if (rec) {
#pragma unroll
                for (int c = 0; c < SD; ++c) tl.next_agent[a * SD + c] = xn[c];
                const float nr = sqrtf(sq);
                const bool col = collides_prev<PD, SD>(x, tl.row_start_prev[a], tl.row_deg_prev[a], tl.edge_src_prev,
                                                       tl.agent_prev, d.two_r);
                bool in_obs = false;
                if (O > 0) {
                    const float* ob = obstacles + (d.obs_per_graph ? (size_t)g * O * OBW : 0);
                    in_obs = inside_any<PD>(ob, O, x, d.radius);
                }
                acc[0] += nr * nr;
                acc[1] += col ? 1.f : 0.f;
                acc[2] += in_obs ? 1.f : 0.f;
            }
        }
        if (rec) reduce_reward_cost<GB_WARPS>(acc, &s_red[0][0], N, reward + g, cost + g);
    }
    __syncthreads();
    if (PD == 2) {   // derived fields for the (conservative, exactness-preserving) far-obstacle skip
        derive_far_fields(sobs, O, d.comm_radius, tid, blockDim.x);
        __syncthreads();
    }

    // A CTA serves `rounds` groups of GB_WARPS agents: at ~60 registers per thread one 1024-thread CTA fills an SM, so
    // the grid is sized to one wave (graph_build_impl) instead of paying the prologue (and the fused tail) per wave.
    for (int round = 0; round < rounds; ++round) {
    const int i = (blockIdx.x * rounds + round) * GB_WARPS + warp;
    const bool valid = i < N;
    const int ii = valid ? i : 0;
    float p[PD];
#pragma unroll
    for (int c = 0; c < PD; ++c) p[c] = spos[ii * PD + c];
    const size_t a_glob = (size_t)g * N + ii;
    float* my_hits = hits + a_glob * R * PD;

    // ---------------- LiDAR (env/utils.py:49-131)
    if (do_cast && valid) {
        if (PD == 2) {
            lidar2d_warp(p, stab, sobs, O, d.n_rays, R, lane, my_hits);
        } else {
            const bool is_in = (O > 0) ? inside_any<PD>(sobs, O, p, 0.f) : false;
            const float keep = 1.f - (is_in ? 1.f : 0.f);
            float* al = salpha + warp * d.n_rays;
            const float x1 = p[0], y1 = p[1], z1 = p[PD - 1];
            for (int r = lane; r < d.n_rays; r += 32) {
                const float x2 = x1 + stab[r * PD + 0], y2 = y1 + stab[r * PD + 1], z2 = z1 + stab[r * PD + PD - 1];
                float alpha;
                if (O == 0) {
                    alpha = 1.f * NO_HIT;
                } else {
                    alpha = sphere_raytrace(sobs, x1, y1, z1, x2, y2, z2);
                    for (int o = 1; o < O; ++o)
                        alpha = nanmin(alpha, sphere_raytrace(sobs + 4 * o, x1, y1, z1, x2, y2, z2));
                    alpha = alpha * keep;
                }
                al[r] = alpha;
            }
            __syncwarp();
            // ---- argsort(alpha)[:R] (env/utils.py:127-131), stable.  Almost every ray misses (alpha == 1e6 exactly) and
            // argsort is stable, so the result is [the few real returns sorted by (alpha, ray)] followed by the first
            // missing rays in ray order.  Fast path (measured: the R-round arg-min below was more than half of this kernel
            // at 514 rays): if at most 32 rays have alpha < 1e6 and no alpha is NaN / above 1e6, compact those rays, sort
            // them with one 32-key warp sort and fill up with the lowest-index misses -- the same permutation.
            bool fast = false;
            if (R <= 32) {
                int nA = 0;
                bool odd = false;
                for (int r = lane; r < d.n_rays; r += 32) {
                    const float a = al[r];
                    odd = odd || !(a <= NO_HIT);            // NaN or above the miss value: leave it to the general path
                    nA += (a < NO_HIT) ? 1 : 0;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) nA += __shfl_xor_sync(0xffffffffu, nA, o);
                fast = !__any_sync(0xffffffffu, odd) && nA <= 32 && (d.n_rays - nA) >= R;
                if (fast) {
                    // [0,32) ray of a return, [32,64) its alpha bits, [64,96) first misses: up to R <= 32 of them are
                    // needed (no returns at all)
                    int* tk = stk + warp * 96;
                    const unsigned lt = (1u << lane) - 1u;
                    int nret = 0, nmiss = 0;
                    for (int r0 = 0; r0 < d.n_rays; r0 += 32) {
                        const int r = r0 + lane;
                        const float a = (r < d.n_rays) ? al[r] : NO_HIT;
                        const bool is_ret = (r < d.n_rays) && (a < NO_HIT);
                        const bool is_miss = (r < d.n_rays) && !(a < NO_HIT);
                        const unsigned rb = __ballot_sync(0xffffffffu, is_ret), mb = __ballot_sync(0xffffffffu, is_miss);
                        if (is_ret) {
                            const int pos = nret + __popc(rb & lt);
                            tk[pos] = r;
                            tk[32 + pos] = __float_as_int(a);
                        }
                        if (is_miss) {
                            const int pos = nmiss + __popc(mb & lt);
                            if (pos < 32) tk[64 + pos] = r;
                        }
                        nret += __popc(rb);
                        nmiss += __popc(mb);
                    }
                    __syncwarp();
                    SortKey k;
                    k.flag = (lane < nret) ? 0 : 2;
                    k.alpha = (lane < nret) ? __int_as_float(tk[32 + lane]) : 0.f;
                    k.idx = (lane < nret) ? tk[lane] : (0x40000000 + lane);
                    if (nret > 1) k = warp_sort32(k, lane);
                    if (lane < R) {
                        const int r = (lane < nret) ? k.idx : tk[64 + lane - nret];   // lane - nret < R - nret <= 32
                        const float a = (lane < nret) ? k.alpha : NO_HIT;
                        const float x2 = x1 + stab[r * PD + 0], y2 = y1 + stab[r * PD + 1], z2 = z1 + stab[r * PD + PD - 1];
                        my_hits[lane * PD + 0] = x1 + (x2 - x1) * a;
                        my_hits[lane * PD + 1] = y1 + (y2 - y1) * a;
                        my_hits[lane * PD + PD - 1] = z1 + (z2 - z1) * a;
                    }
                }
            }
            // general path: R rounds of stable arg-min with removal
            for (int rank = 0; rank < (fast ? 0 : R); ++rank) {
                SortKey best;
                best.flag = 3;
                best.alpha = 0.f;
                best.idx = 0x7fffffff;
                for (int r = lane; r < d.n_rays; r += 32) {
                    const float a = al[r];
                    SortKey k;
                    k.flag = (__float_as_uint(a) == 0xffc00001u) ? 3 : (isnan(a) ? 1 : 0);
                    k.alpha = a;
                    k.idx = r;
                    if (key_less(k, best)) best = k;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    SortKey other;
                    other.flag = __shfl_xor_sync(0xffffffffu, best.flag, o);
                    other.alpha = __shfl_xor_sync(0xffffffffu, best.alpha, o);
                    other.idx = __shfl_xor_sync(0xffffffffu, best.idx, o);
                    if (key_less(other, best)) best = other;
                }
                if (lane == 0) {
                    const int r = best.idx;
                    const float a = best.alpha;
                    const float x2 = x1 + stab[r * PD + 0], y2 = y1 + stab[r * PD + 1], z2 = z1 + stab[r * PD + PD - 1];
                    my_hits[rank * PD + 0] = x1 + (x2 - x1) * a;
                    my_hits[rank * PD + 1] = y1 + (y2 - y1) * a;
                    my_hits[rank * PD + PD - 1] = z1 + (z2 - z1) * a;
                    al[r] = __uint_as_float(0xffc00001u);  // tombstone (a NaN payload no alpha can have)
                }
                __syncwarp();
            }
        }
        __syncwarp();
    }
    __syncwarp();

    // ---------------- active hit nodes and neighbours; the ballots are kept in shared memory for the fill pass
    const unsigned hit_bits = active_hit_bits<PD>(d, p, my_hits, lane, valid);
    int cnt = 0;
    unsigned* my_bits = sbits + warp * n_words;
    if (valid) cnt = neighbour_bits<PD, PD>(d, p, i, spos, lane, my_bits);
    const int deg = valid ? (1 + cnt + __popc(hit_bits)) : 0;
    if (lane == 0) s_off[warp + 1] = deg;
    __syncthreads();
    if (tid == 0) {
        s_off[0] = 0;
        for (int w = 0; w < GB_WARPS; ++w) s_off[w + 1] += s_off[w];
        s_base = (s_off[GB_WARPS] > 0) ? atomicAdd(&counters[0], s_off[GB_WARPS]) : 0;
    }
    __syncthreads();
    const int base = s_base + s_off[warp];
    const int a_id = (int)a_glob;
    if (valid && base + deg > d.edge_cap) {
        if (lane == 0) {
            atomicOr(&counters[1], 1);
            row_start[a_id] = 0;
            row_deg[a_id] = 0;
        }
    } else if (valid) {
        if (lane == 0) {
            row_start[a_id] = base;
            row_deg[a_id] = deg;
        }
        fill_row(edge_recv, edge_src, base, a_id, g * N, my_bits, n_words, hit_bits, lane);
    }
    __syncthreads();   // s_off / s_base / the per-warp scratch are reused by the next round
    }
}

// ------------------------------------------------------------------------------------
// canonical edge layout.  graph_build_kernel places each CTA's rows at a base taken from an atomic ticket, so the row
// order in edge_recv / edge_src depends on which CTA ran first.  Two passes move the rows into batch-agent order
// (row_start[a + 1] = row_start[a] + row_deg[a], row_start[0] = 0) with edge_recv as staging; every sum over the edge
// arrays (the train step's reductions) then sees the same layout on every run.  No CTA waits on another: each CTA
// adds up the degrees of all agents before its own chunk itself (A^2 / (2 CANON_T) loads in all, a few microseconds
// at the graph sizes a minibatch or a rollout chain holds).
// ------------------------------------------------------------------------------------
constexpr int CANON_T = 512;

// pass 1: row_start <- exclusive prefix of row_deg; the row at the ticket position in edge_src is copied to its
// canonical position in edge_recv.  Overflowed rows have row_deg = 0 and move nothing.
__global__ void __launch_bounds__(CANON_T)
edge_canon_stage_kernel(const int A, const int cap, int32_t* __restrict__ row_start, const int32_t* __restrict__ row_deg,
                        const int32_t* __restrict__ edge_src, int32_t* __restrict__ edge_recv) {
    __shared__ int s_warp[CANON_T / 32];
    __shared__ int s_scan[CANON_T];
    __shared__ int s_old[CANON_T];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int a0 = blockIdx.x * CANON_T;
    int pre = 0;
    for (int a = t; a < a0; a += CANON_T) pre += row_deg[a];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) pre += __shfl_xor_sync(0xffffffffu, pre, o);
    if (lane == 0) s_warp[warp] = pre;
    const int a = a0 + t;
    const int deg = a < A ? row_deg[a] : 0;
    s_old[t] = a < A ? row_start[a] : 0;
    s_scan[t] = deg;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < CANON_T / 32; ++w) base += s_warp[w];
    for (int o = 1; o < CANON_T; o <<= 1) {     // inclusive scan of the chunk's degrees
        const int v = t >= o ? s_scan[t - o] : 0;
        __syncthreads();
        s_scan[t] += v;
        __syncthreads();
    }
    if (a < A) row_start[a] = base + s_scan[t] - deg;
    for (int q = warp; q < CANON_T && a0 + q < A; q += CANON_T / 32) {
        const int d = row_deg[a0 + q], from = s_old[q], to = base + s_scan[q] - d;
        if (from < 0 || from + d > cap || to + d > cap) continue;
        for (int k = lane; k < d; k += 32) edge_recv[to + k] = edge_src[from + k];
    }
}

// pass 2: the staged rows go back to edge_src, and edge_recv gets the receiver ids
__global__ void __launch_bounds__(CANON_T)
edge_canon_final_kernel(const int A, const int cap, const int32_t* __restrict__ row_start,
                        const int32_t* __restrict__ row_deg, int32_t* __restrict__ edge_src,
                        int32_t* __restrict__ edge_recv) {
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; a < A; a += warps) {
        const int rs = row_start[a], d = row_deg[a];
        if (rs < 0 || rs + d > cap) continue;
        for (int k = lane; k < d; k += 32) {
            edge_src[rs + k] = edge_recv[rs + k];
            edge_recv[rs + k] = a;
        }
    }
}

// ------------------------------------------------------------------------------------
// env step: one CTA per graph (deterministic reward / cost reductions).
// ------------------------------------------------------------------------------------
template <int KIND>
__global__ void __launch_bounds__(256)
env_step_kernel(const gcbf_env_desc d, const float* __restrict__ agent, const float* __restrict__ goal,
                const float* __restrict__ obstacles, const float* __restrict__ pi,
                const int32_t* __restrict__ row_start, const int32_t* __restrict__ row_deg,
                const int32_t* __restrict__ edge_src, float* __restrict__ action, float* __restrict__ next_agent,
                float* __restrict__ reward, float* __restrict__ cost, const int mode) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU, PD = T::PD;
    constexpr int OBW = (PD == 2) ? 16 : 4;
    extern __shared__ float smem[];
    float* sobs = smem;  // [O, OBW]
    __shared__ float red_r[256];
    __shared__ float red_c[256];
    __shared__ float red_o[256];
    const int g = blockIdx.x, N = d.n_agents, O = d.n_obs;
    if (O > 0) {
        const float* ob = obstacles + (d.obs_per_graph ? (size_t)g * O * OBW : 0);
        for (int i = threadIdx.x; i < O * OBW; i += blockDim.x) sobs[i] = ob[i];
    }
    __syncthreads();
    float r_acc = 0.f, c_acc = 0.f, o_acc = 0.f;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const size_t a = (size_t)g * N + i;
        float x[SD], gl[SD], ur[NU], act[NU], xn[SD];
#pragma unroll
        for (int c = 0; c < SD; ++c) {
            x[c] = agent[a * SD + c];
            gl[c] = goal[a * SD + c];
        }
        u_ref_dev<KIND>(d, x, gl, ur);
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            // mode 0: a = 2 pi + u_ref (gcbf_plus.py:182-186); 1 / 3: given action; 2: a = u_ref (test.py --u-ref)
            act[c] = (mode == 0) ? (2.f * pi[a * NU + c] + ur[c]) : ((mode == 1 || mode == 3) ? action[a * NU + c] : ur[c]);
            if (mode == 0 || mode == 2) action[a * NU + c] = act[c];
        }
        const float sq = step_agent<KIND>(d, x, gl, act, ur, mode != 3, xn);   // mode 3: DubinsCar stop mask off
#pragma unroll
        for (int c = 0; c < SD; ++c) next_agent[a * SD + c] = xn[c];
        const float nr = sqrtf(sq);
        r_acc += nr * nr;  // (jnp.linalg.norm(...) ** 2)
        const bool col = collides_prev<PD, SD>(x, row_start[a], row_deg[a], edge_src, agent, d.two_r);
        c_acc += col ? 1.f : 0.f;
        o_acc += (O > 0 && inside_any<PD>(sobs, O, x, d.radius)) ? 1.f : 0.f;
    }
    red_r[threadIdx.x] = r_acc;
    red_c[threadIdx.x] = c_acc;
    red_o[threadIdx.x] = o_acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            red_r[threadIdx.x] += red_r[threadIdx.x + s];
            red_c[threadIdx.x] += red_c[threadIdx.x + s];
            red_o[threadIdx.x] += red_o[threadIdx.x + s];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        reward[g] = -(red_r[0] / (float)N);
        cost[g] = red_c[0] / (float)N + red_o[0] / (float)N;
    }
}

// ------------------------------------------------------------------------------------
// masks: warp per agent; brute force over the graph's agents + own hit nodes.
// ------------------------------------------------------------------------------------
template <int KIND>
__global__ void __launch_bounds__(GB_WARPS * 32)
masks_kernel(const gcbf_env_desc d, const float* __restrict__ agent, const float* __restrict__ goal,
             const float* __restrict__ hits, const float* __restrict__ obstacles, uint8_t* __restrict__ unsafe,
             uint8_t* __restrict__ collision, uint8_t* __restrict__ finish, uint8_t* __restrict__ safe) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, PD = T::PD;
    constexpr int OBW = (PD == 2) ? 16 : 4;
    extern __shared__ float smem[];
    const int N = d.n_agents, O = d.n_obs, R = d.n_hits;
    float* spos = smem;
    float* sobs = spos + N * PD;
    const int g = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < N; i += blockDim.x) {
        const float* a = agent + ((size_t)g * N + i) * SD;
#pragma unroll
        for (int c = 0; c < PD; ++c) spos[i * PD + c] = a[c];
    }
    if (O > 0) {
        const float* ob = obstacles + (d.obs_per_graph ? (size_t)g * O * OBW : 0);
        for (int i = tid; i < O * OBW; i += blockDim.x) sobs[i] = ob[i];
    }
    __syncthreads();
    const int i = blockIdx.x * GB_WARPS + warp;
    if (i >= N) return;
    const size_t a = (size_t)g * N + i;
    float x[SD];
#pragma unroll
    for (int c = 0; c < SD; ++c) x[c] = agent[a * SD + c];
    // heading for the "unsafe direction" test (double_integrator.py:393-415 / dubins_car.py:445-462)
    float hx = 0.f, hy = 0.f;
    if (KIND == GCBF_ENV_DOUBLE_INTEGRATOR) {
        const float sp = sqrtf(x[2] * x[2] + x[3] * x[3]);
        hx = x[2] / (sp + 0.0001f);
        hy = x[3] / (sp + 0.0001f);
    } else if (KIND == GCBF_ENV_DUBINS_CAR) {
        hx = cosf(x[2]);
        hy = sinf(x[2]);
    }
    bool any_unsafe_agent = false, any_col = false, all_safe = true, any_dir = false;
    for (int j0 = 0; j0 < N; j0 += 32) {
        const int j = j0 + lane;
        if (j < N) {
            // unsafe_mask uses pos[j] - pos[i]; collision/safe use pos[i] - pos[j]: same norm bitwise
            float dl[PD];
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < PD; ++c) {
                dl[c] = spos[j * PD + c] - x[c];
                acc = (c == 0) ? dl[c] * dl[c] : acc + dl[c] * dl[c];
            }
            const float nrm = sqrtf(acc);
            const float dist = nrm + ((j == i) ? d.two_r_p1 : 0.f);
            any_unsafe_agent = any_unsafe_agent || (dist < d.unsafe_agent);
            any_col = any_col || (dist < d.two_r);
            all_safe = all_safe && (dist > d.safe_agent);
            if (KIND == GCBF_ENV_DOUBLE_INTEGRATOR || KIND == GCBF_ENV_DUBINS_CAR) {
                const bool warn = dist < d.warn_agent;
                const float vx = dl[0] / (nrm + 0.0001f), vy = dl[1] / (nrm + 0.0001f);
                const float inner = vx * hx + vy * hy;
                const float th = atan2f(d.two_r, sqrtf(dist * dist - d.four_r_sq));
                any_dir = any_dir || (warn && (inner > cosf(th)));
            }
        }
    }
    if ((KIND == GCBF_ENV_DOUBLE_INTEGRATOR || KIND == GCBF_ENV_DUBINS_CAR) && hits != nullptr && lane < R) {
        const float* h = hits + (a * R + lane) * PD;
        const float dx = h[0] - x[0], dy = h[1] - x[1];
        const float dist = sqrtf(dx * dx + dy * dy);
        const bool warn = dist < d.warn_obs;
        const float vx = dx / (dist + 0.0001f), vy = dy / (dist + 0.0001f);
        const float inner = vx * hx + vy * hy;
        const float th = atan2f(d.radius, sqrtf(dist * dist - d.r_sq));
        any_dir = any_dir || (warn && (inner > cosf(th)));
    }
    any_unsafe_agent = __any_sync(0xffffffffu, any_unsafe_agent);
    any_col = __any_sync(0xffffffffu, any_col);
    all_safe = __all_sync(0xffffffffu, all_safe);
    any_dir = __any_sync(0xffffffffu, any_dir);
    if (lane == 0) {
        const bool in_unsafe = (O > 0) && inside_any<PD>(sobs, O, x, d.unsafe_obs);
        const bool in_col = (O > 0) && inside_any<PD>(sobs, O, x, d.radius);
        if (unsafe) unsafe[a] = (any_unsafe_agent || in_unsafe || any_dir) ? 1 : 0;
        if (collision) collision[a] = (any_col || in_col) ? 1 : 0;
        if (finish) {
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < PD; ++c) {
                const float dlt = x[c] - goal[a * SD + c];
                acc = (c == 0) ? dlt * dlt : acc + dlt * dlt;
            }
            finish[a] = (sqrtf(acc) < d.two_r) ? 1 : 0;
        }
        if (safe) {
            const bool in_safe = (O > 0) && inside_any<PD>(sobs, O, x, d.safe_obs);
            safe[a] = (all_safe && !in_safe) ? 1 : 0;
        }
    }
}

// action = (pi ? 2 pi : 0) + u_ref   (GCBFPlus.act, gcbf_plus.py:176-180; env.u_ref)
template <int KIND>
__global__ void act_kernel(const gcbf_env_desc d, const float* __restrict__ agent, const float* __restrict__ goal,
                           const float* __restrict__ pi, float* __restrict__ action) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= d.n_graphs * d.n_agents) return;
    float x[SD], gl[SD], ur[NU];
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        x[c] = agent[(size_t)a * SD + c];
        gl[c] = goal[(size_t)a * SD + c];
    }
    u_ref_dev<KIND>(d, x, gl, ur);
#pragma unroll
    for (int c = 0; c < NU; ++c) action[(size_t)a * NU + c] = pi ? (2.f * pi[(size_t)a * NU + c] + ur[c]) : ur[c];
}

// GCBFPlus.safe_mask (gcbf_plus.py:160-174): safe[t] = !any(unsafe[t .. t+H]) ; safe[0] = 1.
__global__ void safe_horizon_kernel(const uint8_t* __restrict__ unsafe, uint8_t* __restrict__ safe, int n_roll, int T,
                                    int N, int H) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_roll * N) return;
    const int b = idx / N, n = idx % N;
    const uint8_t* u = unsafe + (size_t)b * T * N + n;
    uint8_t* s = safe + (size_t)b * T * N + n;
    // sliding count of unsafe flags in the window [t, min(t+H, T-1)]
    int cnt = 0;
    for (int t = 0; t <= min(H, T - 1); ++t) cnt += u[(size_t)t * N];
    for (int t = 0; t < T; ++t) {
        s[(size_t)t * N] = (t == 0) ? 1 : (cnt == 0 ? 1 : 0);
        cnt -= u[(size_t)t * N];
        if (t + H + 1 < T) cnt += u[(size_t)(t + H + 1) * N];
    }
}

}  // namespace gcbf

using namespace gcbf;

static int32_t check_desc(const gcbf_env_desc* d) {
    GCBF_REQUIRE(d != nullptr, "desc is NULL");
    GCBF_REQUIRE(d->env_kind >= 0 && d->env_kind <= 3, "bad env_kind %d", d->env_kind);
    GCBF_REQUIRE(d->n_graphs > 0 && d->n_agents > 0, "n_graphs/n_agents must be positive");
    GCBF_REQUIRE(d->n_obs >= 0 && d->n_hits > 0 && d->n_hits <= 32, "n_obs >= 0 and 0 < n_hits <= 32 required");
    GCBF_REQUIRE((int64_t)d->n_graphs * d->n_agents < (int64_t)1 << 30, "too many agents");
    if (env_pd(d->env_kind) == 2)
        GCBF_REQUIRE(d->n_rays >= 1 && d->n_rays <= 32 && d->n_hits == d->n_rays,
                     "2-D envs need 1 <= n_rays <= 32 and n_hits == n_rays (got %d, %d)", d->n_rays, d->n_hits);
    else
        GCBF_REQUIRE(d->n_rays >= d->n_hits, "3-D env needs n_rays >= n_hits");
    return 0;
}

namespace gcbf {
int32_t graph_build_impl(const gcbf_env_desc* desc, const float* agent, const float* obstacles, const float* ray_table,
                         float* hits, int32_t* row_start, int32_t* row_deg, int32_t* edge_recv, int32_t* edge_src,
                         int32_t* counters, int32_t flags, const TailArgs& tail, float* reward, float* cost, void* stream);

}  // namespace gcbf

extern "C" __attribute__((visibility("default"))) int32_t gcbf_graph_build(const gcbf_env_desc* desc, const float* agent, const float* obstacles,
                                    const float* ray_table, float* hits, int32_t* row_start, int32_t* row_deg,
                                    int32_t* edge_recv, int32_t* edge_src, int32_t* counters, int32_t flags,
                                    void* stream) {
    TailArgs none;
    memset(&none, 0, sizeof(none));
    return graph_build_impl(desc, agent, obstacles, ray_table, hits, row_start, row_deg, edge_recv, edge_src, counters,
                            flags, none, nullptr, nullptr, stream);
}

int32_t gcbf::graph_build_impl(const gcbf_env_desc* desc, const float* agent, const float* obstacles,
                               const float* ray_table, float* hits, int32_t* row_start, int32_t* row_deg,
                               int32_t* edge_recv, int32_t* edge_src, int32_t* counters, int32_t flags,
                               const TailArgs& tail, float* reward, float* cost, void* stream) {
    if (int32_t rc = check_desc(desc)) return rc;
    GCBF_REQUIRE((agent || tail.z) && hits && row_start && row_deg && edge_recv && edge_src && counters,
                 "NULL pointer argument");
    GCBF_REQUIRE(!tail.z || (tail.bHO && tail.agent_prev && tail.goal && tail.row_start_prev && tail.row_deg_prev &&
                             tail.edge_src_prev && tail.action && tail.next_agent && reward && cost &&
                             tail.row_start_prev != row_start && tail.edge_src_prev != edge_src),
                 "fused policy tail: NULL argument or edge lists not double-buffered");
    GCBF_REQUIRE(desc->n_obs == 0 || obstacles, "obstacles is NULL but n_obs > 0");
    GCBF_REQUIRE(!(flags & 1) || ray_table, "ray_table is NULL");
    GCBF_REQUIRE(desc->edge_cap > 0, "edge_cap must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    const int pd = env_pd(desc->env_kind);
    const int obw = pd == 2 ? 16 : 4;
    const size_t smem = sizeof(float) * ((size_t)desc->n_agents * pd + (size_t)desc->n_obs * (pd == 2 ? 24 : 4) +
                                         (size_t)desc->n_rays * pd + (pd == 3 ? (size_t)GB_WARPS * desc->n_rays : 0) +
                                         (size_t)GB_WARPS * ((desc->n_agents + 31) / 32) + (pd == 3 ? (size_t)GB_WARPS * 96 : 0));
    GCBF_REQUIRE(smem <= 200 * 1024, "graph_build needs %zu B shared memory (> 200 KB): too many agents/obstacles", smem);
    if (!(flags & 4)) {   // bit 2: the caller's previous kernel already cleared counters[0]
        cudaError_t e = cudaMemsetAsync(counters, 0, sizeof(int32_t), st);
        if (e != cudaSuccess) { set_error("cudaMemsetAsync: %s", cudaGetErrorString(e)); return (int32_t)e; }
    }
    // one wave: a 1024-thread CTA owns an SM (register-bound), so each CTA takes `rounds` groups of GB_WARPS agents
    const int groups = (desc->n_agents + GB_WARPS - 1) / GB_WARPS;
    int rounds = 1;
    while (rounds < groups && (int64_t)((groups + rounds - 1) / rounds) * desc->n_graphs > sm_count()) ++rounds;
    dim3 grid((groups + rounds - 1) / rounds, desc->n_graphs);
    GCBF_DISPATCH_ENV(desc->env_kind, {
        auto kern = graph_build_kernel<KIND>;
        if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        kern<<<grid, GB_WARPS * 32, smem, st>>>(*desc, agent, obstacles, ray_table, hits, row_start, row_deg,
                                                edge_recv, edge_src, counters, flags & 1, tail, reward, cost, rounds);
    });
    count_launch();
    if (int32_t rc = check_launch("graph_build_kernel")) return rc;
    // the fused rollout step and callers that set flags bit 3 (the rollout engine) keep ticket order: rollout outputs do
    // not depend on the layout (every edge row is computed on its own and each receiver sums its own row in order)
    if (tail.z || (flags & 8)) return 0;
    const int A = desc->n_graphs * desc->n_agents, cap = desc->edge_cap;
    const int chunks = (A + CANON_T - 1) / CANON_T;
    edge_canon_stage_kernel<<<chunks, CANON_T, 0, st>>>(A, cap, row_start, row_deg, edge_src, edge_recv);
    count_launch();
    if (int32_t rc = check_launch("edge_canon_stage_kernel")) return rc;
    edge_canon_final_kernel<<<chunks, CANON_T, 0, st>>>(A, cap, row_start, row_deg, edge_src, edge_recv);
    count_launch();
    return check_launch("edge_canon_final_kernel");
}

// ------------------------------------------------------------------------------------
// reset: start / goal positions of every environment (env/utils.py:134-226 get_node_goal_rng), one warp per
// environment, with jax.random's threefry key chain (gcbfplus_b200/utils/jrandom.py describes the algorithm; the host
// restatement there is the cross-check, tests/test_gpu_reset.py).  Sequential rejection sampling per agent: the lanes
// share the key arithmetic and split the distance scan over the already placed agents.
// ------------------------------------------------------------------------------------
namespace gcbf {
struct TfKey { uint32_t a, b; };
__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__device__ __forceinline__ void threefry2x32(TfKey k, uint32_t c0, uint32_t c1, uint32_t& y0, uint32_t& y1) {
    const uint32_t ks[3] = {k.a, k.b, k.a ^ k.b ^ 0x1BD11BDAu};
    uint32_t x0 = c0 + ks[0], x1 = c1 + ks[1];
#pragma unroll
    for (int g = 0; g < 5; ++g) {
        const int* rot = (g & 1) ? (const int[4]){17, 29, 16, 24} : (const int[4]){13, 15, 26, 6};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            x0 += x1;
            x1 = rotl32(x1, rot[r]);
            x1 ^= x0;
        }
        x0 += ks[(g + 1) % 3];
        x1 += ks[(g + 2) % 3] + (uint32_t)(g + 1);
    }
    y0 = x0;
    y1 = x1;
}
// jr.split(key, 2) / jr.split(key, 3).  PART = false: jax's legacy layout, threefry over iota(2 num) split in halves;
// PART = true: jax_threefry_partitionable (default from JAX 0.5.0): child i = the output pair of threefry(key, (0, i)).
template <bool PART>
__device__ __forceinline__ void tf_split2(TfKey k, TfKey& k0, TfKey& k1) {
    if (PART) {
        TfKey c0, c1;
        threefry2x32(k, 0u, 0u, c0.a, c0.b);
        threefry2x32(k, 0u, 1u, c1.a, c1.b);
        k0 = c0;
        k1 = c1;
        return;
    }
    uint32_t a0, a1, b0, b1;
    threefry2x32(k, 0u, 2u, a0, a1);
    threefry2x32(k, 1u, 3u, b0, b1);
    k0 = {a0, b0};
    k1 = {a1, b1};
}
template <bool PART>
__device__ __forceinline__ void tf_split3(TfKey k, TfKey& k0, TfKey& k1, TfKey& k2) {
    if (PART) {
        TfKey c0, c1, c2;
        threefry2x32(k, 0u, 0u, c0.a, c0.b);
        threefry2x32(k, 0u, 1u, c1.a, c1.b);
        threefry2x32(k, 0u, 2u, c2.a, c2.b);
        k0 = c0;
        k1 = c1;
        k2 = c2;
        return;
    }
    uint32_t a0, a1, b0, b1, c0, c1;
    threefry2x32(k, 0u, 3u, a0, a1);
    threefry2x32(k, 1u, 4u, b0, b1);
    threefry2x32(k, 2u, 5u, c0, c1);
    k0 = {a0, b0};
    k1 = {c0, a1};
    k2 = {b1, c1};
}
__device__ __forceinline__ float tf_unit(uint32_t bits) { return __uint_as_float((bits >> 9) | 0x3F800000u) - 1.0f; }
// jr.uniform(key, (PD,), minval, maxval): max(minval, f * (maxval - minval) + minval), fp32 (this TU has no FMA)
template <int PD, bool PART>
__device__ __forceinline__ void tf_uniform(TfKey k, float lo, float hi, float* out) {
    uint32_t y0, y1;
    if (PART) {   // element i: bits = y0 ^ y1 of threefry(key, (0, i))
#pragma unroll
        for (int c = 0; c < PD; ++c) {
            threefry2x32(k, 0u, (uint32_t)c, y0, y1);
            out[c] = fmaxf(lo, tf_unit(y0 ^ y1) * (hi - lo) + lo);
        }
        return;
    }
    if (PD == 2) {
        threefry2x32(k, 0u, 1u, y0, y1);
        out[0] = fmaxf(lo, tf_unit(y0) * (hi - lo) + lo);
        out[1] = fmaxf(lo, tf_unit(y1) * (hi - lo) + lo);
    } else {   // iota(3) zero-padded to 4: halves [0, 1] and [2, 0]
        uint32_t z0, z1;
        threefry2x32(k, 0u, 2u, y0, y1);
        threefry2x32(k, 1u, 0u, z0, z1);
        out[0] = fmaxf(lo, tf_unit(y0) * (hi - lo) + lo);
        out[1] = fmaxf(lo, tf_unit(z0) * (hi - lo) + lo);
        out[PD - 1] = fmaxf(lo, tf_unit(y1) * (hi - lo) + lo);
    }
}

template <int PD, bool PART>
__global__ void __launch_bounds__(32)
reset_kernel(const int N, const int O, const int sd, const uint32_t* __restrict__ keys,
             const float* __restrict__ obstacles, const float L, const float min_dist, const float max_travel,
             float* __restrict__ agent, float* __restrict__ goal) {
    constexpr int OBW = (PD == 2) ? 16 : 4;
    extern __shared__ float rsm[];
    float* st = rsm;                 // [N, PD] placed start positions (zeros until placed: reference quirk)
    float* gl = st + (size_t)N * PD; // [N, PD]
    const int g = blockIdx.x, lane = threadIdx.x;
    const float* ob = obstacles + (size_t)g * O * OBW;
    const bool has_mt = max_travel >= 0.f;
    const int max_iter = 1024;
    for (int i = lane; i < N * PD; i += 32) { st[i] = 0.f; gl[i] = 0.f; }
    __syncwarp();
    // any slot within min_dist (sqrt of the fp32 sum, like jnp.linalg.norm)
    auto too_close = [&](const float* tab, const float* p) {
        bool hit = false;
        for (int j = lane; j < N; j += 32) {
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < PD; ++c) {
                const float dlt = tab[j * PD + c] - p[c];
                acc = (c == 0) ? dlt * dlt : acc + dlt * dlt;
            }
            hit = hit || (sqrtf(acc) <= min_dist);
        }
        return __any_sync(0xffffffffu, hit);
    };
    TfKey this_key = {keys[2 * g], keys[2 * g + 1]};
    int agent_id = 0;
    while (agent_id < N) {
        TfKey agent_key, goal_key;
        tf_split3<PART>(this_key, agent_key, goal_key, this_key);
        // ---- start position
        float cand[PD];
        tf_uniform<PD, PART>(agent_key, 0.f, L, cand);
        int it_a = 0;
        TfKey k = agent_key;
        while ((too_close(st, cand) || inside_any<PD>(ob, O, cand, min_dist)) && it_a < max_iter) {
            TfKey use;
            tf_split2<PART>(k, use, k);
            ++it_a;
            tf_uniform<PD, PART>(use, 0.f, L, cand);
        }
        __syncwarp();
        if (lane == 0) {
#pragma unroll
            for (int c = 0; c < PD; ++c) st[agent_id * PD + c] = cand[c];
        }
        // ---- goal position
        float gp[PD];
        if (!has_mt) {
            tf_uniform<PD, PART>(goal_key, 0.f, L, gp);
        } else {
            tf_uniform<PD, PART>(goal_key, 0.f, max_travel, gp);
#pragma unroll
            for (int c = 0; c < PD; ++c) gp[c] = gp[c] + cand[c];
        }
        int it_g = 0;
        k = goal_key;
        while (true) {
            bool bad = too_close(gl, gp) || inside_any<PD>(ob, O, gp, min_dist);
#pragma unroll
            for (int c = 0; c < PD; ++c) bad = bad || (gp[c] < 0.f) || (gp[c] > L);
            if (has_mt) {
                float acc = 0.f;
#pragma unroll
                for (int c = 0; c < PD; ++c) {
                    const float dlt = gp[c] - cand[c];
                    acc = (c == 0) ? dlt * dlt : acc + dlt * dlt;
                }
                bad = bad || (sqrtf(acc) > max_travel);
            }
            if (!bad || it_g >= max_iter) break;
            TfKey use;
            tf_split2<PART>(k, use, k);
            ++it_g;
            if (!has_mt) {
                tf_uniform<PD, PART>(use, 0.f, L, gp);
            } else {
                tf_uniform<PD, PART>(use, -max_travel, max_travel, gp);
#pragma unroll
                for (int c = 0; c < PD; ++c) gp[c] = gp[c] + cand[c];
            }
        }
        __syncwarp();
        if (lane == 0) {
#pragma unroll
            for (int c = 0; c < PD; ++c) gl[agent_id * PD + c] = gp[c];
        }
        ++agent_id;
        if (it_a >= max_iter || it_g >= max_iter) {   // "if no solution is found, start over" (same key chain)
            agent_id = 0;
            __syncwarp();
            for (int i = lane; i < N * PD; i += 32) { st[i] = 0.f; gl[i] = 0.f; }
        }
        __syncwarp();
    }
    for (int i = lane; i < N * PD; i += 32) {
        const int a = i / PD, c = i % PD;
        agent[((size_t)g * N + a) * sd + c] = st[i];
        goal[((size_t)g * N + a) * sd + c] = gl[i];
    }
}
}  // namespace gcbf

template <int PD, bool PART>
static void launch_reset(const gcbf_env_desc* desc, int sd, size_t smem, const uint32_t* keys, const float* obstacles,
                         float area_size, float min_dist, float max_travel, float* agent, float* goal, cudaStream_t st) {
    auto kern = gcbf::reset_kernel<PD, PART>;
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<desc->n_graphs, 32, smem, st>>>(desc->n_agents, desc->n_obs, sd, keys, obstacles, area_size, min_dist, max_travel,
                                           agent, goal);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_reset_positions_ex(
    const gcbf_env_desc* desc, const uint32_t* keys, const float* obstacles, float area_size, float min_dist,
    float max_travel, int32_t threefry_partitionable, float* agent, float* goal, void* stream) {
    GCBF_REQUIRE(desc && keys && agent && goal, "gcbf_reset_positions: NULL pointer argument");
    GCBF_REQUIRE(desc->env_kind >= 0 && desc->env_kind <= 3 && desc->n_graphs > 0 && desc->n_agents > 0,
                 "gcbf_reset_positions: bad descriptor");
    GCBF_REQUIRE(desc->n_obs == 0 || obstacles, "obstacles is NULL but n_obs > 0");
    GCBF_REQUIRE(desc->obs_per_graph == 1 || desc->n_obs == 0, "gcbf_reset_positions: one obstacle set per environment");
    const int pd = env_pd(desc->env_kind), sd = env_sd(desc->env_kind);
    const size_t smem = sizeof(float) * 2 * (size_t)desc->n_agents * pd;
    GCBF_REQUIRE(smem <= 200 * 1024, "gcbf_reset_positions: too many agents (%d)", desc->n_agents);
    cudaStream_t st = (cudaStream_t)stream;
    const bool part = threefry_partitionable != 0;
    if (pd == 2) {
        if (part) launch_reset<2, true>(desc, sd, smem, keys, obstacles, area_size, min_dist, max_travel, agent, goal, st);
        else launch_reset<2, false>(desc, sd, smem, keys, obstacles, area_size, min_dist, max_travel, agent, goal, st);
    } else {
        if (part) launch_reset<3, true>(desc, sd, smem, keys, obstacles, area_size, min_dist, max_travel, agent, goal, st);
        else launch_reset<3, false>(desc, sd, smem, keys, obstacles, area_size, min_dist, max_travel, agent, goal, st);
    }
    count_launch();
    return check_launch("reset_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_reset_positions(
    const gcbf_env_desc* desc, const uint32_t* keys, const float* obstacles, float area_size, float min_dist,
    float max_travel, float* agent, float* goal, void* stream) {
    return gcbf_reset_positions_ex(desc, keys, obstacles, area_size, min_dist, max_travel, 0, agent, goal, stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_env_step(const gcbf_env_desc* desc, const float* agent, const float* goal,
                                 const float* obstacles, const float* pi, const int32_t* row_start,
                                 const int32_t* row_deg, const int32_t* edge_src, float* action, float* next_agent,
                                 float* reward, float* cost, int32_t mode, void* stream) {
    if (int32_t rc = check_desc(desc)) return rc;
    GCBF_REQUIRE(agent && goal && row_start && row_deg && edge_src && action && next_agent && reward && cost,
                 "NULL pointer argument");
    GCBF_REQUIRE(desc->n_obs == 0 || obstacles, "obstacles is NULL but n_obs > 0");
    GCBF_REQUIRE(mode >= 0 && mode <= 3 && (mode != 0 || pi), "bad mode %d (mode 0 needs pi)", mode);
    const int obw = env_pd(desc->env_kind) == 2 ? 16 : 4;
    const size_t smem = sizeof(float) * (size_t)desc->n_obs * obw;
    GCBF_REQUIRE(smem <= 40 * 1024, "too many obstacles for env_step");
    cudaStream_t st = (cudaStream_t)stream;
    GCBF_DISPATCH_ENV(desc->env_kind, {
        env_step_kernel<KIND><<<desc->n_graphs, 256, smem, st>>>(*desc, agent, goal, obstacles, pi, row_start, row_deg,
                                                                 edge_src, action, next_agent, reward, cost, mode);
    });
    count_launch();
    return check_launch("env_step_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_act(const gcbf_env_desc* desc, const float* agent,
                                                                   const float* goal, const float* pi, float* action,
                                                                   void* stream) {
    if (int32_t rc = check_desc(desc)) return rc;
    GCBF_REQUIRE(agent && goal && action, "NULL pointer argument");
    const int A = desc->n_graphs * desc->n_agents;
    GCBF_DISPATCH_ENV(desc->env_kind, {
        act_kernel<KIND><<<(A + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*desc, agent, goal, pi, action);
    });
    count_launch();
    return check_launch("act_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_masks(const gcbf_env_desc* desc, const float* agent, const float* goal, const float* hits,
                              const float* obstacles, uint8_t* unsafe, uint8_t* collision, uint8_t* finish,
                              uint8_t* safe, void* stream) {
    if (int32_t rc = check_desc(desc)) return rc;
    GCBF_REQUIRE(agent && goal, "NULL pointer argument");
    GCBF_REQUIRE(desc->n_obs == 0 || obstacles, "obstacles is NULL but n_obs > 0");
    const int pd = env_pd(desc->env_kind);
    const int obw = pd == 2 ? 16 : 4;
    if (unsafe && (desc->env_kind == GCBF_ENV_DOUBLE_INTEGRATOR || desc->env_kind == GCBF_ENV_DUBINS_CAR))
        GCBF_REQUIRE(hits, "unsafe_mask of DoubleIntegrator/DubinsCar needs the hit nodes");
    const size_t smem = sizeof(float) * ((size_t)desc->n_agents * pd + (size_t)desc->n_obs * obw);
    GCBF_REQUIRE(smem <= 200 * 1024, "masks: too many agents/obstacles for shared memory");
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((desc->n_agents + GB_WARPS - 1) / GB_WARPS, desc->n_graphs);
    GCBF_DISPATCH_ENV(desc->env_kind, {
        auto kern = masks_kernel<KIND>;
        if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        kern<<<grid, GB_WARPS * 32, smem, st>>>(*desc, agent, goal, hits, obstacles, unsafe, collision, finish, safe);
    });
    count_launch();
    return check_launch("masks_kernel");
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_safe_horizon(const uint8_t* unsafe, uint8_t* safe, int32_t n_rollouts, int32_t T,
                                     int32_t n_agents, int32_t horizon, void* stream) {
    GCBF_REQUIRE(unsafe && safe && n_rollouts > 0 && T > 0 && n_agents > 0 && horizon >= 0, "bad argument");
    const int n = n_rollouts * n_agents;
    safe_horizon_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(unsafe, safe, n_rollouts, T, n_agents, horizon);
    count_launch();
    return check_launch("safe_horizon_kernel");
}
