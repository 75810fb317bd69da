// cbfqp.cu -- the hand-written CBF-QP baseline controllers DecShareCBF and CentralizedCBF
// (gcbfplus/algo/dec_share_cbf.py:61-150, centralized_cbf.py:64-117) and their pairwise CBFs
// (gcbfplus/algo/utils.py:44-349, get_pwise_cbf_fn :413-439) for a batch of G graphs.
// Compiled with -fmad=false: the candidate distances (and so the k-nearest sets) are bit-exact against the CPU
// oracle, which evaluates them in the same operation order.
//
// Pairwise CBF of agent i (k = 3): the candidates are [the N agents | the R hit nodes of agent i] (hit state =
// [hit_pos, 0...]; every hit counts, "no-hit" rays included), d_c = |p_i - p_c|^2 with the self entry forced to 100,
// the k smallest in stable argsort order (ties -> lower index; NaN last).  With dp = p_i - p_c, dv = v_i - v_c:
//   SingleIntegrator  h = d - 4 (1.01 r)^2
//   DoubleIntegrator  h = 2 dp.dv + 10 (d - 4 r^2)
//   DubinsCar         h = 2 dp.dv + 5 (d - 4 r^2)     v = speed (cos th, sin th); a hit has zero velocity
//   LinearDrone       h = 2 dp.dv + 3 (d - 4 (1.01 r)^2)
// Its Jacobian wrt ALL agent states (the reference's jax.jacfwd) has at most two non-zero blocks: agent i and, when
// the pick is another agent j, agent j (dh/des_j = -dh/des_i); hit nodes are constants and the self pick has a
// constant distance and dp = dv = 0, so its gradient is exactly 0.  Lie terms along env.control_affine_dyn
// (qp_lie.cuh): Lf_h = dh/dx_i f(x_i) + dh/dx_j f(x_j), Lg_self = dh/dx_i g(x_i), Lg_other = dh/dx_j g(x_j).
//
// Both controllers solve the QP of dual_qp.cuh, which the reference hands to JaxProxQP with max_iter = 100, exactly
// on its dual with the momentum scalar in fp64.  A NaN u_ref component (u_ref is NaN exactly at the goal) takes part
// as 0 and comes out NaN, as it passes through the reference's solve.
//   DecShareCBF: one 3-row problem per agent (own Lg block only), b = resp (Lf_h + alpha h), resp = 1 for an
//     obstacle pick, 0.5 for an agent pick.  Thread per agent.
//   CentralizedCBF: one 3N-row problem per graph, row (i, k) touching u_i and, for an agent pick, u_j;
//     b = Lf_h + alpha h.  One CTA per graph, everything in shared memory.
#include <math.h>

#include "common.cuh"
#include "dual_qp.cuh"
#include "geometry_dev.cuh"
#include "qp_lie.cuh"

namespace gcbf {

constexpr int CBF_K = 3;
constexpr float CBF_SELF_DIST = 1e2f;      // utils.py: o_dist_sq.at[agent_idx].set(1e2)
constexpr int CBF_WARPS = 8;               // agents (warps) per CTA of the pairwise kernel
constexpr int CBF_CENTRAL_THREADS = 512;

// ------------------------------------------------------------------------------------------------------------------
// pairwise CBF + Lie terms: one warp per agent
// ------------------------------------------------------------------------------------------------------------------
struct CbfKey {
    float d;
    int idx;
};
// stable argsort order: numbers ascending, NaN after every number, ties by index
__device__ __forceinline__ bool cbf_less(const CbfKey& a, const CbfKey& b) {
    const bool na = isnan(a.d), nb = isnan(b.d);
    if (na != nb) return nb;
    if (!na && a.d != b.d) return a.d < b.d;
    return a.idx < b.idx;
}

struct CbfPairOut {
    int32_t* idx;        // [A, 3] candidate index: j < N agent j of the graph, N + k hit node k of this agent
    uint8_t* isobs;      // [A, 3] idx >= N
    float* h;            // [A, 3]
    float* lf;           // [A, 3]
    float* lg_self;      // [A, 3, NU]
    float* lg_other;     // [A, 3, NU] or NULL
};

template <int KIND>
__global__ void __launch_bounds__(CBF_WARPS * 32)
cbf_pairwise_kernel(const gcbf_env_desc d, const float* __restrict__ agent, const float* __restrict__ hits,
                    const float h_off, const CbfPairOut out) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, PD = T::PD, NU = T::NU;
    extern __shared__ float cbf_sx[];   // [N, SD] agent states of the graph
    const int N = d.n_agents, R = d.n_hits;
    const int g = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t = threadIdx.x; t < N * SD; t += blockDim.x) cbf_sx[t] = agent[(size_t)g * N * SD + t];
    __syncthreads();
    const int i = blockIdx.x * CBF_WARPS + warp;
    if (i >= N) return;
    const size_t a = (size_t)g * N + i;
    const float* xi = cbf_sx + i * SD;
    const float* hi = hits + a * R * PD;

    // ---- per-lane top-3 over the candidates lane, lane + 32, ...
    CbfKey top[CBF_K];
#pragma unroll
    for (int q = 0; q < CBF_K; ++q) top[q] = CbfKey{NAN, 0x7fffffff};
    for (int c = lane; c < N + R; c += 32) {
        const float* pc = (c < N) ? cbf_sx + c * SD : hi + (c - N) * PD;
        float dd = 0.f;
#pragma unroll
        for (int q = 0; q < PD; ++q) {
            const float dl = xi[q] - pc[q];
            dd = (q == 0) ? dl * dl : dd + dl * dl;
        }
        if (c == i) dd = CBF_SELF_DIST;
        CbfKey k{dd, c};
#pragma unroll
        for (int q = 0; q < CBF_K; ++q) {
            if (cbf_less(k, top[q])) { const CbfKey t = top[q]; top[q] = k; k = t; }
        }
    }
    // ---- warp merge: three rounds of an argmin over the lanes' heads, the winner pops its head
    CbfKey pick[CBF_K];
#pragma unroll
    for (int q = 0; q < CBF_K; ++q) {
        CbfKey m = top[0];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            CbfKey other;
            other.d = __shfl_xor_sync(0xffffffffu, m.d, o);
            other.idx = __shfl_xor_sync(0xffffffffu, m.idx, o);
            if (cbf_less(other, m)) m = other;
        }
        pick[q] = m;
        if (top[0].idx == m.idx) { top[0] = top[1]; top[1] = top[2]; top[2] = CbfKey{NAN, 0x7fffffff}; }
    }
    if (lane >= CBF_K) return;
    CbfKey kk = pick[0];
#pragma unroll
    for (int q = 1; q < CBF_K; ++q)
        if (lane == q) kk = pick[q];
    const int c = kk.idx;   // N + R >= 3 always (N >= 1, R >= 2)

    // ---- h and dh/des_i (es = edge state: position, velocity vector)
    constexpr bool VEL = (KIND != GCBF_ENV_SINGLE_INTEGRATOR);
    constexpr int VD = VEL ? PD : 0;
    float pc[PD], vi[PD], vc[PD];
    const bool is_agent = c < N, is_other = is_agent && c != i;
    const float* xc = is_agent ? cbf_sx + c * SD : nullptr;
#pragma unroll
    for (int q = 0; q < PD; ++q) pc[q] = is_agent ? xc[q] : hi[(c - N) * PD + q];
    if (KIND == GCBF_ENV_DUBINS_CAR) {
        vi[0] = xi[3] * cosf(xi[2]);
        vi[1] = xi[3] * sinf(xi[2]);
        vc[0] = is_agent ? xc[3] * cosf(xc[2]) : 0.f;
        vc[1] = is_agent ? xc[3] * sinf(xc[2]) : 0.f;
    } else {
#pragma unroll
        for (int q = 0; q < VD; ++q) {
            vi[q] = xi[PD + q];
            vc[q] = is_agent ? xc[PD + q] : 0.f;
        }
    }
    float dp[PD], dv[PD];
#pragma unroll
    for (int q = 0; q < PD; ++q) {
        dp[q] = xi[q] - pc[q];
        dv[q] = VEL ? vi[q] - vc[q] : 0.f;
    }
    const float h0 = kk.d - h_off;
    float h, de[2 * PD];
    if (!VEL) {
        h = h0;
#pragma unroll
        for (int q = 0; q < PD; ++q) de[q] = is_other || !is_agent ? 2.f * dp[q] : 0.f;
    } else {
        const float cgain = (KIND == GCBF_ENV_DOUBLE_INTEGRATOR) ? 10.f : ((KIND == GCBF_ENV_DUBINS_CAR) ? 5.f : 3.f);
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < PD; ++q) s = (q == 0) ? dp[q] * dv[q] : s + dp[q] * dv[q];
        h = 2.f * s + cgain * h0;
        const bool live = is_other || !is_agent;
#pragma unroll
        for (int q = 0; q < PD; ++q) {
            de[q] = live ? 2.f * dv[q] + cgain * (2.f * dp[q]) : 0.f;
            de[PD + q] = live ? 2.f * dp[q] : 0.f;
        }
    }
    float lf, lg[NU], lfj = 0.f, lgj[NU];
    qp_lie_terms<KIND>(d, xi, de, &lf, lg);
#pragma unroll
    for (int q = 0; q < NU; ++q) lgj[q] = 0.f;
    if (is_other) {
        float nde[2 * PD];
#pragma unroll
        for (int q = 0; q < 2 * PD; ++q) nde[q] = -de[q];
        qp_lie_terms<KIND>(d, xc, nde, &lfj, lgj);
    }
    const size_t o = a * CBF_K + lane;
    out.idx[o] = c;
    out.isobs[o] = c >= N ? 1 : 0;
    out.h[o] = h;
    out.lf[o] = lf + lfj;
#pragma unroll
    for (int q = 0; q < NU; ++q) {
        out.lg_self[o * NU + q] = lg[q];
        if (out.lg_other) out.lg_other[o * NU + q] = lgj[q];
    }
}

// ------------------------------------------------------------------------------------------------------------------
// DecShareCBF: one 3-multiplier dual per agent, thread per agent
// ------------------------------------------------------------------------------------------------------------------
// The steps of dual_cta_solve on a thread-local problem held in registers (no block reduction).
// iters[a] = iterations | (1 << 30) when the cap was hit before the stopping test passed
template <int KIND>
__global__ void __launch_bounds__(128)
cbf_dec_share_kernel(const gcbf_env_desc d, const float alpha, const int max_iter, const double tol,
                     const float* __restrict__ agent, const float* __restrict__ goal, const CbfPairOut pw,
                     float* __restrict__ out_u, float* __restrict__ out_r, int32_t* __restrict__ iters) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU, K = CBF_K;
    const int A = d.n_graphs * d.n_agents;
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A) return;
    float x[SD], gl[SD], urf[NU];
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        x[c] = agent[(size_t)a * SD + c];
        gl[c] = goal[(size_t)a * SD + c];
    }
    u_ref_dev<KIND>(d, x, gl, urf);
    double L[K][NU], b[K], s[K], ur[NU], mu[K], y[K];
    const double ul = (double)d.u_lim;
    double fro = 0.0, s2max = 0.0;
#pragma unroll
    for (int c = 0; c < NU; ++c) ur[c] = (double)urf[c];
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const size_t o = (size_t)a * K + k;
        const float resp = pw.isobs[o] ? 1.0f : 0.5f;
        b[k] = (double)(resp * (pw.lf[o] + alpha * pw.h[o]));
        double sq = 0.0, rs = 0.0;
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            L[k][c] = (double)pw.lg_self[o * NU + c];
            sq += L[k][c] * L[k][c];
            rs += fabs(L[k][c]);
        }
        s[k] = 1.0 / sqrt(sq + 1.0 / QP_RELAX_WEIGHT);
        fro += s[k] * s[k] * sq;
        s2max = fmax(s2max, s[k] * s[k]);
        mu[k] = dual_warm_start(-rs * ul - b[k], s[k]);
        y[k] = mu[k];
    }
    // step 1 / lip with |S Lg|_F^2 >= |S Lg|_2^2
    const double lip = dual_lipschitz(fro, s2max), step = 1.0 / lip;
    double t = 1.0;
    int it = 0;
    bool conv = false;
    double u[NU];
    for (it = 1; it <= max_iter; ++it) {
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            double v = ur[c];
#pragma unroll
            for (int k = 0; k < K; ++k) v = fma(L[k][c], s[k] * y[k], v);
            u[c] = isnan(v) ? 0.0 : fmin(fmax(v, -ul), ul);   // NaN u_ref: as 0 here, NaN in the result
        }
        double res = 0.0, dotp = 0.0, mn[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            double lgu = 0.0;
#pragma unroll
            for (int c = 0; c < NU; ++c) lgu = fma(L[k][c], u[c], lgu);
            mn[k] = dual_row_step(k, s[k] * y[k], s, b, y, mu, lgu, step, res, dotp);
        }
        const double beta = dual_momentum(dotp, t);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            y[k] = dual_extrapolate(beta, mn[k], mu[k]);
            mu[k] = mn[k];
        }
        if (dual_converged(res, lip, tol)) { conv = true; break; }
    }
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        double v = ur[c];
#pragma unroll
        for (int k = 0; k < K; ++k) v = fma(L[k][c], s[k] * mu[k], v);
        out_u[(size_t)a * NU + c] = isnan(v) ? NAN : (float)fmin(fmax(v, -ul), ul);
    }
    if (out_r) {
#pragma unroll
        for (int k = 0; k < K; ++k)
            out_r[(size_t)a * K + k] = (float)dual_relax(s[k] * mu[k]);
    }
    if (iters) iters[a] = min(it, max_iter) | (conv ? 0 : (1 << 30));
}

// ------------------------------------------------------------------------------------------------------------------
// CentralizedCBF: one 3N-row dual per graph, one CTA per graph
// ------------------------------------------------------------------------------------------------------------------
// The problem of dual_cta_solve: row (i, k) = self block ls of agent i plus, for an agent pick j, other block lo of
// agent j.  u is fp64, and a NaN u_ref component takes part as 0 until the returned iterate, which keeps the NaN.
template <int NU>
struct CentralRows {
    const float* ls; const float* lo; const float* ur;   // [M, NU], [M, NU], [N, NU]
    const int* oth; const int* toff; const int* trow;   // other agent of each row; transposed index
    double* u;                                          // [N, NU]
    int N;
    double ul;
    // u = clip(u_ref + Lg^T lam): own rows (self block) + the transposed list (other block)
    __device__ __forceinline__ void primal(const double* lam, const bool last) const {
        for (int j = threadIdx.x; j < N; j += blockDim.x) {
            double v[NU];
#pragma unroll
            for (int q = 0; q < NU; ++q) v[q] = (double)ur[j * NU + q];
            for (int k = 0; k < CBF_K; ++k) {
                const double l = lam[j * CBF_K + k];
#pragma unroll
                for (int q = 0; q < NU; ++q) v[q] = fma((double)ls[(j * CBF_K + k) * NU + q], l, v[q]);
            }
            for (int w = toff[j]; w < toff[j + 1]; ++w) {
                const int r = trow[w];
                const double l = lam[r];
#pragma unroll
                for (int q = 0; q < NU; ++q) v[q] = fma((double)lo[r * NU + q], l, v[q]);
            }
#pragma unroll
            for (int q = 0; q < NU; ++q)
                u[j * NU + q] = isnan(v[q]) ? (last ? NAN : 0.0) : fmin(fmax(v[q], -ul), ul);
        }
    }
    __device__ __forceinline__ double row_dot(const int r) const {
        const int i = r / CBF_K, j = oth[r];
        double lgu = 0.0;
#pragma unroll
        for (int q = 0; q < NU; ++q) lgu = fma((double)ls[r * NU + q], u[i * NU + q], lgu);
        if (j >= 0) {
#pragma unroll
            for (int q = 0; q < NU; ++q) lgu = fma((double)lo[r * NU + q], u[j * NU + q], lgu);
        }
        return lgu;
    }
};

// Shared memory, M = 3N rows: mu, y, lam [M] fp64 | u [N, NU] fp64 | red [64] fp64 | s, b [M] | lg_self, lg_other
// [M, NU] | u_ref [N, NU] | other [M] int (agent j of the row or -1) | toff [N + 1] int | trow [M] int (transposed
// index: rows whose OTHER block is agent j, grouped by j).  u stays fp64: an fp32 u puts ~1e-7 |Lg| of noise into the
// dual gradient, and the stopping test on it then stalls.
inline size_t cbf_central_smem(int N, int NU) {
    const size_t M = 3 * (size_t)N;
    return (3 * M + (size_t)N * NU + 64) * sizeof(double) + (2 * M + 2 * M * NU + (size_t)N * NU) * sizeof(float) +
           (M + (N + 1) + M) * sizeof(int);
}

template <int KIND>
__global__ void __launch_bounds__(CBF_CENTRAL_THREADS)
cbf_central_kernel(const gcbf_env_desc d, const float alpha, const int max_iter, const double tol,
                   const float* __restrict__ agent, const float* __restrict__ goal, const CbfPairOut pw,
                   float* __restrict__ out_u, float* __restrict__ out_r, int32_t* __restrict__ iters) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU, K = CBF_K;
    extern __shared__ __align__(16) unsigned char cbf_csm[];
    const int N = d.n_agents, M = K * N;
    double* mu = reinterpret_cast<double*>(cbf_csm);
    double* y = mu + M;
    double* lam = y + M;
    double* u = lam + M;
    double* red = u + (size_t)N * NU;
    float* sc = reinterpret_cast<float*>(red + 64);
    float* bb = sc + M;
    float* ls = bb + M;
    float* lo = ls + (size_t)M * NU;
    float* ur = lo + (size_t)M * NU;
    int* oth = reinterpret_cast<int*>(ur + (size_t)N * NU);
    int* toff = oth + M;
    int* trow = toff + N + 1;
    const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const size_t base = (size_t)g * N;
    const double ul = (double)d.u_lim;

    // ---- load the rows; count every agent's references as the OTHER block of a row
    for (int j = tid; j <= N; j += nt) toff[j] = 0;
    __syncthreads();
    for (int r = tid; r < M; r += nt) {
        const size_t o = base * K + r;
        const int i = r / K, c = pw.idx[o];
        const int j = (c < N && c != i) ? c : -1;
        oth[r] = j;
        bb[r] = pw.lf[o] + alpha * pw.h[o];
        float sq = 0.f;
#pragma unroll
        for (int q = 0; q < NU; ++q) {
            ls[r * NU + q] = pw.lg_self[o * NU + q];
            lo[r * NU + q] = pw.lg_other[o * NU + q];
            sq += ls[r * NU + q] * ls[r * NU + q] + lo[r * NU + q] * lo[r * NU + q];
        }
        sc[r] = rsqrtf(sq + (float)(1.0 / QP_RELAX_WEIGHT));
        if (j >= 0) atomicAdd(&toff[j + 1], 1);
    }
    for (int j = tid; j < N; j += nt) {
        float x[SD], gl[SD], uf[NU];
#pragma unroll
        for (int c = 0; c < SD; ++c) {
            x[c] = agent[(base + j) * SD + c];
            gl[c] = goal[(base + j) * SD + c];
        }
        u_ref_dev<KIND>(d, x, gl, uf);
#pragma unroll
        for (int c = 0; c < NU; ++c) ur[j * NU + c] = uf[c];
    }
    __syncthreads();
    if (tid == 0) {   // serial scan, once per graph
        for (int j = 0; j < N; ++j) toff[j + 1] += toff[j];
    }
    __syncthreads();
    // transposed index: the thread owning agent j lists the rows whose other block is j, in row order (deterministic)
    for (int j = tid; j < N; j += nt) {
        int w = toff[j];
        for (int r = 0; r < M; ++r)
            if (oth[r] == j) trow[w++] = r;
    }
    __syncthreads();

    // ---- step bound L = |S Lg|_1 |S Lg|_inf + max(s^2) / 10 and the relaxed-row warm start
    double rowmax = 0.0, colmax = 0.0, s2max = 0.0;
    for (int r = tid; r < M; r += nt) {
        double rs = 0.0;
#pragma unroll
        for (int q = 0; q < NU; ++q) rs += fabs((double)ls[r * NU + q]) + fabs((double)lo[r * NU + q]);
        rowmax = fmax(rowmax, (double)sc[r] * rs);
        s2max = fmax(s2max, (double)sc[r] * (double)sc[r]);
        const double m0 = dual_warm_start(-rs * ul - (double)bb[r], (double)sc[r]);
        mu[r] = m0;
        y[r] = m0;
    }
    for (int j = tid; j < N; j += nt) {
#pragma unroll
        for (int q = 0; q < NU; ++q) {
            double cs = 0.0;
            for (int k = 0; k < K; ++k) cs += (double)sc[j * K + k] * fabs((double)ls[(j * K + k) * NU + q]);
            for (int w = toff[j]; w < toff[j + 1]; ++w) cs += (double)sc[trow[w]] * fabs((double)lo[trow[w] * NU + q]);
            colmax = fmax(colmax, cs);
        }
    }
    rowmax = block_max(rowmax, red);
    colmax = block_max(colmax, red);
    s2max = block_max(s2max, red);
    const double lip = dual_lipschitz(rowmax * colmax, s2max);
    __syncthreads();

    CentralRows<NU> P{ls, lo, ur, oth, toff, trow, u, N, ul};
    bool conv;
    const int it = dual_cta_solve<double>(P, M, max_iter, tol, lip, mu, y, lam, sc, bb, red, conv);
    for (int j = tid; j < N; j += nt) {
#pragma unroll
        for (int q = 0; q < NU; ++q) out_u[(base + j) * NU + q] = (float)u[j * NU + q];
    }
    if (out_r) {
        for (int r = tid; r < M; r += nt)
            out_r[base * K + r] = (float)dual_relax(lam[r]);
    }
    if (iters && tid == 0) iters[g] = it | (conv ? 0 : (1 << 30));
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
// h0 offset of the env: 4 r^2 (DoubleIntegrator, DubinsCar) is the descriptor's four_r_sq; 4 (1.01 r)^2
// (SingleIntegrator, LinearDrone) is 1.0201 four_r_sq rounded once, which gives the fp32 the reference's weak typing
// makes of the python float for the shipped radius (tests/test_cbfqp_oracle.py checks it).
static float cbf_h_offset(const gcbf_env_desc& d) {
    if (d.env_kind == GCBF_ENV_SINGLE_INTEGRATOR || d.env_kind == GCBF_ENV_LINEAR_DRONE)
        return (float)(1.0201 * (double)d.four_r_sq);
    return d.four_r_sq;
}

static int32_t cbf_check(const gcbf_env_desc* desc, const float* agent, const float* hits) {
    GCBF_REQUIRE(desc, "NULL descriptor");
    GCBF_REQUIRE(desc->n_graphs > 0 && desc->n_agents > 0 && desc->n_hits >= 0, "bad batch sizes");
    GCBF_REQUIRE(desc->n_agents + desc->n_hits >= CBF_K, "fewer than 3 candidates (n_agents + n_hits < 3)");
    GCBF_REQUIRE(desc->env_kind >= 0 && desc->env_kind <= 3, "unknown env_kind %d", desc->env_kind);
    GCBF_REQUIRE(agent && (hits || desc->n_hits == 0), "NULL pointer argument");
    const size_t smem = sizeof(float) * (size_t)desc->n_agents * env_sd(desc->env_kind);
    GCBF_REQUIRE(smem <= 200 * 1024, "cbf pairwise: %d agents do not fit in shared memory", desc->n_agents);
    return 0;
}

static int32_t cbf_pairwise_launch(const gcbf_env_desc& d, const float* agent, const float* hits, const CbfPairOut& out,
                                   cudaStream_t st) {
    const size_t smem = sizeof(float) * (size_t)d.n_agents * env_sd(d.env_kind);
    const dim3 grid((d.n_agents + CBF_WARPS - 1) / CBF_WARPS, d.n_graphs);
    GCBF_DISPATCH_ENV(d.env_kind, {
        if (smem > 48 * 1024)
            cudaFuncSetAttribute(cbf_pairwise_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        cbf_pairwise_kernel<KIND><<<grid, CBF_WARPS * 32, smem, st>>>(d, agent, hits, cbf_h_offset(d), out);
    });
    count_launch();
    return check_launch("cbf_pairwise_kernel");
}

// workspace layout (floats): idx [3A] int32 | h [3A] | lf [3A] | lg_self [3A, NU] | lg_other [3A, NU] | isobs [3A] u8
static CbfPairOut cbf_ws_layout(const gcbf_env_desc& d, float* ws) {
    const size_t A3 = (size_t)d.n_graphs * d.n_agents * CBF_K;
    const int NU = env_nu(d.env_kind);
    CbfPairOut o;
    o.idx = reinterpret_cast<int32_t*>(ws);
    o.h = ws + A3;
    o.lf = o.h + A3;
    o.lg_self = o.lf + A3;
    o.lg_other = o.lg_self + A3 * NU;
    o.isobs = reinterpret_cast<uint8_t*>(o.lg_other + A3 * NU);
    return o;
}
static int64_t cbf_ws_floats(const gcbf_env_desc& d) {
    const int64_t A3 = (int64_t)d.n_graphs * d.n_agents * CBF_K;
    return A3 * (3 + 2 * env_nu(d.env_kind)) + (A3 + 3) / 4;
}

enum CbfAlgo { CBF_DEC_SHARE = 0, CBF_CENTRAL = 1 };

static int32_t cbf_qp(int which, const gcbf_env_desc* desc, float alpha, int32_t max_iter, float tol, const float* agent,
                      const float* goal, const float* hits, float* u, float* r, int32_t* iters, float* workspace,
                      int64_t workspace_floats, void* stream) {
    if (int32_t rc = cbf_check(desc, agent, hits)) return rc;
    GCBF_REQUIRE(goal && u && workspace, "NULL pointer argument");
    GCBF_REQUIRE(max_iter >= 1, "max_iter must be >= 1");
    GCBF_REQUIRE(tol >= 0.f, "tol must be >= 0");
    GCBF_REQUIRE(workspace_floats >= cbf_ws_floats(*desc), "workspace too small: %lld < %lld floats",
                 (long long)workspace_floats, (long long)cbf_ws_floats(*desc));
    const gcbf_env_desc d = *desc;
    cudaStream_t st = (cudaStream_t)stream;
    const CbfPairOut pw = cbf_ws_layout(d, workspace);
    size_t csm = 0;
    if (which == CBF_CENTRAL) {
        csm = cbf_central_smem(d.n_agents, env_nu(d.env_kind));
        GCBF_REQUIRE(d.n_agents <= GCBF_CBFQP_CENTRAL_MAX_AGENTS && csm <= 227 * 1024,
                     "centralized_cbf: %d agents per graph exceed the shared-memory limit (%d; LinearDrone 999)",
                     d.n_agents, GCBF_CBFQP_CENTRAL_MAX_AGENTS);
    }
    if (int32_t rc = cbf_pairwise_launch(d, agent, hits, pw, st)) return rc;
    const int A = d.n_graphs * d.n_agents;
    if (which == CBF_DEC_SHARE) {
        GCBF_DISPATCH_ENV(d.env_kind, {
            cbf_dec_share_kernel<KIND><<<(A + 127) / 128, 128, 0, st>>>(d, alpha, max_iter, (double)tol, agent, goal, pw,
                                                                        u, r, iters);
        });
        count_launch();
        return check_launch("cbf_dec_share_kernel");
    }
    GCBF_DISPATCH_ENV(d.env_kind, {
        cudaFuncSetAttribute(cbf_central_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)csm);
        cbf_central_kernel<KIND><<<d.n_graphs, CBF_CENTRAL_THREADS, csm, st>>>(d, alpha, max_iter, (double)tol, agent, goal,
                                                                               pw, u, r, iters);
    });
    count_launch();
    return check_launch("cbf_central_kernel");
}

}  // namespace gcbf

using namespace gcbf;

extern "C" __attribute__((visibility("default"))) int32_t gcbf_cbf_pairwise(
    const gcbf_env_desc* desc, const float* agent, const float* hits, int32_t* k_idx, uint8_t* k_isobs, float* k_h,
    float* k_lf_h, float* k_lg_self, float* k_lg_other, void* stream) {
    if (int32_t rc = cbf_check(desc, agent, hits)) return rc;
    GCBF_REQUIRE(k_idx && k_isobs && k_h && k_lf_h && k_lg_self, "NULL pointer argument");
    CbfPairOut o{k_idx, k_isobs, k_h, k_lf_h, k_lg_self, k_lg_other};
    return cbf_pairwise_launch(*desc, agent, hits, o, (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int64_t gcbf_cbfqp_workspace_floats(const gcbf_env_desc* desc) {
    if (!desc || desc->n_graphs <= 0 || desc->n_agents <= 0 || desc->env_kind < 0 || desc->env_kind > 3) return -1;
    return cbf_ws_floats(*desc);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_cbfqp_dec_share(
    const gcbf_env_desc* desc, float alpha, int32_t max_iter, float tol, const float* agent, const float* goal,
    const float* hits, float* u, float* r, int32_t* iters, float* workspace, int64_t workspace_floats, void* stream) {
    return cbf_qp(CBF_DEC_SHARE, desc, alpha, max_iter, tol, agent, goal, hits, u, r, iters, workspace, workspace_floats,
                  stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_cbfqp_centralized(
    const gcbf_env_desc* desc, float alpha, int32_t max_iter, float tol, const float* agent, const float* goal,
    const float* hits, float* u, float* r, int32_t* iters, float* workspace, int64_t workspace_floats, void* stream) {
    return cbf_qp(CBF_CENTRAL, desc, alpha, max_iter, tol, agent, goal, hits, u, r, iters, workspace, workspace_floats,
                  stream);
}
