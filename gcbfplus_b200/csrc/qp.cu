// qp.cu -- CBF-QP action labels u_qp (gcbfplus/algo/gcbf_plus.py:299-352 get_qp_action, :193-211 get_b_u_qp).
// Uses u_ref_dev of geometry_dev.cuh and, from the train step (internal.cuh), the data-only mode of gnn_backward_impl.
//
// Per graph with N agents, x = [u | r]:
//     min 1/2 |u|^2 - u_ref.u + 5 |r|^2 + 1000 sum r   s.t.  -Lg_h u - r <= Lf_h + 0.1 alpha h,  |u| <= u_lim,  r >= 0
// The safety filter (gcbf_qp_filter) solves the same QP with a given nominal action u_nom in place of u_ref.
// The reference hands the dense [N, N nu] problem to JaxProxQP.  Here:
//   * h(x) is a ONE-layer GNN, so row i of dh/dx is non-zero only at i and at i's agent neighbours: the
//     Jacobian is one data-only backward pass with upstream 1 (every receiver's gradient stays on its own
//     edges), kept per edge -- Lg_h is stored on the edge list (self block + one nu-block per agent edge);
//   * H is diagonal, so the dual is a box-projected concave problem in N multipliers whose inner minimisers
//     are closed-form: u(lam) = clip(u_ref + Lg^T lam), r(lam) = max(0, (lam - 1000) / 10).  One CTA per graph
//     runs an accelerated projected-gradient ascent with gradient restart on the row-scaled dual, everything
//     in shared memory; Lg^T lam uses the symmetric radius graph (edge j->i has the mirror edge i->j).
// The minimiser is unique (H > 0), so any exact method returns the reference's label up to solver tolerance.
#include "geometry_dev.cuh"
#include "gnn.cuh"
#include "internal.cuh"
#include "qp_lie.cuh"

namespace gcbf {

constexpr float QP_RELAX_PENALTY = 1e3f;   // gcbf_plus.py:302
constexpr float QP_RELAX_WEIGHT = 10.f;    // gcbf_plus.py:331
constexpr float QP_H_SCALE = 0.1f;         // gcbf_plus.py:334
constexpr int QP_MAX_AGENTS = 2048;

// Thread per agent i: row i of the QP.  JE[e][0..ED) = d h_i / d feat_e (feat = es_recv - es_sender), so
// d h_i / d es_i = +sum_e JE[e] and d h_i / d es_j = -JE[e] for the agent edge j -> i.
//   QB[i] = Lf_h_i + 0.1 alpha h_i     QS[i][c] = Lg_h[i, i, c]     QE[e][c] = Lg_h[i, j, c]
//   UR[i] = the nominal action: u_nom_i ([A, NU]) where u_nom is given, u_ref_i otherwise
//   REV[e] = index of the mirror edge i -> j in row j (or -1)        QSC[i] = row scale 1 / sqrt(|row|^2 + 0.1)
template <int KIND>
__global__ void __launch_bounds__(128)
qp_assemble_kernel(const gcbf_env_desc d, const float alpha, const float* __restrict__ agent,
                   const float* __restrict__ goal, const float* __restrict__ h, const float* __restrict__ JE,
                   const int32_t* __restrict__ row_start, const int32_t* __restrict__ row_deg,
                   const int32_t* __restrict__ edge_src, const float* __restrict__ u_nom, float* __restrict__ QB,
                   float* __restrict__ QS, float* __restrict__ QE, float* __restrict__ UR, float* __restrict__ QSC,
                   int32_t* __restrict__ REV) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU, ED = T::ED;
    const int A = d.n_graphs * d.n_agents;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A) return;
    const int rs = row_start[i];
    int rd = row_deg[i];
    if (rs < 0 || rs + rd > d.edge_cap) rd = 0;
    float xi[SD], gl[SD], ci[ED];
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        xi[c] = agent[(size_t)i * SD + c];
        gl[c] = goal[(size_t)i * SD + c];
    }
#pragma unroll
    for (int c = 0; c < ED; ++c) ci[c] = 0.f;
    float lf_sum = 0.f, sq = 0.f;
    for (int e = rs; e < rs + rd; ++e) {
        float je[ED];
#pragma unroll
        for (int c = 0; c < ED; ++c) {
            je[c] = JE[(size_t)e * 8 + c];
            ci[c] += je[c];
        }
        const int code = edge_src[e];
        int rev = -1;
        if (code >= 0 && code < A) {
            float xj[SD], nje[ED], lf, lg[NU];
#pragma unroll
            for (int c = 0; c < SD; ++c) xj[c] = agent[(size_t)code * SD + c];
#pragma unroll
            for (int c = 0; c < ED; ++c) nje[c] = -je[c];
            qp_lie_terms<KIND>(d, xj, nje, &lf, lg);
            lf_sum += lf;
#pragma unroll
            for (int c = 0; c < NU; ++c) {
                QE[(size_t)e * 4 + c] = lg[c];
                sq = fmaf(lg[c], lg[c], sq);
            }
            // mirror edge i -> code in row `code` (radius graph is symmetric)
            const int rs2 = row_start[code];
            int rd2 = row_deg[code];
            if (rs2 < 0 || rs2 + rd2 > d.edge_cap) rd2 = 0;
            for (int e2 = rs2; e2 < rs2 + rd2; ++e2)
                if (edge_src[e2] == i) { rev = e2; break; }
        } else {
#pragma unroll
            for (int c = 0; c < NU; ++c) QE[(size_t)e * 4 + c] = 0.f;
        }
        REV[e] = rev;
    }
    float lf, lg[NU], ur[NU];
    qp_lie_terms<KIND>(d, xi, ci, &lf, lg);
    lf_sum += lf;
    if (u_nom) {
#pragma unroll
        for (int c = 0; c < NU; ++c) ur[c] = u_nom[(size_t)i * NU + c];
    } else {
        u_ref_dev<KIND>(d, xi, gl, ur);
    }
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        QS[(size_t)i * 4 + c] = lg[c];
        UR[(size_t)i * 4 + c] = ur[c];
        sq = fmaf(lg[c], lg[c], sq);
    }
    QB[i] = lf_sum + alpha * QP_H_SCALE * h[i];
    QSC[i] = rsqrtf(sq + 1.f / QP_RELAX_WEIGHT);
}

__device__ __forceinline__ float qp_block_max(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float r = red[0];
    for (int w = 1; w < nw; ++w) r = fmaxf(r, red[w]);
    return r;
}
// (max of a, sum of b) over the block in one round trip; the sum runs in a fixed order (deterministic).
__device__ __forceinline__ void qp_block_max_sum(double& a, double& b, double* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a = fmax(a, __shfl_xor_sync(0xffffffffu, a, o));
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    __syncthreads();
    if (lane == 0) { red[warp] = a; red[32 + warp] = b; }
    __syncthreads();
    a = red[0];
    b = red[32];
    for (int w = 1; w < nw; ++w) { a = fmax(a, red[w]); b += red[32 + w]; }
}

// Neighbour access of the dual iteration.  SM: the graph's agent-agent blocks compacted into shared memory
// (CSR: off / nj / lg / lgt); otherwise straight from the edge list in global memory (graphs too dense to fit).
template <int NU, bool SM>
struct QpRows {
    const int* off; const int* nj; const float* lg; const float* lgt;           // shared CSR
    const int32_t* row_start; const int32_t* row_deg; const int32_t* edge_src;  // global edge list
    const float* QE; const int32_t* REV;
    int base, N, edge_cap;
    __device__ __forceinline__ void range(int i, int& beg, int& end) const {
        if (SM) { beg = off[i]; end = off[i + 1]; return; }
        beg = row_start[base + i];
        int rd = row_deg[base + i];
        if (beg < 0 || beg + rd > edge_cap) rd = 0;
        end = beg + rd;
    }
    // neighbour index of slot k (or -1: not an agent edge / no mirror) and pointers to Lg[i, j, :] and Lg[j, i, :]
    __device__ __forceinline__ int nbr(int k, const float*& row_blk, const float*& col_blk) const {
        if (SM) { row_blk = lg + (size_t)k * NU; col_blk = lgt + (size_t)k * NU; return nj[k]; }
        const int code = edge_src[k];
        if (code < base || code >= base + N) return -1;
        const int rv = REV[k];
        if (rv < 0) return -1;
        row_blk = QE + (size_t)k * 4;
        col_blk = QE + (size_t)rv * 4;
        return code - base;
    }
};

template <int NU, bool SM>
__device__ __forceinline__ void qp_primal_u(const QpRows<NU, SM>& R, const int N, const float u_lim, const double* lam,
                                            const float* ls, const float* ur, float* u) {
    // u = clip(u_ref + Lg^T lam): column block j collects Lg[i, j] lam_i over j's neighbours i (mirror edges)
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
        int beg, end;
        R.range(j, beg, end);
        const double lj = lam[j];
        double v[NU];
#pragma unroll
        for (int c = 0; c < NU; ++c) v[c] = fma((double)ls[j * NU + c], lj, (double)ur[j * NU + c]);
        for (int k = beg; k < end; ++k) {
            const float *rb, *cb;
            const int i = R.nbr(k, rb, cb);
            if (i < 0) continue;
            const double li = lam[i];
#pragma unroll
            for (int c = 0; c < NU; ++c) v[c] = fma((double)cb[c], li, v[c]);
        }
#pragma unroll
        for (int c = 0; c < NU; ++c) u[j * NU + c] = (float)fmin(fmax(v[c], -(double)u_lim), (double)u_lim);
    }
}

template <int NU, bool SM>
__device__ __forceinline__ int qp_iterate(const QpRows<NU, SM>& R, const int N, const float u_lim, const int max_iter,
                                          const double tol, const double lip, double* mu, double* y, double* lam,
                                          const float* sc, const float* bb, const float* ls, const float* ur, float* u,
                                          double* red) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const double step = 1.0 / lip;
    float t = 1.f;                                  // momentum schedule: fp32 is ample (only beta depends on it)
    int it;
    for (int i = tid; i < N; i += nt) lam[i] = (double)sc[i] * y[i];
    __syncthreads();
    for (it = 1; it <= max_iter; ++it) {            // 4 block barriers per iteration
        qp_primal_u<NU, SM>(R, N, u_lim, lam, ls, ur, u);
        __syncthreads();
        // dual gradient s (-Lg u - r - b), projected step, restart test
        double res = 0.0, dotp = 0.0;
        for (int i = tid; i < N; i += nt) {
            int beg, end;
            R.range(i, beg, end);
            double lgu = 0.0;
#pragma unroll
            for (int c = 0; c < NU; ++c) lgu = fma((double)ls[i * NU + c], (double)u[i * NU + c], lgu);
            for (int k = beg; k < end; ++k) {
                const float *rb, *cb;
                const int j = R.nbr(k, rb, cb);
                if (j < 0) continue;
#pragma unroll
                for (int c = 0; c < NU; ++c) lgu = fma((double)rb[c], (double)u[j * NU + c], lgu);
            }
            const double r = fmax(0.0, (lam[i] - (double)QP_RELAX_PENALTY) / (double)QP_RELAX_WEIGHT);
            const double grad = (double)sc[i] * (-lgu - r - (double)bb[i]);
            const double mn = fmax(0.0, fma(step, grad, y[i]));
            res = fmax(res, fabs(mn - y[i]));
            dotp = fma(grad, mn - mu[i], dotp);
            lam[i] = mn;   // lam carries mu_new until the momentum update below (u is already formed)
        }
        qp_block_max_sum(res, dotp, red);
        const bool restart = dotp < 0.0;
        const float t_new = restart ? 1.f : 0.5f * (1.f + sqrtf(1.f + 4.f * t * t));
        const double beta = restart ? 0.0 : (double)((t - 1.f) / t_new);
        for (int i = tid; i < N; i += nt) {
            const double mn = lam[i];
            const double yn = fma(beta, mn - mu[i], mn);
            y[i] = yn;
            mu[i] = mn;
            lam[i] = (double)sc[i] * yn;            // multipliers of the next iterate (read by every thread after the barrier)
        }
        t = t_new;
        __syncthreads();
        if (res * lip < tol) break;
    }
    for (int i = tid; i < N; i += nt) lam[i] = (double)sc[i] * mu[i];
    __syncthreads();
    qp_primal_u<NU, SM>(R, N, u_lim, lam, ls, ur, u);
    __syncthreads();
    return min(it, max_iter);
}

// One CTA per graph.  Dual variables mu = lam / s (row-scaled), FISTA with gradient restart, step 1 / L with the
// guaranteed bound L = |S Lg|_1 |S Lg|_inf + max(s^2) / 10 >= |S Lg|_2^2 + max(s^2) / 10.
// The multipliers are iterated in fp64: a relaxed row sits at lam ~ 1e3 while its fixed point is decided at the
// 1e-6 level (fp32 stalls ~600 ulp short: measured primal residual 3.7e-3); the matrix entries stay fp32.
// Shared memory: per agent mu, y, lam (fp64), s, b, u[NU], u_ref[NU], Lg_self[NU]; then the compacted agent-agent
// blocks of the graph (nbr_cap entries; graphs with more fall back to the global edge list).
// out_u [A, NU] clipped label; optional out_aux [A, 2] = (lam, r); optional out_iters [G].
template <int NU>
__global__ void __launch_bounds__(1024)
qp_solve_kernel(const int N, const int edge_cap, const int nbr_cap, const float u_lim, const int max_iter, const float tol,
                const float* __restrict__ QB, const float* __restrict__ QS, const float* __restrict__ QE,
                const float* __restrict__ UR, const float* __restrict__ QSC, const int32_t* __restrict__ REV,
                const int32_t* __restrict__ row_start, const int32_t* __restrict__ row_deg,
                const int32_t* __restrict__ edge_src, float* __restrict__ out_u, float* __restrict__ out_aux,
                int32_t* __restrict__ out_iters) {
    extern __shared__ __align__(16) unsigned char qsm_raw[];
    double* mu = reinterpret_cast<double*>(qsm_raw);
    double* y = mu + N;
    double* lam = y + N;
    double* red = lam + N;                      // 64 doubles
    float* sc = reinterpret_cast<float*>(red + 64);
    float* bb = sc + N;
    float* u = bb + N;
    float* ur = u + (size_t)N * NU;
    float* ls = ur + (size_t)N * NU;
    int* off = reinterpret_cast<int*>(ls + (size_t)N * NU);   // N + 1 (+ 1 flag)
    int* nj = off + N + 2;
    float* lg = reinterpret_cast<float*>(nj + nbr_cap);
    float* lgt = lg + (size_t)nbr_cap * NU;
    const int g = blockIdx.x;
    const int base = g * N;
    const int tid = threadIdx.x, nt = blockDim.x;

    // ---- load rows, count agent-agent blocks
    for (int i = tid; i < N; i += nt) {
        const int a = base + i;
        sc[i] = QSC[a];
        bb[i] = QB[a];
        mu[i] = 0.0;
        y[i] = 0.0;
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            ur[i * NU + c] = UR[(size_t)a * 4 + c];
            ls[i * NU + c] = QS[(size_t)a * 4 + c];
        }
        const int rs = row_start[a];
        int rd = row_deg[a];
        if (rs < 0 || rs + rd > edge_cap) rd = 0;
        int cnt = 0;
        for (int e = rs; e < rs + rd; ++e) {
            const int code = edge_src[e];
            cnt += (code >= base && code < base + N && REV[e] >= 0) ? 1 : 0;
        }
        off[i + 1] = cnt;
    }
    __syncthreads();
    if (tid == 0) {   // serial scan: N <= 2048, once per graph
        int acc = 0;
        off[0] = 0;
        for (int i = 0; i < N; ++i) { acc += off[i + 1]; off[i + 1] = acc; }
        off[N + 1] = (acc <= nbr_cap) ? 1 : 0;
    }
    __syncthreads();
    const bool in_smem = off[N + 1] != 0;
    // ---- norms for the step size (+ fill of the shared CSR)
    float rowmax = 0.f, colmax = 0.f, s2max = 0.f;
    for (int i = tid; i < N; i += nt) {
        const int a = base + i;
        const int rs = row_start[a];
        int rd = row_deg[a];
        if (rs < 0 || rs + rd > edge_cap) rd = 0;
        const float s = sc[i];
        float rsum = 0.f, csum[NU];
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            rsum += fabsf(ls[i * NU + c]);
            csum[c] = s * fabsf(ls[i * NU + c]);
        }
        int k = in_smem ? off[i] : 0;
        for (int e = rs; e < rs + rd; ++e) {
            const int code = edge_src[e];
            if (code < base || code >= base + N) continue;
            const int rv = REV[e];
            if (rv < 0) continue;
            const float sj = sc[code - base];
            if (in_smem) nj[k] = code - base;
#pragma unroll
            for (int c = 0; c < NU; ++c) {
                const float vr = QE[(size_t)e * 4 + c], vc = QE[(size_t)rv * 4 + c];
                rsum += fabsf(vr);
                csum[c] += sj * fabsf(vc);
                if (in_smem) { lg[(size_t)k * NU + c] = vr; lgt[(size_t)k * NU + c] = vc; }
            }
            ++k;
        }
        rowmax = fmaxf(rowmax, s * rsum);
#pragma unroll
        for (int c = 0; c < NU; ++c) colmax = fmaxf(colmax, csum[c]);
        s2max = fmaxf(s2max, s * s);
        // A row that no admissible u can satisfy (violation >= vmin > 0 over the whole box) is relaxed at the
        // optimum with r_i >= vmin, i.e. lam_i >= 1000 + 10 vmin: start there instead of climbing from 0
        // (the climb costs ~sqrt(1000 / (step * violation)) accelerated steps).
        const float vmin = -rsum * u_lim - bb[i];
        if (vmin > 0.f) {
            const double m0 = ((double)QP_RELAX_PENALTY + (double)QP_RELAX_WEIGHT * (double)vmin) / (double)s;
            mu[i] = m0;
            y[i] = m0;
        }
    }
    float* redf = reinterpret_cast<float*>(red);
    rowmax = qp_block_max(rowmax, redf);
    colmax = qp_block_max(colmax, redf);
    s2max = qp_block_max(s2max, redf);
    const double lip = (double)rowmax * (double)colmax + (double)s2max / (double)QP_RELAX_WEIGHT;
    __syncthreads();

    int it;
    if (in_smem) {
        QpRows<NU, true> R{off, nj, lg, lgt, row_start, row_deg, edge_src, QE, REV, base, N, edge_cap};
        it = qp_iterate<NU, true>(R, N, u_lim, max_iter, (double)tol, lip, mu, y, lam, sc, bb, ls, ur, u, red);
    } else {
        QpRows<NU, false> R{off, nj, lg, lgt, row_start, row_deg, edge_src, QE, REV, base, N, edge_cap};
        it = qp_iterate<NU, false>(R, N, u_lim, max_iter, (double)tol, lip, mu, y, lam, sc, bb, ls, ur, u, red);
    }
    for (int j = tid; j < N; j += nt) {
        const int a = base + j;
#pragma unroll
        for (int c = 0; c < NU; ++c) out_u[(size_t)a * NU + c] = u[j * NU + c];
        if (out_aux) {
            const double lj = lam[j];
            out_aux[(size_t)a * 2 + 0] = (float)lj;
            out_aux[(size_t)a * 2 + 1] = (float)fmax(0.0, (lj - (double)QP_RELAX_PENALTY) / (double)QP_RELAX_WEIGHT);
        }
    }
    if (out_iters && tid == 0) out_iters[g] = it | (in_smem ? 0 : (1 << 30));
}

// shared-memory bytes of qp_solve_kernel for N agents and nbr_cap compacted blocks
inline size_t qp_solve_smem(int N, int NU, int nbr_cap) {
    return (size_t)(3 * N + 64) * sizeof(double) + (size_t)(2 + 3 * NU) * N * sizeof(float) + (size_t)(N + 2) * sizeof(int) +
           (size_t)nbr_cap * (sizeof(int) + 2 * NU * sizeof(float));
}

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

}  // namespace gcbf

using namespace gcbf;

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
