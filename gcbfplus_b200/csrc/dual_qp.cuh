// dual_qp.cuh -- the method of every device QP: the GCBF+ labels and safety filter (qp.cu), both CBF-QP baselines
// (cbfqp.cu).  Each solves  min 1/2 |u|^2 - u_ref.u + 5 |r|^2 + 1000 sum r  s.t.  -Lg u - r <= b, |u| <= u_lim, r >= 0
// (H > 0: the minimiser is unique) on its dual.  With multipliers lam >= 0 the inner minimisers are closed-form,
// u(lam) = clip(u_ref + Lg^T lam) and r(lam) = max(0, (lam - 1000) / 10), so the dual is a box-projected concave
// problem.  It is row-scaled (mu = lam / s, s = 1 / sqrt(|row|^2 + 0.1)) and solved by projected-gradient ascent with
// FISTA momentum and gradient restart, step 1 / L, in fp64, until res L < tol (res = largest projected step).
// The callers own their rows, their u (precision and NaN rule) and the meaning of bit 30 of their iteration word.
#pragma once

#include "common.cuh"

namespace gcbf {

constexpr double QP_RELAX_PENALTY = 1e3;   // gcbf_plus.py:302, dec_share_cbf.py:103 relax_penalty
constexpr double QP_RELAX_WEIGHT = 10.0;   // H[-k:, -k:] = 10 (gcbf_plus.py:331)

__device__ __forceinline__ double dual_relax(const double lam) {
    return fmax(0.0, (lam - QP_RELAX_PENALTY) / QP_RELAX_WEIGHT);
}

// A row no u in the box satisfies (violation >= vmin > 0) is relaxed at the optimum with lam >= 1000 + 10 vmin: start
// there instead of climbing from 0 (~sqrt(1000 / (step * violation)) accelerated steps).
__device__ __forceinline__ double dual_warm_start(const double vmin, const double s) {
    return vmin > 0.0 ? (QP_RELAX_PENALTY + QP_RELAX_WEIGHT * vmin) / s : 0.0;
}

// L = norm2 + max(s^2) / 10, from a bound norm2 >= |S Lg|_2^2
__device__ __forceinline__ double dual_lipschitz(const double norm2, const double s2max) {
    return norm2 + s2max / QP_RELAX_WEIGHT;
}

// Row r of the projected dual-gradient step at y (lam = s[r] y[r], lgu = (Lg u(lam))_r): returns the new mu[r] and
// folds the row into res (max projected step) and dotp (the restart product grad . (mu_new - mu)).  The row is read
// from the caller's arrays (shared memory or registers) where each operand is used: loading the operands ahead costs
// the CTA solves spills.
template <class S>
__device__ __forceinline__ double dual_row_step(const int r, const double lam, const S* s, const S* b, const double* y,
                                                const double* mu, const double lgu, const double step, double& res,
                                                double& dotp) {
    const double rel = dual_relax(lam);
    const double grad = (double)s[r] * (-lgu - rel - (double)b[r]);
    const double mn = fmax(0.0, fma(step, grad, y[r]));
    res = fmax(res, fabs(mn - y[r]));
    dotp = fma(grad, mn - mu[r], dotp);
    return mn;
}

// FISTA schedule with gradient restart: advances t and returns the momentum beta.  T is the type t is kept in (the
// labels keep it in fp32, the baselines in fp64); beta is fp64 either way.
template <class T>
__device__ __forceinline__ double dual_momentum(const double dotp, T& t) {
    const bool restart = dotp < 0.0;
    const T t_new = restart ? T(1) : T(0.5) * (T(1) + sqrt(T(1) + T(4) * t * t));
    const double beta = restart ? 0.0 : (double)((t - T(1)) / t_new);
    t = t_new;
    return beta;
}

__device__ __forceinline__ double dual_extrapolate(const double beta, const double mn, const double mu) {
    return fma(beta, mn - mu, mn);   // y of the next iterate
}
__device__ __forceinline__ bool dual_converged(const double res, const double lip, const double tol) {
    return res * lip < tol;
}

// Block-wide max of v (red: 32 V of shared scratch).
template <class V>
__device__ __forceinline__ V block_max(V v, V* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    V r = red[0];
    for (int w = 1; w < nw; ++w) r = fmax(r, red[w]);
    return r;
}

// (max of a, sum of b) over the block in one round trip (red: 64 doubles); the sum runs in a fixed order
// (deterministic).
__device__ __forceinline__ void block_max_sum(double& a, double& b, double* red) {
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

// One M-row problem solved by a whole CTA, 4 block barriers per iteration.  Shared memory: mu, y (holding the warm
// start), lam (fp64), row scale sc and right-hand side bb (fp32), red (64 doubles).  The problem P supplies
//   void primal(const double* lam, bool last)  u(lam) into its u, strided over the CTA (last: the returned iterate)
//   double row_dot(int r) const                (Lg u)_r in fp64
// On return lam = s mu and u = u(lam).  Returns the iterations run (<= max_iter); conv: the stopping test passed.
template <class T, class P>
__device__ __forceinline__ int dual_cta_solve(const P& p, const int M, const int max_iter, const double tol,
                                              const double lip, double* mu, double* y, double* lam, const float* sc,
                                              const float* bb, double* red, bool& conv) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const double step = 1.0 / lip;
    T t = T(1);
    int it;
    conv = false;
    for (int r = tid; r < M; r += nt) lam[r] = (double)sc[r] * y[r];
    __syncthreads();
    for (it = 1; it <= max_iter; ++it) {
        p.primal(lam, false);
        __syncthreads();
        double res = 0.0, dotp = 0.0;
        for (int r = tid; r < M; r += nt) {
            const double lgu = p.row_dot(r);
            // lam carries mu_new until the momentum update below (u is already formed)
            lam[r] = dual_row_step(r, lam[r], sc, bb, y, mu, lgu, step, res, dotp);
        }
        block_max_sum(res, dotp, red);
        const double beta = dual_momentum(dotp, t);
        for (int r = tid; r < M; r += nt) {
            const double mn = lam[r];
            const double yn = dual_extrapolate(beta, mn, mu[r]);
            y[r] = yn;
            mu[r] = mn;
            lam[r] = (double)sc[r] * yn;            // multipliers of the next iterate (read by every thread after the barrier)
        }
        __syncthreads();
        if (dual_converged(res, lip, tol)) { conv = true; break; }
    }
    for (int r = tid; r < M; r += nt) lam[r] = (double)sc[r] * mu[r];
    __syncthreads();
    p.primal(lam, true);
    __syncthreads();
    return min(it, max_iter);
}

}  // namespace gcbf
