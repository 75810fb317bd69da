// geometry_dev.cuh -- device functions shared by geometry.cu, rollout_persist.cu, train.cu, qp.cu, refine.cu and
// falsify.cu: obstacle primitives (Rectangle / Sphere inside + ray cast), the stable 32-key warp sort of the LiDAR
// returns, u_ref, the Euler step, their state Jacobians (the CBF-condition gradient of falsify.cu), the chain of the
// train step's and the refinement's backward through the Euler step (dyn_chain_dev), the policy tail and reward / cost
// terms of an env step, and the per-warp pieces of the graph build (2-D LiDAR, active hits, neighbour scan, edge-row
// fill).  The 5-launch rollout step and the persistent rollout kernel run these
// same functions, which is what keeps the two paths bit-identical.
// Every including unit is compiled with -fmad=false: every arithmetic step keeps the reference's
// one-rounding-per-op semantics (bit-exact index sets / hit ordering / masks against the CPU oracle).
//
// Replaces (reference paths): gcbfplus/env/obstacle.py:53-96 (Rectangle), :234-270 (Sphere), env/utils.py:82-131,
// env/double_integrator.py:128-143 (Euler), :332-338 (u_ref) and their SingleIntegrator / DubinsCar / LinearDrone twins.
#pragma once
#include <math.h>

#include "common.cuh"

namespace gcbf {

static constexpr int GB_WARPS = 32;  // agents (warps) per CTA in graph_build
#define NO_HIT 1e6f

// ------------------------------------------------------------------------------------
// obstacle primitives
// ------------------------------------------------------------------------------------
// Rectangle.inside (obstacle.py:53-63); ob = 16-float packed rectangle.
__device__ __forceinline__ bool rect_inside(const float* ob, float px, float py, float r) {
    float rel_x = px - ob[0];
    float rel_y = py - ob[1];
    float rel_xx = fabsf(rel_x * ob[4] + rel_y * ob[5]) - ob[2];
    float rel_yy = fabsf(rel_x * ob[5] - rel_y * ob[4]) - ob[3];
    bool is_in_down = (rel_xx < r) && (rel_yy < 0.f);
    bool is_in_up = (rel_xx < 0.f) && (rel_yy < r);
    bool is_out_corner = (rel_xx > 0.f) && (rel_yy > 0.f);
    bool is_in_circle = sqrtf(rel_xx * rel_xx + rel_yy * rel_yy) < r;
    return (is_in_down || is_in_up) || (is_out_corner && is_in_circle);
}

__device__ __forceinline__ float nanmin(float a, float b) {  // jnp.min: NaN-propagating
    return (isnan(a) || isnan(b)) ? NAN : fminf(a, b);
}

// Rectangle.raytracing (obstacle.py:65-96): min over the 4 edges.
__device__ __forceinline__ float rect_raytrace(const float* ob, float x1, float y1, float x2, float y2) {
    float best = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int kp = (k + 3) & 3;  // points[[-1,0,1,2]]
        float x3 = ob[6 + 2 * k], y3 = ob[7 + 2 * k];
        float x4 = ob[6 + 2 * kp], y4 = ob[7 + 2 * kp];
        float det = (x1 - x2) * (y4 - y3) - (y1 - y2) * (x4 - x3);
        float sgn = (det > 0.f) ? 1.f : ((det < 0.f) ? -1.f : det);  // jnp.sign (0 -> 0, NaN -> NaN)
        det = sgn * fminf(fmaxf(fabsf(det), 1e-7f), 1e7f);
        float alpha = ((y4 - y3) * (x1 - x3) - (x4 - x3) * (y1 - y3)) / det;
        float beta = (-(y1 - y2) * (x1 - x3) + (x1 - x2) * (y1 - y3)) / det;
        float v = ((alpha <= 1.f && alpha >= 0.f) && (beta <= 1.f && beta >= 0.f)) ? 1.f : 0.f;
        alpha = v * alpha + (1.f - v) * NO_HIT;
        best = (k == 0) ? alpha : nanmin(best, alpha);
    }
    return best;
}

// Sphere.inside / raytracing (obstacle.py:234-270); ob = cx,cy,cz,r.
__device__ __forceinline__ bool sphere_inside(const float* ob, float px, float py, float pz, float r) {
    float dx = px - ob[0], dy = py - ob[1], dz = pz - ob[2];
    return sqrtf(dx * dx + dy * dy + dz * dz) <= ob[3] + r;
}
__device__ __forceinline__ float sphere_raytrace(const float* ob, float x1, float y1, float z1, float x2,
                                                 float y2, float z2) {
    float dx = x2 - x1, dy = y2 - y1, dz = z2 - z1;
    float rmax = sqrtf(dx * dx + dy * dy + dz * dz);
    float A = rmax * rmax;
    float ex = x1 - ob[0], ey = y1 - ob[1], ez = z1 - ob[2];
    float B = 2.f * (dx * ex + dy * ey + dz * ez);
    float C = ex * ex + ey * ey + ez * ez - ob[3] * ob[3];
    float delta = B * B - 4.f * A * C;
    // the line misses the sphere (the common case: 4 small spheres, 514 rays): valid1 = 0 makes both roots
    // (-B -+ 0) / (2A) * 0 + 1 = 1 exactly (finite operands), alphas = 1 and the result 0 * 1 + 1 * 1e6 = 1e6 -- returned
    // directly, skipping the square root and the two divisions (identical bits; NaN inputs fail `delta < 0` and take the
    // full path)
    if (delta < 0.f && A > 1e-20f && fabsf(B) < 1e18f) return NO_HIT;
    float valid1 = (delta >= 0.f) ? 1.f : 0.f;
    float sq = sqrtf(delta * valid1);
    float alpha1 = (-B - sq) / (2.f * A) * valid1 + (1.f - valid1);
    float alpha2 = (-B + sq) / (2.f * A) * valid1 + (1.f - valid1);
    float a1 = ((alpha1 >= 0.f) ? 1.f : 0.f) * alpha1 + ((alpha1 < 0.f) ? 1.f : 0.f) * 1.f;
    float a2 = ((alpha2 >= 0.f) ? 1.f : 0.f) * alpha2 + ((alpha2 < 0.f) ? 1.f : 0.f) * 1.f;
    float alphas = fminf(a1, a2);
    alphas = fminf(fmaxf(alphas, 0.f), 1.f);
    return valid1 * alphas + (1.f - valid1) * NO_HIT;
}

// inside_obstacles (env/utils.py:82-107) for one point against the graph's obstacle set; obstacle o at sobs + OSTRIDE o
// (packed rows by default; OBS2D for the shared-memory rows of the graph build).
template <int PD, int OSTRIDE = (PD == 2 ? 16 : 4)>
__device__ __forceinline__ bool inside_any(const float* sobs, int O, const float* p, float r) {
    bool in = false;
    if (PD == 2) {
        for (int o = 0; o < O; ++o) in = in || rect_inside(sobs + OSTRIDE * o, p[0], p[1], r);
    } else {
        for (int o = 0; o < O; ++o) in = in || sphere_inside(sobs + OSTRIDE * o, p[0], p[1], p[2], r);
    }
    return in;
}

// ------------------------------------------------------------------------------------
// stable ascending sort of 32 (alpha, idx) keys held one per lane (argsort, env/utils.py:127)
// key order: (flag, alpha, idx); flag 0 = number, 1 = NaN (sorts last), 2 = padding lane.
// ------------------------------------------------------------------------------------
struct SortKey {
    int flag;
    float alpha;
    int idx;
};
__device__ __forceinline__ bool key_less(const SortKey& a, const SortKey& b) {
    if (a.flag != b.flag) return a.flag < b.flag;
    if (a.flag == 0 && a.alpha != b.alpha) return a.alpha < b.alpha;
    return a.idx < b.idx;
}
__device__ __forceinline__ SortKey warp_sort32(SortKey k, int lane) {
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
        for (int j = size >> 1; j > 0; j >>= 1) {
            SortKey o;
            o.flag = __shfl_xor_sync(0xffffffffu, k.flag, j);
            o.alpha = __shfl_xor_sync(0xffffffffu, k.alpha, j);
            o.idx = __shfl_xor_sync(0xffffffffu, k.idx, j);
            const bool up = ((lane & size) == 0);
            const bool lower = ((lane & j) == 0);
            const bool keep_min = (up == lower);
            const bool o_less = key_less(o, k);
            if (keep_min ? o_less : !o_less) k = o;
        }
    }
    return k;
}

// ------------------------------------------------------------------------------------
// u_ref (double_integrator.py:332-338; dubins_car.py:328-379)
// ------------------------------------------------------------------------------------
template <int KIND>
__device__ __forceinline__ void u_ref_dev(const gcbf_env_desc& d, const float* x, const float* gl, float* u) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU;
    if (KIND == GCBF_ENV_DUBINS_CAR) {
        const float PI_F = 3.14159265358979323846f;
        const float TWO_PI = 6.283185307179586f;
        const float pdx = x[0] - gl[0], pdy = x[1] - gl[1];
        const float dist = sqrtf(pdx * pdx + pdy * pdy);
        float theta_t = atan2f(-pdy, -pdx);
        theta_t = theta_t - floorf(theta_t / TWO_PI) * TWO_PI;  // python-style mod
        float theta = x[2] - floorf(x[2] / TWO_PI) * TWO_PI;
        const float theta_diff = theta_t - theta;
        const float dot = (-pdx) * cosf(theta) + (-pdy) * sinf(theta);
        const float tb = acosf(fminf(fmaxf(dot / (dist + 0.0001f), -1.f), 1.f));
        float omega = 0.f;
        const bool c1 = (theta_diff < PI_F) && (theta_diff >= 0.f);
        if (c1 && theta <= PI_F) omega = 1.0f * tb;
        if (!c1 && theta <= PI_F) omega = -1.0f * tb;
        const bool c2 = (theta_diff > -PI_F) && (theta_diff <= 0.f);
        if (c2 && theta > PI_F) omega = -1.0f * tb;
        if (!c2 && theta > PI_F) omega = 1.0f * tb;
        omega = fminf(fmaxf(omega, -5.f), 5.f);
        const float nrm = sqrtf(1e-6f + (pdx * pdx + pdy * pdy));
        const float coef = (nrm > d.comm_radius) ? d.comm_radius / fmaxf(nrm, d.comm_radius) : 1.f;
        const float qx = coef * pdx, qy = coef * pdy;
        u[0] = omega;
        u[1] = -2.5f * x[3] + 2.3f * sqrtf(qx * qx + qy * qy);
        return;
    }
    float err[SD];
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        err[c] = gl[c] - x[c];
        acc = (c == 0) ? err[c] * err[c] : acc + err[c] * err[c];
    }
    const float nrm = sqrtf(acc);
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        const float emax = fabsf(err[c] / nrm * d.comm_radius);
        // jnp.clip(x, lo, hi) = minimum(maximum(x, lo), hi), NaN-propagating
        float e = err[c];
        e = (isnan(e) || isnan(emax)) ? NAN : fminf(fmaxf(e, -emax), emax);
        err[c] = e;
    }
#pragma unroll
    for (int a = 0; a < NU; ++a) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < SD; ++c) s = (c == 0) ? err[c] * d.K[a * SD + c] : s + err[c] * d.K[a * SD + c];
        u[a] = isnan(s) ? NAN : fminf(fmaxf(s, -d.u_lim), d.u_lim);
    }
}

// dx += du . d u_ref / dx (the state Jacobian of u_ref_dev, applied to du).  Kinks as torch autograd differentiates the
// reference's formulas: a clip passes no gradient outside its limits (strictly inside: gradient 1), the branch
// conditions of the DubinsCar law and the python-style mod of theta are piecewise constant.
template <int KIND>
__device__ __forceinline__ void u_ref_vjp_dev(const gcbf_env_desc& d, const float* x, const float* gl, const float* du,
                                              float* dx) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU;
    if (KIND == GCBF_ENV_DUBINS_CAR) {
        const float PI_F = 3.14159265358979323846f;
        const float TWO_PI = 6.283185307179586f;
        const float pdx = x[0] - gl[0], pdy = x[1] - gl[1];
        const float dist = sqrtf(pdx * pdx + pdy * pdy);
        float theta_t = atan2f(-pdy, -pdx);
        theta_t = theta_t - floorf(theta_t / TWO_PI) * TWO_PI;
        const float theta = x[2] - floorf(x[2] / TWO_PI) * TWO_PI;
        const float theta_diff = theta_t - theta;
        const float cth = cosf(theta), sth = sinf(theta);
        const float dot = (-pdx) * cth + (-pdy) * sth;
        const float D = dist + 0.0001f;
        const float q = dot / D;
        // omega = s tb (s = +-1 by the branch conditions, 0 never: one of the four cases always holds)
        const bool c1 = (theta_diff < PI_F) && (theta_diff >= 0.f);
        const bool c2 = (theta_diff > -PI_F) && (theta_diff <= 0.f);
        const float s = (theta <= PI_F) ? (c1 ? 1.f : -1.f) : (c2 ? -1.f : 1.f);
        const float tb = acosf(fminf(fmaxf(q, -1.f), 1.f));
        const float om = s * tb;
        const float dom = (om > -5.f && om < 5.f) ? du[0] : 0.f;
        const float dq = (q > -1.f && q < 1.f) ? dom * s * (-1.f / sqrtf(1.f - q * q)) : 0.f;
        // q = dot / (dist + 1e-4)
        const float dD = -dq * dot / (D * D);
        float gx = dq * (-cth) / D + dD * pdx / dist;
        float gy = dq * (-sth) / D + dD * pdy / dist;
        const float gth = dq * (pdx * sth - pdy * cth) / D;
        // u[1] = -2.5 v + 2.3 |coef pd|, coef = rc / nrm where nrm = sqrt(1e-6 + |pd|^2) > rc
        const float nrm = sqrtf(1e-6f + (pdx * pdx + pdy * pdy));
        const bool clip = nrm > d.comm_radius;
        const float coef = clip ? d.comm_radius / fmaxf(nrm, d.comm_radius) : 1.f;
        const float qx = coef * pdx, qy = coef * pdy;
        const float r = sqrtf(qx * qx + qy * qy);
        const float dr = 2.3f * du[1];
        const float dqx = dr * qx / r, dqy = dr * qy / r;
        gx += coef * dqx;
        gy += coef * dqy;
        if (clip) {
            const float dn = (dqx * pdx + dqy * pdy) * (-d.comm_radius / (nrm * nrm));
            gx += dn * pdx / nrm;
            gy += dn * pdy / nrm;
        }
        dx[0] += gx;
        dx[1] += gy;
        dx[2] += gth;
        dx[3] += -2.5f * du[1];
        return;
    }
    // e = clip(err, -|err| rc / |err|, |err| rc / |err|) componentwise with err = goal - x: a clipped component is
    // err_c rc / |err|;  u = clip(K e, -u_lim, u_lim)
    float err[SD], e[SD];
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        err[c] = gl[c] - x[c];
        acc = (c == 0) ? err[c] * err[c] : acc + err[c] * err[c];
    }
    const float nrm = sqrtf(acc);
    bool clipped[SD];
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        const float emax = fabsf(err[c] / nrm * d.comm_radius);
        clipped[c] = err[c] > emax || err[c] < -emax;
        e[c] = fminf(fmaxf(err[c], -emax), emax);
    }
    float de[SD];
#pragma unroll
    for (int c = 0; c < SD; ++c) de[c] = 0.f;
#pragma unroll
    for (int a = 0; a < NU; ++a) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < SD; ++c) s = (c == 0) ? e[c] * d.K[a * SD + c] : s + e[c] * d.K[a * SD + c];
        const float ds = (s > -d.u_lim && s < d.u_lim) ? du[a] : 0.f;
#pragma unroll
        for (int c = 0; c < SD; ++c) de[c] += ds * d.K[a * SD + c];
    }
    const float k = d.comm_radius / nrm;
    float dot = 0.f;   // sum over the clipped components of de_c err_c
#pragma unroll
    for (int c = 0; c < SD; ++c) dot += clipped[c] ? de[c] * err[c] : 0.f;
    const float w = k * dot / (nrm * nrm);
#pragma unroll
    for (int c = 0; c < SD; ++c) dx[c] -= (clipped[c] ? k * de[c] : de[c]) - w * err[c];   // d err / dx = -1
}

// agent_step_euler (double_integrator.py:128-143; SI :104-109; Dubins :104-122; LD :123-134)
// stop = false: the DubinsCar stop mask is off (env.enable_stop = False, dubins_car.py:138-142)
template <int KIND>
__device__ __forceinline__ void euler_dev(const gcbf_env_desc& d, const float* x, const float* gl, const float* u,
                                          float* xn, const bool stop_mask = true) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU;
    float xd[SD];
    if (KIND == GCBF_ENV_SINGLE_INTEGRATOR) {
        xd[0] = u[0];
        xd[1] = u[1];
    } else if (KIND == GCBF_ENV_DOUBLE_INTEGRATOR) {
        xd[0] = x[2];
        xd[1] = x[3];
        xd[2] = u[0] / d.mass;
        xd[3] = u[1] / d.mass;
    } else if (KIND == GCBF_ENV_DUBINS_CAR) {
        const float ddx = x[0] - gl[0], ddy = x[1] - gl[1];
        const float stop = (stop_mask && sqrtf(ddx * ddx + ddy * ddy) < d.half_r) ? 1.f : 0.f;
        const float keep = 1.f - stop;
        xd[0] = (cosf(x[2]) * x[3]) * keep;
        xd[1] = (sinf(x[2]) * x[3]) * keep;
        xd[2] = (u[0] * 20.f) * keep;
        xd[3] = u[1] * keep;
    } else {
#pragma unroll
        for (int r = 0; r < SD; ++r) {
            float s = 0.f;
#pragma unroll
            for (int c = 0; c < SD; ++c) s += x[c] * d.A[r * SD + c];
            float t = 0.f;
#pragma unroll
            for (int c = 0; c < NU; ++c) t += u[c] * d.B[r * NU + c];
            xd[r] = s + t;
        }
    }
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        float v = xd[c] * d.dt + x[c];
        const bool limited = (KIND == GCBF_ENV_DOUBLE_INTEGRATOR && c >= 2) || (KIND == GCBF_ENV_DUBINS_CAR && c == 3) ||
                             (KIND == GCBF_ENV_LINEAR_DRONE && c >= 3);
        if (limited) v = isnan(v) ? v : fminf(fmaxf(v, -d.v_lim), d.v_lim);
        xn[c] = v;
    }
}

// The transposed Jacobians of euler_dev (stop mask on) at (x, u): dx = dxn . dx'/dx and du = dxn . dx'/du, where dxn
// is the gradient wrt x' after the velocity clip (the caller zeroes the clipped components).  The DubinsCar stop
// mask is piecewise constant in x.
template <int KIND>
__device__ __forceinline__ void euler_vjp_dev(const gcbf_env_desc& d, const float* x, const float* gl, const float* dxn,
                                              float* dx, float* du) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU;
#pragma unroll
    for (int c = 0; c < SD; ++c) dx[c] = dxn[c];
    if (KIND == GCBF_ENV_SINGLE_INTEGRATOR) {
        du[0] = dxn[0] * d.dt;
        du[1] = dxn[1] * d.dt;
    } else if (KIND == GCBF_ENV_DOUBLE_INTEGRATOR) {
        dx[2] += dxn[0] * d.dt;
        dx[3] += dxn[1] * d.dt;
        du[0] = dxn[2] * d.dt / d.mass;
        du[1] = dxn[3] * d.dt / d.mass;
    } else if (KIND == GCBF_ENV_DUBINS_CAR) {
        const float ddx = x[0] - gl[0], ddy = x[1] - gl[1];
        const float keep = (sqrtf(ddx * ddx + ddy * ddy) < d.half_r) ? 0.f : 1.f;
        const float c = cosf(x[2]), s = sinf(x[2]), kt = keep * d.dt;
        dx[2] += (dxn[0] * (-s * x[3]) + dxn[1] * (c * x[3])) * kt;
        dx[3] += (dxn[0] * c + dxn[1] * s) * kt;
        du[0] = dxn[2] * 20.f * kt;
        du[1] = dxn[3] * kt;
    } else {
#pragma unroll
        for (int c = 0; c < SD; ++c) {
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < SD; ++r) s += dxn[r] * d.A[r * SD + c];
            dx[c] += s * d.dt;
        }
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < SD; ++r) s += dxn[r] * d.B[r * NU + c];
            du[c] = s * d.dt;
        }
    }
}

// d_es (edge-state grads of x') -> d a.   x' = clip_state(x + xdot(x, u) dt), u = clip_action(a)
// (gcbf_plus.py:386-391; double_integrator.py:128-143,340-354 and twins): the chain edge state -> state ->
// clip_state -> Euler -> clip_action of agent `a`, shared by the train step and the policy refinement.
template <int KIND>
__device__ __forceinline__ void dyn_chain_dev(const gcbf_env_desc& d, const float* agent, const float* goal,
                                              const float* action, const float* xnext, const float* d_es, const int a,
                                              float* g) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU, ED = T::ED;
    float dx[SD], xn[SD], de[ED];
#pragma unroll
    for (int c = 0; c < ED; ++c) de[c] = d_es[(size_t)a * ED + c];
#pragma unroll
    for (int c = 0; c < SD; ++c) xn[c] = xnext[(size_t)a * SD + c];
    if (KIND == GCBF_ENV_DUBINS_CAR) {  // es = (x, y, v cos th, v sin th)
        const float th = xn[2], v = xn[3];
        dx[0] = de[0];
        dx[1] = de[1];
        dx[2] = de[2] * (-v * sinf(th)) + de[3] * (v * cosf(th));
        dx[3] = de[2] * cosf(th) + de[3] * sinf(th);
    } else {
#pragma unroll
        for (int c = 0; c < SD; ++c) dx[c] = de[c];
    }
    // clip_state: zero gradient on clipped velocity components
#pragma unroll
    for (int c = 0; c < SD; ++c) {
        const bool limited = (KIND == GCBF_ENV_DOUBLE_INTEGRATOR && c >= 2) || (KIND == GCBF_ENV_DUBINS_CAR && c == 3) ||
                             (KIND == GCBF_ENV_LINEAR_DRONE && c >= 3);
        if (limited && !(xn[c] > -d.v_lim && xn[c] < d.v_lim)) dx[c] = 0.f;
    }
    float du[NU];
    if (KIND == GCBF_ENV_SINGLE_INTEGRATOR) {
        du[0] = dx[0] * d.dt;
        du[1] = dx[1] * d.dt;
    } else if (KIND == GCBF_ENV_DOUBLE_INTEGRATOR) {
        du[0] = dx[2] * d.dt / d.mass;
        du[1] = dx[3] * d.dt / d.mass;
    } else if (KIND == GCBF_ENV_DUBINS_CAR) {
        const float ddx = agent[(size_t)a * SD + 0] - goal[(size_t)a * SD + 0];
        const float ddy = agent[(size_t)a * SD + 1] - goal[(size_t)a * SD + 1];
        const float keep = (sqrtf(ddx * ddx + ddy * ddy) < d.half_r) ? 0.f : 1.f;
        du[0] = dx[2] * 20.f * d.dt * keep;
        du[1] = dx[3] * d.dt * keep;
    } else {
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < SD; ++r) s += dx[r] * d.B[r * NU + c];
            du[c] = s * d.dt;
        }
    }
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        const float act = action[(size_t)a * NU + c];
        g[c] = (act > -d.u_lim && act < d.u_lim) ? du[c] : 0.f;  // clip_action
    }
}

// u = clip_action(act), x' = agent_step_euler(x, u); returns ||u - u_ref||^2, the control term of the reward
// (double_integrator.py:145-198)
template <int KIND>
__device__ __forceinline__ float step_agent(const gcbf_env_desc& d, const float* x, const float* gl, const float* act,
                                            const float* ur, const bool stop_mask, float* xn) {
    constexpr int NU = EnvTraits<KIND>::NU;
    float u[NU], sq = 0.f;
#pragma unroll
    for (int c = 0; c < NU; ++c) {
        u[c] = isnan(act[c]) ? act[c] : fminf(fmaxf(act[c], -d.u_lim), d.u_lim);
        const float df = u[c] - ur[c];
        sq = (c == 0) ? df * df : sq + df * df;
    }
    euler_dev<KIND>(d, x, gl, u, xn, stop_mask);
    return sq;
}

// policy tail of a rollout step: pi = tanh(z + bHO) (policy.py:72), a = 2 pi + u_ref (gcbf_plus.py:182-186)
template <int KIND>
__device__ __forceinline__ void policy_action(const gcbf_env_desc& d, const float* x, const float* gl, const float* z,
                                              const float* bHO, float* ur, float* act) {
    u_ref_dev<KIND>(d, x, gl, ur);
#pragma unroll
    for (int c = 0; c < EnvTraits<KIND>::NU; ++c) act[c] = 2.f * tanhf(z[c] + bHO[c]) + ur[c];
}

// get_cost's agent term (double_integrator.py:183-198): any neighbour j of the previous graph with 2r > ||x - x_j||.
// edge_src holds the agent's edge row [rs, rs + rd): self / goal edge first, then agent senders, then hit codes (< 0).
template <int PD, int SD>
__device__ __forceinline__ bool collides_prev(const float* x, int rs, int rd, const int32_t* edge_src,
                                              const float* agent_prev, float two_r) {
    bool col = false;
    for (int e = rs + 1; e < rs + rd; ++e) {
        const int s = edge_src[e];
        if (s < 0) break;
        float dd = 0.f;
#pragma unroll
        for (int c = 0; c < PD; ++c) {
            const float dlt = x[c] - agent_prev[(size_t)s * SD + c];
            dd = (c == 0) ? dlt * dlt : dd + dlt * dlt;
        }
        col = col || (two_r > sqrtf(dd));
    }
    return col;
}

// Smallest fp32 a whose correctly rounded sqrtf is >= r, so that (sqrtf(x) < r) == (x < a) and (r > sqrtf(x)) ==
// (x < a) for every fp32 x (NaN: both false).  The device twin of _lib.sqrt_threshold, which the host uses for
// comm_sq_thr / lidar_sq_thr; r <= 0 gives 0, which no x is below.
__device__ __forceinline__ float sqrt_threshold(float r) {
    float a = r * r;
    while (a > 0.f && sqrtf(a) >= r) a = nextafterf(a, 0.f);
    while (sqrtf(a) < r) a = nextafterf(a, INFINITY);
    return a;
}

// Reward and cost of one graph from per-thread sums acc = [sum ||u - u_ref||^2, #colliding, #inside an obstacle]:
// warp sums, then thread 0 adds the NW warp sums in warp order.  Warps without agents add +0, so CTAs of different
// widths give the same bits.  Every thread of the CTA calls it.
template <int NW>
__device__ __forceinline__ void reduce_reward_cost(const float* acc, float* s_red, int N, float* reward, float* cost) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const float v = warp_sum(acc[q]);
        if (lane == 0) s_red[q * NW + warp] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float t[3] = {0.f, 0.f, 0.f};
        for (int w = 0; w < NW; ++w) {
            t[0] += s_red[0 * NW + w];
            t[1] += s_red[1 * NW + w];
            t[2] += s_red[2 * NW + w];
        }
        *reward = -(t[0] / (float)N);
        *cost = t[1] / (float)N + t[2] / (float)N;
    }
}

// ------------------------------------------------------------------------------------
// graph build of one agent per warp (graph_build_kernel and the persistent rollout kernel; the persistent kernel fills
// FILL_NA rows per warp at once)
// ------------------------------------------------------------------------------------
// 2-D obstacle rows in shared memory are 24 floats: the packed rectangle, then the derived fields of the far-obstacle
// skip at [14] reach^2, [15..18] edge dx, [19..22] edge dy.
constexpr int OBS2D = 24;
__device__ __forceinline__ void derive_far_fields(float* sobs, int O, float comm_radius, int tid, int nthreads) {
    for (int o = tid; o < O; o += nthreads) {
        float* ob = sobs + OBS2D * o;
        const float reach = comm_radius + sqrtf(ob[2] * ob[2] + ob[3] * ob[3]) + 2e-3f;
        ob[14] = reach * reach;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int kp = (k + 3) & 3;
            ob[15 + k] = ob[6 + 2 * kp] - ob[6 + 2 * k];   // x4 - x3
            ob[19 + k] = ob[7 + 2 * kp] - ob[7 + 2 * k];   // y4 - y3
        }
    }
}

// 2-D LiDAR (env/utils.py:49-131) of the agent at p, one ray per lane: the R closest returns in stable argsort order
// -> my_hits[R][2], and lane r < R also returns hit r in (hx, hy), so that the active-hit test need not read the
// global store back.  sobs: O obstacle rows of OBS2D floats (derive_far_fields), stab: [n_rays][2] ray offsets.
__device__ __forceinline__ void lidar2d_warp(const float* p, const float* stab, const float* sobs, int O, int n_rays,
                                             int R, int lane, float* my_hits, float& hx_out, float& hy_out) {
    const bool ray_ok = lane < n_rays;
    const int rl = ray_ok ? lane : 0;
    const float x1 = p[0], y1 = p[1];
    const float x2 = x1 + stab[rl * 2 + 0], y2 = y1 + stab[rl * 2 + 1];
    const float rdx = x1 - x2, rdy = y1 - y2;
    float alpha;
    if (O == 0) {
        alpha = 1.f * NO_HIT;
    } else {
        // A rectangle whose bounding circle is out of the ray's reach cannot be hit or contain the agent:
        // every edge test gives valid = 0 and alpha = 0 * alpha + 1e6 = 1e6 exactly -- unless an edge is
        // exactly parallel to the ray (det == 0 -> alpha = x/0 -> NaN in the reference, obstacle.py:88-94).
        // The skip is taken only when it is bit-identical to the full evaluation (agent-uniform branch).
        alpha = NO_HIT;
        bool is_in = false;
        for (int o = 0; o < O; ++o) {
            const float* ob = sobs + OBS2D * o;
            const float cx = x1 - ob[0], cy = y1 - ob[1];
            const bool far = (cx * cx + cy * cy) > ob[14];
            bool degenerate = false;
            if (far) {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float det = rdx * ob[19 + k] - rdy * ob[15 + k];
                    degenerate = degenerate || !(det != 0.f);   // det == 0 or NaN
                }
            }
            if (!far) is_in = is_in || rect_inside(ob, x1, y1, 0.f);
            if (!far || __any_sync(0xffffffffu, degenerate))
                alpha = nanmin(alpha, rect_raytrace(ob, x1, y1, x2, y2));
        }
        alpha = alpha * (1.f - (is_in ? 1.f : 0.f));
    }
    const float hx = x1 + (x2 - x1) * alpha;
    const float hy = y1 + (y2 - y1) * alpha;
    SortKey k;
    k.flag = ray_ok ? (isnan(alpha) ? 1 : 0) : 2;
    k.alpha = alpha;
    k.idx = lane;
    // argsort is stable: when no ray of this agent hit anything (every alpha == 1e6) the order is the
    // identity and the 15-stage warp sort can be skipped (warp-uniform, the common case in open space)
    const bool all_miss = __all_sync(0xffffffffu, !ray_ok || alpha == NO_HIT);
    if (!all_miss) k = warp_sort32(k, lane);
    const float shx = __shfl_sync(0xffffffffu, hx, k.idx);
    const float shy = __shfl_sync(0xffffffffu, hy, k.idx);
    if (lane < R) {
        my_hits[lane * 2 + 0] = shx;
        my_hits[lane * 2 + 1] = shy;
    }
    hx_out = shx;
    hy_out = shy;
}

// active hit nodes: ||p - hit|| < comm_radius - 0.1 (double_integrator.py:254-257); bit r = hit r (ballot, lane r).
// h: hit `lane` (read only on lanes < n_hits).
template <int PD>
__device__ __forceinline__ unsigned active_hit_bits(const gcbf_env_desc& d, const float* p, const float* h, int lane,
                                                    bool valid) {
    bool act = false;
    if (valid && lane < d.n_hits) {
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < PD; ++c) {
            const float dlt = p[c] - h[c];
            acc = (c == 0) ? dlt * dlt : acc + dlt * dlt;
        }
        act = acc < d.lidar_sq_thr;   // == (sqrtf(acc) < lidar_radius), threshold precomputed exactly on the host
    }
    return __ballot_sync(0xffffffffu, act);
}

// Neighbour words of the n agents i0 .. i0 + n - 1 of a graph: ||p_i - p_j|| < comm_radius, j != i
// (double_integrator.py:227-232), agent j's position at pos + j * STRIDE.  Word w of agent i0 + s goes to
// bits[s * bstride + w], bit b = candidate 32 w + b.  sqrtf(acc) < Rc  <=>  acc < d.comm_sq_thr (smallest fp32 whose
// correctly rounded sqrt is >= Rc; host-computed), so the scan needs no sqrt.
// One thread per (word, agent), tasks tid, tid + nthreads, ...: consecutive threads take consecutive agents of the same
// word, so each candidate load is a shared-memory broadcast, and every thread runs an independent 32-candidate chain
// (no ballot, no warp-wide dependence).  An odd bstride keeps the word stores of 32 consecutive agents conflict-free.
// COL: also set col[s] = 1 when some other agent j has acc < col_thr (= two_r_sq_thr: 2r > ||p_i - p_j||; the caller
// zeroes col).  Only the candidates already in the word are tested, which finds them all when col_thr <= comm_sq_thr:
// the caller's condition for using the flag.
template <int PD, int STRIDE, bool COL = false>
__device__ __forceinline__ void neighbour_words(const gcbf_env_desc& d, const float* pos, int i0, int n, unsigned* bits,
                                                int bstride, int tid, int nthreads, float col_thr = 0.f,
                                                uint8_t* col = nullptr) {
    const int N = d.n_agents, n_words = (N + 31) >> 5;
    const float thr = d.comm_sq_thr;
    for (int task = tid; task < n * n_words; task += nthreads) {
        const int w = task / n, s = task - w * n;
        const int i = i0 + s;
        float p[PD];
#pragma unroll
        for (int c = 0; c < PD; ++c) p[c] = pos[i * STRIDE + c];
        const float* q = pos + (w << 5) * STRIDE;
        unsigned word = 0u;
        if ((w << 5) + 32 <= N) {
#pragma unroll
            for (int b = 0; b < 32; ++b) {
                float acc;
                if (PD == 2) {
                    const float2 qq = *reinterpret_cast<const float2*>(q + b * STRIDE);
                    const float dx = p[0] - qq.x, dy = p[1] - qq.y;
                    acc = dx * dx;
                    acc = acc + dy * dy;
                } else {
#pragma unroll
                    for (int c = 0; c < PD; ++c) {
                        const float dlt = p[c] - q[b * STRIDE + c];
                        acc = (c == 0) ? dlt * dlt : acc + dlt * dlt;
                    }
                }
                word |= (acc < thr ? 1u : 0u) << b;
            }
        } else {
            const int nb = N - (w << 5);
            for (int b = 0; b < nb; ++b) {
                float acc;
#pragma unroll
                for (int c = 0; c < PD; ++c) {
                    const float dlt = p[c] - q[b * STRIDE + c];
                    acc = (c == 0) ? dlt * dlt : acc + dlt * dlt;
                }
                word |= (acc < thr ? 1u : 0u) << b;
            }
        }
        if (w == (i >> 5)) word &= ~(1u << (i & 31));
        bits[s * bstride + w] = word;
        if (COL && word != 0u) {   // the same acc expression as above, for the few neighbours
            bool c = false;
            for (unsigned m = word; m != 0u; m &= m - 1u) {
                const int b = __ffs(m) - 1;
                float acc;
#pragma unroll
                for (int c2 = 0; c2 < PD; ++c2) {
                    const float dlt = p[c2] - q[b * STRIDE + c2];
                    acc = (c2 == 0) ? dlt * dlt : acc + dlt * dlt;
                }
                c = c || (acc < col_thr);
            }
            if (c) col[s] = 1;
        }
    }
}

// neighbour count of one agent from its words (warp-wide; every lane returns it)
__device__ __forceinline__ int word_count(const unsigned* my_bits, int n_words, int lane) {
    int cnt = 0;
    for (int w = lane; w < n_words; w += 32) cnt += __popc(my_bits[w]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    return cnt;
}

// Edge rows of NA receivers a_id[a] at rbase[a]: [goal | agents ascending | active hits ascending] (edge codes:
// gcbf_b200.h); rows with ok[a] false are not written.  Agent j of the graph is sender sender0 + j.
// Lane w holds word w of every row (32 words per round), so the word loads of all NA rows issue at once and the row
// walks only the non-empty words (most words of a sparse neighbourhood are empty).
template <int NA>
__device__ __forceinline__ void fill_row(int32_t* er, int32_t* es, const int (&rbase)[NA], const int (&a_id)[NA],
                                         const bool (&ok)[NA], int sender0, const unsigned* const (&my_bits)[NA],
                                         int n_words, const unsigned (&hit_bits)[NA], int lane) {
    const unsigned lt = (1u << lane) - 1u;
    int pos[NA];
#pragma unroll
    for (int a = 0; a < NA; ++a) {
        if (ok[a] && lane == 0) {
            er[rbase[a]] = a_id[a];
            es[rbase[a]] = -1;
        }
        pos[a] = rbase[a] + 1;
    }
    for (int w0 = 0; w0 < n_words; w0 += 32) {
        unsigned words[NA], nz[NA];
#pragma unroll
        for (int a = 0; a < NA; ++a) words[a] = (ok[a] && w0 + lane < n_words) ? my_bits[a][w0 + lane] : 0u;
#pragma unroll
        for (int a = 0; a < NA; ++a) nz[a] = __ballot_sync(0xffffffffu, words[a] != 0u);
#pragma unroll
        for (int a = 0; a < NA; ++a) {
            for (unsigned m = nz[a]; m != 0u; m &= m - 1u) {      // warp-uniform
                const int wl = __ffs(m) - 1;
                const unsigned bits = __shfl_sync(0xffffffffu, words[a], wl);
                if ((bits >> lane) & 1u) {
                    const int e = pos[a] + __popc(bits & lt);
                    er[e] = a_id[a];
                    es[e] = sender0 + ((w0 + wl) << 5) + lane;
                }
                pos[a] += __popc(bits);
            }
        }
    }
#pragma unroll
    for (int a = 0; a < NA; ++a) {
        if (ok[a] && ((hit_bits[a] >> lane) & 1u)) {
            const int e = pos[a] + __popc(hit_bits[a] & lt);
            er[e] = a_id[a];
            es[e] = -2 - lane;
        }
    }
}

}  // namespace gcbf
