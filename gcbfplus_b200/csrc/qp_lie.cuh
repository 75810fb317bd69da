// qp_lie.cuh -- Lie derivatives of a scalar function of the edge states along the control-affine dynamics
// (env.control_affine_dyn).  Shared by the GCBF+ QP labels (qp.cu) and the CBF-QP baselines (cbfqp.cu).
#pragma once

#include "common.cuh"

namespace gcbf {

// d es / d x applied to an edge-state cotangent (Dubins: es = (x, y, v cos th, v sin th)), then contracted with
// the control-affine dynamics of THAT agent: lf = dx . f(x), lg[c] = dx . g(x)[:, c].
// f, g: single_integrator.py:231-238, double_integrator.py:266-273, dubins_car.py:243-254 (g = diag(10, 1) on
// (theta, v) here, not the 20 of the step), linear_drone.py:255-262.
template <int KIND>
__device__ __forceinline__ void qp_lie_terms(const gcbf_env_desc& d, const float* x, const float* de, float* lf,
                                             float* lg) {
    using T = EnvTraits<KIND>;
    constexpr int SD = T::SD, NU = T::NU;
    float dx[SD];
    if (KIND == GCBF_ENV_DUBINS_CAR) {
        const float th = x[2], v = x[3];
        float sn, cs;
        sincosf(th, &sn, &cs);
        dx[0] = de[0];
        dx[1] = de[1];
        dx[2] = de[2] * (-v * sn) + de[3] * (v * cs);
        dx[3] = de[2] * cs + de[3] * sn;
        *lf = dx[0] * (cs * v) + dx[1] * (sn * v);
        lg[0] = dx[2] * 10.f;
        lg[1] = dx[3];
    } else if (KIND == GCBF_ENV_SINGLE_INTEGRATOR) {
        *lf = 0.f;
        lg[0] = de[0];
        lg[1] = de[1];
    } else if (KIND == GCBF_ENV_DOUBLE_INTEGRATOR) {
#pragma unroll
        for (int c = 0; c < SD; ++c) dx[c] = de[c];
        *lf = dx[0] * x[2] + dx[1] * x[3];
        lg[0] = dx[2] / d.mass;
        lg[1] = dx[3] / d.mass;
    } else {
#pragma unroll
        for (int c = 0; c < SD; ++c) dx[c] = de[c];
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < SD; ++r) {
            float fr = 0.f;
#pragma unroll
            for (int c = 0; c < SD; ++c) fr += d.A[r * SD + c] * x[c];
            s += dx[r] * fr;
        }
        *lf = s;
#pragma unroll
        for (int c = 0; c < NU; ++c) {
            float t = 0.f;
#pragma unroll
            for (int r = 0; r < SD; ++r) t += dx[r] * d.B[r * NU + c];
            lg[c] = t;
        }
    }
}

}  // namespace gcbf
