// common.cuh -- shared host/device helpers for libgcbf_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/gcbf_b200.h"

namespace gcbf {

// ---- error reporting (thread-local, no exceptions, no aborts) -----------------------
void set_error(const char* fmt, ...);
int32_t check_launch(const char* what);  // returns cudaGetLastError() mapped to >0 status
void count_launch(int64_t n = 1);
int sm_count();

#define GCBF_REQUIRE(cond, ...)            \
    do {                                   \
        if (!(cond)) {                     \
            gcbf::set_error(__VA_ARGS__);  \
            return -1;                     \
        }                                  \
    } while (0)

// ---- fused policy tail of the rollout step (z == nullptr: plain graph build from `agent`).
struct TailArgs {
    const float* z;            // [parts][z_cap][4] output-layer partial sums (no bias / tanh)
    int parts, z_cap;
    const float* bHO;          // output-layer bias
    const float* agent_prev;   // states the action is computed for
    const float* goal;
    const int32_t* row_start_prev;   // previous graph (cost: any neighbour within 2r)
    const int32_t* row_deg_prev;
    const int32_t* edge_src_prev;
    float* action;             // out [A, nu] (unclipped 2 pi + u_ref)
    float* next_agent;         // out [A, sd]
};

// ---- workspace layouts: consecutive slots, each rounded up to `align` floats (a power of two) --------------------
struct WsSlots {
    int64_t align, off = 0;
    int64_t take(int64_t n) {
        const int64_t r = off;
        off += (n + align - 1) & ~(align - 1);
        return r;
    }
};

// ---- per-environment compile-time traits -------------------------------------------
template <int KIND> struct EnvTraits;
template <> struct EnvTraits<GCBF_ENV_SINGLE_INTEGRATOR> { static constexpr int SD = 2, ED = 2, NU = 2, PD = 2; };
template <> struct EnvTraits<GCBF_ENV_DOUBLE_INTEGRATOR> { static constexpr int SD = 4, ED = 4, NU = 2, PD = 2; };
template <> struct EnvTraits<GCBF_ENV_DUBINS_CAR> { static constexpr int SD = 4, ED = 4, NU = 2, PD = 2; };
template <> struct EnvTraits<GCBF_ENV_LINEAR_DRONE> { static constexpr int SD = 6, ED = 6, NU = 3, PD = 3; };

inline int env_sd(int kind) { return kind == 0 ? 2 : (kind == 3 ? 6 : 4); }
inline int env_ed(int kind) { return env_sd(kind); }
inline int env_nu(int kind) { return kind == 3 ? 3 : 2; }
inline int env_pd(int kind) { return kind == 3 ? 3 : 2; }

// Dispatch a generic lambda-like functor over the env kind.
#define GCBF_DISPATCH_ENV(kind, ...)                                                      \
    switch (kind) {                                                                       \
        case GCBF_ENV_SINGLE_INTEGRATOR: { constexpr int KIND = GCBF_ENV_SINGLE_INTEGRATOR; __VA_ARGS__; } break; \
        case GCBF_ENV_DOUBLE_INTEGRATOR: { constexpr int KIND = GCBF_ENV_DOUBLE_INTEGRATOR; __VA_ARGS__; } break; \
        case GCBF_ENV_DUBINS_CAR: { constexpr int KIND = GCBF_ENV_DUBINS_CAR; __VA_ARGS__; } break;               \
        case GCBF_ENV_LINEAR_DRONE: { constexpr int KIND = GCBF_ENV_LINEAR_DRONE; __VA_ARGS__; } break;           \
        default: gcbf::set_error("unknown env_kind %d", (int)(kind)); return -1;          \
    }

// ---- flat parameter layout (one network) --------------------------------------------
// Forward order of the 12 Dense layers (SURVEY A.3); offsets in floats, 4-float aligned.
struct ParamLayout {
    int w[12];
    int b[12];
    int in[12];
    int out[12];
    int total;
};
enum { L_MSG0 = 0, L_MSG1, L_MSGOUT, L_ATT0, L_ATT1, L_GATE, L_UPD0, L_UPD1, L_UPDOUT, L_HEAD0, L_HEAD1, L_OUT };

inline ParamLayout make_layout(int edge_dim, int out_dim) {
    ParamLayout L;
    const int in[12] = {edge_dim + 6, 256, 256, 128, 128, 128, 131, 256, 256, 128, 256, 256};
    const int out[12] = {256, 256, 128, 128, 128, 1, 256, 256, 128, 256, 256, out_dim};
    int off = 0;
    for (int i = 0; i < 12; ++i) {
        L.in[i] = in[i];
        L.out[i] = out[i];
        L.w[i] = off;
        off += in[i] * out[i];
        off = (off + 3) & ~3;
        L.b[i] = off;
        off += out[i];
        off = (off + 3) & ~3;
    }
    L.total = off;
    return L;
}

// ---- flat parameter layout of an n_layers-deep network (gnn.py:78-104 with n_layers > 1) -----------------------
// Forward order: the 9 Dense layers of GNN layer 0, ..., of layer n - 1, then the 3 of the head.  layer[l] views GNN
// layer l plus the head as a 12-entry ParamLayout (its `total` is the whole network's).  From layer 1 on, msg/Dense_0
// reads [edge | y_sender | y_receiver] (ed + 256 rows) and update/Dense_0 reads [y | aggregate] (256 rows); every layer
// outputs 128.  n_layers = 1 gives make_layout's offsets.
constexpr int GCBF_MAX_LAYERS = 8;
struct DeepLayout {
    int n_layers;
    ParamLayout layer[GCBF_MAX_LAYERS];
    int total;
};
inline DeepLayout make_deep_layout(int edge_dim, int out_dim, int n_layers) {
    DeepLayout D;
    D.n_layers = n_layers;
    const ParamLayout L0 = make_layout(edge_dim, out_dim);
    int off = 0;
    auto place = [&](ParamLayout& P, int i, int in) {
        P.in[i] = in;
        P.out[i] = L0.out[i];
        P.w[i] = off;
        off += in * L0.out[i];
        off = (off + 3) & ~3;
        P.b[i] = off;
        off += L0.out[i];
        off = (off + 3) & ~3;
    };
    for (int l = 0; l < n_layers; ++l)
        for (int i = 0; i < L_HEAD0; ++i)
            place(D.layer[l], i, l == 0 ? L0.in[i] : (i == L_MSG0 ? edge_dim + 256 : (i == L_UPD0 ? 256 : L0.in[i])));
    for (int i = L_HEAD0; i <= L_OUT; ++i) place(D.layer[0], i, L0.in[i]);
    for (int l = 0; l < n_layers; ++l) {
        for (int i = L_HEAD0; i <= L_OUT; ++i) {
            D.layer[l].in[i] = D.layer[0].in[i];
            D.layer[l].out[i] = D.layer[0].out[i];
            D.layer[l].w[i] = D.layer[0].w[i];
            D.layer[l].b[i] = D.layer[0].b[i];
        }
        D.layer[l].total = off;
    }
    D.total = off;
    return D;
}

// tf32(x) rounded to nearest (13 low mantissa bits cleared, so the tensor core's own fp32->tf32 conversion is exact);
// the hi / lo planes of the 3xTF32 GEMMs are rn_tf32(x) and rn_tf32(x - hi).
__device__ __forceinline__ float rn_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace gcbf
