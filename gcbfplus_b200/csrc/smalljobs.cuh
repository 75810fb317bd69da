// smalljobs.cuh -- batched small dense products on parameter-sized matrices (<= 256 x 256 x 256), one launch per
// dependency wave: folding the linear tails of the MLP blocks for inference / the folded train step
// (gcbf_prepare_infer) and un-folding the gradients of the folded weights back onto the flax parameters
// (gcbf_train_step).  Plus the plane builder: transposed / straight tf32 hi-lo planes of the GEMM weights.  Their
// kernels and launch() are in dense.cu.
//
// The layers folded here are the ones gcbfplus/nn/mlp.py:23-29 applies with act_final=False, i.e. back to back with
// no nonlinearity (gcbfplus/nn/gnn.py:53-72, algo/module/cbf.py:12-21, policy.py:63-73).
#pragma once
#include "common.cuh"

namespace gcbf {

// C[i, j] (+)= sum_k A(i, k) B(k, j) + u[i] v[j] + bias[j];  A(i, k) = A[i a_rs + k a_cs], B(k, j) = B[k b_rs + j b_cs].
// One accumulator per output, sequential fused multiply-adds over ascending k, then the rank-1 term, then the bias.
struct SmallJob {
    const float* A;
    const float* B;
    float* C;
    const float* u;
    const float* v;
    const float* bias;
    int m, n, k;
    int a_rs, a_cs, b_rs, b_cs;
    int accumulate;
};
constexpr int SMALL_MAX_JOBS = 40;   // 40 x 80 B + offsets < the 4 KB kernel-parameter limit
struct SmallJobs {
    int n;
    int blk0[SMALL_MAX_JOBS + 1];
    SmallJob j[SMALL_MAX_JOBS];
};

struct SmallJobList {
    SmallJobs J;
    SmallJobList() { J.n = 0; J.blk0[0] = 0; }
    // C[m, n] (+)= A B + u (x) v + bias   (pass nullptr for absent terms)
    void add(float* C, int m, int n, int k, const float* A, int a_rs, int a_cs, const float* B, int b_rs, int b_cs,
             const float* u, const float* v, const float* bias, bool accumulate) {
        SmallJob& q = J.j[J.n];
        q.A = A; q.B = B; q.C = C; q.u = u; q.v = v; q.bias = bias;
        q.m = m; q.n = n; q.k = k;
        q.a_rs = a_rs; q.a_cs = a_cs; q.b_rs = b_rs; q.b_cs = b_cs;
        q.accumulate = accumulate ? 1 : 0;
        J.blk0[J.n + 1] = J.blk0[J.n] + ((m + 31) / 32) * ((n + 31) / 32);
        ++J.n;
    }
    bool full() const { return J.n >= SMALL_MAX_JOBS; }
    int32_t launch(cudaStream_t st);
};

// ---- tf32 hi / lo planes of a [rows, cols] matrix, straight or transposed, several matrices per launch
constexpr int PLANE_MAX_JOBS = 18;   // the planes of a one-layer network (PlaneLayout): 9 transposed + 9 straight
struct PlaneJobs {
    int n;
    int tile0[PLANE_MAX_JOBS + 1];
    const float* src[PLANE_MAX_JOBS];
    float* hi[PLANE_MAX_JOBS];
    float* lo[PLANE_MAX_JOBS];
    int rows[PLANE_MAX_JOBS], cols[PLANE_MAX_JOBS], trans[PLANE_MAX_JOBS];
};
struct PlaneJobList {
    PlaneJobs J;
    PlaneJobList() { J.n = 0; J.tile0[0] = 0; }
    void add(const float* src, int rows, int cols, bool transpose, float* hi, float* lo) {
        const int q = J.n;
        J.src[q] = src; J.hi[q] = hi; J.lo[q] = lo;
        J.rows[q] = rows; J.cols[q] = cols; J.trans[q] = transpose ? 1 : 0;
        J.tile0[q + 1] = J.tile0[q] + ((rows + 31) / 32) * ((cols + 31) / 32);
        ++J.n;
    }
    int32_t launch(cudaStream_t st);
};

}  // namespace gcbf
