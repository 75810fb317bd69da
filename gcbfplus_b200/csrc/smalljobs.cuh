// smalljobs.cuh -- batched small dense products on parameter-sized matrices (<= 256 x 256 x 256), one launch per
// dependency wave: folding the linear tails of the MLP blocks for inference / the folded train step
// (gcbf_prepare_infer) and un-folding the gradients of the folded weights back onto the flax parameters
// (gcbf_train_step).  Plus the plane builder: transposed / straight tf32 hi-lo planes of the GEMM weights.
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

// 32 x 32 output tile per CTA (256 threads, 4 outputs each), operand tiles staged through shared memory with the
// global loads coalesced along whichever index has unit stride.  Every output is still ONE accumulator fed in ascending
// k by fused multiply-adds, then the rank-1 term, then the bias: same bits as a thread-per-output loop.
static __global__ void __launch_bounds__(256) small_jobs_kernel(const SmallJobs J) {
    __shared__ float As[32][33];   // [i][kk]
    __shared__ float Bs[32][33];   // [kk][j]
    int q = 0;
    while (q + 1 < J.n && (int)blockIdx.x >= J.blk0[q + 1]) ++q;
    const SmallJob& job = J.j[q];
    const int t = blockIdx.x - J.blk0[q];
    const int tiles_n = (job.n + 31) / 32;
    const int r0 = (t / tiles_n) * 32, c0 = (t % tiles_n) * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (job.A != nullptr) {
        const bool a_k_fast = job.a_cs == 1;     // A(i, k): k contiguous -> lanes along k, else lanes along i
        const bool b_j_fast = job.b_cs == 1;     // B(k, j): j contiguous -> lanes along j, else lanes along k
        // register double buffer: the global loads of k-tile t + 1 are in flight while tile t is consumed
        float ra[4], rb[4];
        auto fetch = [&](int k0) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int s = ty + 8 * q;
                const int i = a_k_fast ? s : tx, kk = a_k_fast ? tx : s;
                const int r = r0 + i, k = k0 + kk;
                ra[q] = (r < job.m && k < job.k) ? job.A[(size_t)r * job.a_rs + (size_t)k * job.a_cs] : 0.f;
                const int kb = b_j_fast ? s : tx, jb = b_j_fast ? tx : s;
                const int kq = k0 + kb, c = c0 + jb;
                rb[q] = (kq < job.k && c < job.n) ? job.B[(size_t)kq * job.b_rs + (size_t)c * job.b_cs] : 0.f;
            }
        };
        fetch(0);
        for (int k0 = 0; k0 < job.k; k0 += 32) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int s = ty + 8 * q;
                As[a_k_fast ? s : tx][a_k_fast ? tx : s] = ra[q];
                Bs[b_j_fast ? s : tx][b_j_fast ? tx : s] = rb[q];
            }
            __syncthreads();
            if (k0 + 32 < job.k) fetch(k0 + 32);
            const int kmax = min(32, job.k - k0);
            if (kmax == 32) {
#pragma unroll 8
                for (int kk = 0; kk < 32; ++kk) {
                    const float bv = Bs[kk][tx];
#pragma unroll
                    for (int o = 0; o < 4; ++o) acc[o] = fmaf(As[ty + 8 * o][kk], bv, acc[o]);
                }
            } else {
                for (int kk = 0; kk < kmax; ++kk) {
                    const float bv = Bs[kk][tx];
#pragma unroll
                    for (int o = 0; o < 4; ++o) acc[o] = fmaf(As[ty + 8 * o][kk], bv, acc[o]);
                }
            }
            __syncthreads();
        }
    }
#pragma unroll
    for (int o = 0; o < 4; ++o) {
        const int r = r0 + ty + 8 * o, c = c0 + tx;
        if (r >= job.m || c >= job.n) continue;
        float sv = acc[o];
        if (job.u != nullptr) sv = fmaf(job.u[r], job.v[c], sv);
        if (job.bias != nullptr) sv += job.bias[c];
        const size_t idx = (size_t)r * job.n + c;
        job.C[idx] = job.accumulate ? job.C[idx] + sv : sv;
    }
}

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
    int32_t launch(cudaStream_t st) {
        if (J.n == 0) return 0;
        small_jobs_kernel<<<J.blk0[J.n], 256, 0, st>>>(J);
        count_launch();
        const int32_t rc = check_launch("small_jobs_kernel");
        J.n = 0;
        return rc;
    }
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
static __global__ void __launch_bounds__(256) plane_jobs_kernel(const PlaneJobs J) {
    __shared__ float tile[32][33];
    int j = 0;
    while (j + 1 < J.n && (int)blockIdx.x >= J.tile0[j + 1]) ++j;
    const int t = blockIdx.x - J.tile0[j];
    const int rows = J.rows[j], cols = J.cols[j];
    const int tiles_c = (cols + 31) / 32;
    const int c0 = (t % tiles_c) * 32, r0 = (t / tiles_c) * 32;
    const float* in = J.src[j];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    if (!J.trans[j]) {
        for (int i = ty; i < 32; i += 8) {
            const int r = r0 + i, c = c0 + tx;
            if (r < rows && c < cols) {
                const float x = in[(size_t)r * cols + c];
                const float h = rn_tf32(x);
                J.hi[j][(size_t)r * cols + c] = h;
                J.lo[j][(size_t)r * cols + c] = rn_tf32(x - h);
            }
        }
        return;
    }
    for (int i = ty; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + tx;
        if (r < rows && c < cols) tile[i][tx] = in[(size_t)r * cols + c];
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + tx;
        if (r < rows && c < cols) {
            const float x = tile[tx][i];
            const float h = rn_tf32(x);
            J.hi[j][(size_t)c * rows + r] = h;
            J.lo[j][(size_t)c * rows + r] = rn_tf32(x - h);
        }
    }
}
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
    int32_t launch(cudaStream_t st) {
        if (J.n == 0) return 0;
        plane_jobs_kernel<<<J.tile0[J.n], 256, 0, st>>>(J);
        count_launch();
        const int32_t rc = check_launch("plane_jobs_kernel");
        J.n = 0;
        return rc;
    }
};

}  // namespace gcbf
