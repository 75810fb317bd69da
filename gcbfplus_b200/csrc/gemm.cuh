// gemm.cuh -- types and constants of the dense-layer GEMMs of the GNN: the epilogues, the ordered partial sums and the
// row counts.  The kernels and their launchers are in dense.cu (declared in internal.cuh): the fp32 SIMT GEMM family
// (strict-fp32 parity path; SURVEY 8c: fp32 FMA is the parity default) and the tensor-core GEMMs of gemm_tc.cuh.  All
// operands row-major, contiguous.
//
//   gemm_nn : C[M,N] = epi(A[M,K] @ B[K,N])     forward (B = W) and backward-data (B = W^T)
//   gemm_tn : C[K1,N] += sum_m w[m] * X[m,K1] * dY[m,N]   backward-weight (split over M, ordered partial sums)
//   colsum  : db[N] += sum_m w[m] * dY[m,N]
//
// No float atomics: a kernel that splits a sum over CTAs writes one partial per CTA to a workspace and
// partial_sum_kernel adds the partials in CTA order, so every result is bit-identical from run to run.
#pragma once
#include "common.cuh"

namespace gcbf {

enum GemmEpi {
    EPI_BIAS = 0,       // C = acc + bias (+ bias2)
    EPI_BIAS_RELU = 1,  // C = relu(acc + bias (+ bias2))
    EPI_NONE = 2,       // C = acc
    EPI_RELU_MASK = 3,  // C = aux > 0 ? acc : 0      (backward through ReLU, aux = saved activation)
                        // 4 is unassigned: the C ABI passes these values, so they keep their numbers
    EPI_RELU_DOTN = 5,  // C[(part*m_cap + m)*4 + q] = sum_{n in column tile `part`} relu(acc + bias)[n] * aux[n*ndot + q]
                        // (tensor-core path only: the output layer folded into the last hidden layer's epilogue)
};

// ------------------------------------------------------------------------------------ ordered partial sums
// Floats of the partials workspace every split reduction of the train step shares (one reduction at a time, in stream
// order): 160 CTAs of a [128 x 256] weight-gradient tile plus its 256 column sums.  Launchers cap their CTA count so
// that their partials fit.
constexpr int64_t PART_FLOATS = 160 * (128 * 256 + 256);
constexpr int DW_MAX_CTAS_TC = 160;     // tensor-core dW GEMM: [128 x N] partial (+ N column sums) per CTA
constexpr int DW_MAX_CTAS_SIMT = 320;   // SIMT dW GEMM: [128 x 128] partial per CTA

// destination segments of one reduction: element i of a partial maps to segment k, offset j; dst2 (optional) receives
// the same sum (a bias gradient shared by two parameters)
struct PartSeg {
    float* dst;
    float* dst2;
    int n;
};
struct PartSegs {
    PartSeg s[3];
    int count = 0;
    PartSegs& add(float* dst, int n, float* dst2 = nullptr) {
        s[count++] = PartSeg{dst, dst2, n};
        return *this;
    }
    int total() const {
        int n = 0;
        for (int k = 0; k < count; ++k) n += s[k].n;
        return n;
    }
};

struct RowCount {
    const int32_t* ptr;  // device row count (edges) or nullptr
    int fixed;           // host row count when ptr == nullptr
    int cap;             // buffer capacity in rows
};

}  // namespace gcbf
