// translayout.cuh -- the GEMM weights of a network in the layouts the GEMMs read: transposed fp32 copies (TransLayout,
// the backward-data operands of the SIMT path) and tf32 hi / lo planes (PlaneLayout, the tensor-core path).
#pragma once
#include "common.cuh"

namespace gcbf {

static __global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[i][threadIdx.x] = in[(size_t)r * cols + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) out[(size_t)c * rows + r] = tile[threadIdx.x][i];
    }
}

static int32_t launch_transpose(const float* in, float* out, int rows, int cols, cudaStream_t st) {
    dim3 grid((cols + 31) / 32, (rows + 31) / 32), block(32, 8);
    transpose_kernel<<<grid, block, 0, st>>>(in, out, rows, cols);
    count_launch();
    return check_launch("transpose_kernel");
}

// Transposed copies of the GEMM weights of one network (backward-data operands).
struct TransLayout {
    int w[12];
    int total;
};
static TransLayout make_trans_layout(const ParamLayout& L) {
    TransLayout T;
    int off = 0;
    for (int i = 0; i < 12; ++i) {
        T.w[i] = off;
        int rows = L.in[i];
        if (i == L_UPD0) rows = 128;  // only the aggregated-message rows 3..130
        if (i == L_MSG0 || i == L_GATE || i == L_OUT) { T.w[i] = -1; continue; }
        off += rows * L.out[i];
    }
    T.total = off;
    return T;
}
static int32_t build_transposes(const ParamLayout& L, const TransLayout& T, const float* P, float* PT, cudaStream_t st) {
    for (int i = 0; i < 12; ++i) {
        if (T.w[i] < 0) continue;
        const float* src = P + L.w[i] + (i == L_UPD0 ? 3 * 256 : 0);
        const int rows = (i == L_UPD0) ? 128 : L.in[i];
        if (int32_t rc = launch_transpose(src, PT + T.w[i], rows, L.out[i], st)) return rc;
    }
    return 0;
}

// tf32 hi / lo planes of the GEMM weights of an n_layers-deep network (gcbf_prepare_params_l): the one prepared-weights
// format of the unfolded network.  Slot i < 12 is Dense layer i of DeepLayout layer[l] (L_MSG0 holds Ws, DEEP_WR holds
// Wr at l >= 1; the head lives in layer 0's slots); layer 0's update/Dense_0 is its rows 3..130, which multiply the
// aggregate.  src / rows / cols: the weight in the parameters.  Per slot:
//   t[l][i]: W^T hi, then W^T lo at + rows * cols (K-major B operand of the forward); -1: not a GEMM operand;
//   s[i] (n_layers = 1 only, else -1): W hi, then W lo (K-major B operand of the backward-data GEMM dX = dY W^T).
constexpr int DEEP_WR = 12;
struct PlaneLayout {
    int t[GCBF_MAX_LAYERS][13], src[GCBF_MAX_LAYERS][13], rows[GCBF_MAX_LAYERS][13], cols[GCBF_MAX_LAYERS][13];
    int s[13];
    int total;
};
inline PlaneLayout make_plane_layout(const DeepLayout& D, int ed) {
    PlaneLayout Q;
    int off = 0;
    for (int l = 0; l < D.n_layers; ++l) {
        const ParamLayout& L = D.layer[l];
        for (int i = 0; i < 13; ++i) {
            int src = -1, rows = 0;
            if (i == L_MSG0 || i == DEEP_WR) {
                if (l > 0) { src = L.w[L_MSG0] + (ed + (i == DEEP_WR ? 128 : 0)) * 256; rows = 128; }
            } else if (i == L_UPD0) {
                src = L.w[i] + (l == 0 ? 3 * 256 : 0);
                rows = l == 0 ? 128 : 256;
            } else if (i == L_HEAD0 || i == L_HEAD1) {
                if (l == 0) { src = L.w[i]; rows = L.in[i]; }
            } else if (i != L_GATE && i != L_OUT) {
                src = L.w[i];
                rows = L.in[i];
            }
            const int cols = (i == DEEP_WR) ? 256 : L.out[i];
            Q.src[l][i] = src;
            Q.rows[l][i] = rows;
            Q.cols[l][i] = cols;
            Q.t[l][i] = src < 0 ? -1 : off;
            if (src >= 0) off += 2 * rows * cols;
            if (l > 0) continue;
            Q.s[i] = (src < 0 || D.n_layers > 1) ? -1 : off;
            if (Q.s[i] >= 0) off += 2 * rows * cols;
        }
    }
    Q.total = off;
    return Q;
}

}  // namespace gcbf
