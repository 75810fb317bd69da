// gemm_tc_prod.cuh -- tensor-core GEMMs whose A operand is PRODUCED inside the kernel (rollout / inference
// path), so the per-edge inputs never round-trip through HBM and a launch disappears:
//
//   A[e, :] = relu(feat_e @ W1[:ed] + W1[ed + sender_type] + W1[ed+3+2] + b1)   (edge_l1_kernel)
//   feat_e from agent / goal / hit states through the receiver-grouped edge lists
//
// Each consumer thread computes the elements of its own register A fragment (two edge rows, 4 columns per k8 step),
// splits them into tf32 hi / lo and feeds them to the register-A form of wgmma; B (weights, pre-split) arrives by TMA.
// The device functions here are shared by edge_chain_kernel (gnn.cu) and the persistent rollout kernel.
#pragma once
#include "gemm_tc.cuh"
#include "gnn.cuh"

namespace gcbf {
namespace tc {

struct ProdArgs {
    gcbf_env_desc d;
    const float *W1, *b1, *agent, *goal, *hits;
    const int32_t *edge_recv, *edge_src;
    int clip_all;
};

// edge_chain_kernel: a second GEMM is chained onto the message tile while it is still on the SM --
//   logit[m] = relu(MSG[m, :128] @ A1 + b_g) . avec + c            (gate layer + folded gate vector, gnn.py:64-67)
// The message tile is handed over in shared memory (tf32 hi / lo planes in the K-major SWIZZLE_128B layout, 4 k-blocks
// of 32 = 128 KB over the drained pipeline stages 0-1) and the gate weights stream through the third stage (two 32 KB
// slots).  One launch (and one round trip of MSG through L2) less per env-step.
struct ChainArgs {
    const float* bias_g;   // [128] gate hidden-layer bias
    const float* avec;     // [128] folded gate vector
    const float* cst;      // [1]   folded gate constant
    float* logits;         // [M]   out
};

constexpr int L1_FLOATS = 9 * 256;   // message layer 1 in shared memory: W1[:ED] and the per-sender-type bias rows

// Position of column c in a row of the layer-1 table: inside each group of 8 columns, c and c + 4 are neighbours
// (8 a + 4 h + j -> 8 a + 2 j + h), so the two columns of a k8 step's A fragment are one 8-byte load.
__device__ __forceinline__ int l1_pos(int c) { return (c & ~7) | ((c & 3) << 1) | ((c >> 2) & 1); }

// W1[:ED] and the per-sender-type bias table sW[(ED + t) * 256 + l1_pos(c)] = W1[ED + t] + W1[ED + 3 + 2] + b1
template <int ED>
__device__ __forceinline__ void load_l1_table(float* sW, const float* W1, const float* b1, int tid, int nthreads) {
    for (int i = tid; i < ED * 256; i += nthreads) sW[(i & ~255) + l1_pos(i & 255)] = W1[i];
    for (int i = tid; i < 3 * 256; i += nthreads) {
        const int t = i / 256, c = i % 256;
        sW[(ED + t) * 256 + l1_pos(c)] = W1[(ED + t) * 256 + c] + W1[(ED + 3 + 2) * 256 + c] + b1[c];
    }
}

// message layer 1 at columns n0 + j and n0 + j + 4 (n0 = 8 k8-steps, j = lane % 4) of the thread's two fragment rows
// (features f[h], sender-type table row bias[h], h = 0: row frag_row0, h = 1: row + 8; rows that are not ok give 0)
// -> the tf32 hi / lo register A fragment of that k8 step
template <int ED>
__device__ __forceinline__ void produce_l1_k8(uint32_t (&ah)[4], uint32_t (&al)[4], int n0, int j, const bool (&ok)[2],
                                              const float* sW, const float* const (&bias)[2], const float (&f)[2][ED]) {
    const int p = n0 + 2 * j;                  // l1_pos(n0 + j); l1_pos(n0 + j + 4) = p + 1
    float2 y[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) y[h] = *reinterpret_cast<const float2*>(bias[h] + p);
#pragma unroll
    for (int q = 0; q < ED; ++q) {
        const float2 w = *reinterpret_cast<const float2*>(sW + q * 256 + p);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            y[h].x = fmaf(f[h][q], w.x, y[h].x);
            y[h].y = fmaf(f[h][q], w.y, y[h].y);
        }
    }
    const float v[4] = {ok[0] ? fmaxf(y[0].x, 0.f) : 0.f, ok[1] ? fmaxf(y[1].x, 0.f) : 0.f,
                        ok[0] ? fmaxf(y[0].y, 0.f) : 0.f, ok[1] ? fmaxf(y[1].y, 0.f) : 0.f};
    split_frag(v, ah, al);
}

// message tile of warpgroup g -> global rows (bias added; tile row r lands at msg + r * 128, rows >= n_valid skipped)
// and -> shared memory as the tf32 hi / lo A operand of the chained gate GEMM (k-block c / 32 at smem + 32 KB (c / 32):
// hi plane, then lo plane)
__device__ __forceinline__ void drain_msg(const float (&d)[64], uint8_t* smem, int g, int wt, const float* bias,
                                          float* msg, int n_valid) {
    const int r0 = 64 * g + frag_row0(wt);
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
        const int r = r0 + 8 * ((i >> 1) & 1);
        const int c = frag_col(wt, i);
        const float2 o = make_float2(d[i] + bias[c], d[i + 1] + bias[c + 1]);
        if (r < n_valid) *reinterpret_cast<float2*>(msg + (size_t)r * 128 + c) = o;
        const float2 h = make_float2(rn_tf32(o.x), rn_tf32(o.y));
        const float2 l = make_float2(rn_tf32(o.x - h.x), rn_tf32(o.y - h.y));
        const int off = (c >> 5) * 32768 + swz(r, (c & 31) >> 2) + (c & 3) * 4;
        *reinterpret_cast<float2*>(smem + off) = h;
        *reinterpret_cast<float2*>(smem + off + 16384) = l;
    }
}

// the 3 x 4 chained gate MMAs of warpgroup g over the hand-over planes (k-block kb2) and a gate-weight slot
__device__ __forceinline__ void chain_kblock(float (&d)[64], uint8_t* smem, int g, int kb2, int slot) {
    const uint32_t a_hi = smem_u32(smem + kb2 * 32768) + g * WG_ROWS_BYTES;
    const uint32_t b_hi = smem_u32(smem + 2 * STG + slot * 32768);
    mma_kblock(d, a_hi, a_hi + 16384, b_hi, b_hi + 16384, kb2 == 0);
}

// edge rows of tile `tile`: per-row edge features, sender type
template <int KIND>
__device__ __forceinline__ void edge_row_setup(const ProdArgs& pa, int m, bool row_ok, float (&f)[EnvTraits<KIND>::ED],
                                               int& stype) {
    using T = EnvTraits<KIND>;
    constexpr int ED = T::ED, SD = T::SD;
    const int A_tot = pa.d.n_graphs * pa.d.n_agents;
#pragma unroll
    for (int c = 0; c < ED; ++c) f[c] = 0.f;
    stype = 0;
    if (row_ok) {
        const int a = min(max(pa.edge_recv[m], 0), A_tot - 1);
        const int code = min(pa.edge_src[m], A_tot - 1);
        float er[ED], es[ED], coef, nrm;
        edge_state_dev<KIND>(pa.agent + (size_t)a * SD, er);
        sender_state_dev<KIND>(code, a, pa.d.n_hits, pa.agent, pa.goal, pa.hits, es);
        edge_feat_dev<KIND>(er, es, pa.clip_all || code == -1, pa.d.comm_radius, f, &coef, &nrm);
        stype = (code >= 0) ? 2 : ((code == -1) ? 1 : 0);
    }
}

// Row set-up of the two fragment rows of a thread (h = 0: frag_row0, h = 1: + 8): lanes 4 i, 4 i + 1 of a quad set up
// row h = 0, lanes 4 i + 2, 4 i + 3 row h = 1 (setup_row), and share_rows hands both to the whole quad.
__device__ __forceinline__ int setup_row(int lane) { return (lane >> 1) & 1; }
template <int ED>
__device__ __forceinline__ void share_rows(const float (&fs)[ED], int ss, int lane, float (&f)[2][ED], int (&stype)[2]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int src = (lane & ~3) | (2 * h);
#pragma unroll
        for (int q = 0; q < ED; ++q) f[h][q] = __shfl_sync(0xffffffffu, fs[q], src);
        stype[h] = __shfl_sync(0xffffffffu, ss, src);
    }
}

// main loop of an edge tile: 8 k-blocks of message layer 1 produced in-kernel x W23 (K = 256, N = 128), one k8 step
// at a time as in tma_a_mainloop; the first k8 step of a k-block is produced before the wait for its weights
template <int ED>
__device__ __forceinline__ void edge_tile_mainloop(float (&d)[64], uint8_t* smem, uint64_t* full, uint64_t* empty,
                                                   uint32_t& it, int lane, const bool (&ok)[2], const float* sW,
                                                   const float (&f)[2][ED], const int (&stype)[2]) {
    const float* const bias[2] = {sW + (ED + stype[0]) * 256, sW + (ED + stype[1]) * 256};
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    for (int kb = 0; kb < 8; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t b_hi = smem_u32(smem + s * STG) + 2 * PLANE;
#pragma unroll
        for (int k = 0; k < BK / WK; ++k) {
            uint32_t ah[4], al[4];
            produce_l1_k8<ED>(ah, al, kb * BK + k * WK, lane & 3, ok, sW, bias, f);
            if (k == 0) mbar_wait(&full[s], (it / STAGES) & 1);
            mma_k8_rs(d, ah, al, b_hi + k * WK * 4, b_hi + PLANE + k * WK * 4, kb == 0 && k == 0);
            wg_wait<1>();                      // all but this step's hi MMAs retired; at k = 0 that includes the last
            if (k == 0 && kb > 0) mbar_arrive(&empty[(it - 1) % STAGES]);   // MMAs of k-block kb - 1
        }
    }
    wg_wait<0>();
    mbar_arrive(&empty[(it - 1) % STAGES]);
}

}  // namespace tc
}  // namespace gcbf
