// gemm_tc_prod.cuh -- tensor-core GEMMs whose A operand is PRODUCED inside the kernel (rollout / inference
// path), so the per-edge inputs never round-trip through HBM and a launch disappears:
//
//   A[e, :] = relu(feat_e @ W1[:ed] + W1[ed + sender_type] + W1[ed+3+2] + b1)   (edge_l1_kernel)
//   feat_e from agent / goal / hit states through the receiver-grouped edge lists
//
// Each consumer thread computes the elements of its own register A fragment (two edge rows, 4 columns per k8 step),
// splits them into tf32 hi / lo and feeds them to the register-A form of wgmma; B (weights, pre-split) arrives by TMA.
#pragma once
#include "gemm_tc.cuh"
#include "gnn.cuh"
#include "internal.cuh"

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

// edge message GEMM + chained gate GEMM (see ChainArgs).  Barriers: full / empty = the 3-stage ring of W23 planes;
// main_done = both warpgroups' main-loop MMAs retired (stage 2 free for the gate weights); b2_full / b2_empty = the two
// gate-weight slots; t2f = the chained GEMM retired (the stages may be refilled for the next tile).
template <int KIND>
__global__ void __launch_bounds__(THREADS_NN, 1)
edge_chain_kernel(const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
                  const __grid_constant__ CUtensorMap tmB2h, const __grid_constant__ CUtensorMap tmB2l,
                  const __grid_constant__ ProdArgs pa, const float* __restrict__ bias, float* __restrict__ C,
                  const int32_t* __restrict__ m_ptr, const int m_cap, const ChainArgs ch) {
    constexpr int ED = EnvTraits<KIND>::ED;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align1024(smem_raw);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STG);
    uint64_t* full = bars;                 // [3]
    uint64_t* empty = bars + 3;            // [3]
    uint64_t* b2_full = bars + 6;          // [2]
    uint64_t* b2_empty = bars + 8;         // [2]
    uint64_t* main_done = bars + 10;
    uint64_t* t2f = bars + 11;
    float* sW = reinterpret_cast<float*>(smem + STAGES * STG + 256);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < 3; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], CONSUMERS);
        }
        for (int i = 0; i < 2; ++i) {
            mbar_init(&b2_full[i], 1);
            mbar_init(&b2_empty[i], CONSUMERS);
        }
        mbar_init(main_done, CONSUMERS);
        mbar_init(t2f, CONSUMERS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    load_l1_table<ED>(sW, pa.W1, pa.b1, threadIdx.x, blockDim.x);
    __syncthreads();
    const int M = min(*m_ptr, m_cap);
    const int n_tiles = (M + BM - 1) / BM;

    if (warp == 8) {
        if (lane == 0) {
            uint32_t it = 0, tc_ = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tc_) {
                if (tc_ > 0) mbar_wait(t2f, (tc_ - 1) & 1);       // the previous tile's chained GEMM still reads the stages
                for (int kb = 0; kb < 8; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
                    uint8_t* st = smem + s * STG;
                    mbar_expect_tx(&full[s], 2 * PLANE);
                    tma_load_2d(st + 2 * PLANE, &tmBh, &full[s], kb * BK, 0);
                    tma_load_2d(st + 3 * PLANE, &tmBl, &full[s], kb * BK, 0);
                }
                mbar_wait(main_done, tc_ & 1);                    // main-loop MMAs retired: stage 2 is free
                for (int kb2 = 0; kb2 < 4; ++kb2) {
                    const uint32_t j2 = tc_ * 4 + kb2, slot = j2 & 1, use = j2 >> 1;
                    mbar_wait(&b2_empty[slot], (use & 1) ^ 1);
                    uint8_t* sl = smem + 2 * STG + slot * 32768;
                    mbar_expect_tx(&b2_full[slot], 32768);
                    tma_load_2d(sl, &tmB2h, &b2_full[slot], kb2 * BK, 0);
                    tma_load_2d(sl + 16384, &tmB2l, &b2_full[slot], kb2 * BK, 0);
                }
            }
        }
        return;
    }
    const int g = warp >> 2, wt = threadIdx.x & 127;
    const int r = 64 * g + frag_row0(wt);      // the thread's fragment rows r, r + 8 of the tile
    const int rs = r + 8 * setup_row(lane);    // ... and the one it sets up
    uint32_t it = 0, tc_ = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++tc_) {
        const int m0 = tile * BM;
        float fs[ED], f[2][ED];
        int ss, stype[2];
        edge_row_setup<KIND>(pa, m0 + rs, m0 + rs < M, fs, ss);
        share_rows<ED>(fs, ss, lane, f, stype);
        const bool ok[2] = {m0 + r < M, m0 + r + 8 < M};
        float d[64];
        edge_tile_mainloop<ED>(d, smem, full, empty, it, lane, ok, sW, f, stype);
        mbar_arrive(main_done);
        bar_consumers();                       // both warpgroups' main loops retired: the hand-over may overwrite stages 0-1
        drain_msg(d, smem, g, wt, bias, C + (size_t)m0 * 128, M - m0);
        fence_async_smem();
        bar_wg(g);                             // the chained GEMM of warpgroup g reads its own hand-over rows only
        float d2[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) d2[i] = 0.f;
        for (int kb2 = 0; kb2 < 4; ++kb2) {
            const uint32_t j2 = tc_ * 4 + kb2, slot = j2 & 1, use = j2 >> 1;
            mbar_wait(&b2_full[slot], use & 1);
            wg_fence();
            chain_kblock(d2, smem, g, kb2, slot);
            wg_commit();
            wg_wait<0>();
            mbar_arrive(&b2_empty[slot]);
        }
        float q[2][1];
        frag_relu_dot<1>(d2, ch.bias_g, ch.avec, 1, 1, wt, q);
        if ((lane & 3) == 0) {
            const int rr = m0 + 64 * g + frag_row0(wt);
            if (rr < M) ch.logits[rr] = q[0][0] + ch.cst[0];
            if (rr + 8 < M) ch.logits[rr + 8] = q[1][0] + ch.cst[0];
        }
        mbar_arrive(t2f);
    }
}

constexpr int PROD_SMEM = STAGES * STG + 256 + L1_FLOATS * 4 + 1024;

// MSG[e, :128] = relu-layer-1(edge e) @ W23 + b23: edge_l1 producer + folded message GEMM (K = 256, N = 128), with the
// gate layer (K = N = 128, weights gate_Bt_*) and its folded gate vector chained in the same kernel: the logits are
// written to chain.logits.
inline int32_t launch_edge_msg(const gcbf_env_desc* d, const float* W1, const float* b1, const GraphRefs& g,
                               int clip_all, const float* Bt_hi, const float* Bt_lo, const float* bias, float* msg,
                               cudaStream_t st, const float* gate_Bt_hi, const float* gate_Bt_lo,
                               const ChainArgs& chain) {
    if (!g.counters) {
        set_error("launch_edge_msg: the chained gate GEMM needs the device edge counter");
        return -1;
    }
    ProdArgs pa;
    memset(&pa, 0, sizeof(pa));
    pa.d = *d;
    pa.W1 = W1; pa.b1 = b1; pa.agent = g.agent; pa.goal = g.goal; pa.hits = g.hits;
    pa.edge_recv = g.edge_recv; pa.edge_src = g.edge_src; pa.clip_all = clip_all;
    const int K = 256, N = 128;
    CUtensorMap tmB, tmBl, tmG, tmGl;
    if (int32_t r = make_map(&tmB, Bt_hi, N, K, N)) return r;
    if (int32_t r = make_map(&tmBl, Bt_lo, N, K, N)) return r;
    if (int32_t r = make_map(&tmG, gate_Bt_hi, 128, 128, 128)) return r;
    if (int32_t r = make_map(&tmGl, gate_Bt_lo, 128, 128, 128)) return r;
    const int grid = min((d->edge_cap + BM - 1) / BM, sm_count());
    GCBF_DISPATCH_ENV(d->env_kind, {
        auto kern = edge_chain_kernel<KIND>;
        static bool attr_done = false;
        if (!attr_done) {
            cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, PROD_SMEM);
            attr_done = true;
        }
        kern<<<grid, THREADS_NN, PROD_SMEM, st>>>(tmB, tmBl, tmG, tmGl, pa, bias, msg, g.counters, d->edge_cap, chain);
        count_launch();
        return check_launch("edge_chain_kernel");
    });
    return -1;
}

}  // namespace tc
}  // namespace gcbf
