// gemm_tc.cuh -- Hopper tensor-core GEMM for the dense MLP layers: wgmma.mma_async (tf32) with fp32 operands split
// as x = hi + lo (3xTF32: hi*hi + hi*lo + lo*hi, fp32 accumulation in registers), operands in shared memory in the
// K-major SWIZZLE_128B layout, staged by TMA through an mbarrier pipeline.
//
//   C[M,N] = epi( A[M,K] @ Bt[N,K]^T )        A, Bt row-major fp32 (both "K-major")
//
// Accuracy: each product carries a relative error ~2^-21 (the dropped lo*lo term and the tf32
// truncation of lo), i.e. fp32-class results (tests: <= 2e-6 relative to |A||B|), which keeps the
// <= 1e-5 parity bar of the GNN outputs -- a single-pass TF32/BF16 MMA (2^-11 / 2^-8) would not.
//
// CTA layout of the kernels here (288 threads): warps 0-7 are two consumer warpgroups, warpgroup g owning rows
// [64 g, 64 g + 64) of a 128 x 128 output tile (one m64n128k8 accumulator: 64 registers per thread); warp 8 issues
// the TMA loads.  The consumers hold A in registers: each thread splits its own A fragment into tf32 hi / lo (the
// weight planes arrive pre-split in shared memory) and feeds it to the register-A form of wgmma -- the split of k8
// step j + 1 overlaps the MMAs of step j -- and runs the epilogue straight from the accumulator registers.
// Persistent tile loop; M may come from a device counter (edge count) so the launch is CUDA-graph friendly.
// gemm_tn_tc_kernel (weight gradient) is described at its definition.
// This header holds the device code the kernels share with the persistent rollout kernel and the tensor-map helpers;
// the kernels and their launchers are in dense.cu.
#pragma once
#include <cuda.h>

#include <cstdlib>

#include "common.cuh"
#include "gemm.cuh"

namespace gcbf {
namespace tc {

constexpr int BM = 128;                   // rows per tile (two m64 warpgroups)
constexpr int BN = 128;                   // columns per tile (wgmma n128)
constexpr int BK = 32;                    // fp32 elements per k-block = one 128-byte swizzle row
constexpr int WK = 8;                     // tf32: 32 bytes of K per MMA
constexpr int CONSUMERS = 256;            // two warpgroups
constexpr int THREADS_NN = CONSUMERS + 32;
constexpr int PLANE = BM * BK * 4;        // 16 KB: one hi or lo plane of a 128-row k-block
constexpr int STG = 4 * PLANE;            // pipeline stage: A (fp32) | (unused) | B hi | B lo
constexpr int STAGES = 3;
constexpr int WG_ROWS_BYTES = 64 * 128;   // the 64 rows of one warpgroup inside a plane

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// The dynamic shared-memory window rounded up to the 1024-byte alignment SWIZZLE_128B needs.  The result is the
// __shared__ array plus a byte offset: a round trip through uintptr_t would erase its address space, and every access
// through it would become a generic 64-bit LD / ST instead of LDS / STS.
__device__ __forceinline__ uint8_t* smem_align1024(uint8_t* raw) { return raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug must end in a trap (error return), never in a hung GPU.  The bound is wall time
// (%globaltimer, ns), 60 s: every wait of a correct kernel here is a few microseconds, so even a 1000x slowdown under
// compute-sanitizer stays far below it.
constexpr unsigned long long MBAR_TIMEOUT_NS = 60ull * 1000000000ull;
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    unsigned long long t0 = 0;
    while (true) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (done) break;
        const unsigned long long t = global_ns();         // the clock is read only once the barrier is not ready
        if (t0 == 0) t0 = t;
        else if (t - t0 > MBAR_TIMEOUT_NS) __trap();
    }
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// generic-proxy shared-memory writes -> reads by the async proxy (wgmma operands, TMA)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barriers of the consumers: 1 = both warpgroups, 2 + g = warpgroup g
__device__ __forceinline__ void bar_consumers() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void bar_wg(int g) { asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory"); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA layout): start >> 4 [0,14) | LBO >> 4 [16,30)
// (unused for swizzled K-major, 1) | SBO >> 4 [32,46) = 1024 B between 8-row groups | layout [62,64) = 1 (128B swizzle).
// Tile bases are 1024-byte aligned; the K offset of an MMA inside the 128-byte row is added to the start address.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

#define GCBF_ACC8(i)                                                                                               \
    "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), \
        "+f"(d[i + 7])
// D[64 x 128] (+)= A[64 x 8] B[8 x 128], tf32 operands from shared memory, fp32 accumulator in registers
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n"
        "}\n"
        : GCBF_ACC8(0), GCBF_ACC8(8), GCBF_ACC8(16), GCBF_ACC8(24), GCBF_ACC8(32), GCBF_ACC8(40), GCBF_ACC8(48),
          GCBF_ACC8(56)
        : "l"(da), "l"(db), "r"(accumulate)
        : "memory");
}
// D[64 x 128] (+)= A[64 x 8] B[8 x 128], A (tf32 bit patterns) from registers, B from shared memory.  A fragment of
// thread `lane` of warp w of the warpgroup (PTX ISA, wgmma .tf32 register fragment of A): a[0] = (row 16 w + lane / 4,
// column lane % 4), a[1] = (row + 8, same column), a[2] = (same row, column + 4), a[3] = (row + 8, column + 4).  The
// registers are read asynchronously: they must stay unchanged until a wgmma.wait_group retires the MMA.
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1;\n"
        "}\n"
        : GCBF_ACC8(0), GCBF_ACC8(8), GCBF_ACC8(16), GCBF_ACC8(24), GCBF_ACC8(32), GCBF_ACC8(40), GCBF_ACC8(48),
          GCBF_ACC8(56)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate)
        : "memory");
}
#undef GCBF_ACC8

// 12 MMAs of one 32-wide k-block of a 3xTF32 product (small terms first): a_* = the warpgroup's 64 rows, b_* = 128 rows
__device__ __forceinline__ void mma_kblock(float (&d)[64], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                           bool first) {
#pragma unroll
    for (int k = 0; k < BK / WK; ++k) {
        const uint32_t koff = k * WK * 4;   // bytes inside the 128-byte swizzle row
        wgmma_tf32(d, make_desc(a_lo + koff), make_desc(b_hi + koff), (first && k == 0) ? 0u : 1u);
        wgmma_tf32(d, make_desc(a_hi + koff), make_desc(b_lo + koff), 1u);
        wgmma_tf32(d, make_desc(a_hi + koff), make_desc(b_hi + koff), 1u);
    }
}

// The 3 MMAs of one k8 step of a 3xTF32 product, A from registers, in the order of mma_kblock: lo * Bhi, hi * Blo,
// hi * Bhi.  b_hi / b_lo: shared-memory address of the k8 step's B columns (k-block plane + 32 bytes per k8 step).
// The lo MMA and the two hi MMAs are committed as two groups, so the wg_wait<1> that follows in the main loops retires
// the lo group of this step (and everything before it): the next step's fragment is then produced while only the 4 hi
// registers of this step are in flight, which keeps the persistent rollout kernel within its 128 registers.
__device__ __forceinline__ void mma_k8_rs(float (&d)[64], const uint32_t (&a_hi)[4], const uint32_t (&a_lo)[4],
                                          uint32_t b_hi, uint32_t b_lo, bool first) {
    wg_fence();                                // the fragment registers were just written
    wgmma_tf32_rs(d, a_lo, make_desc(b_hi), first ? 0u : 1u);
    wg_commit();
    wgmma_tf32_rs(d, a_hi, make_desc(b_lo), 1u);
    wgmma_tf32_rs(d, a_hi, make_desc(b_hi), 1u);
    wg_commit();
}

// Accumulator fragment of an m64n128 wgmma: element i of thread t of the warpgroup (warp w = t / 32, lane l) holds
// row 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.
__device__ __forceinline__ int frag_row0(int wt) { return 16 * (wt >> 5) + ((wt & 31) >> 2); }
__device__ __forceinline__ int frag_col(int wt, int i) { return 8 * (i >> 2) + 2 * (wt & 3) + (i & 1); }

// hi = rn_tf32(x), lo = rn_tf32(x - hi): |x - hi - lo| <= 2^-24 |x|.
__device__ __forceinline__ void split_tf32(const float4& v, float4& h, float4& l) {
    h.x = rn_tf32(v.x); h.y = rn_tf32(v.y); h.z = rn_tf32(v.z); h.w = rn_tf32(v.w);
    l.x = rn_tf32(v.x - h.x); l.y = rn_tf32(v.y - h.y); l.z = rn_tf32(v.z - h.z); l.w = rn_tf32(v.w - h.w);
}
// the same split of a register A fragment (wgmma_tf32_rs operands)
__device__ __forceinline__ void split_frag(const float (&v)[4], uint32_t (&h)[4], uint32_t (&l)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float x = rn_tf32(v[i]);
        h[i] = __float_as_uint(x);
        l[i] = __float_as_uint(rn_tf32(v[i] - x));
    }
}
// byte offset of 16-byte chunk c (columns 4c .. 4c + 3 of a k-block) of row r in a K-major SWIZZLE_128B plane
__device__ __forceinline__ int swz(int r, int c) { return r * 128 + ((c ^ (r & 7)) << 4); }

// relu(acc + bias) . vec over the tile's 128 columns, for the two rows of the thread (out[h]: row frag_row0 + 8 h).
// Each thread chains its 32 columns in column order, then the 4 threads of a row add their partial sums (butterfly:
// the same bits in all four).  Every kernel that produces a gate logit or output-layer sum uses this order.
template <int NQ>
__device__ __forceinline__ void frag_relu_dot(const float (&d)[64], const float* bias, const float* vec, int vstride,
                                              int nq, int wt, float (&out)[2][NQ]) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < NQ; ++q) out[h][q] = 0.f;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        const int c = frag_col(wt, i);
        const float x = fmaxf(d[i] + bias[c], 0.f);
#pragma unroll
        for (int q = 0; q < NQ; ++q)
            if (q < nq) out[(i >> 1) & 1][q] = fmaf(x, vec[c * vstride + q], out[(i >> 1) & 1][q]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
            out[h][q] += __shfl_xor_sync(0xffffffffu, out[h][q], 1);
            out[h][q] += __shfl_xor_sync(0xffffffffu, out[h][q], 2);
        }
}

// Main loop of one 128 x 128 tile whose A arrives by TMA (stage layout A | (unused) | B hi | B lo, A as plain fp32):
// each consumer thread loads its A fragment of a k8 step from the fp32 tile -- for one k8 step the 8 rows of a quad
// column sit in 8 distinct 16-byte chunks of the swizzled rows, so the loads are free of bank conflicts -- splits it
// into tf32 hi / lo in registers and issues the step's 3 MMAs (mma_k8_rs): the split of step j + 1 overlaps the hi
// MMAs of step j, and 12 A registers are live.  `empty` counts the 256 consumer threads.
__device__ __forceinline__ void tma_a_mainloop(float (&d)[64], uint8_t* smem, uint64_t* full, uint64_t* empty,
                                               uint32_t& it, int nkb, int g, int wt) {
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    const int r = frag_row0(wt);               // fragment rows r, r + 8 of the warpgroup's 64; column wt % 4 (+ 4)
    // byte offset of (row r, column wt % 4) in chunk 0 of the swizzled tile; chunk c is at off ^ (c << 4) (swz)
    const uint32_t off = g * WG_ROWS_BYTES + swz(r, 0) + (wt & 3) * 4;
    for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = it % STAGES;
        mbar_wait(&full[s], (it / STAGES) & 1);
        // the chunk XOR is applied to the stage-dependent offset, so the 16 fragment addresses of a k-block are not
        // loop-invariant registers
        const uint32_t a = s * STG + off;
        const uint32_t b_hi = smem_u32(smem + s * STG) + 2 * PLANE;
#pragma unroll
        for (int k = 0; k < BK / WK; ++k) {
            const uint32_t o0 = a ^ (2 * k << 4), o1 = a ^ ((2 * k + 1) << 4);
            const float v[4] = {*reinterpret_cast<const float*>(smem + o0),
                                *reinterpret_cast<const float*>(smem + o0 + 8 * 128),
                                *reinterpret_cast<const float*>(smem + o1),
                                *reinterpret_cast<const float*>(smem + o1 + 8 * 128)};
            uint32_t ah[4], al[4];
            split_frag(v, ah, al);
            mma_k8_rs(d, ah, al, b_hi + k * WK * 4, b_hi + PLANE + k * WK * 4, kb == 0 && k == 0);
            wg_wait<1>();                      // all but this step's hi MMAs retired; at k = 0 that includes the last
            if (k == 0 && kb > 0) mbar_arrive(&empty[(it - 1) % STAGES]);   // MMAs of k-block kb - 1
        }
    }
    wg_wait<0>();
    mbar_arrive(&empty[(it - 1) % STAGES]);
}

// ---- host side ----------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            p = nullptr;
        return (EncodeTiledFn)p;
    }();
    return fn;
}

// 2-D fp32 [rows, cols] tensor with row stride ld floats, box = [box_rows, box_cols]
inline int32_t make_map_box(CUtensorMap* map, const float* ptr, int rows, int cols, int ld, int box_rows, int box_cols,
                            CUtensorMapSwizzle swz) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled unavailable");
        return -2;
    }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d ld=%d", (int)r, rows, cols, ld);
        return -2;
    }
    return 0;
}
// row-major [rows, cols] tensor, box = [box_rows, BK cols] with the 128-byte swizzle the MMA descriptors expect
inline int32_t make_map(CUtensorMap* map, const float* ptr, int rows, int cols, int box_rows) {
    return make_map_box(map, ptr, rows, cols, cols, box_rows, BK, CU_TENSOR_MAP_SWIZZLE_128B);
}
// `depth` row-major [rows, cols] tensors `stride` floats apart as one 3-D map (the stack index outermost, a multiple of
// 4 floats), box = [1, box_rows, BK cols] with make_map's swizzle: a load with third coordinate k lands the same tile
// of tensor k that make_map's load lands of tensor 0
inline int32_t make_map_stack(CUtensorMap* map, const float* ptr, int rows, int cols, int box_rows, int depth,
                              int64_t stride) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled unavailable");
        return -2;
    }
    cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)depth};
    cuuint64_t strides[2] = {(cuuint64_t)cols * 4, (cuuint64_t)stride * 4};
    cuuint32_t box[3] = {(cuuint32_t)BK, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d depth=%d stride=%lld", (int)r, rows, cols, depth,
                  (long long)stride);
        return -2;
    }
    return 0;
}

}  // namespace tc
}  // namespace gcbf
