// gemm.cuh -- fp32 SIMT GEMM family for the dense MLP layers of the GNN (strict-fp32 parity
// path; SURVEY 8c: fp32 FMA is the parity default).  All operands row-major, contiguous.
//
//   gemm_nn : C[M,N] = epi(A[M,K] @ B[K,N])     forward (B = W) and backward-data (B = W^T)
//   gemm_tn : C[K1,N] += sum_m w[m] * X[m,K1] * dY[m,N]   backward-weight (split over M, ordered partial sums)
//   colsum  : db[N] += sum_m w[m] * dY[m,N]
//
// No float atomics: a kernel that splits a sum over CTAs writes one partial per CTA to a workspace and
// partial_sum_kernel adds the partials in CTA order, so every result is bit-identical from run to run.
//
// Tiling: CTA tile 128x128, BK = 16, 256 threads, 8x8 register tile per thread split as
// 2x2 blocks of 4x4 (conflict-free LDS.128), register-prefetch double buffering, persistent
// tile loop (grid = k * #SM) so that a device-side row count (edge count) can drive the
// launch inside a CUDA graph.
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

constexpr int GEMM_BM = 128, GEMM_BN = 128, GEMM_BK = 16, GEMM_THREADS = 256;
constexpr int GEMM_LDA = GEMM_BM + 4;  // padded: transposed A tile

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

// dst[i] += sum_{p < P} part[p * stride + i], the p in increasing order: a CTA takes 32 consecutive elements, warp w
// sums the partials p = w, w + 8, ... and warp 0 adds the 8 warp sums in warp order.  P = nparts, or, with a device row
// count, the number of parts that had rows: min(nparts, ceil(M / rows_per_part)) (the other parts wrote nothing).
static __global__ void __launch_bounds__(256)
partial_sum_kernel(const float* __restrict__ part, const int64_t stride, const int nparts, const PartSegs segs,
                   const int n_total, const int32_t* __restrict__ m_ptr, const int m_cap, const int rows_per_part) {
    __shared__ float red[8][32];
    int P = nparts;
    if (m_ptr) {
        const int M = min(*m_ptr, m_cap);
        P = min(P, (M + rows_per_part - 1) / rows_per_part);
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + lane;
    float s = 0.f;
    if (i < n_total) {
#pragma unroll 4
        for (int p = w; p < P; p += 8) s += part[(size_t)p * stride + i];
    }
    red[w][lane] = s;
    __syncthreads();
    if (w != 0 || i >= n_total) return;
    for (int k = 1; k < 8; ++k) s += red[k][lane];
    int j = i;
    for (int k = 0; k < segs.count; ++k) {
        if (j < segs.s[k].n) {
            segs.s[k].dst[j] += s;
            if (segs.s[k].dst2) segs.s[k].dst2[j] += s;
            return;
        }
        j -= segs.s[k].n;
    }
}

inline int32_t launch_partial_sum(const float* part, int64_t stride, int nparts, const PartSegs& segs, cudaStream_t st,
                                  const int32_t* m_ptr = nullptr, int m_cap = 0, int rows_per_part = 1) {
    const int n = segs.total();
    if (n <= 0 || nparts <= 0) return 0;
    partial_sum_kernel<<<(n + 31) / 32, 256, 0, st>>>(part, stride, nparts, segs, n, m_ptr, m_cap, rows_per_part);
    count_launch();
    return check_launch("partial_sum_kernel");
}

template <int EPI, bool ACCUM>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
gemm_nn_kernel(const float* __restrict__ A, const float* __restrict__ B, const float* __restrict__ bias,
               const float* __restrict__ bias2, float* __restrict__ C, const float* __restrict__ aux,
               const int32_t* __restrict__ m_ptr, const int m_fixed, const int m_cap, const int K, const int N) {
    __shared__ __align__(16) float As[2][GEMM_BK][GEMM_LDA];
    __shared__ __align__(16) float Bs[2][GEMM_BK][GEMM_BN];
    int M = m_ptr ? *m_ptr : m_fixed;
    M = min(M, m_cap);
    const int tiles_n = N / GEMM_BN;
    const int tiles_m = (M + GEMM_BM - 1) / GEMM_BM;
    const int tid = threadIdx.x;
    const int ty = tid >> 4, tx = tid & 15;
    // global->smem load assignment
    const int a_row0 = tid >> 2, a_kq = (tid & 3) * 4;          // A: rows a_row0, a_row0+64 ; 4 consecutive k
    const int b_row0 = tid >> 5, b_c4 = (tid & 31) * 4;         // B: k rows b_row0, b_row0+8 ; 4 consecutive n

    for (int tile = blockIdx.x; tile < tiles_m * tiles_n; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * GEMM_BM;
        const int n0 = (tile % tiles_n) * GEMM_BN;
        float acc[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

        float4 ra[2], rb[2];
        auto load_global = [&](int k0) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + a_row0 + h * 64;
                ra[h] = (m < M) ? *reinterpret_cast<const float4*>(A + (size_t)m * K + k0 + a_kq)
                                : make_float4(0.f, 0.f, 0.f, 0.f);
                rb[h] = *reinterpret_cast<const float4*>(B + (size_t)(k0 + b_row0 + h * 8) * N + n0 + b_c4);
            }
        };
        auto store_smem = [&](int buf) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = a_row0 + h * 64;
                As[buf][a_kq + 0][r] = ra[h].x;
                As[buf][a_kq + 1][r] = ra[h].y;
                As[buf][a_kq + 2][r] = ra[h].z;
                As[buf][a_kq + 3][r] = ra[h].w;
                *reinterpret_cast<float4*>(&Bs[buf][b_row0 + h * 8][b_c4]) = rb[h];
            }
        };
        load_global(0);
        store_smem(0);
        __syncthreads();
        const int nk = K / GEMM_BK;
        for (int kt = 0; kt < nk; ++kt) {
            const int buf = kt & 1;
            if (kt + 1 < nk) load_global((kt + 1) * GEMM_BK);
#pragma unroll
            for (int k = 0; k < GEMM_BK; ++k) {
                const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
                const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
                const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
                const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
                const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            }
            if (kt + 1 < nk) {
                store_smem(buf ^ 1);
            }
            __syncthreads();
        }
        // ---- epilogue
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = m0 + ((i < 4) ? (ty * 4 + i) : (64 + ty * 4 + i - 4));
            if (m >= M) continue;
#pragma unroll
            for (int jh = 0; jh < 2; ++jh) {
                const int n = n0 + jh * 64 + tx * 4;
                float4 v = make_float4(acc[i][jh * 4 + 0], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]);
                if (EPI == EPI_BIAS || EPI == EPI_BIAS_RELU) {
                    const float4 bb = *reinterpret_cast<const float4*>(bias + n);
                    v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w;
                    if (bias2) {
                        const float4 b2 = *reinterpret_cast<const float4*>(bias2 + n);
                        v.x += b2.x; v.y += b2.y; v.z += b2.z; v.w += b2.w;
                    }
                    if (EPI == EPI_BIAS_RELU) {
                        v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
                    }
                } else if (EPI == EPI_RELU_MASK) {
                    const float4 mk = *reinterpret_cast<const float4*>(aux + (size_t)m * N + n);
                    v.x = mk.x > 0.f ? v.x : 0.f; v.y = mk.y > 0.f ? v.y : 0.f;
                    v.z = mk.z > 0.f ? v.z : 0.f; v.w = mk.w > 0.f ? v.w : 0.f;
                }
                float4* dst = reinterpret_cast<float4*>(C + (size_t)m * N + n);
                if (ACCUM) {
                    const float4 old = *dst;
                    v.x += old.x; v.y += old.y; v.z += old.z; v.w += old.w;
                }
                *dst = v;
            }
        }
        __syncthreads();
    }
}

// backward-weight: C[K1,N] += sum_m w(m) X[m, K1] dY[m, N]; K1, N multiples of 128.
// grid = (K1/128 * N/128) * splits ; each CTA walks m-chunks {split, split+S, ...}.
// `roww`: optional per-agent weights; `row2agent`: optional row -> agent map (edges -> receiver).
// `part` (splits > 1): the CTA stores its tile to part[split][K1][N] and partial_sum_kernel adds the splits to C;
// otherwise (one split) the CTA adds its tile to C itself.
static __global__ void __launch_bounds__(GEMM_THREADS, 2)
gemm_tn_kernel(const float* __restrict__ X, const int ldx, const float* __restrict__ dY, float* __restrict__ C,
               const float* __restrict__ roww, const int32_t* __restrict__ row2agent,
               const int32_t* __restrict__ m_ptr, const int m_fixed, const int m_cap, const int K1, const int N,
               const int splits, const int n_agents_total, float* __restrict__ part) {
    __shared__ __align__(16) float As[2][GEMM_BK][GEMM_BM];
    __shared__ __align__(16) float Bs[2][GEMM_BK][GEMM_BN];
    int M = m_ptr ? *m_ptr : m_fixed;
    M = min(M, m_cap);
    const int tiles_n = N / GEMM_BN;
    const int tile = blockIdx.x / splits, split = blockIdx.x % splits;
    const int k0 = (tile / tiles_n) * GEMM_BM, n0 = (tile % tiles_n) * GEMM_BN;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const int l_row0 = tid >> 5, l_c4 = (tid & 31) * 4;  // rows l_row0, l_row0+8
    const int n_chunks = (M + GEMM_BK - 1) / GEMM_BK;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    if (split >= n_chunks) return;
    float4 ra[2], rb[2];
    auto load_global = [&](int chunk) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = chunk * GEMM_BK + l_row0 + h * 8;
            if (m < M) {
                ra[h] = *reinterpret_cast<const float4*>(X + (size_t)m * ldx + k0 + l_c4);
                rb[h] = *reinterpret_cast<const float4*>(dY + (size_t)m * N + n0 + l_c4);
                if (roww) {
                    int ag = row2agent ? row2agent[m] : m;
                    ag = min(max(ag, 0), n_agents_total - 1);
                    const float w = roww[ag];
                    rb[h].x *= w; rb[h].y *= w; rb[h].z *= w; rb[h].w *= w;
                }
            } else {
                ra[h] = make_float4(0.f, 0.f, 0.f, 0.f);
                rb[h] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
    };
    auto store_smem = [&](int buf) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            *reinterpret_cast<float4*>(&As[buf][l_row0 + h * 8][l_c4]) = ra[h];
            *reinterpret_cast<float4*>(&Bs[buf][l_row0 + h * 8][l_c4]) = rb[h];
        }
    };
    load_global(split);
    store_smem(0);
    __syncthreads();
    int it = 0;
    for (int chunk = split; chunk < n_chunks; chunk += splits, ++it) {
        const int buf = it & 1;
        const bool more = (chunk + splits) < n_chunks;
        if (more) load_global(chunk + splits);
#pragma unroll
        for (int k = 0; k < GEMM_BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (more) store_smem(buf ^ 1);
        __syncthreads();
    }
    float* dst = part ? part + (size_t)split * K1 * N : C;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int kr = k0 + ((i < 4) ? (ty * 4 + i) : (64 + ty * 4 + i - 4));
#pragma unroll
        for (int jh = 0; jh < 2; ++jh) {
            float4* p = reinterpret_cast<float4*>(dst + (size_t)kr * N + n0 + jh * 64 + tx * 4);
            float4 v = make_float4(acc[i][jh * 4 + 0], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]);
            if (!part) {
                const float4 o = *p;
                v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
            }
            *p = v;
        }
    }
}

// db[n] += sum_m w(m) dY[m, n]; N in {128, 256}.  Bandwidth kernel: a CTA of 256 threads reads 8 rows x 128
// float4-columns (N = 128: 8 rows of 32 float4) per step with 4 loads in flight per thread and block-reduces
// through shared memory in row order.  `part`: the CTA stores its column sums to part[blockIdx.x][N] (reduced in
// CTA order by partial_sum_kernel); otherwise (one CTA) it adds them to db (and db2).
static __global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ dY, float* __restrict__ db, float* __restrict__ db2,
              const float* __restrict__ roww, const int32_t* __restrict__ row2agent, const int32_t* __restrict__ m_ptr,
              const int m_fixed, const int m_cap, const int N, const int n_agents_total, float* __restrict__ part) {
    __shared__ float4 red[256];
    int M = m_ptr ? *m_ptr : m_fixed;
    M = min(M, m_cap);
    const int vec_per_row = N / 4;                    // 32 or 64
    const int rows_per_step = 256 / vec_per_row;      // 8 or 4
    const int c4 = threadIdx.x % vec_per_row, r0 = threadIdx.x / vec_per_row;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const int stride = gridDim.x * rows_per_step;
    for (int m = blockIdx.x * rows_per_step + r0; m < M; m += 4 * stride) {
        float4 v[4];
        float w[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int mm = m + u * stride;
            if (mm < M) {
                v[u] = *reinterpret_cast<const float4*>(dY + (size_t)mm * N + c4 * 4);
                w[u] = 1.f;
                if (roww) {
                    int ag = row2agent ? row2agent[mm] : mm;
                    ag = min(max(ag, 0), n_agents_total - 1);
                    w[u] = roww[ag];
                }
            } else {
                v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                w[u] = 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            acc.x = fmaf(w[u], v[u].x, acc.x);
            acc.y = fmaf(w[u], v[u].y, acc.y);
            acc.z = fmaf(w[u], v[u].z, acc.z);
            acc.w = fmaf(w[u], v[u].w, acc.w);
        }
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    if (r0 == 0) {
        for (int r = 1; r < rows_per_step; ++r) {
            const float4 o = red[r * vec_per_row + c4];
            acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
        }
        if (part) {
            *reinterpret_cast<float4*>(part + (size_t)blockIdx.x * N + c4 * 4) = acc;
            return;
        }
        float* outs[2] = {db, db2};
        for (int q = 0; q < 2; ++q) {
            if (!outs[q]) continue;
            float4* p = reinterpret_cast<float4*>(outs[q] + c4 * 4);
            float4 o = *p;
            o.x += acc.x; o.y += acc.y; o.z += acc.z; o.w += acc.w;
            *p = o;
        }
    }
}

struct RowCount {
    const int32_t* ptr;  // device row count (edges) or nullptr
    int fixed;           // host row count when ptr == nullptr
    int cap;             // buffer capacity in rows
};

inline int32_t launch_gemm_nn(int epi, bool accum, const float* A, const float* B, const float* bias,
                              const float* bias2, float* C, const float* aux, RowCount rc, int K, int N,
                              cudaStream_t st) {
    if (K % GEMM_BK != 0 || N % GEMM_BN != 0) {
        set_error("gemm_nn: K=%d N=%d unsupported", K, N);
        return -1;
    }
    const int rows = rc.ptr ? rc.cap : min(rc.fixed, rc.cap);
    const int tiles = ((rows + GEMM_BM - 1) / GEMM_BM) * (N / GEMM_BN);
    if (tiles <= 0) return 0;
    const int grid = min(tiles, 2 * sm_count());
#define GCBF_GEMM_CASE(E, ACC)                                                                                     \
    gemm_nn_kernel<E, ACC><<<grid, GEMM_THREADS, 0, st>>>(A, B, bias, bias2, C, aux, rc.ptr, rc.fixed, rc.cap, K, N)
    if (!accum) {
        switch (epi) {
            case EPI_BIAS: GCBF_GEMM_CASE(EPI_BIAS, false); break;
            case EPI_BIAS_RELU: GCBF_GEMM_CASE(EPI_BIAS_RELU, false); break;
            case EPI_NONE: GCBF_GEMM_CASE(EPI_NONE, false); break;
            case EPI_RELU_MASK: GCBF_GEMM_CASE(EPI_RELU_MASK, false); break;
            default: set_error("bad epilogue"); return -1;
        }
    } else {
        switch (epi) {
            case EPI_NONE: GCBF_GEMM_CASE(EPI_NONE, true); break;
            case EPI_RELU_MASK: GCBF_GEMM_CASE(EPI_RELU_MASK, true); break;
            default: set_error("bad accumulate epilogue"); return -1;
        }
    }
#undef GCBF_GEMM_CASE
    count_launch();
    return check_launch("gemm_nn_kernel");
}

// `part` (optional, PART_FLOATS): split-M over up to DW_MAX_CTAS_SIMT CTAs with an ordered reduction of the splits;
// without it one CTA per output tile walks all rows.
inline int32_t launch_gemm_tn(const float* X, int ldx, const float* dY, float* C, const float* roww,
                              const int32_t* row2agent, RowCount rc, int K1, int N, int n_agents_total,
                              cudaStream_t st, float* part = nullptr) {
    if (K1 % GEMM_BM != 0 || N % GEMM_BN != 0) {
        set_error("gemm_tn: K1=%d N=%d unsupported", K1, N);
        return -1;
    }
    const int tiles = (K1 / GEMM_BM) * (N / GEMM_BN);
    const int rows = rc.ptr ? rc.cap : min(rc.fixed, rc.cap);
    const int chunks = (rows + GEMM_BK - 1) / GEMM_BK;
    if (chunks <= 0) return 0;
    int splits = max(1, (2 * sm_count()) / tiles);
    splits = min(splits, max(1, chunks / 8));  // at least 8 chunks (128 rows) per CTA
    splits = part ? min(splits, max(1, DW_MAX_CTAS_SIMT / tiles)) : 1;
    gemm_tn_kernel<<<tiles * splits, GEMM_THREADS, 0, st>>>(X, ldx, dY, C, roww, row2agent, rc.ptr, rc.fixed, rc.cap,
                                                            K1, N, splits, n_agents_total, splits > 1 ? part : nullptr);
    count_launch();
    if (int32_t r = check_launch("gemm_tn_kernel")) return r;
    if (splits == 1) return 0;
    return launch_partial_sum(part, (int64_t)K1 * N, splits, PartSegs().add(C, K1 * N), st, rc.ptr, rc.cap, GEMM_BK);
}

// db (and db2, optional) += sum_m w(m) dY[m, :].  `part` (optional, PART_FLOATS): many CTAs and an ordered reduction;
// without it one CTA walks all rows.
inline int32_t launch_colsum(const float* dY, float* db, const float* roww, const int32_t* row2agent, RowCount rc,
                             int N, int n_agents_total, cudaStream_t st, float* part = nullptr, float* db2 = nullptr) {
    if (N != 128 && N != 256) {
        set_error("colsum: N=%d unsupported (128 or 256)", N);
        return -1;
    }
    const int rows = rc.ptr ? rc.cap : min(rc.fixed, rc.cap);
    if (rows <= 0) return 0;
    const int grid = part ? min(min(max(1, rows / 128), 4 * sm_count()), (int)(PART_FLOATS / N)) : 1;
    colsum_kernel<<<grid, 256, 0, st>>>(dY, db, db2, roww, row2agent, rc.ptr, rc.fixed, rc.cap, N, n_agents_total,
                                        grid > 1 ? part : nullptr);
    count_launch();
    if (int32_t r = check_launch("colsum_kernel")) return r;
    if (grid == 1) return 0;
    return launch_partial_sum(part, N, grid, PartSegs().add(db, N, db2), st);
}

}  // namespace gcbf
