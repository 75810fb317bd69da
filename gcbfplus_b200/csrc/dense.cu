// dense.cu -- the dense-layer kernels of the GNN and their launchers: the strict-fp32 SIMT GEMM family and the ordered
// partial sums (types in gemm.cuh), the wgmma 3xTF32 GEMMs (device code in gemm_tc.cuh), the batched small products and
// the plane builder (smalljobs.cuh), the transposed weights (translayout.cuh), and the building-block entry points
// exported for unit tests and bench.py's isolated kernel timing.  The launchers other units call are declared in
// internal.cuh.
#include "gemm.cuh"
#include "gemm_tc.cuh"
#include "smalljobs.cuh"
#include "translayout.cuh"
#include "internal.cuh"

namespace gcbf {

// Tiling: CTA tile 128x128, BK = 16, 256 threads, 8x8 register tile per thread split as
// 2x2 blocks of 4x4 (conflict-free LDS.128), register-prefetch double buffering, persistent
// tile loop (grid = k * #SM) so that a device-side row count (edge count) can drive the
// launch inside a CUDA graph.
constexpr int GEMM_BM = 128, GEMM_BN = 128, GEMM_BK = 16, GEMM_THREADS = 256;
constexpr int GEMM_LDA = GEMM_BM + 4;  // padded: transposed A tile

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

int32_t launch_partial_sum(const float* part, int64_t stride, int nparts, const PartSegs& segs, cudaStream_t st,
                           const int32_t* m_ptr, int m_cap, int rows_per_part) {
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

int32_t launch_gemm_nn(int epi, bool accum, const float* A, const float* B, const float* bias, const float* bias2,
                       float* C, const float* aux, RowCount rc, int K, int N, cudaStream_t st) {
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
int32_t launch_gemm_tn(const float* X, int ldx, const float* dY, float* C, const float* roww, const int32_t* row2agent,
                       RowCount rc, int K1, int N, int n_agents_total, cudaStream_t st, float* part) {
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
int32_t launch_colsum(const float* dY, float* db, const float* roww, const int32_t* row2agent, RowCount rc, int N,
                      int n_agents_total, cudaStream_t st, float* part, float* db2) {
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

namespace tc {

// Weights are split once per parameter update (gcbf_prepare_params_l); activations are split in shared memory.
static __global__ void split_tf32_kernel(const float* __restrict__ in, float* __restrict__ hi, float* __restrict__ lo, int n) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float x = in[i];
        const float h = rn_tf32(x);
        hi[i] = h;
        lo[i] = rn_tf32(x - h);
    }
}

template <int EPI, bool ACCUM>
__global__ void __launch_bounds__(THREADS_NN, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBh,
               const __grid_constant__ CUtensorMap tmBl, const float* __restrict__ bias,
               const float* __restrict__ bias2, float* __restrict__ C, const float* __restrict__ aux,
               const int32_t* __restrict__ m_ptr, const int m_fixed, const int m_cap, const int K, const int N,
               const int ndot) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align1024(smem_raw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STG);   // [STAGES] TMA bytes landed
    uint64_t* empty = full + STAGES;                                      // [STAGES] MMAs of the stage retired

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_n = N / BN;                // 1, or 2 for a 256-wide layer
    const int nkb = K / BK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], CONSUMERS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    int M = m_ptr ? *m_ptr : m_fixed;
    M = min(M, m_cap);
    const int n_tiles = ((M + BM - 1) / BM) * tiles_n;

    if (warp == 8) {
        // ================= TMA producer =================
        if (lane == 0) {
            uint32_t it = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN;
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
                    uint8_t* st = smem + s * STG;
                    mbar_expect_tx(&full[s], 3 * PLANE);
                    tma_load_2d(st, &tmA, &full[s], kb * BK, m0);
                    tma_load_2d(st + 2 * PLANE, &tmBh, &full[s], kb * BK, n0);
                    tma_load_2d(st + 3 * PLANE, &tmBl, &full[s], kb * BK, n0);
                }
            }
        }
        return;
    }
    // ================= consumers: A split, MMAs, epilogue =================
    const int g = warp >> 2, wt = threadIdx.x & 127;
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN;
        float d[64];
        tma_a_mainloop(d, smem, full, empty, it, nkb, g, wt);

        const int r0 = m0 + 64 * g + frag_row0(wt);
        if (EPI == EPI_RELU_DOTN) {   // output-layer partial sums over this column tile
            float q[2][4];
            frag_relu_dot<4>(d, bias + n0, aux + (size_t)n0 * ndot, ndot, ndot, wt, q);
            if ((lane & 3) == 0)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (r0 + 8 * h < M)
                        *reinterpret_cast<float4*>(C + ((size_t)(n0 / BN) * m_cap + r0 + 8 * h) * 4) =
                            make_float4(q[h][0], q[h][1], q[h][2], q[h][3]);
            continue;
        }
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int m = r0 + 8 * ((i >> 1) & 1);
            if (m >= M) continue;
            const int n = n0 + frag_col(wt, i);
            float2 o = make_float2(d[i], d[i + 1]);
            if (EPI == EPI_BIAS || EPI == EPI_BIAS_RELU) {
                const float2 bb = *reinterpret_cast<const float2*>(bias + n);
                o.x += bb.x; o.y += bb.y;
                if (bias2) {
                    const float2 b2 = *reinterpret_cast<const float2*>(bias2 + n);
                    o.x += b2.x; o.y += b2.y;
                }
                if (EPI == EPI_BIAS_RELU) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
            } else if (EPI == EPI_RELU_MASK) {
                const float2 mk = *reinterpret_cast<const float2*>(aux + (size_t)m * N + n);
                o.x = mk.x > 0.f ? o.x : 0.f;
                o.y = mk.y > 0.f ? o.y : 0.f;
            }
            float2* cp = reinterpret_cast<float2*>(C + (size_t)m * N + n);
            if (ACCUM) {
                const float2 old = *cp;
                o.x += old.x; o.y += old.y;
            }
            *cp = o;
        }
    }
}

template <int EPI, bool ACC>
static void launch_nn_inst(int grid, cudaStream_t st, const CUtensorMap& tmA, const CUtensorMap& tmB,
                           const CUtensorMap& tmBl, const float* bias, const float* bias2, float* C, const float* aux,
                           RowCount rc, int K, int N, int ndot) {
    constexpr int smem = STAGES * STG + 1024 + 256;
    auto kern = gemm_tc_kernel<EPI, ACC>;
    static bool attr_done = false;
    if (!attr_done) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        attr_done = true;
    }
    kern<<<grid, THREADS_NN, smem, st>>>(tmA, tmB, tmBl, bias, bias2, C, aux, rc.ptr, rc.fixed, rc.cap, K, N, ndot);
}

// C[M,N] = epi(A[M,K] @ Bt[N,K]^T) with Bt given as its tf32 split (Bt_hi + Bt_lo, split_tf32_kernel).
// A must be backed by at least rc.cap rows.  A 256-wide layer runs as two 128-wide column tiles; EPI_RELU_DOTN writes
// one partial sum per column tile (*parts_out = N / BN).
int32_t launch_gemm_tc(int epi, bool accum, const float* A, const float* Bt_hi, const float* Bt_lo, const float* bias,
                       const float* bias2, float* C, const float* aux, RowCount rc, int K, int N, cudaStream_t st,
                       int ndot, int* parts_out) {
    if (K % BK != 0 || (N != 128 && N != 256) || ndot > 4) {
        set_error("gemm_tc: K=%d N=%d epi=%d unsupported", K, N, epi);
        return -1;
    }
    if (parts_out) *parts_out = N / BN;
    const int rows = rc.ptr ? rc.cap : min(rc.fixed, rc.cap);
    if (rows <= 0) return 0;
    const int tiles_m = (rows + BM - 1) / BM;
    CUtensorMap tmA, tmB, tmBl;
    if (int32_t r = make_map(&tmA, A, rc.cap, K, BM)) return r;
    if (int32_t r = make_map(&tmB, Bt_hi, N, K, BN)) return r;
    if (int32_t r = make_map(&tmBl, Bt_lo, N, K, BN)) return r;
    const int grid = min(tiles_m * (N / BN), sm_count());
#define GCBF_TC_CASE(E, ACC) launch_nn_inst<E, ACC>(grid, st, tmA, tmB, tmBl, bias, bias2, C, aux, rc, K, N, ndot)
    if (!accum) {
        switch (epi) {
            case EPI_BIAS: GCBF_TC_CASE(EPI_BIAS, false); break;
            case EPI_BIAS_RELU: GCBF_TC_CASE(EPI_BIAS_RELU, false); break;
            case EPI_NONE: GCBF_TC_CASE(EPI_NONE, false); break;
            case EPI_RELU_MASK: GCBF_TC_CASE(EPI_RELU_MASK, false); break;
            case EPI_RELU_DOTN: GCBF_TC_CASE(EPI_RELU_DOTN, false); break;
            default: set_error("bad epilogue"); return -1;
        }
    } else {
        switch (epi) {
            case EPI_NONE: GCBF_TC_CASE(EPI_NONE, true); break;
            case EPI_RELU_MASK: GCBF_TC_CASE(EPI_RELU_MASK, true); break;
            default: set_error("bad accumulate epilogue"); return -1;
        }
    }
#undef GCBF_TC_CASE
    count_launch();
    return check_launch("gemm_tc_kernel");
}

// =====================================================================================================
// backward-weight on tensor cores:  C[K1, N] += sum_m w(m) X[m, k1] dY[m, n]
// D[128 k1-rows, BN n-columns] += A B^T with A = X^T and B = dY^T: the MMA-K index is the row index m of X / dY.
// tf32 wgmma reads both operands K-major only, so TMA lands plain [32 m x 32] boxes of X and dY (a "raw" ring of
// 2 stages) and the consumers transpose them while splitting into K-major SWIZZLE_128B hi / lo planes ([128 k1][32 m]
// and [BN n][32 m]; double-buffered for BN = 128, single for BN = 256).  Rows m >= M are selected to zero (they may
// hold stale data, possibly NaN), dY is scaled by the row weight, and the column sums sum_m w(m) dY[m, n] are taken
// from the very values converted.  Split over M: CTA (tile, split) walks 32-row chunks {split, split + S, ...}.  With
// more than one split each CTA stores its tile (and its column sums) to a workspace and partial_sum_kernel adds the
// splits to C in split order: no float atomics, the same bits on every run.
// =====================================================================================================
constexpr int TN_RAWS = 2;

template <int BNT>
struct TnCfg {
    static constexpr int NH = BNT / 128;                     // 128-wide accumulators per warpgroup
    static constexpr int PB = (BNT == 256) ? 1 : 2;          // plane buffers
    static constexpr int RAW = (4 + BNT / 32) * 4096;        // 4 boxes of X, BNT / 32 boxes of dY
    static constexpr int PLANES = 2 * PLANE + 2 * BNT * 128; // A hi | A lo | B hi | B lo
    static constexpr int SMEM = TN_RAWS * RAW + PB * PLANES + 1024 + 256;
};

// `cs1` / `cs2` (optional): column sums sum_m w(m) dY[m, n] -- the bias gradient of the same layer (and the agent
// one-hot row of the update layer) -- accumulated by the converting threads, so no separate pass over dY is needed.
// Only the CTAs of k1-tile 0 contribute.
// `part` (splits > 1): CTA (tile, split) stores its tile to part[split][K1][N] and its column sums to
// part[split][K1 * N + n] (stride K1 * N + N); otherwise (one split) it adds them to C / cs1 / cs2 itself.
template <int BNT>
__global__ void __launch_bounds__(THREADS_NN, 1)
gemm_tn_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                  float* __restrict__ C, const float* __restrict__ roww, const int32_t* __restrict__ row2agent,
                  const int32_t* __restrict__ m_ptr, const int m_fixed, const int m_cap, const int N, const int splits,
                  const int n_agents_total, float* __restrict__ cs1, float* __restrict__ cs2, const int K1,
                  float* __restrict__ part) {
    using CF = TnCfg<BNT>;
    constexpr int MR = 32 * BNT / 256;                       // m rows of dY converted per thread
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_align1024(smem_raw);
    uint8_t* planes = smem + TN_RAWS * CF::RAW;
    uint64_t* full = reinterpret_cast<uint64_t*>(planes + CF::PB * CF::PLANES);
    uint64_t* empty = full + TN_RAWS;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int M = m_ptr ? *m_ptr : m_fixed;
    M = min(M, m_cap);
    const int tile = blockIdx.x / splits, split = blockIdx.x % splits;
    const int k1_0 = tile * 128;
    const int n_chunks = (M + 31) / 32;
    const int n_my = (split < n_chunks) ? (n_chunks - split + splits - 1) / splits : 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < TN_RAWS; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], CONSUMERS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            for (int it = 0; it < n_my; ++it) {
                const int s = it % TN_RAWS;
                const int m0 = (split + it * splits) * 32;
                mbar_wait(&empty[s], ((it / TN_RAWS) & 1) ^ 1);
                uint8_t* st = smem + s * CF::RAW;
                mbar_expect_tx(&full[s], CF::RAW);
#pragma unroll
                for (int i = 0; i < 4; ++i) tma_load_2d(st + i * 4096, &tmX, &full[s], k1_0 + 32 * i, m0);
#pragma unroll
                for (int j = 0; j < BNT / 32; ++j) tma_load_2d(st + (4 + j) * 4096, &tmY, &full[s], 32 * j, m0);
            }
        }
        return;
    }
    const int t = threadIdx.x;                 // 0..255
    const int g = warp >> 2, wt = t & 127;
    const int xk = t & 127, xm = (t >> 7) * 16;          // X: column k1 = xk, rows xm .. xm + 15
    const int yn = t % BNT, ym = (t / BNT) * MR;         // dY: column n = yn, rows ym .. ym + MR - 1
    const bool do_cs = (cs1 != nullptr) && tile == 0;
    float csum = 0.f;
    float d[CF::NH][64];
#pragma unroll
    for (int h = 0; h < CF::NH; ++h)
#pragma unroll
        for (int i = 0; i < 64; ++i) d[h][i] = 0.f;
    for (int it = 0; it < n_my; ++it) {
        const int s = it % TN_RAWS;
        const int m0 = (split + it * splits) * 32;
        uint8_t* raw = smem + s * CF::RAW;
        uint8_t* pl = planes + (it % CF::PB) * CF::PLANES;
        mbar_wait(&full[s], (it / TN_RAWS) & 1);
        bar_consumers();                       // the MMAs that last read this plane buffer have retired in both warpgroups
        {   // X -> A planes [k1][m]
            const float* xs = reinterpret_cast<const float*>(raw + (xk >> 5) * 4096) + (xk & 31);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float v[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int m = xm + 4 * c + j;
                    v[j] = (m0 + m < M) ? xs[m * 32] : 0.f;
                }
                float4 h, l;
                split_tf32(make_float4(v[0], v[1], v[2], v[3]), h, l);
                const int off = swz(xk, (xm >> 2) + c);
                *reinterpret_cast<float4*>(pl + off) = h;
                *reinterpret_cast<float4*>(pl + PLANE + off) = l;
            }
        }
        {   // dY (scaled by the row weight) -> B planes [n][m]
            const float* ys = reinterpret_cast<const float*>(raw + (4 + (yn >> 5)) * 4096) + (yn & 31);
            uint8_t* bh = pl + 2 * PLANE;
            uint8_t* bl = bh + BNT * 128;
#pragma unroll
            for (int c = 0; c < MR / 4; ++c) {
                float v[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int m = ym + 4 * c + j;
                    const int gm = m0 + m;
                    float y = 0.f;
                    if (gm < M) {
                        float w = 1.f;
                        if (roww) {
                            int ag = row2agent ? row2agent[gm] : gm;
                            ag = min(max(ag, 0), n_agents_total - 1);
                            w = roww[ag];
                        }
                        y = ys[m * 32] * w;
                    }
                    csum += y;
                    v[j] = y;
                }
                float4 h, l;
                split_tf32(make_float4(v[0], v[1], v[2], v[3]), h, l);
                const int off = swz(yn, (ym >> 2) + c);
                *reinterpret_cast<float4*>(bh + off) = h;
                *reinterpret_cast<float4*>(bl + off) = l;
            }
        }
        fence_async_smem();
        bar_consumers();
        mbar_arrive(&empty[s]);                // raw stage consumed
        wg_fence();
        const uint32_t a_hi = smem_u32(pl) + g * WG_ROWS_BYTES;
        const uint32_t b_hi = smem_u32(pl) + 2 * PLANE;
#pragma unroll
        for (int h = 0; h < CF::NH; ++h)
            mma_kblock(d[h], a_hi, a_hi + PLANE, b_hi + h * 128 * 128, b_hi + BNT * 128 + h * 128 * 128, it == 0);
        wg_commit();
        wg_wait<CF::PB - 1>();
    }
    wg_wait<0>();
    if (n_my == 0) return;
    if (do_cs) {
        bar_consumers();                       // every MMA has retired: the plane buffers are free
        float* s_cs = reinterpret_cast<float*>(planes);
        s_cs[t] = csum;                        // [t / BNT][n]
        bar_consumers();
        if (t < BNT) {
            float v = s_cs[t];
            if (BNT == 128) v += s_cs[t + 128];
            if (part) {
                part[(size_t)split * ((size_t)K1 * N + N) + (size_t)K1 * N + t] = v;
            } else {
                cs1[t] += v;
                if (cs2) cs2[t] += v;
            }
        }
    }
    float* dst = part ? part + (size_t)split * ((size_t)K1 * N + N) : C;
    const int r0 = 64 * g + frag_row0(wt);
#pragma unroll
    for (int h = 0; h < CF::NH; ++h)
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            float2* p = reinterpret_cast<float2*>(dst + (size_t)(k1_0 + r0 + 8 * ((i >> 1) & 1)) * N + h * 128 + frag_col(wt, i));
            float2 v = make_float2(d[h][i], d[h][i + 1]);
            if (!part) {
                const float2 o = *p;
                v.x += o.x;
                v.y += o.y;
            }
            *p = v;
        }
}

// C[K1, N] += sum_m w(m) X[m, :K1] dY[m, :N]; X row stride ldx (>= K1, multiple of 4), K1 % 128 == 0, N in {128, 256}.
// cs1 / cs2 (optional): += sum_m w(m) dY[m, :N] (bias gradient fused into the same pass over dY).
// `part` (optional, PART_FLOATS): split-M over up to DW_MAX_CTAS_TC CTAs with an ordered reduction of the splits;
// without it one CTA per 128-row tile of C walks all rows.
int32_t launch_gemm_tn_tc(const float* X, int ldx, const float* dY, float* C, const float* roww,
                          const int32_t* row2agent, RowCount rc, int K1, int N, int n_agents_total, cudaStream_t st,
                          float* cs1, float* cs2, float* part) {
    if (K1 % 128 != 0 || (N != 128 && N != 256) || ldx % 4 != 0) {
        set_error("gemm_tn_tc: K1=%d N=%d ldx=%d unsupported", K1, N, ldx);
        return -1;
    }
    const int rows = rc.ptr ? rc.cap : min(rc.fixed, rc.cap);
    if (rows <= 0) return 0;
    CUtensorMap tmX, tmY;
    if (int32_t r = make_map_box(&tmX, X, rc.cap, K1, ldx, 32, 32, CU_TENSOR_MAP_SWIZZLE_NONE)) return r;
    if (int32_t r = make_map_box(&tmY, dY, rc.cap, N, N, 32, 32, CU_TENSOR_MAP_SWIZZLE_NONE)) return r;
    const int tiles = K1 / 128;
    const int chunks = (rows + 31) / 32;
    int splits = max(1, sm_count() / tiles);
    splits = min(splits, max(1, chunks * 32 / 128));       // >= 128 rows per CTA
    splits = part ? min(splits, max(1, DW_MAX_CTAS_TC / tiles)) : 1;
    float* kpart = splits > 1 ? part : nullptr;
    const int grid = tiles * splits;
#define GCBF_TN_CASE(BN_)                                                                                             \
    do {                                                                                                              \
        constexpr int smem = TnCfg<BN_>::SMEM;                                                                        \
        static bool done = false;                                                                                     \
        if (!done) { cudaFuncSetAttribute(gemm_tn_tc_kernel<BN_>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); done = true; } \
        gemm_tn_tc_kernel<BN_><<<grid, THREADS_NN, smem, st>>>(tmX, tmY, C, roww, row2agent, rc.ptr, rc.fixed, rc.cap, N, \
                                                               splits, n_agents_total, cs1, cs2, K1, kpart);          \
    } while (0)
    if (N == 256) GCBF_TN_CASE(256);
    else GCBF_TN_CASE(128);
#undef GCBF_TN_CASE
    count_launch();
    if (int32_t r = check_launch("gemm_tn_tc_kernel")) return r;
    if (splits == 1) return 0;
    PartSegs segs;
    segs.add(C, K1 * N);
    if (cs1) segs.add(cs1, N, cs2);
    return launch_partial_sum(part, (int64_t)K1 * N + N, splits, segs, st, rc.ptr, rc.cap, 32);
}

}  // namespace tc

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

int32_t SmallJobList::launch(cudaStream_t st) {
    if (J.n == 0) return 0;
    small_jobs_kernel<<<J.blk0[J.n], 256, 0, st>>>(J);
    count_launch();
    const int32_t rc = check_launch("small_jobs_kernel");
    J.n = 0;
    return rc;
}

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

int32_t PlaneJobList::launch(cudaStream_t st) {
    if (J.n == 0) return 0;
    plane_jobs_kernel<<<J.tile0[J.n], 256, 0, st>>>(J);
    count_launch();
    const int32_t rc = check_launch("plane_jobs_kernel");
    J.n = 0;
    return rc;
}

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

int32_t build_transposes(const ParamLayout& L, const TransLayout& T, const float* P, float* PT, cudaStream_t st) {
    for (int i = 0; i < 12; ++i) {
        if (T.w[i] < 0) continue;
        const float* src = P + L.w[i] + (i == L_UPD0 ? 3 * 256 : 0);
        const int rows = (i == L_UPD0) ? 128 : L.in[i];
        if (int32_t rc = launch_transpose(src, PT + T.w[i], rows, L.out[i], st)) return rc;
    }
    return 0;
}

}  // namespace gcbf

using namespace gcbf;

// ---- building blocks exported for unit tests and for bench.py's isolated kernel timing ----
extern "C" __attribute__((visibility("default"))) int32_t gcbf_gemm_nn(int32_t epi, int32_t accum, const float* A,
                                                                       const float* B, const float* bias,
                                                                       const float* bias2, float* C, const float* aux,
                                                                       const int32_t* m_ptr, int32_t m_fixed,
                                                                       int32_t m_cap, int32_t K, int32_t N,
                                                                       void* stream) {
    GCBF_REQUIRE(A && B && C, "gcbf_gemm_nn: NULL pointer");
    GCBF_REQUIRE((epi != EPI_BIAS && epi != EPI_BIAS_RELU) || bias, "gcbf_gemm_nn: bias required");
    GCBF_REQUIRE(epi != EPI_RELU_MASK || aux, "gcbf_gemm_nn: aux required");
    return launch_gemm_nn(epi, accum != 0, A, B, bias, bias2, C, aux, RowCount{m_ptr, m_fixed, m_cap}, K, N,
                          (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_gemm_tn(const float* X, int32_t ldx, const float* dY,
                                                                       float* C, const float* roww,
                                                                       const int32_t* row2agent, const int32_t* m_ptr,
                                                                       int32_t m_fixed, int32_t m_cap, int32_t K1,
                                                                       int32_t N, int32_t n_agents_total, void* stream) {
    GCBF_REQUIRE(X && dY && C, "gcbf_gemm_tn: NULL pointer");
    return launch_gemm_tn(X, ldx, dY, C, roww, row2agent, RowCount{m_ptr, m_fixed, m_cap}, K1, N, n_agents_total,
                          (cudaStream_t)stream);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_colsum(const float* dY, float* db, const float* roww,
                                                                      const int32_t* row2agent, const int32_t* m_ptr,
                                                                      int32_t m_fixed, int32_t m_cap, int32_t N,
                                                                      int32_t n_agents_total, void* stream) {
    GCBF_REQUIRE(dY && db, "gcbf_colsum: NULL pointer");
    return launch_colsum(dY, db, roww, row2agent, RowCount{m_ptr, m_fixed, m_cap}, N, n_agents_total,
                         (cudaStream_t)stream);
}

// ---- tensor-core (wgmma 3xTF32) variant of gcbf_gemm_nn: C = epi(A[M,K] @ Bt[N,K]^T) ----
extern "C" __attribute__((visibility("default"))) int32_t gcbf_gemm_tc(int32_t epi, int32_t accum, const float* A,
                                                                       const float* Bt_hi, const float* Bt_lo,
                                                                       const float* bias,
                                                                       const float* bias2, float* C, const float* aux,
                                                                       const int32_t* m_ptr, int32_t m_fixed,
                                                                       int32_t m_cap, int32_t K, int32_t N,
                                                                       int32_t ndot, void* stream) {
    GCBF_REQUIRE(A && Bt_hi && Bt_lo && C, "gcbf_gemm_tc: NULL pointer");
    GCBF_REQUIRE(epi != EPI_RELU_DOTN || (bias && aux), "gcbf_gemm_tc: bias and aux required");
    GCBF_REQUIRE(epi != EPI_RELU_DOTN || (ndot >= 1 && ndot <= 4), "gcbf_gemm_tc: ndot must be in [1, 4]");
    GCBF_REQUIRE((epi != EPI_BIAS && epi != EPI_BIAS_RELU) || bias, "gcbf_gemm_tc: bias required");
    GCBF_REQUIRE(epi != EPI_RELU_MASK || aux, "gcbf_gemm_tc: aux required");
    GCBF_REQUIRE((((uintptr_t)A | (uintptr_t)Bt_hi | (uintptr_t)Bt_lo | (uintptr_t)C) & 15) == 0,
                 "gcbf_gemm_tc: 16-byte alignment required");
    return gcbf::tc::launch_gemm_tc(epi, accum != 0, A, Bt_hi, Bt_lo, bias, bias2, C, aux,
                                    RowCount{m_ptr, m_fixed, m_cap}, K, N, (cudaStream_t)stream, ndot);
}

extern "C" __attribute__((visibility("default"))) int32_t gcbf_split_tf32(const float* in, float* hi, float* lo, int32_t n,
                                                                          void* stream) {
    GCBF_REQUIRE(in && hi && lo && n > 0, "gcbf_split_tf32: bad argument");
    gcbf::tc::split_tf32_kernel<<<min((n + 255) / 256, 4 * sm_count()), 256, 0, (cudaStream_t)stream>>>(in, hi, lo, n);
    count_launch();
    return check_launch("split_tf32_kernel");
}
extern "C" __attribute__((visibility("default"))) int32_t gcbf_gemm_tn_tc(const float* X, int32_t ldx, const float* dY,
                                                                          float* C, const float* roww,
                                                                          const int32_t* row2agent,
                                                                          const int32_t* m_ptr, int32_t m_fixed,
                                                                          int32_t m_cap, int32_t K1, int32_t N,
                                                                          int32_t n_agents_total, float* cs1, float* cs2,
                                                                          void* stream) {
    GCBF_REQUIRE(X && dY && C, "gcbf_gemm_tn_tc: NULL pointer");
    GCBF_REQUIRE(cs1 || !cs2, "gcbf_gemm_tn_tc: cs2 without cs1");
    GCBF_REQUIRE((((uintptr_t)X | (uintptr_t)dY | (uintptr_t)C) & 15) == 0, "gcbf_gemm_tn_tc: 16-byte alignment required");
    return gcbf::tc::launch_gemm_tn_tc(X, ldx, dY, C, roww, row2agent, RowCount{m_ptr, m_fixed, m_cap}, K1, N,
                                       n_agents_total, (cudaStream_t)stream, cs1, cs2);
}
