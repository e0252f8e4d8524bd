// K5 — CSR / CSC build of the GCN aggregation pattern, and K9 — induced subgraph with relabelling.
//
// Reference behaviour replaced (per call, paths in the reference repository): large/ours.py:26-33 (PyG degree -> edge weights ->
// torch_sparse.SparseTensor(row=col, col=row): argsort of target*N+source + rowptr), medium/models.py:22-37
// (PyG gcn_norm: add_remaining_self_loops + degree), large/main-batch.py:139 (PyG subgraph, CPU, O(E) per batch).
//
// Pipeline (all HBM-bound integer work, no tensor cores):
//   count   : one pass over the int64 edge list, atomicAdd into int32 row counters        (8 B/edge read)
//   scan    : 3-kernel exclusive scan of the counters -> int64 rowptr                       (12 B/node)
//   fill    : second pass, cursor atomics, writes int32 column ids                          (16 B/edge read, 4 B write)
//   sort    : per-row sort of the column ids (warp rank-sort <=32, block bitonic in smem <=2048, block bitonic
//             in global memory above) so the arrays are deterministic and bit-exact with the reference's
//             (target, source)-sorted storage
//   dinv    : dinv[i] = sqrt(1/len_i) (0 for empty rows)
//
// Weighted build (sgf_csr_build_weighted, edge_weight of the medium GCN / DIFFormer, DESIGN.md §4.10): the fill writes 64-bit keys
// (col << 32 | eid + 1) instead of column ids, so the same sort tiers order every row by (col, eid) and carry the source edge's
// position along; an unpack pass then splits the keys into col / eid and gathers val[j] = w[eid[j]].
#include <cstdlib>

#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

namespace sgf {

constexpr int kScanBlock = 1024;
constexpr int kScanItems = 4;  // per thread -> 4096 per block

// rows [row_begin, row_end) of a matrix with n_cols columns are built; edges whose key falls outside are skipped.
// (bound by the L2's atomic rate; issuing four independent loads per thread changes nothing.)
__global__ void csr_count_kernel(const int64_t* __restrict__ key, const int64_t* __restrict__ val, int64_t nnz,
                                 int64_t row_begin, int64_t row_end, int64_t n_cols, int drop_self_loops,
                                 int* __restrict__ counts, int* __restrict__ err) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        int64_t k = key[e], v = val[e];
        if (k < 0 || k >= n_cols || v < 0 || v >= n_cols) { atomicExch(err, 1); continue; }
        if (k < row_begin || k >= row_end) continue;
        if (drop_self_loops && k == v) continue;
        atomicAdd(&counts[k - row_begin], 1);
    }
}

// counts[i] (+1 if add_loop) -> block-local exclusive scan into rowptr[i]; block totals to block_sums
__global__ void scan_local_kernel(const int* __restrict__ counts, int64_t n, int add_loop, int64_t* __restrict__ rowptr,
                                  int64_t* __restrict__ block_sums) {
    __shared__ int64_t warp_tot[32];
    const int tid = threadIdx.x;
    const int64_t base = ((int64_t)blockIdx.x * kScanBlock + tid) * kScanItems;
    int64_t v[kScanItems];
    int64_t tsum = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        int64_t idx = base + i;
        v[i] = idx < n ? (int64_t)counts[idx] + add_loop : 0;
        tsum += v[i];
    }
    // inclusive warp scan of tsum
    int64_t x = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if ((tid & 31) >= o) x += y;
    }
    if ((tid & 31) == 31) warp_tot[tid >> 5] = x;
    __syncthreads();
    if (tid < 32) {
        int64_t w = warp_tot[tid];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int64_t y = __shfl_up_sync(0xffffffffu, w, o);
            if (tid >= o) w += y;
        }
        warp_tot[tid] = w;  // inclusive over warps
    }
    __syncthreads();
    int64_t excl = x - tsum + ((tid >> 5) > 0 ? warp_tot[(tid >> 5) - 1] : 0);
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        int64_t idx = base + i;
        if (idx < n) rowptr[idx] = excl;
        excl += v[i];
    }
    if (tid == kScanBlock - 1) block_sums[blockIdx.x] = warp_tot[31];
}

// single block: exclusive scan of block_sums in place; total -> *total_out
__global__ void scan_block_sums_kernel(int64_t* __restrict__ block_sums, int64_t nblocks, int64_t* __restrict__ total_out) {
    __shared__ int64_t warp_tot[32];
    __shared__ int64_t carry_s;
    const int tid = threadIdx.x;
    if (tid == 0) carry_s = 0;
    __syncthreads();
    for (int64_t base = 0; base < nblocks; base += kScanBlock) {
        int64_t idx = base + tid;
        int64_t v = idx < nblocks ? block_sums[idx] : 0;
        int64_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int64_t y = __shfl_up_sync(0xffffffffu, x, o);
            if ((tid & 31) >= o) x += y;
        }
        if ((tid & 31) == 31) warp_tot[tid >> 5] = x;
        __syncthreads();
        if (tid < 32) {
            int64_t w = warp_tot[tid];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int64_t y = __shfl_up_sync(0xffffffffu, w, o);
                if (tid >= o) w += y;
            }
            warp_tot[tid] = w;
        }
        __syncthreads();
        int64_t carry = carry_s;
        int64_t excl = carry + x - v + ((tid >> 5) > 0 ? warp_tot[(tid >> 5) - 1] : 0);
        if (idx < nblocks) block_sums[idx] = excl;
        __syncthreads();
        if (tid == 0) carry_s = carry + warp_tot[31];
        __syncthreads();
    }
    if (tid == 0) *total_out = carry_s;
}

__global__ void scan_add_kernel(int64_t* __restrict__ rowptr, int64_t n, const int64_t* __restrict__ block_sums,
                                const int64_t* __restrict__ total, int* __restrict__ cursor, int add_loop) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += stride) {
        if (i == n) { rowptr[n] = *total; continue; }
        rowptr[i] += block_sums[i / (kScanBlock * kScanItems)];
        cursor[i] = 0;
    }
}

__global__ void csr_fill_kernel(const int64_t* __restrict__ key, const int64_t* __restrict__ val, int64_t nnz, int64_t shard_begin,
                                int64_t row_begin, int64_t row_end, int64_t n_cols, int drop_self_loops,
                                const int64_t* __restrict__ rowptr, int* __restrict__ cursor, int32_t* __restrict__ col) {
    // [row_begin, row_end) is the row window of THIS launch (sgf_csr_build_rot runs one launch per window so that the scattered
    // 4-byte writes of a launch stay inside one piece of `col`); rowptr / cursor are indexed relative to shard_begin.
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        int64_t k = key[e];
        if (k < row_begin || k >= row_end) continue;
        int64_t v = val[e];
        if (v < 0 || v >= n_cols) continue;
        if (drop_self_loops && k == v) continue;
        k -= shard_begin;
        int pos = atomicAdd(&cursor[k], 1);
        col[rowptr[k] + pos] = (int32_t)v;
    }
}

// Row-sharded runs with pushed operand blocks (sgf_spmm_flagged): column ids are stored ROTATED, col' = (col - rot) mod `mod`, so
// that the rank's own row block comes first in every row and the gathered operand buffer is indexed by arrival slot.
__global__ void csr_rotate_cols_kernel(int32_t* __restrict__ col, const int64_t* __restrict__ rowptr, int64_t n, int64_t rot, int64_t mod) {
    const int64_t total = rowptr[n];
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        int64_t v = (int64_t)col[i] - rot;
        if (v < 0) v += mod;
        col[i] = (int32_t)v;
    }
}

// splits[t][r] = number of entries of row r whose (sorted) column id is < thr[t]  (binary search; thresholds ascending)
__global__ void csr_row_splits_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col, int64_t n, int n_thr,
                                      const int32_t* __restrict__ thr, int32_t* __restrict__ splits) {
    const int64_t total = n * n_thr;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int t = (int)(i / n);
        const int64_t r = i - (int64_t)t * n;
        const int64_t s = rowptr[r];
        int64_t lo = s, hi = rowptr[r + 1];
        const int32_t key = thr[t];
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (col[mid] < key) lo = mid + 1; else hi = mid;
        }
        splits[i] = (int32_t)(lo - s);
    }
}

__global__ void csr_add_loops_kernel(int64_t n, int64_t row_begin, const int64_t* __restrict__ rowptr, int* __restrict__ cursor,
                                     int32_t* __restrict__ col) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        int pos = atomicAdd(&cursor[i], 1);
        col[rowptr[i] + pos] = (int32_t)(row_begin + i);
    }
}

// ---- per-row sort ---------------------------------------------------------------------------------
constexpr int kSortSmemMax = 2048;

// Sort keys: int32 column ids, or the int64 (col << 32 | eid + 1) keys of the weighted build.  key_pad sorts after every key.
template <typename T> __device__ __forceinline__ T key_pad();
template <> __device__ __forceinline__ int32_t key_pad<int32_t>() { return INT32_MAX; }
template <> __device__ __forceinline__ int64_t key_pad<int64_t>() { return INT64_MAX; }
__device__ __forceinline__ int32_t key_min(int32_t a, int32_t b) { return min(a, b); }
__device__ __forceinline__ int32_t key_max(int32_t a, int32_t b) { return max(a, b); }
__device__ __forceinline__ int64_t key_min(int64_t a, int64_t b) { return a < b ? a : b; }
__device__ __forceinline__ int64_t key_max(int64_t a, int64_t b) { return a < b ? b : a; }

template <typename T>
__device__ __forceinline__ void bitonic_block(T* a, int npow2, int tid, int nthreads) {
    for (int k = 2; k <= npow2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < npow2; i += nthreads) {
                int ixj = i ^ j;
                if (ixj > i) {
                    T x = a[i], y = a[ixj];
                    bool up = (i & k) == 0;
                    if ((x > y) == up) { a[i] = y; a[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
}

// Ascending sort of col[s, s + len), 2 <= len <= kWarpSortMax, by one warp: <= 64 entries by a bitonic network in registers (one or
// two entries per lane, shuffles), longer rows by a bitonic network in `sm` (kWarpSortMax ints of per-warp scratch).
constexpr int kWarpSortMax = 256;
// bitonic network over 32 * NREG entries held NREG per lane (entry i = lane + 32 * reg): compare-exchange partners at distance
// j < 32 by shfl.xor, at distance 32 inside the lane.  ~8 instructions per stage and register instead of the ~9 per ENTRY of a rank sort.
template <int NREG, typename T>
__device__ __forceinline__ void warp_bitonic(T (&v)[NREG], int lane) {
#pragma unroll
    for (int k = 2; k <= 32 * NREG; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            if (j == 32) {                      // NREG == 2, k == 64: ascending everywhere
                const T lo = key_min(v[0], v[NREG - 1]), hi = key_max(v[0], v[NREG - 1]);
                v[0] = lo; v[NREG - 1] = hi;
            } else {
                const bool lower = (lane & j) == 0;
#pragma unroll
                for (int r = 0; r < NREG; ++r) {
                    const T o = __shfl_xor_sync(0xffffffffu, v[r], j);
                    const bool up = ((lane + 32 * r) & k) == 0;
                    v[r] = (lower == up) ? key_min(v[r], o) : key_max(v[r], o);
                }
            }
        }
    }
}

template <typename T>
__device__ __forceinline__ void warp_sort_row(T* __restrict__ col, int64_t s, int len, T* sm, int lane) {
    if (len <= 32) {
        T v[1] = {lane < len ? col[s + lane] : key_pad<T>()};      // padding sorts to the end (column ids are < INT32_MAX)
        warp_bitonic<1>(v, lane);
        if (lane < len) col[s + lane] = v[0];
        return;
    }
    if (len <= 64) {
        T v[2] = {col[s + lane], lane + 32 < len ? col[s + lane + 32] : key_pad<T>()};
        warp_bitonic<2>(v, lane);
        col[s + lane] = v[0];
        if (lane + 32 < len) col[s + lane + 32] = v[1];
        return;
    }
    int p2 = 128;
    while (p2 < len) p2 <<= 1;
    for (int i = lane; i < p2; i += 32) sm[i] = i < len ? col[s + i] : key_pad<T>();
    __syncwarp();
    for (int k = 2; k <= p2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < p2; i += 32) {
                int ixj = i ^ j;
                if (ixj > i) {
                    T x = sm[i], y = sm[ixj];
                    bool up = (i & k) == 0;
                    if ((x > y) == up) { sm[i] = y; sm[ixj] = x; }
                }
            }
            __syncwarp();
        }
    }
    for (int i = lane; i < len; i += 32) col[s + i] = sm[i];
    __syncwarp();
}

// one warp per row; rows longer than kWarpSortMax are queued for the block kernels
template <typename T>
__global__ void __launch_bounds__(256) csr_sort_rows_warp_kernel(const int64_t* __restrict__ rowptr, int64_t n,
                                                                  T* __restrict__ col, int64_t* __restrict__ long_rows,
                                                                  int* __restrict__ n_long) {
    __shared__ T sm_all[8][kWarpSortMax];
    const int lane = threadIdx.x & 31;
    T* sm = sm_all[threadIdx.x >> 5];
    int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        int64_t s = rowptr[r], e = rowptr[r + 1];
        int64_t len64 = e - s;
        if (len64 <= 1) continue;
        if (len64 > kWarpSortMax) {
            if (lane == 0) long_rows[atomicAdd(n_long, 1)] = r;
            continue;
        }
        warp_sort_row(col, s, (int)len64, sm, lane);
    }
}

// one block per queued long row whose padded length p2 satisfies min_p2 < p2 <= max_p2
template <typename T>
__global__ void csr_sort_rows_block_kernel(const int64_t* __restrict__ rowptr, T* __restrict__ col,
                                           const int64_t* __restrict__ long_rows, const int* __restrict__ n_long,
                                           T* __restrict__ scratch, int64_t scratch_per_block, int64_t min_p2,
                                           int64_t max_p2) {
    __shared__ T sm[kSortSmemMax];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int nq = *n_long;
    for (int q = blockIdx.x; q < nq; q += gridDim.x) {
        int64_t r = long_rows[q];
        int64_t s = rowptr[r];
        int64_t len = rowptr[r + 1] - s;
        int64_t p2 = 1;
        while (p2 < len) p2 <<= 1;
        if (p2 <= min_p2 || p2 > max_p2) continue;  // block-uniform
        if (p2 <= kSortSmemMax) {
            for (int i = tid; i < p2; i += nt) sm[i] = i < len ? col[s + i] : key_pad<T>();
            __syncthreads();
            bitonic_block(sm, (int)p2, tid, nt);
            for (int i = tid; i < len; i += nt) col[s + i] = sm[i];
            __syncthreads();
        } else {
            // hub rows: bitonic network in global scratch (padded to a power of two)
            T* g = scratch + (int64_t)blockIdx.x * scratch_per_block;
            for (int64_t i = tid; i < p2; i += nt) g[i] = i < len ? col[s + i] : key_pad<T>();
            __syncthreads();
            for (int64_t k = 2; k <= p2; k <<= 1) {
                for (int64_t j = k >> 1; j > 0; j >>= 1) {
                    for (int64_t i = tid; i < p2; i += nt) {
                        int64_t ixj = i ^ j;
                        if (ixj > i) {
                            T x = g[i], y = g[ixj];
                            bool up = (i & k) == 0;
                            if ((x > y) == up) { g[i] = y; g[ixj] = x; }
                        }
                    }
                    __syncthreads();
                }
            }
            for (int64_t i = tid; i < len; i += nt) col[s + i] = g[i];
            __syncthreads();
        }
    }
}

__global__ void csr_dinv_kernel(const int64_t* __restrict__ rowptr, int64_t n, float* __restrict__ dinv) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float d = (float)(rowptr[i + 1] - rowptr[i]);
        // same operation order as the reference: (1/d).sqrt(), inf -> 0   (large/ours.py:29-32)
        dinv[i] = d > 0.f ? sqrtf(1.0f / d) : 0.0f;
    }
}

// ---- weighted build ----------------------------------------------------------------------------------
// last[i] = position of node i's last self loop in edge order (-1: none); an atomicMax, so the result does not depend on the
// order in which the threads run (PyG's GPU scatter leaves that choice undefined).
__global__ void csr_last_loop_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ dst, int64_t nnz, int64_t n,
                                     long long* __restrict__ last) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        const int64_t r = src[e];
        if (r == dst[e] && r >= 0 && r < n) atomicMax(&last[r], (long long)e);
    }
}

// csr_fill_kernel writing the 64-bit key (col << 32 | e + 1) of edge e
__global__ void csr_fill_keyed_kernel(const int64_t* __restrict__ key, const int64_t* __restrict__ val, int64_t nnz,
                                      int64_t row_begin, int64_t row_end, int64_t n_cols, int drop_self_loops,
                                      const int64_t* __restrict__ rowptr, int* __restrict__ cursor, int64_t* __restrict__ keys) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        int64_t k = key[e];
        if (k < row_begin || k >= row_end) continue;
        int64_t v = val[e];
        if (v < 0 || v >= n_cols) continue;
        if (drop_self_loops && k == v) continue;
        int pos = atomicAdd(&cursor[k], 1);
        keys[rowptr[k] + pos] = (v << 32) | (e + 1);
    }
}

// the added self loop of node i takes the weight of i's last existing self loop (eid = last[i], -1 -> weight 1)
__global__ void csr_add_loops_keyed_kernel(int64_t n, const long long* __restrict__ last, const int64_t* __restrict__ rowptr,
                                           int* __restrict__ cursor, int64_t* __restrict__ keys) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        int pos = atomicAdd(&cursor[i], 1);
        keys[rowptr[i] + pos] = (i << 32) | (int64_t)(last[i] + 1);
    }
}

__global__ void csr_unpack_weighted_kernel(const int64_t* __restrict__ keys, const int64_t* __restrict__ rowptr, int64_t n,
                                           const float* __restrict__ w, int32_t* __restrict__ col, int64_t* __restrict__ eid,
                                           float* __restrict__ val) {
    const int64_t total = rowptr[n];
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < total; j += stride) {
        const int64_t k = keys[j];
        const int64_t e = (k & 0xffffffffLL) - 1;
        col[j] = (int32_t)(k >> 32);
        eid[j] = e;
        val[j] = e >= 0 ? w[e] : 1.0f;
    }
}

// weighted gcn_norm: deg[i] = sum of row i's values in CSR order (fp64, fixed order: bit-identical run to run),
// dinv = deg^-1/2 with inf -> 0 (a negative degree gives NaN, as PyG's pow does)
__global__ void csr_weighted_dinv_kernel(const int64_t* __restrict__ rowptr, const float* __restrict__ val, int64_t n,
                                         float* __restrict__ dinv) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        double d = 0.0;
        for (int64_t j = rowptr[i]; j < rowptr[i + 1]; ++j) d += (double)val[j];
        const float df = (float)d;
        dinv[i] = df == 0.f ? 0.f : (float)(1.0 / sqrt((double)df));
    }
}

__global__ void max_row_len_kernel(const int64_t* __restrict__ rowptr, int64_t n, unsigned long long* __restrict__ out) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned long long m = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        unsigned long long l = (unsigned long long)(rowptr[i + 1] - rowptr[i]);
        m = l > m ? l : m;
    }
    for (int o = 16; o > 0; o >>= 1) {
        unsigned long long t = __shfl_xor_sync(0xffffffffu, m, o);
        m = t > m ? t : m;
    }
    if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

// ---- K9: induced subgraph --------------------------------------------------------------------------
__global__ void fill_i32_kernel(int32_t* p, int64_t n, int32_t v) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}
__global__ void subgraph_map_kernel(const int64_t* __restrict__ subset, int64_t n_sub, int64_t n, int32_t* __restrict__ node_map) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_sub; i += stride) {
        int64_t v = subset[i];
        if (v >= 0 && v < n) node_map[v] = (int32_t)i;
    }
}
// flag + block-local count, order-preserving compaction in three steps (flags -> scan -> scatter)
__global__ void subgraph_flag_kernel(const int64_t* __restrict__ ei, int64_t nnz, int64_t n, const int32_t* __restrict__ node_map,
                                     int* __restrict__ flags) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        int64_t r = ei[e], c = ei[nnz + e];
        int keep = (r >= 0 && r < n && c >= 0 && c < n) ? (node_map[r] >= 0 && node_map[c] >= 0) : 0;
        flags[e] = keep;
    }
}
__global__ void subgraph_scatter_kernel(const int64_t* __restrict__ ei, int64_t nnz, const int32_t* __restrict__ node_map,
                                        const int* __restrict__ flags, const int64_t* __restrict__ pos,
                                        int64_t* __restrict__ out, int64_t out_pitch) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        if (!flags[e]) continue;
        int64_t p = pos[e];
        out[p] = node_map[ei[e]];
        out[out_pitch + p] = node_map[ei[nnz + e]];
    }
}

// ---- K9 on the CSR: induced subgraph of a node subset, emitted directly as the subset's CSR -----------------------------
// O(sum of the subset rows' lengths) instead of the O(E) mask over all edges of PyG subgraph (large/main-batch.py:139).
__global__ void subset_unmap_kernel(const int64_t* __restrict__ subset, int64_t n_sub, int64_t n, int32_t* __restrict__ node_map) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_sub; i += stride) {
        int64_t v = subset[i];
        if (v >= 0 && v < n) node_map[v] = -1;
    }
}
__global__ void subset_count_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                    const int64_t* __restrict__ subset, int64_t n_sub, int64_t n,
                                    const int32_t* __restrict__ node_map, int* __restrict__ counts) {
    const int lane = threadIdx.x & 31;
    int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n_sub; i += nwarps) {
        const int64_t v = subset[i];
        int c = 0;
        if (v >= 0 && v < n)
            for (int64_t j = rowptr[v] + lane; j < rowptr[v + 1]; j += 32) c += node_map[col[j]] >= 0;
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) counts[i] = c;
    }
}
// The caller's out_col holds `capacity` entries (a no-sync bound on the induced nnz): clamp the scanned row pointers to it so
// that the fill / sort / degree kernels never touch memory past the buffer, and report the true total so the host can tell.
__global__ void subset_clamp_kernel(int64_t* __restrict__ out_rowptr, int64_t n_sub, int64_t capacity, int64_t* __restrict__ needed) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n_sub; i += stride) {
        const int64_t v = out_rowptr[i];
        if (i == n_sub && needed) *needed = v;
        if (v > capacity) out_rowptr[i] = capacity;
    }
}
__global__ void subset_fill_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                   const int64_t* __restrict__ subset, int64_t n_sub, int64_t n,
                                   const int32_t* __restrict__ node_map, const int64_t* __restrict__ out_rowptr,
                                   int32_t* __restrict__ out_col) {
    const int lane = threadIdx.x & 31;
    int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n_sub; i += nwarps) {
        const int64_t v = subset[i];
        if (v < 0 || v >= n) continue;
        int64_t w = out_rowptr[i];
        const int64_t lim = out_rowptr[i + 1];      // == w + induced row length unless clamped to the buffer capacity
        const int64_t s = rowptr[v], e = rowptr[v + 1];
        for (int64_t base = s; base < e && w < lim; base += 32) {
            const int64_t j = base + lane;
            const int32_t m = j < e ? node_map[col[j]] : -1;
            const unsigned keep = __ballot_sync(0xffffffffu, m >= 0);
            const int64_t pos = w + __popc(keep & ((1u << lane) - 1u));
            if (m >= 0 && pos < lim) out_col[pos] = m;
            w += __popc(keep);
        }
    }
}

// ---- K10: graph preprocessing (torch_geometric.utils.to_undirected / remove_self_loops / add_self_loops) -----------------------
// remove_self_loops: order-preserving filter (flags -> scan -> scatter)
__global__ void selfloop_flag_kernel(const int64_t* __restrict__ ei, int64_t nnz, int* __restrict__ flags) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) flags[e] = ei[e] != ei[nnz + e];
}
__global__ void compact_edges_kernel(const int64_t* __restrict__ ei, int64_t nnz, const int* __restrict__ flags,
                                     const int64_t* __restrict__ pos, int64_t* __restrict__ out, int64_t out_pitch) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        if (!flags[e]) continue;
        int64_t p = pos[e];
        out[p] = ei[e];
        out[out_pitch + p] = ei[nnz + e];
    }
}
// add_self_loops: [edge_index | (i, i) for i in 0..n)
__global__ void add_self_loops_kernel(const int64_t* __restrict__ ei, int64_t nnz, int64_t n, int64_t* __restrict__ out) {
    const int64_t pitch = nnz + n;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < pitch; e += stride) {
        out[e] = e < nnz ? ei[e] : e - nnz;
        out[pitch + e] = e < nnz ? ei[nnz + e] : e - nnz;
    }
}
// to_undirected = coalesce([ei | ei.flip(0)]): the doubled list is never materialised - the CSR count / fill kernels run once per
// direction into the same rows, rows are sorted, then a sorted row's first occurrences are counted and emitted as COO (row, col).
__global__ void __launch_bounds__(256) row_unique_count_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                               int64_t n, int* __restrict__ ucount) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp0; r < n; r += nwarps) {
        const int64_t s = rowptr[r], e = rowptr[r + 1];
        int cnt = 0;
        for (int64_t j = s + lane; j < e; j += 32) cnt += (j == s || col[j] != col[j - 1]) ? 1 : 0;
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if (lane == 0) ucount[r] = cnt;
    }
}
__global__ void __launch_bounds__(256) row_unique_emit_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                              int64_t n, const int64_t* __restrict__ uptr,
                                                              int64_t* __restrict__ out, int64_t out_pitch) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp0; r < n; r += nwarps) {
        const int64_t s = rowptr[r], e = rowptr[r + 1];
        int64_t base = uptr[r];
        for (int64_t j0 = s; j0 < e; j0 += 32) {
            const int64_t j = j0 + lane;
            const bool keep = j < e && (j == s || col[j] != col[j - 1]);
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (keep) {
                const int64_t p = base + __popc(m & ((1u << lane) - 1u));
                out[p] = r;
                out[out_pitch + p] = col[j];
            }
            base += __popc(m);
        }
    }
}

// Order-independent 64-bit hash sums of {(r,c)} and {(c,r)}: equal sums <=> the edge multiset is symmetric (up to a 2^-64 collision).
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x *= 0x9E3779B97F4A7C15ULL; x ^= x >> 29;
    x *= 0xBF58476D1CE4E5B9ULL; x ^= x >> 32;
    x *= 0x94D049BB133111EBULL; x ^= x >> 31;
    return x;
}
__global__ void __launch_bounds__(256) edge_symmetry_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ dst, int64_t nnz,
                                                            uint64_t n, unsigned long long* __restrict__ out) {
    uint64_t h1 = 0, h2 = 0;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        const uint64_t r = (uint64_t)src[e], c = (uint64_t)dst[e];
        h1 += mix64(r * n + c);
        h2 += mix64(c * n + r);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        h1 += __shfl_xor_sync(0xffffffffu, h1, o);
        h2 += __shfl_xor_sync(0xffffffffu, h2, o);
    }
    __shared__ uint64_t sm[2][8];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) { sm[0][w] = h1; sm[1][w] = h2; }
    __syncthreads();
    if (threadIdx.x < 2) {
        uint64_t t = 0;
        for (int i = 0; i < 8; ++i) t += sm[threadIdx.x][i];
        atomicAdd(&out[threadIdx.x], (unsigned long long)t);
    }
}

// as edge_symmetry_kernel over {(r, c, w)} and {(c, r, w)}: the weight's bit pattern is mixed into every term, so a symmetric
// pattern whose weights are not symmetric hashes differently
__global__ void __launch_bounds__(256) edge_symmetry_weighted_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ dst,
                                                                     const float* __restrict__ w, int64_t nnz, uint64_t n,
                                                                     unsigned long long* __restrict__ out) {
    uint64_t h1 = 0, h2 = 0;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        const uint64_t r = (uint64_t)src[e], c = (uint64_t)dst[e];
        const uint64_t wb = mix64((uint64_t)__float_as_uint(w[e]) + 0x632BE59BD9B4E019ULL);
        h1 += mix64(mix64(r * n + c) ^ wb);
        h2 += mix64(mix64(c * n + r) ^ wb);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        h1 += __shfl_xor_sync(0xffffffffu, h1, o);
        h2 += __shfl_xor_sync(0xffffffffu, h2, o);
    }
    __shared__ uint64_t sm[2][8];
    const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
    if (lane == 0) { sm[0][wi] = h1; sm[1][wi] = h2; }
    __syncthreads();
    if (threadIdx.x < 2) {
        uint64_t t = 0;
        for (int i = 0; i < 8; ++i) t += sm[threadIdx.x][i];
        atomicAdd(&out[threadIdx.x], (unsigned long long)t);
    }
}

static inline int grid_for(int64_t work, int block, int per_sm = 8) {
    int64_t g = (work + block - 1) / block;
    int64_t cap = (int64_t)num_sms() * per_sm;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Row-window size of the CSR fill in bytes of `col` (SGF_CSR_FILL_WINDOW_MB, 0 = one launch); at most kMaxFillWindows launches, so
// beyond kMaxFillWindows x window bytes the windows simply grow.
static constexpr int64_t kMaxFillWindows = 12;
static inline int64_t fill_window_bytes() {
    static const int64_t v = [] {
        const char* e = std::getenv("SGF_CSR_FILL_WINDOW_MB");
        return (int64_t)(e ? std::atoi(e) : 128) << 20;
    }();
    return v;
}

// Row windows [lo, hi) of the fill, each written by one launch (sizes: fill_window_bytes of entry_bytes-sized entries)
template <typename Launch>
static int for_fill_windows(int64_t nnz, int64_t row_begin, int64_t row_end, int64_t entry_bytes, Launch launch) {
    const int64_t n = row_end - row_begin;
    const int64_t win_bytes = fill_window_bytes();
    int64_t nwin = win_bytes > 0 ? ((nnz + n) * entry_bytes + win_bytes - 1) / win_bytes : 1;
    if (nwin > kMaxFillWindows) nwin = kMaxFillWindows;
    if (nwin < 1 || n == 0) nwin = 1;
    const int64_t rows_per = (n + nwin - 1) / nwin;
    for (int64_t wi = 0; wi < nwin; ++wi) {
        const int64_t lo = row_begin + wi * rows_per, hi = lo + rows_per < row_end ? lo + rows_per : row_end;
        if (nwin > 1 && lo >= hi) break;
        launch(nwin > 1 ? lo : row_begin, nwin > 1 ? hi : row_end);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    return SGF_OK;
}

// exclusive scan of int counts (+add) into int64 out[0..n], using block_sums scratch
static int launch_scan(const int* counts, int64_t n, int add_loop, int64_t* rowptr, int64_t* block_sums,
                       int64_t* total, int* cursor, cudaStream_t st) {
    int64_t per_block = (int64_t)kScanBlock * kScanItems;
    int64_t nblocks = (n + per_block - 1) / per_block;
    if (nblocks < 1) nblocks = 1;
    scan_local_kernel<<<(unsigned)nblocks, kScanBlock, 0, st>>>(counts, n, add_loop, rowptr, block_sums);
    SGF_LAUNCH_CHECK(); count_launch();
    scan_block_sums_kernel<<<1, kScanBlock, 0, st>>>(block_sums, nblocks, total);
    SGF_LAUNCH_CHECK(); count_launch();
    scan_add_kernel<<<grid_for(n + 1, 256), 256, 0, st>>>(rowptr, n, block_sums, total, cursor, add_loop);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

}  // namespace sgf

using namespace sgf;

// workspace layout: counts int32[n] | cursor int32[n] | block_sums int64[nb] | total int64 | err int32 | n_long int32 |
//                   maxlen u64 | long_rows int64[n] | hub scratch int32[...]
struct CsrWs {
    int* counts; int* cursor; int64_t* block_sums; int64_t* total; int* err; int* n_long;
    unsigned long long* maxlen; int64_t* long_rows; int32_t* scratch; int64_t scratch_elems;
    size_t bytes;
};
static constexpr int kHubBlocks = 16;
// hub-row scratch cap (ints): rows longer than this (only possible with > 2^26 parallel edges into one node) are left
// in fill order — still a valid CSR for the SpMM, but not bit-comparable.
static constexpr int64_t kHubScratchMax = (int64_t)1 << 26;

static CsrWs carve_ws(void* ws, int64_t nnz, int64_t n, size_t key_bytes = 4) {
    CsrWs w;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    int64_t per_block = (int64_t)kScanBlock * kScanItems;
    int64_t nb = (n + per_block - 1) / per_block + 1;
    char* base = (char*)ws;
    size_t o_counts = take((size_t)(n + 1) * 4), o_cursor = take((size_t)(n + 1) * 4), o_bs = take((size_t)nb * 8);
    size_t o_misc = take(64), o_long = take((size_t)(n + 1) * 8);
    // hub scratch: each of kHubBlocks blocks may need next_pow2(longest row) <= next_pow2(nnz + n) ints; sized lazily:
    // we reserve 2*(nnz+n) ints in total and give every block an equal share (rows longer than a share are split... never:
    // a row longer than share means few such rows exist; the kernel is launched with fewer blocks in that case).
    int64_t tot = nnz + n;
    int64_t p2 = kSortSmemMax * kHubBlocks;
    while (p2 < tot && p2 < kHubScratchMax) p2 <<= 1;
    size_t o_scr = take((size_t)p2 * key_bytes);
    w.counts = (int*)(base + o_counts); w.cursor = (int*)(base + o_cursor); w.block_sums = (int64_t*)(base + o_bs);
    w.total = (int64_t*)(base + o_misc); w.err = (int*)(base + o_misc + 8); w.n_long = (int*)(base + o_misc + 12);
    w.maxlen = (unsigned long long*)(base + o_misc + 16);
    w.long_rows = (int64_t*)(base + o_long); w.scratch = (int32_t*)(base + o_scr); w.scratch_elems = p2;
    w.bytes = off;
    return w;
}

// per-row ascending sort of col (tiers by row length; see the kernels)
template <typename T> static int sort_long_rows(const int64_t* rowptr, T* col, const CsrWs& w, cudaStream_t st);
template <typename T>
static int sort_rows(const int64_t* rowptr, T* col, int64_t n, const CsrWs& w, cudaStream_t st) {
    csr_sort_rows_warp_kernel<<<grid_for(n * 32, 256), 256, 0, st>>>(rowptr, n, col, w.long_rows, w.n_long);
    SGF_LAUNCH_CHECK(); count_launch();
    return sort_long_rows(rowptr, col, w, st);
}
// the rows queued in w.long_rows (longer than kWarpSortMax)
template <typename T>
static int sort_long_rows(const int64_t* rowptr, T* col, const CsrWs& w, cudaStream_t st) {
    T* scratch = reinterpret_cast<T*>(w.scratch);
    int64_t share = w.scratch_elems / kHubBlocks;
    // queued rows: (256, 2048] in shared memory across the whole chip; (2048, share] in global scratch by kHubBlocks
    // blocks; (share, scratch] by a single block.
    csr_sort_rows_block_kernel<<<num_sms() * 4, 256, 0, st>>>(rowptr, col, w.long_rows, w.n_long, scratch, 0, 0, kSortSmemMax);
    SGF_LAUNCH_CHECK(); count_launch();
    csr_sort_rows_block_kernel<<<kHubBlocks, 1024, 0, st>>>(rowptr, col, w.long_rows, w.n_long, scratch, share, kSortSmemMax, share);
    SGF_LAUNCH_CHECK(); count_launch();
    csr_sort_rows_block_kernel<<<1, 1024, 0, st>>>(rowptr, col, w.long_rows, w.n_long, scratch, w.scratch_elems, share, w.scratch_elems);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_csr_build_ws_bytes(int64_t nnz, int64_t n, size_t* bytes) {
    if (!bytes || nnz < 0 || n < 0) return SGF_ERR_ARG;
    *bytes = carve_ws(nullptr, nnz, n).bytes;
    return SGF_OK;
}

extern "C" int sgf_csr_build_rect(const int64_t* edge_index, int64_t nnz, int64_t row_begin, int64_t row_end, int64_t n_cols,
                                  int by_source, int self_loop_mode, int64_t* rowptr, int32_t* col, float* dinv, void* ws,
                                  size_t ws_bytes, void* stream) {
    return sgf_csr_build_rot(edge_index, nnz, row_begin, row_end, n_cols, by_source, self_loop_mode, 0, 0, rowptr, col, dinv, ws,
                             ws_bytes, stream);
}

extern "C" int sgf_csr_build_rot(const int64_t* edge_index, int64_t nnz, int64_t row_begin, int64_t row_end, int64_t n_cols,
                                 int by_source, int self_loop_mode, int64_t col_rot, int64_t col_mod, int64_t* rowptr, int32_t* col,
                                 float* dinv, void* ws, size_t ws_bytes, void* stream) {
    const int64_t n = row_end - row_begin;
    if (nnz < 0 || n < 0 || row_begin < 0 || row_end > n_cols || n_cols >= (int64_t)INT32_MAX || !rowptr ||
        (!col && nnz + n > 0) || !ws)
        return SGF_ERR_ARG;
    if (col_mod != 0 && (col_mod < n_cols || col_mod >= (int64_t)INT32_MAX || col_rot < 0 || col_rot >= col_mod)) return SGF_ERR_ARG;
    if (nnz > 0 && !edge_index) return SGF_ERR_ARG;
    if (self_loop_mode != 0 && self_loop_mode != 1) return SGF_ERR_ARG;
    CsrWs w = carve_ws(ws, nnz, n);
    if (ws_bytes < w.bytes) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t* key = by_source ? edge_index : edge_index + nnz;
    const int64_t* val = by_source ? edge_index + nnz : edge_index;
    SGF_CUDA_TRY(cudaMemsetAsync(w.total, 0, 64, st));
    SGF_CUDA_TRY(cudaMemsetAsync(w.counts, 0, (size_t)(n + 1) * 4, st));
    if (nnz > 0) {
        csr_count_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(key, val, nnz, row_begin, row_end, n_cols, self_loop_mode, w.counts, w.err);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    int rc = launch_scan(w.counts, n, self_loop_mode, rowptr, w.block_sums, w.total, w.cursor, st);
    if (rc) return rc;
    if (nnz > 0) {
        // The fill scatters 4-byte entries over `col`; when `col` is much larger than the L2 every write is a DRAM sector
        // read-modify-write.  Row windows confine the writes of a launch to a piece of `col`, so that more of them hit lines
        // already in L2 and are written back whole, at the price of re-reading the keys once per window.  The 128 MB window
        // exceeds the 50 MB L2 of an H100 yet builds the products-shaped CSR faster than a 40 MB one (13.9 vs 16.0 ms,
        // scripts/bench_csr.py on an H100 at a 400 W power limit): fewer windows re-read the keys fewer times.
        const int rcf = for_fill_windows(nnz, row_begin, row_end, 4, [&](int64_t lo, int64_t hi) {
            csr_fill_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(key, val, nnz, row_begin, lo, hi, n_cols, self_loop_mode, rowptr,
                                                               w.cursor, col);
        });
        if (rcf) return rcf;
    }
    if (self_loop_mode == 1 && n > 0) {
        csr_add_loops_kernel<<<grid_for(n, 256), 256, 0, st>>>(n, row_begin, rowptr, w.cursor, col);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    if (n > 0) {
        if (col_mod > 0 && nnz + n > 0) {
            csr_rotate_cols_kernel<<<grid_for(nnz + n, 256), 256, 0, st>>>(col, rowptr, n, col_rot, col_mod);
            SGF_LAUNCH_CHECK(); count_launch();
        }
        int rcs = sort_rows(rowptr, col, n, w, st);
        if (rcs) return rcs;
        if (dinv) {
            csr_dinv_kernel<<<grid_for(n, 256), 256, 0, st>>>(rowptr, n, dinv);
            SGF_LAUNCH_CHECK(); count_launch();
        }
    } else {
        SGF_CUDA_TRY(cudaMemsetAsync(rowptr, 0, 8, st));
    }
    return SGF_OK;
}

extern "C" int sgf_csr_row_splits(const int64_t* rowptr, const int32_t* col, int64_t n_rows, const int32_t* thresholds, int n_thr,
                                  int32_t* splits, void* stream) {
    if (!rowptr || n_rows < 0 || n_thr < 0 || (n_thr > 0 && (!thresholds || !splits))) return SGF_ERR_ARG;
    if (n_rows == 0 || n_thr == 0) return SGF_OK;
    csr_row_splits_kernel<<<grid_for(n_rows * n_thr, 256), 256, 0, (cudaStream_t)stream>>>(rowptr, col, n_rows, n_thr, thresholds, splits);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_csr_build(const int64_t* edge_index, int64_t nnz, int64_t n, int by_source, int self_loop_mode,
                             int64_t* rowptr, int32_t* col, float* dinv, void* ws, size_t ws_bytes, void* stream) {
    return sgf_csr_build_rect(edge_index, nnz, 0, n, n, by_source, self_loop_mode, rowptr, col, dinv, ws, ws_bytes, stream);
}

// workspace: flags int32[nnz] | pos int64[nnz+1] | block_sums | total
extern "C" int sgf_subgraph_ws_bytes(int64_t nnz, int64_t n, size_t* bytes) {
    if (!bytes || nnz < 0 || n < 0) return SGF_ERR_ARG;
    int64_t per_block = (int64_t)kScanBlock * kScanItems;
    int64_t nb = (nnz + per_block - 1) / per_block + 1;
    *bytes = align_up((size_t)(nnz + 1) * 4, 256) * 2 + align_up((size_t)(nnz + 1) * 8, 256) + align_up((size_t)nb * 8, 256) + 256;
    return SGF_OK;
}

extern "C" int sgf_subgraph(const int64_t* edge_index, int64_t nnz, int64_t n, const int64_t* subset, int64_t n_sub,
                            int32_t* node_map, int64_t* out_edge_index, int64_t* out_count, void* ws, size_t ws_bytes,
                            void* stream) {
    if (nnz < 0 || n < 0 || n_sub < 0 || !node_map || !out_count || !ws) return SGF_ERR_ARG;
    size_t need = 0;
    sgf_subgraph_ws_bytes(nnz, n, &need);
    if (ws_bytes < need) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    char* base = (char*)ws;
    size_t off = 0;
    int* flags = (int*)(base + off); off += align_up((size_t)(nnz + 1) * 4, 256);
    int* cursor = (int*)(base + off); off += align_up((size_t)(nnz + 1) * 4, 256);
    int64_t* pos = (int64_t*)(base + off); off += align_up((size_t)(nnz + 1) * 8, 256);
    int64_t per_block = (int64_t)kScanBlock * kScanItems;
    int64_t nb = (nnz + per_block - 1) / per_block + 1;
    int64_t* block_sums = (int64_t*)(base + off); off += align_up((size_t)nb * 8, 256);
    (void)cursor;
    fill_i32_kernel<<<grid_for(n, 256), 256, 0, st>>>(node_map, n, -1);
    SGF_LAUNCH_CHECK(); count_launch();
    if (n_sub > 0) {
        subgraph_map_kernel<<<grid_for(n_sub, 256), 256, 0, st>>>(subset, n_sub, n, node_map);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    if (nnz == 0) {
        SGF_CUDA_TRY(cudaMemsetAsync(out_count, 0, 8, st));
        return SGF_OK;
    }
    subgraph_flag_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(edge_index, nnz, n, node_map, flags);
    SGF_LAUNCH_CHECK(); count_launch();
    int rc = launch_scan(flags, nnz, 0, pos, block_sums, out_count, cursor, st);
    if (rc) return rc;
    subgraph_scatter_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(edge_index, nnz, node_map, flags, pos, out_edge_index, nnz);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

// workspace: counts int32[n_sub+1] | cursor int32[n_sub+1] | block_sums | misc | long_rows int64[n_sub+1] | sort scratch
extern "C" int sgf_csr_subset_ws_bytes(int64_t n_sub, int64_t max_out_nnz, size_t* bytes) {
    if (!bytes || n_sub < 0 || max_out_nnz < 0) return SGF_ERR_ARG;
    *bytes = carve_ws(nullptr, max_out_nnz, n_sub).bytes;
    return SGF_OK;
}

extern "C" int sgf_csr_subset(const int64_t* rowptr, const int32_t* col, int64_t n, const int64_t* subset, int64_t n_sub,
                              int32_t* node_map, int64_t* out_rowptr, int32_t* out_col, int64_t out_col_capacity, float* dinv,
                              int64_t* out_needed, void* ws, size_t ws_bytes, void* stream) {
    if (!rowptr || n < 0 || n_sub < 0 || !node_map || !out_rowptr || !ws || (n_sub > 0 && !subset) || out_col_capacity < 0)
        return SGF_ERR_ARG;
    CsrWs w = carve_ws(ws, out_col_capacity, n_sub);
    if (ws_bytes < w.bytes) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (n_sub == 0) {
        SGF_CUDA_TRY(cudaMemsetAsync(out_rowptr, 0, 8, st));
        if (out_needed) SGF_CUDA_TRY(cudaMemsetAsync(out_needed, 0, 8, st));
        return SGF_OK;
    }
    SGF_CUDA_TRY(cudaMemsetAsync(w.total, 0, 64, st));
    // node_map holds -1 everywhere on entry (maintained by the caller across batches) and is restored on exit
    subgraph_map_kernel<<<grid_for(n_sub, 256), 256, 0, st>>>(subset, n_sub, n, node_map);
    SGF_LAUNCH_CHECK(); count_launch();
    subset_count_kernel<<<grid_for(n_sub * 32, 256), 256, 0, st>>>(rowptr, col, subset, n_sub, n, node_map, w.counts);
    SGF_LAUNCH_CHECK(); count_launch();
    int rc = launch_scan(w.counts, n_sub, 0, out_rowptr, w.block_sums, w.total, w.cursor, st);
    if (rc) return rc;
    subset_clamp_kernel<<<grid_for(n_sub + 1, 256), 256, 0, st>>>(out_rowptr, n_sub, out_col_capacity, out_needed);
    SGF_LAUNCH_CHECK(); count_launch();
    subset_fill_kernel<<<grid_for(n_sub * 32, 256), 256, 0, st>>>(rowptr, col, subset, n_sub, n, node_map, out_rowptr, out_col);
    SGF_LAUNCH_CHECK(); count_launch();
    subset_unmap_kernel<<<grid_for(n_sub, 256), 256, 0, st>>>(subset, n_sub, n, node_map);
    SGF_LAUNCH_CHECK(); count_launch();
    // local ids are a permutation of the global ones: restore sorted rows (canonical CSR)
    csr_sort_rows_warp_kernel<<<grid_for(n_sub * 32, 256), 256, 0, st>>>(out_rowptr, n_sub, out_col, w.long_rows, w.n_long);
    SGF_LAUNCH_CHECK(); count_launch();
    int64_t share = w.scratch_elems / kHubBlocks;
    csr_sort_rows_block_kernel<<<num_sms() * 4, 256, 0, st>>>(out_rowptr, out_col, w.long_rows, w.n_long, w.scratch, 0, 0, kSortSmemMax);
    SGF_LAUNCH_CHECK(); count_launch();
    csr_sort_rows_block_kernel<<<kHubBlocks, 1024, 0, st>>>(out_rowptr, out_col, w.long_rows, w.n_long, w.scratch, share, kSortSmemMax, share);
    SGF_LAUNCH_CHECK(); count_launch();
    if (dinv) {
        csr_dinv_kernel<<<grid_for(n_sub, 256), 256, 0, st>>>(out_rowptr, n_sub, dinv);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    return SGF_OK;
}

// ---- K10 host side ---------------------------------------------------------------------------------------------------------
// workspace of remove_self_loops: flags int32[nnz+1] | pos int64[nnz+1] | block_sums
extern "C" int sgf_remove_self_loops_ws_bytes(int64_t nnz, size_t* bytes) {
    if (!bytes || nnz < 0) return SGF_ERR_ARG;
    int64_t per_block = (int64_t)kScanBlock * kScanItems;
    int64_t nb = (nnz + per_block - 1) / per_block + 1;
    *bytes = align_up((size_t)(nnz + 1) * 4, 256) * 2 + align_up((size_t)(nnz + 1) * 8, 256) + align_up((size_t)nb * 8, 256) + 256;
    return SGF_OK;
}

extern "C" int sgf_remove_self_loops(const int64_t* edge_index, int64_t nnz, int64_t* out_edge_index, int64_t* out_count, void* ws,
                                     size_t ws_bytes, void* stream) {
    if (nnz < 0 || !out_count || !ws || (nnz > 0 && (!edge_index || !out_edge_index))) return SGF_ERR_ARG;
    size_t need = 0;
    sgf_remove_self_loops_ws_bytes(nnz, &need);
    if (ws_bytes < need) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (nnz == 0) {
        SGF_CUDA_TRY(cudaMemsetAsync(out_count, 0, 8, st));
        return SGF_OK;
    }
    char* base = (char*)ws;
    size_t off = 0;
    int* flags = (int*)(base + off); off += align_up((size_t)(nnz + 1) * 4, 256);
    int* cursor = (int*)(base + off); off += align_up((size_t)(nnz + 1) * 4, 256);
    int64_t* pos = (int64_t*)(base + off); off += align_up((size_t)(nnz + 1) * 8, 256);
    int64_t* block_sums = (int64_t*)(base + off);
    selfloop_flag_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(edge_index, nnz, flags);
    SGF_LAUNCH_CHECK(); count_launch();
    int rc = launch_scan(flags, nnz, 0, pos, block_sums, out_count, cursor, st);
    if (rc) return rc;
    compact_edges_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(edge_index, nnz, flags, pos, out_edge_index, nnz);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_add_self_loops(const int64_t* edge_index, int64_t nnz, int64_t n, int64_t* out_edge_index, void* stream) {
    if (nnz < 0 || n < 0 || (nnz > 0 && !edge_index) || (nnz + n > 0 && !out_edge_index)) return SGF_ERR_ARG;
    if (nnz + n == 0) return SGF_OK;
    add_self_loops_kernel<<<grid_for(nnz + n, 256), 256, 0, (cudaStream_t)stream>>>(edge_index, nnz, n, out_edge_index);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

// workspace of to_undirected: CsrWs(2 nnz, n) | rowptr int64[n+1] | uptr int64[n+1] | ucount int32[n+1] | ucursor int32[n+1] |
//                             block_sums2 | col int32[2 nnz]
struct UndWs {
    CsrWs csr; int64_t* rowptr; int64_t* uptr; int* ucount; int* ucursor; int64_t* block_sums2; int32_t* col; size_t bytes;
};
static UndWs carve_und(void* ws, int64_t nnz, int64_t n) {
    UndWs u;
    u.csr = carve_ws(ws, 2 * nnz, n);
    size_t off = align_up(u.csr.bytes, 256);
    auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
    char* base = (char*)ws;
    int64_t per_block = (int64_t)kScanBlock * kScanItems;
    int64_t nb = (n + per_block - 1) / per_block + 1;
    size_t o_rp = take((size_t)(n + 1) * 8), o_up = take((size_t)(n + 1) * 8), o_uc = take((size_t)(n + 1) * 4);
    size_t o_cu = take((size_t)(n + 1) * 4), o_bs = take((size_t)nb * 8), o_col = take((size_t)(2 * nnz + 1) * 4);
    u.rowptr = (int64_t*)(base + o_rp); u.uptr = (int64_t*)(base + o_up); u.ucount = (int*)(base + o_uc);
    u.ucursor = (int*)(base + o_cu); u.block_sums2 = (int64_t*)(base + o_bs); u.col = (int32_t*)(base + o_col);
    u.bytes = off;
    return u;
}

extern "C" int sgf_to_undirected_ws_bytes(int64_t nnz, int64_t n, size_t* bytes) {
    if (!bytes || nnz < 0 || n < 0) return SGF_ERR_ARG;
    *bytes = carve_und(nullptr, nnz, n).bytes;
    return SGF_OK;
}

extern "C" int sgf_to_undirected(const int64_t* edge_index, int64_t nnz, int64_t n, int64_t* out_edge_index, int64_t* out_count,
                                 void* ws, size_t ws_bytes, void* stream) {
    if (nnz < 0 || n < 0 || n >= (int64_t)INT32_MAX || !out_count || !ws || (nnz > 0 && (!edge_index || !out_edge_index)))
        return SGF_ERR_ARG;
    UndWs u = carve_und(ws, nnz, n);
    if (ws_bytes < u.bytes) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (nnz == 0 || n == 0) {
        SGF_CUDA_TRY(cudaMemsetAsync(out_count, 0, 8, st));
        return nnz == 0 ? SGF_OK : SGF_ERR_ARG;
    }
    const CsrWs& w = u.csr;
    const int64_t* row = edge_index;
    const int64_t* colv = edge_index + nnz;
    SGF_CUDA_TRY(cudaMemsetAsync(w.counts, 0, (size_t)(n + 1) * 4, st));
    SGF_CUDA_TRY(cudaMemsetAsync(w.total, 0, 64, st));
    // both directions into the same rows: (row -> col) and (col -> row)
    csr_count_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(row, colv, nnz, 0, n, n, 0, w.counts, w.err);
    SGF_LAUNCH_CHECK(); count_launch();
    csr_count_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(colv, row, nnz, 0, n, n, 0, w.counts, w.err);
    SGF_LAUNCH_CHECK(); count_launch();
    int rc = launch_scan(w.counts, n, 0, u.rowptr, w.block_sums, w.total, w.cursor, st);
    if (rc) return rc;
    csr_fill_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(row, colv, nnz, 0, 0, n, n, 0, u.rowptr, w.cursor, u.col);
    SGF_LAUNCH_CHECK(); count_launch();
    csr_fill_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(colv, row, nnz, 0, 0, n, n, 0, u.rowptr, w.cursor, u.col);
    SGF_LAUNCH_CHECK(); count_launch();
    if ((rc = sort_rows(u.rowptr, u.col, n, w, st))) return rc;
    row_unique_count_kernel<<<grid_for(n * 32, 256), 256, 0, st>>>(u.rowptr, u.col, n, u.ucount);
    SGF_LAUNCH_CHECK(); count_launch();
    if ((rc = launch_scan(u.ucount, n, 0, u.uptr, u.block_sums2, out_count, u.ucursor, st))) return rc;
    row_unique_emit_kernel<<<grid_for(n * 32, 256), 256, 0, st>>>(u.rowptr, u.col, n, u.uptr, out_edge_index, 2 * nnz);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_edge_symmetry(const int64_t* edge_index, int64_t nnz, int64_t n, uint64_t* out2, void* stream) {
    if (nnz < 0 || n < 0 || !out2 || (nnz > 0 && !edge_index)) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    SGF_CUDA_TRY(cudaMemsetAsync(out2, 0, 16, st));
    if (nnz == 0) return SGF_OK;
    edge_symmetry_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(edge_index, edge_index + nnz, nnz, (uint64_t)n,
                                                            reinterpret_cast<unsigned long long*>(out2));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

// ---- weighted build ----------------------------------------------------------------------------------------------------------
// workspace: CsrWs with 8-byte sort scratch | keys int64[nnz + n] | last int64[n]
struct WCsrWs { CsrWs csr; int64_t* keys; long long* last; size_t bytes; };
static WCsrWs carve_wws(void* ws, int64_t nnz, int64_t n) {
    WCsrWs u;
    u.csr = carve_ws(ws, nnz, n, 8);
    size_t off = align_up(u.csr.bytes, 256);
    char* base = (char*)ws;
    u.keys = (int64_t*)(base + off); off = align_up(off + (size_t)(nnz + n + 1) * 8, 256);
    u.last = (long long*)(base + off); off = align_up(off + (size_t)(n + 1) * 8, 256);
    u.bytes = off;
    return u;
}

extern "C" int sgf_csr_build_weighted_ws_bytes(int64_t nnz, int64_t n, size_t* bytes) {
    if (!bytes || nnz < 0 || n < 0) return SGF_ERR_ARG;
    *bytes = carve_wws(nullptr, nnz, n).bytes;
    return SGF_OK;
}

extern "C" int sgf_csr_build_weighted(const int64_t* edge_index, const float* weight, int64_t nnz, int64_t n, int by_source,
                                      int self_loop_mode, int64_t* rowptr, int32_t* col, int64_t* eid, float* val, float* dinv,
                                      void* ws, size_t ws_bytes, void* stream) {
    if (nnz < 0 || n < 0 || n >= (int64_t)INT32_MAX || nnz >= (int64_t)UINT32_MAX || !rowptr || !ws) return SGF_ERR_ARG;
    if (nnz + n > 0 && (!col || !eid || !val)) return SGF_ERR_ARG;
    if (nnz > 0 && (!edge_index || !weight)) return SGF_ERR_ARG;
    if (self_loop_mode != 0 && self_loop_mode != 1) return SGF_ERR_ARG;
    WCsrWs u = carve_wws(ws, nnz, n);
    if (ws_bytes < u.bytes) return SGF_ERR_ARG;
    const CsrWs& w = u.csr;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t* key = by_source ? edge_index : edge_index + nnz;
    const int64_t* other = by_source ? edge_index + nnz : edge_index;
    SGF_CUDA_TRY(cudaMemsetAsync(w.total, 0, 64, st));
    SGF_CUDA_TRY(cudaMemsetAsync(w.counts, 0, (size_t)(n + 1) * 4, st));
    if (n == 0) return cudaMemsetAsync(rowptr, 0, 8, st) == cudaSuccess ? SGF_OK : SGF_ERR_ARG;
    if (nnz > 0) {
        csr_count_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(key, other, nnz, 0, n, n, self_loop_mode, w.counts, w.err);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    int rc = launch_scan(w.counts, n, self_loop_mode, rowptr, w.block_sums, w.total, w.cursor, st);
    if (rc) return rc;
    if (nnz > 0) {
        rc = for_fill_windows(nnz, 0, n, 8, [&](int64_t lo, int64_t hi) {
            csr_fill_keyed_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(key, other, nnz, lo, hi, n, self_loop_mode, rowptr, w.cursor,
                                                                     u.keys);
        });
        if (rc) return rc;
    }
    if (self_loop_mode == 1) {
        SGF_CUDA_TRY(cudaMemsetAsync(u.last, 0xff, (size_t)n * 8, st));      // -1: no self loop
        if (nnz > 0) {
            csr_last_loop_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(edge_index, edge_index + nnz, nnz, n, u.last);
            SGF_LAUNCH_CHECK(); count_launch();
        }
        csr_add_loops_keyed_kernel<<<grid_for(n, 256), 256, 0, st>>>(n, u.last, rowptr, w.cursor, u.keys);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    if ((rc = sort_rows(rowptr, u.keys, n, w, st))) return rc;
    csr_unpack_weighted_kernel<<<grid_for(nnz + n, 256), 256, 0, st>>>(u.keys, rowptr, n, weight, col, eid, val);
    SGF_LAUNCH_CHECK(); count_launch();
    if (dinv) {
        if (self_loop_mode == 1) csr_weighted_dinv_kernel<<<grid_for(n, 256), 256, 0, st>>>(rowptr, val, n, dinv);
        else csr_dinv_kernel<<<grid_for(n, 256), 256, 0, st>>>(rowptr, n, dinv);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    return SGF_OK;
}

extern "C" int sgf_edge_symmetry_weighted(const int64_t* edge_index, const float* weight, int64_t nnz, int64_t n, uint64_t* out2,
                                          void* stream) {
    if (nnz < 0 || n < 0 || !out2 || (nnz > 0 && (!edge_index || !weight))) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    SGF_CUDA_TRY(cudaMemsetAsync(out2, 0, 16, st));
    if (nnz == 0) return SGF_OK;
    edge_symmetry_weighted_kernel<<<grid_for(nnz, 256), 256, 0, st>>>(edge_index, edge_index + nnz, weight, nnz, (uint64_t)n,
                                                                     reinterpret_cast<unsigned long long*>(out2));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}
