// K6 / K7 — CSR SpMM  y[r,:] = row_scale[r] * sum_{j in row r} x[col[j], :]
//
// Replaces torch_sparse.matmul(adj, x) (reference large/ours.py:34, 100M/ours.py:80; torch_sparse 0.6.10 spmm_kernel:
// fp32, int64 indices, value array, one warp per row x 32 feature columns) and its autograd transpose.
//
// Design (pure HBM-bound gather, no tensor cores):
//   * no value array: Â = D^-1/2 A D^-1/2 is applied as a row pre-scale in the producer of x and `row_scale` here,
//     which removes 4 B/nnz and one dependent gather;
//   * int32 column ids, int64 rowptr (nnz may exceed 2^31);
//   * one warp per output row; a feature row is split into 16-byte chunks, `lpr` lanes cover one neighbour row with
//     128-bit ld.global.nc.L1::no_allocate loads (512 B row at h=256 bf16 = one fully coalesced warp load); when a row
//     needs fewer than 32 lanes the warp gathers 32/lpr neighbours at once and folds them with shuffles at the end;
//   * column ids are read 32 at a time (one coalesced 128 B load) and broadcast with __shfl_sync;
//   * kUnroll neighbour rows are in flight per lane group before the fp32 accumulation (memory-level parallelism:
//     >= 64 KB in flight per SM at 32 resident warps, above the ~44 KB latency-bandwidth product of one SM's HBM share).
// Algorithmic bytes per launch: nnz*4 + (n+1)*8 + nnz*h*b + n*h*b (DESIGN.md §SpMM).
//
// Weighted graphs (edge_weight, DESIGN.md §4.10): the WEIGHTED instantiations also read the fp32 value array `val` next to `col`
// (32 at a time, broadcast by shuffle like the column ids) and FMA it into the fp32 accumulation: nnz*8 index + value bytes
// instead of nnz*4.  The dinv pre-scale by the producer and the row_scale post-scale stay as they are.  The value pointer is the
// kernels' last parameter, so the unweighted instantiations compile to the same code as before.
//
// Unscaled sums (the large variant's GCNConv(normalize=False), DESIGN.md §4.11): the SCALED=false instantiations of the row kernel
// and of the hub-row finalize kernel compute y[r,:] = sum_{j in row r} x[col[j], :] with no row_scale read and no multiply; the
// segment kernel has no scale and is shared.  SCALED is the last template parameter and defaults to true, so the existing
// instantiations compile to the same SASS as before.
#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

namespace sgf {

constexpr int kSpmmBlock = 256;
#ifndef SGF_SPMM_UNROLL
#define SGF_SPMM_UNROLL 4
#endif
#ifndef SGF_SPMM_MIN_BLOCKS
#define SGF_SPMM_MIN_BLOCKS 4
#endif
// Tuning knobs (scripts/bench_spmm.py times the variants): rows in flight per lane group x CTAs per SM, and software-pipelining
// the rowptr -> column-id -> feature-row chain across a warp's rows (SGF_SPMM_PIPELINE=1).  Once the gather saturates the memory
// system extra memory-level parallelism buys nothing, so the simple loop is the default.
#ifndef SGF_SPMM_PIPELINE
#define SGF_SPMM_PIPELINE 0
#endif
constexpr int kUnroll = SGF_SPMM_UNROLL;
constexpr int kMinBlocks = SGF_SPMM_MIN_BLOCKS;

// gather-accumulate up to 32 neighbour rows whose ids sit one per lane in my_idx (cnt valid), all lane groups cooperating
template <typename T, int CPL, bool COH = false, bool WEIGHTED = false>
__device__ __forceinline__ void gather_item(int my_idx, int cnt, const T* __restrict__ x, int64_t ldx, int groups, int grp,
                                            const int (&coff)[CPL], const bool (&cval)[CPL], float (&acc)[CPL][Vec16<T>::N],
                                            float my_w = 0.f) {
    constexpr int VN = Vec16<T>::N;
    for (int j0 = 0; j0 < cnt; j0 += groups * kUnroll) {
        uint4 v[kUnroll][CPL];
        int nb[kUnroll];
        float wt[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            int j = j0 + u * groups + grp;
            int t = __shfl_sync(0xffffffffu, my_idx, j & 31);
            nb[u] = j < cnt ? t : -1;
            if constexpr (WEIGHTED) wt[u] = __shfl_sync(0xffffffffu, my_w, j & 31);
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const T* src = x + (int64_t)(nb[u] < 0 ? 0 : nb[u]) * ldx;
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                if (nb[u] >= 0 && cval[c]) v[u][c] = COH ? ldg_na(src + coff[c]) : ldg_nc_na(src + coff[c]);
                else v[u][c] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                float f[VN];
                Vec16<T>::unpack(v[u][c], f);
                if constexpr (WEIGHTED) {
#pragma unroll
                    for (int i = 0; i < VN; ++i) acc[c][i] = fmaf(wt[u], f[i], acc[c][i]);
                } else {
#pragma unroll
                    for (int i = 0; i < VN; ++i) acc[c][i] += f[i];
                }
            }
    }
}

// gather-accumulate the neighbour rows col[s..e) of x into acc (fp32)
// (WEIGHTED: entry j contributes val[j] * x[col[j], :])
template <typename T, int CPL, bool WEIGHTED = false>
__device__ __forceinline__ void gather_range(const int32_t* __restrict__ col, const T* __restrict__ x, int64_t ldx, int64_t s, int64_t e,
                                             int lane, int groups, int grp, const int (&coff)[CPL], const bool (&cval)[CPL],
                                             float (&acc)[CPL][Vec16<T>::N], const float* __restrict__ val = nullptr) {
    for (int64_t base = s; base < e; base += 32) {
        const int cnt = (int)((e - base) < 32 ? (e - base) : 32);
        const int my_idx = lane < cnt ? ldg_nc_na_s32(col + base + lane) : -1;
        if constexpr (WEIGHTED) {
            const float my_w = lane < cnt ? __ldg(val + base + lane) : 0.f;
            gather_item<T, CPL, false, true>(my_idx, cnt, x, ldx, groups, grp, coff, cval, acc, my_w);
        } else {
            gather_item<T, CPL>(my_idx, cnt, x, ldx, groups, grp, coff, cval, acc);
        }
    }
}

// ---- row-sharded runs: operand blocks pushed by the peers while the kernel runs ------------------------------------------------
// x is the gathered operand [n_slots * slot_rows, h]: slot 0 = this rank's own rows (present), slot s > 0 = the rows of rank
// (rank + s) mod world, written by that rank's copy engine over NVLink; flags[s] != 0 once slot s has landed (set by the sender
// after its copy, sgf_signal).  Column ids are rotated (sgf_csr_build_rot), rows sorted by them, so a row's neighbours are met in
// slot order: a warp waits for a slot the first time one of its 32 current column ids falls into it.  One warp per CTA polls the
// global flags (acquire.sys); the others watch the CTA's shared `ready` counter.  Bounded spin: a protocol error traps.
struct SlotWait {
    const uint32_t* flags;
    int64_t slot_rows;
    int n_slots;
};
__device__ __forceinline__ int wait_slots(int need, volatile int* s_ready, int* s_lock, const uint32_t* flags) {
    uint32_t spins = 0;
    while (true) {
        const int r = *s_ready;
        if (r >= need) { __threadfence_block(); return r; }
        if (atomicCAS(s_lock, 0, 1) == 0) {             // this warp polls for the CTA
            int got = *s_ready;
            while (got < need && ld_acquire_sys_u32(flags + got + 1) != 0u) ++got;
            if (got > r) atomicMax(const_cast<int*>(s_ready), got);
            __threadfence_block();
            atomicExch(s_lock, 0);
            if (got >= need) return got;
            __nanosleep(400);
        } else {
            __nanosleep(200);
        }
        if (++spins > (1u << 24)) __trap();             // ~ seconds: the peers never delivered
    }
}
template <typename T, int CPL>
__device__ __forceinline__ void gather_range_flagged(const int32_t* __restrict__ col, const T* __restrict__ x, int64_t ldx, int64_t s,
                                                     int64_t e, int lane, int groups, int grp, const int (&coff)[CPL],
                                                     const bool (&cval)[CPL], float (&acc)[CPL][Vec16<T>::N], const SlotWait& sw,
                                                     int& ready, volatile int* s_ready, int* s_lock) {
    for (int64_t base = s; base < e; base += 32) {
        const int cnt = (int)((e - base) < 32 ? (e - base) : 32);
        const int my_idx = lane < cnt ? ldg_nc_na_s32(col + base + lane) : -1;
        const int slot = my_idx >= 0 ? (int)(my_idx / sw.slot_rows) : 0;
        const int need = __reduce_max_sync(0xffffffffu, slot);
        if (need > ready) {
            int got = 0;
            if (lane == 0) got = wait_slots(need < sw.n_slots ? need : sw.n_slots - 1, s_ready, s_lock, sw.flags);
            ready = __shfl_sync(0xffffffffu, got, 0);
        }
        gather_item<T, CPL, true>(my_idx, cnt, x, ldx, groups, grp, coff, cval, acc);
    }
}

// One warp per output row, rows r = warp, warp + nwarps, ...; rows longer than max_len (> 0) are left to the segmented path
// below.  SGF_SPMM_PIPELINE=1 software-pipelines the dependent chain rowptr -> column ids -> feature rows across the warp's work
// items (an item = up to 32 neighbours of one row): while the gathers of item i are in flight, the column ids of item i+1 (same
// row or the warp's next row) and the rowptr entries of the row after next are already loading (off by default, see above).
// Row range of a phased SpMM (row-sharded runs, dist.Comm._spmm_phased): the launch handles entries [lo[r], hi[r]) of every row r
// (offsets relative to the row start; null = row start / row end), starts from the fp32 partial sums of the previous phases
// (part_in, nullable) and either hands fp32 partials on (part_out) or scales and stores the finished row.
struct RowRange {
    const int32_t* lo;
    const int32_t* hi;
    const float* part_in;
    float* part_out;
    int64_t ld_part;
};
template <typename T, int CPL>
__global__ void __launch_bounds__(kSpmmBlock, kMinBlocks)
spmm_range_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ row_scale,
                  const T* __restrict__ x, int64_t ldx, T* __restrict__ y, int64_t ldy, int64_t n_rows, int chunks, int lpr_log2,
                  RowRange rr) {
    constexpr int VN = Vec16<T>::N;
    const int lane = threadIdx.x & 31;
    const int lpr = 1 << lpr_log2;
    const int groups = 32 >> lpr_log2;
    const int grp = lane >> lpr_log2;
    const int sub = lane & (lpr - 1);
    const int64_t warp0 = ((int64_t)blockIdx.x * kSpmmBlock + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * kSpmmBlock) >> 5;
    int coff[CPL];
    bool cval[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
        int ch = sub + c * lpr;
        cval[c] = ch < chunks;
        coff[c] = ch * VN;
    }
    for (int64_t r = warp0; r < n_rows; r += nwarps) {
        const int64_t s0 = rowptr[r];
        const int64_t s = rr.lo ? s0 + rr.lo[r] : s0;
        const int64_t e = rr.hi ? s0 + rr.hi[r] : rowptr[r + 1];
        float acc[CPL][VN];
#pragma unroll
        for (int c = 0; c < CPL; ++c)
#pragma unroll
            for (int i = 0; i < VN; ++i) acc[c][i] = 0.f;
        gather_range<T, CPL>(col, x, ldx, s, e, lane, groups, grp, coff, cval, acc);
        for (int o = lpr; o < 32; o <<= 1) {
#pragma unroll
            for (int c = 0; c < CPL; ++c)
#pragma unroll
                for (int i = 0; i < VN; ++i) acc[c][i] += __shfl_xor_sync(0xffffffffu, acc[c][i], o);
        }
        if (grp == 0) {
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                if (!cval[c]) continue;
                if (rr.part_in) {
                    const float4* pi = reinterpret_cast<const float4*>(rr.part_in + r * rr.ld_part + coff[c]);
#pragma unroll
                    for (int q = 0; q < VN / 4; ++q) {
                        const float4 v = pi[q];
                        acc[c][4 * q] += v.x; acc[c][4 * q + 1] += v.y; acc[c][4 * q + 2] += v.z; acc[c][4 * q + 3] += v.w;
                    }
                }
                if (rr.part_out) {
                    float4* po = reinterpret_cast<float4*>(rr.part_out + r * rr.ld_part + coff[c]);
#pragma unroll
                    for (int q = 0; q < VN / 4; ++q) po[q] = make_float4(acc[c][4 * q], acc[c][4 * q + 1], acc[c][4 * q + 2], acc[c][4 * q + 3]);
                } else {
                    const float rs = row_scale ? row_scale[r] : 1.0f;
                    float f[VN];
#pragma unroll
                    for (int i = 0; i < VN; ++i) f[i] = acc[c][i] * rs;
                    stg_na(y + r * ldy + coff[c], Vec16<T>::pack(f));
                }
            }
        }
    }
}

template <typename T, int CPL, bool FLAGS = false, bool WEIGHTED = false, bool SCALED = true>
__global__ void __launch_bounds__(kSpmmBlock, kMinBlocks)
spmm_rows_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ row_scale,
                 const T* __restrict__ x, int64_t ldx, T* __restrict__ y, int64_t ldy, int64_t n_rows, int chunks, int lpr_log2,
                 int64_t max_len, SlotWait sw, const float* __restrict__ val = nullptr) {
    constexpr int VN = Vec16<T>::N;
    __shared__ int s_ready, s_lock;
    int ready = 0;
    if (FLAGS) {
        if (threadIdx.x == 0) { s_ready = 0; s_lock = 0; }
        __syncthreads();
    }
    const int lane = threadIdx.x & 31;
    const int lpr = 1 << lpr_log2;
    const int groups = 32 >> lpr_log2;
    const int grp = lane >> lpr_log2;
    const int sub = lane & (lpr - 1);
    const int64_t warp0 = ((int64_t)blockIdx.x * kSpmmBlock + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * kSpmmBlock) >> 5;
    int coff[CPL];
    bool cval[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
        int ch = sub + c * lpr;
        cval[c] = ch < chunks;
        coff[c] = ch * VN;
    }
#if SGF_SPMM_PIPELINE
    static_assert(!FLAGS && !WEIGHTED, "the flagged and weighted variants use the simple loop");
    int64_t r = warp0;
    if (r >= n_rows) return;
    // current row [s, e) (a skipped hub row behaves like an empty row that is not stored), next row [sn, en)
    int64_t s = rowptr[r], e = rowptr[r + 1];
    bool skip = max_len > 0 && e - s > max_len;
    if (skip) e = s;
    int64_t rn = r + nwarps, sn = 0, en = 0;
    if (rn < n_rows) { sn = rowptr[rn]; en = rowptr[rn + 1]; }
    int64_t base = s;
    int idx = (base + lane < e) ? ldg_nc_na_s32(col + base + lane) : -1;
    float acc[CPL][VN];
#pragma unroll
    for (int c = 0; c < CPL; ++c)
#pragma unroll
        for (int i = 0; i < VN; ++i) acc[c][i] = 0.f;
    while (true) {
        const int cnt = (int)((e - base) < 32 ? (e - base) : 32);      // 0 for an empty row
        const bool last = base + 32 >= e;                               // last item of this row
        // ---- put the next item's column ids (and, at a row end, the rowptr pair of the row after next) in flight ----
        int64_t nbase, ne;
        bool nskip = false;
        int64_t rnn = rn, snn = 0, enn = 0;
        if (!last) { nbase = base + 32; ne = e; }
        else {
            nskip = max_len > 0 && en - sn > max_len;
            nbase = sn; ne = nskip ? sn : en;
            rnn = rn + nwarps;
            if (rnn < n_rows) { snn = rowptr[rnn]; enn = rowptr[rnn + 1]; }
        }
        const bool have_next = !last || rn < n_rows;
        const int nidx = (have_next && nbase + lane < ne) ? ldg_nc_na_s32(col + nbase + lane) : -1;
        // ---- this item ----
        gather_item<T, CPL>(idx, cnt, x, ldx, groups, grp, coff, cval, acc);
        if (last) {
            if (!skip) {
                for (int o = lpr; o < 32; o <<= 1) {
#pragma unroll
                    for (int c = 0; c < CPL; ++c)
#pragma unroll
                        for (int i = 0; i < VN; ++i) acc[c][i] += __shfl_xor_sync(0xffffffffu, acc[c][i], o);
                }
                const float rs = (SCALED && row_scale) ? row_scale[r] : 1.0f;
                if (grp == 0) {
                    T* dst = y + r * ldy;
#pragma unroll
                    for (int c = 0; c < CPL; ++c) {
                        if (!cval[c]) continue;
                        float f[VN];
#pragma unroll
                        for (int i = 0; i < VN; ++i) f[i] = SCALED ? acc[c][i] * rs : acc[c][i];
                        stg_na(dst + coff[c], Vec16<T>::pack(f));
                    }
                }
            }
            if (rn >= n_rows) break;
            r = rn; s = sn; e = ne; skip = nskip;
            rn = rnn; sn = snn; en = enn;
#pragma unroll
            for (int c = 0; c < CPL; ++c)
#pragma unroll
                for (int i = 0; i < VN; ++i) acc[c][i] = 0.f;
        }
        base = nbase;
        idx = nidx;
    }
#else
    for (int64_t r = warp0; r < n_rows; r += nwarps) {
        const int64_t s = rowptr[r];
        const int64_t e = rowptr[r + 1];
        if (max_len > 0 && e - s > max_len) continue;
        float acc[CPL][VN];
#pragma unroll
        for (int c = 0; c < CPL; ++c)
#pragma unroll
            for (int i = 0; i < VN; ++i) acc[c][i] = 0.f;
        if (FLAGS) gather_range_flagged<T, CPL>(col, x, ldx, s, e, lane, groups, grp, coff, cval, acc, sw, ready, &s_ready, &s_lock);
        else gather_range<T, CPL, WEIGHTED>(col, x, ldx, s, e, lane, groups, grp, coff, cval, acc, val);
        for (int o = lpr; o < 32; o <<= 1) {
#pragma unroll
            for (int c = 0; c < CPL; ++c)
#pragma unroll
                for (int i = 0; i < VN; ++i) acc[c][i] += __shfl_xor_sync(0xffffffffu, acc[c][i], o);
        }
        const float rs = (SCALED && row_scale) ? row_scale[r] : 1.0f;
        if (grp == 0) {
            T* dst = y + r * ldy;
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                if (!cval[c]) continue;
                float f[VN];
#pragma unroll
                for (int i = 0; i < VN; ++i) f[i] = SCALED ? acc[c][i] * rs : acc[c][i];
                stg_na(dst + coff[c], Vec16<T>::pack(f));
            }
        }
    }
#endif
}

// hub rows (power-law graphs): a row longer than the threshold is cut into segments, one warp per segment writes an fp32
// partial sum, and a second kernel adds a row's partials in fixed order (deterministic), scales and stores the row.
template <typename T, int CPL, bool WEIGHTED = false>
__global__ void __launch_bounds__(kSpmmBlock, kMinBlocks)
spmm_segments_kernel(const int32_t* __restrict__ col, const T* __restrict__ x, int64_t ldx, const int64_t* __restrict__ seg_start,
                     const int32_t* __restrict__ seg_len, int64_t n_seg, float* __restrict__ partial, int h, int chunks,
                     int lpr_log2, const float* __restrict__ val = nullptr) {
    constexpr int VN = Vec16<T>::N;
    const int lane = threadIdx.x & 31;
    const int lpr = 1 << lpr_log2;
    const int groups = 32 >> lpr_log2;
    const int grp = lane >> lpr_log2;
    const int sub = lane & (lpr - 1);
    const int64_t warp0 = ((int64_t)blockIdx.x * kSpmmBlock + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * kSpmmBlock) >> 5;
    int coff[CPL];
    bool cval[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
        int ch = sub + c * lpr;
        cval[c] = ch < chunks;
        coff[c] = ch * VN;
    }
    for (int64_t sg = warp0; sg < n_seg; sg += nwarps) {
        const int64_t s = seg_start[sg];
        float acc[CPL][VN];
#pragma unroll
        for (int c = 0; c < CPL; ++c)
#pragma unroll
            for (int i = 0; i < VN; ++i) acc[c][i] = 0.f;
        gather_range<T, CPL, WEIGHTED>(col, x, ldx, s, s + seg_len[sg], lane, groups, grp, coff, cval, acc, val);
        for (int o = lpr; o < 32; o <<= 1) {
#pragma unroll
            for (int c = 0; c < CPL; ++c)
#pragma unroll
                for (int i = 0; i < VN; ++i) acc[c][i] += __shfl_xor_sync(0xffffffffu, acc[c][i], o);
        }
        if (grp == 0) {
            float* dst = partial + sg * h;
#pragma unroll
            for (int c = 0; c < CPL; ++c)
                if (cval[c])
#pragma unroll
                    for (int i = 0; i < VN; ++i) dst[coff[c] + i] = acc[c][i];
        }
    }
}

template <typename T, bool SCALED = true>
__global__ void spmm_heavy_finalize_kernel(const float* __restrict__ partial, const int64_t* __restrict__ heavy_rows,
                                           const int64_t* __restrict__ heavy_seg_ptr, int64_t n_heavy,
                                           const float* __restrict__ row_scale, T* __restrict__ y, int64_t ldy, int h) {
    const int64_t total = n_heavy * h;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = t / h;
        const int c = (int)(t - i * h);
        float s = 0.f;
        for (int64_t sg = heavy_seg_ptr[i]; sg < heavy_seg_ptr[i + 1]; ++sg) s += partial[sg * h + c];
        const int64_t r = heavy_rows[i];
        y[r * ldy + c] = from_f32<T>(SCALED ? s * (row_scale ? row_scale[r] : 1.f) : s);
    }
}

template <typename T, bool SCALED = true>
static int launch_spmm(const int64_t* rowptr, const int32_t* col, const float* row_scale, const void* x, int64_t ldx,
                       void* y, int64_t ldy, int64_t n_rows, int h, int64_t max_len, cudaStream_t st, const SlotWait* slots = nullptr,
                       const float* val = nullptr) {
    constexpr int VN = Vec16<T>::N;
    if (h % VN != 0 || ldx % VN != 0 || ldy % VN != 0) return SGF_ERR_ARG;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15)) return SGF_ERR_ARG;
    const int chunks = h / VN;
    int lpr_log2 = 0;
    while ((1 << lpr_log2) < chunks && lpr_log2 < 5) ++lpr_log2;
    const int lpr = 1 << lpr_log2;
    const int cpl = (chunks + lpr - 1) / lpr;
    if (n_rows == 0) return SGF_OK;
    int64_t warps_needed = n_rows;
    int64_t blocks = (warps_needed * 32 + kSpmmBlock - 1) / kSpmmBlock;
    int64_t cap = (int64_t)num_sms() * kMinBlocks * 8;  // 8 waves of the resident CTAs per SM, grid-stride beyond
    if (blocks > cap) blocks = cap;
    // flagged variant: ONE wave of resident CTAs (grid-stride over the rows).  Its CTAs may spin on operand blocks that have not
    // arrived; with no CTA queued behind them the SMs keep room for the 1-thread signal kernels of this GPU's own pushes
    // (another stream), so two GPUs can never wait on each other's signals.
    if (slots && blocks > (int64_t)num_sms() * kMinBlocks) blocks = (int64_t)num_sms() * kMinBlocks;
    const T* xp = static_cast<const T*>(x);
    T* yp = static_cast<T*>(y);
    const SlotWait sw = slots ? *slots : SlotWait{nullptr, 1, 1};
#define SGF_SPMM_CASE(N)                                                                                              \
    case N:                                                                                                           \
        if (slots)                                                                                                    \
            spmm_rows_kernel<T, N, true><<<(unsigned)blocks, kSpmmBlock, 0, st>>>(rowptr, col, row_scale, xp, ldx, yp, ldy, \
                                                                                  n_rows, chunks, lpr_log2, max_len, sw);   \
        else if (val)                                                                                                 \
            spmm_rows_kernel<T, N, false, true><<<(unsigned)blocks, kSpmmBlock, 0, st>>>(rowptr, col, row_scale, xp, ldx, yp, \
                                                                                   ldy, n_rows, chunks, lpr_log2, max_len, sw, val); \
        else                                                                                                          \
            spmm_rows_kernel<T, N, false, false, SCALED><<<(unsigned)blocks, kSpmmBlock, 0, st>>>(                   \
                rowptr, col, row_scale, xp, ldx, yp, ldy, n_rows, chunks, lpr_log2, max_len, sw);                        \
        break;
    switch (cpl) {
        SGF_SPMM_CASE(1)
        SGF_SPMM_CASE(2)
        SGF_SPMM_CASE(3)
        SGF_SPMM_CASE(4)
        default: return SGF_ERR_UNSUPPORTED;  // rows wider than 2 KB
    }
#undef SGF_SPMM_CASE
    SGF_LAUNCH_CHECK();
    count_launch();
    return SGF_OK;
}

template <typename T>
static int launch_range(const int64_t* rowptr, const int32_t* col, const float* row_scale, const void* x, int64_t ldx, void* y,
                        int64_t ldy, int64_t n_rows, int h, const RowRange& rr, cudaStream_t st) {
    constexpr int VN = Vec16<T>::N;
    if (h % VN != 0 || ldx % VN != 0 || (y && ldy % VN != 0) || rr.ld_part % 4 != 0) return SGF_ERR_ARG;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15) || (reinterpret_cast<uintptr_t>(rr.part_in) & 15) ||
        (reinterpret_cast<uintptr_t>(rr.part_out) & 15))
        return SGF_ERR_ARG;
    const int chunks = h / VN;
    int lpr_log2 = 0;
    while ((1 << lpr_log2) < chunks && lpr_log2 < 5) ++lpr_log2;
    const int lpr = 1 << lpr_log2;
    const int cpl = (chunks + lpr - 1) / lpr;
    if (n_rows == 0) return SGF_OK;
    int64_t blocks = (n_rows * 32 + kSpmmBlock - 1) / kSpmmBlock;
    int64_t cap = (int64_t)num_sms() * kMinBlocks * 8;
    if (blocks > cap) blocks = cap;
    const T* xp = static_cast<const T*>(x);
    T* yp = static_cast<T*>(y);
#define SGF_RANGE_CASE(N)                                                                                             \
    case N:                                                                                                           \
        spmm_range_kernel<T, N><<<(unsigned)blocks, kSpmmBlock, 0, st>>>(rowptr, col, row_scale, xp, ldx, yp, ldy,     \
                                                                         n_rows, chunks, lpr_log2, rr);                \
        break;
    switch (cpl) {
        SGF_RANGE_CASE(1)
        SGF_RANGE_CASE(2)
        SGF_RANGE_CASE(3)
        SGF_RANGE_CASE(4)
        default: return SGF_ERR_UNSUPPORTED;
    }
#undef SGF_RANGE_CASE
    SGF_LAUNCH_CHECK();
    count_launch();
    return SGF_OK;
}

template <typename T, bool SCALED = true>
static int launch_heavy(const int32_t* col, const float* row_scale, const void* x, int64_t ldx, void* y, int64_t ldy, int h,
                        const int64_t* seg_start, const int32_t* seg_len, int64_t n_seg, float* partial,
                        const int64_t* heavy_rows, const int64_t* heavy_seg_ptr, int64_t n_heavy, cudaStream_t st,
                        const float* val = nullptr) {
    constexpr int VN = Vec16<T>::N;
    if (h % VN != 0 || ldx % VN != 0) return SGF_ERR_ARG;
    const int chunks = h / VN;
    int lpr_log2 = 0;
    while ((1 << lpr_log2) < chunks && lpr_log2 < 5) ++lpr_log2;
    const int lpr = 1 << lpr_log2;
    const int cpl = (chunks + lpr - 1) / lpr;
    int64_t blocks = (n_seg * 32 + kSpmmBlock - 1) / kSpmmBlock;
    int64_t cap = (int64_t)num_sms() * kMinBlocks * 8;
    if (blocks > cap) blocks = cap;
    const T* xp = static_cast<const T*>(x);
#define SGF_SEG_CASE(N)                                                                                                 \
    case N:                                                                                                             \
        if (val)                                                                                                        \
            spmm_segments_kernel<T, N, true><<<(unsigned)blocks, kSpmmBlock, 0, st>>>(col, xp, ldx, seg_start, seg_len, n_seg, \
                                                                                      partial, h, chunks, lpr_log2, val); \
        else                                                                                                            \
            spmm_segments_kernel<T, N><<<(unsigned)blocks, kSpmmBlock, 0, st>>>(col, xp, ldx, seg_start, seg_len, n_seg, \
                                                                                partial, h, chunks, lpr_log2);          \
        break;
    switch (cpl) {
        SGF_SEG_CASE(1)
        SGF_SEG_CASE(2)
        SGF_SEG_CASE(3)
        SGF_SEG_CASE(4)
        default: return SGF_ERR_UNSUPPORTED;
    }
#undef SGF_SEG_CASE
    SGF_LAUNCH_CHECK();
    count_launch();
    int64_t fb = (n_heavy * h + 255) / 256;
    if (fb > cap) fb = cap;
    spmm_heavy_finalize_kernel<T, SCALED><<<(unsigned)fb, 256, 0, st>>>(partial, heavy_rows, heavy_seg_ptr, n_heavy, row_scale,
                                                                static_cast<T*>(y), ldy, h);
    SGF_LAUNCH_CHECK();
    count_launch();
    return SGF_OK;
}

__global__ void signal_kernel(uint32_t* flag, uint32_t value) { st_release_sys_u32(flag, value); }
__global__ void wait_flags_kernel(const uint32_t* flags, int n) {
    uint32_t spins = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        while (ld_acquire_sys_u32(flags + i) == 0u) {
            __nanosleep(500);
            if (++spins > (1u << 24)) __trap();
        }
}

}  // namespace sgf

extern "C" int sgf_spmm_flagged(const int64_t* rowptr, const int32_t* col, const float* row_scale, const void* x, int64_t ldx,
                                void* y, int64_t ldy, int64_t n_rows, int h, int dtype, int64_t max_row_len, const uint32_t* flags,
                                int64_t slot_rows, int n_slots, void* stream) {
    if (!rowptr || n_rows < 0 || h <= 0 || (n_rows > 0 && (!x || !y)) || max_row_len < 0 || !flags || slot_rows <= 0 || n_slots < 1)
        return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const sgf::SlotWait sw{flags, slot_rows, n_slots};
    if (dtype == 0) return sgf::launch_spmm<float>(rowptr, col, row_scale, x, ldx, y, ldy, n_rows, h, max_row_len, st, &sw);
    if (dtype == 1) return sgf::launch_spmm<__nv_bfloat16>(rowptr, col, row_scale, x, ldx, y, ldy, n_rows, h, max_row_len, st, &sw);
    return SGF_ERR_ARG;
}

extern "C" int sgf_spmm_range(const int64_t* rowptr, const int32_t* col, const float* row_scale, const void* x, int64_t ldx, void* y,
                              int64_t ldy, int64_t n_rows, int h, int dtype, const int32_t* lo, const int32_t* hi,
                              const float* part_in, float* part_out, int64_t ld_part, void* stream) {
    if (!rowptr || n_rows < 0 || h <= 0 || (n_rows > 0 && !x) || (!part_out && n_rows > 0 && !y)) return SGF_ERR_ARG;
    if ((part_in || part_out) && ld_part < h) return SGF_ERR_ARG;
    const sgf::RowRange rr{lo, hi, part_in, part_out, ld_part};
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0) return sgf::launch_range<float>(rowptr, col, row_scale, x, ldx, y, ldy, n_rows, h, rr, st);
    if (dtype == 1) return sgf::launch_range<__nv_bfloat16>(rowptr, col, row_scale, x, ldx, y, ldy, n_rows, h, rr, st);
    return SGF_ERR_ARG;
}

extern "C" int sgf_signal(uint32_t* flag, uint32_t value, void* stream) {
    if (!flag) return SGF_ERR_ARG;
    sgf::signal_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(flag, value);
    SGF_LAUNCH_CHECK(); sgf::count_launch();
    return SGF_OK;
}

extern "C" int sgf_memcpy_async(void* dst, const void* src, size_t bytes, void* stream) {
    if (!dst || !src) return SGF_ERR_ARG;
    if (bytes == 0) return SGF_OK;
    SGF_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
    return SGF_OK;
}

extern "C" int sgf_wait_flags(const uint32_t* flags, int n, void* stream) {
    if (!flags || n < 0) return SGF_ERR_ARG;
    if (n == 0) return SGF_OK;
    sgf::wait_flags_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(flags, n);
    SGF_LAUNCH_CHECK(); sgf::count_launch();
    return SGF_OK;
}

extern "C" int sgf_spmm(const int64_t* rowptr, const int32_t* col, const float* row_scale, const void* x, int64_t ldx,
                        void* y, int64_t ldy, int64_t n_rows, int h, int dtype, int64_t max_row_len, void* stream) {
    if (!rowptr || n_rows < 0 || h <= 0 || (n_rows > 0 && (!x || !y)) || max_row_len < 0) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0) return sgf::launch_spmm<float>(rowptr, col, row_scale, x, ldx, y, ldy, n_rows, h, max_row_len, st);
    if (dtype == 1) return sgf::launch_spmm<__nv_bfloat16>(rowptr, col, row_scale, x, ldx, y, ldy, n_rows, h, max_row_len, st);
    return SGF_ERR_ARG;
}

extern "C" int sgf_spmm_heavy(const int32_t* col, const float* row_scale, const void* x, int64_t ldx, void* y, int64_t ldy, int h,
                              int dtype, const int64_t* seg_start, const int32_t* seg_len, int64_t n_seg, float* partial,
                              const int64_t* heavy_rows, const int64_t* heavy_seg_ptr, int64_t n_heavy, void* stream) {
    if (!col || !x || !y || h <= 0 || n_seg < 0 || n_heavy < 0) return SGF_ERR_ARG;
    if (n_seg == 0 || n_heavy == 0) return SGF_OK;
    if (!seg_start || !seg_len || !partial || !heavy_rows || !heavy_seg_ptr) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0)
        return sgf::launch_heavy<float>(col, row_scale, x, ldx, y, ldy, h, seg_start, seg_len, n_seg, partial, heavy_rows,
                                        heavy_seg_ptr, n_heavy, st);
    if (dtype == 1)
        return sgf::launch_heavy<__nv_bfloat16>(col, row_scale, x, ldx, y, ldy, h, seg_start, seg_len, n_seg, partial, heavy_rows,
                                                heavy_seg_ptr, n_heavy, st);
    return SGF_ERR_ARG;
}

extern "C" int sgf_spmm_weighted(const int64_t* rowptr, const int32_t* col, const float* val, const float* row_scale, const void* x,
                                 int64_t ldx, void* y, int64_t ldy, int64_t n_rows, int h, int dtype, int64_t max_row_len,
                                 void* stream) {
    if (!rowptr || n_rows < 0 || h <= 0 || (n_rows > 0 && (!x || !y || !val)) || max_row_len < 0) return SGF_ERR_ARG;
    if (n_rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0) return sgf::launch_spmm<float>(rowptr, col, row_scale, x, ldx, y, ldy, n_rows, h, max_row_len, st, nullptr, val);
    if (dtype == 1)
        return sgf::launch_spmm<__nv_bfloat16>(rowptr, col, row_scale, x, ldx, y, ldy, n_rows, h, max_row_len, st, nullptr, val);
    return SGF_ERR_ARG;
}

extern "C" int sgf_spmm_heavy_weighted(const int32_t* col, const float* val, const float* row_scale, const void* x, int64_t ldx,
                                       void* y, int64_t ldy, int h, int dtype, const int64_t* seg_start, const int32_t* seg_len,
                                       int64_t n_seg, float* partial, const int64_t* heavy_rows, const int64_t* heavy_seg_ptr,
                                       int64_t n_heavy, void* stream) {
    if (!col || !val || !x || !y || h <= 0 || n_seg < 0 || n_heavy < 0) return SGF_ERR_ARG;
    if (n_seg == 0 || n_heavy == 0) return SGF_OK;
    if (!seg_start || !seg_len || !partial || !heavy_rows || !heavy_seg_ptr) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0)
        return sgf::launch_heavy<float>(col, row_scale, x, ldx, y, ldy, h, seg_start, seg_len, n_seg, partial, heavy_rows,
                                        heavy_seg_ptr, n_heavy, st, val);
    if (dtype == 1)
        return sgf::launch_heavy<__nv_bfloat16>(col, row_scale, x, ldx, y, ldy, h, seg_start, seg_len, n_seg, partial, heavy_rows,
                                                heavy_seg_ptr, n_heavy, st, val);
    return SGF_ERR_ARG;
}

extern "C" int sgf_spmm_sum(const int64_t* rowptr, const int32_t* col, const void* x, int64_t ldx, void* y, int64_t ldy,
                            int64_t n_rows, int h, int dtype, int64_t max_row_len, void* stream) {
    if (!rowptr || n_rows < 0 || h <= 0 || (n_rows > 0 && (!col || !x || !y)) || max_row_len < 0) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0) return sgf::launch_spmm<float, false>(rowptr, col, nullptr, x, ldx, y, ldy, n_rows, h, max_row_len, st);
    if (dtype == 1) return sgf::launch_spmm<__nv_bfloat16, false>(rowptr, col, nullptr, x, ldx, y, ldy, n_rows, h, max_row_len, st);
    return SGF_ERR_ARG;
}

extern "C" int sgf_spmm_heavy_sum(const int32_t* col, const void* x, int64_t ldx, void* y, int64_t ldy, int h, int dtype,
                                  const int64_t* seg_start, const int32_t* seg_len, int64_t n_seg, float* partial,
                                  const int64_t* heavy_rows, const int64_t* heavy_seg_ptr, int64_t n_heavy, void* stream) {
    if (!col || !x || !y || h <= 0 || n_seg < 0 || n_heavy < 0) return SGF_ERR_ARG;
    if (n_seg == 0 || n_heavy == 0) return SGF_OK;
    if (!seg_start || !seg_len || !partial || !heavy_rows || !heavy_seg_ptr) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0)
        return sgf::launch_heavy<float, false>(col, nullptr, x, ldx, y, ldy, h, seg_start, seg_len, n_seg, partial, heavy_rows,
                                               heavy_seg_ptr, n_heavy, st);
    if (dtype == 1)
        return sgf::launch_heavy<__nv_bfloat16, false>(col, nullptr, x, ldx, y, ldy, h, seg_start, seg_len, n_seg, partial,
                                                       heavy_rows, heavy_seg_ptr, n_heavy, st);
    return SGF_ERR_ARG;
}
