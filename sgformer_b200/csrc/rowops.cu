// Row-streaming kernels: LayerNorm / BatchNorm / ReLU / dropout / residual mixes / column statistics / casts.
//
// Replace the ATen passes of the reference's TransConv.forward / GraphConv.forward (large/ours.py:74-94,194-219),
// torch.norm (medium/ours.py:16-17) and their autograd backward.  All are HBM-bound: 128-bit loads/stores, every
// activation read once per kernel, fp32 math, row reductions by warp shuffles, column reductions by per-lane register
// accumulators -> shared-memory atomics -> one global atomic per column per block.
//
// Geometry shared by all kernels: a feature row of h elements is split into 16-byte chunks; `lpr` (a power of two
// <= 32) lanes cover one row, each lane owning chunks {sub, sub+lpr, ...} (CPL of them); a warp processes 32/lpr rows
// at a time.  Because the lane -> column mapping is fixed, column sums accumulate in registers across the row loop.
#include <cstdlib>

#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

namespace sgf {

constexpr int kRowBlock = 256;
constexpr float kLnEps = 1e-5f;

// Dropout seed as the kernels receive it: the host seed of the call plus an optional device-resident epoch word
// (sgf_set_dropout_epoch).  A step captured in a CUDA graph bakes the host seed into the graph; the epoch, advanced by a
// node of the same graph, is what makes every replay draw fresh masks (forward and backward of one step read the same value).
static const uint64_t* g_dropout_epoch = nullptr;
const uint64_t* dropout_epoch_word() { return g_dropout_epoch; }
struct SeedArg {
    uint64_t base;
    const uint64_t* epoch;
    SeedArg(uint64_t s) : base(s), epoch(g_dropout_epoch) {}
    __device__ __forceinline__ uint64_t get() const {
        return epoch ? base + (*epoch) * 0xD1B54A32D192ED03ULL : base;
    }
};

struct RowGeom {
    int chunks, lpr_log2, cpl;
};
template <typename T>
static inline bool make_geom(int h, RowGeom& g) {
    constexpr int VN = Vec16<T>::N;
    if (h <= 0 || h % VN != 0) return false;
    g.chunks = h / VN;
    g.lpr_log2 = 0;
    while ((1 << g.lpr_log2) < g.chunks && g.lpr_log2 < 5) ++g.lpr_log2;
    g.cpl = (g.chunks + (1 << g.lpr_log2) - 1) >> g.lpr_log2;
    return g.cpl <= 4;
}
static inline int row_grid(int64_t rows, const RowGeom& g) {
    int rpw = 32 >> g.lpr_log2;
    int64_t warps = (rows + rpw - 1) / rpw;
    int64_t blocks = (warps * 32 + kRowBlock - 1) / kRowBlock;
    int64_t cap = (int64_t)num_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (int)blocks;
}

template <typename T, int CPL>
struct Lane {
    static constexpr int VN = Vec16<T>::N;
    int lane, lpr, sub, grp, rpw;
    int coff[CPL];
    bool cval[CPL];
    int64_t row0, row_step;
    __device__ __forceinline__ Lane(int chunks, int lpr_log2) {
        lane = threadIdx.x & 31;
        lpr = 1 << lpr_log2;
        sub = lane & (lpr - 1);
        grp = lane >> lpr_log2;
        rpw = 32 >> lpr_log2;
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
            int ch = sub + c * lpr;
            cval[c] = ch < chunks;
            coff[c] = ch * VN;
        }
        int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
        int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
        row0 = warp * rpw + grp;
        row_step = nwarps * rpw;
    }
    __device__ __forceinline__ void load(const T* base, int64_t ld, int64_t r, float (&f)[CPL][Vec16<T>::N]) const {
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
            if (cval[c]) {
                uint4 u = ldg_nc_na(base + r * ld + coff[c]);
                Vec16<T>::unpack(u, f[c]);
            } else {
#pragma unroll
                for (int i = 0; i < VN; ++i) f[c][i] = 0.f;
            }
        }
    }
    // raw 16-byte loads (kept packed while in flight: software prefetch of the next row costs 4 registers per chunk)
    __device__ __forceinline__ void load_raw(const T* base, int64_t ld, int64_t r, uint4 (&u)[CPL]) const {
#pragma unroll
        for (int c = 0; c < CPL; ++c) u[c] = cval[c] ? ldg_nc_na(base + r * ld + coff[c]) : make_uint4(0u, 0u, 0u, 0u);
    }
    __device__ __forceinline__ void unpack(const uint4 (&u)[CPL], float (&f)[CPL][Vec16<T>::N]) const {
#pragma unroll
        for (int c = 0; c < CPL; ++c) Vec16<T>::unpack(u[c], f[c]);
    }
    __device__ __forceinline__ void store(T* base, int64_t ld, int64_t r, const float (&f)[CPL][Vec16<T>::N]) const {
#pragma unroll
        for (int c = 0; c < CPL; ++c)
            if (cval[c]) stg_na(base + r * ld + coff[c], Vec16<T>::pack(f[c]));
    }
    // sum over the lanes that share a row
    __device__ __forceinline__ float row_sum(float v) const {
        for (int o = 1; o < lpr; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    }
    // dropout on the lane's chunks of row r (mask = f(seed, row, chunk))
    __device__ __forceinline__ void dropout(float (&f)[CPL][Vec16<T>::N], uint64_t seed, int64_t r, int chunks, uint32_t thr16,
                                            float inv_keep) const {
#pragma unroll
        for (int c = 0; c < CPL; ++c)
            dropout_chunk<VN>(seed, (uint64_t)r * (uint64_t)chunks + (uint64_t)(coff[c] / VN), thr16, inv_keep, f[c]);
    }
    __device__ __forceinline__ void load_vec(const float* p, float (&f)[CPL][Vec16<T>::N], float fill) const {
#pragma unroll
        for (int c = 0; c < CPL; ++c)
#pragma unroll
            for (int i = 0; i < VN; ++i) f[c][i] = (cval[c] && p) ? p[coff[c] + i] : fill;
    }
};

// ------------------------------------------------------------------------------------------------
// Deterministic cross-block sums.  fp32 atomics would add the blocks' partials in whatever order they arrive, so two runs of
// the same step would differ in the last bits (and a training run would drift apart).  Instead every reducing call site of a
// kernel owns a slot of the caller's workspace (sgf_reduce_ws_bytes): block b writes its partial to row b of the slot, and the
// last block to arrive adds the rows in block order.  The launcher zeroes the slots' arrival counters on its stream.
// ------------------------------------------------------------------------------------------------
constexpr int kRedSlots = 5;
constexpr size_t kRedHeader = 256;   // bytes of the workspace that hold the counters
struct RedWs {
    float* part;      // [kRedSlots][gridDim.x][width]
    unsigned* cnt;    // [kRedSlots] arrival counters
};

// gout[0..n) += sum over the blocks of part[0..n) (shared memory of every block, complete), in block order
__device__ __forceinline__ void grid_reduce_add(const float* part, int n, int width, int slot, float* gout, const RedWs& red) {
    __shared__ unsigned s_last;
    float* base = red.part + (size_t)slot * gridDim.x * width;
    for (int i = threadIdx.x; i < n; i += blockDim.x) base[(size_t)blockIdx.x * width + i] = part[i];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&red.cnt[slot], 1u) == gridDim.x - 1;
    __syncthreads();
    if (s_last) {
        // columns in tiles of w <= blockDim.x; the G = blockDim.x / w thread groups of a tile take every G-th block row (8 loads
        // in flight per thread), then group sums are added in group order
        __shared__ float s_grp[kRowBlock];
        __threadfence();
        for (int i0 = 0; i0 < n; i0 += blockDim.x) {
            const int w = n - i0 < (int)blockDim.x ? n - i0 : (int)blockDim.x;
            const int G = blockDim.x / w, grp = threadIdx.x / w, i = i0 + threadIdx.x % w;
            if (grp < G) {
                float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                unsigned b = grp;
                for (; b + 7 * G < gridDim.x; b += 8 * G)
#pragma unroll
                    for (int j = 0; j < 8; ++j) a[j] += __ldcg(base + (size_t)(b + j * G) * width + i);
                for (; b < gridDim.x; b += G) a[0] += __ldcg(base + (size_t)b * width + i);
                s_grp[grp * w + threadIdx.x % w] = ((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7]));
            }
            __syncthreads();
            if ((int)threadIdx.x < w) {
                float t = 0.f;
                for (int q = 0; q < G; ++q) t += s_grp[q * w + threadIdx.x];
                gout[i0 + threadIdx.x] += t;
            }
            __syncthreads();
        }
    }
    __syncthreads();
}

static inline int red_max_grid() { return num_sms() * 16; }      // >= every grid of a reducing launch (row_grid, ew_grid)

// the caller's workspace as the kernels see it; zeroes the arrival counters on the stream
static int red_args(void* ws, size_t ws_bytes, int64_t width, cudaStream_t st, RedWs& red) {
    const size_t need = kRedHeader + (size_t)kRedSlots * red_max_grid() * (size_t)width * sizeof(float);
    if (!ws || ws_bytes < need || (reinterpret_cast<uintptr_t>(ws) & 15)) return SGF_ERR_ARG;
    red.cnt = static_cast<unsigned*>(ws);
    red.part = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + kRedHeader);
    SGF_CUDA_TRY(cudaMemsetAsync(ws, 0, kRedSlots * sizeof(unsigned), st));
    return SGF_OK;
}

// fold per-lane column accumulators of a block into gout (deterministic: warps in order, then blocks in order)
template <typename T, int CPL>
__device__ __forceinline__ void flush_columns(const Lane<T, CPL>& L, float (&acc)[CPL][Vec16<T>::N], float* sm /* [h] */, int h,
                                              float* gout, int slot, const RedWs& red) {
    constexpr int VN = Vec16<T>::N;
    for (int i = threadIdx.x; i < h; i += blockDim.x) sm[i] = 0.f;
    __syncthreads();
    for (int o = L.lpr; o < 32; o <<= 1) {
#pragma unroll
        for (int c = 0; c < CPL; ++c)
#pragma unroll
            for (int i = 0; i < VN; ++i) acc[c][i] += __shfl_xor_sync(0xffffffffu, acc[c][i], o);
    }
    const int nw = blockDim.x >> 5;
    for (int w = 0; w < nw; ++w) {
        if ((int)(threadIdx.x >> 5) == w && L.grp == 0) {
#pragma unroll
            for (int c = 0; c < CPL; ++c)
                if (L.cval[c])
#pragma unroll
                    for (int i = 0; i < VN; ++i) sm[L.coff[c] + i] += acc[c][i];
        }
        __syncthreads();
    }
    grid_reduce_add(sm, h, h, slot, gout, red);
}

#define SGF_ZERO(a)                                   \
    _Pragma("unroll") for (int c_ = 0; c_ < CPL; ++c_) \
        _Pragma("unroll") for (int i_ = 0; i_ < VN; ++i_) a[c_][i_] = 0.f;
#define SGF_FOR_ELEMS _Pragma("unroll") for (int c = 0; c < CPL; ++c) _Pragma("unroll") for (int i = 0; i < VN; ++i)

// ------------------------------------------------------------------------------------------------
// rows in flight per lane group / live registers of the colstats loop (packed loads + two fp32 accumulator sets)
template <typename T, int CPL> __host__ __device__ constexpr int colstats_unroll() { return CPL * Vec16<T>::N <= 8 ? 4 : 2; }
template <typename T, int CPL> __host__ __device__ constexpr int colstats_live() { return colstats_unroll<T, CPL>() * CPL * 4 + 2 * CPL * Vec16<T>::N; }

template <typename T, int CPL>
__global__ void __launch_bounds__(kRowBlock, (colstats_live<T, CPL>() > 56 ? 2 : 3)) colstats_kernel(const T* __restrict__ x, int64_t ldx, int64_t rows, int h, int chunks,
                                                              int lpr_log2, const float* __restrict__ w, float* __restrict__ sum,
                                                              float* __restrict__ sumsq, RedWs red) {
    constexpr int VN = Vec16<T>::N;
    extern __shared__ float sm[];
    Lane<T, CPL> L(chunks, lpr_log2);
    float s1[CPL][VN], s2[CPL][VN];
    SGF_ZERO(s1) SGF_ZERO(s2)
    // 2-4 rows in flight per lane group (packed) before the accumulation: a pure reduction has no other latency hiding.
    // Wide rows (> 56 live registers of loads + accumulators) run 2 CTAs/SM so that U = 2 does not spill.
    constexpr int U = colstats_unroll<T, CPL>();
#pragma unroll 1
    for (int64_t r = L.row0; r < rows; r += U * L.row_step) {
        uint4 raw[U][CPL];
        float wr[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int64_t ru = r + u * L.row_step;
            if (ru < rows) {
                L.load_raw(x, ldx, ru, raw[u]);
                wr[u] = w ? w[ru] : 1.f;
            } else {
#pragma unroll
                for (int c = 0; c < CPL; ++c) raw[u][c] = make_uint4(0u, 0u, 0u, 0u);
                wr[u] = 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            float f[CPL][VN];
            L.unpack(raw[u], f);
            SGF_FOR_ELEMS { s1[c][i] += wr[u] * f[c][i]; s2[c][i] += f[c][i] * f[c][i]; }
        }
    }
    if (sum) flush_columns<T, CPL>(L, s1, sm, h, sum, 0, red);
    if (sumsq) flush_columns<T, CPL>(L, s2, sm, h, sumsq, 1, red);
}

// ------------------------------------------------------------------------------------------------
// LayerNorm family.  u = a*x + b*r (+ c*gy when GY); t = LN?(u); t = relu?(t); y = dropout(t)
template <typename T, int CPL, bool DROP, bool GY = false>
__global__ void __launch_bounds__(kRowBlock, 3) ln_fwd_kernel(const T* __restrict__ x, const T* __restrict__ rr, int64_t ld, int64_t rows,
                                                            int h, int chunks, int lpr_log2, float a, float b,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta, int use_ln,
                                                            int use_relu, float p, SeedArg seed_arg, T* __restrict__ y,
                                                            float* __restrict__ stats, const T* __restrict__ gyy = nullptr, float cy = 0.f) {
    const uint64_t seed = DROP ? seed_arg.get() : 0;
    constexpr int VN = Vec16<T>::N;
    Lane<T, CPL> L(chunks, lpr_log2);
    float g[CPL][VN], be[CPL][VN];
    L.load_vec(use_ln ? gamma : nullptr, g, 1.f);
    L.load_vec(use_ln ? beta : nullptr, be, 0.f);
    const float inv_h = 1.f / (float)h;
    const uint32_t thr16 = dropout_thr16(p);
    const float inv_keep = dropout_inv_keep(thr16);
    // all lanes of a warp must run the same number of iterations (row_sum shuffles): iterate on the warp's first row
    uint4 nx[CPL], nr[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) { nx[c] = make_uint4(0u, 0u, 0u, 0u); nr[c] = nx[c]; }
    if (L.row0 < rows) {
        L.load_raw(x, ld, L.row0, nx);
        if (rr) L.load_raw(rr, ld, L.row0, nr);
    }
#pragma unroll 1
    for (int64_t rb = L.row0 - L.grp; rb < rows; rb += L.row_step) {
        const int64_t r = rb + L.grp;
        const bool live = r < rows;
        float u[CPL][VN];
        L.unpack(nx, u);
        if (rr) {
            float t[CPL][VN];
            L.unpack(nr, t);
            SGF_FOR_ELEMS u[c][i] = a * u[c][i] + b * t[c][i];
        } else {
            SGF_FOR_ELEMS u[c][i] = a * u[c][i];
        }
        if (GY) {                        // the graph term of a DIFFormer layer (not prefetched: it is read once)
            uint4 ny[CPL];
            if (live) L.load_raw(gyy, ld, r, ny);
            else {
#pragma unroll
                for (int c = 0; c < CPL; ++c) ny[c] = make_uint4(0u, 0u, 0u, 0u);
            }
            float t[CPL][VN];
            L.unpack(ny, t);
            SGF_FOR_ELEMS u[c][i] += cy * t[c][i];
        }
        {
            const int64_t rn = r + L.row_step;
            if (rn < rows) {
                L.load_raw(x, ld, rn, nx);
                if (rr) L.load_raw(rr, ld, rn, nr);
            } else {
#pragma unroll
                for (int c = 0; c < CPL; ++c) { nx[c] = make_uint4(0u, 0u, 0u, 0u); nr[c] = nx[c]; }
            }
        }
        float mean = 0.f, rstd = 1.f;
        if (use_ln) {
            float s = 0.f;
            SGF_FOR_ELEMS s += u[c][i];
            mean = L.row_sum(s) * inv_h;
            float v = 0.f;
            SGF_FOR_ELEMS { float d = L.cval[c] ? u[c][i] - mean : 0.f; v += d * d; }
            rstd = rsqrtf(L.row_sum(v) * inv_h + kLnEps);
            SGF_FOR_ELEMS u[c][i] = (u[c][i] - mean) * rstd * g[c][i] + be[c][i];
        }
        if (use_relu) SGF_FOR_ELEMS u[c][i] = fmaxf(u[c][i], 0.f);
        if (DROP) L.dropout(u, seed, r, chunks, thr16, inv_keep);
        if (live) {
            L.store(y, ld, r, u);
            if (stats && L.sub == 0) { stats[2 * r] = mean; stats[2 * r + 1] = rstd; }
        }
    }
}

template <typename T, int CPL, bool DROP>
__global__ void __launch_bounds__(kRowBlock, 3) ln_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ rr,
                                                            int64_t ld, int64_t rows, int h, int chunks, int lpr_log2, float a, float b,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            const float* __restrict__ stats, int use_ln, int use_relu, float p,
                                                            SeedArg seed_arg, float gscale, T* __restrict__ dx, T* __restrict__ dr,
                                                            float* __restrict__ dgamma, float* __restrict__ dbeta, RedWs red) {
    const uint64_t seed = DROP ? seed_arg.get() : 0;
    constexpr int VN = Vec16<T>::N;
    extern __shared__ float sm[];
    Lane<T, CPL> L(chunks, lpr_log2);
    float g[CPL][VN], be[CPL][VN], dg[CPL][VN], db[CPL][VN];
    L.load_vec(use_ln ? gamma : nullptr, g, 1.f);
    L.load_vec(use_ln ? beta : nullptr, be, 0.f);
    SGF_ZERO(dg) SGF_ZERO(db)
    const float inv_h = 1.f / (float)h;
    const uint32_t thr16 = dropout_thr16(p);
    const float inv_keep = dropout_inv_keep(thr16);
    uint4 nx[CPL], nr[CPL], ng[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) { nx[c] = make_uint4(0u, 0u, 0u, 0u); nr[c] = nx[c]; ng[c] = nx[c]; }
    float nmean = 0.f, nrstd = 1.f;
    if (L.row0 < rows) {
        L.load_raw(x, ld, L.row0, nx);
        if (rr) L.load_raw(rr, ld, L.row0, nr);
        L.load_raw(dy, ld, L.row0, ng);
        if (use_ln) { nmean = stats[2 * L.row0]; nrstd = stats[2 * L.row0 + 1]; }
    }
#pragma unroll 1
    for (int64_t rb = L.row0 - L.grp; rb < rows; rb += L.row_step) {
        const int64_t r = rb + L.grp;
        const bool live = r < rows;
        float u[CPL][VN], gy[CPL][VN];
        const float mean = nmean, rstd = nrstd;
        L.unpack(nx, u);
        L.unpack(ng, gy);
        if (rr) {
            float t[CPL][VN];
            L.unpack(nr, t);
            SGF_FOR_ELEMS u[c][i] = a * u[c][i] + b * t[c][i];
        } else {
            SGF_FOR_ELEMS u[c][i] = a * u[c][i];
        }
        {
            const int64_t rn = r + L.row_step;
            if (rn < rows) {
                L.load_raw(x, ld, rn, nx);
                if (rr) L.load_raw(rr, ld, rn, nr);
                L.load_raw(dy, ld, rn, ng);
                if (use_ln) { nmean = stats[2 * rn]; nrstd = stats[2 * rn + 1]; }
            } else {
#pragma unroll
                for (int c = 0; c < CPL; ++c) { nx[c] = make_uint4(0u, 0u, 0u, 0u); nr[c] = nx[c]; ng[c] = nx[c]; }
                nmean = 0.f; nrstd = 1.f;
            }
        }
        SGF_FOR_ELEMS gy[c][i] *= gscale;
        if (DROP) L.dropout(gy, seed, r, chunks, thr16, inv_keep);
        float du[CPL][VN];
        if (use_ln) {
            float s1 = 0.f, s2 = 0.f;
            SGF_FOR_ELEMS {
                float xh = L.cval[c] ? (u[c][i] - mean) * rstd : 0.f;
                float pre = xh * g[c][i] + be[c][i];
                float gg = (use_relu && pre <= 0.f) ? 0.f : gy[c][i];
                dg[c][i] += gg * xh;
                db[c][i] += gg;
                gg *= g[c][i];
                u[c][i] = xh;
                gy[c][i] = gg;
                s1 += gg;
                s2 += gg * xh;
            }
            s1 = L.row_sum(s1) * inv_h;
            s2 = L.row_sum(s2) * inv_h;
            SGF_FOR_ELEMS du[c][i] = rstd * (gy[c][i] - s1 - u[c][i] * s2);
        } else {
            SGF_FOR_ELEMS du[c][i] = (use_relu && u[c][i] <= 0.f) ? 0.f : gy[c][i];
        }
        if (live) {
            float o[CPL][VN];
            SGF_FOR_ELEMS o[c][i] = a * du[c][i];
            L.store(dx, ld, r, o);
            if (dr) {
                SGF_FOR_ELEMS o[c][i] = b * du[c][i];
                L.store(dr, ld, r, o);
            }
        }
    }
    if (use_ln && dgamma) flush_columns<T, CPL>(L, dg, sm, h, dgamma, 0, red);
    if (use_ln && dbeta) flush_columns<T, CPL>(L, db, sm, h, dbeta, 1, red);
}

// LayerNorm backward of y = dropout(relu?(LN?(a*o + b*r))) fused with the row prologue of the Gram-form attention backward
// (engine.attention_gram_backward): with ga = a*du (gradient of the attention output o) and den~ = the forward's normalised
// denominator,   gnum' = ga / den~,   gden' = -(ga . o) / den~,   dr = b*du,
// and the column sums cs = sum_r gnum'[r,:], pg = sum_r xa[r,:]*gden'[r], sg = sum_r gden'[r] that the h x h backward algebra
// needs (sgf_attn_gram_prepare_bwd) accumulate in registers like dgamma / dbeta.  xa = the attention layer's input (== r when
// the layer has a residual connection: then it is not loaded twice).
template <typename T, int CPL, bool DROP, bool RELU, int MINB, bool GY = false>
__global__ void __launch_bounds__(kRowBlock, (CPL >= 2 ? 1 : MINB)) ln_bwd_attn_kernel(const T* __restrict__ dy, const T* __restrict__ o, const T* __restrict__ rr,
                                                                    const T* __restrict__ xa, int64_t ld, int64_t rows, int h, int chunks,
                                                                    int lpr_log2, float a, float b, const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta, const float* __restrict__ stats,
                                                                    int use_ln, float p, SeedArg seed_arg, float gscale,
                                                                    const float* __restrict__ den, T* __restrict__ gnum,
                                                                    float* __restrict__ gden, T* __restrict__ dr,
                                                                    float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                                    float* __restrict__ cs, float* __restrict__ pg, float* __restrict__ sg,
                                                                    RedWs red, const T* __restrict__ gyy = nullptr,
                                                                    const float* __restrict__ dinv = nullptr, float cy = 0.f,
                                                                    T* __restrict__ ys = nullptr) {
    const uint64_t seed = DROP ? seed_arg.get() : 0;
    constexpr int VN = Vec16<T>::N;
    extern __shared__ float sm[];
    Lane<T, CPL> L(chunks, lpr_log2);
    // register budget (85 at 3 CTAs/SM): gamma + four column accumulators live across the row loop; beta only exists in the
    // RELU instantiation (the mask needs the LayerNorm output); o and the layer input stay packed until they are used
    float g[CPL][VN], dg[CPL][VN], db[CPL][VN], acs[CPL][VN], apg[CPL][VN];
    L.load_vec(use_ln ? gamma : nullptr, g, 1.f);
    SGF_ZERO(dg) SGF_ZERO(db) SGF_ZERO(acs) SGF_ZERO(apg)
    float asg = 0.f;
    const float inv_h = 1.f / (float)h;
    const uint32_t thr16 = dropout_thr16(p);
    const float inv_keep = dropout_inv_keep(thr16);
    const bool xa_is_r = (xa == rr);
    uint4 nx[CPL], nr[CPL], ng[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) { nx[c] = make_uint4(0u, 0u, 0u, 0u); nr[c] = nx[c]; ng[c] = nx[c]; }
    float nmean = 0.f, nrstd = 1.f, ninv = 0.f;
    if (L.row0 < rows) {
        L.load_raw(o, ld, L.row0, nx);
        if (rr) L.load_raw(rr, ld, L.row0, nr);
        L.load_raw(dy, ld, L.row0, ng);
        if (use_ln) { nmean = stats[2 * L.row0]; nrstd = stats[2 * L.row0 + 1]; }
        ninv = 1.f / den[L.row0];
    }
#pragma unroll 1
    for (int64_t rb = L.row0 - L.grp; rb < rows; rb += L.row_step) {
        const int64_t r = rb + L.grp;
        const bool live = r < rows;
        float u[CPL][VN], gy[CPL][VN];
        uint4 co[CPL], cr[CPL];          // packed copies of this row's o and residual (4 registers per chunk)
        const float mean = nmean, rstd = nrstd, inv_den = ninv;
#pragma unroll
        for (int c = 0; c < CPL; ++c) { co[c] = nx[c]; cr[c] = nr[c]; }
        L.unpack(nx, u);
        L.unpack(ng, gy);
        if (rr) {
            float t[CPL][VN];
            L.unpack(cr, t);
            SGF_FOR_ELEMS u[c][i] = a * u[c][i] + b * t[c][i];
        } else {
            SGF_FOR_ELEMS u[c][i] = a * u[c][i];
        }
        if (GY) {                        // u also holds c*y (the forward's graph term)
            uint4 ny[CPL];
            if (live) L.load_raw(gyy, ld, r, ny);
            else {
#pragma unroll
                for (int c = 0; c < CPL; ++c) ny[c] = make_uint4(0u, 0u, 0u, 0u);
            }
            float t[CPL][VN];
            L.unpack(ny, t);
            SGF_FOR_ELEMS u[c][i] += cy * t[c][i];
        }
        if (!xa_is_r) {
            if (live) L.load_raw(xa, ld, r, cr);
            else {
#pragma unroll
                for (int c = 0; c < CPL; ++c) cr[c] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
        {
            const int64_t rn = r + L.row_step;
            if (rn < rows) {
                L.load_raw(o, ld, rn, nx);
                if (rr) L.load_raw(rr, ld, rn, nr);
                L.load_raw(dy, ld, rn, ng);
                if (use_ln) { nmean = stats[2 * rn]; nrstd = stats[2 * rn + 1]; }
                ninv = 1.f / den[rn];
            } else {
#pragma unroll
                for (int c = 0; c < CPL; ++c) { nx[c] = make_uint4(0u, 0u, 0u, 0u); nr[c] = nx[c]; ng[c] = nx[c]; }
                nmean = 0.f; nrstd = 1.f; ninv = 0.f;
            }
        }
        SGF_FOR_ELEMS gy[c][i] *= gscale;
        if (DROP) L.dropout(gy, seed, r, chunks, thr16, inv_keep);
        // du (gradient w.r.t. u = a*o + b*r) overwrites gy
        if (use_ln) {
            float s1 = 0.f, s2 = 0.f;
            SGF_FOR_ELEMS {
                const float xh = L.cval[c] ? (u[c][i] - mean) * rstd : 0.f;
                float gg = gy[c][i];
                if (RELU) {
                    const float be = L.cval[c] ? beta[L.coff[c] + i] : 0.f;
                    if (xh * g[c][i] + be <= 0.f) gg = 0.f;
                }
                dg[c][i] += gg * xh;
                db[c][i] += gg;
                gg *= g[c][i];
                u[c][i] = xh;
                gy[c][i] = gg;
                s1 += gg;
                s2 += gg * xh;
            }
            s1 = L.row_sum(s1) * inv_h;
            s2 = L.row_sum(s2) * inv_h;
            SGF_FOR_ELEMS gy[c][i] = rstd * (gy[c][i] - s1 - u[c][i] * s2);
        } else if (RELU) {
            SGF_FOR_ELEMS if (u[c][i] <= 0.f) gy[c][i] = 0.f;
        }
        if (live && dr) {
            SGF_FOR_ELEMS u[c][i] = b * gy[c][i];
            L.store(dr, ld, r, u);
        }
        if (GY && live) {                // dinv (.) (c*du): the operand of the transposed SpMM of the graph term
            const float sr = cy * dinv[r];
            SGF_FOR_ELEMS u[c][i] = sr * gy[c][i];
            L.store(ys, ld, r, u);
        }
        // attention-backward prologue on ga = a*du
        L.unpack(co, u);                 // o again
        float dot = 0.f;
        SGF_FOR_ELEMS { const float ga = L.cval[c] ? a * gy[c][i] : 0.f; dot += ga * u[c][i]; gy[c][i] = ga * inv_den; }
        dot = L.row_sum(dot);
        const float gd = live ? -dot * inv_den : 0.f;
        L.unpack(cr, u);                 // the layer input
        SGF_FOR_ELEMS { acs[c][i] += gy[c][i]; apg[c][i] += u[c][i] * gd; }
        if (L.sub == 0) asg += gd;
        if (live) {
            L.store(gnum, ld, r, gy);
            if (L.sub == 0) gden[r] = gd;
        }
    }
    if (use_ln && dgamma) flush_columns<T, CPL>(L, dg, sm, h, dgamma, 0, red);
    if (use_ln && dbeta) flush_columns<T, CPL>(L, db, sm, h, dbeta, 1, red);
    flush_columns<T, CPL>(L, acs, sm, h, cs, 2, red);
    flush_columns<T, CPL>(L, apg, sm, h, pg, 3, red);
    asg = warp_sum(asg);
    if (threadIdx.x == 0) sm[0] = 0.f;
    __syncthreads();
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {         // warps in order
        if (L.lane == 0 && (int)(threadIdx.x >> 5) == w) sm[0] += asg;
        __syncthreads();
    }
    grid_reduce_add(sm, 1, h, 4, sg, red);
}

// ------------------------------------------------------------------------------------------------
// BatchNorm family (column statistics supplied)
__global__ void bn_finalize_kernel(const float* __restrict__ sum, const float* __restrict__ sumsq, int64_t rows, int h, float eps,
                                   float momentum, const float* __restrict__ zbias, float* __restrict__ mean,
                                   float* __restrict__ rstd, float* __restrict__ rmean, float* __restrict__ rvar) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= h) return;
    if (sum) {  // batch statistics (training); statistics are of z (without zbias), the bias only shifts the mean
        double n = (double)rows;
        double m = (double)sum[c] / n;
        double var = (double)sumsq[c] / n - m * m;
        if (var < 0.0) var = 0.0;
        if (zbias) m += (double)zbias[c];
        mean[c] = (float)m;
        rstd[c] = (float)(1.0 / sqrt(var + (double)eps));
        if (rmean) {
            double unb = rows > 1 ? var * n / (n - 1.0) : var;
            rmean[c] = (1.f - momentum) * rmean[c] + momentum * (float)m;
            rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)unb;
        }
    } else {  // running statistics (eval)
        mean[c] = rmean[c];
        rstd[c] = rsqrtf(rvar[c] + eps);
    }
}

// Jumping knowledge over a GCN stack (GCNJK, medium/models.py:157-205), fused into the BatchNorm passes the GCN schedule makes.
// kJkMax: `buf` [rows, ld] (activation dtype) holds the running element-wise maximum over the layers' activations and `idx`
// [rows, ld] (uint8) the layer it came from.  Layer 0 initialises both; layer l > 0 replaces an element only when its value is
// strictly greater, so a tie keeps the lowest layer index (torch.max's first maximal index).  Values are compared as stored
// (rounded to the activation dtype).  kJkCat: `buf` is layer l's column block of the [rows, L*h] concatenation (pitch ld).
// Backward: the JK gradient g (`buf`) is added to the gradient of layer l's activation after the dropout mask (JK reads the
// pre-dropout value): where idx == l (kJkMax), or everywhere (kJkCat, g = column block l of g_out W^T).
constexpr int kJkNone = 0, kJkMax = 1, kJkCat = 2;
struct JkArgs {
    void* buf;
    int64_t ld;
    uint8_t* idx;
    int layer;
};

template <int VN>
__device__ __forceinline__ void ld_idx(const uint8_t* p, uint8_t (&b)[VN]) {
    if constexpr (VN == 4) {
        const uint32_t u = *reinterpret_cast<const uint32_t*>(p);
#pragma unroll
        for (int i = 0; i < 4; ++i) b[i] = (uint8_t)(u >> (8 * i));
    } else {
        const uint2 u = *reinterpret_cast<const uint2*>(p);
#pragma unroll
        for (int i = 0; i < 4; ++i) { b[i] = (uint8_t)(u.x >> (8 * i)); b[4 + i] = (uint8_t)(u.y >> (8 * i)); }
    }
}
template <int VN>
__device__ __forceinline__ void st_idx(uint8_t* p, const uint8_t (&b)[VN]) {
    if constexpr (VN == 4) {
        *reinterpret_cast<uint32_t*>(p) = (uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24);
    } else {
        uint2 u;
        u.x = (uint32_t)b[0] | ((uint32_t)b[1] << 8) | ((uint32_t)b[2] << 16) | ((uint32_t)b[3] << 24);
        u.y = (uint32_t)b[4] | ((uint32_t)b[5] << 8) | ((uint32_t)b[6] << 16) | ((uint32_t)b[7] << 24);
        *reinterpret_cast<uint2*>(p) = u;
    }
}

template <typename T, int CPL, int JK>
__device__ __forceinline__ void jk_fwd_row(const Lane<T, CPL>& L, const float (&v)[CPL][Vec16<T>::N], const JkArgs& jk, int64_t r) {
    constexpr int VN = Vec16<T>::N;
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
        if (!L.cval[c]) continue;
        const int64_t o = r * jk.ld + L.coff[c];
        T* bp = static_cast<T*>(jk.buf) + o;
        const uint4 pa = Vec16<T>::pack(v[c]);
        if constexpr (JK == kJkCat) {
            stg_na(bp, pa);
        } else {
            uint8_t id[VN];
            if (jk.layer == 0) {
#pragma unroll
                for (int i = 0; i < VN; ++i) id[i] = 0;
                stg_na(bp, pa);
            } else {
                float a[VN], m[VN];
                Vec16<T>::unpack(pa, a);
                Vec16<T>::unpack(*reinterpret_cast<const uint4*>(bp), m);
                ld_idx<VN>(jk.idx + o, id);
#pragma unroll
                for (int i = 0; i < VN; ++i)
                    if (a[i] > m[i]) { m[i] = a[i]; id[i] = (uint8_t)jk.layer; }
                stg_na(bp, Vec16<T>::pack(m));
            }
            st_idx<VN>(jk.idx + o, id);
        }
    }
}

// gy += the JK gradient of row r (see above)
template <typename T, int CPL, int JK>
__device__ __forceinline__ void jk_bwd_row(const Lane<T, CPL>& L, float (&gy)[CPL][Vec16<T>::N], const JkArgs& jk, int64_t r) {
    constexpr int VN = Vec16<T>::N;
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
        if (!L.cval[c]) continue;
        const int64_t o = r * jk.ld + L.coff[c];
        float t[VN];
        Vec16<T>::unpack(ldg_nc_na(static_cast<const T*>(jk.buf) + o), t);
        if constexpr (JK == kJkMax) {
            uint8_t id[VN];
            ld_idx<VN>(jk.idx + o, id);
#pragma unroll
            for (int i = 0; i < VN; ++i) gy[c][i] += id[i] == (uint8_t)jk.layer ? t[i] : 0.f;
        } else {
#pragma unroll
            for (int i = 0; i < VN; ++i) gy[c][i] += t[i];
        }
    }
}

template <typename T, int CPL, bool DROP, int JK = kJkNone>
__global__ void __launch_bounds__(kRowBlock, 3) bn_fwd_kernel(const T* __restrict__ z, const T* __restrict__ res, const T* __restrict__ mix,
                                                            int64_t ld, int64_t rows, int h, int chunks, int lpr_log2,
                                                            const float* __restrict__ mean, const float* __restrict__ rstd,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            const float* __restrict__ zbias, int use_bn,
                                                            int use_relu, float p, SeedArg seed_arg, float gw,
                                                            const float* __restrict__ row_scale, T* __restrict__ y,
                                                            T* __restrict__ y_scaled, JkArgs jk) {
    const uint64_t seed = DROP ? seed_arg.get() : 0;
    constexpr int VN = Vec16<T>::N;
    Lane<T, CPL> L(chunks, lpr_log2);
    float sc[CPL][VN], sh[CPL][VN];
    {
        float m[CPL][VN], rs[CPL][VN], g[CPL][VN], be[CPL][VN], zb[CPL][VN];
        L.load_vec(use_bn ? mean : nullptr, m, 0.f);
        L.load_vec(use_bn ? rstd : nullptr, rs, 1.f);
        L.load_vec(use_bn ? gamma : nullptr, g, 1.f);
        L.load_vec(use_bn ? beta : nullptr, be, 0.f);
        L.load_vec(zbias, zb, 0.f);
        SGF_FOR_ELEMS { sc[c][i] = rs[c][i] * g[c][i]; sh[c][i] = be[c][i] + (zb[c][i] - m[c][i]) * sc[c][i]; }
    }
    const uint32_t thr16 = dropout_thr16(p);
    const float inv_keep = dropout_inv_keep(thr16);
    uint4 nz[CPL], nr[CPL], nm[CPL];
    if (L.row0 < rows) {
        L.load_raw(z, ld, L.row0, nz);
        if (res) L.load_raw(res, ld, L.row0, nr);
        if (mix) L.load_raw(mix, ld, L.row0, nm);
    }
#pragma unroll 1
    for (int64_t r = L.row0; r < rows; r += L.row_step) {
        float v[CPL][VN], tr[CPL][VN], tm[CPL][VN];
        L.unpack(nz, v);
        if (res) L.unpack(nr, tr);
        if (mix) L.unpack(nm, tm);
        const int64_t rn = r + L.row_step;
        if (rn < rows) {
            L.load_raw(z, ld, rn, nz);
            if (res) L.load_raw(res, ld, rn, nr);
            if (mix) L.load_raw(mix, ld, rn, nm);
        }
        SGF_FOR_ELEMS v[c][i] = v[c][i] * sc[c][i] + sh[c][i];
        if (use_relu == kActElu) SGF_FOR_ELEMS v[c][i] = v[c][i] > 0.f ? v[c][i] : expm1f(v[c][i]);
        else if (use_relu) SGF_FOR_ELEMS v[c][i] = fmaxf(v[c][i], 0.f);
        if constexpr (JK != kJkNone) jk_fwd_row<T, CPL, JK>(L, v, jk, r);      // the pre-dropout activation
        if (DROP) L.dropout(v, seed, r, chunks, thr16, inv_keep);
        if (res) SGF_FOR_ELEMS v[c][i] += tr[c][i];
        if (y_scaled) {
            const float s = row_scale[r];
            float t[CPL][VN];
            SGF_FOR_ELEMS t[c][i] = v[c][i] * s;
            L.store(y_scaled, ld, r, t);
        }
        if (mix) SGF_FOR_ELEMS v[c][i] = gw * v[c][i] + (1.f - gw) * tm[c][i];
        if (y) L.store(y, ld, r, v);
    }
}

// g_raw = gscale * (dy + rs2[r]*dy2);  dres (+)= g_raw;  g = g_raw * dropmask * relumask
// REDUCE: sums[0:h] += g, sums[h:2h] += g*xhat.   APPLY: dz = BN-backward(g) (* out_scale[r]); dz_colsum += dz (unscaled)
// RING: the rows of the next kRingDepth iterations travel through a per-thread staging ring in shared memory (cp.async) instead
// of one row of packed registers: at 123-128 registers the kernel holds 2 CTAs = 16 warps per SM, and one 512-byte row per warp and
// tensor in flight is 16-32 KB per SM - ncu (r2l): 45 % (reduce) / 57-62 % (apply) of the DRAM peak at 25 % occupancy.
constexpr int kRingDepth = 4, kRingTensors = 4;
template <typename T, int CPL, bool APPLY, bool DROP, bool RING, int JK = kJkNone>
__global__ void __launch_bounds__(kRowBlock, 2) bn_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ dy2,
                                                               const float* __restrict__ rs2, const T* __restrict__ z, int64_t ld,
                                                               int64_t rows, int h, int chunks, int lpr_log2, const float* __restrict__ mean,
                                                               const float* __restrict__ rstd, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, const float* __restrict__ zbias, int use_bn,
                                                               int use_relu, int training, float p, SeedArg seed_arg, float gscale,
                                                               int64_t stat_rows, float* __restrict__ sums, T* __restrict__ dz,
                                                               T* __restrict__ dres,
                                                               int dres_acc, float* __restrict__ dz_colsum,
                                                               const float* __restrict__ out_scale, RedWs red, JkArgs jk) {
    static_assert(JK == kJkNone || !RING, "the JK addend is read by the register pipeline");
    const uint64_t seed = DROP ? seed_arg.get() : 0;
    constexpr int VN = Vec16<T>::N;
    extern __shared__ float sm[];
    Lane<T, CPL> L(chunks, lpr_log2);
    // per-column constants, folded so that few stay live in the row loop:
    //   xhat = z*rs + xoff,  pre-activation = z*sc + sh,  dz = sc*g - c0 - c1*z   (sc = gamma*rstd, or 1 without BN)
    float sc[CPL][VN], sh[CPL][VN], q0[CPL][VN], q1[CPL][VN];   // REDUCE: q0 = rs, q1 = xoff | APPLY: q0 = c0, q1 = c1
    {
        float m[CPL][VN], rs[CPL][VN], g[CPL][VN], be[CPL][VN], zb[CPL][VN];
        L.load_vec(use_bn ? mean : nullptr, m, 0.f);
        L.load_vec(use_bn ? rstd : nullptr, rs, 1.f);
        L.load_vec(use_bn ? gamma : nullptr, g, 1.f);
        L.load_vec(use_bn ? beta : nullptr, be, 0.f);
        L.load_vec(zbias, zb, 0.f);
        float m1[CPL][VN], m2[CPL][VN];
        if (APPLY && use_bn && training) {
            const float inv_n = 1.f / (float)(stat_rows > 0 ? stat_rows : rows);
            L.load_vec(sums, m1, 0.f);
            L.load_vec(sums + h, m2, 0.f);
            SGF_FOR_ELEMS { m1[c][i] *= inv_n; m2[c][i] *= inv_n; }
        } else {
            SGF_ZERO(m1) SGF_ZERO(m2)
        }
        SGF_FOR_ELEMS {
            const float xoff = (zb[c][i] - m[c][i]) * rs[c][i];
            sc[c][i] = rs[c][i] * g[c][i];
            sh[c][i] = xoff * g[c][i] + be[c][i];
            if (APPLY) {
                q0[c][i] = sc[c][i] * (m1[c][i] + m2[c][i] * xoff);
                q1[c][i] = sc[c][i] * m2[c][i] * rs[c][i];
            } else {
                q0[c][i] = rs[c][i];
                q1[c][i] = xoff;
            }
        }
    }
    float a1[CPL][VN], a2[CPL][VN];   // REDUCE: sum g, sum g*xhat | APPLY: a1 = column sum of dz
    SGF_ZERO(a1) SGF_ZERO(a2)
    const uint32_t thr16 = dropout_thr16(p);
    const float inv_keep = dropout_inv_keep(thr16);
    // software pipeline: the next row's 16-byte chunks are in flight (packed registers, or kRingDepth rows in the shared-memory ring)
    // while the current row is processed
    const bool acc_res = APPLY && dres && dres_acc;
    uint4 nz[CPL], n1[CPL], n2[CPL], n3[CPL];
    float ns2 = 1.f;
    uint4* ring = nullptr;
    if (RING) {
        const uint32_t base = static_cast<uint32_t>(__cvta_generic_to_shared(sm));
        const uint32_t off = ((base + (uint32_t)h * 4u + 15u) & ~15u) - base;
        ring = reinterpret_cast<uint4*>(reinterpret_cast<char*>(sm) + off);
    }
    // slot of (stage, tensor, chunk) of this thread: consecutive threads -> consecutive 16-byte slots (conflict-free LDS.128)
    auto slot = [&](int stage, int t, int c) -> uint4* { return ring + ((stage * kRingTensors + t) * CPL + c) * kRowBlock + threadIdx.x; };
    auto issue = [&](int stage, int64_t row) {
        if (row < rows) {
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                if (!L.cval[c]) continue;
                const int64_t o = row * ld + L.coff[c];
                cp_async16(slot(stage, 0, c), z + o);
                if (dy) cp_async16(slot(stage, 1, c), dy + o);
                if (dy2) cp_async16(slot(stage, 2, c), dy2 + o);
                if (acc_res) cp_async16(slot(stage, 3, c), dres + o);
            }
        }
        cp_async_commit();          // one group per stage, empty past the last row: wait_group counts stay uniform
    };
    int stage = 0;
    if (RING) {
#pragma unroll
        for (int s = 0; s < kRingDepth; ++s) issue(s, L.row0 + s * L.row_step);
        if (dy2 && rs2 && L.row0 < rows) ns2 = rs2[L.row0];
    } else if (L.row0 < rows) {
        L.load_raw(z, ld, L.row0, nz);
        if (dy) L.load_raw(dy, ld, L.row0, n1);
        if (dy2) { L.load_raw(dy2, ld, L.row0, n2); ns2 = rs2 ? rs2[L.row0] : 1.f; }
        if (acc_res) L.load_raw(dres, ld, L.row0, n3);
    }
#pragma unroll 1
    for (int64_t r = L.row0; r < rows; r += L.row_step) {
        float gy[CPL][VN], zz[CPL][VN];
        uint4 c3[CPL];
        const float s2 = ns2;
        const int64_t rn = r + L.row_step;
        if (RING) {
            cp_async_wait<kRingDepth - 1>();      // the oldest group (this row) has landed
            const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                nz[c] = L.cval[c] ? *slot(stage, 0, c) : zero;
                n1[c] = (L.cval[c] && dy) ? *slot(stage, 1, c) : zero;
                n2[c] = (L.cval[c] && dy2) ? *slot(stage, 2, c) : zero;
                c3[c] = (L.cval[c] && acc_res) ? *slot(stage, 3, c) : zero;
            }
            if (dy2 && rs2 && rn < rows) ns2 = rs2[rn];
        }
        L.unpack(nz, zz);
        if (dy) L.unpack(n1, gy);
        else SGF_ZERO(gy)
        if (dy2) {
            float t[CPL][VN];
            L.unpack(n2, t);
            SGF_FOR_ELEMS gy[c][i] += s2 * t[c][i];
        }
        if (RING) {
            issue(stage, r + (int64_t)kRingDepth * L.row_step);      // refill the stage just consumed (its data is in registers)
            stage = stage + 1 == kRingDepth ? 0 : stage + 1;
        } else {
            if (acc_res) {
#pragma unroll
                for (int c = 0; c < CPL; ++c) c3[c] = n3[c];
            }
            if (rn < rows) {
                L.load_raw(z, ld, rn, nz);
                if (dy) L.load_raw(dy, ld, rn, n1);
                if (dy2) { L.load_raw(dy2, ld, rn, n2); ns2 = rs2 ? rs2[rn] : 1.f; }
                if (acc_res) L.load_raw(dres, ld, rn, n3);
            }
        }
        SGF_FOR_ELEMS gy[c][i] *= gscale;
        if (APPLY && dres) {
            if (dres_acc) {
                float t[CPL][VN];
                L.unpack(c3, t);
                SGF_FOR_ELEMS t[c][i] += gy[c][i];
                L.store(dres, ld, r, t);
            } else {
                L.store(dres, ld, r, gy);
            }
        }
        if (DROP) L.dropout(gy, seed, r, chunks, thr16, inv_keep);
        if constexpr (JK != kJkNone) jk_bwd_row<T, CPL, JK>(L, gy, jk, r);
        const float os = (APPLY && out_scale) ? out_scale[r] : 1.f;
        SGF_FOR_ELEMS {
            const float zv = zz[c][i];
            float gg = gy[c][i];
            if (use_relu == kActElu) {
                const float pre = zv * sc[c][i] + sh[c][i];
                if (pre <= 0.f) gg *= expf(pre);
            } else if (use_relu && zv * sc[c][i] + sh[c][i] <= 0.f) {
                gg = 0.f;
            }
            if (APPLY) {
                const float d = sc[c][i] * gg - q0[c][i] - q1[c][i] * zv;
                a1[c][i] += L.cval[c] ? d : 0.f;
                gy[c][i] = d * os;
            } else {
                a1[c][i] += gg;
                a2[c][i] += gg * (zv * q0[c][i] + q1[c][i]);
            }
        }
        if (APPLY && dz) L.store(dz, ld, r, gy);
    }
    if (RING) cp_async_wait<0>();
    if (!APPLY) {
        flush_columns<T, CPL>(L, a1, sm, h, sums, 0, red);
        flush_columns<T, CPL>(L, a2, sm, h, sums + h, 1, red);
    } else if (dz_colsum) {
        flush_columns<T, CPL>(L, a1, sm, h, dz_colsum, 0, red);
    }
}

// ------------------------------------------------------------------------------------------------
template <typename TI, typename TO>
__global__ void __launch_bounds__(kRowBlock) axpby_kernel(const TI* __restrict__ x, int64_t ldx, const TI* __restrict__ y, int64_t ldy,
                                                           float a, float b, const float* __restrict__ row_scale, TO* __restrict__ out,
                                                           int64_t ldo, int64_t rows, int h) {
    // 4 elements per thread-step; rows may have different pitches so index by (row, col4)
    const int h4 = (h + 3) >> 2;
    const int64_t total = rows * h4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t r = t / h4;
        const int c0 = (int)(t - r * h4) * 4;
        const float s = row_scale ? row_scale[r] : 1.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int c = c0 + i;
            if (c < h) {
                float v = a * to_f32(x[r * ldx + c]);
                if (y) v += b * to_f32(y[r * ldy + c]);
                out[r * ldo + c] = from_f32<TO>(v * s);
            }
        }
    }
}

// fp32 [rows, cols] (pitch ld_src) -> bf16 operand dst[r_out, c_out] (optionally transposed), K padded with zeros to kp,
// one plane (plane_ld == 0) or three planes side by side (value ~= p0 + p1 + p2; fp32-accurate tensor-core products).
// Optional exact fp32 column sums of the source (bias gradients).
__global__ void __launch_bounds__(kRowBlock) pack_operand_kernel(const float* __restrict__ src, int64_t ld_src, int64_t rows, int cols,
                                                                  int transpose, __nv_bfloat16* __restrict__ dst, int64_t ld_dst,
                                                                  int kp, int64_t plane_ld, float* __restrict__ colsum,
                                                                  const int64_t* __restrict__ row_index, RedWs red) {
    extern __shared__ float sm[];
    const int64_t rows_out = transpose ? cols : rows;
    const int cols_out = transpose ? (int)rows : cols;
    const int64_t total = rows_out * kp;
    const int64_t per_block = (total + gridDim.x - 1) / gridDim.x;
    const int64_t t0 = (int64_t)blockIdx.x * per_block;
    const int64_t t1 = t0 + per_block < total ? t0 + per_block : total;
    for (int64_t t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
        const int64_t r = t / kp;
        const int c = (int)(t - r * kp);
        float v = 0.f;
        if (c < cols_out) {
            v = transpose ? src[(int64_t)c * ld_src + r] : src[(row_index ? row_index[r] : r) * ld_src + c];
        }
        __nv_bfloat16 p0 = __float2bfloat16_rn(v);
        __nv_bfloat16* o = dst + r * ld_dst + c;
        o[0] = p0;
        if (plane_ld > 0) {
            float r1 = v - __bfloat162float(p0);
            __nv_bfloat16 p1 = __float2bfloat16_rn(r1);
            o[plane_ld] = p1;
            o[2 * plane_ld] = __float2bfloat16_rn(r1 - __bfloat162float(p1));
        }
    }
    if (colsum) {
        // the block's share of every source column, summed in element order, then the blocks in order (deterministic)
        for (int k = threadIdx.x; k < cols; k += blockDim.x) {
            float s = 0.f;
            if (!transpose) {                    // source column k = output column: elements t = r * kp + k
                for (int64_t r = t0 / kp; r * kp < t1; ++r) {
                    const int64_t t = r * kp + k;
                    if (t >= t0 && t < t1) s += src[(row_index ? row_index[r] : r) * ld_src + k];
                }
            } else {                             // source column k = output row: elements t = k * kp + c, c < cols_out
                const int64_t c0 = t0 - (int64_t)k * kp > 0 ? t0 - (int64_t)k * kp : 0;
                const int64_t c1e = t1 - (int64_t)k * kp;
                const int64_t c1 = c1e < cols_out ? c1e : cols_out;
                for (int64_t c = c0; c < c1; ++c) s += src[c * ld_src + k];
            }
            sm[k] = s;
        }
        __syncthreads();
        grid_reduce_add(sm, cols, cols, 0, colsum, red);
    }
}

// vector path of pack_operand for the common case (no transpose, no column sums, 8-column aligned): a thread converts 8
// consecutive columns with two 16-byte loads and one 16-byte store per plane
__global__ void __launch_bounds__(kRowBlock) pack_rows_vec_kernel(const float* __restrict__ src, int64_t ld_src, int64_t rows, int cols,
                                                                   __nv_bfloat16* __restrict__ dst, int64_t ld_dst, int kp,
                                                                   int64_t plane_ld, const int64_t* __restrict__ row_index) {
    const int cpr = kp >> 3;                                  // 8-column chunks per output row
    const int64_t total = rows * cpr;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t r = t / cpr;
        const int c = (int)(t - r * cpr) << 3;
        float v[8];
        if (c < cols) {                                       // cols % 8 == 0: a chunk is entirely inside or outside
            const float4* sp = reinterpret_cast<const float4*>(src + (row_index ? row_index[r] : r) * ld_src + c);
            const float4 a = __ldg(sp), b = __ldg(sp + 1);
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = 0.f;
        }
        __nv_bfloat16* o = dst + r * ld_dst + c;
        *reinterpret_cast<uint4*>(o) = Vec16<__nv_bfloat16>::pack(v);
        if (plane_ld > 0) {
            float r1[8], r2[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const __nv_bfloat16 p0 = __float2bfloat16_rn(v[i]);
                r1[i] = v[i] - __bfloat162float(p0);
                const __nv_bfloat16 p1 = __float2bfloat16_rn(r1[i]);
                r2[i] = r1[i] - __bfloat162float(p1);
            }
            *reinterpret_cast<uint4*>(o + plane_ld) = Vec16<__nv_bfloat16>::pack(r1);
            *reinterpret_cast<uint4*>(o + 2 * plane_ld) = Vec16<__nv_bfloat16>::pack(r2);
        }
    }
}

// multi-head attention backward: the norm-gradient scalar is shared by all heads (one ||q||_F over [N,H,M])
__global__ void attn_combine_scal_kernel(float* __restrict__ scal_bwd, int heads, int stride, const float* __restrict__ scal_fwd) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        float c = 0.f;
        for (int i = 0; i < heads; ++i) c += scal_bwd[i * stride + 3];
        const float inq = scal_fwd[0], ink = scal_fwd[1];
        for (int i = 0; i < heads; ++i) {
            scal_bwd[i * stride + 1] = -c * inq * inq;
            scal_bwd[i * stride + 2] = -c * ink * ink;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kRowBlock) head_mean_kernel(const T* __restrict__ x, int64_t ldx, int64_t rows, int heads, int d,
                                                               T* __restrict__ out, int64_t ldo) {
    const int64_t total = rows * d;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const float inv = 1.f / (float)heads;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t r = t / d;
        const int c = (int)(t - r * d);
        float s = 0.f;
        for (int hh = 0; hh < heads; ++hh) s += to_f32(x[r * ldx + (int64_t)hh * d + c]);
        out[r * ldo + c] = from_f32<T>(s * inv);
    }
}

// gnum = g/den ; gden = -(g.o)/den
template <typename T, int CPL>
__global__ void __launch_bounds__(kRowBlock) attn_bwd_prep_kernel(const T* __restrict__ g, const T* __restrict__ o, int64_t ld,
                                                                   int64_t ld_o, const float* __restrict__ den, int64_t rows, int d, int chunks,
                                                                   int lpr_log2, float gscale, T* __restrict__ gnum, int64_t ld_gnum,
                                                                   float* __restrict__ gden) {
    constexpr int VN = Vec16<T>::N;
    Lane<T, CPL> L(chunks, lpr_log2);
#pragma unroll 1
    for (int64_t rb = L.row0 - L.grp; rb < rows; rb += L.row_step) {
        const int64_t r = rb + L.grp;
        const bool live = r < rows;
        float gg[CPL][VN], oo[CPL][VN];
        float inv = 0.f;
        if (live) {
            L.load(g, ld, r, gg);
            L.load(o, ld_o, r, oo);
            inv = gscale / den[r];
        } else {
            SGF_ZERO(gg) SGF_ZERO(oo)
        }
        float s = 0.f;
        SGF_FOR_ELEMS { s += gg[c][i] * oo[c][i]; gg[c][i] *= inv; }
        s = L.row_sum(s);
        if (live) {
            L.store(gnum, ld_gnum, r, gg);
            if (L.sub == 0) gden[r] = -s * inv;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// tiny h x h glue of the linear attention (one block per row of the output operand)
__device__ __forceinline__ void store_operand(__nv_bfloat16* base, int64_t ld, int64_t plane_ld, int r, int c, float v) {
    __nv_bfloat16 p0 = __float2bfloat16_rn(v);
    base[r * ld + c] = p0;
    if (plane_ld > 0) {
        float r1 = v - __bfloat162float(p0);
        __nv_bfloat16 p1 = __float2bfloat16_rn(r1);
        base[r * ld + plane_ld + c] = p1;
        base[r * ld + 2 * plane_ld + c] = __float2bfloat16_rn(r1 - __bfloat162float(p1));
    }
}

// scal[0]=1/nq scal[1]=1/nk scal[2]=1/(nq*nk)
__global__ void attn_prepare_fwd_kernel(const float* __restrict__ s_raw, const float* __restrict__ z_raw, const float* __restrict__ nq2v,
                                        int nq2_len, const float* __restrict__ nk2v, int nk2_len, int m, int d,
                                        __nv_bfloat16* __restrict__ bmat, int64_t ld_bmat, __nv_bfloat16* __restrict__ btail,
                                        int64_t ld_btail, int64_t plane_ld, float* __restrict__ scal) {
    __shared__ float s_inv;
    if (threadIdx.x < 32) {
        float a = 0.f, b = 0.f;
        for (int i = threadIdx.x; i < nq2_len; i += 32) a += nq2v[i];
        for (int i = threadIdx.x; i < nk2_len; i += 32) b += nk2v[i];
        a = warp_sum(a);
        b = warp_sum(b);
        if (threadIdx.x == 0) {
            float inq = rsqrtf(a), ink = rsqrtf(b);
            s_inv = inq * ink;
            if (blockIdx.x == 0) { scal[0] = inq; scal[1] = ink; scal[2] = inq * ink; scal[3] = 0.f; }
        }
    }
    __syncthreads();
    const float inv = s_inv;
    const int row = blockIdx.x;  // output row: d index for bmat rows [0,d), tail rows [d, d+16)
    if (row < d) {
        for (int mm = threadIdx.x; mm < m; mm += blockDim.x) store_operand(bmat, ld_bmat, plane_ld, row, mm, s_raw[(int64_t)mm * d + row] * inv);
    } else {
        const int tr = row - d;
        for (int mm = threadIdx.x; mm < m; mm += blockDim.x) store_operand(btail, ld_btail, plane_ld, tr, mm, tr == 0 ? z_raw[mm] * inv : 0.f);
    }
}

// Backward glue (SURVEY Appendix A.1, written for raw q,k and raw partials):
//   alpha = inq*ink (raw partials S' = k^T v, z' = k^T 1, dS_raw = q^T gnum, dz_raw = q^T gden)
//   b_dq[m, d]  = S'[m,d]               (B of dq~ = gnum . S^T, scaled by alpha in the epilogue)
//   b_dv[d, m]  = dS_raw[m,d]           (B of dv  = k . dS, scaled by alpha)
//   b_dk[m, d]  = dS_raw[m,d]           (B of dk~ = v . dS^T, scaled by alpha)
//   r1_col[m]   = alpha * z'[m]         (rank-1 term gden (x) z of dq)
//   dk_bias[m]  = alpha * dz_raw[m]
//   scal_bwd[0] = alpha, [1] = -c*inq^2, [2] = -c*ink^2, [3] = c     with c = alpha * (<dS_raw,S'> + <dz_raw,z'>)
__global__ void attn_prepare_bwd_kernel(const float* __restrict__ s_raw, const float* __restrict__ z_raw, const float* __restrict__ ds_raw,
                                        const float* __restrict__ dz_raw, const float* __restrict__ scal_fwd, int m, int d,
                                        __nv_bfloat16* __restrict__ b_dq, int64_t ld_b_dq, __nv_bfloat16* __restrict__ b_dv,
                                        int64_t ld_b_dv, __nv_bfloat16* __restrict__ b_dk, int64_t ld_b_dk, int64_t plane_ld_d,
                                        int64_t plane_ld_m, float* __restrict__ r1_col, float* __restrict__ dk_bias,
                                        float* __restrict__ scal_bwd) {
    const float alpha = scal_fwd[2];
    const int row = blockIdx.x;  // over m
    if (row < m) {
        for (int dd = threadIdx.x; dd < d; dd += blockDim.x) {
            float sv = s_raw[(int64_t)row * d + dd], dsv = ds_raw[(int64_t)row * d + dd];
            store_operand(b_dq, ld_b_dq, plane_ld_d, row, dd, sv);
            store_operand(b_dk, ld_b_dk, plane_ld_d, row, dd, dsv);
            store_operand(b_dv, ld_b_dv, plane_ld_m, dd, row, dsv);
        }
        if (threadIdx.x == 0) { r1_col[row] = alpha * z_raw[row]; dk_bias[row] = alpha * dz_raw[row]; }
    } else {
        // last block: the scalar c
        __shared__ float red[32];
        float acc = 0.f;
        for (int64_t i = threadIdx.x; i < (int64_t)m * d; i += blockDim.x) acc += s_raw[i] * ds_raw[i];
        for (int i = threadIdx.x; i < m; i += blockDim.x) acc += z_raw[i] * dz_raw[i];
        acc = warp_sum(acc);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x < 32) {
            float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
            v = warp_sum(v);
            if (threadIdx.x == 0) {
                float inq = scal_fwd[0], ink = scal_fwd[1];
                float c = alpha * v;  // <dS,S> + <dz,z> with dS = inq*dS_raw, S = ink*S'
                scal_bwd[0] = alpha;
                scal_bwd[1] = -c * inq * inq;
                scal_bwd[2] = -c * ink * ink;
                scal_bwd[3] = c;
            }
        }
    }
}

// fused log_softmax + NLL (mean over `denom` rows) forward AND gradient in one pass over the logits:
//   loss += -scale * log_softmax(x[r])[y[r]]   and   dlogits[r,:] = scale * (softmax(x[r]) - onehot(y[r]))   (0 for masked rows)
// Replaces F.log_softmax + nn.NLLLoss on out[train_mask] (reference large/main.py:139-141) and their backward.
__global__ void __launch_bounds__(kRowBlock) softmax_nll_kernel(const float* __restrict__ x, int64_t ldx, const int64_t* __restrict__ y,
                                                                 const uint8_t* __restrict__ mask, int64_t rows, int c, float scale,
                                                                 float* __restrict__ loss, float* __restrict__ dx, int64_t lddx,
                                                                 RedWs red) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    float acc = 0.f;
    for (int64_t r = warp; r < rows; r += nwarps) {
        const bool on = mask ? mask[r] != 0 : true;
        const float* xr = x + r * ldx;
        float m = -INFINITY;
        for (int j = lane; j < c; j += 32) m = fmaxf(m, xr[j]);
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float se = 0.f;
        for (int j = lane; j < c; j += 32) se += __expf(xr[j] - m);
        se = warp_sum(se);
        const float lse = m + __logf(se);
        const int64_t lab = y[r];
        if (on && lane == 0 && lab >= 0 && lab < c) acc += lse - xr[lab];
        if (dx) {
            float* dr = dx + r * lddx;
            const float s = on ? scale : 0.f;
            for (int j = lane; j < c; j += 32) dr[j] = s * (__expf(xr[j] - lse) - (j == lab ? 1.f : 0.f));
        }
    }
    acc = warp_sum(acc);
    __shared__ float s_acc[kRowBlock / 32];
    if (lane == 0) s_acc[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {                      // warps in order, then the blocks in order (deterministic)
        float b = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) b += s_acc[w];
        s_acc[0] = b * scale;
    }
    __syncthreads();
    grid_reduce_add(s_acc, 1, 1, 0, loss, red);
}

// K11 - evaluation on the device: accuracy (argmax == label) and summed NLL of log_softmax over the rows idx[0..m) (all rows if
// idx is NULL).  Replaces eval_acc (reference large/data_utils.py:210-220: argmax -> D2H -> numpy loop) and the valid_loss of
// evaluate() (large/eval.py:28-31) for single-column integer labels.  Ties: first maximum, as numpy/torch argmax.
__global__ void __launch_bounds__(kRowBlock) eval_acc_kernel(const float* __restrict__ x, int64_t ldx, const int64_t* __restrict__ y,
                                                              const int64_t* __restrict__ idx, int64_t m, int64_t rows, int c,
                                                              unsigned long long* __restrict__ correct, double* __restrict__ nll_sum) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    unsigned long long hit = 0;
    double acc = 0.0;
    for (int64_t i = warp; i < m; i += nwarps) {
        const int64_t r = idx ? idx[i] : i;
        if (r < 0 || r >= rows) continue;
        const float* xr = x + r * ldx;
        float best = -INFINITY;
        int arg = c;
        for (int j = lane; j < c; j += 32) {
            const float v = xr[j];
            if (v > best) { best = v; arg = j; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
        }
        const int64_t lab = y[r];
        if (lane == 0 && lab == arg) ++hit;
        if (nll_sum) {
            float se = 0.f;
            for (int j = lane; j < c; j += 32) se += expf(xr[j] - best);
            se = warp_sum(se);
            if (lane == 0 && lab >= 0 && lab < c) acc += (double)(best + logf(se) - xr[lab]);
        }
    }
    if (lane == 0) {
        if (hit) atomicAdd(correct, hit);
        if (nll_sum && acc != 0.0) atomicAdd(nll_sum, acc);
    }
}

}  // namespace sgf

using namespace sgf;

#define SGF_DISPATCH_T_CPL(dtype, cpl, KERNEL_CALL)                                                        \
    do {                                                                                                   \
        if ((dtype) == 0) {                                                                                \
            using T = float;                                                                               \
            switch (cpl) {                                                                                 \
                case 1: { constexpr int CPL = 1; KERNEL_CALL; } break;                                     \
                case 2: { constexpr int CPL = 2; KERNEL_CALL; } break;                                     \
                case 3: { constexpr int CPL = 3; KERNEL_CALL; } break;                                     \
                default: { constexpr int CPL = 4; KERNEL_CALL; } break;                                    \
            }                                                                                              \
        } else {                                                                                           \
            using T = __nv_bfloat16;                                                                       \
            switch (cpl) {                                                                                 \
                case 1: { constexpr int CPL = 1; KERNEL_CALL; } break;                                     \
                case 2: { constexpr int CPL = 2; KERNEL_CALL; } break;                                     \
                case 3: { constexpr int CPL = 3; KERNEL_CALL; } break;                                     \
                default: { constexpr int CPL = 4; KERNEL_CALL; } break;                                    \
            }                                                                                              \
        }                                                                                                  \
    } while (0)

// as above plus a compile-time DROP flag (dropout code only in the p > 0 instantiation)
#define SGF_DISPATCH_T_CPL_DROP(dtype, cpl, drop, KERNEL_CALL)                                             \
    do {                                                                                                   \
        if (drop) { constexpr bool DROP = true; SGF_DISPATCH_T_CPL(dtype, cpl, KERNEL_CALL); }             \
        else { constexpr bool DROP = false; SGF_DISPATCH_T_CPL(dtype, cpl, KERNEL_CALL); }                 \
    } while (0)

// T and DROP only (kernels instantiated for one CPL)
#define SGF_DISPATCH_T_DROP(dtype, drop, ...)                                                              \
    do {                                                                                                   \
        if ((dtype) == 0) {                                                                                \
            using T = float;                                                                               \
            if (drop) { constexpr bool DROP = true; __VA_ARGS__ } else { constexpr bool DROP = false; __VA_ARGS__ } \
        } else {                                                                                           \
            using T = __nv_bfloat16;                                                                       \
            if (drop) { constexpr bool DROP = true; __VA_ARGS__ } else { constexpr bool DROP = false; __VA_ARGS__ } \
        }                                                                                                  \
    } while (0)

// SGF_BN_BWD_RING (default on): shared-memory staging ring in the BatchNorm backward (rows of <= 32 chunks) instead of the
// register pipeline.
static inline bool bn_bwd_ring() {
    static const bool v = [] { const char* e = std::getenv("SGF_BN_BWD_RING"); return e ? std::atoi(e) != 0 : true; }();
    return v;
}
static inline size_t bn_bwd_ring_smem(int h) {
    return (size_t)h * sizeof(float) + 16 + (size_t)kRingDepth * kRingTensors * kRowBlock * 16;
}

static inline bool geom_for(int dtype, int h, RowGeom& g) {
    if (dtype == 0) return make_geom<float>(h, g);
    if (dtype == 1) return make_geom<__nv_bfloat16>(h, g);
    return false;
}
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static inline bool ld_ok(int dtype, int64_t ld) { return ld % (dtype == 0 ? 4 : 8) == 0; }

extern "C" int sgf_reduce_ws_bytes(int32_t width, size_t* bytes) {
    if (width <= 0 || !bytes) return SGF_ERR_ARG;
    *bytes = kRedHeader + (size_t)kRedSlots * red_max_grid() * (size_t)width * sizeof(float);
    return SGF_OK;
}

extern "C" int sgf_colstats(const void* x, int64_t ldx, int64_t rows, int h, int dtype, const float* w, float* sum, float* sumsq, void* ws, size_t ws_bytes,
                            void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !aligned16(x) || !ld_ok(dtype, ldx) || rows < 0) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    RedWs red;
    if (int rc = red_args(ws, ws_bytes, h, st, red)) return rc;
    SGF_DISPATCH_T_CPL(dtype, g.cpl, (colstats_kernel<T, CPL><<<row_grid(rows, g), kRowBlock, h * sizeof(float), st>>>(
                                         (const T*)x, ldx, rows, h, g.chunks, g.lpr_log2, w, sum, sumsq, red)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_ln_fwd(const void* x, const void* r, int64_t ld, int64_t rows, int h, int dtype, float a, float b,
                          const float* gamma, const float* beta, int use_ln, int use_relu, float p, uint64_t seed, void* y,
                          float* stats, void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !aligned16(x) || !aligned16(y) || !aligned16(r) || !ld_ok(dtype, ld) || rows < 0) return SGF_ERR_ARG;
    if (use_ln && (!gamma || !beta)) return SGF_ERR_ARG;
    if (p < 0.f || p >= 1.f) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (ln_fwd_kernel<T, CPL, DROP><<<row_grid(rows, g), kRowBlock, 0, st>>>(
                                         (const T*)x, (const T*)r, ld, rows, h, g.chunks, g.lpr_log2, a, b, gamma, beta, use_ln,
                                         use_relu, p, seed, (T*)y, stats)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_ln_fwd_graph(const void* x, const void* r, const void* gy, int64_t ld, int64_t rows, int h, int dtype, float a,
                                float b, float c, const float* gamma, const float* beta, int use_ln, int use_relu, float p,
                                uint64_t seed, void* y, float* stats, void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !x || !gy || !aligned16(x) || !aligned16(gy) || !aligned16(y) || !aligned16(r) || !ld_ok(dtype, ld) ||
        rows < 0)
        return SGF_ERR_ARG;
    if (use_ln && (!gamma || !beta)) return SGF_ERR_ARG;
    if (p < 0.f || p >= 1.f) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (ln_fwd_kernel<T, CPL, DROP, true><<<row_grid(rows, g), kRowBlock, 0, st>>>(
                                         (const T*)x, (const T*)r, ld, rows, h, g.chunks, g.lpr_log2, a, b, gamma, beta, use_ln,
                                         use_relu, p, seed, (T*)y, stats, (const T*)gy, c)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_ln_bwd(const void* dy, const void* x, const void* r, int64_t ld, int64_t rows, int h, int dtype, float a,
                          float b, const float* gamma, const float* beta, const float* stats, int use_ln, int use_relu, float p,
                          uint64_t seed, float gscale, void* dx, void* dr, float* dgamma, float* dbeta, void* ws, size_t ws_bytes,
                          void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !aligned16(x) || !aligned16(dy) || !aligned16(dx) || !aligned16(r) || !aligned16(dr) ||
        !ld_ok(dtype, ld) || rows < 0)
        return SGF_ERR_ARG;
    if (use_ln && (!gamma || !beta || !stats)) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    RedWs red;
    if (int rc = red_args(ws, ws_bytes, h, st, red)) return rc;
    SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (ln_bwd_kernel<T, CPL, DROP><<<row_grid(rows, g), kRowBlock, h * sizeof(float), st>>>(
                                         (const T*)dy, (const T*)x, (const T*)r, ld, rows, h, g.chunks, g.lpr_log2, a, b, gamma, beta,
                                         stats, use_ln, use_relu, p, seed, gscale, (T*)dx, (T*)dr, dgamma, dbeta, red)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_ln_bwd_attn(const void* dy, const void* o, const void* r, const void* xa, int64_t ld, int64_t rows, int h,
                               int dtype, float a, float b, const float* gamma, const float* beta, const float* stats, int use_ln,
                               int use_relu, float p, uint64_t seed, float gscale, const float* den, void* gnum, float* gden,
                               void* dr, float* dgamma, float* dbeta, float* cs, float* pg, float* sg, void* ws, size_t ws_bytes,
                               void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !aligned16(o) || !aligned16(dy) || !aligned16(gnum) || !aligned16(r) || !aligned16(dr) ||
        !aligned16(xa) || !ld_ok(dtype, ld) || rows < 0)
        return SGF_ERR_ARG;
    if (!o || !dy || !xa || !den || !gnum || !gden || !cs || !pg || !sg) return SGF_ERR_ARG;
    if (use_ln && (!gamma || !beta || !stats)) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    RedWs red;
    if (int rc = red_args(ws, ws_bytes, h, st, red)) return rc;
    // resident CTAs per SM for the one-chunk-per-lane geometry: 2 (no spills; default) or 3 (fewer registers, some spilled)
    static const int minb = [] { const char* e = getenv("SGF_LNATTN_BLOCKS"); return (e && e[0] == '3') ? 3 : 2; }();
    if (minb == 2 && !use_relu) {
        SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (ln_bwd_attn_kernel<T, CPL, DROP, false, 2><<<row_grid(rows, g), kRowBlock, h * sizeof(float), st>>>(
                                             (const T*)dy, (const T*)o, (const T*)r, (const T*)xa, ld, rows, h, g.chunks, g.lpr_log2, a, b,
                                             gamma, beta, stats, use_ln, p, seed, gscale, den, (T*)gnum, gden, (T*)dr, dgamma,
                                             dbeta, cs, pg, sg, red)));
    } else if (use_relu) {
        SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (ln_bwd_attn_kernel<T, CPL, DROP, true, 3><<<row_grid(rows, g), kRowBlock, h * sizeof(float), st>>>(
                                             (const T*)dy, (const T*)o, (const T*)r, (const T*)xa, ld, rows, h, g.chunks, g.lpr_log2, a, b,
                                             gamma, beta, stats, use_ln, p, seed, gscale, den, (T*)gnum, gden, (T*)dr, dgamma,
                                             dbeta, cs, pg, sg, red)));
    } else {
        SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (ln_bwd_attn_kernel<T, CPL, DROP, false, 3><<<row_grid(rows, g), kRowBlock, h * sizeof(float), st>>>(
                                             (const T*)dy, (const T*)o, (const T*)r, (const T*)xa, ld, rows, h, g.chunks, g.lpr_log2, a, b,
                                             gamma, beta, stats, use_ln, p, seed, gscale, den, (T*)gnum, gden, (T*)dr, dgamma,
                                             dbeta, cs, pg, sg, red)));
    }
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_ln_bwd_attn_graph(const void* dy, const void* o, const void* r, const void* xa, const void* gy, int64_t ld, int64_t rows, int h,
                                     int dtype, float a, float b, float c, const float* gamma, const float* beta, const float* stats,
                                     int use_ln, float p, uint64_t seed, float gscale, const float* den, const float* dinv,
                                     void* gnum, float* gden, void* dr, void* ys, float* dgamma, float* dbeta, float* cs, float* pg,
                                     float* sg, void* ws, size_t ws_bytes, void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !aligned16(o) || !aligned16(dy) || !aligned16(gnum) || !aligned16(r) || !aligned16(dr) ||
        !aligned16(xa) || !aligned16(gy) || !aligned16(ys) || !ld_ok(dtype, ld) || rows < 0)
        return SGF_ERR_ARG;
    if (!o || !dy || !xa || !gy || !den || !dinv || !gnum || !gden || !ys || !cs || !pg || !sg) return SGF_ERR_ARG;
    if (use_ln && (!gamma || !beta || !stats)) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    RedWs red;
    if (int rc = red_args(ws, ws_bytes, h, st, red)) return rc;
    SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (ln_bwd_attn_kernel<T, CPL, DROP, false, 2, true><<<row_grid(rows, g), kRowBlock, h * sizeof(float), st>>>(
                                         (const T*)dy, (const T*)o, (const T*)r, (const T*)xa, ld, rows, h, g.chunks, g.lpr_log2, a, b,
                                         gamma, beta, stats, use_ln, p, seed, gscale, den, (T*)gnum, gden, (T*)dr, dgamma,
                                         dbeta, cs, pg, sg, red, (const T*)gy, dinv, c, (T*)ys)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_bn_finalize(const float* sum, const float* sumsq, int64_t rows, int h, float eps, float momentum,
                               const float* zbias, float* mean, float* rstd, float* running_mean, float* running_var, void* stream) {
    if (h <= 0 || !mean || !rstd) return SGF_ERR_ARG;
    if (!sum && (!running_mean || !running_var)) return SGF_ERR_ARG;
    if (sum && (!sumsq || rows <= 0)) return SGF_ERR_ARG;
    bn_finalize_kernel<<<(h + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sum, sumsq, rows, h, eps, momentum, zbias, mean, rstd,
                                                                          running_mean, running_var);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

// the JK modes as template instances: the mode-0 instances are the plain BatchNorm kernels
#define SGF_DISPATCH_JK(mode, ...)                                                             \
    do {                                                                                       \
        if ((mode) == kJkMax) { constexpr int JK = kJkMax; __VA_ARGS__; }                      \
        else if ((mode) == kJkCat) { constexpr int JK = kJkCat; __VA_ARGS__; }                 \
        else { constexpr int JK = kJkNone; __VA_ARGS__; }                                      \
    } while (0)

static int jk_check(int jk_mode, int dtype, const JkArgs& jk) {
    if (jk_mode == kJkNone) return SGF_OK;
    if (jk_mode != kJkMax && jk_mode != kJkCat) return SGF_ERR_ARG;
    if (!jk.buf || !aligned16(jk.buf) || !ld_ok(dtype, jk.ld) || jk.layer < 0 || jk.layer > 255) return SGF_ERR_ARG;
    if (jk_mode == kJkMax && (!jk.idx || (reinterpret_cast<uintptr_t>(jk.idx) & (dtype == 0 ? 3 : 7)))) return SGF_ERR_ARG;
    return SGF_OK;
}

static int bn_fwd_launch(const void* z, const void* res, const void* mix, int64_t ld, int64_t rows, int h, int dtype,
                         const float* mean, const float* rstd, const float* gamma, const float* beta, const float* zbias,
                         int use_bn, int use_relu, float p, uint64_t seed, float gw, const float* row_scale, void* y,
                         void* y_scaled, int jk_mode, JkArgs jk, void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !aligned16(z) || !aligned16(res) || !aligned16(mix) || !aligned16(y) || !aligned16(y_scaled) ||
        !ld_ok(dtype, ld) || rows < 0)
        return SGF_ERR_ARG;
    if (use_bn && (!mean || !rstd || !gamma || !beta)) return SGF_ERR_ARG;
    if (y_scaled && !row_scale) return SGF_ERR_ARG;
    if (p < 0.f || p >= 1.f) return SGF_ERR_ARG;
    if (int rc = jk_check(jk_mode, dtype, jk)) return rc;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    SGF_DISPATCH_JK(jk_mode, SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (bn_fwd_kernel<T, CPL, DROP, JK><<<row_grid(rows, g), kRowBlock, 0, st>>>(
                                         (const T*)z, (const T*)res, (const T*)mix, ld, rows, h, g.chunks, g.lpr_log2, mean, rstd,
                                         gamma, beta, zbias, use_bn, use_relu, p, seed, gw, row_scale, (T*)y, (T*)y_scaled, jk))));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_bn_fwd(const void* z, const void* res, const void* mix, int64_t ld, int64_t rows, int h, int dtype,
                          const float* mean, const float* rstd, const float* gamma, const float* beta, const float* zbias,
                          int use_bn, int use_relu, float p, uint64_t seed, float gw, const float* row_scale, void* y,
                          void* y_scaled, void* stream) {
    return bn_fwd_launch(z, res, mix, ld, rows, h, dtype, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, gw, row_scale, y,
                         y_scaled, kJkNone, JkArgs{nullptr, 0, nullptr, 0}, stream);
}

extern "C" int sgf_bn_fwd_jk(const void* z, int64_t ld, int64_t rows, int h, int dtype, const float* mean, const float* rstd,
                             const float* gamma, const float* beta, const float* zbias, int use_bn, int use_relu, float p,
                             uint64_t seed, void* y, int jk_mode, void* jk, int64_t ld_jk, uint8_t* jk_idx, int jk_layer,
                             void* stream) {
    if (jk_mode == kJkNone) return SGF_ERR_ARG;
    return bn_fwd_launch(z, nullptr, nullptr, ld, rows, h, dtype, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed, 1.f,
                         nullptr, y, nullptr, jk_mode, JkArgs{jk, ld_jk, jk_idx, jk_layer}, stream);
}

static int bn_bwd_reduce_launch(const void* dy, const void* dy2, const float* row_scale2, const void* z, int64_t ld, int64_t rows,
                                int h, int dtype, const float* mean, const float* rstd, const float* gamma, const float* beta,
                                const float* zbias, int use_bn, int use_relu, float p, uint64_t seed, float gscale, float* sums,
                                int jk_mode, JkArgs jk, void* ws, size_t ws_bytes, void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !aligned16(dy) || !aligned16(dy2) || !aligned16(z) || !ld_ok(dtype, ld) || rows < 0 || !sums ||
        (!dy && !dy2 && jk_mode == kJkNone))
        return SGF_ERR_ARG;
    if (use_bn && (!mean || !rstd || !gamma || !beta)) return SGF_ERR_ARG;
    if (int rc = jk_check(jk_mode, dtype, jk)) return rc;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    RedWs red;
    if (int rc = red_args(ws, ws_bytes, h, st, red)) return rc;
    if (g.cpl == 1 && bn_bwd_ring() && jk_mode == kJkNone) {
        const size_t smem = bn_bwd_ring_smem(h);
        SGF_DISPATCH_T_DROP(dtype, p > 0.f, {
            SGF_CUDA_TRY(cudaFuncSetAttribute(bn_bwd_kernel<T, 1, false, DROP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            bn_bwd_kernel<T, 1, false, DROP, true><<<row_grid(rows, g), kRowBlock, smem, st>>>(
                (const T*)dy, (const T*)dy2, row_scale2, (const T*)z, ld, rows, h, g.chunks, g.lpr_log2, mean, rstd, gamma, beta, zbias,
                use_bn, use_relu, 1, p, seed, gscale, (int64_t)0, sums, (T*)nullptr, (T*)nullptr, 0, (float*)nullptr,
                (const float*)nullptr, red, jk);
        });
        SGF_LAUNCH_CHECK(); count_launch();
        return SGF_OK;
    }
    SGF_DISPATCH_JK(jk_mode, SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (bn_bwd_kernel<T, CPL, false, DROP, false, JK><<<row_grid(rows, g), kRowBlock, h * sizeof(float), st>>>(
                                         (const T*)dy, (const T*)dy2, row_scale2, (const T*)z, ld, rows, h, g.chunks, g.lpr_log2, mean,
                                         rstd, gamma, beta, zbias, use_bn, use_relu, 1, p, seed, gscale, (int64_t)0, sums,
                                         (T*)nullptr, (T*)nullptr, 0, (float*)nullptr, (const float*)nullptr, red, jk))));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_bn_bwd_reduce(const void* dy, const void* dy2, const float* row_scale2, const void* z, int64_t ld, int64_t rows,
                                 int h, int dtype, const float* mean, const float* rstd, const float* gamma, const float* beta,
                                 const float* zbias, int use_bn, int use_relu, float p, uint64_t seed, float gscale, float* sums,
                                 void* ws, size_t ws_bytes, void* stream) {
    return bn_bwd_reduce_launch(dy, dy2, row_scale2, z, ld, rows, h, dtype, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed,
                                gscale, sums, kJkNone, JkArgs{nullptr, 0, nullptr, 0}, ws, ws_bytes, stream);
}

static int bn_bwd_apply_launch(const void* dy, const void* dy2, const float* row_scale2, const void* z, int64_t ld, int64_t rows,
                               int h, int dtype, const float* mean, const float* rstd, const float* gamma, const float* beta,
                               const float* zbias, int use_bn, int use_relu, int training, float p, uint64_t seed, float gscale,
                               int64_t stat_rows, const float* sums, void* dz, void* dres, int dres_accumulate,
                               float* dz_colsum, const float* out_row_scale, int jk_mode, JkArgs jk, void* ws, size_t ws_bytes,
                               void* stream) {
    RowGeom g;
    if (!geom_for(dtype, h, g) || !aligned16(dy) || !aligned16(dy2) || !aligned16(z) || !aligned16(dz) || !aligned16(dres) ||
        !ld_ok(dtype, ld) || rows < 0 || (!dy && !dy2 && jk_mode == kJkNone))
        return SGF_ERR_ARG;
    if (use_bn && (!mean || !rstd || !gamma || !beta)) return SGF_ERR_ARG;
    if (use_bn && training && !sums) return SGF_ERR_ARG;
    if (int rc = jk_check(jk_mode, dtype, jk)) return rc;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    RedWs red;
    if (int rc = red_args(ws, ws_bytes, h, st, red)) return rc;
    if (g.cpl == 1 && bn_bwd_ring() && jk_mode == kJkNone) {
        const size_t smem = bn_bwd_ring_smem(h);
        SGF_DISPATCH_T_DROP(dtype, p > 0.f, {
            SGF_CUDA_TRY(cudaFuncSetAttribute(bn_bwd_kernel<T, 1, true, DROP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            bn_bwd_kernel<T, 1, true, DROP, true><<<row_grid(rows, g), kRowBlock, smem, st>>>(
                (const T*)dy, (const T*)dy2, row_scale2, (const T*)z, ld, rows, h, g.chunks, g.lpr_log2, mean, rstd, gamma, beta, zbias,
                use_bn, use_relu, training, p, seed, gscale, stat_rows, const_cast<float*>(sums), (T*)dz, (T*)dres, dres_accumulate,
                dz_colsum, out_row_scale, red, jk);
        });
        SGF_LAUNCH_CHECK(); count_launch();
        return SGF_OK;
    }
    SGF_DISPATCH_JK(jk_mode, SGF_DISPATCH_T_CPL_DROP(dtype, g.cpl, p > 0.f, (bn_bwd_kernel<T, CPL, true, DROP, false, JK><<<row_grid(rows, g), kRowBlock, h * sizeof(float), st>>>(
                                         (const T*)dy, (const T*)dy2, row_scale2, (const T*)z, ld, rows, h, g.chunks, g.lpr_log2, mean,
                                         rstd, gamma, beta, zbias, use_bn, use_relu, training, p, seed, gscale, stat_rows,
                                         const_cast<float*>(sums), (T*)dz, (T*)dres, dres_accumulate, dz_colsum, out_row_scale, red, jk))));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_bn_bwd_apply(const void* dy, const void* dy2, const float* row_scale2, const void* z, int64_t ld, int64_t rows,
                                int h, int dtype, const float* mean, const float* rstd, const float* gamma, const float* beta,
                                const float* zbias, int use_bn, int use_relu, int training, float p, uint64_t seed, float gscale,
                                int64_t stat_rows, const float* sums, void* dz, void* dres, int dres_accumulate,
                                float* dz_colsum, const float* out_row_scale, void* ws, size_t ws_bytes,
                                void* stream) {
    return bn_bwd_apply_launch(dy, dy2, row_scale2, z, ld, rows, h, dtype, mean, rstd, gamma, beta, zbias, use_bn, use_relu, training, p,
                               seed, gscale, stat_rows, sums, dz, dres, dres_accumulate, dz_colsum, out_row_scale, kJkNone,
                               JkArgs{nullptr, 0, nullptr, 0}, ws, ws_bytes, stream);
}

extern "C" int sgf_bn_bwd_reduce_jk(const void* dy, const void* z, int64_t ld, int64_t rows, int h, int dtype, const float* mean,
                                    const float* rstd, const float* gamma, const float* beta, const float* zbias, int use_bn,
                                    int use_relu, float p, uint64_t seed, float* sums, int jk_mode, const void* jk_g, int64_t ld_jk,
                                    const uint8_t* jk_idx, int jk_layer, void* ws, size_t ws_bytes, void* stream) {
    if (jk_mode == kJkNone) return SGF_ERR_ARG;
    return bn_bwd_reduce_launch(dy, nullptr, nullptr, z, ld, rows, h, dtype, mean, rstd, gamma, beta, zbias, use_bn, use_relu, p, seed,
                                1.f, sums, jk_mode, JkArgs{const_cast<void*>(jk_g), ld_jk, const_cast<uint8_t*>(jk_idx), jk_layer},
                                ws, ws_bytes, stream);
}

extern "C" int sgf_bn_bwd_apply_jk(const void* dy, const void* z, int64_t ld, int64_t rows, int h, int dtype, const float* mean,
                                   const float* rstd, const float* gamma, const float* beta, const float* zbias, int use_bn,
                                   int use_relu, int training, float p, uint64_t seed, const float* sums, void* dz, float* dz_colsum,
                                   const float* out_row_scale, int jk_mode, const void* jk_g, int64_t ld_jk, const uint8_t* jk_idx,
                                   int jk_layer, void* ws, size_t ws_bytes, void* stream) {
    if (jk_mode == kJkNone) return SGF_ERR_ARG;
    return bn_bwd_apply_launch(dy, nullptr, nullptr, z, ld, rows, h, dtype, mean, rstd, gamma, beta, zbias, use_bn, use_relu, training, p,
                               seed, 1.f, 0, sums, dz, nullptr, 0, dz_colsum, out_row_scale, jk_mode,
                               JkArgs{const_cast<void*>(jk_g), ld_jk, const_cast<uint8_t*>(jk_idx), jk_layer}, ws, ws_bytes, stream);
}

static inline int ew_grid(int64_t total) {
    int64_t b = (total + kRowBlock - 1) / kRowBlock;
    int64_t cap = (int64_t)num_sms() * 16;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

extern "C" int sgf_axpby(const void* x, int64_t ldx, int x_dtype, const void* y, int64_t ldy, int y_dtype, float a, float b,
                         const float* row_scale, void* out, int64_t ldo, int out_dtype, int64_t rows, int h, void* stream) {
    if (!x || !out || rows < 0 || h <= 0 || (y && y_dtype != x_dtype)) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int grid = ew_grid(rows * ((h + 3) / 4));
    if (x_dtype == 0 && out_dtype == 0)
        axpby_kernel<float, float><<<grid, kRowBlock, 0, st>>>((const float*)x, ldx, (const float*)y, ldy, a, b, row_scale, (float*)out, ldo, rows, h);
    else if (x_dtype == 0 && out_dtype == 1)
        axpby_kernel<float, __nv_bfloat16><<<grid, kRowBlock, 0, st>>>((const float*)x, ldx, (const float*)y, ldy, a, b, row_scale, (__nv_bfloat16*)out, ldo, rows, h);
    else if (x_dtype == 1 && out_dtype == 0)
        axpby_kernel<__nv_bfloat16, float><<<grid, kRowBlock, 0, st>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)y, ldy, a, b, row_scale, (float*)out, ldo, rows, h);
    else if (x_dtype == 1 && out_dtype == 1)
        axpby_kernel<__nv_bfloat16, __nv_bfloat16><<<grid, kRowBlock, 0, st>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)y, ldy, a, b, row_scale, (__nv_bfloat16*)out, ldo, rows, h);
    else
        return SGF_ERR_ARG;
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_pack_operand(const float* src, int64_t ld_src, int64_t rows, int cols, int transpose, void* dst,
                                int64_t ld_dst, int kp, int64_t plane_ld, float* colsum, const int64_t* row_index, void* ws,
                                size_t ws_bytes, void* stream) {
    if (!src || !dst || rows <= 0 || cols <= 0 || kp <= 0 || (row_index && transpose)) return SGF_ERR_ARG;
    const int64_t cols_out = transpose ? rows : cols;
    if (kp < cols_out || (plane_ld > 0 && plane_ld < kp) || ld_dst < (plane_ld > 0 ? 2 * plane_ld + kp : kp)) return SGF_ERR_ARG;
    if (colsum && cols > 8192) return SGF_ERR_UNSUPPORTED;
    const int64_t rows_out = transpose ? cols : rows;
    // 16-byte vectorised row pack (the arxiv-shaped fp32 step packs 28 activations per step into bf16x3 planes);
    // SGF_PACK_VEC=0 selects the scalar kernel
    static const bool vec_on = [] { const char* e = getenv("SGF_PACK_VEC"); return !(e && e[0] == '0'); }();
    const bool vec = vec_on && !transpose && !colsum && cols % 8 == 0 && kp % 8 == 0 && ld_src % 4 == 0 && ld_dst % 8 == 0 &&
                     plane_ld % 8 == 0 && aligned16(src) && aligned16(dst);
    RedWs red{nullptr, nullptr};
    if (colsum)
        if (int rc = red_args(ws, ws_bytes, cols, (cudaStream_t)stream, red)) return rc;
    if (vec)
        pack_rows_vec_kernel<<<ew_grid(rows_out * (kp / 8)), kRowBlock, 0, (cudaStream_t)stream>>>(
            src, ld_src, rows, cols, (__nv_bfloat16*)dst, ld_dst, kp, plane_ld, row_index);
    else
        pack_operand_kernel<<<ew_grid(rows_out * kp), kRowBlock, colsum ? cols * sizeof(float) : 0, (cudaStream_t)stream>>>(
            src, ld_src, rows, cols, transpose, (__nv_bfloat16*)dst, ld_dst, kp, plane_ld, colsum, row_index, red);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_attn_combine_scal(float* scal_bwd, int heads, int stride, const float* scal_fwd, void* stream) {
    if (!scal_bwd || !scal_fwd || heads <= 0 || stride < 4) return SGF_ERR_ARG;
    attn_combine_scal_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(scal_bwd, heads, stride, scal_fwd);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_head_mean(const void* x, int64_t ldx, int64_t rows, int heads, int d, int dtype, void* out, int64_t ldo, void* stream) {
    if (!x || !out || rows < 0 || heads <= 0 || d <= 0) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == 0) head_mean_kernel<float><<<ew_grid(rows * d), kRowBlock, 0, st>>>((const float*)x, ldx, rows, heads, d, (float*)out, ldo);
    else if (dtype == 1) head_mean_kernel<__nv_bfloat16><<<ew_grid(rows * d), kRowBlock, 0, st>>>((const __nv_bfloat16*)x, ldx, rows, heads, d, (__nv_bfloat16*)out, ldo);
    else return SGF_ERR_ARG;
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_attn_bwd_prep(const void* g, int64_t ld, const void* o, int64_t ld_o, const float* den, int64_t rows, int d,
                                 int dtype, float gscale, void* gnum, int64_t ld_gnum, float* gden, void* stream) {
    RowGeom gm;
    if (!geom_for(dtype, d, gm) || !aligned16(g) || !aligned16(o) || !aligned16(gnum) || !ld_ok(dtype, ld) || !ld_ok(dtype, ld_o) ||
        !ld_ok(dtype, ld_gnum) || !den || !gden || rows < 0)
        return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    SGF_DISPATCH_T_CPL(dtype, gm.cpl, (attn_bwd_prep_kernel<T, CPL><<<row_grid(rows, gm), kRowBlock, 0, st>>>(
                                          (const T*)g, (const T*)o, ld, ld_o, den, rows, d, gm.chunks, gm.lpr_log2, gscale, (T*)gnum, ld_gnum, gden)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_attn_prepare_fwd(const float* s_raw, const float* z_raw, const float* nq2, int nq2_len, const float* nk2,
                                    int nk2_len, int m, int d, void* bmat, int64_t ld_bmat, void* btail, int64_t ld_btail,
                                    int64_t plane_ld, float* scal, void* stream) {
    if (!s_raw || !z_raw || !nq2 || !nk2 || !bmat || !btail || !scal || m <= 0 || d <= 0) return SGF_ERR_ARG;
    attn_prepare_fwd_kernel<<<d + 16, 128, 0, (cudaStream_t)stream>>>(s_raw, z_raw, nq2, nq2_len, nk2, nk2_len, m, d,
                                                                      (__nv_bfloat16*)bmat, ld_bmat, (__nv_bfloat16*)btail, ld_btail,
                                                                      plane_ld, scal);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_attn_prepare_bwd(const float* s_raw, const float* z_raw, const float* ds_raw, const float* dz_raw,
                                    const float* scal_fwd, int m, int d, void* b_dq, int64_t ld_b_dq, void* b_dv, int64_t ld_b_dv,
                                    void* b_dk, int64_t ld_b_dk, int64_t plane_ld_d, int64_t plane_ld_m, float* r1_col,
                                    float* dk_bias, float* scal_bwd, void* stream) {
    if (!s_raw || !z_raw || !ds_raw || !dz_raw || !scal_fwd || !b_dq || !b_dv || !b_dk || !r1_col || !dk_bias || !scal_bwd ||
        m <= 0 || d <= 0)
        return SGF_ERR_ARG;
    attn_prepare_bwd_kernel<<<m + 1, 128, 0, (cudaStream_t)stream>>>(s_raw, z_raw, ds_raw, dz_raw, scal_fwd, m, d,
                                                                     (__nv_bfloat16*)b_dq, ld_b_dq, (__nv_bfloat16*)b_dv, ld_b_dv,
                                                                     (__nv_bfloat16*)b_dk, ld_b_dk, plane_ld_d, plane_ld_m, r1_col,
                                                                     dk_bias, scal_bwd);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_softmax_nll(const float* logits, int64_t ld, const int64_t* labels, const uint8_t* mask, int64_t rows, int c,
                               float scale, float* loss, float* dlogits, int64_t ld_d, void* ws, size_t ws_bytes,
                               void* stream) {
    if (!logits || !labels || !loss || rows < 0 || c <= 0) return SGF_ERR_ARG;
    if (rows == 0) return SGF_OK;
    int64_t blocks = (rows * 32 + kRowBlock - 1) / kRowBlock;
    int64_t cap = (int64_t)num_sms() * 8;
    if (blocks > cap) blocks = cap;
    RedWs red;
    if (int rc = red_args(ws, ws_bytes, 1, (cudaStream_t)stream, red)) return rc;
    softmax_nll_kernel<<<(unsigned)blocks, kRowBlock, 0, (cudaStream_t)stream>>>(logits, ld, labels, mask, rows, c, scale, loss,
                                                                               dlogits, ld_d, red);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_eval_acc(const float* logits, int64_t ld, const int64_t* labels, const int64_t* idx, int64_t m, int64_t rows,
                            int c, int64_t* correct, double* nll_sum, void* stream) {
    if (m < 0 || rows < 0 || c <= 0 || !correct || (m > 0 && (!logits || !labels)) || ld < c) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    SGF_CUDA_TRY(cudaMemsetAsync(correct, 0, 8, st));
    if (nll_sum) SGF_CUDA_TRY(cudaMemsetAsync(nll_sum, 0, 8, st));
    if (m == 0) return SGF_OK;
    int64_t blocks = (m * 32 + kRowBlock - 1) / kRowBlock;
    int64_t cap = (int64_t)num_sms() * 8;
    if (blocks > cap) blocks = cap;
    eval_acc_kernel<<<(unsigned)blocks, kRowBlock, 0, st>>>(logits, ld, labels, idx, m, rows, c,
                                                            reinterpret_cast<unsigned long long*>(correct), nll_sum);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

// Device-resident dropout epoch (see SeedArg).
namespace sgf {
__global__ void advance_epoch_kernel(uint64_t* e) { *e += 1; }
}  // namespace sgf

extern "C" int sgf_set_dropout_epoch(const uint64_t* epoch_dev) {
    sgf::g_dropout_epoch = epoch_dev;
    return SGF_OK;
}

extern "C" int sgf_advance_dropout_epoch(uint64_t* epoch_dev, void* stream) {
    if (!epoch_dev) return SGF_ERR_ARG;
    sgf::advance_epoch_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(epoch_dev);
    SGF_LAUNCH_CHECK(); sgf::count_launch();
    return SGF_OK;
}
