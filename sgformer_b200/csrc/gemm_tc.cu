// Dense contractions of the SGFormer encoder on Hopper tensor cores (wgmma, sm_90a).
//
//  gemm_nt : out[rows, n_out] = epilogue( sum_seg A_seg[rows, k] . B_seg[n_out, k]^T )      "row-streaming"
//            rows = nodes (huge), n_out, k <= a few hundred.  Replaces nn.Linear forward / input-gradient,
//            q~.(K^T V) and the attention backward products (reference medium/ours.py:22,28,76-85; large/ours.py:38-40,
//            123-128,141,199,275).  Both operands K-major bf16, TMA SWIZZLE_128B tiles, BM=128 x BN<=256(+16) x BK=64,
//            3-stage smem ring, fp32 accumulators in registers, warp-specialised: warp 8 = TMA producer, warps 0-7 = two
//            consumer warpgroups (64 rows of the tile each) that issue the wgmma and run the epilogue of their rows.
//  gemm_tn : out[m, n] = alpha * sum_rows A[rows, m]^T B[rows, n]                               "node-contracting"
//            Replaces K^T V (medium/ours.py:21), its backward q^T gnum and every weight gradient dW = dY^T X.
//            Both operands are MN-major for the MMA (features contiguous), loaded as [64 feat x 64 node] boxes;
//            the node range is split across CTAs, per-CTA partials go to a workspace and are reduced deterministically.
//
// Descriptor formats follow cute/atom/mma_traits_sm90_gmma.hpp (canonical SW128 layouts).
#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

#include <cstdlib>
#include <cstring>
#include <mutex>

namespace sgf {

// ------------------------------------------------------------------------------------------------
// host: cuTensorMapEncodeTiled through the runtime's driver entry point (no link dependency on libcuda)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)p;
    });
    return fn;
}

// 2-D row-major [rows, cols] (pitch ld elements) of bf16 (dtype 1) or fp32 (dtype 0); box = [box_rows x 128 bytes],
// 128-byte swizzle, OOB loads -> 0, OOB stores clipped
static int make_tmap_2d(CUtensorMap* tm, const void* base, int dtype, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return SGF_ERR_DRIVER;
    const int es = dtype == 1 ? 2 : 4;
    if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld * es) % 16 != 0 || rows <= 0 || cols <= 0 || box_rows <= 0 || box_rows > 256)
        return SGF_ERR_ARG;
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstr[1] = {(cuuint64_t)ld * es};
    cuuint32_t box[2] = {(cuuint32_t)(128 / es), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1u, 1u};
    CUresult r = enc(tm, dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                     const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? SGF_OK : SGF_ERR_DRIVER;
}
static int make_tmap_bf16(CUtensorMap* tm, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
    return make_tmap_2d(tm, base, 1, rows, cols, ld, box_rows);
}

// ================================================================================================
// gemm_nt
// ================================================================================================
namespace nt {
constexpr int BM = 128, BK = 64, STAGES = 3;
constexpr int MMA_WARPS = 8;                      // two consumer warpgroups: tile rows [0,64) and [64,128)
constexpr int THREADS = 32 * (MMA_WARPS + 4);     // warps 0..7 MMA + epilogue, warp 8 TMA producer (warps 9..11 idle)
constexpr int A_BYTES = BM * BK * 2;              // 16 KB
constexpr int B_BYTES_MAX = (256 + 16) * BK * 2;  // 34 KB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES_MAX;
constexpr int WSTG_BYTES = 16 * 128;              // output staging: a warp's 16 rows x 128 bytes (SW128), stored by its own TMA store
constexpr int BAR_BYTES = 512;
constexpr int STAT_COLS = 1024;                   // fused column statistics cover n_out <= 1024
constexpr int STAT_BYTES = 2 * STAT_COLS * 4;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + MMA_WARPS * 2 * WSTG_BYTES + BAR_BYTES + STAT_BYTES + 1024;
// Resident-B mode (p.b_res): the whole B operand of one n-block (all k-blocks) stays in shared memory across the row tiles
// of a CTA, so that only A streams through the ring.  Without it every 128-row tile re-fetches K x n_block of weights from
// L2, and at short K the few k-blocks of a tile cannot cover that latency.
constexpr int RES_BYTES = (256 + 16) * 256 * 2;   // 136 KB: K = 256 x (256 + 16-column tail)
constexpr int RES_MAX_KB = 16;                    // one full/empty mbarrier pair per resident k-block
constexpr int RES_STAGES = 3;                     // A-only ring
constexpr int SMEM_BYTES_RES = RES_BYTES + RES_STAGES * A_BYTES + MMA_WARPS * WSTG_BYTES + BAR_BYTES + STAT_BYTES + 1024;
static_assert(SMEM_BYTES <= 232448 && SMEM_BYTES_RES <= 232448, "exceeds the 227 KB of dynamic shared memory per CTA");

struct Seg {
    int a_idx, a_koff, b_idx, b_koff, k_blocks;
};
struct Params {
    int64_t rows;
    int n_out, bn_main, bn_pad, has_tail, n_blocks;   // bn_pad: bn_main rounded up to the 64-column MMA chunk
    int64_t num_tiles;
    int b_res;          // 1: resident-B schedule (see RES_BYTES)
    int64_t chunk;      // b_res: row tiles per CTA between two reloads of B (only matters when n_blocks > 1)
    int n_seg, total_kb;
    Seg seg[SGF_MAX_SEG];
    int epi;
    void* out; int64_t ldo; int out_dtype;
    const float* bias;
    const void* aux; int64_t ld_aux; int aux_dtype;
    const float* row_scale;
    float alpha, beta;
    const float* alpha_dev; const float* beta_dev;
    int relu, accumulate;
    float nf; const float* nf_dev; float* den_out;
    const float* r1_row; const float* r1_col;
    int tma_store;   // 1: epilogue stages 128-byte rows in smem and stores them with TMA; 0: direct global stores
    float* col_sum; float* col_sumsq;   // optional fused column statistics of the STORED output (tma_store path only)
};
struct Tmaps {
    CUtensorMap a[SGF_MAX_SRC];
    CUtensorMap b[SGF_MAX_SRC];
    CUtensorMap tail;
    CUtensorMap out;
};

__device__ __forceinline__ float load1(const void* base, int dtype, int64_t off) {
    return dtype == 1 ? __bfloat162float(static_cast<const __nv_bfloat16*>(base)[off]) : static_cast<const float*>(base)[off];
}
__device__ __forceinline__ void store1(void* base, int dtype, int64_t off, float v) {
    if (dtype == 1) static_cast<__nv_bfloat16*>(base)[off] = __float2bfloat16_rn(v);
    else static_cast<float*>(base)[off] = v;
}
// The two warp roles walk the CTA's tiles in the same order.
//  streaming:  tile = blockIdx.x + i*gridDim.x over (m_blk, n_blk) pairs, n_blk fastest.
//  resident-B: the CTA owns row tiles m = blockIdx.x + i*gridDim.x; they are visited in chunks of p.chunk, and inside a chunk
//              n_blk is the OUTER loop: B(n_blk) is loaded once per (chunk, n_blk) "group", the chunk's A tiles are re-read
//              from L2 for the following n-blocks (a chunk is sized to stay L2-resident).
struct TileIter {
    const Params& p;
    bool started = false;
    int64_t tile = 0;                 // streaming
    int64_t cnt = 0, c0 = 0, i = 0;   // resident
    int nb = 0;
    int64_t group = 0;
    int m_blk = 0, n_blk = 0;
    bool first = false, last = false;   // first / last tile of its group (resident)
    __device__ explicit TileIter(const Params& pp) : p(pp) {
        if (p.b_res) {
            const int64_t m_tiles = p.num_tiles / p.n_blocks;
            cnt = m_tiles > blockIdx.x ? (m_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        }
    }
    __device__ bool next() {
        if (!p.b_res) {
            tile = started ? tile + gridDim.x : blockIdx.x;
            started = true;
            if (tile >= p.num_tiles) return false;
            m_blk = (int)(tile / p.n_blocks);
            n_blk = (int)(tile % p.n_blocks);
            return true;
        }
        if (!started) {
            started = true;
            if (cnt == 0) return false;
        } else {
            ++i;
            const int64_t cend = c0 + p.chunk < cnt ? c0 + p.chunk : cnt;
            if (i >= cend) {
                ++group;
                if (++nb >= p.n_blocks) {
                    nb = 0;
                    c0 += p.chunk;
                    if (c0 >= cnt) return false;
                }
                i = c0;
            }
        }
        const int64_t cend = c0 + p.chunk < cnt ? c0 + p.chunk : cnt;
        m_blk = (int)(blockIdx.x + i * gridDim.x);
        n_blk = nb;
        first = i == c0;
        last = i == cend - 1;
        return true;
    }
};

// Epilogue feature bits.  A specialised instantiation gemm_nt_kernel<F> compiles exactly the features in F (present and
// unconditional: bf16 output through the TMA-store path, every 32-column piece complete, bf16 aligned addends); the
// F_GENERIC instantiation reads every feature from Params at run time and handles ragged widths, fp32 and unaligned tensors.
enum : int { F_BIAS = 1, F_AUX = 2, F_RELU = 4, F_ROWSCALE = 8, F_ACCUM = 16, F_R1 = 32, F_ATTN = 64, F_GENERIC = 128 };

// 16 addends of a 32-column piece in accumulator layout (d[4c + 2s + e]: row rows[s], column col0 + 8c + e)
template <bool GEN>
__device__ __forceinline__ void load_piece(const void* src, int dtype, int64_t ld, const int64_t* rows, const bool* row_ok,
                                           int col0, int n_out, bool nc, float* d) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const int col = col0 + 8 * c;
            const int64_t off = rows[s] * ld + col;
            float a0 = 0.f, a1 = 0.f;
            if (!GEN) {
                if (row_ok[s]) {
                    const uint32_t* q = reinterpret_cast<const uint32_t*>(static_cast<const __nv_bfloat16*>(src) + off);
                    unpack_bf16x2(nc ? __ldg(q) : *q, a0, a1);
                }
            } else {
                if (row_ok[s] && col < n_out) a0 = load1(src, dtype, off);
                if (row_ok[s] && col + 1 < n_out) a1 = load1(src, dtype, off + 1);
            }
            d[4 * c + 2 * s] = a0;
            d[4 * c + 2 * s + 1] = a1;
        }
}

template <int F>
__global__ void __launch_bounds__(THREADS, 1) gemm_nt_kernel(const __grid_constant__ Tmaps tm, const __grid_constant__ Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    // streaming: [ring: STAGES x (A | B)] [staging];  resident: [B: RES_BYTES] [ring: RES_STAGES x A] [staging]
    const bool res = p.b_res != 0;
    uint8_t* bres = smem;
    uint8_t* ring = res ? smem + RES_BYTES : smem;
    const int ring_stages = res ? RES_STAGES : STAGES;
    const int ring_stride = res ? A_BYTES : STAGE_BYTES;
    const int stg_per_warp = res ? 1 : 2;                 // warp-private [16 rows x 128 B] staging tiles
    uint8_t* staging = ring + ring_stages * ring_stride;
    uint64_t* full = reinterpret_cast<uint64_t*>(staging + MMA_WARPS * stg_per_warp * WSTG_BYTES);
    uint64_t* empty = full + STAGES;
    uint64_t* bres_full = empty + STAGES;
    uint64_t* bres_empty = bres_full + RES_MAX_KB;
    float* stat_sm = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full) + BAR_BYTES);   // [2][STAT_COLS]: sum, sumsq
    static_assert((2 * STAGES + 2 * RES_MAX_KB) * 8 <= BAR_BYTES, "barrier area");
    static_assert(RES_STAGES <= STAGES, "ring barriers");
    const bool want_stats = p.col_sum != nullptr || p.col_sumsq != nullptr;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const uint32_t b_tx = p.bn_pad * BK * 2 + (p.has_tail ? 16 * BK * 2 : 0);
    if (want_stats)
        for (int i = threadIdx.x; i < 2 * STAT_COLS; i += THREADS) stat_sm[i] = 0.f;

    if (threadIdx.x == 0) {
        for (int i = 0; i < p.n_seg; ++i) {
            tma_prefetch_desc(&tm.a[p.seg[i].a_idx]);
            tma_prefetch_desc(&tm.b[p.seg[i].b_idx]);
        }
        if (p.has_tail) tma_prefetch_desc(&tm.tail);
        if (p.tma_store) tma_prefetch_desc(&tm.out);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], MMA_WARPS); }
        for (int s = 0; s < RES_MAX_KB; ++s) { mbar_init(&bres_full[s], 1); mbar_init(&bres_empty[s], MMA_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= MMA_WARPS) {
        producer_regs();
        if (warp == MMA_WARPS && lane == 0) {
            // ===== TMA producer =====
            int stage = 0; uint32_t phase = 0;
            TileIter ti(p);
            while (ti.next()) {
                int kbg = 0;
                for (int s = 0; s < p.n_seg; ++s) {
                    const Seg sg = p.seg[s];
                    for (int kb = 0; kb < sg.k_blocks; ++kb, ++kbg) {
                        mbar_wait(&empty[stage], phase ^ 1);
                        uint8_t* sa = ring + stage * ring_stride;
                        if (!res) {
                            uint8_t* sb = sa + A_BYTES;
                            mbar_arrive_expect_tx(&full[stage], A_BYTES + b_tx);
                            tma_load_2d(sa, &tm.a[sg.a_idx], &full[stage], sg.a_koff + kb * BK, ti.m_blk * BM);
                            tma_load_2d(sb, &tm.b[sg.b_idx], &full[stage], sg.b_koff + kb * BK, ti.n_blk * p.bn_main);
                            if (p.has_tail) tma_load_2d(sb + p.bn_pad * BK * 2, &tm.tail, &full[stage], sg.b_koff + kb * BK, 0);
                        } else {
                            // A first (its ring slot frees early), then - on the first tile of a group - the k-block of B,
                            // as soon as the previous group's last tile has consumed the old one
                            mbar_arrive_expect_tx(&full[stage], A_BYTES);
                            tma_load_2d(sa, &tm.a[sg.a_idx], &full[stage], sg.a_koff + kb * BK, ti.m_blk * BM);
                            if (ti.first) {
                                mbar_wait(&bres_empty[kbg], (uint32_t)(ti.group & 1) ^ 1);
                                uint8_t* sb = bres + (size_t)kbg * b_tx;
                                mbar_arrive_expect_tx(&bres_full[kbg], b_tx);
                                tma_load_2d(sb, &tm.b[sg.b_idx], &bres_full[kbg], sg.b_koff + kb * BK, ti.n_blk * p.bn_main);
                                if (p.has_tail) tma_load_2d(sb + p.bn_pad * BK * 2, &tm.tail, &bres_full[kbg], sg.b_koff + kb * BK, 0);
                            }
                        }
                        if (++stage == ring_stages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
        return;
    }
    consumer_regs();

    // ===== consumers: wgmma over the tile's k-blocks, then the epilogue of the warpgroup's 64 rows =====
    constexpr bool GEN = (F & F_GENERIC) != 0;
    const bool f_bias = GEN ? p.bias != nullptr : (F & F_BIAS) != 0;
    const bool f_aux = GEN ? p.aux != nullptr : (F & F_AUX) != 0;
    const bool f_relu = GEN ? p.relu != 0 : (F & F_RELU) != 0;
    const bool f_rs = GEN ? p.row_scale != nullptr : (F & F_ROWSCALE) != 0;
    const bool f_acc = GEN ? p.accumulate != 0 : (F & F_ACCUM) != 0;
    const bool f_r1 = GEN ? p.r1_row != nullptr : (F & F_R1) != 0;
    const bool f_attn = GEN ? (p.epi == SGF_EPI_ATTN_APPLY || p.epi == SGF_EPI_ATTN_GRAM) : (F & F_ATTN) != 0;
    const bool f_tma = GEN ? p.tma_store != 0 : true;
    const bool f_stats = GEN ? want_stats : false;
    const int out_dtype = GEN ? p.out_dtype : 1;
    const int wg = warp >> 2;      // warpgroup: tile rows [64 wg, 64 wg + 64)
    const int wq = warp & 3;       // warp in the warpgroup: 16 of those rows
    const int rr = lane >> 2;      // accumulator rows rr and rr + 8 of the warp's 16
    const int cq = 2 * (lane & 3); // accumulator columns cq, cq + 1 of every 8
    float alpha = p.alpha, beta = p.beta;
    if (p.alpha_dev) alpha *= *p.alpha_dev;
    if (p.beta_dev) beta *= *p.beta_dev;
    const float nfv = (f_attn && p.nf_dev) ? *p.nf_dev : p.nf;
    const int GW = out_dtype == 1 ? 64 : 32;              // columns per 128-byte staging row
    const int ppg = GW / 32;                              // pieces per staging group (bf16: 2, fp32: 1)
    const int n_pieces = (p.bn_main + 31) / 32;
    const int nch = p.bn_pad / 64;                        // 64-column MMA chunks
    uint8_t* wstg = staging + warp * stg_per_warp * WSTG_BYTES;
    const uint32_t a_off = wg * 64 * BK * 2;

    float acc[4][32];
    float acct[8];
    uint32_t gcount = 0;
    int stage = 0; uint32_t phase = 0;
    TileIter ti(p);
    while (ti.next()) {
        for (int kbg = 0; kbg < p.total_kb; ++kbg) {
            if (res && ti.first) mbar_wait(&bres_full[kbg], (uint32_t)(ti.group & 1));
            mbar_wait(&full[stage], phase);
            const uint32_t sa = smem_u32(ring + stage * ring_stride) + a_off;
            const uint32_t sb = res ? smem_u32(bres) + (uint32_t)kbg * b_tx : smem_u32(ring + stage * ring_stride) + A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                const uint64_t da = make_smem_desc_sw128(sa + k * 32, 16, 1024);
                const uint32_t sc = (kbg > 0 || k > 0) ? 1u : 0u;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (j < nch) wgmma_n64<0, 0>(acc[j], da, make_smem_desc_sw128(sb + j * 8192 + k * 32, 16, 1024), sc);
                if (p.has_tail) wgmma_n16<0, 0>(acct, da, make_smem_desc_sw128(sb + p.bn_pad * BK * 2 + k * 32, 16, 1024), sc);
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < 4; ++j) fence_regs(acc[j]);
            fence_regs(acct);
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&empty[stage]);
                if (res && ti.last) mbar_arrive(&bres_empty[kbg]);
            }
            if (++stage == ring_stages) { stage = 0; phase ^= 1; }
        }

        // -------- epilogue --------
        const int m_blk = ti.m_blk, n_blk = ti.n_blk;
        const int64_t row_w = (int64_t)m_blk * BM + wg * 64 + wq * 16;     // first row of this warp's 16
        const int64_t rows[2] = {row_w + rr, row_w + rr + 8};
        const bool row_ok[2] = {rows[0] < p.rows, rows[1] < p.rows};
        const int col_base = n_blk * p.bn_main;
        float rs[2] = {1.f, 1.f}, r1r[2] = {0.f, 0.f}, inv_den[2] = {1.f, 1.f};
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            if (f_rs && row_ok[s]) rs[s] = p.row_scale[rows[s]];
            if (f_r1 && row_ok[s]) r1r[s] = p.r1_row[rows[s]];
        }
        if (f_attn) {
            // tail column 0 of rows rr / rr + 8 is held by lane 4 rr
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const float den = __shfl_sync(0xffffffffu, acct[2 * s], lane & ~3) + nfv;
                inv_den[s] = 1.f / den;
                if (row_ok[s] && p.den_out && n_blk == 0 && (lane & 3) == 0) p.den_out[rows[s]] = den;
            }
        }
        // -------- 32-column pieces; piece pc covers tile columns [32 pc, 32 pc + 32) --------
#pragma unroll
        for (int pc = 0; pc < 8; ++pc) {
            if (pc >= n_pieces) break;
            const int g = pc / ppg, pp = pc % ppg;
            const uint32_t buf = stg_per_warp == 2 ? (gcount & 1) : 0;
            if (f_tma && pp == 0) {
                if (lane == 0) {                                   // the store that last used this buffer has drained
                    if (stg_per_warp == 2) bulk_wait_read<1>(); else bulk_wait_read<0>();
                }
                __syncwarp();
            }
            float v[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = acc[pc >> 1][(pc & 1) * 16 + i];
            const int col0 = col_base + pc * 32 + cq;              // column of v[0]; v[4c + 2s + e] is column col0 + 8c + e
            float ax[16], old[16];
            if (f_aux) load_piece<GEN>(p.aux, p.aux_dtype, p.ld_aux, rows, row_ok, col0, p.n_out, true, ax);
            if (f_acc) load_piece<GEN>(p.out, out_dtype, p.ldo, rows, row_ok, col0, p.n_out, false, old);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int s = (i >> 1) & 1;
                const int col = col0 + 8 * (i >> 2) + (i & 1);
                const bool cok = !GEN || col < p.n_out;
                float x = v[i];
                if (f_attn) {
                    // out = (acc + nf*aux + bias) / (tail + nf): ATTN_APPLY carries aux (= v), ATTN_GRAM the bias bt
                    if (f_aux) x += nfv * ax[i];
                    if (f_bias && cok) x += __ldg(p.bias + col);
                    x *= inv_den[s];
                } else {
                    x *= alpha;
                    if (f_aux) x += beta * ax[i];
                    if (f_bias && cok) x += __ldg(p.bias + col);
                    if (f_r1 && cok) x += r1r[s] * __ldg(p.r1_col + col);
                    if (f_relu) x = fmaxf(x, 0.f);
                    if (f_rs) x *= rs[s];
                }
                if (f_acc) x += old[i];
                v[i] = x;
            }
            if (f_tma) {
                // 128-byte staging rows, 16-byte chunks XOR-swizzled with (row & 7) (== TMA SWIZZLE_128B); OOB rows/cols
                // are clipped by the TMA store, so garbage there is harmless
                uint8_t* tile = wstg + buf * WSTG_BYTES;
#pragma unroll
                for (int c = 0; c < 4; ++c)
#pragma unroll
                    for (int s = 0; s < 2; ++s) {
                        const int r = rr + 8 * s;
                        if (out_dtype == 1) {
                            const int chunk = (pp * 4 + c) ^ (r & 7);
                            *reinterpret_cast<uint32_t*>(tile + r * 128 + chunk * 16 + 2 * cq) = pack_bf16x2(v[4 * c + 2 * s], v[4 * c + 2 * s + 1]);
                        } else {
                            const int chunk = (2 * c + (cq >> 2)) ^ (r & 7);
                            *reinterpret_cast<float2*>(tile + r * 128 + chunk * 16 + 4 * (cq & 3)) = make_float2(v[4 * c + 2 * s], v[4 * c + 2 * s + 1]);
                        }
                    }
            } else if constexpr (GEN) {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int s = (i >> 1) & 1;
                    const int col = col0 + 8 * (i >> 2) + (i & 1);
                    if (row_ok[s] && col < p.n_out) store1(p.out, out_dtype, rows[s] * p.ldo + col, v[i]);
                }
            }
            if (f_tma && (pp == ppg - 1 || pc == n_pieces - 1)) {
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) {
                    tma_store_2d(&tm.out, wstg + buf * WSTG_BYTES, col_base + g * GW, (int32_t)row_w);
                    bulk_commit();
                }
                if (f_stats) {
                    // column sums of the staged (already rounded) 16-row tile: lane l owns columns l (and l + 32 for bf16);
                    // the buffer is rewritten only after this warp's next bulk_wait_read + __syncwarp
                    const uint8_t* tile = wstg + buf * WSTG_BYTES;
                    const int64_t valid_rows = p.rows - row_w;
                    for (int cg = lane; cg < GW; cg += 32) {
                        const int colg = col_base + g * GW + cg;
                        if (colg >= p.n_out || colg >= col_base + p.bn_main) continue;
                        float s1 = 0.f, s2 = 0.f;
                        for (int r = 0; r < 16 && r < valid_rows; ++r) {
                            float x;
                            if (out_dtype == 1) {
                                const int chunk = (cg >> 3) ^ (r & 7);
                                x = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(tile + r * 128 + chunk * 16 + (cg & 7) * 2));
                            } else {
                                const int chunk = (cg >> 2) ^ (r & 7);
                                x = *reinterpret_cast<const float*>(tile + r * 128 + chunk * 16 + (cg & 3) * 4);
                            }
                            s1 += x;
                            s2 += x * x;
                        }
                        atomicAdd(&stat_sm[colg], s1);
                        atomicAdd(&stat_sm[STAT_COLS + colg], s2);
                    }
                }
                ++gcount;
            }
        }
    }
    if (f_tma && lane == 0) bulk_wait<0>();
    if (f_stats) {
        named_bar_sync(3, 32 * MMA_WARPS);
        for (int i = threadIdx.x; i < p.n_out; i += 32 * MMA_WARPS) {
            if (p.col_sum) atomicAdd(&p.col_sum[i], stat_sm[i]);
            if (p.col_sumsq) atomicAdd(&p.col_sumsq[i], stat_sm[STAT_COLS + i]);
        }
    }
}
}  // namespace nt

// ================================================================================================
// node-contracting products (gemm_tn, gram): flushing the register accumulators
// ================================================================================================
// The error of one wgmma accumulator grows with the number of nodes it sums: measured on an H100, sgf_gram over 300 k rows of
// bf16x3 operands (about 4500 rows per accumulator) missed fp64 by 2.7e-5 relative, beyond the 2e-5 that tests/test_gpu_kernels.py
// allows (a bias consistent with truncating fp32 accumulation).  Every FLUSH_KB node blocks (1024 rows) a thread adds its
// accumulators into its own fp32 workspace partial (round-to-nearest, fixed order: deterministic) and restarts them from zero.
constexpr int FLUSH_KB = 16;
// ws[col * mp + row] (+)= acc for the accumulator rows mrow, mrow + 8 and columns 64 j + 8c + cq + e < ncols of the chunks
// j in [j0, 4); acc is zeroed.
__device__ __forceinline__ void flush_acc(float (&acc)[4][32], float* ws, int mp, int mrow, int cq, int j0, int ncols, bool add) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j < j0) continue;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int col = 64 * j + 8 * (i >> 2) + cq + (i & 1);
            float* w = ws + (int64_t)col * mp + mrow + 8 * ((i >> 1) & 1);
            if (col < ncols) *w = add ? *w + acc[j][i] : acc[j][i];
            acc[j][i] = 0.f;
        }
    }
}

// ================================================================================================
// gemm_tn
// ================================================================================================
// CTA (x, y): features [128 x, 128 x + 128) of A (one warpgroup per 64) against all n of B, over the y-th slice of the
// node blocks.  CTAs that share a node slice run side by side, so the second read of B hits L2.
namespace tn {
constexpr int BKN = 64, STAGES = 4, MMA_WARPS = 8, THREADS = 32 * (MMA_WARPS + 4);   // + the producer warpgroup
constexpr int CHUNK_BYTES = 64 * BKN * 2;   // one [64 feat x 64 node] box = 8 KB
constexpr int A_BYTES = 2 * CHUNK_BYTES;    // the CTA's 128 features of A
constexpr int B_BYTES = 4 * CHUNK_BYTES;    // up to 256 features of B
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;  // 48 KB
constexpr int BAR_BYTES = 256;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + 1024;

struct Params {
    int64_t rows;
    int m, n, mp, n_chunks, un;   // mp = m rounded up to 128, un = n rounded up to 16
    int64_t kb_total;
    float* ws;  // [gridDim.y][un][mp]
    int n_pairs;                                  // partial products accumulated per node block (1, or the 6 of bf16x3)
    int a_off[SGF_TN_MAX_PAIRS], b_off[SGF_TN_MAX_PAIRS];   // column offset (elements) of the plane each product reads
};
struct Tmaps {
    CUtensorMap a, b;
};

__global__ void __launch_bounds__(THREADS, 1) gemm_tn_kernel(const __grid_constant__ Tmaps tm, const __grid_constant__ Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    // contiguous slice of 64-row node blocks for this CTA
    const int64_t per = p.kb_total / gridDim.y, rem = p.kb_total % gridDim.y;
    const int64_t kb0 = blockIdx.y * per + (blockIdx.y < rem ? blockIdx.y : rem);
    const int64_t kb1 = kb0 + per + (blockIdx.y < rem ? 1 : 0);
    const int m0 = blockIdx.x * 128;
    const int a_chunks = (p.m - m0) >= 128 ? 2 : ((p.m - m0) + 63) / 64;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm.a);
        tma_prefetch_desc(&tm.b);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], MMA_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= MMA_WARPS) {
        producer_regs();
        if (warp == MMA_WARPS && lane == 0) {
            const uint32_t stage_tx = (a_chunks + p.n_chunks) * CHUNK_BYTES;
            int stage = 0; uint32_t phase = 0;
            // all partial products of a node block before the next block: the planes re-read by later products hit L2
            for (int64_t kb = kb0; kb < kb1; ++kb) {
                for (int pr = 0; pr < p.n_pairs; ++pr) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * STAGE_BYTES;
                    uint8_t* sb = sa + A_BYTES;
                    mbar_arrive_expect_tx(&full[stage], stage_tx);
                    for (int c = 0; c < a_chunks; ++c)
                        tma_load_2d(sa + c * CHUNK_BYTES, &tm.a, &full[stage], p.a_off[pr] + m0 + c * 64, (int32_t)(kb * BKN));
                    for (int c = 0; c < p.n_chunks; ++c)
                        tma_load_2d(sb + c * CHUNK_BYTES, &tm.b, &full[stage], p.b_off[pr] + c * 64, (int32_t)(kb * BKN));
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }
    consumer_regs();

    const int wg = warp >> 2, wq = warp & 3;
    const bool active = wg < a_chunks;
    float acc[4][32];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
    // partial [un][mp] of this node slice: accumulator row = feature of A, column = feature of B
    float* ws = p.ws + (int64_t)blockIdx.y * p.un * p.mp;
    const int mrow = m0 + wg * 64 + wq * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    bool flushed = false;
    int stage = 0; uint32_t phase = 0;
    for (int64_t kb = kb0; kb < kb1; ++kb) {
        for (int pr = 0; pr < p.n_pairs; ++pr) {
            mbar_wait(&full[stage], phase);
            if (active) {
                const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + wg * CHUNK_BYTES;
                const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES) + A_BYTES;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BKN / 16; ++k) {
                    // MN-major SW128: LBO = stride between 64-element feature chunks, SBO = stride between 8-row node groups
                    const uint64_t da = make_smem_desc_sw128(sa + k * 2048, CHUNK_BYTES, 1024);
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (j < p.n_chunks) wgmma_n64<1, 1>(acc[j], da, make_smem_desc_sw128(sb + j * CHUNK_BYTES + k * 2048, CHUNK_BYTES, 1024), 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();
#pragma unroll
                for (int j = 0; j < 4; ++j) fence_regs(acc[j]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if (active && (kb - kb0 + 1) % FLUSH_KB == 0 && kb + 1 < kb1) {
            flush_acc(acc, ws, p.mp, mrow, cq, 0, p.un, flushed);
            flushed = true;
        }
    }
    flush_acc(acc, ws, p.mp, mrow, cq, 0, p.un, flushed);
}

// out[i,j] = alpha * sum_cta ws[cta][j][i] (+ beta*out[i,j]);  i < m, j < n
__global__ void tn_reduce_kernel(const float* __restrict__ ws, int nparts, int mp, int un, int m, int n, float alpha,
                                 const float* __restrict__ alpha_dev, float beta, float* __restrict__ out, int64_t ldo, int transpose_out) {
    const int64_t total = (int64_t)n * mp;
    const float a = alpha * (alpha_dev ? *alpha_dev : 1.f);
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(t / mp), i = (int)(t % mp);
        if (i >= m) continue;
        float s = 0.f;
        for (int c = 0; c < nparts; ++c) s += ws[((int64_t)c * un + j) * mp + i];
        float* o = transpose_out ? &out[(int64_t)j * ldo + i] : &out[(int64_t)i * ldo + j];
        *o = a * s + (beta != 0.f ? beta * *o : 0.f);
    }
}
}  // namespace tn
// ================================================================================================
// gram : G[h,h] = X^T X and s[h] = X^T 1 of one bf16 operand X [rows, h <= 256] — pass 1 of the Gram-form attention
// ================================================================================================
// The node-contracting product of gemm_tn specialised for A == B (reference contractions it replaces: k^T v, k^T 1, ||q||^2,
// ||k||^2 of medium/ours.py:16-31 — all functions of X^T X, see csrc/attn_gram.cu):
//  * every [64 feat x 64 node] box is loaded ONCE and feeds both operands of the MMA (A and B descriptors point into the same
//    shared-memory tile), so the kernel moves rows*h*2 bytes for 2*rows*h^2 flops instead of twice that;
//  * G is symmetric: of the 64 x 64 feature blocks only those with column block >= row block are accumulated, the
//    reduction kernel mirrors the rest.  A warpgroup owns one row block; CTA x pairs row blocks x and 2*m_blocks-1-x so that
//    both CTAs of h = 256 issue the same number of MMAs;
//  * X^T 1 rides along as an N = 16 MMA against a constant all-ones tile;
//  * bf16x3 operands (fp32 mode): the six plane pairs of kernels._PAIRS3 accumulate into the same registers.
// The node range is split across the CTAs; per-CTA partials -> workspace -> fixed-order reduction (deterministic).
namespace gramk {
constexpr int BKN = 64, MMA_WARPS = 8, THREADS = 32 * (MMA_WARPS + 4);   // + the producer warpgroup
constexpr int CHUNK_BYTES = 64 * BKN * 2;        // one [64 feat x 64 node] box = 8 KB
constexpr int ONES_BYTES = CHUNK_BYTES;          // constant tile of bf16 1.0
constexpr int BAR_BYTES = 256;
constexpr int SMEM_BUDGET = 200 * 1024;          // stages * planes * chunks * 8 KB
constexpr int MAX_STAGES = 8;

struct Params {
    int64_t rows, kb_total;
    int h, chunks, m_blocks, un, mp, n_planes, stages;
    int plane_off[3];                             // column offset (elements) of each plane
    int n_pairs, pa[6], pb[6];
    float* ws;                                    // [gridDim.y][un + 1][mp]: G rows (features) x columns, then X^T 1
};

__global__ void __launch_bounds__(THREADS, 1) gram_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    const int c0 = blockIdx.x;                       // first feature chunk this CTA reads
    const int nld = p.chunks - c0;                   // chunks [c0, chunks) are loaded
    const int plane_bytes = nld * CHUNK_BYTES;
    const int stage_stride = p.n_planes * p.chunks * CHUNK_BYTES;
    uint8_t* ones = smem + p.stages * stage_stride;
    uint64_t* full = reinterpret_cast<uint64_t*>(ones + ONES_BYTES);
    uint64_t* empty = full + MAX_STAGES;
    static_assert(2 * MAX_STAGES * 8 <= BAR_BYTES, "barrier area");

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t per = p.kb_total / gridDim.y, rem = p.kb_total % gridDim.y;
    const int64_t kb0 = blockIdx.y * per + (blockIdx.y < rem ? blockIdx.y : rem);
    const int64_t kb1 = kb0 + per + (blockIdx.y < rem ? 1 : 0);

    for (int i = threadIdx.x; i < ONES_BYTES / 4; i += THREADS) reinterpret_cast<uint32_t*>(ones)[i] = 0x3F803F80u;   // bf16 1.0 x2
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm);
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], MMA_WARPS); }
        fence_barrier_init();
    }
    fence_proxy_async_smem();        // the generic-proxy writes of the ones tile must be visible to the tensor core (async proxy)
    __syncthreads();

    if (warp >= MMA_WARPS) {
        producer_regs();
        if (warp == MMA_WARPS && lane == 0) {
            int stage = 0; uint32_t phase = 0;
            for (int64_t kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * stage_stride;
                mbar_arrive_expect_tx(&full[stage], (uint32_t)(p.n_planes * plane_bytes));
                for (int pl = 0; pl < p.n_planes; ++pl)
                    for (int c = 0; c < nld; ++c)
                        tma_load_2d(sa + pl * plane_bytes + c * CHUNK_BYTES, &tm, &full[stage], p.plane_off[pl] + (c0 + c) * 64, (int32_t)(kb * BKN));
                if (++stage == p.stages) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }
    consumer_regs();

    const int wg = warp >> 2, wq = warp & 3;
    const int ic = wg == 0 ? blockIdx.x : 2 * p.m_blocks - 1 - blockIdx.x;    // this warpgroup's row block
    const bool active = ic < p.chunks;
    float acc[4][32], accs[8];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) accs[i] = 0.f;
    const uint32_t s_ones = smem_u32(ones);
    float* ws = p.ws + (int64_t)blockIdx.y * (p.un + 1) * p.mp;
    const int mrow = ic * 64 + wq * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    bool flushed = false;
    // G partial of the chunks j >= ic, then column 0 of the ones product (X^T 1) as workspace column un
    auto flush = [&]() {
        flush_acc(acc, ws, p.mp, mrow, cq, ic, p.un, flushed);
        if (cq == 0) {
            float* w = ws + (int64_t)p.un * p.mp + mrow;
            w[0] = flushed ? w[0] + accs[0] : accs[0];
            w[8] = flushed ? w[8] + accs[2] : accs[2];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) accs[i] = 0.f;
        flushed = true;
    };
    int stage = 0; uint32_t phase = 0;
    for (int64_t kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full[stage], phase);
        if (active) {
            const uint32_t sa = smem_u32(smem + stage * stage_stride);
            wgmma_fence();
            for (int pr = 0; pr < p.n_pairs; ++pr) {
                const uint32_t a0 = sa + p.pa[pr] * plane_bytes + (ic - c0) * CHUNK_BYTES, b0 = sa + p.pb[pr] * plane_bytes;
#pragma unroll
                for (int k = 0; k < BKN / 16; ++k) {
                    // MN-major SW128: LBO = stride between 64-element feature chunks, SBO = stride between 8-row node groups
                    const uint64_t da = make_smem_desc_sw128(a0 + k * 2048, CHUNK_BYTES, 1024);
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (j >= ic && j < p.chunks)
                            wgmma_n64<1, 1>(acc[j], da, make_smem_desc_sw128(b0 + (j - c0) * CHUNK_BYTES + k * 2048, CHUNK_BYTES, 1024), 1u);
                }
            }
            for (int pl = 0; pl < p.n_planes; ++pl) {
                const uint32_t a0 = sa + pl * plane_bytes + (ic - c0) * CHUNK_BYTES;
#pragma unroll
                for (int k = 0; k < BKN / 16; ++k)
                    wgmma_n16<1, 1>(accs, make_smem_desc_sw128(a0 + k * 2048, CHUNK_BYTES, 1024),
                                    make_smem_desc_sw128(s_ones + k * 2048, CHUNK_BYTES, 1024), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < 4; ++j) fence_regs(acc[j]);
            fence_regs(accs);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
        if (active && (kb - kb0 + 1) % FLUSH_KB == 0 && kb + 1 < kb1) flush();
    }
    if (active) flush();
}

// G (both triangles) and s from the per-CTA partials, summed in CTA order (deterministic).  Entries below the block
// diagonal were not accumulated: they read their mirror image.
__global__ void gram_reduce_kernel(const float* __restrict__ ws, int nparts, int un, int mp, int h, float* __restrict__ G,
                                   int64_t ldg, float* __restrict__ s) {
    const int total = h * h + h;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        int i, c;
        if (t < h * h) {
            const int r = t / h, q = t % h;
            const bool upper = (q >> 6) >= (r >> 6);
            i = upper ? r : q;
            c = upper ? q : r;
        } else {
            i = t - h * h;
            c = un;
        }
        float acc = 0.f;
        for (int part = 0; part < nparts; ++part) acc += ws[((int64_t)part * (un + 1) + c) * mp + i];
        if (t < h * h) G[(int64_t)(t / h) * ldg + t % h] = acc;
        else s[i] = acc;
    }
}
}  // namespace gramk
}  // namespace sgf

using namespace sgf;

extern "C" int sgf_gemm_nt(const sgf_gemm_nt_args* a, void* stream) {
    if (!a || a->rows < 0 || a->n_out <= 0 || a->n_seg <= 0 || a->n_seg > SGF_MAX_SEG || a->n_a <= 0 || a->n_a > SGF_MAX_SRC ||
        a->n_b <= 0 || a->n_b > SGF_MAX_SRC || !a->out)
        return SGF_ERR_ARG;
    if (a->out_dtype != 0 && a->out_dtype != 1) return SGF_ERR_ARG;
    if (a->aux && a->aux_dtype != 0 && a->aux_dtype != 1) return SGF_ERR_ARG;
    if (a->rows == 0) return SGF_OK;
    const bool has_tail = a->b_tail != nullptr;
    if (has_tail && (a->n_b != 1 || a->n_out > 256)) return SGF_ERR_ARG;
    if (a->epi == SGF_EPI_ATTN_APPLY && (!has_tail || !a->aux)) return SGF_ERR_ARG;
    if (a->epi == SGF_EPI_ATTN_GRAM && (!has_tail || !a->bias || !a->nf_dev || a->aux)) return SGF_ERR_ARG;
    if (a->epi != SGF_EPI_AFFINE && a->epi != SGF_EPI_ATTN_APPLY && a->epi != SGF_EPI_ATTN_GRAM) return SGF_ERR_ARG;
    if ((a->r1_row == nullptr) != (a->r1_col == nullptr)) return SGF_ERR_ARG;

    nt::Params p;
    memset(&p, 0, sizeof(p));
    nt::Tmaps tm;
    memset(&tm, 0, sizeof(tm));
    p.rows = a->rows;
    p.n_out = a->n_out;
    const int n16 = (a->n_out + 15) / 16 * 16;
    p.n_blocks = (n16 + 255) / 256;
    // a 256-wide output with a 16-column tail is one n-block when the whole B (all k-blocks of the 256 + 16 columns) can stay
    // resident in shared memory: A is read once and B never again.  Otherwise it is split into two 128(+16) blocks (the tail
    // is recomputed, cheap), so that a streamed stage of B fits the ring.
    bool tail_one_block = false;
    if (has_tail && n16 + 16 > 256) {
        static const bool res_ok = [] { const char* e = getenv("SGF_ATTN_RESIDENT"); return !(e && e[0] == '0'); }();
        int kb = 0;
        for (int s = 0; s < a->n_seg; ++s) kb += (a->seg_klen[s] + nt::BK - 1) / nt::BK;
        tail_one_block = res_ok && a->schedule != SGF_GEMM_STREAM_B && n16 <= 256 && kb <= nt::RES_MAX_KB &&
                         (int64_t)((n16 + 63) / 64 * 64 + 16) * nt::BK * 2 * kb <= nt::RES_BYTES;
        if (!tail_one_block) p.n_blocks = 2;
    }
    // equal-width n-blocks: a multiple of 16 (UMMA N), and of 64 when there are several - the epilogue stores 128-byte
    // groups (64 bf16 / 32 fp32 columns), which must not reach into the next n-block's columns
    p.bn_main = p.n_blocks == 1 ? n16 : ((n16 / p.n_blocks + 63) / 64) * 64;
    if (p.bn_main > 256) return SGF_ERR_UNSUPPORTED;
    p.n_blocks = (n16 + p.bn_main - 1) / p.bn_main;
    p.bn_pad = (p.bn_main + 63) / 64 * 64;
    p.has_tail = has_tail ? 1 : 0;
    const int64_t m_blocks = (a->rows + nt::BM - 1) / nt::BM;
    p.num_tiles = m_blocks * p.n_blocks;
    p.n_seg = a->n_seg;
    p.total_kb = 0;
    for (int s = 0; s < a->n_seg; ++s) {
        const int ai = a->seg_a[s], bi = a->seg_b[s];
        if (ai < 0 || ai >= a->n_a || bi < 0 || bi >= a->n_b || a->seg_klen[s] <= 0) return SGF_ERR_ARG;
        const int klen = a->seg_klen[s];
        // A partial last k-block (klen % 64 != 0) reads A/B columns past koff+klen: the caller guarantees that those A
        // columns are zero (zero padding or the end of the tensor, where TMA zero-fills) and the B columns finite.
        if (a->seg_akoff[s] + klen > a->a_cols[ai] || a->seg_bkoff[s] + klen > a->b_cols[bi]) return SGF_ERR_ARG;
        p.seg[s].a_idx = ai; p.seg[s].a_koff = a->seg_akoff[s];
        p.seg[s].b_idx = bi; p.seg[s].b_koff = a->seg_bkoff[s];
        p.seg[s].k_blocks = (klen + nt::BK - 1) / nt::BK;
        p.total_kb += p.seg[s].k_blocks;
    }
    // explicit resident-B request: narrow the n-blocks until one block of B fits (A is then re-read from L2 per n-block)
    if (a->schedule == SGF_GEMM_RESIDENT_B && !has_tail) {
        while ((int64_t)p.bn_pad * nt::BK * 2 * p.total_kb > nt::RES_BYTES && p.bn_main > 64) {
            p.bn_main = p.bn_pad = p.bn_pad - 64;
            p.n_blocks = (n16 + p.bn_main - 1) / p.bn_main;
        }
        p.num_tiles = m_blocks * p.n_blocks;
    }
    int rc;
    for (int i = 0; i < a->n_a; ++i)
        if ((rc = make_tmap_bf16(&tm.a[i], a->a[i], a->rows, a->a_cols[i], a->lda[i], nt::BM))) return rc;
    for (int i = 0; i < a->n_b; ++i)
        if ((rc = make_tmap_bf16(&tm.b[i], a->b[i], a->n_out, a->b_cols[i], a->ldb[i], p.bn_pad))) return rc;
    if (has_tail && (rc = make_tmap_bf16(&tm.tail, a->b_tail, 16, a->b_cols[0], a->ldb_tail, 16))) return rc;

    p.epi = a->epi;
    p.out = a->out; p.ldo = a->ldo; p.out_dtype = a->out_dtype;
    p.bias = a->bias;
    p.aux = a->aux; p.ld_aux = a->ld_aux; p.aux_dtype = a->aux_dtype;
    p.row_scale = a->row_scale;
    p.alpha = a->alpha; p.beta = a->beta; p.alpha_dev = a->alpha_dev; p.beta_dev = a->beta_dev;
    p.relu = a->relu; p.accumulate = a->accumulate;
    p.nf = a->nf; p.nf_dev = a->nf_dev; p.den_out = a->den_out;
    p.r1_row = a->r1_row; p.r1_col = a->r1_col;
    {
        const int es = a->out_dtype == 1 ? 2 : 4;
        p.tma_store = ((reinterpret_cast<uintptr_t>(a->out) & 15) == 0 && (a->ldo * es) % 16 == 0) ? 1 : 0;
        if (p.tma_store && (rc = make_tmap_2d(&tm.out, a->out, a->out_dtype, a->rows, a->n_out, a->ldo, 16))) return rc;
        p.col_sum = a->col_sum; p.col_sumsq = a->col_sumsq;
        if ((p.col_sum || p.col_sumsq) && (!p.tma_store || a->n_out > nt::STAT_COLS)) return SGF_ERR_UNSUPPORTED;
    }

    // resident-B schedule whenever one n-block of B (all k-blocks) fits: see nt::RES_BYTES
    {
        const int64_t b_tx = (int64_t)(p.bn_pad + (has_tail ? 16 : 0)) * nt::BK * 2;
        const bool fits = p.total_kb <= nt::RES_MAX_KB && b_tx * p.total_kb <= nt::RES_BYTES;
        if (a->schedule == SGF_GEMM_RESIDENT_B && !fits) return SGF_ERR_UNSUPPORTED;
        // AUTO: resident when the whole B is one n-block (loaded once per CTA), where short K leaves a tile too few k-blocks
        // to cover the latency of re-fetching B.  With several n-blocks the per-chunk reload of B stalls the MMA.
        p.b_res = (fits && (a->schedule == SGF_GEMM_RESIDENT_B || (a->schedule == SGF_GEMM_AUTO && p.n_blocks == 1))) ? 1 : 0;
        // several n-blocks: B is re-loaded per (chunk, n-block); a chunk of 4 row tiles per CTA keeps the A tiles that are
        // re-read for the following n-blocks inside the 50 MB L2 (132 CTAs x 4 x 128 rows x K x 2 B = 35 MB at K = 256)
        p.chunk = p.n_blocks == 1 ? (int64_t)1 << 40 : 4;
    }
    // resident-B: one CTA per SM over ROW tiles (every CTA visits all n-blocks of its rows)
    const int64_t work = p.b_res ? m_blocks : p.num_tiles;
    const int64_t grid = work < num_sms() ? work : num_sms();
    const int smem_bytes = p.b_res ? nt::SMEM_BYTES_RES : nt::SMEM_BYTES;

    // epilogue specialisation: the exact feature set of this call if it has a compiled instantiation, else the generic kernel
    int feat = (a->bias ? nt::F_BIAS : 0) | (a->aux ? nt::F_AUX : 0) | (a->relu ? nt::F_RELU : 0) |
               (a->row_scale ? nt::F_ROWSCALE : 0) | (a->accumulate ? nt::F_ACCUM : 0) | (a->r1_row ? nt::F_R1 : 0) |
               (a->epi != SGF_EPI_AFFINE ? nt::F_ATTN : 0);
    const bool al16 = (!a->bias || (reinterpret_cast<uintptr_t>(a->bias) & 15) == 0) &&
                      (!a->r1_col || (reinterpret_cast<uintptr_t>(a->r1_col) & 15) == 0) &&
                      (!a->aux || (a->aux_dtype == 1 && (reinterpret_cast<uintptr_t>(a->aux) & 15) == 0 && (a->ld_aux * 2) % 16 == 0));
    const bool fast_ok = p.tma_store && a->out_dtype == 1 && a->n_out % 32 == 0 && al16 && !p.col_sum && !p.col_sumsq &&
                         p.n_blocks * p.bn_main == a->n_out;     // every 32-column piece of every n-block is complete
    static const bool no_special = [] { const char* e = getenv("SGF_GEMM_NT_GENERIC"); return e && e[0] == '1'; }();
    if (!fast_ok || no_special) feat = nt::F_GENERIC;
    const int smem_max = nt::SMEM_BYTES > nt::SMEM_BYTES_RES ? nt::SMEM_BYTES : nt::SMEM_BYTES_RES;
#define SGF_NT_CASE(FEAT)                                                                                                   \
    case (FEAT): {                                                                                                         \
        static bool attr_set = false;                                                                                      \
        if (!attr_set) {                                                                                                   \
            SGF_CUDA_TRY(cudaFuncSetAttribute(nt::gemm_nt_kernel<(FEAT)>, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                              smem_max));                                                                  \
            attr_set = true;                                                                                               \
        }                                                                                                                  \
        nt::gemm_nt_kernel<(FEAT)><<<(unsigned)grid, nt::THREADS, smem_bytes, (cudaStream_t)stream>>>(tm, p);              \
        launched = true;                                                                                                   \
    } break;
    for (int attempt = 0; attempt < 2; ++attempt) {
        bool launched = false;
        switch (feat) {
            SGF_NT_CASE(0)
            SGF_NT_CASE(nt::F_BIAS)
            SGF_NT_CASE(nt::F_BIAS | nt::F_RELU)
            SGF_NT_CASE(nt::F_ROWSCALE)
            SGF_NT_CASE(nt::F_ACCUM)
            SGF_NT_CASE(nt::F_AUX)
            SGF_NT_CASE(nt::F_AUX | nt::F_ACCUM)
            SGF_NT_CASE(nt::F_AUX | nt::F_BIAS)
            SGF_NT_CASE(nt::F_AUX | nt::F_R1)
            SGF_NT_CASE(nt::F_AUX | nt::F_ATTN)
            SGF_NT_CASE(nt::F_BIAS | nt::F_ATTN)
            SGF_NT_CASE(nt::F_BIAS | nt::F_R1)
            SGF_NT_CASE(nt::F_BIAS | nt::F_R1 | nt::F_ACCUM)
            SGF_NT_CASE(nt::F_GENERIC)
            default: break;
        }
        if (launched) break;
        feat = nt::F_GENERIC;     // no instantiation for this feature set
    }
#undef SGF_NT_CASE
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

// node slices per 128-feature block of A: one wave of CTAs over all blocks
static inline int tn_splits(int64_t kb_total, int m_blocks) {
    const int64_t cap = num_sms() / m_blocks > 0 ? num_sms() / m_blocks : 1;
    return (int)(kb_total < cap ? (kb_total < 1 ? 1 : kb_total) : cap);
}

extern "C" int sgf_gemm_tn_ws_bytes(int32_t m, int32_t n, int64_t rows, size_t* bytes) {
    if (!bytes || m <= 0 || m > 256 || n <= 0 || n > 256 || rows < 0) return SGF_ERR_ARG;
    const int m_blocks = (m + 127) / 128, un = (n + 15) / 16 * 16;
    const int64_t kb_total = (rows + tn::BKN - 1) / tn::BKN;
    *bytes = (size_t)tn_splits(kb_total, m_blocks) * un * m_blocks * 128 * sizeof(float);
    return SGF_OK;
}

extern "C" int sgf_gemm_tn(const sgf_gemm_tn_args* a, void* stream) {
    if (!a || a->m <= 0 || a->m > 256 || a->n <= 0 || a->n > 256 || a->rows < 0 || !a->out || !a->ws) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    tn::Params p;
    memset(&p, 0, sizeof(p));
    p.rows = a->rows; p.m = a->m; p.n = a->n;
    const int m_blocks = (a->m + 127) / 128;
    p.mp = m_blocks * 128;
    p.un = (a->n + 15) / 16 * 16;
    p.n_chunks = (p.un + 63) / 64;
    p.kb_total = (a->rows + tn::BKN - 1) / tn::BKN;
    p.ws = (float*)a->ws;
    if (a->n_pairs < 0 || a->n_pairs > SGF_TN_MAX_PAIRS) return SGF_ERR_ARG;
    p.n_pairs = a->n_pairs > 0 ? a->n_pairs : 1;
    int64_t a_span = a->m, b_span = a->n;      // columns the tensor maps must cover
    for (int i = 0; i < p.n_pairs; ++i) {
        p.a_off[i] = a->n_pairs > 0 ? a->a_off[i] : 0;
        p.b_off[i] = a->n_pairs > 0 ? a->b_off[i] : 0;
        if (p.a_off[i] < 0 || p.b_off[i] < 0 || p.a_off[i] % 64 || p.b_off[i] % 64) return SGF_ERR_ARG;
        if (p.a_off[i] + a->m > a_span) a_span = p.a_off[i] + a->m;
        if (p.b_off[i] + a->n > b_span) b_span = p.b_off[i] + a->n;
    }
    const int mp = p.mp;
    int grid = 0;
    if (a->rows > 0) {
        size_t need = 0;
        sgf_gemm_tn_ws_bytes(a->m, a->n, a->rows, &need);
        if (a->ws_bytes < need) return SGF_ERR_ARG;
        tn::Tmaps tm;
        memset(&tm, 0, sizeof(tm));
        int rc;
        if ((rc = make_tmap_bf16(&tm.a, a->a, a->rows, a_span, a->lda, tn::BKN))) return rc;
        if ((rc = make_tmap_bf16(&tm.b, a->b, a->rows, b_span, a->ldb, tn::BKN))) return rc;
        static bool attr_set = false;
        if (!attr_set) {
            SGF_CUDA_TRY(cudaFuncSetAttribute(tn::gemm_tn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tn::SMEM_BYTES));
            attr_set = true;
        }
        grid = tn_splits(p.kb_total, m_blocks);
        tn::gemm_tn_kernel<<<dim3(m_blocks, grid), tn::THREADS, tn::SMEM_BYTES, st>>>(tm, p);
        SGF_LAUNCH_CHECK(); count_launch();
    }
    int64_t total = (int64_t)a->n * mp;
    int rgrid = (int)((total + 255) / 256);
    tn::tn_reduce_kernel<<<rgrid, 256, 0, st>>>(p.ws, grid, mp, p.un, a->m, a->n, a->alpha, a->alpha_dev, a->beta, a->out, a->ldo,
                                                a->transpose_out);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}


static int gram_geometry(int h, int planes, int64_t rows, gramk::Params& p) {
    if (h <= 0 || h > 256 || (planes != 1 && planes != 3) || rows < 0) return SGF_ERR_ARG;
    memset(&p, 0, sizeof(p));
    p.rows = rows; p.h = h;
    p.chunks = (h + 63) / 64;
    p.m_blocks = h > 128 ? 2 : 1;
    p.un = (h + 15) / 16 * 16;
    p.mp = p.m_blocks * 128;
    p.n_planes = planes;
    p.kb_total = (rows + gramk::BKN - 1) / gramk::BKN;
    p.stages = gramk::SMEM_BUDGET / (planes * p.chunks * gramk::CHUNK_BYTES);
    if (p.stages > gramk::MAX_STAGES) p.stages = gramk::MAX_STAGES;
    if (p.stages < 2) return SGF_ERR_UNSUPPORTED;
    return SGF_OK;
}

extern "C" int sgf_gram_ws_bytes(int32_t h, int32_t planes, int64_t rows, size_t* bytes) {
    gramk::Params p;
    int rc = gram_geometry(h, planes, rows, p);
    if (rc || !bytes) return rc ? rc : SGF_ERR_ARG;
    *bytes = (size_t)tn_splits(p.kb_total, p.m_blocks) * (p.un + 1) * p.mp * sizeof(float);
    return SGF_OK;
}

extern "C" int sgf_gram(const void* x, int64_t ldx, int64_t rows, int32_t h, int32_t planes, int64_t plane_ld, float* G, int64_t ldg,
                        float* s, void* ws, size_t ws_bytes, void* stream) {
    gramk::Params p;
    int rc = gram_geometry(h, planes, rows, p);
    if (rc) return rc;
    if (!x || !G || !s || !ws || ldg < h || (planes == 3 && (plane_ld < h || plane_ld % 64 != 0))) return SGF_ERR_ARG;
    size_t need = 0;
    sgf_gram_ws_bytes(h, planes, rows, &need);
    if (ws_bytes < need) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    p.ws = (float*)ws;
    for (int i = 0; i < planes; ++i) p.plane_off[i] = (int)(i * plane_ld);
    if (planes == 1) {
        p.n_pairs = 1;
    } else {      // bf16x3: the six partial products, smallest terms first (kernels._PAIRS3)
        static const int PA[6] = {0, 2, 1, 0, 1, 0}, PB[6] = {2, 0, 1, 1, 0, 0};
        p.n_pairs = 6;
        for (int i = 0; i < 6; ++i) { p.pa[i] = PA[i]; p.pb[i] = PB[i]; }
    }
    const int grid = tn_splits(p.kb_total, p.m_blocks);
    if (rows > 0) {
        CUtensorMap tm;
        memset(&tm, 0, sizeof(tm));
        const int64_t span = planes == 1 ? h : 2 * plane_ld + h;
        if ((rc = make_tmap_bf16(&tm, x, rows, span, ldx, gramk::BKN))) return rc;
        const int smem_bytes = p.stages * planes * p.chunks * gramk::CHUNK_BYTES + gramk::ONES_BYTES + gramk::BAR_BYTES + 1024;
        static int attr_set = 0;
        if (attr_set < smem_bytes) {
            SGF_CUDA_TRY(cudaFuncSetAttribute(gramk::gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
            attr_set = 227 * 1024;
        }
        gramk::gram_kernel<<<dim3(p.m_blocks, grid), gramk::THREADS, smem_bytes, st>>>(tm, p);
        SGF_LAUNCH_CHECK(); count_launch();
    } else {
        SGF_CUDA_TRY(cudaMemsetAsync(ws, 0, need, st));
    }
    gramk::gram_reduce_kernel<<<(h * h + h + 255) / 256, 256, 0, st>>>(p.ws, grid, p.un, p.mp, h, G, ldg, s);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}
