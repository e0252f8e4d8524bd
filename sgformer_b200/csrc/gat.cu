// K12 — GAT edge softmax over the CSR (replaces PyG GATConv's propagate: per-edge logits, torch_scatter softmax over the in-edges
// of every target, attention dropout, weighted scatter-add; medium/models.py:116-155 with PyG's GATConv defaults).
//
// Conventions: the CSR rows are edge targets with sorted source columns (sgf_csr_build, self_loop_mode 1 = remove_self_loops +
// one self loop per node); xp = x W^T is [N, H*C] (head h = columns [hC, hC+C)); a_src, a_dst, lse, r are fp32 [N, H];
// da_src, da_dst are fp32 [H, N] (head-major, so that a head's column feeds sgf_colstats as its row weight).
//
//   e_ij = leaky_relu(a_src[j] + a_dst[i], 0.2),   alpha_ij = exp(e_ij - lse_i),   lse_i = log sum_j exp(e_ij)   (per head)
//   y_i = sum_j alpha_ij d_ij xp_j      (d_ij = attention-dropout factor: 0 or 1/(1-p))
//   out_i = concat_h y_i + bias  |  mean_h y_i + bias
//
// Geometry: one warp per CSR row; a feature row of H*C elements is cut into 16-byte chunks, lpr lanes cover one gathered row
// (each lane owns chunks sub, sub+lpr, ...: CPL of them) and a warp gathers 32/lpr neighbours at once (as spmm_rows_kernel).
// Per-head dot products are reduced over the lpr lanes of a group with xor shuffles; per-head sums over the groups at row end.
// Every sum runs in a fixed order, so a launch is bit-identical run to run (no float atomics).
//
// Attention dropout is a counter-based hash of (seed + epoch, target, source, duplicate rank, head).  The duplicate rank (0 for the
// first of several identical edges j -> i, 1 for the next, ...) is the entry's position within its run of equal columns; runs of
// (i, j) in row i of the CSR and of (j, i) in row j of the transposed CSR have the same length, so both traversals draw the same
// mask for the same edge.
#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

namespace sgf {

constexpr int kGatBlock = 256;
constexpr int kGatMaxH = SGF_GAT_MAX_HEADS;
constexpr int kGatUnroll = 2;
constexpr float kGatSlope = 0.2f;

__device__ __forceinline__ uint64_t gat_mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
    x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
    x ^= x >> 33;
    return x;
}

// attention-dropout factor of edge src -> dst (duplicate rank `rank`), head h
__device__ __forceinline__ float gat_keep(uint64_t seed, int64_t dst, int64_t src, int rank, int h, uint32_t thr16, float inv_keep) {
    if (thr16 == 0u) return 1.f;
    const uint64_t key = ((uint64_t)dst << 32) | (uint64_t)(uint32_t)src;
    const uint64_t x = gat_mix64(seed + key * 0x9E3779B97F4A7C15ULL + (((uint64_t)rank << 8) | (uint64_t)h) * 0xD1B54A32D192ED03ULL);
    return ((uint32_t)x & 0xFFFFu) >= thr16 ? inv_keep : 0.f;
}

__device__ __forceinline__ uint64_t gat_seed(uint64_t base, const uint64_t* epoch) {
    return epoch ? base + (*epoch) * 0xD1B54A32D192ED03ULL : base;
}

__device__ __forceinline__ float lrelu(float v) { return v > 0.f ? v : kGatSlope * v; }
__device__ __forceinline__ float lrelu_grad(float v) { return v > 0.f ? 1.f : kGatSlope; }

// Column ids of entries [base, base+32) of a row (-1 past its end) and each entry's duplicate rank; (run_val, run_cnt) carry the
// run of equal columns that ends the previous batch.
__device__ __forceinline__ void gat_batch(const int32_t* __restrict__ col, int64_t base, int64_t e, int lane, int& idx, int& rank,
                                          int& cnt, int& run_val, int& run_cnt) {
    cnt = (int)((e - base) < 32 ? (e - base) : 32);
    idx = lane < cnt ? ldg_nc_na_s32(col + base + lane) : -1;
    const unsigned same = __match_any_sync(0xffffffffu, idx);
    rank = __popc(same & ((1u << lane) - 1u));
    if (idx >= 0 && idx == run_val) rank += run_cnt;
    const int last = __shfl_sync(0xffffffffu, idx, cnt - 1);
    const int last_n = __popc(__shfl_sync(0xffffffffu, same, cnt - 1));
    run_cnt = last == run_val ? run_cnt + last_n : last_n;
    run_val = last;
}

template <typename T, int CPL>
struct GatLanes {
    static constexpr int VN = Vec16<T>::N;
    int lane, lpr_log2, lpr, groups, grp, sub;
    int coff[CPL];      // element offset of the chunk in the [H*C] row
    int hd[CPL];        // head of the chunk
    bool cval[CPL];
    __device__ __forceinline__ GatLanes(int chunks, int lpr_log2_, int C) {
        lane = threadIdx.x & 31;
        lpr_log2 = lpr_log2_;
        lpr = 1 << lpr_log2;
        groups = 32 >> lpr_log2;
        grp = lane >> lpr_log2;
        sub = lane & (lpr - 1);
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
            const int ch = sub + c * lpr;
            cval[c] = ch < chunks;
            coff[c] = ch * VN;
            hd[c] = cval[c] ? coff[c] / C : 0;
        }
    }
    // offset of chunk c in a row of the gradient / output: the same chunk (concat) or its position within the head (mean)
    __device__ __forceinline__ int goff(int c, int C, bool mean) const { return mean ? coff[c] - hd[c] * C : coff[c]; }
    // per-head sums of part[c] over the chunks of this lane group (every lane of the group receives them)
    __device__ __forceinline__ void head_dots(const float (&part)[CPL], float (&hv)[kGatMaxH]) const {
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) {
            float v = 0.f;
#pragma unroll
            for (int c = 0; c < CPL; ++c) v += (cval[c] && hd[c] == h) ? part[c] : 0.f;
            hv[h] = v;
        }
        for (int o = 1; o < lpr; o <<= 1) {
#pragma unroll
            for (int h = 0; h < kGatMaxH; ++h) hv[h] += __shfl_xor_sync(0xffffffffu, hv[h], o);
        }
    }
    __device__ __forceinline__ float pick(const float (&v)[kGatMaxH], int c) const {
        float r = 0.f;
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) r = hd[c] == h ? v[h] : r;
        return r;
    }
};

template <typename T, int CPL>
__device__ __forceinline__ void load_chunks(const T* __restrict__ row, const GatLanes<T, CPL>& L, bool valid, const int* offs,
                                            float (&f)[CPL][Vec16<T>::N]) {
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
        const uint4 u = (valid && L.cval[c]) ? ldg_nc_na(row + offs[c]) : make_uint4(0u, 0u, 0u, 0u);
        Vec16<T>::unpack(u, f[c]);
    }
}

// ---- logits: a_src[n,h] = <xp[n,h,:], att_src[h,:]>, a_dst likewise (one lane group per row) -------------------------------------
template <typename T, int CPL>
__global__ void __launch_bounds__(kGatBlock) gat_logits_kernel(const T* __restrict__ xp, int64_t ldx, int64_t n, int H, int C, int chunks,
                                                               int lpr_log2, const float* __restrict__ att_src,
                                                               const float* __restrict__ att_dst, float* __restrict__ a_src,
                                                               float* __restrict__ a_dst) {
    constexpr int VN = Vec16<T>::N;
    GatLanes<T, CPL> L(chunks, lpr_log2, C);
    float ws[CPL][VN], wd[CPL][VN];
#pragma unroll
    for (int c = 0; c < CPL; ++c)
#pragma unroll
        for (int t = 0; t < VN; ++t) {
            ws[c][t] = L.cval[c] ? att_src[L.coff[c] + t] : 0.f;
            wd[c][t] = L.cval[c] ? att_dst[L.coff[c] + t] : 0.f;
        }
    const int64_t warp0 = ((int64_t)blockIdx.x * kGatBlock + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * kGatBlock) >> 5;
    for (int64_t base = warp0 * L.groups; base < n; base += nwarps * L.groups) {
        const int64_t r = base + L.grp;
        const bool valid = r < n;
        float x[CPL][VN];
        load_chunks<T, CPL>(xp + (valid ? r : 0) * ldx, L, valid, L.coff, x);
        float ps[CPL], pd[CPL];
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
            ps[c] = 0.f; pd[c] = 0.f;
#pragma unroll
            for (int t = 0; t < VN; ++t) { ps[c] += x[c][t] * ws[c][t]; pd[c] += x[c][t] * wd[c][t]; }
        }
        float hs[kGatMaxH], hdst[kGatMaxH];
        L.head_dots(ps, hs);
        L.head_dots(pd, hdst);
        if (valid && L.sub == 0) {
#pragma unroll
            for (int h = 0; h < kGatMaxH; ++h)
                if (h < H) { a_src[r * H + h] = hs[h]; a_dst[r * H + h] = hdst[h]; }
        }
    }
}

// ---- forward ---------------------------------------------------------------------------------------------------------------------
template <typename T, int CPL>
__global__ void __launch_bounds__(kGatBlock) gat_fwd_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                            const T* __restrict__ xp, int64_t ldx, const float* __restrict__ a_src,
                                                            const float* __restrict__ a_dst, int64_t n_rows, int H, int C, int chunks,
                                                            int lpr_log2, int mean, const float* __restrict__ bias, T* __restrict__ out,
                                                            int64_t ldo, float* __restrict__ lse_out, uint32_t thr16, float inv_keep,
                                                            uint64_t seed_base, const uint64_t* __restrict__ epoch) {
    constexpr int VN = Vec16<T>::N;
    extern __shared__ float s_row[];                 // one finished fp32 row of H*C per warp
    float* srow = s_row + (threadIdx.x >> 5) * (H * C);
    const uint64_t seed = gat_seed(seed_base, epoch);
    GatLanes<T, CPL> L(chunks, lpr_log2, C);
    const int lane = L.lane;
    const int64_t warp0 = ((int64_t)blockIdx.x * kGatBlock + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * kGatBlock) >> 5;
    for (int64_t i = warp0; i < n_rows; i += nwarps) {
        const int64_t s = rowptr[i], e = rowptr[i + 1];
        float ad[kGatMaxH], mx[kGatMaxH], sm[kGatMaxH];
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) { ad[h] = h < H ? a_dst[i * H + h] : 0.f; mx[h] = -INFINITY; sm[h] = 0.f; }
        // 1) per-head online max / sum of exp over the row's logits (one edge per lane)
        for (int64_t b = s; b < e; b += 32) {
            const int64_t p = b + lane;
            if (p < e) {
                const int64_t j = col[p];
#pragma unroll
                for (int h = 0; h < kGatMaxH; ++h) {
                    if (h >= H) break;
                    const float v = lrelu(a_src[j * H + h] + ad[h]);
                    if (v > mx[h]) { sm[h] = sm[h] * expf(mx[h] - v) + 1.f; mx[h] = v; }
                    else sm[h] += expf(v - mx[h]);
                }
            }
        }
        float lse[kGatMaxH];
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) {
            float m = mx[h];
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float t = mx[h] == -INFINITY ? 0.f : sm[h] * expf(mx[h] - m);
            t = warp_sum(t);
            lse[h] = m + logf(t);
        }
        if (lane == 0) {
#pragma unroll
            for (int h = 0; h < kGatMaxH; ++h)
                if (h < H) lse_out[i * H + h] = lse[h];
        }
        float adc[CPL], lsec[CPL];
#pragma unroll
        for (int c = 0; c < CPL; ++c) { adc[c] = L.pick(ad, c); lsec[c] = L.pick(lse, c); }
        // 2) gather: y = sum_j alpha_ij d_ij xp_j
        float acc[CPL][VN];
#pragma unroll
        for (int c = 0; c < CPL; ++c)
#pragma unroll
            for (int t = 0; t < VN; ++t) acc[c][t] = 0.f;
        int run_val = -2, run_cnt = 0;
        for (int64_t b = s; b < e; b += 32) {
            int idx, rank, cnt;
            gat_batch(col, b, e, lane, idx, rank, cnt, run_val, run_cnt);
            for (int j0 = 0; j0 < cnt; j0 += L.groups * kGatUnroll) {
                int src[kGatUnroll], rk[kGatUnroll];
                float x[kGatUnroll][CPL][VN];
#pragma unroll
                for (int u = 0; u < kGatUnroll; ++u) {
                    const int jj = j0 + u * L.groups + L.grp;
                    const int t0 = __shfl_sync(0xffffffffu, idx, jj & 31), t1 = __shfl_sync(0xffffffffu, rank, jj & 31);
                    src[u] = jj < cnt ? t0 : -1;
                    rk[u] = t1;
                    load_chunks<T, CPL>(xp + (int64_t)(src[u] < 0 ? 0 : src[u]) * ldx, L, src[u] >= 0, L.coff, x[u]);
                }
#pragma unroll
                for (int u = 0; u < kGatUnroll; ++u) {
                    if (src[u] < 0) continue;
#pragma unroll
                    for (int c = 0; c < CPL; ++c) {
                        if (!L.cval[c]) continue;
                        const float w = expf(lrelu(a_src[(int64_t)src[u] * H + L.hd[c]] + adc[c]) - lsec[c]) *
                                        gat_keep(seed, i, src[u], rk[u], L.hd[c], thr16, inv_keep);
#pragma unroll
                        for (int t = 0; t < VN; ++t) acc[c][t] += w * x[u][c][t];
                    }
                }
            }
        }
        for (int o = L.lpr; o < 32; o <<= 1) {
#pragma unroll
            for (int c = 0; c < CPL; ++c)
#pragma unroll
                for (int t = 0; t < VN; ++t) acc[c][t] += __shfl_xor_sync(0xffffffffu, acc[c][t], o);
        }
        if (L.grp == 0) {
#pragma unroll
            for (int c = 0; c < CPL; ++c)
                if (L.cval[c]) {
#pragma unroll
                    for (int t = 0; t < VN; ++t) srow[L.coff[c] + t] = acc[c][t];
                }
        }
        __syncwarp();
        T* orow = out + i * ldo;
        if (mean) {
            const float inv_h = 1.f / (float)H;
            for (int k = lane; k < C; k += 32) {
                float v = 0.f;
                for (int h = 0; h < H; ++h) v += srow[h * C + k];
                orow[k] = from_f32<T>(v * inv_h + (bias ? bias[k] : 0.f));
            }
        } else {
            for (int k = lane; k < H * C; k += 32) orow[k] = from_f32<T>(srow[k] + (bias ? bias[k] : 0.f));
        }
        __syncwarp();
    }
}

// ---- backward pass 1 (forward CSR, row = target i): r_i = sum_j alpha_ij dalpha_ij,  da_dst_i = sum_j de_ij lrelu'_ij ------------
// with dalpha_ij = d_ij <g_i, xp_j> and de_ij = alpha_ij (dalpha_ij - r_i):  da_dst = A - r B,  A = sum alpha dalpha lrelu',
// B = sum alpha lrelu'.
template <typename T, int CPL>
__global__ void __launch_bounds__(kGatBlock) gat_bwd_dst_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                                const T* __restrict__ xp, int64_t ldx, const float* __restrict__ a_src,
                                                                const float* __restrict__ a_dst, const float* __restrict__ lse,
                                                                const T* __restrict__ g, int64_t ldg, int64_t n_rows, int H, int C,
                                                                int chunks, int lpr_log2, int mean, float* __restrict__ r_out,
                                                                float* __restrict__ da_dst, uint32_t thr16, float inv_keep,
                                                                uint64_t seed_base, const uint64_t* __restrict__ epoch) {
    constexpr int VN = Vec16<T>::N;
    const uint64_t seed = gat_seed(seed_base, epoch);
    GatLanes<T, CPL> L(chunks, lpr_log2, C);
    const int lane = L.lane;
    const float gsc = mean ? 1.f / (float)H : 1.f;
    int goffs[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) goffs[c] = L.goff(c, C, mean);
    const int64_t warp0 = ((int64_t)blockIdx.x * kGatBlock + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * kGatBlock) >> 5;
    for (int64_t i = warp0; i < n_rows; i += nwarps) {
        const int64_t s = rowptr[i], e = rowptr[i + 1];
        float gi[CPL][VN];
        load_chunks<T, CPL>(g + i * ldg, L, true, goffs, gi);
        float ad[kGatMaxH], ls[kGatMaxH], R[kGatMaxH], A[kGatMaxH], B[kGatMaxH];
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) {
            ad[h] = h < H ? a_dst[i * H + h] : 0.f;
            ls[h] = h < H ? lse[i * H + h] : 0.f;
            R[h] = A[h] = B[h] = 0.f;
        }
        int run_val = -2, run_cnt = 0;
        for (int64_t b = s; b < e; b += 32) {
            int idx, rank, cnt;
            gat_batch(col, b, e, lane, idx, rank, cnt, run_val, run_cnt);
            for (int j0 = 0; j0 < cnt; j0 += L.groups) {
                const int jj = j0 + L.grp;
                const int t0 = __shfl_sync(0xffffffffu, idx, jj & 31), rk = __shfl_sync(0xffffffffu, rank, jj & 31);
                const int src = jj < cnt ? t0 : -1;
                float x[CPL][VN];
                load_chunks<T, CPL>(xp + (int64_t)(src < 0 ? 0 : src) * ldx, L, src >= 0, L.coff, x);
                float part[CPL];
#pragma unroll
                for (int c = 0; c < CPL; ++c) {
                    part[c] = 0.f;
#pragma unroll
                    for (int t = 0; t < VN; ++t) part[c] += gi[c][t] * x[c][t];
                }
                float dot[kGatMaxH];
                L.head_dots(part, dot);
                if (src >= 0) {
#pragma unroll
                    for (int h = 0; h < kGatMaxH; ++h) {
                        if (h >= H) break;
                        const float pre = a_src[(int64_t)src * H + h] + ad[h];
                        const float lg = lrelu_grad(pre);
                        const float al = expf(lrelu(pre) - ls[h]);
                        const float da = gat_keep(seed, i, src, rk, h, thr16, inv_keep) * dot[h] * gsc;
                        R[h] += al * da;
                        A[h] += al * da * lg;
                        B[h] += al * lg;
                    }
                }
            }
        }
        // the lanes of a group hold identical copies: sum one copy per group
        if (L.sub != 0) {
#pragma unroll
            for (int h = 0; h < kGatMaxH; ++h) R[h] = A[h] = B[h] = 0.f;
        }
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) { R[h] = warp_sum(R[h]); A[h] = warp_sum(A[h]); B[h] = warp_sum(B[h]); }
        if (lane == 0) {
#pragma unroll
            for (int h = 0; h < kGatMaxH; ++h)
                if (h < H) { r_out[i * H + h] = R[h]; da_dst[(int64_t)h * n_rows + i] = A[h] - R[h] * B[h]; }
        }
    }
}

// ---- backward pass 2 (transposed CSR, row = source j): dxp_j = sum_i alpha_ij d_ij g_i + da_src_j att_src + da_dst_j att_dst,
// da_src_j = sum_i de_ij lrelu'_ij --------------------------------------------------------------------------------------------------
template <typename T, int CPL>
__global__ void __launch_bounds__(kGatBlock) gat_bwd_src_kernel(const int64_t* __restrict__ rowptr_t, const int32_t* __restrict__ col_t,
                                                                const T* __restrict__ xp, int64_t ldx, const float* __restrict__ a_src,
                                                                const float* __restrict__ a_dst, const float* __restrict__ lse,
                                                                const float* __restrict__ r_in, const T* __restrict__ g, int64_t ldg,
                                                                const float* __restrict__ da_dst, const float* __restrict__ att_src,
                                                                const float* __restrict__ att_dst, int64_t n_rows, int H, int C,
                                                                int chunks, int lpr_log2, int mean, T* __restrict__ dxp, int64_t ldd,
                                                                float* __restrict__ da_src, uint32_t thr16, float inv_keep,
                                                                uint64_t seed_base, const uint64_t* __restrict__ epoch) {
    constexpr int VN = Vec16<T>::N;
    const uint64_t seed = gat_seed(seed_base, epoch);
    GatLanes<T, CPL> L(chunks, lpr_log2, C);
    const int lane = L.lane;
    const float gsc = mean ? 1.f / (float)H : 1.f;
    int goffs[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) goffs[c] = L.goff(c, C, mean);
    const int64_t warp0 = ((int64_t)blockIdx.x * kGatBlock + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * kGatBlock) >> 5;
    for (int64_t j = warp0; j < n_rows; j += nwarps) {
        const int64_t s = rowptr_t[j], e = rowptr_t[j + 1];
        float xj[CPL][VN];
        load_chunks<T, CPL>(xp + j * ldx, L, true, L.coff, xj);
        float as[kGatMaxH], S[kGatMaxH];
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) { as[h] = h < H ? a_src[j * H + h] : 0.f; S[h] = 0.f; }
        float acc[CPL][VN];
#pragma unroll
        for (int c = 0; c < CPL; ++c)
#pragma unroll
            for (int t = 0; t < VN; ++t) acc[c][t] = 0.f;
        int run_val = -2, run_cnt = 0;
        for (int64_t b = s; b < e; b += 32) {
            int idx, rank, cnt;
            gat_batch(col_t, b, e, lane, idx, rank, cnt, run_val, run_cnt);
            for (int j0 = 0; j0 < cnt; j0 += L.groups) {
                const int jj = j0 + L.grp;
                const int t0 = __shfl_sync(0xffffffffu, idx, jj & 31), rk = __shfl_sync(0xffffffffu, rank, jj & 31);
                const int dst = jj < cnt ? t0 : -1;
                float gv[CPL][VN];
                load_chunks<T, CPL>(g + (int64_t)(dst < 0 ? 0 : dst) * ldg, L, dst >= 0, goffs, gv);
                float part[CPL];
#pragma unroll
                for (int c = 0; c < CPL; ++c) {
                    part[c] = 0.f;
#pragma unroll
                    for (int t = 0; t < VN; ++t) part[c] += gv[c][t] * xj[c][t];
                }
                float dot[kGatMaxH], coef[kGatMaxH];
                L.head_dots(part, dot);
#pragma unroll
                for (int h = 0; h < kGatMaxH; ++h) {
                    coef[h] = 0.f;
                    if (dst < 0 || h >= H) continue;
                    const int64_t o = (int64_t)dst * H + h;
                    const float pre = as[h] + a_dst[o];
                    const float al = expf(lrelu(pre) - lse[o]);
                    const float kp = gat_keep(seed, dst, j, rk, h, thr16, inv_keep);
                    const float de = al * (kp * dot[h] * gsc - r_in[o]);
                    S[h] += de * lrelu_grad(pre);
                    coef[h] = al * kp * gsc;
                }
#pragma unroll
                for (int c = 0; c < CPL; ++c) {
                    const float w = L.pick(coef, c);
#pragma unroll
                    for (int t = 0; t < VN; ++t) acc[c][t] += w * gv[c][t];
                }
            }
        }
        if (L.sub != 0) {
#pragma unroll
            for (int h = 0; h < kGatMaxH; ++h) S[h] = 0.f;
        }
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) S[h] = warp_sum(S[h]);
        for (int o = L.lpr; o < 32; o <<= 1) {
#pragma unroll
            for (int c = 0; c < CPL; ++c)
#pragma unroll
                for (int t = 0; t < VN; ++t) acc[c][t] += __shfl_xor_sync(0xffffffffu, acc[c][t], o);
        }
        if (L.grp == 0) {
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                if (!L.cval[c]) continue;
                const int h = L.hd[c];
                const float ss = L.pick(S, c), sd = da_dst[(int64_t)h * n_rows + j];
                float f[VN];
#pragma unroll
                for (int t = 0; t < VN; ++t) f[t] = acc[c][t] + ss * att_src[L.coff[c] + t] + sd * att_dst[L.coff[c] + t];
                stg_na(dxp + j * ldd + L.coff[c], Vec16<T>::pack(f));
            }
        }
        if (lane == 0) {
#pragma unroll
            for (int h = 0; h < kGatMaxH; ++h)
                if (h < H) da_src[(int64_t)h * n_rows + j] = S[h];
        }
    }
}

// ---- input dropout of a dense fp32 matrix (GAT's F.dropout of the node features): one hash per element ----------------------------
__global__ void dense_dropout_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, uint32_t thr16,
                                     float inv_keep, uint64_t seed_base, const uint64_t* __restrict__ epoch, float* __restrict__ y,
                                     int64_t ldy) {
    const uint64_t seed = gat_seed(seed_base, epoch);
    const int64_t total = rows * cols;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += stride) {
        const int64_t r = k / cols, c = k - r * cols;
        const uint64_t h = gat_mix64(seed + (uint64_t)k * 0x9E3779B97F4A7C15ULL);
        y[r * ldy + c] = ((uint32_t)h & 0xFFFFu) >= thr16 ? x[r * ldx + c] * inv_keep : 0.f;
    }
}

struct GatGeom {
    int chunks, lpr_log2, cpl;
};
static bool gat_geom(int dtype, int H, int C, GatGeom& g) {
    const int vn = dtype == SGF_BF16 ? 8 : 4;
    if ((dtype != SGF_F32 && dtype != SGF_BF16) || H < 1 || H > kGatMaxH || C <= 0 || C % vn != 0) return false;
    g.chunks = H * C / vn;
    g.lpr_log2 = 0;
    while ((1 << g.lpr_log2) < g.chunks && g.lpr_log2 < 5) ++g.lpr_log2;
    g.cpl = (g.chunks + (1 << g.lpr_log2) - 1) >> g.lpr_log2;
    return g.cpl <= 4;
}
static int gat_grid(int64_t warps) {
    int64_t blocks = (warps * 32 + kGatBlock - 1) / kGatBlock;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    return (int)(blocks < 1 ? 1 : blocks);
}
static bool ld_ok16(int dtype, int64_t ld) { return ld > 0 && (ld * (dtype == SGF_BF16 ? 2 : 4)) % 16 == 0; }
static bool al16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

#define SGF_GAT_DISPATCH(dtype, cpl, LAUNCH)                                      \
    do {                                                                          \
        if (dtype == SGF_F32) {                                                   \
            using T = float;                                                      \
            switch (cpl) {                                                        \
                case 1: { constexpr int CPL = 1; LAUNCH; } break;                 \
                case 2: { constexpr int CPL = 2; LAUNCH; } break;                 \
                case 3: { constexpr int CPL = 3; LAUNCH; } break;                 \
                default: { constexpr int CPL = 4; LAUNCH; } break;                \
            }                                                                     \
        } else {                                                                  \
            using T = __nv_bfloat16;                                              \
            switch (cpl) {                                                        \
                case 1: { constexpr int CPL = 1; LAUNCH; } break;                 \
                case 2: { constexpr int CPL = 2; LAUNCH; } break;                 \
                case 3: { constexpr int CPL = 3; LAUNCH; } break;                 \
                default: { constexpr int CPL = 4; LAUNCH; } break;                \
            }                                                                     \
        }                                                                         \
    } while (0)

static bool drop_args(float p, uint32_t& thr16, float& inv_keep) {
    if (!(p >= 0.f && p < 1.f)) return false;
    thr16 = dropout_thr16(p);
    inv_keep = dropout_inv_keep(thr16);
    return true;
}

}  // namespace sgf

using namespace sgf;

extern "C" int sgf_gat_logits(const void* xp, int64_t ldx, int64_t n, int heads, int c, int dtype, const float* att_src,
                              const float* att_dst, float* a_src, float* a_dst, void* stream) {
    GatGeom g;
    if (!gat_geom(dtype, heads, c, g) || n < 0 || !ld_ok16(dtype, ldx) || !al16(xp) || !att_src || !att_dst || !a_src || !a_dst)
        return SGF_ERR_ARG;
    if (n == 0) return SGF_OK;
    const int groups = 32 >> g.lpr_log2;
    SGF_GAT_DISPATCH(dtype, g.cpl, (gat_logits_kernel<T, CPL><<<gat_grid((n + groups - 1) / groups), kGatBlock, 0, (cudaStream_t)stream>>>(
                                       (const T*)xp, ldx, n, heads, c, g.chunks, g.lpr_log2, att_src, att_dst, a_src, a_dst)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_gat_fwd(const int64_t* rowptr, const int32_t* col, const void* xp, int64_t ldx, const float* a_src,
                           const float* a_dst, int64_t n, int heads, int c, int dtype, int mean, const float* bias, void* out,
                           int64_t ldo, float* lse, float p, uint64_t seed, void* stream) {
    GatGeom g;
    uint32_t thr16; float inv_keep;
    if (!gat_geom(dtype, heads, c, g) || n < 0 || !ld_ok16(dtype, ldx) || !al16(xp) || !drop_args(p, thr16, inv_keep) || !rowptr ||
        !a_src || !a_dst || !out || !lse || ldo < (mean ? c : (int64_t)heads * c))
        return SGF_ERR_ARG;
    if (n == 0) return SGF_OK;
    const size_t smem = (size_t)(kGatBlock / 32) * heads * c * sizeof(float);     // <= 32 KB (H*C <= 512 fp32 / 1024 bf16)
    const uint64_t* ep = dropout_epoch_word();
    SGF_GAT_DISPATCH(dtype, g.cpl, (gat_fwd_kernel<T, CPL><<<gat_grid(n), kGatBlock, smem, (cudaStream_t)stream>>>(
                                       rowptr, col, (const T*)xp, ldx, a_src, a_dst, n, heads, c, g.chunks, g.lpr_log2, mean, bias,
                                       (T*)out, ldo, lse, thr16, inv_keep, seed, ep)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_gat_bwd(const int64_t* rowptr, const int32_t* col, const int64_t* rowptr_t, const int32_t* col_t, const void* xp,
                           int64_t ldx, const float* a_src, const float* a_dst, const float* lse, const void* g, int64_t ldg,
                           const float* att_src, const float* att_dst, int64_t n, int heads, int c, int dtype, int mean, float p,
                           uint64_t seed, float* r_ws, float* da_src, float* da_dst, void* dxp, int64_t ldd, void* stream) {
    GatGeom gg;
    uint32_t thr16; float inv_keep;
    if (!gat_geom(dtype, heads, c, gg) || n < 0 || !ld_ok16(dtype, ldx) || !ld_ok16(dtype, ldg) || !ld_ok16(dtype, ldd) || !al16(xp) ||
        !al16(g) || !al16(dxp) || !drop_args(p, thr16, inv_keep) || !rowptr || !rowptr_t || !a_src || !a_dst || !lse || !att_src ||
        !att_dst || !r_ws || !da_src || !da_dst)
        return SGF_ERR_ARG;
    if (n == 0) return SGF_OK;
    const uint64_t* ep = dropout_epoch_word();
    cudaStream_t st = (cudaStream_t)stream;
    SGF_GAT_DISPATCH(dtype, gg.cpl, (gat_bwd_dst_kernel<T, CPL><<<gat_grid(n), kGatBlock, 0, st>>>(
                                        rowptr, col, (const T*)xp, ldx, a_src, a_dst, lse, (const T*)g, ldg, n, heads, c, gg.chunks,
                                        gg.lpr_log2, mean, r_ws, da_dst, thr16, inv_keep, seed, ep)));
    SGF_LAUNCH_CHECK(); count_launch();
    SGF_GAT_DISPATCH(dtype, gg.cpl, (gat_bwd_src_kernel<T, CPL><<<gat_grid(n), kGatBlock, 0, st>>>(
                                        rowptr_t, col_t, (const T*)xp, ldx, a_src, a_dst, lse, r_ws, (const T*)g, ldg, da_dst, att_src,
                                        att_dst, n, heads, c, gg.chunks, gg.lpr_log2, mean, (T*)dxp, ldd, da_src, thr16, inv_keep, seed,
                                        ep)));
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_dense_dropout(const float* x, int64_t ldx, int64_t rows, int64_t cols, float p, uint64_t seed, float* y, int64_t ldy,
                                 void* stream) {
    uint32_t thr16; float inv_keep;
    if (rows < 0 || cols < 0 || ldx < cols || ldy < cols || !drop_args(p, thr16, inv_keep) || (rows * cols > 0 && (!x || !y)))
        return SGF_ERR_ARG;
    if (rows * cols == 0) return SGF_OK;
    int64_t blocks = (rows * cols + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    dense_dropout_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, ldx, rows, cols, thr16, inv_keep, seed,
                                                                              dropout_epoch_word(), y, ldy);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}
