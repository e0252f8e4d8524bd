// Fused softmax attention of SGFormerSOFT (medium/ablation/oursSOFT.py:14-34) that never stores an N x N tile.
//
//   q~ = q/||q||_F,  k~ = k/||k||_F   (one Frobenius norm over all nodes and heads)
//   s[n,l,h] = q~[n,h].k~[l,h],  P = softmax over the HEAD axis h of s[n,l,:],  o[n,h] = sum_l P[n,l,h] v[l,h]
// (v[l,h] = v[l] when v is shared).  This is what the reference computes: its einsum "nhm,lhm->nlh" builds [N, L, H] scores and
// F.softmax(..., dim=-1) normalises over the last axis, the heads (oursSOFT.py:21-22).  With one head every weight is 1 and
// o[n] = sum_l v[l].
//
// The bound the kernels rely on: by Cauchy-Schwarz |q_nh . k_lh| <= ||q_nh|| ||k_lh|| <= ||q||_F ||k||_F, so |s| <= 1.  Hence
// exp(s) lies in [1/e, e] and the per-pair denominator sum_h exp(s[n,l,h]) in [H/e, H e]: no maximum is subtracted (torch's
// max subtraction differs from this only at rounding level).  The kernels work on the raw q, k with c = 1/(||q||_F ||k||_F)
// applied to the dot products (s = c q.k); ||q||^2, ||k||^2 are the fixed-order sums of the projection's column sums of squares.
//
// Structure (4 warps, 16 rows each, a CTA owns 64 resident rows with every head's q (or k) columns; the other side streams
// through shared memory in tiles of BS rows, double-buffered with cp.async; every product is an mma.sync m16n8k16 bf16
// tensor-core product with fp32 accumulation, 16 streamed rows at a time).  A CTA writes one head h; the softmax over heads
// needs every head's score of the same (n, l) pair, so each 16 x 16 block computes the scores of all H heads (H times the
// score work of a per-head softmax):
//   fwd      query tile x head x 128-column block of v_h:   P_h = E_h / sum_h' E_h' (E = exp(c S)),  o_h = sum_l P_h V_h
//   bwd_q    query tile x head x 128-column block of q_h:   dS_h = P_h (dP_h - sum_h' P_h' dP_h'),  dP = G V^T,  Aq_h = c dS_h K_h
//   bwd_kv   key tile x head x (128-column block of k_h | of v_h):  Ak_h = c dS_h^T Q_h,  dV_h = gs P_h^T G_h
//            (a shared v sums its heads' P_h^T G_h in head order inside one CTA: no float atomics anywhere)
//   norm     dq = gs (Aq - <q,Aq>/||q||^2 q),  dk = gs (Ak - <k,Ak>/||k||^2 k)  (the norm backward; <q,Aq> from per-CTA partials
//            that bwd_q / bwd_kv write, summed in a fixed order)
// G is the gradient of o (per head, or one [n, d] block shared by every head: the head mean's); gs (gscale) scales every output.
//
// Scaled mode (SCALED, args.scaled = 1): the scaled dot-product attention of SGFormerGAT (medium/ablation/oursGAT.py:31-44),
//   s[n,l,h] = c q[n,h].k[l,h] with a host constant c = args.scale (1/sqrt(dk)), the same softmax over the heads and the same o.
// Nothing bounds these scores (exp overflows fp32 once c q.k > 88), so each pair's exponents are taken relative to the pair's
// maximum over the heads.  The thread that holds a pair's score fragment holds that pair's score for every head, so the maximum
// needs no cross-thread reduction; it is kept online while the head loop runs: E_h' = exp(c (s_h' - mx)) against the running
// maximum mx, and when a head raises mx every term accumulated so far (E_h, den, and the backward's numerator) is rescaled by
// exp(c (mx_old - mx_new)).  A separate max pass would recompute every head's score tile (H more 16 x 16 mma blocks per block
// of pairs) to save one multiply per accumulated term; the online rescale costs one exp2f per head and pair, as the
// unscaled mode does.  Every exponent is <= 0 and the own head's or the maximum's term is 1, so den lies in [1, H].
// The backward recomputes the same maximum and the same dS_h; there is no norm backward: the sweeps write
//   dq_h = gs c dS_h K_h (bwd_q) and dk_h = gs c dS_h^T Q_h (bwd_kv) directly in the activation dtype, no <q,Aq> partials.
// dV is unchanged (v is always per head in this mode).  With one head P = 1 and dS = 0 exactly, as in the unscaled mode.
// Precision: bf16 activations use one bf16 plane; fp32 activations split every operand (and P, dS in registers) into bf16 hi/lo
// planes and accumulate hi.hi + hi.lo + lo.hi (the bf16x3 scheme of the GEMMs: fp32-accurate products).
#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

#include <type_traits>

namespace sgf {
namespace soft {

constexpr int kRows = 64;        // resident rows per CTA
constexpr int kThreads = 128;
constexpr int kOutCols = 128;    // output columns per CTA (accumulator: 16 n8 tiles)
constexpr float kLog2e = 1.4426950408889634f;

__host__ __device__ constexpr int ceil16(int x) { return (x + 15) & ~15; }
// shared-memory row stride in elements: padded width plus 16 bytes (shifts banks between rows)
template <typename T> __host__ __device__ constexpr int row_stride(int w) { return ceil16(w) + 16 / (int)sizeof(T); }

struct FragA { uint32_t h[4], l[4]; };
struct FragB { uint32_t h[2], l[2]; };

__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    hi = pack_bf16x2(x0, x1);
    float h0, h1;
    unpack_bf16x2(hi, h0, h1);
    lo = pack_bf16x2(x0 - h0, x1 - h1);
}
// (p[0], p[stride]) -> bf16x2 planes
__device__ __forceinline__ void ld_pair(const float* p, int stride, uint32_t& hi, uint32_t& lo) { split_pair(p[0], p[stride], hi, lo); }
__device__ __forceinline__ void ld_pair(const __nv_bfloat16* p, int stride, uint32_t& hi, uint32_t& lo) {
    const uint32_t a = *reinterpret_cast<const uint16_t*>(p), b = *reinterpret_cast<const uint16_t*>(p + stride);
    hi = a | (b << 16);
    lo = 0u;
}
__device__ __forceinline__ void ld_pair2(const float* p, uint32_t& hi, uint32_t& lo) {
    const float2 v = *reinterpret_cast<const float2*>(p);
    split_pair(v.x, v.y, hi, lo);
}
__device__ __forceinline__ void ld_pair2(const __nv_bfloat16* p, uint32_t& hi, uint32_t& lo) {
    hi = *reinterpret_cast<const uint32_t*>(p);
    lo = 0u;
}

__device__ __forceinline__ void mma1(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
template <bool SPLIT>
__device__ __forceinline__ void mma(float (&c)[4], const FragA& a, const FragB& b) {
    mma1(c, a.h, b.h);
    if (SPLIT) {
        mma1(c, a.h, b.l);
        mma1(c, a.l, b.h);
    }
}

// A fragment (16 x 16) of a row-major tile X: rows r0.., columns k0..
template <typename T>
__device__ __forceinline__ FragA ld_a(const T* X, int ld, int r0, int k0, int lane) {
    const int g = lane >> 2, c = lane & 3;
    const T* p = X + (r0 + g) * ld + k0 + 2 * c;
    FragA f;
    ld_pair2(p, f.h[0], f.l[0]);
    ld_pair2(p + 8 * ld, f.h[1], f.l[1]);
    ld_pair2(p + 8, f.h[2], f.l[2]);
    ld_pair2(p + 8 * ld + 8, f.h[3], f.l[3]);
    return f;
}
// B fragment (16 x 8) with B[k][n] = X[n0+n][k0+k] (contiguous along k)
template <typename T>
__device__ __forceinline__ FragB ld_b_n(const T* X, int ld, int n0, int k0, int lane) {
    const int g = lane >> 2, c = lane & 3;
    const T* p = X + (n0 + g) * ld + k0 + 2 * c;
    FragB f;
    ld_pair2(p, f.h[0], f.l[0]);
    ld_pair2(p + 8, f.h[1], f.l[1]);
    return f;
}
// B fragment (16 x 8) with B[k][n] = X[k0+k][n0+n] (strided along k)
template <typename T>
__device__ __forceinline__ FragB ld_b_k(const T* X, int ld, int k0, int n0, int lane) {
    const int g = lane >> 2, c = lane & 3;
    const T* p = X + (k0 + 2 * c) * ld + n0 + g;
    FragB f;
    ld_pair(p, ld, f.h[0], f.l[0]);
    ld_pair(p + 8 * ld, ld, f.h[1], f.l[1]);
    return f;
}
// A fragment from two 16 x 8 accumulator tiles (columns 0-7 and 8-15 of a 16 x 16 block)
__device__ __forceinline__ FragA a_from_acc(const float (&t0)[4], const float (&t1)[4]) {
    FragA f;
    split_pair(t0[0], t0[1], f.h[0], f.l[0]);
    split_pair(t0[2], t0[3], f.h[1], f.l[1]);
    split_pair(t1[0], t1[1], f.h[2], f.l[2]);
    split_pair(t1[2], t1[3], f.h[3], f.l[3]);
    return f;
}

// rows [r0, r0+rows) x columns [c0, c0+w) of a global [n, *] matrix (pitch ld) -> shared tile (stride sl, width ceil16(w)); rows
// past n and columns past w are zero.  w is a multiple of 16 bytes of T, and so are the pointer and the pitch (checked on the host).
template <typename T>
__device__ __forceinline__ void load_tile(T* S, int sl, const T* X, int64_t ld, int64_t r0, int rows, int64_t n, int c0, int w) {
    constexpr int E = 16 / sizeof(T);
    const int cpr = ceil16(w) / E;
    for (int i = threadIdx.x; i < rows * cpr; i += kThreads) {
        const int r = i / cpr, ch = i % cpr;
        T* dst = S + r * sl + ch * E;
        if (r0 + r < n && ch * E < w) cp_async16(dst, X + (r0 + r) * ld + c0 + ch * E);
        else *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
    }
}

// sums of the column sums of squares in a fixed order (double): every kernel gets a bit-identical c = 1/(||q|| ||k||)
__device__ double fixed_sum(const float* v, int len) {
    double t = 0.0;
    for (int i = 0; i < len; ++i) t += (double)v[i];
    return t;
}

// Column block of head hh inside a shared tile whose rows hold every head's block padded to 16 elements.
template <typename T>
__device__ __forceinline__ void load_heads(T* S, int sl, const T* X, int64_t ld, int64_t r0, int rows, int64_t n, int nh, int w) {
    for (int hh = 0; hh < nh; ++hh) load_tile(S + hh * ceil16(w), sl, X + (int64_t)hh * w, ld, r0, rows, n, 0, w);
}

// 16 x 16 score tile of one head: rows r0.. of A (row-major, columns a0..) against rows b0.. of B (columns b0c..), over kw
template <bool SPLIT, typename T>
__device__ __forceinline__ void tile16(float (&s)[2][4], const T* A, int lda, int r0, int ac0, const T* B, int ldb, int b0, int bc0,
                                       int kw, int lane) {
#pragma unroll
    for (int j = 0; j < 2; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
    for (int ks = 0; ks < kw; ks += 16) {
        const FragA fa = ld_a(A, lda, r0, ac0 + ks, lane);
#pragma unroll
        for (int j = 0; j < 2; ++j) mma<SPLIT>(s[j], fa, ld_b_n(B, ldb, b0 + j * 8, bc0 + ks, lane));
    }
}

__device__ __forceinline__ float c_scale(const sgf_attn_softmax_args& a) {
    return (float)(1.0 / (sqrt(fixed_sum(a.sq_q, a.heads * a.m)) * sqrt(fixed_sum(a.sq_k, a.heads * a.m))));
}
template <bool SCALED> __device__ __forceinline__ float score_scale(const sgf_attn_softmax_args& a) {
    return SCALED ? a.scale : c_scale(a);
}

// Scaled mode: the first head's raw score s of a pair starts its running maximum; its term is exp(0) = 1.
__device__ __forceinline__ void max_first(float (&s)[2][4], float (&mx)[2][4], float (&eh)[2][4], float (&den)[2][4]) {
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) { mx[j][e] = s[j][e]; eh[j][e] = den[j][e] = 1.f; }
}
// Scaled mode: one more head's raw score s of a pair.  ex = exp(-c |s - mx|): below the running maximum it is the new term;
// above it, the factor r that rescales what has been accumulated (and the new head's term is 1; else r = 1).  Returns the new
// term.
__device__ __forceinline__ float max_step(float s, float cl2, float& mx, float& eh, float& den, float& r) {
    const float dd = (s - mx) * cl2;
    const float ex = exp2f(-fabsf(dd));
    if (dd > 0.f) {
        r = ex;
        eh *= ex;
        den = fmaf(den, ex, 1.f);
        mx = s;
        return 1.f;
    }
    r = 1.f;
    den += ex;
    return ex;
}

// ---------------------------------------------------------------------------------------------------------------------------
// forward: query tile x head h x 128-column block of v_h.  Per 16-key block: E_h' = exp(c Q_h' K_h'^T) for every head,
// P_h = E_h / sum_h' E_h', o_h += P_h V_h.
// ---------------------------------------------------------------------------------------------------------------------------
template <typename T, int BS, bool SCALED>
__global__ void __launch_bounds__(kThreads, 1) fwd_kernel(const __grid_constant__ sgf_attn_softmax_args a) {
    constexpr bool SPLIT = std::is_same<T, float>::value;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ float s_c;
    const int n = a.n, H = a.heads, M = a.m, D = a.d, Mp = ceil16(M);
    const int h = blockIdx.y;
    const int dc0 = blockIdx.z * kOutCols, dw = min(kOutCols, D - dc0);
    const int slq = H * Mp + 16 / (int)sizeof(T), slv = row_stride<T>(dw);
    T* Qs = reinterpret_cast<T*>(smem_raw);
    T* Ks = Qs + kRows * slq;                 // [2][BS][slq]
    T* Vs = Ks + 2 * BS * slq;                // [2][BS][slv]
    const T* q = static_cast<const T*>(a.q);
    const T* k = static_cast<const T*>(a.k);
    const T* v = static_cast<const T*>(a.v) + (a.shared_v ? 0 : (int64_t)h * D);
    const int64_t row0 = (int64_t)blockIdx.x * kRows;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c4 = lane & 3;
    if (threadIdx.x == 0) s_c = score_scale<SCALED>(a);

    const int nt = (n + BS - 1) / BS;
    load_heads(Qs, slq, q, a.ldq, row0, kRows, n, H, M);
    load_heads(Ks, slq, k, a.ldk, 0, BS, n, H, M);
    load_tile(Vs, slv, v, a.ldv, 0, BS, n, dc0, dw);
    cp_async_commit();
    __syncthreads();
    const float cl2 = s_c * kLog2e;
    const int ndt = (dw + 7) / 8;
    const int r0 = warp * 16;
    float acc[16][4];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int t = 0; t < nt; ++t) {
        const int buf = t & 1;
        if (t + 1 < nt) {
            load_heads(Ks + (buf ^ 1) * BS * slq, slq, k, a.ldk, (int64_t)(t + 1) * BS, BS, n, H, M);
            load_tile(Vs + (buf ^ 1) * BS * slv, slv, v, a.ldv, (int64_t)(t + 1) * BS, BS, n, dc0, dw);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const T* Kb = Ks + buf * BS * slq;
        const T* Vb = Vs + buf * BS * slv;
#pragma unroll 1
        for (int sb = 0; sb < BS; sb += 16) {
            float s[2][4], eh[2][4], den[2][4], mx[2][4];
            tile16<SPLIT>(s, Qs, slq, r0, h * Mp, Kb, slq, sb, h * Mp, Mp, lane);
            if (SCALED) {
                max_first(s, mx, eh, den);
            } else {
#pragma unroll
                for (int j = 0; j < 2; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e) den[j][e] = eh[j][e] = exp2f(s[j][e] * cl2);
            }
            for (int hp = 0; hp < H; ++hp) {      // the other heads' terms of the softmax over heads, in head order
                if (hp == h) continue;
                tile16<SPLIT>(s, Qs, slq, r0, hp * Mp, Kb, slq, sb, hp * Mp, Mp, lane);
#pragma unroll
                for (int j = 0; j < 2; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        if (SCALED) {
                            float r;
                            max_step(s[j][e], cl2, mx[j][e], eh[j][e], den[j][e], r);
                        } else {
                            den[j][e] += exp2f(s[j][e] * cl2);
                        }
                    }
            }
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int64_t key = (int64_t)t * BS + sb + j * 8 + 2 * c4 + (e & 1);
                    s[j][e] = key < n ? eh[j][e] / den[j][e] : 0.f;
                }
            const FragA pa = a_from_acc(s[0], s[1]);
#pragma unroll
            for (int dj = 0; dj < 16; ++dj)
                if (dj < ndt) mma<SPLIT>(acc[dj], pa, ld_b_k(Vb, slv, sb, dj * 8, lane));
        }
        __syncthreads();
    }
    T* o = static_cast<T*>(a.o) + (int64_t)h * D + dc0;
#pragma unroll
    for (int e2 = 0; e2 < 2; ++e2) {
        const int64_t row = row0 + r0 + g + 8 * e2;
        if (row >= n) continue;
#pragma unroll
        for (int dj = 0; dj < 16; ++dj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = dj * 8 + 2 * c4 + e;
                if (dj < ndt && col < dw) o[row * a.ldo + col] = from_f32<T>(acc[dj][2 * e2 + e]);
            }
    }
}

// sum over the CTA of per-thread partials, fixed order (warp shuffle tree, then warps in order) -> one float
__device__ __forceinline__ void cta_partial(float v, float* red, float* out) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) *out = red[0] + red[1] + red[2] + red[3];
}

// dS_h of a 16 x 16 block: with E_h' = exp(c S_h') and dP_h' of every head (own head h first),
//   dS_h = P_h (dP_h - sum_h' P_h' dP_h') = (E_h / den) * (sum_h' E_h' (dP_h - dP_h')) / den,   den = sum_h' E_h'.
// The difference form is exactly zero when every head has the same dP (one head, or a shared v under the head mean).
// Scaled mode: the same with E_h' relative to the pair's running maximum (num rescaled with den and E_h).
template <bool SPLIT, bool SCALED, typename T>
__device__ __forceinline__ void dscore16(float (&ds)[2][4], int h, int H, float cl2, const T* Qa, int lda, int r0, const T* Kb, int ldb,
                                         int b0, int Mp, const T* Ga, int ldga, const T* Vb, int ldvb, int Dp, bool shared_ga, bool shared_vb,
                                         int lane) {
    float s[2][4], dp[2][4], dpo[2][4], eh[2][4], den[2][4], num[2][4], mx[2][4];
    tile16<SPLIT>(s, Qa, lda, r0, h * Mp, Kb, ldb, b0, h * Mp, Mp, lane);
    tile16<SPLIT>(dp, Ga, ldga, r0, shared_ga ? 0 : h * Dp, Vb, ldvb, b0, shared_vb ? 0 : h * Dp, Dp, lane);
    if (SCALED) max_first(s, mx, eh, den);
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            if (!SCALED) den[j][e] = eh[j][e] = exp2f(s[j][e] * cl2);
            num[j][e] = 0.f;
        }
    for (int hp = 0; hp < H; ++hp) {
        if (hp == h) continue;
        tile16<SPLIT>(s, Qa, lda, r0, hp * Mp, Kb, ldb, b0, hp * Mp, Mp, lane);
        tile16<SPLIT>(dpo, Ga, ldga, r0, shared_ga ? 0 : hp * Dp, Vb, ldvb, b0, shared_vb ? 0 : hp * Dp, Dp, lane);
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (SCALED) {
                    float r;
                    const float ex = max_step(s[j][e], cl2, mx[j][e], eh[j][e], den[j][e], r);
                    num[j][e] = fmaf(num[j][e], r, ex * (dp[j][e] - dpo[j][e]));
                } else {
                    const float ex = exp2f(s[j][e] * cl2);
                    den[j][e] += ex;
                    num[j][e] += ex * (dp[j][e] - dpo[j][e]);
                }
            }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) ds[j][e] = (eh[j][e] / den[j][e]) * (num[j][e] / den[j][e]);
}

// ---------------------------------------------------------------------------------------------------------------------------
// backward, query sweep: query tile x head h x 128-column block of q_h:  Aq_h = c dS_h K_h
// ---------------------------------------------------------------------------------------------------------------------------
template <typename T, int BS, bool SCALED>
__global__ void __launch_bounds__(kThreads) bwd_q_kernel(const __grid_constant__ sgf_attn_softmax_args a) {
    constexpr bool SPLIT = std::is_same<T, float>::value;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ float s_c, s_red[4];
    const int n = a.n, H = a.heads, M = a.m, D = a.d, Mp = ceil16(M), Dp = ceil16(D);
    const bool sg = a.g_hstride == 0, sv = a.shared_v != 0;
    const int GH = sg ? 1 : H, VH = sv ? 1 : H;
    const int h = blockIdx.y;
    const int mc0 = blockIdx.z * kOutCols, mw = min(kOutCols, M - mc0);
    constexpr int E = 16 / (int)sizeof(T);
    const int slq = H * Mp + E, slg = GH * Dp + E, slv = VH * Dp + E;
    T* Qs = reinterpret_cast<T*>(smem_raw);
    T* Gs = Qs + kRows * slq;
    T* Ks = Gs + kRows * slg;                 // [2][BS][slq]
    T* Vs = Ks + 2 * BS * slq;                // [2][BS][slv]
    const T* q = static_cast<const T*>(a.q);
    const T* k = static_cast<const T*>(a.k);
    const T* v = static_cast<const T*>(a.v);
    const T* gp = static_cast<const T*>(a.g);
    const int64_t row0 = (int64_t)blockIdx.x * kRows;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c4 = lane & 3;
    if (threadIdx.x == 0) s_c = score_scale<SCALED>(a);

    const int nt = (n + BS - 1) / BS;
    load_heads(Qs, slq, q, a.ldq, row0, kRows, n, H, M);
    load_heads(Gs, slg, gp, a.ldg, row0, kRows, n, GH, D);
    load_heads(Ks, slq, k, a.ldk, 0, BS, n, H, M);
    load_heads(Vs, slv, v, a.ldv, 0, BS, n, VH, D);
    cp_async_commit();
    __syncthreads();
    const float cl2 = s_c * kLog2e;
    const int nmt = (mw + 7) / 8;
    const int r0 = warp * 16;
    float acc[16][4];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int t = 0; t < nt; ++t) {
        const int buf = t & 1;
        if (t + 1 < nt) {
            load_heads(Ks + (buf ^ 1) * BS * slq, slq, k, a.ldk, (int64_t)(t + 1) * BS, BS, n, H, M);
            load_heads(Vs + (buf ^ 1) * BS * slv, slv, v, a.ldv, (int64_t)(t + 1) * BS, BS, n, VH, D);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const T* Kb = Ks + buf * BS * slq;
        const T* Vb = Vs + buf * BS * slv;
#pragma unroll 1
        for (int sb = 0; sb < BS; sb += 16) {
            float ds[2][4];
            dscore16<SPLIT, SCALED>(ds, h, H, cl2, Qs, slq, r0, Kb, slq, sb, Mp, Gs, slg, Vb, slv, Dp, sg, sv, lane);
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if ((int64_t)t * BS + sb + j * 8 + 2 * c4 + (e & 1) >= n) ds[j][e] = 0.f;
            const FragA da = a_from_acc(ds[0], ds[1]);
#pragma unroll
            for (int mj = 0; mj < 16; ++mj)
                if (mj < nmt) mma<SPLIT>(acc[mj], da, ld_b_k(Kb, slq, sb, h * Mp + mc0 + mj * 8, lane));
        }
        __syncthreads();
    }
    if (SCALED) {       // dq = gs c acc
        const float f = a.gscale * s_c;
        T* dq = static_cast<T*>(a.dq) + (int64_t)h * M + mc0;
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            const int64_t row = row0 + r0 + g + 8 * e2;
            if (row >= n) continue;
#pragma unroll
            for (int mj = 0; mj < 16; ++mj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = mj * 8 + 2 * c4 + e;
                    if (mj < nmt && col < mw) dq[row * a.lddq + col] = from_f32<T>(f * acc[mj][2 * e2 + e]);
                }
        }
        return;
    }
    // Aq = c * acc; partial <q, Aq> of this CTA
    const float cs = s_c;
    float* aq = a.aq + (int64_t)h * M + mc0;
    float part = 0.f;
#pragma unroll
    for (int e2 = 0; e2 < 2; ++e2) {
        const int r = r0 + g + 8 * e2;
        const int64_t row = row0 + r;
        if (row >= n) continue;
#pragma unroll
        for (int mj = 0; mj < 16; ++mj)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = mj * 8 + 2 * c4 + e;
                if (mj < nmt && col < mw) {
                    const float val = cs * acc[mj][2 * e2 + e];
                    aq[row * a.ld_a + col] = val;
                    part += val * to_f32(Qs[r * slq + h * Mp + mc0 + col]);
                }
            }
    }
    cta_partial(part, s_red, a.ws + ((int64_t)blockIdx.z * H + h) * gridDim.x + blockIdx.x);
}

// ---------------------------------------------------------------------------------------------------------------------------
// backward, key sweep: key tile x head h x (128-column block of k_h: Ak_h = c dS_h^T Q_h | of v_h: dV_h = gs P_h^T G_h)
// ---------------------------------------------------------------------------------------------------------------------------
template <typename T, int BS, bool SCALED>
__global__ void __launch_bounds__(kThreads) bwd_kv_kernel(const __grid_constant__ sgf_attn_softmax_args a) {
    constexpr bool SPLIT = std::is_same<T, float>::value;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ float s_c, s_red[4];
    const int n = a.n, H = a.heads, M = a.m, D = a.d, Mp = ceil16(M), Dp = ceil16(D);
    const bool sg = a.g_hstride == 0, sv = a.shared_v != 0;
    const int GH = sg ? 1 : H, VH = sv ? 1 : H;
    const int n_mc = (M + kOutCols - 1) / kOutCols;
    const bool want_dk = (int)blockIdx.z < n_mc;
    if (!want_dk && sv && blockIdx.y > 0) return;      // a shared v: head 0's CTAs sum every head
    const int oc0 = (want_dk ? blockIdx.z : blockIdx.z - n_mc) * kOutCols;
    const int ow = min(kOutCols, (want_dk ? M : D) - oc0);
    constexpr int E = 16 / (int)sizeof(T);
    const int slq = H * Mp + E, slg = GH * Dp + E, slv = VH * Dp + E;
    T* Ks = reinterpret_cast<T*>(smem_raw);
    T* Vs = Ks + kRows * slq;
    T* Qs = Vs + kRows * slv;                 // [2][BS][slq]
    T* Gs = Qs + 2 * BS * slq;                // [2][BS][slg]
    const T* q = static_cast<const T*>(a.q);
    const T* k = static_cast<const T*>(a.k);
    const T* v = static_cast<const T*>(a.v);
    const T* gp = static_cast<const T*>(a.g);
    const int64_t row0 = (int64_t)blockIdx.x * kRows;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c4 = lane & 3;
    if (threadIdx.x == 0) s_c = score_scale<SCALED>(a);
    const int nj = (ow + 7) / 8;
    const int r0 = warp * 16;
    const int nt = (n + BS - 1) / BS;
    const int h_begin = want_dk || !sv ? (int)blockIdx.y : 0, h_end = want_dk || !sv ? h_begin + 1 : H;
    load_heads(Ks, slq, k, a.ldk, row0, kRows, n, H, M);
    if (want_dk) load_heads(Vs, slv, v, a.ldv, row0, kRows, n, VH, D);
    __syncthreads();
    const float cl2 = s_c * kLog2e;
    float acc[16][4];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int hd = h_begin; hd < h_end; ++hd) {
        load_heads(Qs, slq, q, a.ldq, 0, BS, n, H, M);
        load_heads(Gs, slg, gp, a.ldg, 0, BS, n, GH, D);
        cp_async_commit();
        for (int t = 0; t < nt; ++t) {
            const int buf = t & 1;
            if (t + 1 < nt) {
                load_heads(Qs + (buf ^ 1) * BS * slq, slq, q, a.ldq, (int64_t)(t + 1) * BS, BS, n, H, M);
                load_heads(Gs + (buf ^ 1) * BS * slg, slg, gp, a.ldg, (int64_t)(t + 1) * BS, BS, n, GH, D);
                cp_async_commit();
                cp_async_wait<1>();
            } else {
                cp_async_wait<0>();
            }
            __syncthreads();
            const T* Qb = Qs + buf * BS * slq;
            const T* Gb = Gs + buf * BS * slg;
            const int gc = sg ? 0 : hd * Dp;
#pragma unroll 1
            for (int sb = 0; sb < BS; sb += 16) {
                float w[2][4];
                if (want_dk) {
                    dscore16<SPLIT, SCALED>(w, hd, H, cl2, Ks, slq, r0, Qb, slq, sb, Mp, Vs, slv, Gb, slg, Dp, sv, sg, lane);
                } else {       // P_h^T
                    float s[2][4], den[2][4], mx[2][4];
                    tile16<SPLIT>(s, Ks, slq, r0, hd * Mp, Qb, slq, sb, hd * Mp, Mp, lane);
                    if (SCALED) {
                        max_first(s, mx, w, den);
                    } else {
#pragma unroll
                        for (int j = 0; j < 2; ++j)
#pragma unroll
                            for (int e = 0; e < 4; ++e) den[j][e] = w[j][e] = exp2f(s[j][e] * cl2);
                    }
                    for (int hp = 0; hp < H; ++hp) {
                        if (hp == hd) continue;
                        tile16<SPLIT>(s, Ks, slq, r0, hp * Mp, Qb, slq, sb, hp * Mp, Mp, lane);
#pragma unroll
                        for (int j = 0; j < 2; ++j)
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                if (SCALED) {
                                    float r;
                                    max_step(s[j][e], cl2, mx[j][e], w[j][e], den[j][e], r);
                                } else {
                                    den[j][e] += exp2f(s[j][e] * cl2);
                                }
                            }
                    }
#pragma unroll
                    for (int j = 0; j < 2; ++j)
#pragma unroll
                        for (int e = 0; e < 4; ++e) w[j][e] /= den[j][e];
                }
#pragma unroll
                for (int j = 0; j < 2; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if ((int64_t)t * BS + sb + j * 8 + 2 * c4 + (e & 1) >= n) w[j][e] = 0.f;
                const FragA fa = a_from_acc(w[0], w[1]);
                if (want_dk) {
#pragma unroll
                    for (int mj = 0; mj < 16; ++mj)
                        if (mj < nj) mma<SPLIT>(acc[mj], fa, ld_b_k(Qb, slq, sb, hd * Mp + oc0 + mj * 8, lane));
                } else {
#pragma unroll
                    for (int dj = 0; dj < 16; ++dj)
                        if (dj < nj) mma<SPLIT>(acc[dj], fa, ld_b_k(Gb, slg, sb, gc + oc0 + dj * 8, lane));
                }
            }
            __syncthreads();
        }
    }
    if (SCALED && want_dk) {        // dk = gs c acc
        const float f = a.gscale * s_c;
        T* dk = static_cast<T*>(a.dk) + (int64_t)blockIdx.y * M + oc0;
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            const int64_t row = row0 + r0 + g + 8 * e2;
            if (row >= n) continue;
#pragma unroll
            for (int mj = 0; mj < 16; ++mj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = mj * 8 + 2 * c4 + e;
                    if (mj < nj && col < ow) dk[row * a.lddk + col] = from_f32<T>(f * acc[mj][2 * e2 + e]);
                }
        }
    } else if (want_dk) {      // Ak = c * acc; partial <k, Ak> of this CTA
        const float cs = s_c;
        float* ak = a.ak + (int64_t)blockIdx.y * M + oc0;
        float part = 0.f;
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            const int r = r0 + g + 8 * e2;
            const int64_t row = row0 + r;
            if (row >= n) continue;
#pragma unroll
            for (int mj = 0; mj < 16; ++mj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = mj * 8 + 2 * c4 + e;
                    if (mj < nj && col < ow) {
                        const float val = cs * acc[mj][2 * e2 + e];
                        ak[row * a.ld_a + col] = val;
                        part += val * to_f32(Ks[r * slq + blockIdx.y * Mp + oc0 + col]);
                    }
                }
        }
        const int64_t n_q = (int64_t)gridDim.x * H * n_mc;     // bwd_q's partials come first in ws
        cta_partial(part, s_red, a.ws + n_q + ((int64_t)blockIdx.z * H + blockIdx.y) * gridDim.x + blockIdx.x);
    } else {            // dv (+)= gs * acc
        T* dv = static_cast<T*>(a.dv) + (sv ? 0 : (int64_t)blockIdx.y * D) + oc0;
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            const int64_t row = row0 + r0 + g + 8 * e2;
            if (row >= n) continue;
#pragma unroll
            for (int dj = 0; dj < 16; ++dj)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = dj * 8 + 2 * c4 + e;
                    if (dj < nj && col < ow) {
                        T* p = dv + row * a.lddv + col;
                        const float val = a.gscale * acc[dj][2 * e2 + e];
                        *p = from_f32<T>(a.dv_accumulate ? to_f32(*p) + val : val);
                    }
                }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// norm backward: out = gs (A - (sum(part)/||x||^2) x), blockIdx.y = 0: q, 1: k
// ---------------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) norm_kernel(const __grid_constant__ sgf_attn_softmax_args a, int64_t n_part_q, int64_t n_part_k) {
    __shared__ float s_t;
    const bool isk = blockIdx.y == 1;
    const int HM = a.heads * a.m;
    if (threadIdx.x < 32) {       // lanes sum strided partials, then a fixed shuffle tree
        const float* part = a.ws + (isk ? n_part_q : 0);
        const int64_t np = isk ? n_part_k : n_part_q;
        double t = 0.0;
        for (int64_t i = threadIdx.x; i < np; i += 32) t += (double)part[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (threadIdx.x == 0) s_t = (float)(t / fixed_sum(isk ? a.sq_k : a.sq_q, HM));
    }
    __syncthreads();
    const float t = s_t, gs = a.gscale;
    const float* A = isk ? a.ak : a.aq;
    const T* x = static_cast<const T*>(isk ? a.k : a.q);
    const int64_t ldx = isk ? a.ldk : a.ldq;
    T* out = static_cast<T*>(isk ? a.dk : a.dq);
    const int64_t ldo = isk ? a.lddk : a.lddq;
    const int64_t total = (int64_t)a.n * HM;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / HM, cidx = i % HM;
        out[r * ldo + cidx] = from_f32<T>(gs * (A[r * a.ld_a + cidx] - t * to_f32(x[r * ldx + cidx])));
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// visualisation: att[n, l] = mean_h P[n, l, h]  (the head mean of the softmax over heads; inference only, O(N^2) output)
// ---------------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) probs_kernel(const __grid_constant__ sgf_attn_softmax_args a, float* att, int64_t ld_att) {
    __shared__ float s_c;
    const int n = a.n, H = a.heads, M = a.m;
    if (threadIdx.x == 0) s_c = c_scale(a);
    __syncthreads();
    const float cl2 = s_c * kLog2e;
    const int64_t total = (int64_t)n * n;
    const T* q = static_cast<const T*>(a.q);
    const T* k = static_cast<const T*>(a.k);
    auto score = [&](int64_t r, int64_t l, int hd) {
        float s = 0.f;
        for (int j = 0; j < M; ++j) s += to_f32(q[r * a.ldq + hd * M + j]) * to_f32(k[l * a.ldk + hd * M + j]);
        return exp2f(s * cl2);
    };
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / n, l = i % n;
        float den = 0.f;
        for (int hd = 0; hd < H; ++hd) den += score(r, l, hd);
        float tot = 0.f;
        for (int hd = 0; hd < H; ++hd) tot += score(r, l, hd) / den;
        att[r * ld_att + l] = tot / (float)H;
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int kSmemMax = 227 * 1024;

struct Widths {      // shared-memory row strides (elements) of the all-head q/k rows, the v rows and the g rows; d: v's width
    int slq, slv, slg, d;
};
template <typename T> static Widths widths(int heads, int m, int d, bool shared_v, bool shared_g) {
    constexpr int E = 16 / sizeof(T);
    const int gh = shared_g ? 1 : heads, vh = shared_v ? 1 : heads;
    return Widths{heads * ceil16(m) + E, vh * ceil16(d) + E, gh * ceil16(d) + E, d};
}
// largest streamed tile (64, 32 or 16 rows) whose double buffer fits next to the resident tiles; the static shared memory is
// counted with a margin.  kind 0: fwd, 1: bwd_q, 2: bwd_kv.  0: none fits.
template <typename T> static int pick_bs(const Widths& w, int kind, size_t* bytes) {
    const int dw = w.d < kOutCols ? w.d : kOutCols;
    for (int bs : {64, 32, 16}) {
        size_t e = 0;
        if (kind == 0) e = (size_t)kRows * w.slq + 2 * (size_t)bs * (w.slq + row_stride<T>(dw));
        if (kind == 1) e = (size_t)kRows * (w.slq + w.slg) + 2 * (size_t)bs * (w.slq + w.slv);
        if (kind == 2) e = (size_t)kRows * (w.slq + w.slv) + 2 * (size_t)bs * (w.slq + w.slg);
        *bytes = e * sizeof(T);
        if (*bytes + 1024 <= (size_t)kSmemMax) return bs;
    }
    return 0;
}
template <typename T> static int pick_bs(const sgf_attn_softmax_args* a, int kind, size_t* bytes) {
    return pick_bs<T>(widths<T>(a->heads, a->m, a->d, a->shared_v != 0, a->g_hstride == 0), kind, bytes);
}

template <typename T> static bool aligned16(const void* p, int64_t ld) {
    return p && (reinterpret_cast<uintptr_t>(p) & 15u) == 0 && (ld * (int64_t)sizeof(T)) % 16 == 0;
}

// m and d are multiples of 16 bytes, and the padded head blocks of one q/k row and of one v row each take at most
// SGF_ATTN_SOFTMAX_MAX_ROW_BYTES
template <typename T> static bool shape_ok(int heads, int m, int d, bool shared_v) {
    constexpr int E = 16 / sizeof(T);
    const int64_t vh = shared_v ? 1 : heads;
    return m % E == 0 && d % E == 0 && (int64_t)heads * ceil16(m) * sizeof(T) <= SGF_ATTN_SOFTMAX_MAX_ROW_BYTES &&
           vh * ceil16(d) * sizeof(T) <= SGF_ATTN_SOFTMAX_MAX_ROW_BYTES;
}

template <typename T> static int check_common(const sgf_attn_softmax_args* a) {
    if (!a || a->n <= 0 || a->heads <= 0 || a->m <= 0 || a->d <= 0) return SGF_ERR_ARG;
    if (a->scaled != 0 && a->scaled != 1) return SGF_ERR_ARG;
    if (a->scaled ? !(a->scale > 0.f && a->scale < INFINITY) || a->shared_v : !a->sq_q || !a->sq_k) return SGF_ERR_ARG;
    if (!shape_ok<T>(a->heads, a->m, a->d, a->shared_v != 0)) return SGF_ERR_UNSUPPORTED;
    if (!aligned16<T>(a->q, a->ldq) || !aligned16<T>(a->k, a->ldk) || !aligned16<T>(a->v, a->ldv)) return SGF_ERR_ARG;
    return SGF_OK;
}

// host only (no CUDA call): the streamed-tile heights the fwd, bwd_q and bwd_kv launches would pick
template <typename T> static int tile_rows(int heads, int m, int d, bool shared_v, bool shared_g, int32_t* rows) {
    if (!shape_ok<T>(heads, m, d, shared_v)) return SGF_ERR_UNSUPPORTED;
    const Widths w = widths<T>(heads, m, d, shared_v, shared_g);
    size_t bytes = 0;
    for (int kind = 0; kind < 3; ++kind) rows[kind] = pick_bs<T>(w, kind, &bytes);
    return SGF_OK;
}

template <typename K> static int launch(K kernel, dim3 grid, int threads, size_t smem, const sgf_attn_softmax_args* a, cudaStream_t st) {
    SGF_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, threads, smem, st>>>(*a);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

#define SGF_SOFT_LAUNCH(kern, kind, grid)                                                        \
    do {                                                                                         \
        size_t sm = 0;                                                                           \
        const int bs = pick_bs<T>(a, kind, &sm);                                                 \
        if (a->scaled) {                                                                         \
            if (bs == 64) return launch(kern<T, 64, true>, grid, kThreads, sm, a, st);           \
            if (bs == 32) return launch(kern<T, 32, true>, grid, kThreads, sm, a, st);           \
            if (bs == 16) return launch(kern<T, 16, true>, grid, kThreads, sm, a, st);           \
            return SGF_ERR_UNSUPPORTED;                                                          \
        }                                                                                        \
        if (bs == 64) return launch(kern<T, 64, false>, grid, kThreads, sm, a, st);              \
        if (bs == 32) return launch(kern<T, 32, false>, grid, kThreads, sm, a, st);              \
        if (bs == 16) return launch(kern<T, 16, false>, grid, kThreads, sm, a, st);              \
        return SGF_ERR_UNSUPPORTED;                                                              \
    } while (0)

template <typename T> static int fwd(const sgf_attn_softmax_args* a, cudaStream_t st) {
    int rc = check_common<T>(a);
    if (rc) return rc;
    if (!a->o || (reinterpret_cast<uintptr_t>(a->o) % sizeof(T))) return SGF_ERR_ARG;
    const dim3 grid((a->n + kRows - 1) / kRows, a->heads, (a->d + kOutCols - 1) / kOutCols);
    SGF_SOFT_LAUNCH(fwd_kernel, 0, grid);
}

static int64_t parts_q(int n, int heads, int m) { return (int64_t)((n + kRows - 1) / kRows) * heads * ((m + kOutCols - 1) / kOutCols); }

template <typename T> static int bwd_check(const sgf_attn_softmax_args* a) {
    int rc = check_common<T>(a);
    if (rc) return rc;
    if (!aligned16<T>(a->g, a->ldg) || (a->g_hstride != 0 && a->g_hstride != a->d)) return SGF_ERR_ARG;
    if (a->scaled) return SGF_OK;       // no partial sums
    if (!a->ws) return SGF_ERR_ARG;
    int64_t need = 0;
    sgf_attn_softmax_ws_floats(a->n, a->heads, a->m, a->d, &need);
    return a->ws_floats < need ? SGF_ERR_ARG : SGF_OK;
}

// the sweep's output: aq / ak (fp32, pitch ld_a), or in scaled mode dq / dk (dtype, pitch lddq / lddk)
template <typename T> static bool grad_out_ok(const sgf_attn_softmax_args* a, const float* acc, const void* out, int64_t ld) {
    const int64_t hm = (int64_t)a->heads * a->m;
    if (!a->scaled) return acc && a->ld_a >= hm;
    return out && (reinterpret_cast<uintptr_t>(out) % sizeof(T)) == 0 && ld >= hm;
}

template <typename T> static int bwd_q(const sgf_attn_softmax_args* a, cudaStream_t st) {
    int rc = bwd_check<T>(a);
    if (rc) return rc;
    if (!grad_out_ok<T>(a, a->aq, a->dq, a->lddq)) return SGF_ERR_ARG;
    const dim3 grid((a->n + kRows - 1) / kRows, a->heads, (a->m + kOutCols - 1) / kOutCols);
    SGF_SOFT_LAUNCH(bwd_q_kernel, 1, grid);
}

template <typename T> static int bwd_kv(const sgf_attn_softmax_args* a, cudaStream_t st) {
    int rc = bwd_check<T>(a);
    if (rc) return rc;
    if (!grad_out_ok<T>(a, a->ak, a->dk, a->lddk) || !a->dv) return SGF_ERR_ARG;
    const int n_mc = (a->m + kOutCols - 1) / kOutCols, n_dc = (a->d + kOutCols - 1) / kOutCols;
    const dim3 grid((a->n + kRows - 1) / kRows, a->heads, n_mc + n_dc);
    SGF_SOFT_LAUNCH(bwd_kv_kernel, 2, grid);
}

template <typename T> static int bwd_norm(const sgf_attn_softmax_args* a, cudaStream_t st) {
    if (!a || a->n <= 0 || a->heads <= 0 || a->m <= 0 || !a->aq || !a->ak || !a->dq || !a->dk || !a->q || !a->k || !a->ws ||
        !a->sq_q || !a->sq_k || a->scaled)      // the scaled mode's sweeps write dq, dk themselves
        return SGF_ERR_ARG;
    const int64_t nq = parts_q(a->n, a->heads, a->m);
    const int64_t total = (int64_t)a->n * a->heads * a->m;
    const int blocks = (int)((total + 255) / 256 < 4 * num_sms() ? (total + 255) / 256 : 4 * num_sms());
    norm_kernel<T><<<dim3(blocks, 2), 256, 0, st>>>(*a, nq, nq);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

template <typename T> static int probs(const sgf_attn_softmax_args* a, float* att, int64_t ld_att, cudaStream_t st) {
    if (!a || a->n <= 0 || a->heads <= 0 || a->m <= 0 || !a->q || !a->k || !a->sq_q || !a->sq_k || !att || ld_att < a->n ||
        a->scaled)
        return SGF_ERR_ARG;
    const int64_t total = (int64_t)a->n * a->n;
    const int blocks = (int)((total + 255) / 256 < 8 * num_sms() ? (total + 255) / 256 : 8 * num_sms());
    probs_kernel<T><<<blocks, 256, 0, st>>>(*a, att, ld_att);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

}  // namespace soft
}  // namespace sgf

using namespace sgf::soft;

extern "C" int sgf_attn_softmax_ws_floats(int n, int heads, int m, int d, int64_t* n_floats) {
    if (!n_floats || n <= 0 || heads <= 0 || m <= 0 || d <= 0) return SGF_ERR_ARG;
    *n_floats = 2 * parts_q(n, heads, m);        // bwd_q's and bwd_kv's per-CTA partials (same grid extent)
    return SGF_OK;
}

extern "C" int sgf_attn_softmax_tile_rows(int heads, int m, int d, int dtype, int shared_v, int shared_g, int32_t rows[3]) {
    if (!rows || heads <= 0 || m <= 0 || d <= 0) return SGF_ERR_ARG;
    if (dtype == 0) return tile_rows<float>(heads, m, d, shared_v != 0, shared_g != 0, rows);
    if (dtype == 1) return tile_rows<__nv_bfloat16>(heads, m, d, shared_v != 0, shared_g != 0, rows);
    return SGF_ERR_ARG;
}

#define SGF_SOFT_DISPATCH(fn, ...)                                                                 \
    do {                                                                                           \
        if (!a) return SGF_ERR_ARG;                                                                \
        if (a->dtype == 0) return fn<float>(a, ##__VA_ARGS__, (cudaStream_t)stream);               \
        if (a->dtype == 1) return fn<__nv_bfloat16>(a, ##__VA_ARGS__, (cudaStream_t)stream);       \
        return SGF_ERR_ARG;                                                                        \
    } while (0)

extern "C" int sgf_attn_softmax_fwd(const sgf_attn_softmax_args* a, void* stream) { SGF_SOFT_DISPATCH(fwd); }
extern "C" int sgf_attn_softmax_bwd_q(const sgf_attn_softmax_args* a, void* stream) { SGF_SOFT_DISPATCH(bwd_q); }
extern "C" int sgf_attn_softmax_bwd_kv(const sgf_attn_softmax_args* a, void* stream) { SGF_SOFT_DISPATCH(bwd_kv); }
extern "C" int sgf_attn_softmax_bwd_norm(const sgf_attn_softmax_args* a, void* stream) { SGF_SOFT_DISPATCH(bwd_norm); }
extern "C" int sgf_attn_softmax_probs(const sgf_attn_softmax_args* a, float* att, int64_t ld_att, void* stream) {
    SGF_SOFT_DISPATCH(probs, att, ld_att);
}
