// Gram-form linear attention: the h x h algebra between the node passes (fp32, SIMT).
//
// full_attention_conv on projected inputs (reference medium/ours.py:14-34 with q/k/v = Linear(x), :76-85; large/ours.py:123-149;
// 100M/ours.py:12-43,175-184) only ever contracts q, k, v over the NODE dimension.  With q = x Wq^T + bq (k, v alike) those
// contractions are functions of G = x^T x and s = x^T 1:
//     kx := k^T x = Wk G + bk s^T            z1 := k^T 1 = Wk s + N bk           (qx, q1, vx, v1 alike)
//     S  := k^T v = kx Wv^T + z1 bv^T        ||k||^2 = <kx, Wk> + z1.bk          ||q||^2 = <qx, Wq> + q1.bq
// so with alpha = 1/(||q|| ||k||), beta = alpha/N the whole layer is   out = (x Bt^T + bt) / (x ct + dt),
//     Bt = beta S^T Wq + Wv [d,h],  bt = beta S^T bq + bv,  ct = beta Wq^T z1,  dt = beta bq.z1 + 1
// (numerator and denominator of medium/ours.py:21-31 divided by N).  sgf_attn_gram_prepare_fwd evaluates this from G, s and the
// weights; the node passes themselves are wgmma GEMMs (sgf_gemm_tn x^T x, sgf_gemm_nt with SGF_EPI_ATTN_GRAM).
// Backward (SURVEY.md Appendix A.1 pushed through the projections): with gnum' = g/den~, gden' = -(g.o)/den~ (sgf_ln_bwd_attn),
// P = x^T gnum', pg = x^T gden', cs = 1^T gnum', sg = 1^T gden':
//     dS = Wq P + bq cs^T,  dz = Wq pg + bq sg,  c = beta(<dS,S> + <dz,z1>),  cq = -c/||q||^2,  ck = -c/||k||^2
//     dWq = beta S P^T + beta z1 pg^T + cq qx          dbq = beta (S cs + sg z1) + cq q1
//     dWk = beta dS vx + beta dz s^T + ck kx           dbk = beta dS v1 + alpha dz + ck z1
//     dWv = beta dS^T kx + P^T                         dbv = beta dS^T z1 + cs
//     dx  = gnum' Bt + x A3 + gden' (x) ct + 1 (x) a4,   A3 = cq Wq^T Wq + ck Wk^T Wk + beta (Wk^T dS Wv + (Wk^T dS Wv)^T),
//     a4  = cq Wq^T bq + ck Wk^T bk + beta (Wk^T (dz + dS bv) + Wv^T dS^T bk)
// (checked against autograd of the reference formula in fp64: tests/test_gram_attention_math.py).
// Everything here is O(h^3) work on matrices of at most a few hundred rows: one generic batched small-GEMM kernel
// (several independent products per launch), a batched dot-product kernel and two scalar kernels.
#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

#include <cstring>

namespace sgf {
namespace gram {

// scalar slots of sgf_attn_gram_args.sc (mirrored in sgformer_b200/kernels.py)
enum : int { SC_NQ2 = 0, SC_NK2 = 1, SC_ALPHA = 2, SC_BETA = 3, SC_DEN = 4, SC_N = 5, SC_ONE = 6, SC_BQZ = 7, SC_IP = 8, SC_C = 9,
             SC_CQ = 10, SC_CK = 11 };

struct Mat {          // element (i, j) = p[i*rs + j*cs]; p == nullptr: absent
    const float* p;
    int64_t rs, cs;
};
struct Coef {         // value = s * (dev ? *dev : 1)
    float s;
    const float* dev;
};
// C[m,n] = c1 * A1[m,k1] B1[k1,n] + c2 * A2[m,k2] B2[k2,n] + ce * E[m,n] + cg * u[m] (x) v[n]     (every term optional)
struct Op {
    int m, n, k1, k2;
    Mat A1, B1, A2, B2, E;
    Coef c1, c2, ce, cg;
    const float* u; const float* v;
    int64_t us, vs;
    float* C;
    int64_t c_rs, c_cs;
    int tiles_n, tile0;
};
constexpr int MAX_OPS = 8;
struct Batch {
    int n_ops, total_tiles;
    Op op[MAX_OPS];
};
constexpr int TILE = 32, KC = 16;

__device__ __forceinline__ float coef(const Coef& c) { return c.dev ? c.s * *c.dev : c.s; }

__global__ void __launch_bounds__(256) small_ops_kernel(const __grid_constant__ Batch bt) {
    __shared__ float As[TILE][KC + 1];
    __shared__ float Bs[KC][TILE + 1];
    int oi = 0;
    while (oi + 1 < bt.n_ops && (int)blockIdx.x >= bt.op[oi + 1].tile0) ++oi;
    const Op& op = bt.op[oi];
    const int t = blockIdx.x - op.tile0;
    const int i0 = (t / op.tiles_n) * TILE, j0 = (t % op.tiles_n) * TILE;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float tot[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    for (int term = 0; term < 2; ++term) {
        const Mat& A = term ? op.A2 : op.A1;
        const Mat& B = term ? op.B2 : op.B1;
        const int k = term ? op.k2 : op.k1;
        if (k <= 0 || !A.p) continue;
        float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
        for (int k0 = 0; k0 < k; k0 += KC) {
            for (int e = threadIdx.x; e < TILE * KC; e += 256) {
                const int i = e / KC, kk = e % KC;
                As[i][kk] = (i0 + i < op.m && k0 + kk < k) ? A.p[(int64_t)(i0 + i) * A.rs + (int64_t)(k0 + kk) * A.cs] : 0.f;
                const int kb = e / TILE, j = e % TILE;
                Bs[kb][j] = (j0 + j < op.n && k0 + kb < k) ? B.p[(int64_t)(k0 + kb) * B.rs + (int64_t)(j0 + j) * B.cs] : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < KC; ++kk) {
                const float a0 = As[ty][kk], a1 = As[ty + 16][kk], b0 = Bs[kk][tx], b1 = Bs[kk][tx + 16];
                acc[0][0] += a0 * b0; acc[0][1] += a0 * b1; acc[1][0] += a1 * b0; acc[1][1] += a1 * b1;
            }
            __syncthreads();
        }
        const float c = coef(term ? op.c2 : op.c1);
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b) tot[a][b] += c * acc[a][b];
    }
    const float ce = op.E.p ? coef(op.ce) : 0.f;
    const float cg = op.u ? coef(op.cg) : 0.f;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int i = i0 + ty + 16 * a, j = j0 + tx + 16 * b;
            if (i >= op.m || j >= op.n) continue;
            float r = tot[a][b];
            if (op.E.p) r += ce * op.E.p[(int64_t)i * op.E.rs + (int64_t)j * op.E.cs];
            if (op.u) r += cg * op.u[(int64_t)i * op.us] * op.v[(int64_t)j * op.vs];
            op.C[(int64_t)i * op.c_rs + (int64_t)j * op.c_cs] = r;
        }
}

// Frobenius inner products <A, B> = sum_{i<m, j<n} A(i,j) B(i,j): DOT_SPLIT blocks per product write their slice's sum to
// part[d][blockIdx.y]; the scalar kernels add a slot's partials in fixed order (deterministic, no atomics).
constexpr int DOT_SPLIT = 32;
struct Dot {
    Mat A, B;
    int m, n;
    int slot;           // partial sums go to part[slot_part0 .. +DOT_SPLIT)
};
struct DotBatch {
    int n;
    float* part;        // [n][DOT_SPLIT]
    Dot d[MAX_OPS];
};
__global__ void __launch_bounds__(256) dots_kernel(const __grid_constant__ DotBatch db) {
    const Dot& d = db.d[blockIdx.x];
    float s = 0.f;
    const int64_t total = (int64_t)d.m * d.n;
    for (int64_t e = (int64_t)blockIdx.y * 256 + threadIdx.x; e < total; e += 256 * DOT_SPLIT) {
        const int64_t i = e / d.n, j = e % d.n;
        s += d.A.p[i * d.A.rs + j * d.A.cs] * d.B.p[i * d.B.rs + j * d.B.cs];
    }
    __shared__ float red[8];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tsum = 0.f;
        for (int w = 0; w < 8; ++w) tsum += red[w];
        db.part[blockIdx.x * DOT_SPLIT + blockIdx.y] = tsum;
    }
}
// sum of the partials of dot products [d0, d1) in fixed order
__device__ __forceinline__ double dot_sum(const float* part, int d0, int d1) {
    double t = 0.0;
    for (int i = d0 * DOT_SPLIT; i < d1 * DOT_SPLIT; ++i) t += (double)part[i];
    return t;
}

__global__ void init_sc_kernel(float* sc, float nf) {
    if (threadIdx.x < 16) sc[threadIdx.x] = threadIdx.x == SC_N ? nf : (threadIdx.x == SC_ONE ? 1.f : 0.f);
}
// forward dot products (in launch order): 0 <kx,Wk>  1 z1.bk  2 <qx,Wq>  3 q1.bq  4 bq.z1
__global__ void scal_fwd_kernel(float* sc, const float* part) {
    // alpha = 1/(||q|| ||k||) in double: the two norms are sums over ~N*h terms
    const double nk2 = dot_sum(part, 0, 2), nq2 = dot_sum(part, 2, 4);
    sc[SC_NQ2] = (float)nq2;
    sc[SC_NK2] = (float)nk2;
    sc[SC_BQZ] = (float)dot_sum(part, 4, 5);
    const double alpha = 1.0 / (sqrt(nq2) * sqrt(nk2));
    const double beta = alpha / (double)sc[SC_N];
    sc[SC_ALPHA] = (float)alpha;
    sc[SC_BETA] = (float)beta;
    sc[SC_DEN] = (float)(beta * (double)sc[SC_BQZ] + 1.0);
}
// backward dot products: 0 <dS,S>  1 dz.z1
__global__ void scal_bwd_kernel(float* sc, const float* part) {
    const double ip = dot_sum(part, 0, 2);
    sc[SC_IP] = (float)ip;
    const double c = (double)sc[SC_BETA] * ip;
    sc[SC_C] = (float)c;
    sc[SC_CQ] = (float)(-c / (double)sc[SC_NQ2]);
    sc[SC_CK] = (float)(-c / (double)sc[SC_NK2]);
}

// ---- host-side builders -------------------------------------------------------------------------
static inline Mat mat(const float* p, int64_t rs, int64_t cs = 1) { return Mat{p, rs, cs}; }
static inline Mat matT(const float* p, int64_t ld) { return Mat{p, 1, ld}; }      // transpose view of a row-major [*, ld] matrix
static inline Mat vec(const float* p) { return Mat{p, 1, 0}; }                   // column vector [k,1] / [m,1]
static inline Coef cf(float s, const float* dev = nullptr) { return Coef{s, dev}; }

struct BatchBuilder {
    Batch b;
    BatchBuilder() { memset(&b, 0, sizeof(b)); }
    Op& add(int m, int n, float* C, int64_t c_rs, int64_t c_cs = 1) {
        Op& o = b.op[b.n_ops++];
        o.m = m; o.n = n; o.C = C; o.c_rs = c_rs; o.c_cs = c_cs;
        o.tiles_n = (n + TILE - 1) / TILE;
        o.tile0 = b.total_tiles;
        b.total_tiles += ((m + TILE - 1) / TILE) * o.tiles_n;
        return o;
    }
    int launch(cudaStream_t st) {
        if (b.n_ops == 0) return SGF_OK;
        small_ops_kernel<<<b.total_tiles, 256, 0, st>>>(b);
        SGF_LAUNCH_CHECK(); count_launch();
        return SGF_OK;
    }
};
static inline void prod1(Op& o, Coef c, Mat A, Mat B, int k) { o.c1 = c; o.A1 = A; o.B1 = B; o.k1 = k; }
static inline void prod2(Op& o, Coef c, Mat A, Mat B, int k) { o.c2 = c; o.A2 = A; o.B2 = B; o.k2 = k; }
static inline void addend(Op& o, Coef c, Mat E) { o.ce = c; o.E = E; }
static inline void rank1(Op& o, Coef c, const float* u, int64_t us, const float* v, int64_t vs) {
    o.cg = c; o.u = u; o.us = us; o.v = v; o.vs = vs;
}
struct DotBuilder {
    DotBatch b;
    explicit DotBuilder(float* part) { memset(&b, 0, sizeof(b)); b.part = part; }
    void add(Mat A, Mat B, int m, int n) { b.d[b.n] = Dot{A, B, m, n, b.n}; ++b.n; }
    int launch(cudaStream_t st) {
        dots_kernel<<<dim3(b.n, DOT_SPLIT), 256, 0, st>>>(b);
        SGF_LAUNCH_CHECK(); count_launch();
        return SGF_OK;
    }
};

static bool args_ok(const sgf_attn_gram_args* a) {
    return a && a->h > 0 && a->m > 0 && a->d > 0 && a->n_nodes > 0 && a->wq && a->bq && a->wk && a->bk && a->wv && a->bv &&
           a->ld_wq >= a->h && a->ld_wk >= a->h && a->ld_wv >= a->h && a->G && a->s && a->kx && a->qx && a->vx && a->z1 && a->q1 &&
           a->v1 && a->S && a->Bt && a->tail && a->bt && a->sc;
}
}  // namespace gram
}  // namespace sgf

using namespace sgf;
using namespace sgf::gram;

extern "C" int sgf_attn_gram_ws_floats(int h, int m, int d, int64_t* n_floats) {
    if (!n_floats || h <= 0 || m <= 0 || d <= 0) return SGF_ERR_ARG;
    *n_floats = (int64_t)m * d /* dS */ + m /* dz */ + (int64_t)m * h /* U */ + m /* t1 */ + d /* t2 */ +
                MAX_OPS * DOT_SPLIT /* dot-product partials */;
    return SGF_OK;
}

extern "C" int sgf_attn_gram_prepare_fwd(const sgf_attn_gram_args* a, void* stream) {
    if (!args_ok(a) || !a->ws) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    const int h = a->h, m = a->m, d = a->d;
    int64_t need = 0;
    sgf_attn_gram_ws_floats(h, m, d, &need);
    if (a->ws_floats < need) return SGF_ERR_ARG;
    float* part = a->ws + (need - MAX_OPS * DOT_SPLIT);
    float* sc = a->sc;
    const float* scN = sc + SC_N;
    const float* beta = sc + SC_BETA;
    int rc;
    init_sc_kernel<<<1, 32, 0, st>>>(sc, (float)a->n_nodes);
    SGF_LAUNCH_CHECK(); count_launch();
    {   // level 1: the node-contracted first moments of q, k, v
        BatchBuilder bb;
        { Op& o = bb.add(m, h, a->kx, h); prod1(o, cf(1.f), mat(a->wk, a->ld_wk), mat(a->G, h), h); rank1(o, cf(1.f), a->bk, 1, a->s, 1); }
        { Op& o = bb.add(m, h, a->qx, h); prod1(o, cf(1.f), mat(a->wq, a->ld_wq), mat(a->G, h), h); rank1(o, cf(1.f), a->bq, 1, a->s, 1); }
        { Op& o = bb.add(d, h, a->vx, h); prod1(o, cf(1.f), mat(a->wv, a->ld_wv), mat(a->G, h), h); rank1(o, cf(1.f), a->bv, 1, a->s, 1); }
        { Op& o = bb.add(m, 1, a->z1, 1); prod1(o, cf(1.f), mat(a->wk, a->ld_wk), vec(a->s), h); rank1(o, cf(1.f), a->bk, 1, scN, 0); }
        { Op& o = bb.add(m, 1, a->q1, 1); prod1(o, cf(1.f), mat(a->wq, a->ld_wq), vec(a->s), h); rank1(o, cf(1.f), a->bq, 1, scN, 0); }
        { Op& o = bb.add(d, 1, a->v1, 1); prod1(o, cf(1.f), mat(a->wv, a->ld_wv), vec(a->s), h); rank1(o, cf(1.f), a->bv, 1, scN, 0); }
        if ((rc = bb.launch(st))) return rc;
    }
    {   // level 2: S = k^T v and the two squared norms
        BatchBuilder bb;
        { Op& o = bb.add(m, d, a->S, d); prod1(o, cf(1.f), mat(a->kx, h), matT(a->wv, a->ld_wv), h); rank1(o, cf(1.f), a->z1, 1, a->bv, 1); }
        if ((rc = bb.launch(st))) return rc;
        DotBuilder db(part);
        db.add(mat(a->kx, h), mat(a->wk, a->ld_wk), m, h);
        db.add(vec(a->z1), vec(a->bk), m, 1);
        db.add(mat(a->qx, h), mat(a->wq, a->ld_wq), m, h);
        db.add(vec(a->q1), vec(a->bq), m, 1);
        db.add(vec(a->z1), vec(a->bq), m, 1);
        if ((rc = db.launch(st))) return rc;
    }
    scal_fwd_kernel<<<1, 1, 0, st>>>(sc, part);
    SGF_LAUNCH_CHECK(); count_launch();
    {   // level 3: operands of the apply GEMM
        BatchBuilder bb;
        { Op& o = bb.add(d, h, a->Bt, h); prod1(o, cf(1.f, beta), matT(a->S, d), mat(a->wq, a->ld_wq), m); addend(o, cf(1.f), mat(a->wv, a->ld_wv)); }
        { Op& o = bb.add(h, 1, a->tail, 1); prod1(o, cf(1.f, beta), matT(a->wq, a->ld_wq), vec(a->z1), m); }
        { Op& o = bb.add(d, 1, a->bt, 1); prod1(o, cf(1.f, beta), matT(a->S, d), vec(a->bq), m); addend(o, cf(1.f), vec(a->bv)); }
        if ((rc = bb.launch(st))) return rc;
    }
    return SGF_OK;
}

extern "C" int sgf_attn_gram_prepare_bwd(const sgf_attn_gram_args* a, void* stream) {
    if (!args_ok(a) || !a->P || !a->pg || !a->cs || !a->sg || !a->dwq || !a->dbq || !a->dwk || !a->dbk || !a->dwv || !a->dbv ||
        !a->bcat || !a->a4 || !a->ws)
        return SGF_ERR_ARG;
    const int h = a->h, m = a->m, d = a->d;
    int64_t need = 0;
    sgf_attn_gram_ws_floats(h, m, d, &need);
    if (a->ws_floats < need) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    float* sc = a->sc;
    const float *alpha = sc + SC_ALPHA, *beta = sc + SC_BETA, *cq = sc + SC_CQ, *ck = sc + SC_CK, *one = sc + SC_ONE;
    float* dS = a->ws;
    float* dz = dS + (int64_t)m * d;
    float* U = dz + m;
    float* t1 = U + (int64_t)m * h;
    float* t2 = t1 + m;
    float* part = a->ws + (need - MAX_OPS * DOT_SPLIT);
    const int64_t ldc = d + h;       // pitch of bcat = [Bt^T | A3]
    float* A3 = a->bcat + d;
    int rc;
    {   // level 1: dS, dz; the Bt^T half of the dx operand
        BatchBuilder bb;
        { Op& o = bb.add(m, d, dS, d); prod1(o, cf(1.f), mat(a->wq, a->ld_wq), mat(a->P, d), h); rank1(o, cf(1.f), a->bq, 1, a->cs, 1); }
        { Op& o = bb.add(m, 1, dz, 1); prod1(o, cf(1.f), mat(a->wq, a->ld_wq), vec(a->pg), h); rank1(o, cf(1.f), a->bq, 1, a->sg, 0); }
        { Op& o = bb.add(h, d, a->bcat, ldc); addend(o, cf(1.f), matT(a->Bt, h)); }
        if ((rc = bb.launch(st))) return rc;
    }
    {   // level 2: c = beta (<dS,S> + <dz,z1>);  U = dS Wv, t1 = dS bv + dz, t2 = dS^T bk
        DotBuilder db(part);
        db.add(mat(dS, d), mat(a->S, d), m, d);
        db.add(vec(dz), vec(a->z1), m, 1);
        if ((rc = db.launch(st))) return rc;
        scal_bwd_kernel<<<1, 1, 0, st>>>(sc, part);
        SGF_LAUNCH_CHECK(); count_launch();
        BatchBuilder bb;
        { Op& o = bb.add(m, h, U, h); prod1(o, cf(1.f), mat(dS, d), mat(a->wv, a->ld_wv), d); }
        { Op& o = bb.add(m, 1, t1, 1); prod1(o, cf(1.f), mat(dS, d), vec(a->bv), d); addend(o, cf(1.f), vec(dz)); }
        { Op& o = bb.add(d, 1, t2, 1); prod1(o, cf(1.f), matT(dS, d), vec(a->bk), m); }
        if ((rc = bb.launch(st))) return rc;
    }
    {   // level 3: parameter gradients; the norm-gradient part of A3 and a4
        BatchBuilder bb;
        { Op& o = bb.add(m, h, a->dwq, h); prod1(o, cf(1.f, beta), mat(a->S, d), matT(a->P, d), d); addend(o, cf(1.f, cq), mat(a->qx, h));
          rank1(o, cf(1.f, beta), a->z1, 1, a->pg, 1); }
        { Op& o = bb.add(m, 1, a->dbq, 1); prod1(o, cf(1.f, beta), mat(a->S, d), vec(a->cs), d); addend(o, cf(1.f, cq), vec(a->q1));
          rank1(o, cf(1.f, beta), a->z1, 1, a->sg, 0); }
        { Op& o = bb.add(m, h, a->dwk, h); prod1(o, cf(1.f, beta), mat(dS, d), mat(a->vx, h), d); addend(o, cf(1.f, ck), mat(a->kx, h));
          rank1(o, cf(1.f, beta), dz, 1, a->s, 1); }
        { Op& o = bb.add(m, 1, a->dbk, 1); prod1(o, cf(1.f, beta), mat(dS, d), vec(a->v1), d); addend(o, cf(1.f, ck), vec(a->z1));
          rank1(o, cf(1.f, alpha), dz, 1, one, 0); }
        { Op& o = bb.add(d, h, a->dwv, h); prod1(o, cf(1.f, beta), matT(dS, d), mat(a->kx, h), m); addend(o, cf(1.f), matT(a->P, d)); }
        { Op& o = bb.add(d, 1, a->dbv, 1); prod1(o, cf(1.f, beta), matT(dS, d), vec(a->z1), m); addend(o, cf(1.f), vec(a->cs)); }
        { Op& o = bb.add(h, h, A3, ldc); prod1(o, cf(1.f, cq), matT(a->wq, a->ld_wq), mat(a->wq, a->ld_wq), m);
          prod2(o, cf(1.f, ck), matT(a->wk, a->ld_wk), mat(a->wk, a->ld_wk), m); }
        { Op& o = bb.add(h, 1, a->a4, 1); prod1(o, cf(1.f, cq), matT(a->wq, a->ld_wq), vec(a->bq), m);
          prod2(o, cf(1.f, ck), matT(a->wk, a->ld_wk), vec(a->bk), m); }
        if ((rc = bb.launch(st))) return rc;
    }
    {   // level 4: A3 += beta (Wk^T U + U^T Wk),  a4 += beta (Wk^T t1 + Wv^T t2)     (E aliases C: read-then-write per element)
        BatchBuilder bb;
        { Op& o = bb.add(h, h, A3, ldc); prod1(o, cf(1.f, beta), matT(a->wk, a->ld_wk), mat(U, h), m);
          prod2(o, cf(1.f, beta), matT(U, h), mat(a->wk, a->ld_wk), m); addend(o, cf(1.f), mat(A3, ldc)); }
        { Op& o = bb.add(h, 1, a->a4, 1); prod1(o, cf(1.f, beta), matT(a->wk, a->ld_wk), vec(t1), m);
          prod2(o, cf(1.f, beta), matT(a->wv, a->ld_wv), vec(t2), d); addend(o, cf(1.f), vec(a->a4)); }
        if ((rc = bb.launch(st))) return rc;
    }
    return SGF_OK;
}
