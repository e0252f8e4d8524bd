// Gradient of the loss w.r.t. the edge weights of a weighted GCN / DIFFormer layer (DESIGN.md §4.10).
//
// A layer computes y = Â t with Â[c, r] = dis[c] w dis[r] over the CSR of sgf_csr_build_weighted (rows c = edge targets).  With
// the operands the schedule already holds in pre-scaled form, a = dis (.) g (g = dL/dy) and b = dis (.) t, the entry j = (c, r) of
// the CSR, source edge eid[j], receives
//     dL/dw = <a_c, b_r> + q_c,
//     q_c   = -1/2 dis_c (<a_c, y_c> + <b_c, u_c>)       (u = Â^T g; the degree term of weighted gcn_norm, self_loop_mode 1)
// which is dis_c dis_r <g_c, t_r> - 1/2 dis_c^3 dL/ddis_c written without a division (q_c = 0 where dis_c = 0).  DIFFormer's
// gcn_conv normalises by the unweighted degree: no degree term (y = u = NULL).
//
// One warp per row; a row's operand a_c stays in registers while the warp walks the row's entries, gathering b_r like the SpMM.
// Every non-loop edge is one CSR entry, so `out[eid]` is written by one thread of one launch: no atomics, deterministic.  The added
// self loop of a self_loop_mode 1 row has no edge of its own; its gradient goes to loop_grad[c], and a second pass adds it to every
// existing self loop (c, c) of node c (autograd of PyG's `loop_attr[idx] = attr`, which scatters into all of them).
#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

namespace sgf {

constexpr int kEdgeGradMaxPerLane = 16;     // h <= 512

template <typename T>
__global__ void __launch_bounds__(256) edge_weight_grad_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                               const int64_t* __restrict__ eid, int64_t n_rows, int h,
                                                               const T* __restrict__ a, int64_t lda, const T* __restrict__ b,
                                                               int64_t ldb, const T* __restrict__ y, int64_t ldy,
                                                               const T* __restrict__ u, int64_t ldu, const float* __restrict__ dinv,
                                                               float* __restrict__ loop_grad, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t c = warp0; c < n_rows; c += nwarps) {
        float ac[kEdgeGradMaxPerLane];
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < kEdgeGradMaxPerLane; ++k) {
            const int f = lane + 32 * k;
            ac[k] = f < h ? to_f32(a[c * lda + f]) : 0.f;
        }
        if (y) {
            float d = 0.f;
#pragma unroll
            for (int k = 0; k < kEdgeGradMaxPerLane; ++k) {
                const int f = lane + 32 * k;
                if (f < h) d += ac[k] * to_f32(y[c * ldy + f]) + to_f32(b[c * ldb + f]) * to_f32(u[c * ldu + f]);
            }
            q = -0.5f * dinv[c] * warp_sum(d);
        }
        for (int64_t j = rowptr[c]; j < rowptr[c + 1]; ++j) {
            const int64_t r = col[j];
            const T* br = b + r * ldb;
            float d = 0.f;
#pragma unroll
            for (int k = 0; k < kEdgeGradMaxPerLane; ++k) {
                const int f = lane + 32 * k;
                if (f < h) d += ac[k] * to_f32(br[f]);
            }
            d = warp_sum(d) + q;
            if (lane == 0) {
                if (loop_grad && r == c) loop_grad[c] = d;
                else if (eid[j] >= 0) out[eid[j]] += d;
            }
        }
    }
}

// out[e] += loop_grad[i] for every self-loop edge e = (i, i)
__global__ void edge_weight_grad_loops_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ dst, int64_t nnz,
                                              const float* __restrict__ loop_grad, float* __restrict__ out) {
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        const int64_t r = src[e];
        if (r == dst[e]) out[e] += loop_grad[r];
    }
}

static inline int grid_for(int64_t work, int block) {
    int64_t g = (work + block - 1) / block;
    int64_t cap = (int64_t)num_sms() * 8;
    return (int)(g < 1 ? 1 : g > cap ? cap : g);
}

template <typename T>
static int launch_edge_grad(const int64_t* rowptr, const int32_t* col, const int64_t* eid, int64_t n_rows, int h, const void* a,
                            int64_t lda, const void* b, int64_t ldb, const void* y, int64_t ldy, const void* u, int64_t ldu,
                            const float* dinv, float* loop_grad, float* out, cudaStream_t st) {
    edge_weight_grad_kernel<T><<<grid_for(n_rows * 32, 256), 256, 0, st>>>(
        rowptr, col, eid, n_rows, h, static_cast<const T*>(a), lda, static_cast<const T*>(b), ldb, static_cast<const T*>(y), ldy,
        static_cast<const T*>(u), ldu, dinv, loop_grad, out);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

}  // namespace sgf

extern "C" int sgf_edge_weight_grad(const int64_t* rowptr, const int32_t* col, const int64_t* eid, int64_t n_rows, int h, int dtype,
                                    const void* a, int64_t lda, const void* b, int64_t ldb, const void* y, int64_t ldy, const void* u,
                                    int64_t ldu, const float* dinv, const int64_t* edge_index, int64_t nnz, float* loop_grad,
                                    float* out, void* stream) {
    if (!rowptr || n_rows < 0 || h <= 0 || h > 32 * sgf::kEdgeGradMaxPerLane || nnz < 0 || (nnz > 0 && !out)) return SGF_ERR_ARG;
    if (n_rows > 0 && (!col || !eid || !a || !b)) return SGF_ERR_ARG;
    if (y && (!u || !dinv)) return SGF_ERR_ARG;
    if (loop_grad && nnz > 0 && !edge_index) return SGF_ERR_ARG;
    if (n_rows == 0) return SGF_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if (dtype == 0) rc = sgf::launch_edge_grad<float>(rowptr, col, eid, n_rows, h, a, lda, b, ldb, y, ldy, u, ldu, dinv, loop_grad, out, st);
    else if (dtype == 1)
        rc = sgf::launch_edge_grad<__nv_bfloat16>(rowptr, col, eid, n_rows, h, a, lda, b, ldb, y, ldy, u, ldu, dinv, loop_grad, out, st);
    else return SGF_ERR_ARG;
    if (rc || !loop_grad || nnz == 0) return rc;
    sgf::edge_weight_grad_loops_kernel<<<sgf::grid_for(nnz, 256), 256, 0, st>>>(edge_index, edge_index + nnz, nnz, loop_grad, out);
    SGF_LAUNCH_CHECK(); sgf::count_launch();
    return SGF_OK;
}
