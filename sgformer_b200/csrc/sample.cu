// K11 — neighbour sampling of the 100M variant's mini-batches on the device (replaces PyG NeighborLoader(num_neighbors=[15, 10, 5],
// batch_size=1000, shuffle=True) of 100M/nb-sample.py:125-150 and its host workers, relabelling and host->device copy).
//
// One batch, per hop t with fan-out k_t (DESIGN.md §4.15):
//   sample  : one warp per frontier row v draws min(k_t, deg v) distinct entry positions of v's parent CSR row with Floyd's
//             algorithm (k_t = -1: every entry, at most `width` of them), kept sorted by insertion, and writes the entries' global
//             source ids into the row's `width` slots and the count into rowlen[local id of v]
//   relabel : every drawn slot claims its node with atomicMin of its flat key (hop, frontier position, slot) in the per-node int32
//             map; the winners (map == own key) are scanned in key order into new local ids, the map then holds the local id, and
//             the slots are rewritten to local ids.  Local ids of earlier nodes are below every key of later hops, so they are never
//             claimed again: no ordering between threads decides anything
//   edges   : an exclusive scan of rowlen (indexed by local target id) places every drawn slot in the batch's edge list, ordered by
//             (target, slot); the tail up to the static capacity gets padding edges (each its own self loop on a node past every
//             real one) so that sgf_csr_build can run on the fixed-size list; the touched map entries are reset to -1
// Every draw is a pure function of (seed, hop, global target id, draw index): the result does not depend on the launch geometry.
#include "common.cuh"
#include "launch_count.h"
#include "../../include/sgformer_b200.h"

namespace sgf {

constexpr int kNsThreads = 256;
constexpr int kNsScanThreads = 512;
constexpr int kNsScanItems = 8;     // per thread -> 4096 per block
constexpr int64_t kNsScanTile = (int64_t)kNsScanThreads * kNsScanItems;

__device__ __forceinline__ uint64_t fmix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
    x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
    x ^= x >> 33;
    return x;
}
// draw i of hop `hop` at target v (tests/neighbor_sample_ref.py restates it)
__device__ __forceinline__ uint64_t ns_draw(uint64_t seed, int hop, int64_t v, int64_t i) {
    const uint64_t h = fmix64(seed ^ ((uint64_t)v * 0x9E3779B97F4A7C15ULL));
    return fmix64(h ^ ((((uint64_t)hop << 32) | (uint64_t)i) * 0xC2B2AE3D27D4EB4FULL));
}

// ---- sample: one warp per frontier row ----------------------------------------------------------------------------------------
// Floyd's algorithm for `k` distinct positions of [0, deg): for j = deg-k .. deg-1 draw t uniform in [0, j]; take t, or j when t is
// taken already.  The taken set lives in the row's own slots, sorted (insertion at the rank of t), so membership and the final
// ascending order come from one ballot pass over the set per draw.  Only k positions are touched, whatever the row's length.
__global__ void __launch_bounds__(kNsThreads) ns_sample_kernel(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                             const int64_t* __restrict__ idx, const int64_t* __restrict__ bounds,
                                                             int64_t frontier_cap, int k, int width, int hop, uint64_t seed,
                                                             int32_t* cand, int32_t* __restrict__ rowlen,
                                                             unsigned long long* __restrict__ need) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t f0 = bounds[0];
    int64_t nf = bounds[1] - f0;
    if (nf > frontier_cap) nf = frontier_cap;
    for (int64_t i = warp; i < nf; i += nwarps) {
        const int64_t v = idx[f0 + i];
        const int64_t s = rowptr[v];
        const int64_t deg = rowptr[v + 1] - s;
        int32_t* out = cand + i * (int64_t)width;
        int64_t m;
        if (k < 0 || deg <= k) {
            m = deg < width ? deg : width;
            if (k < 0 && deg > width && lane == 0 && need) atomicMax(need, (unsigned long long)deg);
            for (int64_t p = lane; p < m; p += 32) out[p] = col[s + p];
        } else {
            m = k;
            for (int d = 0; d < k; ++d) {
                const int64_t j = deg - k + d;
                const uint64_t h = ns_draw(seed, hop, v, d);
                const int32_t t = (int32_t)(((h >> 32) * (uint64_t)(j + 1)) >> 32);
                int lt = 0;
                bool hit = false;
                for (int base = 0; base < d; base += 32) {
                    const int e = base + lane < d ? out[base + lane] : INT32_MAX;
                    lt += __popc(__ballot_sync(0xffffffffu, e < t));
                    hit |= __any_sync(0xffffffffu, e == t);
                }
                if (hit) {                       // j is above every taken position: append
                    if (lane == 0) out[d] = (int32_t)j;
                } else {                         // shift [lt, d) up by one, top chunk first, then insert t
                    for (int top = d; top > lt; top -= 32) {
                        const int p = top - 1 - lane;
                        const int e = p >= lt ? out[p] : 0;
                        __syncwarp();
                        if (p >= lt) out[p + 1] = e;
                        __syncwarp();
                    }
                    if (lane == 0) out[lt] = t;
                }
                __syncwarp();
            }
            for (int p = lane; p < k; p += 32) out[p] = col[s + out[p]];
        }
        if (lane == 0) rowlen[f0 + i] = (int32_t)m;
    }
}

// ---- exclusive scan of int32 counts into int64 offsets (3 kernels) ----------------------------------------------------------------
__device__ __forceinline__ int64_t ns_block_excl(int64_t tsum, int64_t* warp_tot, int64_t& block_total) {
    const int tid = threadIdx.x;
    int64_t x = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if ((tid & 31) >= o) x += y;
    }
    if ((tid & 31) == 31) warp_tot[tid >> 5] = x;
    __syncthreads();
    if (tid < 32) {
        int64_t w = tid < (int)(blockDim.x >> 5) ? warp_tot[tid] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t y = __shfl_up_sync(0xffffffffu, w, o);
            if (tid >= o) w += y;
        }
        warp_tot[tid] = w;
    }
    __syncthreads();
    block_total = warp_tot[31];
    const int64_t r = x - tsum + ((tid >> 5) > 0 ? warp_tot[(tid >> 5) - 1] : 0);
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(kNsScanThreads) ns_scan_reduce_kernel(const int32_t* __restrict__ in, int64_t n,
                                                                       int64_t* __restrict__ bsum) {
    __shared__ int64_t warp_tot[32];
    const int64_t base = (int64_t)blockIdx.x * kNsScanTile + (int64_t)threadIdx.x * kNsScanItems;
    int64_t t = 0;
#pragma unroll
    for (int i = 0; i < kNsScanItems; ++i) t += base + i < n ? in[base + i] : 0;
    int64_t tot;
    ns_block_excl(t, warp_tot, tot);
    if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}

// single block of 1024: exclusive scan of the block sums in place, plus *base (nullable); *total = *base + sum
__global__ void __launch_bounds__(1024) ns_scan_bsum_kernel(int64_t* __restrict__ bsum, int64_t nb, const int64_t* base,
                                                          int64_t* total) {
    __shared__ int64_t warp_tot[32];
    int64_t carry = base ? *base : 0;
    for (int64_t b0 = 0; b0 < nb; b0 += 1024) {
        const int64_t i = b0 + threadIdx.x;
        const int64_t v = i < nb ? bsum[i] : 0;
        int64_t tot;
        const int64_t e = ns_block_excl(v, warp_tot, tot);
        if (i < nb) bsum[i] = carry + e;
        carry += tot;
    }
    if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(kNsScanThreads) ns_scan_apply_kernel(const int32_t* __restrict__ in, int64_t n,
                                                                      const int64_t* __restrict__ bsum, int64_t* __restrict__ out) {
    __shared__ int64_t warp_tot[32];
    const int64_t base = (int64_t)blockIdx.x * kNsScanTile + (int64_t)threadIdx.x * kNsScanItems;
    int64_t v[kNsScanItems];
    int64_t t = 0;
#pragma unroll
    for (int i = 0; i < kNsScanItems; ++i) {
        v[i] = base + i < n ? in[base + i] : 0;
        t += v[i];
    }
    int64_t tot;
    int64_t e = ns_block_excl(t, warp_tot, tot) + bsum[blockIdx.x];
#pragma unroll
    for (int i = 0; i < kNsScanItems; ++i) {
        if (base + i < n) out[base + i] = e;
        e += v[i];
    }
}

// ---- relabel ------------------------------------------------------------------------------------------------------------------
// slot q = i * width + s of the hop's frontier row i is drawn when i < frontier size and s < rowlen[f0 + i]
__device__ __forceinline__ bool ns_slot(const int64_t* bounds, const int32_t* rowlen, int64_t frontier_cap, int width, int64_t q,
                                        int64_t& row) {
    row = q / width;
    const int64_t f0 = bounds[0];
    return row < frontier_cap && row < bounds[1] - f0 && (q - row * width) < rowlen[f0 + row];
}

__global__ void ns_claim_kernel(const int32_t* __restrict__ cand, const int32_t* __restrict__ rowlen, const int64_t* __restrict__ bounds,
                                int64_t frontier_cap, int width, int64_t key_base, int32_t* __restrict__ node_map) {
    const int64_t slots = frontier_cap * width, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += stride) {
        int64_t row;
        // unsigned: an unclaimed entry (-1) is above every key, a local id of an earlier node below every key of this hop
        if (ns_slot(bounds, rowlen, frontier_cap, width, q, row))
            atomicMin(reinterpret_cast<unsigned int*>(&node_map[cand[q]]), (unsigned int)(key_base + q));
    }
}

__global__ void ns_flag_kernel(const int32_t* __restrict__ cand, const int32_t* __restrict__ rowlen, const int64_t* __restrict__ bounds,
                               int64_t frontier_cap, int width, int64_t key_base, const int32_t* __restrict__ node_map,
                               int32_t* __restrict__ flags) {
    const int64_t slots = frontier_cap * width, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += stride) {
        int64_t row;
        flags[q] = ns_slot(bounds, rowlen, frontier_cap, width, q, row) && node_map[cand[q]] == (int32_t)(key_base + q);
    }
}

// winners take local id pos[q] (the scan already holds the hop's first new id); idx is bounded by max_nodes
__global__ void ns_assign_kernel(const int32_t* __restrict__ cand, const int32_t* __restrict__ flags, const int64_t* __restrict__ pos,
                                 int64_t slots, int64_t max_nodes, int32_t* __restrict__ node_map, int64_t* __restrict__ idx) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += stride) {
        if (!flags[q]) continue;
        const int64_t u = pos[q];
        if (u >= max_nodes) continue;
        node_map[cand[q]] = (int32_t)u;
        idx[u] = cand[q];
    }
}

__global__ void ns_rewrite_kernel(int32_t* cand, const int32_t* __restrict__ rowlen, const int64_t* __restrict__ bounds,
                                  int64_t frontier_cap, int width, const int32_t* __restrict__ node_map) {
    const int64_t slots = frontier_cap * width, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += stride) {
        int64_t row;
        if (ns_slot(bounds, rowlen, frontier_cap, width, q, row)) cand[q] = node_map[cand[q]];
    }
}

// ---- begin / edges / finish ------------------------------------------------------------------------------------------------------
__global__ void ns_begin_kernel(const int64_t* __restrict__ seeds, int64_t b, int32_t* __restrict__ node_map, int64_t* __restrict__ idx,
                                int64_t* __restrict__ bounds) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < b; i += stride) {
        idx[i] = seeds[i];
        node_map[seeds[i]] = (int32_t)i;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { bounds[0] = 0; bounds[1] = b; }
}

__global__ void ns_emit_kernel(const int32_t* __restrict__ cand, const int32_t* __restrict__ rowlen, const int64_t* __restrict__ bounds,
                               int64_t frontier_cap, int width, const int64_t* __restrict__ off, int64_t max_edges,
                               int64_t* __restrict__ edge_index) {
    const int64_t slots = frontier_cap * width, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += stride) {
        int64_t row;
        if (!ns_slot(bounds, rowlen, frontier_cap, width, q, row)) continue;
        const int64_t u = bounds[0] + row;
        const int64_t p = off[u] + (q - row * width);
        if (p >= max_edges) continue;
        edge_index[p] = cand[q];
        edge_index[max_edges + p] = u;
    }
}

// padding edges (max_nodes + p, max_nodes + p) after the real ones; the touched map entries back to -1; counts = (nodes, edges)
__global__ void ns_finish_kernel(const int64_t* __restrict__ idx, const int64_t* __restrict__ bounds_end, int64_t max_nodes,
                                 int64_t max_edges, int32_t* __restrict__ node_map, int64_t* __restrict__ edge_index,
                                 int64_t* __restrict__ counts) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t nn = *bounds_end < max_nodes ? *bounds_end : max_nodes;
    const int64_t ne = counts[1];
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < max_edges || p < nn; p += stride) {
        if (p < nn) node_map[idx[p]] = -1;
        if (p < max_edges && p >= ne) edge_index[p] = edge_index[max_edges + p] = max_nodes + p;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) counts[0] = nn;
}

static inline int ns_grid(int64_t work, int block) {
    int64_t g = (work + block - 1) / block;
    const int64_t cap = (int64_t)num_sms() * 8;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}
static inline size_t ns_align(size_t x) { return (x + 255) / 256 * 256; }

// workspace: flags int32[max(slots, nodes)] | pos int64[max(slots, nodes)] | block sums int64[tiles + 1]
struct NsWs { int32_t* flags; int64_t* pos; int64_t* bsum; size_t bytes; };
static NsWs ns_carve(void* ws, int64_t max_slots, int64_t max_nodes) {
    const int64_t m = (max_slots > max_nodes ? max_slots : max_nodes) + 1;
    const int64_t nb = (m + kNsScanTile - 1) / kNsScanTile + 1;
    NsWs w;
    char* b = (char*)ws;
    const size_t o_pos = ns_align((size_t)m * 4), o_bs = o_pos + ns_align((size_t)m * 8);
    w.flags = (int32_t*)b; w.pos = (int64_t*)(b + o_pos); w.bsum = (int64_t*)(b + o_bs);
    w.bytes = o_bs + ns_align((size_t)nb * 8);
    return w;
}

static int ns_scan(const int32_t* in, int64_t n, int64_t* out, const int64_t* base, int64_t* total, int64_t* bsum, cudaStream_t st) {
    const int64_t nb = n > 0 ? (n + kNsScanTile - 1) / kNsScanTile : 1;
    ns_scan_reduce_kernel<<<(unsigned)nb, kNsScanThreads, 0, st>>>(in, n, bsum);
    SGF_LAUNCH_CHECK(); count_launch();
    ns_scan_bsum_kernel<<<1, 1024, 0, st>>>(bsum, nb, base, total);
    SGF_LAUNCH_CHECK(); count_launch();
    ns_scan_apply_kernel<<<(unsigned)nb, kNsScanThreads, 0, st>>>(in, n, bsum, out);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

}  // namespace sgf

using namespace sgf;

extern "C" int sgf_neighbor_sample_ws_bytes(int64_t max_slots, int64_t max_nodes, size_t* bytes) {
    if (!bytes || max_slots < 0 || max_nodes < 0) return SGF_ERR_ARG;
    *bytes = ns_carve(nullptr, max_slots, max_nodes).bytes;
    return SGF_OK;
}

extern "C" int sgf_neighbor_begin(const int64_t* seeds, int64_t b, int32_t* node_map, int64_t* idx, int64_t* bounds,
                                  int32_t* rowlen, int64_t max_nodes, void* stream) {
    if (b < 0 || b > max_nodes || !node_map || !idx || !bounds || !rowlen || (b > 0 && !seeds)) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (max_nodes > 0) SGF_CUDA_TRY(cudaMemsetAsync(rowlen, 0, (size_t)max_nodes * 4, st));
    ns_begin_kernel<<<ns_grid(b, kNsThreads), kNsThreads, 0, st>>>(seeds, b, node_map, idx, bounds);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_neighbor_sample_hop(const int64_t* rowptr, const int32_t* col, const int64_t* idx, const int64_t* bounds,
                                       int64_t frontier_cap, int k, int width, int hop, uint64_t seed, int32_t* cand,
                                       int32_t* rowlen, int64_t* need, void* stream) {
    if (!rowptr || !idx || !bounds || !cand || !rowlen || frontier_cap < 0 || width < 0 || hop < 0) return SGF_ERR_ARG;
    if ((k >= 0 && width != k) || k < -1) return SGF_ERR_ARG;
    if (frontier_cap == 0 || width == 0) return SGF_OK;
    ns_sample_kernel<<<ns_grid(frontier_cap * 32, kNsThreads), kNsThreads, 0, (cudaStream_t)stream>>>(
        rowptr, col, idx, bounds, frontier_cap, k, width, hop, seed, cand, rowlen, (unsigned long long*)need);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_neighbor_relabel(int32_t* cand, const int32_t* rowlen, int64_t* bounds, int64_t frontier_cap, int width,
                                    int64_t key_base, int64_t max_nodes, int32_t* node_map, int64_t* idx, void* ws, size_t ws_bytes,
                                    void* stream) {
    if (!cand || !rowlen || !bounds || !node_map || !idx || !ws || frontier_cap < 0 || width < 0 || key_base < 0) return SGF_ERR_ARG;
    const int64_t slots = frontier_cap * width;
    if (key_base + slots > (int64_t)INT32_MAX) return SGF_ERR_UNSUPPORTED;
    NsWs w = ns_carve(ws, slots, 0);
    if (ws_bytes < w.bytes) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    if (slots == 0) return cudaMemcpyAsync(bounds + 2, bounds + 1, 8, cudaMemcpyDeviceToDevice, st);
    const int g = ns_grid(slots, kNsThreads);
    ns_claim_kernel<<<g, kNsThreads, 0, st>>>(cand, rowlen, bounds, frontier_cap, width, key_base, node_map);
    SGF_LAUNCH_CHECK(); count_launch();
    ns_flag_kernel<<<g, kNsThreads, 0, st>>>(cand, rowlen, bounds, frontier_cap, width, key_base, node_map, w.flags);
    SGF_LAUNCH_CHECK(); count_launch();
    const int rc = ns_scan(w.flags, slots, w.pos, bounds + 1, bounds + 2, w.bsum, st);
    if (rc) return rc;
    ns_assign_kernel<<<g, kNsThreads, 0, st>>>(cand, w.flags, w.pos, slots, max_nodes, node_map, idx);
    SGF_LAUNCH_CHECK(); count_launch();
    ns_rewrite_kernel<<<g, kNsThreads, 0, st>>>(cand, rowlen, bounds, frontier_cap, width, node_map);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}

extern "C" int sgf_neighbor_edges(const int32_t* cand, const int32_t* widths /* host [hops] */, int hops, int64_t batch_cap,
                                  const int64_t* bounds, const int32_t* rowlen, int64_t max_nodes, int32_t* node_map,
                                  const int64_t* idx, int64_t* edge_index, int64_t max_edges, int64_t* counts, void* ws,
                                  size_t ws_bytes, void* stream) {
    if (hops < 0 || (hops > 0 && (!cand || !widths)) || batch_cap < 0 || !bounds || !rowlen || !node_map || !idx || !counts ||
        !ws || max_nodes < 0 || max_edges < 0 || (max_edges > 0 && !edge_index))
        return SGF_ERR_ARG;
    NsWs w = ns_carve(ws, 0, max_nodes);
    if (ws_bytes < w.bytes) return SGF_ERR_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = ns_scan(rowlen, max_nodes, w.pos, nullptr, counts + 1, w.bsum, st);
    if (rc) return rc;
    int64_t fcap = batch_cap, done = 0;
    for (int t = 0; t < hops; ++t) {
        const int64_t slots = fcap * widths[t];
        if (slots > 0) {
            ns_emit_kernel<<<ns_grid(slots, kNsThreads), kNsThreads, 0, st>>>(cand + done, rowlen, bounds + t, fcap, widths[t], w.pos,
                                                                            max_edges, edge_index);
            SGF_LAUNCH_CHECK(); count_launch();
        }
        done += slots;
        fcap = slots;
    }
    const int64_t work = max_edges > max_nodes ? max_edges : max_nodes;
    ns_finish_kernel<<<ns_grid(work, kNsThreads), kNsThreads, 0, st>>>(idx, bounds + hops + 1, max_nodes, max_edges, node_map,
                                                                      edge_index, counts);
    SGF_LAUNCH_CHECK(); count_launch();
    return SGF_OK;
}
