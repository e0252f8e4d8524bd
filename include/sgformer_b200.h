/* sgformer_b200 — C-ABI of the H100 (sm_90a) SGFormer encoder hot path.
 *
 * The reference (qitianwu/SGFormer) has no FFI: its hot path is `ours.py` calling torch / torch_sparse /
 * torch_geometric ops.  Each entry point below replaces one of those call sites (cited per function,
 * paths relative to the reference root).  Conventions:
 *   - plain pointers + sizes, no torch types; every pointer is DEVICE memory unless marked host;
 *   - `stream` is a cudaStream_t passed as void*; launchers never synchronise and never allocate
 *     (workspaces are passed in; *_ws_bytes tells the size);
 *   - sums across thread blocks are deterministic (fixed order, no float atomics): a result is bit-identical
 *     from run to run.  The launchers that sum columns or a loss across blocks (sgf_colstats, sgf_ln_bwd,
 *     sgf_ln_bwd_attn, sgf_bn_bwd_reduce(_jk), sgf_bn_bwd_apply(_jk), sgf_pack_operand with colsum, sgf_softmax_nll)
 *     take a device workspace `ws` of at least sgf_reduce_ws_bytes(width) bytes (16-byte aligned; width = h,
 *     cols, or 1 for the loss) that holds the blocks' partials and arrival counters; the launcher resets the
 *     counters on `stream`.  Calls whose kernels may run at the same time need distinct workspaces;
 *   - return 0 on success, a positive cudaError_t, or a negative SGF_ERR_* argument error;
 *   - dtype codes: SGF_F32 = 0 (float), SGF_BF16 = 1 (__nv_bfloat16); matrices are row-major with an
 *     explicit leading dimension in ELEMENTS; feature rows must be 16-byte aligned and have a
 *     16-byte-multiple pitch;
 *   - node ids fit int32; rowptr is int64 (nnz of a papers100M-scale graph exceeds 2^31).
 * There is no CPU implementation behind this header and no fallback: without a CUDA device every
 * compute entry point fails with the CUDA error.
 */
#ifndef SGFORMER_B200_H
#define SGFORMER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SGF_F32 0
#define SGF_BF16 1

#define SGF_ERR_ARG (-1)
#define SGF_ERR_UNSUPPORTED (-2)
#define SGF_ERR_DRIVER (-3)

/* library / build info: "sgformer_b200 <version> sm_90a" (host string, static storage) */
const char* sgf_version(void);
/* number of kernels this library has launched since load (host counter; bench.py's gpu_launches) */
int64_t sgf_launch_count(void);
/* select the CUDA device for subsequent launches of the calling thread (the library carries its own static CUDA
 * runtime; the host framework's cudaSetDevice does not reach it).  Returns a cudaError_t. */
int sgf_set_device(int device);

/* ------------------------------------------------------------------------------------------------
 * K5 — graph structure (replaces, per GraphConvLayer.forward call, large/ours.py:26-33:
 *   PyG degree() + per-edge weights + torch_sparse.SparseTensor(row=col, col=row) i.e. argsort of
 *   target*N+source and rowptr build; hoisted here to once per graph).
 * Builds the CSR of the aggregation pattern: by_source = 0 -> rows = edge targets (edge_index[1]),
 * columns = sources; by_source = 1 -> the transpose (used by the backward, large/ours.py autograd of :34).
 * Entries of a row are sorted by column, duplicates kept  => rowptr/col are bit-exact with the
 * reference's SparseTensor storage.
 * self_loop_mode 0: edges as given (large/100M GraphConv).  1: PyG gcn_norm semantics
 * (medium/models.py:22-37 GCNConv): existing self loops dropped, one self loop per node added.
 * dinv (nullable, by_source = 0 only): dinv[i] = sqrt(1/len(row i)) or 0 for empty rows
 * (== (1/d).sqrt() with nan_to_num -> 0, large/ours.py:29-32).
 * col must hold nnz (+ n when self_loop_mode = 1) entries; the true count is rowptr[n].
 * Every node id of edge_index must lie in [0, n) (n_cols for the row shard below): an id outside it is the caller's error.
 * The kernels skip such an edge, so rowptr[n] falls short of nnz and col's tail is left unwritten; kernels.csr_build,
 * csr_build_weighted and to_undirected refuse such an edge list with a ValueError before they launch.
 * ------------------------------------------------------------------------------------------------ */
int sgf_csr_build_ws_bytes(int64_t nnz, int64_t n, size_t* bytes /* host out */);
int sgf_csr_build(const int64_t* edge_index /* [2,nnz] */, int64_t nnz, int64_t n, int by_source,
                  int self_loop_mode, int64_t* rowptr /* [n+1] */, int32_t* col, float* dinv /* [n] or NULL */,
                  void* ws, size_t ws_bytes, void* stream);
/* Row shard of the same CSR: only rows [row_begin, row_end) of the n_cols x n_cols pattern are built (local row =
 * global row - row_begin), column ids stay global.  Used when the nodes are row-sharded across GPUs (SURVEY.md §8e):
 * every rank builds its own rows from the full edge list.  ws sized by sgf_csr_build_ws_bytes(nnz, row_end-row_begin). */
int sgf_csr_build_rect(const int64_t* edge_index, int64_t nnz, int64_t row_begin, int64_t row_end, int64_t n_cols,
                       int by_source, int self_loop_mode, int64_t* rowptr, int32_t* col, float* dinv, void* ws,
                       size_t ws_bytes, void* stream);

/* As sgf_csr_build_rect with ROTATED column ids col' = (col - col_rot) mod col_mod (col_mod >= n_cols; col_mod = 0: no rotation),
 * rows sorted by col'.  A row shard built with col_rot = row_begin, col_mod = world * ceil(n/world) has its own row block first in
 * every row, then the blocks of rank+1, rank+2, ...: the order in which sgf_spmm_flagged consumes the operand blocks that the
 * peers push over NVLink (slot s of the gathered buffer = block of rank (rank + s) mod world). */
int sgf_csr_build_rot(const int64_t* edge_index, int64_t nnz, int64_t row_begin, int64_t row_end, int64_t n_cols, int by_source,
                      int self_loop_mode, int64_t col_rot, int64_t col_mod, int64_t* rowptr, int32_t* col, float* dinv, void* ws,
                      size_t ws_bytes, void* stream);

/* K9 — induced subgraph with relabelling (replaces PyG subgraph(idx, edge_index, num_nodes=n,
 * relabel_nodes=True) at large/main-batch.py:139 / large/eval.py:89): keeps edges whose endpoints are
 * both in `subset` and maps node ids to positions in `subset`.  Output order = input edge order
 * (bit-exact with the reference).  node_map: int32 [n] workspace; out_count: device int64 scalar. */
int sgf_subgraph(const int64_t* edge_index, int64_t nnz, int64_t n, const int64_t* subset, int64_t n_sub,
                 int32_t* node_map, int64_t* out_edge_index /* [2,nnz] capacity, pitch nnz */,
                 int64_t* out_count, void* ws, size_t ws_bytes, void* stream);
int sgf_subgraph_ws_bytes(int64_t nnz, int64_t n, size_t* bytes);

/* K10 — graph preprocessing on the device (SURVEY.md §8f-2), bit-exact with torch_geometric 1.7.2 as the reference calls it:
 *   to_undirected(edge_index)                 large/main.py:76, medium/main.py:94   = coalesce([ei | ei.flip(0)]): every edge
 *                                             in both directions, sorted by (row, col), duplicates removed;
 *   remove_self_loops(edge_index)             large/main.py:78, large/main-batch.py:97: drops row == col, keeps the order;
 *   add_self_loops(edge_index, num_nodes=n)   large/main.py:79, large/main-batch.py:98: appends (i, i), i = 0..n-1.
 * edge_index: int64 [2, nnz] row-major (row r at edge_index + r*nnz).  Outputs are int64 [2, capacity] with the pitch stated
 * per function; out_count is a device int64 scalar (valid prefix length of each output row). */
int sgf_to_undirected_ws_bytes(int64_t nnz, int64_t n, size_t* bytes);
int sgf_to_undirected(const int64_t* edge_index, int64_t nnz, int64_t n, int64_t* out_edge_index /* pitch 2*nnz */,
                      int64_t* out_count, void* ws, size_t ws_bytes, void* stream);
int sgf_remove_self_loops_ws_bytes(int64_t nnz, size_t* bytes);
int sgf_remove_self_loops(const int64_t* edge_index, int64_t nnz, int64_t* out_edge_index /* pitch nnz */, int64_t* out_count,
                          void* ws, size_t ws_bytes, void* stream);
int sgf_add_self_loops(const int64_t* edge_index, int64_t nnz, int64_t n, int64_t* out_edge_index /* [2, nnz+n], pitch nnz+n */,
                       void* stream);
/* Is the edge multiset symmetric ({(r,c)} == {(c,r)})?  out2[0], out2[1] (device) receive order-independent 64-bit hash sums of
 * the two multisets; equal sums <=> symmetric (2^-64 collision odds).  One pass over edge_index.  Decides whether the backward
 * SpMM (A^T, autograd of torch_sparse.matmul, large/ours.py:33) can reuse the forward CSR. */
int sgf_edge_symmetry(const int64_t* edge_index, int64_t nnz, int64_t n, uint64_t* out2, void* stream);
/* Weighted graphs (edge_weight of the medium GCN / DIFFormer, DESIGN.md §4.10).  The CSR of sgf_csr_build (n x n, by_source,
 * self_loop_mode as there) plus, per entry j: eid[j] (int64) = position of the source edge in edge_index, val[j] = weight[eid[j]]
 * (fp32).  Rows are sorted by (col, eid).  self_loop_mode 1 (PyG gcn_norm(add_self_loops=True)): existing self loops are
 * dropped and node i's added loop takes the weight of i's LAST self loop in edge order (eid = its position), or 1 when i has none
 * (eid = -1).  dinv (nullable): mode 1 -> deg[i]^-1/2 with deg[i] = sum of row i's values (summed in fp64 in CSR order, inf -> 0,
 * negative -> NaN); mode 0 -> the count-based dinv of sgf_csr_build (DIFFormer's gcn_conv normalises by the unweighted degree).
 * col / eid / val hold nnz (+ n in mode 1) entries.  nnz < 2^32 - 1.  ws sized by sgf_csr_build_weighted_ws_bytes(nnz, n). */
int sgf_csr_build_weighted_ws_bytes(int64_t nnz, int64_t n, size_t* bytes /* host out */);
int sgf_csr_build_weighted(const int64_t* edge_index, const float* weight /* [nnz] */, int64_t nnz, int64_t n, int by_source,
                           int self_loop_mode, int64_t* rowptr, int32_t* col, int64_t* eid, float* val, float* dinv /* or NULL */,
                           void* ws, size_t ws_bytes, void* stream);
/* sgf_edge_symmetry over the weighted multisets {(r, c, w)} and {(c, r, w)} (the weight's bit pattern is hashed along): equal
 * sums <=> the transposed weighted CSR equals the forward one and can share its storage. */
int sgf_edge_symmetry_weighted(const int64_t* edge_index, const float* weight, int64_t nnz, int64_t n, uint64_t* out2, void* stream);
/* Gradient of a weighted layer y = Â t (Â[c,r] = dinv[c] val[j] dinv[r], CSR of sgf_csr_build_weighted by_source = 0) w.r.t. the
 * edge weights, ADDED into out[nnz] (fp32, one entry per edge of edge_index):  out[eid[j]] += <a_c, b_r> + q_c  for entry
 * j = (c, r), where a = dinv (.) dL/dy and b = dinv (.) t are [n_rows, h] activations (dtype 0 fp32 / 1 bf16, h <= 512), and
 * q_c = -1/2 dinv[c] (<a_c, y_c> + <b_c, u_c>) with u = Â^T dL/dy when y is non-NULL (the degree term of self_loop_mode 1; NULL
 * for DIFFormer's unweighted normalisation).  loop_grad (fp32 [n_rows], nullable): self_loop_mode 1 - the added self loop's
 * gradient is added to EVERY self-loop edge (i, i) of edge_index instead.  No atomics: deterministic. */
int sgf_edge_weight_grad(const int64_t* rowptr, const int32_t* col, const int64_t* eid, int64_t n_rows, int h, int dtype,
                         const void* a, int64_t lda, const void* b, int64_t ldb, const void* y, int64_t ldy, const void* u, int64_t ldu,
                         const float* dinv, const int64_t* edge_index, int64_t nnz, float* loop_grad, float* out, void* stream);
/* K9 on the CSR: the induced subgraph of `subset` emitted directly as the subset's own CSR (rows = subset order, columns
 * = positions in subset, sorted; dinv from the induced in-degrees) — the structure GraphConv needs for a mini-batch, in
 * O(sum of the subset rows' lengths) instead of PyG subgraph's O(E) mask per batch + a CSR rebuild.
 * node_map: int32 [n] scratch that must hold -1 everywhere on entry and is restored to -1 on exit (kept across batches).
 * out_col_capacity >= sum of the subset rows' lengths is always enough.  A smaller capacity never overruns out_col: the row
 * pointers are clamped to it (the tail rows come out truncated / empty) and *out_needed (device int64, nullable) receives the
 * induced nnz the full result needs, so the caller can detect out_needed > out_col_capacity without a sync per batch.
 * Either self-loop mode: the subset of a self_loop_mode 1 CSR equals sgf_csr_build(self_loop_mode = 1) of the subset's edge list
 * (one self loop per row, dinv of its row lengths), as the subset of a mode 0 CSR equals the mode 0 build (csr.cu, subset_half). */
int sgf_csr_subset_ws_bytes(int64_t n_sub, int64_t max_out_nnz, size_t* bytes);
int sgf_csr_subset(const int64_t* rowptr, const int32_t* col, int64_t n, const int64_t* subset, int64_t n_sub,
                   int32_t* node_map, int64_t* out_rowptr /* [n_sub+1] */, int32_t* out_col, int64_t out_col_capacity,
                   float* dinv /* [n_sub] or NULL */, int64_t* out_needed, void* ws, size_t ws_bytes, void* stream);
/* sgf_csr_subset of a directed graph: the subset of the forward CSR (rowptr, col; rows = edge targets) as above, and the subset of
 * its transpose (rowptr_t, col_t of sgf_csr_build by_source = 1; rows = edge sources) into out_rowptr_t / out_col_t, both with
 * the local ids of one fill of node_map.  The transposed half equals sgf_csr_build(by_source = 1) of the subset's edge list and
 * has no dinv.  Each half has out_col_capacity entries, is clamped on its own and reports its own induced nnz (out_needed,
 * out_needed_t; nullable).  ws sized by sgf_csr_subset_ws_bytes(n_sub, out_col_capacity), reused by the two halves in turn. */
int sgf_csr_subset_pair(const int64_t* rowptr, const int32_t* col, const int64_t* rowptr_t, const int32_t* col_t, int64_t n,
                        const int64_t* subset, int64_t n_sub, int32_t* node_map, int64_t* out_rowptr /* [n_sub+1] */,
                        int32_t* out_col, int64_t* out_rowptr_t /* [n_sub+1] */, int32_t* out_col_t, int64_t out_col_capacity,
                        float* dinv /* [n_sub] or NULL */, int64_t* out_needed, int64_t* out_needed_t, void* ws, size_t ws_bytes,
                        void* stream);

/* K11 — neighbour sampling (replaces PyG NeighborLoader(num_neighbors=[15, 10, 5], batch_size=1000) of 100M/nb-sample.py:125-150
 * with replace=False, disjoint=False; DESIGN.md §4.15).  Rows of the parent CSR (sgf_csr_build by_source = 0: rows = edge targets,
 * entries = sources) are sampled hop by hop; the batch's nodes get local ids in order of first appearance ordered by (hop, position
 * of the target in the frontier, slot), seeds first.  Buffers are sized by static bounds (batch_cap = B, hop t's frontier capacity
 * F_0 = B, F_{t+1} = F_t * width_t, width_t = k_t or, for k_t = -1, the caller's row capacity; max_nodes = B + sum F_t width_t,
 * max_edges = sum F_t width_t), so no launcher reads a size back.  bounds: device int64 [hops + 2], bounds[t] = first local id
 * of hop t's frontier (bounds[hops + 1] = node count).  node_map: int32 [n] that holds -1 everywhere between batches.
 * sgf_neighbor_begin: idx[0:b] = seeds (distinct ids in [0, n)), node_map[seeds[i]] = i, bounds[0..1] = (0, b), rowlen = 0.
 * sgf_neighbor_sample_hop: hop `hop` (bounds points at bounds[hop]): frontier row i (node v = idx[bounds[0] + i]) draws
 *   min(k, deg v) distinct entry positions of its row (Floyd's algorithm on draws fmix64(fmix64(seed ^ v*phi) ^ (hop<<32 | d)*c),
 *   see sample.cu), or takes its first min(deg, width) entries when k = -1 (deg > width: *need = max(*need, deg), nullable), and
 *   writes their source ids in ascending entry position to cand[i*width ..] and the count to rowlen[bounds[0] + i].
 * sgf_neighbor_relabel: the new nodes of the hop (bounds at bounds[hop]) take local ids from bounds[1] on in key order
 *   (key = key_base + slot, key_base = B + the slots of the earlier hops; key_base + slots < 2^31), idx[local] = global id,
 *   bounds[2] = bounds[1] + their count, and cand is rewritten to local ids.
 * sgf_neighbor_edges: edge_index [2, max_edges] (pitch max_edges) gets one edge (source local, target local) per drawn slot of all
 *   `hops` (cand = every hop's slots back to back, widths host [hops]), ordered by (target, slot), then the padding edges
 *   (max_nodes + p, max_nodes + p) up to max_edges, so that sgf_csr_build(n = max_nodes + max_edges) of the whole list equals
 *   the build of the real edges on their first max_nodes rows; node_map is reset to -1; counts[0..1] = (nodes, edges).
 * ws: sgf_neighbor_sample_ws_bytes(largest hop's F_t * width_t, max_nodes) bytes, shared by relabel and edges in stream order. */
int sgf_neighbor_sample_ws_bytes(int64_t max_slots, int64_t max_nodes, size_t* bytes /* host out */);
int sgf_neighbor_begin(const int64_t* seeds, int64_t b, int32_t* node_map, int64_t* idx /* [max_nodes] */, int64_t* bounds,
                       int32_t* rowlen /* [max_nodes] */, int64_t max_nodes, void* stream);
int sgf_neighbor_sample_hop(const int64_t* rowptr, const int32_t* col, const int64_t* idx, const int64_t* bounds, int64_t frontier_cap,
                            int k, int width, int hop, uint64_t seed, int32_t* cand /* [frontier_cap * width] */, int32_t* rowlen,
                            int64_t* need, void* stream);
int sgf_neighbor_relabel(int32_t* cand, const int32_t* rowlen, int64_t* bounds, int64_t frontier_cap, int width, int64_t key_base,
                         int64_t max_nodes, int32_t* node_map, int64_t* idx, void* ws, size_t ws_bytes, void* stream);
int sgf_neighbor_edges(const int32_t* cand, const int32_t* widths /* host [hops] */, int hops, int64_t batch_cap, const int64_t* bounds,
                       const int32_t* rowlen, int64_t max_nodes, int32_t* node_map, const int64_t* idx, int64_t* edge_index,
                       int64_t max_edges, int64_t* counts /* [2] */, void* ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K6 / K7 — CSR SpMM (replaces torch_sparse.matmul(adj, x), large/ours.py:34, 100M/ours.py:80, and its
 * autograd transpose):  y[r,:] = row_scale[r] * sum_{j in row r} x[col[j], :]   (row_scale nullable).
 * Â = D^-1/2 A D^-1/2 is applied as: producer pre-scales x rows by dinv, row_scale = dinv.
 * out_scaled (nullable): second output out_scaled[r,:] = row_scale[r] * y[r,:] is NOT written here.
 * Pure HBM-bound gather: 128-bit loads of neighbour rows, fp32 accumulation, no tensor cores.
 * ------------------------------------------------------------------------------------------------ */
int sgf_spmm(const int64_t* rowptr, const int32_t* col, const float* row_scale, const void* x, int64_t ldx,
             void* y, int64_t ldy, int64_t n_rows, int h, int dtype,
             int64_t max_row_len /* 0: all rows; > 0: rows longer than this are skipped and must be produced by sgf_spmm_heavy */,
             void* stream);
/* Hub rows of power-law graphs: the rows `heavy_rows[i]` (those longer than max_row_len) are cut into segments
 * [seg_start[s], seg_start[s] + seg_len[s]) of the col array (segments of row i: heavy_seg_ptr[i] .. heavy_seg_ptr[i+1]);
 * one warp gathers one segment into partial[s, :h] (fp32 workspace [n_seg, h]) and a second kernel adds a row's partials in
 * order (deterministic), applies row_scale and writes y[heavy_rows[i], :]. */
int sgf_spmm_heavy(const int32_t* col, const float* row_scale, const void* x, int64_t ldx, void* y, int64_t ldy, int h,
                   int dtype, const int64_t* seg_start, const int32_t* seg_len, int64_t n_seg, float* partial,
                   const int64_t* heavy_rows, const int64_t* heavy_seg_ptr, int64_t n_heavy, void* stream);
/* Weighted SpMM (CSR of sgf_csr_build_weighted):  y[r,:] = row_scale[r] * sum_{j in row r} val[j] * x[col[j], :]  (fp32
 * accumulation), and its hub-row segment path; otherwise as sgf_spmm / sgf_spmm_heavy. */
int sgf_spmm_weighted(const int64_t* rowptr, const int32_t* col, const float* val, const float* row_scale, const void* x, int64_t ldx,
                      void* y, int64_t ldy, int64_t n_rows, int h, int dtype, int64_t max_row_len, void* stream);
int sgf_spmm_heavy_weighted(const int32_t* col, const float* val, const float* row_scale, const void* x, int64_t ldx, void* y,
                            int64_t ldy, int h, int dtype, const int64_t* seg_start, const int32_t* seg_len, int64_t n_seg,
                            float* partial, const int64_t* heavy_rows, const int64_t* heavy_seg_ptr, int64_t n_heavy, void* stream);
/* Unscaled SpMM (GCNConv(normalize=False) of the large variant's GCN):  y[r,:] = sum_{j in row r} x[col[j], :]  over the CSR as
 * built (duplicates kept, no self loops added), fp32 accumulation in CSR order; no row scale is read or applied.  The hub-row
 * segment path likewise; otherwise as sgf_spmm / sgf_spmm_heavy. */
int sgf_spmm_sum(const int64_t* rowptr, const int32_t* col, const void* x, int64_t ldx, void* y, int64_t ldy, int64_t n_rows, int h,
                 int dtype, int64_t max_row_len, void* stream);
int sgf_spmm_heavy_sum(const int32_t* col, const void* x, int64_t ldx, void* y, int64_t ldy, int h, int dtype,
                       const int64_t* seg_start, const int32_t* seg_len, int64_t n_seg, float* partial, const int64_t* heavy_rows,
                       const int64_t* heavy_seg_ptr, int64_t n_heavy, void* stream);

/* ------------------------------------------------------------------------------------------------
 * K12 — GAT edge softmax (replaces PyG GATConv's message passing as medium/models.py:116-155 uses it: per-edge logits, softmax
 * over the in-edges of each target, attention dropout, weighted aggregation).  rowptr/col: the CSR of sgf_csr_build with
 * self_loop_mode 1 (existing self loops dropped, one per node added: remove_self_loops + add_self_loops); rowptr_t/col_t: the
 * same pattern built by_source.  xp = x W^T [n, heads*c] (activation dtype, 16-byte aligned rows); a_src, a_dst, lse, r_ws:
 * fp32 [n, heads]; da_src, da_dst: fp32 [heads, n].  c must be a multiple of 4 (fp32) / 8 (bf16), heads*c at most 512 (fp32) /
 * 1024 (bf16), heads <= SGF_GAT_MAX_HEADS.
 *   e_ij = leaky_relu(a_src[j] + a_dst[i], 0.2);  alpha_ij = exp(e_ij - lse_i);  y_i = sum_j alpha_ij d_ij xp_j
 *   out_i = (mean ? mean over heads of y_i : y_i) + bias  (bias nullable; out [n, c] or [n, heads*c] in the activation dtype)
 * d_ij = attention dropout (p, seed + the dropout epoch): 0 or 1/(1-p) from a hash of (target, source, duplicate rank, head), so the
 * forward and both backward traversals draw the same mask.  No float atomics: every launch is bit-identical run to run.
 * sgf_gat_logits: a_src[n,h] = <xp[n,h,:], att_src[h,:]>, a_dst likewise (att_* fp32 [heads*c]).
 * sgf_gat_bwd, given g = dL/dout: pass 1 over the CSR writes r_i = <g_i, y_i> per head and da_dst; pass 2 over the transposed CSR
 * rebuilds alpha_ij from a_src, a_dst and lse and writes dxp_j = sum_i alpha_ij d_ij g_i + da_src_j att_src + da_dst_j att_dst
 * (the full gradient of xp, logits included) and da_src.
 * sgf_dense_dropout: y = dropout(x) for an fp32 matrix (GAT's input dropout), one hash of (seed + epoch, r*cols + c) per element.
 * ------------------------------------------------------------------------------------------------ */
#define SGF_GAT_MAX_HEADS 8
int sgf_gat_logits(const void* xp, int64_t ldx, int64_t n, int heads, int c, int dtype, const float* att_src, const float* att_dst,
                   float* a_src, float* a_dst, void* stream);
int sgf_gat_fwd(const int64_t* rowptr, const int32_t* col, const void* xp, int64_t ldx, const float* a_src, const float* a_dst,
                int64_t n, int heads, int c, int dtype, int mean, const float* bias, void* out, int64_t ldo, float* lse, float p,
                uint64_t seed, void* stream);
int sgf_gat_bwd(const int64_t* rowptr, const int32_t* col, const int64_t* rowptr_t, const int32_t* col_t, const void* xp, int64_t ldx,
                const float* a_src, const float* a_dst, const float* lse, const void* g, int64_t ldg, const float* att_src,
                const float* att_dst, int64_t n, int heads, int c, int dtype, int mean, float p, uint64_t seed, float* r_ws,
                float* da_src, float* da_dst, void* dxp, int64_t ldd, void* stream);
int sgf_dense_dropout(const float* x, int64_t ldx, int64_t rows, int64_t cols, float p, uint64_t seed, float* y, int64_t ldy,
                      void* stream);

/* Row-sharded SpMM fused with the halo exchange (SURVEY.md §8e C4): as sgf_spmm, but x is the gathered operand
 * [n_slots*slot_rows, h] of which only slot 0 (this rank's own rows) is present at launch; slot s > 0 (the rows of rank
 * (rank + s) mod world) is being written by that rank over NVLink (copy-engine peer copy into this buffer) and is complete once
 * flags[s] != 0 (the sender's sgf_signal after its copy).  col holds ROTATED ids (sgf_csr_build_rot), so every row meets its
 * neighbours in slot order and a warp only waits the first time it touches a slot that has not landed: the gather of the local and
 * the already-arrived blocks overlaps the transfer of the rest.  One wave of resident CTAs; flags[0] is ignored. */
int sgf_spmm_flagged(const int64_t* rowptr, const int32_t* col, const float* row_scale, const void* x, int64_t ldx, void* y,
                     int64_t ldy, int64_t n_rows, int h, int dtype, int64_t max_row_len, const uint32_t* flags, int64_t slot_rows,
                     int n_slots, void* stream);
/* One PHASE of a row-sharded SpMM (dist.Comm, C4 overlap): entries [lo[r], hi[r]) of every row r (int32 offsets relative to the row
 * start, from sgf_csr_row_splits; NULL = row start / row end) are gathered and added to part_in[r,:] (fp32, nullable); the result
 * goes to part_out[r,:] (fp32 partial sums, pitch ld_part) or, when part_out is NULL, is scaled by row_scale[r] and stored to
 * y[r,:] like sgf_spmm.  With the rotated column ids of sgf_csr_build_rot a range is "the neighbours living in slots a..b of the
 * gathered operand": the phase of the local slot runs while the peers' blocks are still in flight, each later phase is launched
 * behind an sgf_wait_flags on the slots it needs. */
int sgf_spmm_range(const int64_t* rowptr, const int32_t* col, const float* row_scale, const void* x, int64_t ldx, void* y,
                   int64_t ldy, int64_t n_rows, int h, int dtype, const int32_t* lo, const int32_t* hi, const float* part_in,
                   float* part_out, int64_t ld_part, void* stream);
/* splits[t*n_rows + r] = number of entries of row r with column id < thresholds[t] (rows sorted; device int32 thresholds) */
int sgf_csr_row_splits(const int64_t* rowptr, const int32_t* col, int64_t n_rows, const int32_t* thresholds, int n_thr,
                       int32_t* splits, void* stream);
/* *flag = value with release semantics at system scope (flag may live in a peer GPU's memory): "my block has landed". */
int sgf_signal(uint32_t* flag, uint32_t value, void* stream);
/* cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault) on `stream`: the copy-engine transfer of an operand block into a peer GPU's
 * symmetric buffer (dst = the peer mapping of that buffer).  A plain stream-ordered memcpy node: no cross-device stream
 * synchronisation and capturable in a CUDA graph (torch's cross-device Tensor.copy_ is neither). */
int sgf_memcpy_async(void* dst, const void* src, size_t bytes, void* stream);
/* returns (on the stream) once flags[0..n) are all non-zero */
int sgf_wait_flags(const uint32_t* flags, int n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense contractions on Hopper tensor cores (wgmma; bf16 operands staged by TMA, fp32 accumulation in registers).
 * Replace nn.Linear / torch.einsum call sites (medium/ours.py:21-22,27-28,76-85; large/ours.py:38-40,
 * 123-128,136-143,199,275).
 * ------------------------------------------------------------------------------------------------ */
#define SGF_MAX_SRC 4
#define SGF_MAX_SEG 16

/* out = epilogue( sum_s A[seg_a[s]][:, koff:koff+klen] . B[seg_b[s]][:, koff:koff+klen]^T )
 * A[i]: bf16 [rows, a_cols[i]] (K-major), B[i]: bf16 [n_out, b_cols[i]] (K-major, e.g. an nn.Linear weight).
 * When seg_klen is not a multiple of 64 the A columns [koff+klen, next multiple of 64) must be zero (zero padding, or
 * the end of the tensor where TMA zero-fills) and the B columns there finite.
 * Optional tail: 16 extra output columns whose B rows come from b_tail [16, b_cols] (bf16), only with a
 * single B source; used for the attention normaliser column.  n_out (+16) <= 272 per n-block of 256. */
#define SGF_EPI_AFFINE 0      /* out = (alpha*acc + beta*aux[r,c] + bias[c] + r1_row[r]*r1_col[c]) -> relu -> *row_scale[r] (+= out) */
#define SGF_EPI_ATTN_APPLY 1  /* out[r,c] = (acc[r,c] + nf*aux[r,c]) / (acc_tail[r,0] + nf); den_out[r] = that denominator */
#define SGF_EPI_ATTN_GRAM 2   /* out[r,c] = (acc[r,c] + bias[c]) / (acc_tail[r,0] + *nf_dev); den_out[r] = that denominator.
                               * Pass 2 of the Gram-form attention (sgf_attn_gram_prepare_fwd): projections, q~.(k~^T v) + N v,
                               * normaliser and divide of full_attention_conv (medium/ours.py:76-85,16-34) as ONE GEMM of the
                               * layer input */

#define SGF_GEMM_AUTO 0
#define SGF_GEMM_STREAM_B 1
#define SGF_GEMM_RESIDENT_B 2
typedef struct {
    const void* a[SGF_MAX_SRC]; int64_t lda[SGF_MAX_SRC]; int64_t a_cols[SGF_MAX_SRC];
    const void* b[SGF_MAX_SRC]; int64_t ldb[SGF_MAX_SRC]; int64_t b_cols[SGF_MAX_SRC];
    int32_t n_a, n_b, n_seg;
    int32_t seg_a[SGF_MAX_SEG], seg_akoff[SGF_MAX_SEG], seg_b[SGF_MAX_SEG], seg_bkoff[SGF_MAX_SEG], seg_klen[SGF_MAX_SEG];
    const void* b_tail; int64_t ldb_tail;      /* NULL = no tail */
    int64_t rows; int32_t n_out;
    /* epilogue */
    int32_t epi;
    void* out; int64_t ldo; int32_t out_dtype;
    const float* bias;                          /* [n_out] or NULL */
    const void* aux; int64_t ld_aux; int32_t aux_dtype;   /* [rows, n_out] or NULL */
    const float* row_scale;                     /* [rows] or NULL */
    float alpha, beta;                          /* host scalars */
    const float* alpha_dev; const float* beta_dev; /* optional device scalars multiplied into alpha/beta */
    int32_t relu, accumulate;
    float nf;                                   /* ATTN_APPLY: node count N as float */
    const float* nf_dev;                        /* ATTN_GRAM: device scalar added to the tail column (replaces nf) */
    float* den_out;                             /* ATTN_APPLY: [rows] fp32 or NULL */
    const float* r1_row; const float* r1_col;   /* AFFINE: optional rank-1 term + r1_row[r]*r1_col[c] (both or neither) */
    float* col_sum; float* col_sumsq;           /* optional (caller-zeroed, fp32 [n_out]): column sums / sums of squares of the
                                                   STORED output accumulated in the epilogue (BatchNorm statistics, K^T 1,
                                                   ||Q||^2, ||K||^2 without a second pass); needs a 16-byte aligned out with a
                                                   16-byte-multiple pitch and n_out <= 1024, else SGF_ERR_UNSUPPORTED */
    int32_t schedule;                           /* SGF_GEMM_AUTO (0), or force one of the two schedules (tests / tuning):
                                                   SGF_GEMM_STREAM_B = weights stream through the TMA ring with A,
                                                   SGF_GEMM_RESIDENT_B = weights of one n-block stay in shared memory across the
                                                   row tiles (SGF_ERR_UNSUPPORTED if they do not fit) */
} sgf_gemm_nt_args;
int sgf_gemm_nt(const sgf_gemm_nt_args* args /* host */, void* stream);

/* Node-contracting product: out[M,N] = alpha * sum_n A[n,:M]^T B[n,:N]  (+ beta*out), fp32 output.
 * A: bf16 [rows, m] row-major, B: bf16 [rows, n] row-major; m <= 256, n <= 256.
 * Used for K^T V (medium/ours.py:21), q^T gnum (its backward) and every weight gradient dW = dY^T X.
 * Deterministic two-stage reduction through `ws` (sgf_gemm_tn_ws_bytes).  transpose_out writes out[N,M]. */
#define SGF_TN_MAX_PAIRS 6
typedef struct {
    const void* a; int64_t lda; int32_t m;
    const void* b; int64_t ldb; int32_t n;
    int64_t rows;
    float* out; int64_t ldo; int32_t transpose_out;
    float alpha, beta; const float* alpha_dev;
    void* ws; size_t ws_bytes;
    int32_t n_pairs;                            /* 0: one product of the columns [0,m) x [0,n).  > 0 (bf16x3 operands): the
                                                   products A[:, a_off[i] : +m]^T B[:, b_off[i] : +n], i < n_pairs, are summed in
                                                   the accumulator (offsets in elements, multiples of 64; lda/ldb cover them) */
    int32_t a_off[SGF_TN_MAX_PAIRS], b_off[SGF_TN_MAX_PAIRS];
} sgf_gemm_tn_args;
int sgf_gemm_tn_ws_bytes(int32_t m, int32_t n, int64_t rows, size_t* bytes);
int sgf_gemm_tn(const sgf_gemm_tn_args* args /* host */, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Row-streaming kernels (replace the ATen elementwise / reduction passes: torch.norm medium/ours.py:16-17,
 * nn.LayerNorm, nn.BatchNorm1d, F.relu, F.dropout, residual mixes large/ours.py:79-93,199-216,270).
 * All take dtype in {SGF_F32, SGF_BF16} for the [rows,h] activations; statistics/parameters are fp32.
 * ------------------------------------------------------------------------------------------------ */

/* Workspace bytes of a reducing launcher (see the conventions above) for rows of `width` floats reduced
 * across thread blocks (h; cols of sgf_pack_operand; 1 for sgf_softmax_nll). */
int sgf_reduce_ws_bytes(int32_t width, size_t* bytes /* host out */);
/* column statistics: sum[c] += w[r]*x[r,c], sumsq[c] += x[r,c]^2 (outputs must be zeroed by the caller;
 * sum, sumsq, w nullable).  Gives K^T 1, ||Q||^2, ||K||^2, q^T gden, BatchNorm batch statistics. */
int sgf_colstats(const void* x, int64_t ldx, int64_t rows, int h, int dtype, const float* w,
                 float* sum, float* sumsq, void* ws, size_t ws_bytes, void* stream);

/* y = dropout( relu?( LN?( a*x + b*r ) ) ), r nullable.  stats: fp32 [rows,2] (mean, rstd) or NULL.
 * (TransConv.forward, large/ours.py:199-216).  p = dropout prob, seed identifies the mask. */
int sgf_ln_fwd(const void* x, const void* r, int64_t ld, int64_t rows, int h, int dtype, float a, float b,
               const float* gamma, const float* beta, int use_ln, int use_relu, float p, uint64_t seed,
               void* y, float* stats, void* stream);
/* sgf_ln_fwd with a third input: u = a*x + b*r + c*gy (gy non-NULL, same dtype and pitch).  A DIFFormer layer
 * (medium/difformer.py:129-137,202-206) mixes its attention output x, the previous layer r and the graph term gy = Â v here. */
int sgf_ln_fwd_graph(const void* x, const void* r, const void* gy, int64_t ld, int64_t rows, int h, int dtype, float a, float b,
                     float c, const float* gamma, const float* beta, int use_ln, int use_relu, float p, uint64_t seed, void* y,
                     float* stats, void* stream);
/* backward of sgf_ln_fwd for the upstream gradient gscale*dy: writes dx = a*du and (if dr != NULL) dr = b*du;
 * accumulates dgamma[c], dbeta[c] (fp32, caller-zeroed, nullable when !use_ln). */
int sgf_ln_bwd(const void* dy, const void* x, const void* r, int64_t ld, int64_t rows, int h, int dtype,
               float a, float b, const float* gamma, const float* beta, const float* stats, int use_ln,
               int use_relu, float p, uint64_t seed, float gscale, void* dx, void* dr, float* dgamma, float* dbeta,
               void* ws, size_t ws_bytes, void* stream);

/* BatchNorm1d (+bias +ReLU +dropout +residual +branch mix) — GraphConv.forward large/ours.py:78-93, GCN.forward
 * medium/models.py:49-63, SGFormer.forward large/ours.py:270.
 * sgf_bn_finalize: batch statistics from column sums of z (training; sum/sumsq non-NULL; updates the running buffers
 * with momentum and the unbiased variance when they are non-NULL) or the running statistics (sum == NULL).  zbias
 * (nullable) is a per-column bias added to z before normalisation (GCNConv's bias): it only shifts the mean.
 * use_relu of the BatchNorm entry points is an activation code: 0 none, 1 ReLU, 2 ELU (alpha 1; GAT's F.elu, backward exp(t) for
 * t <= 0).
 * sgf_bn_fwd:  t = use_bn ? gamma*((z+zbias)-mean)*rstd+beta : z+zbias;  t = act(t);  t = dropout(t);  t += res?;
 *   y_scaled (nullable) = row_scale[r]*t;   if mix: t = gw*t + (1-gw)*mix[r,:];   y (nullable) = t. */
int sgf_bn_finalize(const float* sum, const float* sumsq, int64_t rows, int h, float eps, float momentum,
                    const float* zbias, float* mean, float* rstd, float* running_mean, float* running_var, void* stream);
int sgf_bn_fwd(const void* z, const void* res, const void* mix, int64_t ld, int64_t rows, int h, int dtype,
               const float* mean, const float* rstd, const float* gamma, const float* beta, const float* zbias,
               int use_bn, int use_relu, float p, uint64_t seed, float gw, const float* row_scale, void* y,
               void* y_scaled, void* stream);
/* backward.  Upstream gradient g_raw = gscale*(dy + row_scale2[r]*dy2) (dy or dy2 nullable, not both);
 * g = g_raw * dropout mask * act'(pre-activation).
 * phase 1 (training BN only): sums[0:h] += g, sums[h:2h] += g*xhat   (caller-zeroed fp32 [2h]; == dbeta, dgamma)
 * phase 2: dz = gamma*rstd*(g - sums_g/rows - xhat*sums_gx/rows) (training BN) | gamma*rstd*g (eval BN) | g (no BN);
 *   dz is written times out_row_scale[r] (nullable); dz_colsum[c] += dz (unscaled; bias gradient; nullable);
 *   dres (nullable) = or += g_raw (gradient of the residual input). */
int sgf_bn_bwd_reduce(const void* dy, const void* dy2, const float* row_scale2, const void* z, int64_t ld,
                      int64_t rows, int h, int dtype, const float* mean, const float* rstd, const float* gamma,
                      const float* beta, const float* zbias, int use_bn, int use_relu, float p, uint64_t seed,
                      float gscale, float* sums, void* ws, size_t ws_bytes, void* stream);
int sgf_bn_bwd_apply(const void* dy, const void* dy2, const float* row_scale2, const void* z, int64_t ld,
                     int64_t rows, int h, int dtype, const float* mean, const float* rstd, const float* gamma,
                     const float* beta, const float* zbias, int use_bn, int use_relu, int training, float p,
                     uint64_t seed, float gscale, int64_t stat_rows /* rows the batch statistics span; 0 = rows (the
                     global node count when row-sharded and `sums` was all-reduced) */, const float* sums, void* dz,
                     void* dres, int dres_accumulate, float* dz_colsum, const float* out_row_scale, void* ws,
                     size_t ws_bytes, void* stream);

/* Jumping knowledge over a GCN stack (GCNJK, medium/models.py:157-205), fused into the BatchNorm passes.  jk_mode: 1 max, 2 cat
 * (0 is refused: use the entry points above).  `jk` has the activation dtype, pitch ld_jk (elements; 16-byte aligned rows);
 * jk_idx (max only) is uint8 with the same pitch in bytes.  jk_layer = the layer index l (0..255) of the call.
 * sgf_bn_fwd_jk: sgf_bn_fwd without res/mix/y_scaled; a = act(BN(z + zbias)) before dropout, rounded to the dtype, is
 *   max: l == 0: jk = a, jk_idx = 0;  l > 0: where a > jk (strictly; a tie keeps the lower layer): jk = a, jk_idx = l;
 *   cat: jk[r, :] = a (`jk` points at column block l of the [rows, L*h] concatenation);
 *   y (nullable) = dropout(a) as in sgf_bn_fwd.
 * sgf_bn_bwd_reduce_jk / sgf_bn_bwd_apply_jk: sgf_bn_bwd_reduce / _apply with dy2, dres = NULL and gscale = 1, and the upstream
 *   gradient g = dropout mask * dy (dy nullable) + JK addend, then * act'; the addend is jk[r, c] where jk_idx[r, c] == l (max)
 *   or jk[r, c] (cat: block l of g_out W^T).  dz_colsum includes the addend. */
int sgf_bn_fwd_jk(const void* z, int64_t ld, int64_t rows, int h, int dtype, const float* mean, const float* rstd,
                  const float* gamma, const float* beta, const float* zbias, int use_bn, int use_relu, float p, uint64_t seed,
                  void* y, int jk_mode, void* jk, int64_t ld_jk, uint8_t* jk_idx, int jk_layer, void* stream);
int sgf_bn_bwd_reduce_jk(const void* dy, const void* z, int64_t ld, int64_t rows, int h, int dtype, const float* mean,
                         const float* rstd, const float* gamma, const float* beta, const float* zbias, int use_bn, int use_relu,
                         float p, uint64_t seed, float* sums, int jk_mode, const void* jk_g, int64_t ld_jk, const uint8_t* jk_idx,
                         int jk_layer, void* ws, size_t ws_bytes, void* stream);
int sgf_bn_bwd_apply_jk(const void* dy, const void* z, int64_t ld, int64_t rows, int h, int dtype, const float* mean,
                        const float* rstd, const float* gamma, const float* beta, const float* zbias, int use_bn, int use_relu,
                        int training, float p, uint64_t seed, const float* sums, void* dz, float* dz_colsum,
                        const float* out_row_scale, int jk_mode, const void* jk_g, int64_t ld_jk, const uint8_t* jk_idx,
                        int jk_layer, void* ws, size_t ws_bytes, void* stream);

/* out = (a*x + b*y) * row_scale[r]  (y, row_scale nullable; y has x's dtype); in/out dtypes may differ (casts). */
int sgf_axpby(const void* x, int64_t ldx, int x_dtype, const void* y, int64_t ldy, int y_dtype, float a, float b,
              const float* row_scale, void* out, int64_t ldo, int out_dtype, int64_t rows, int h, void* stream);
/* fp32 [rows, cols] -> bf16 tensor-core operand dst (optionally transposed: dst[c, r] = src[r, c]) whose K extent is
 * zero-padded to kp; plane_ld = 0: one bf16 plane; plane_ld >= kp: three planes side by side along K with
 * src ~= p0 + p1 + p2 (bf16x3 split: fp32-accurate products on the bf16 tensor cores).  colsum (nullable, caller-zeroed):
 * exact fp32 column sums of src (bias gradients). */
int sgf_pack_operand(const float* src, int64_t ld_src, int64_t rows, int cols, int transpose, void* dst,
                     int64_t ld_dst, int kp, int64_t plane_ld, float* colsum,
                     const int64_t* row_index /* nullable: dst row r = src row row_index[r] (mini-batch feature gather,
                     large/main-batch.py:138 x[idx_i]); rows = number of gathered rows; not with transpose */, void* ws, size_t ws_bytes,
                     void* stream);
/* mean over heads: out[r,c] = (1/heads) * sum_h x[r, h*d + c]  (TransConvLayer, medium/ours.py:95) */
int sgf_head_mean(const void* x, int64_t ldx, int64_t rows, int heads, int d, int dtype, void* out, int64_t ldo,
                  void* stream);

/* Fused log_softmax + NLL over the selected rows, forward value and logits gradient in one pass (replaces
 * F.log_softmax + nn.NLLLoss on out[train_mask] and their autograd, large/main.py:139-141):
 *   *loss += scale * sum_{r: mask[r]} -log_softmax(logits[r])[labels[r]]      (caller-zeroed; scale = 1/#selected for 'mean')
 *   dlogits[r,:] = scale * (softmax(logits[r]) - onehot(labels[r])) for selected rows, 0 otherwise (dlogits nullable).
 * mask: uint8 [rows] or NULL (all rows). */
int sgf_softmax_nll(const float* logits, int64_t ld, const int64_t* labels, const uint8_t* mask, int64_t rows, int c,
                    float scale, float* loss, float* dlogits, int64_t ld_d, void* ws, size_t ws_bytes,
                    void* stream);

/* K11 - evaluation on the device (SURVEY.md §8f-3): number of rows r = idx[i], i < m (all rows when idx is NULL, then m = rows)
 * with argmax_j logits[r, j] == labels[r] (first maximum on ties), and optionally the sum of -log_softmax(logits[r])[labels[r]].
 * Replaces eval_acc (large/data_utils.py:210-220: argmax, D2H, numpy loop per split) and the valid_loss of evaluate()
 * (large/eval.py:28-31) for single-column int64 labels.  correct: device int64, nll_sum: device fp64 or NULL. */
int sgf_eval_acc(const float* logits, int64_t ld, const int64_t* labels, const int64_t* idx, int64_t m, int64_t rows, int32_t c,
                 int64_t* correct, double* nll_sum, void* stream);
/* K11 over one batch of a mini-batch evaluation (replaces the three eval_acc calls per batch of large/eval.py:67-118
 * evaluate_batch and their three host syncs).  Row i < m of logits [m, c] (pitch ld) is node r = idx[i] (r = i when idx is
 * NULL; then m <= rows); labels int64 [rows] and split uint8 [rows] are read at r.  split[r] holds one bit per split (1 train,
 * 2 valid, 4 test; overlapping splits set several) and for every bit k set:  counts[2k] += 1,  counts[2k+1] += (argmax_j
 * logits[i, j] == labels[r]), with the argmax of sgf_eval_acc: the first maximum on ties, as torch.max(dim=1), checked against
 * the reference's eval_acc with planted ties in tests/test_gpu_kernels.py (test_eval_acc_matches_reference_semantics) for
 * sgf_eval_acc and tests/test_gpu_eval_batch.py (test_eval_acc_splits_counts_exactly) for this entry point.  Both differ
 * from torch.max on non-finite rows: a NaN entry never wins (torch.max returns the NaN's index), and a row of -inf only
 * has no argmax (torch.max returns 0), so neither counts as a hit.  counts: device int64 [6], ADDED into (the caller zeroes it
 * once per epoch).  Integer sums only: deterministic.  No allocation, no sync. */
int sgf_eval_acc_splits(const float* logits, int64_t ld, int64_t m, int32_t c, const int64_t* labels, const uint8_t* split,
                        const int64_t* idx, int64_t rows, int64_t* counts, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Linear attention glue (full_attention_conv, medium/ours.py:14-34; backward per SURVEY.md Appendix A.1)
 * ------------------------------------------------------------------------------------------------ */
/* Operand format of the small bf16 matrices written by the prepare kernels: plane_ld = 0 -> one bf16 plane;
 * plane_ld > 0 -> three planes side by side along K (value ~= p0+p1+p2, see sgf_split3) for fp32-accurate GEMMs.
 *
 * sgf_attn_prepare_fwd: from the pass-1 partials S'[m,d] = k^T v (sgf_gemm_tn), z'[m] = k^T 1 and the per-column
 * sums of squares of q and k (sgf_colstats; nq2 = sum(nq2v), nk2 = sum(nk2v)) build the B operands of the apply GEMM:
 *   bmat[d, m] = S'[m,d]/(nq*nk) (K-major over m), btail[0, m] = z'[m]/(nq*nk), btail[1..15,:] = 0;
 *   scal[0] = 1/nq, scal[1] = 1/nk, scal[2] = 1/(nq*nk). */
int sgf_attn_prepare_fwd(const float* s_raw, const float* z_raw, const float* nq2v, int nq2_len, const float* nk2v,
                         int nk2_len, int m, int d, void* bmat, int64_t ld_bmat, void* btail, int64_t ld_btail,
                         int64_t plane_ld, float* scal, void* stream);
/* gnum = gscale*g/den, gden = -gscale*(g.o)/den  (per row); gnum: [rows,d] same dtype as g, gden: fp32 [rows] */
int sgf_attn_bwd_prep(const void* g, int64_t ld, const void* o, int64_t ld_o, const float* den, int64_t rows, int d,
                      int dtype, float gscale, void* gnum, int64_t ld_gnum, float* gden, void* stream);
/* multi-head: the norm-gradient scalar c is shared by all heads; sums scal_bwd[i*stride+3] and rewrites entries 1,2 */
int sgf_attn_combine_scal(float* scal_bwd, int heads, int stride, const float* scal_fwd, void* stream);
/* Backward glue (SURVEY.md Appendix A.1 rewritten for raw q,k): with alpha = 1/(nq*nk), dS_raw = q^T gnum,
 * dz_raw = q^T gden:  b_dq[m,d] = S'[m,d], b_dk[m,d] = dS_raw[m,d], b_dv[d,m] = dS_raw[m,d],
 * r1_col[m] = alpha*z'[m], dk_bias[m] = alpha*dz_raw[m], c = alpha*(<dS_raw,S'> + <dz_raw,z'>),
 * scal_bwd = {alpha, -c/nq^2, -c/nk^2, c}.  Then
 *   dq = alpha*(gnum.b_dq^T) + gden (x) r1_col + scal_bwd[1]*q
 *   dk = alpha*(v.b_dk^T) + dk_bias + scal_bwd[2]*k
 *   dv = alpha*(k.b_dv^T) + N*gnum */
int sgf_attn_prepare_bwd(const float* s_raw, const float* z_raw, const float* ds_raw, const float* dz_raw,
                         const float* scal_fwd, int m, int d, void* b_dq, int64_t ld_b_dq, void* b_dv, int64_t ld_b_dv,
                         void* b_dk, int64_t ld_b_dk, int64_t plane_ld_d, int64_t plane_ld_m, float* r1_col,
                         float* dk_bias, float* scal_bwd, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Gram-form linear attention (single head): TransConvLayer.forward = Wq/Wk/Wv projections + full_attention_conv + its
 * autograd (medium/ours.py:14-34,76-95; large/ours.py:123-157; 100M/ours.py:12-43,175-190) WITHOUT materialising q, k, v.
 * Every node contraction of the layer is a function of G = x^T x and s = x^T 1 of the layer input x [N,h] (derivation at the
 * top of csrc/attn_gram.cu), so the layer is:   pass 1  G, s            (sgf_gemm_tn x^T x + sgf_colstats)
 *                                               h x h   sgf_attn_gram_prepare_fwd
 *                                               pass 2  out = (x Bt^T + bt) / (x ct + dt)     (sgf_gemm_nt, SGF_EPI_ATTN_GRAM)
 * and its backward:  sgf_ln_bwd_attn (row prologue) -> P = x^T gnum' (sgf_gemm_tn) -> sgf_attn_gram_prepare_bwd ->
 *                    dx = [gnum' | x] . [Bt | A3] + gden' (x) ct + a4 (sgf_gemm_nt, two segments).
 * All pointers are DEVICE fp32, row-major and dense unless a pitch is given.  use_weight=False (V = x, medium/ours.py:84) is
 * expressed by passing the identity as wv and zeros as bv.
 * ------------------------------------------------------------------------------------------------ */
/* Pass 1: G[h,h] = X^T X (fp32, both triangles, pitch ldg) and s[h] = X^T 1 of a bf16 tensor-core operand X [rows, h <= 256]
 * (planes = 1: one bf16 plane; planes = 3: bf16x3 planes side by side, plane_ld elements apart, the six partial products are
 * accumulated).  wgmma kernel that loads every tile once for both MMA operands and accumulates only the upper block
 * triangle; deterministic two-stage reduction through ws (sgf_gram_ws_bytes). */
int sgf_gram_ws_bytes(int32_t h, int32_t planes, int64_t rows, size_t* bytes);
int sgf_gram(const void* x, int64_t ldx, int64_t rows, int32_t h, int32_t planes, int64_t plane_ld, float* G, int64_t ldg,
             float* s, void* ws, size_t ws_bytes, void* stream);
typedef struct {
    int32_t h, m, d;            /* input width, q/k width (Wq, Wk: [m,h]), v width (Wv: [d,h]) */
    int64_t n_nodes;            /* N of `N*vs` / `+N` (medium/ours.py:25,31): the GLOBAL node count when row-sharded */
    const float *wq, *bq, *wk, *bk, *wv, *bv;
    int64_t ld_wq, ld_wk, ld_wv;
    const float* G;             /* [h,h] x^T x (all-reduced over the row shards) */
    const float* s;             /* [h]   x^T 1 */
    /* written by prepare_fwd, read again by prepare_bwd */
    float *kx, *qx, *vx;        /* [m,h], [m,h], [d,h]: k^T x, q^T x, v^T x */
    float *z1, *q1, *v1;        /* [m], [m], [d]:       k^T 1, q^T 1, v^T 1 */
    float* S;                   /* [m,d] k^T v */
    float* Bt;                  /* [d,h]  B operand of the apply GEMM (K-major over h), before bf16 packing */
    float* tail;                /* [16,h] caller-zeroed; row 0 = ct */
    float* bt;                  /* [d] */
    float* sc;                  /* [16] scalars: 0 ||q||^2, 1 ||k||^2, 2 alpha, 3 beta = alpha/N, 4 dt, 5 N, 6 1.0, 7 bq.z1,
                                   8 <dS,S>+<dz,z1>, 9 c, 10 -c/||q||^2, 11 -c/||k||^2 */
    /* prepare_bwd only */
    const float* P;             /* [h,d] x^T gnum' */
    const float* pg;            /* [h]   x^T gden' */
    const float* cs;            /* [d]   1^T gnum' */
    const float* sg;            /* [1]   1^T gden' */
    float *dwq, *dbq, *dwk, *dbk, *dwv, *dbv;   /* gradients, shapes of the parameters (dense) */
    float* bcat;                /* [h, d+h] = [Bt^T | A3]: B operand of dx = gnum' Bt + x A3 */
    float* a4;                  /* [h] constant row of dx */
    float* ws; int64_t ws_floats;   /* scratch, sgf_attn_gram_ws_floats */
} sgf_attn_gram_args;
int sgf_attn_gram_ws_floats(int h, int m, int d, int64_t* n_floats /* host out */);
int sgf_attn_gram_prepare_fwd(const sgf_attn_gram_args* args /* host */, void* stream);
int sgf_attn_gram_prepare_bwd(const sgf_attn_gram_args* args /* host */, void* stream);
/* Value-sum mode (DIFFormer's `simple` kernel, medium/difformer.py:18-39): the numerator adds the column sum sum_l v_l instead of
 * N v_n.  Same arguments and outputs as above, with  Bt = beta S^T Wq,  bt = beta S^T bq + v1/N  in the forward and
 *   dWv = beta dS^T kx + cs s^T / N,   a4 += Wv^T cs / N     (everything else unchanged)  in the backward. */
int sgf_attn_gram_prepare_fwd_vsum(const sgf_attn_gram_args* args /* host */, void* stream);
int sgf_attn_gram_prepare_bwd_vsum(const sgf_attn_gram_args* args /* host */, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Fused softmax attention of SGFormerSOFT (medium/ablation/oursSOFT.py:14-34; derivation and the |s| <= 1 bound at the top of
 * csrc/attn_softmax.cu): s[n,l,h] = q~[n,h].k~[l,h] with one Frobenius norm over all nodes and heads, P = softmax over the HEADS
 * of s[n,l,:] (the reference's F.softmax(dim=-1) of its [N, L, H] scores), o[n,h] = sum_l P[n,l,h] v[l,h].
 * q, k: [n, heads*m], v: [n, heads*d] (or [n, d] with shared_v: one v for every head), activations of `dtype` (0 fp32, 1 bf16)
 * whose pointers and pitches are 16-byte aligned; m, d multiples of 16 bytes of the dtype; the heads' blocks of one q row, each
 * padded to 16 elements, and those of one v row take at most SGF_ATTN_SOFTMAX_MAX_ROW_BYTES (else SGF_ERR_UNSUPPORTED).
 * sq_q / sq_k: fp32 [heads*m] column sums of squares of q / k (||q||^2 = their sum).
 * No N x N buffer is ever written; every output element is written by one thread in a fixed order (deterministic, no atomics).
 *   fwd:      o [n, heads*d]
 *   bwd_q:    with g the gradient of o (times gscale), head h's block at column h*g_hstride (g_hstride = d, or 0: one [n, d]
 *             block for every head, the head mean's backward):  aq [n, heads*m] (fp32, pitch ld_a) = c dS k per head
 *             (c = 1/(||q|| ||k||), dS_h = P_h (g_h v_h^T - sum_h' P_h' g_h' v_h'^T))
 *   bwd_kv:   ak (fp32, pitch ld_a) = c dS^T q,  dv (+)= gscale P^T g  (with shared_v: the heads summed in head order)
 *   bwd_norm: dq = gscale (aq - <q,aq>/||q||^2 q), dk likewise (dtype, pitches lddq / lddk): the Frobenius-norm backward
 *   probs:    att [n, n] (fp32, pitch ld_att) = the head mean of P (inference, small n)
 * ws: fp32 scratch of sgf_attn_softmax_ws_floats for the bwd kernels' per-CTA partial sums.
 * Scaled mode (scaled = 1; SGFormerGAT, medium/ablation/oursGAT.py:31-44): s[n,l,h] = scale q[n,h].k[l,h] with a host constant
 * scale > 0 (1/sqrt(dk)), the softmax over the heads taken against each pair's maximum over the heads; sq_q, sq_k, ws, aq, ak
 * are unused and v is per head (shared_v = 0).  fwd as above; bwd_q writes dq = gscale scale dS k and bwd_kv writes
 * dk = gscale scale dS^T q (dtype, pitches lddq / lddk) and dv as above.  bwd_norm and probs refuse this mode.
 * tile_rows (host only, no CUDA call): rows[0..2] = the height of the streamed tile (64, 32 or 16 rows) that fwd, bwd_q and bwd_kv
 * pick for this shape in either mode, 0 where no height fits in shared memory (that launch returns SGF_ERR_UNSUPPORTED);
 * shared_g: the backward's g is one [n, d] block for every head (g_hstride = 0), else one block per head.  SGF_ERR_UNSUPPORTED for
 * widths the launches refuse (not multiples of 16 bytes, or past SGF_ATTN_SOFTMAX_MAX_ROW_BYTES). */
#define SGF_ATTN_SOFTMAX_MAX_ROW_BYTES 1024
typedef struct {
    int32_t n, heads, m, d, dtype, shared_v;
    const void* q; int64_t ldq;
    const void* k; int64_t ldk;
    const void* v; int64_t ldv;
    const float *sq_q, *sq_k;
    void* o; int64_t ldo;           /* written by fwd */
    const void* g; int64_t ldg, g_hstride; float gscale;
    float *aq, *ak; int64_t ld_a;
    void* dv; int64_t lddv; int32_t dv_accumulate;
    void* dq; int64_t lddq;
    void* dk; int64_t lddk;
    float* ws; int64_t ws_floats;
    int32_t scaled; float scale;    /* 1: scaled mode (below); 0: the Frobenius-normalised scores above */
} sgf_attn_softmax_args;
int sgf_attn_softmax_ws_floats(int n, int heads, int m, int d, int64_t* n_floats /* host out */);
int sgf_attn_softmax_tile_rows(int heads, int m, int d, int dtype, int shared_v, int shared_g, int32_t rows[3] /* host out */);
int sgf_attn_softmax_fwd(const sgf_attn_softmax_args* args /* host */, void* stream);
int sgf_attn_softmax_bwd_q(const sgf_attn_softmax_args* args /* host */, void* stream);
int sgf_attn_softmax_bwd_kv(const sgf_attn_softmax_args* args /* host */, void* stream);
int sgf_attn_softmax_bwd_norm(const sgf_attn_softmax_args* args /* host */, void* stream);
int sgf_attn_softmax_probs(const sgf_attn_softmax_args* args /* host */, float* att, int64_t ld_att, void* stream);

/* Dropout epoch.  Every kernel that takes (p, seed) draws its mask from hash(seed + epoch * odd, row, chunk); `epoch` is read from
 * the device word registered here (NULL, the default: epoch 0).  The host seed of a call is frozen into a captured CUDA graph;
 * a step that is captured and replayed registers an epoch word and puts sgf_advance_dropout_epoch at the top of the captured
 * step, so that every replay draws fresh masks while forward and backward of one step still agree (F.dropout semantics,
 * large/ours.py:216).  One word per process (one process per GPU). */
int sgf_set_dropout_epoch(const uint64_t* epoch_dev /* device, stays alive; NULL to unregister */);
int sgf_advance_dropout_epoch(uint64_t* epoch_dev, void* stream);   /* *epoch_dev += 1 on the stream */
/* LayerNorm backward of y = dropout(relu?(LN?(a*o + b*r))) (TransConv.forward, large/ours.py:208-216) fused with the row
 * prologue of the attention backward: with du the gradient w.r.t. u = a*o + b*r (as sgf_ln_bwd) and ga = a*du,
 *   gnum[r,:] = ga/den[r],  gden[r] = -(ga . o[r,:])/den[r],  dr (nullable) = b*du,
 *   cs[c] += gnum[r,c],  pg[c] += xa[r,c]*gden[r],  sg[0] += gden[r]      (fp32, caller-zeroed),
 * dgamma/dbeta as sgf_ln_bwd.  o = attention output, den = SGF_EPI_ATTN_GRAM's den_out, xa = the layer input (may alias r). */
int sgf_ln_bwd_attn(const void* dy, const void* o, const void* r, const void* xa, int64_t ld, int64_t rows, int h, int dtype,
                    float a, float b, const float* gamma, const float* beta, const float* stats, int use_ln, int use_relu,
                    float p, uint64_t seed, float gscale, const float* den, void* gnum, float* gden, void* dr, float* dgamma,
                    float* dbeta, float* cs, float* pg, float* sg, void* ws,
                    size_t ws_bytes, void* stream);
/* sgf_ln_bwd_attn for u = a*o + b*r + c*gy (sgf_ln_fwd_graph; no ReLU): additionally writes ys[r,:] = dinv[r] * c * du[r,:],
 * the pre-scaled operand of the transposed SpMM that carries the gradient of the graph term gy = Â v back to v. */
int sgf_ln_bwd_attn_graph(const void* dy, const void* o, const void* r, const void* xa, const void* gy, int64_t ld, int64_t rows, int h, int dtype,
                          float a, float b, float c, const float* gamma, const float* beta, const float* stats, int use_ln, float p,
                          uint64_t seed, float gscale, const float* den, const float* dinv, void* gnum, float* gden, void* dr,
                          void* ys, float* dgamma, float* dbeta, float* cs, float* pg, float* sg, void* ws, size_t ws_bytes,
                          void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused two-group Adam (SURVEY.md §8f-3; replaces torch.optim.Adam([{params1, trans_weight_decay}, {params2,
 * gnn_weight_decay}], lr) of large/main.py:115-119 and its optimizer.step() at :142): all tensors of a step in one launch per
 * SGF_ADAM_MAX_TENSORS, fp32 parameters / gradients / moments, hyper-parameters per tensor (its group's), one step count t per
 * tensor on the device (fp32 scalars advanced by the call itself, so CUDA-graph replays keep counting and a parameter that had no
 * gradient in some step keeps its own count, as in torch).
 *   g += wd*p;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= lr/(1-b1^t) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
 * ------------------------------------------------------------------------------------------------ */
#define SGF_ADAM_MAX_TENSORS 32
typedef struct {
    int32_t n_tensors;
    float* param[SGF_ADAM_MAX_TENSORS]; const float* grad[SGF_ADAM_MAX_TENSORS];
    float* exp_avg[SGF_ADAM_MAX_TENSORS]; float* exp_avg_sq[SGF_ADAM_MAX_TENSORS];
    int64_t numel[SGF_ADAM_MAX_TENSORS];
    float lr[SGF_ADAM_MAX_TENSORS], beta1[SGF_ADAM_MAX_TENSORS], beta2[SGF_ADAM_MAX_TENSORS], eps[SGF_ADAM_MAX_TENSORS],
          weight_decay[SGF_ADAM_MAX_TENSORS];
    float* step[SGF_ADAM_MAX_TENSORS];          /* device fp32 scalars: number of updates each tensor has received so far */
    int32_t chunk0[SGF_ADAM_MAX_TENSORS + 1];   /* filled by sgf_adam_step */
} sgf_adam_args;
int sgf_adam_step(sgf_adam_args* args /* host, chunk0 is written */, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SGFORMER_B200_H */
