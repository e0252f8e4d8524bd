/* Plain-C restatement of the integer part of GraphConvLayer.forward — TEST INFRASTRUCTURE ONLY.
 *
 * Follows the reference's large/ours.py:26-33: in-degree over `col` (PyG degree == scatter_add of
 * ones, :28) and the CSR that torch_sparse.SparseTensor(row=col, col=row, ...) builds (:33): entries
 * ordered by key target*N+source, duplicates kept, rowptr = exclusive scan of the target counts.
 * Built by __graft_entry__.build() into oracle/_build/libcsr_ref.so; only tests/ may load it.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int cmp_i32(const void* a, const void* b) {
    int32_t x = *(const int32_t*)a, y = *(const int32_t*)b;
    return (x > y) - (x < y);
}

/* edge_index: int64 [2, nnz] row-major (row 0 = source `row`, row 1 = target `col`).
 * by_source != 0 builds the transpose pattern (rows = sources, cols = targets) used by the backward.
 * Returns 0, or -1 on an out-of-range node id. */
int sgf_oracle_csr_build(const int64_t* edge_index, int64_t nnz, int64_t n, int by_source,
                         int64_t* rowptr, int32_t* col, int64_t* degree_out) {
    const int64_t* key = by_source ? edge_index : edge_index + nnz;
    const int64_t* val = by_source ? edge_index + nnz : edge_index;
    memset(rowptr, 0, (size_t)(n + 1) * sizeof(int64_t));
    for (int64_t e = 0; e < nnz; ++e) {
        if (key[e] < 0 || key[e] >= n || val[e] < 0 || val[e] >= n) return -1;
        rowptr[key[e] + 1]++;
    }
    if (degree_out)
        for (int64_t i = 0; i < n; ++i) degree_out[i] = rowptr[i + 1];
    for (int64_t i = 0; i < n; ++i) rowptr[i + 1] += rowptr[i];
    int64_t* cursor = (int64_t*)malloc((size_t)(n > 0 ? n : 1) * sizeof(int64_t));
    memcpy(cursor, rowptr, (size_t)n * sizeof(int64_t));
    for (int64_t e = 0; e < nnz; ++e) col[cursor[key[e]]++] = (int32_t)val[e];
    free(cursor);
    for (int64_t i = 0; i < n; ++i)
        qsort(col + rowptr[i], (size_t)(rowptr[i + 1] - rowptr[i]), sizeof(int32_t), cmp_i32);
    return 0;
}
