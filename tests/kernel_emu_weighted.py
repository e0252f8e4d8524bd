"""CPU restatements of the weighted-graph kernels (sgf_csr_build_weighted, sgf_spmm_weighted, sgf_edge_weight_grad) and a dense,
differentiable fp64 restatement of weighted PyG gcn_norm (oracle/sgformer_oracle.py:pyg_gcn_adjacency) and of DIFFormer's
weighted gcn_conv (medium/difformer.py:63-79).  Used by tests/test_weighted.py (CPU) and tests/test_gpu_weighted.py."""
import numpy as np
import torch


def csr_weighted(edge_index, weight, n, by_source=False, self_loop_mode=0):
    """-> (rowptr int64, col int32, eid int64, val, dinv fp32) exactly as sgf_csr_build_weighted builds them (val in fp32, or in
    fp64 for an fp64 weight)."""
    ei = np.asarray(edge_index, dtype=np.int64)
    w = np.asarray(weight)
    w = w if w.dtype == np.float64 else w.astype(np.float32)      # fp32 as the kernels; fp64 for the gradient-formula checks
    src, dst = ei[0], ei[1]
    key, other = (src, dst) if by_source else (dst, src)
    eid = np.arange(src.size, dtype=np.int64)
    if self_loop_mode == 1:
        keep = src != dst
        last = np.full(n, -1, dtype=np.int64)
        for e in np.nonzero(~keep)[0]:
            last[src[e]] = max(last[src[e]], e)            # the LAST self loop in edge order
        ar = np.arange(n, dtype=np.int64)
        key, other, eid = np.concatenate([key[keep], ar]), np.concatenate([other[keep], ar]), np.concatenate([eid[keep], last])
    order = np.lexsort((eid, other, key))
    key, other, eid = key[order], other[order], eid[order]
    rowptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(rowptr, key + 1, 1)
    rowptr = np.cumsum(rowptr)
    val = np.where(eid >= 0, w[np.maximum(eid, 0)], 1.0).astype(w.dtype)
    lens = np.diff(rowptr)
    if self_loop_mode == 1:
        deg = np.array([val[rowptr[i]:rowptr[i + 1]].astype(np.float64).sum() for i in range(n)]).astype(np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            dinv = np.where(deg == 0, 0.0, 1.0 / np.sqrt(deg.astype(np.float64))).astype(np.float32)
    else:
        d = lens.astype(np.float32)
        with np.errstate(divide="ignore"):
            dinv = np.where(d > 0, np.sqrt(np.float32(1.0) / np.maximum(d, 1)), 0).astype(np.float32)
    return rowptr, other.astype(np.int32), eid, val, dinv


def scipy_weighted(rowptr, col, val, n_cols):
    import scipy.sparse as sp
    return sp.csr_matrix((np.asarray(val, np.float64), np.asarray(col, np.int64), np.asarray(rowptr, np.int64)),
                         shape=(rowptr.size - 1, n_cols))


def dense_gcn_adjacency(edge_index, w, n):
    """Differentiable (in w) dense Â of weighted PyG gcn_norm(add_self_loops=True): existing self loops dropped, node i's added
    loop takes the weight of i's last self loop (the CPU shim's loop_attr[idx] = attr) or 1, deg over targets, A[c, r]."""
    src, dst = edge_index[0], edge_index[1]
    keep = src != dst
    loop_w = torch.ones(n, dtype=w.dtype)
    loop_w = loop_w.index_put((src[~keep],), w[~keep])          # sequential put: the last loop wins, gradient to every loop
    r = torch.cat([src[keep], torch.arange(n)])
    c = torch.cat([dst[keep], torch.arange(n)])
    ww = torch.cat([w[keep], loop_w])
    deg = torch.zeros(n, dtype=w.dtype).index_add(0, c, ww)
    dis = deg.pow(-0.5)
    dis = torch.where(torch.isinf(dis), torch.zeros_like(dis), dis)
    return torch.zeros(n, n, dtype=w.dtype).index_put((c, r), dis[c] * ww * dis[r], accumulate=True)


def dense_gcn_conv_adjacency(edge_index, w, n):
    """Dense Â of DIFFormer's weighted gcn_conv: value = w d[c]^-1/2 d[r]^-1/2 with the UNWEIGHTED in-degree d over targets."""
    src, dst = edge_index[0], edge_index[1]
    d = torch.zeros(n, dtype=w.dtype).index_add(0, dst, torch.ones_like(w))
    dis = torch.nan_to_num(d.pow(-0.5), nan=0.0, posinf=0.0, neginf=0.0)
    return torch.zeros(n, n, dtype=w.dtype).index_put((dst, src), w * dis[dst] * dis[src], accumulate=True)


def edge_weight_grad(edge_index, weight, n, t, g, self_loop_mode=1):
    """dL/dw of L = <g, Â t> by the formulas of sgf_edge_weight_grad, walked over the CSR restatement (fp64):
    mode 1: dis_c dis_r <g_c, t_r> - 1/2 dis_c^3 dL/ddis_c, the added loop's share to every self loop of its node;
    mode 0 (gcn_conv): dis_c dis_r <g_c, t_r> with the unweighted dis."""
    t, g = np.asarray(t, np.float64), np.asarray(g, np.float64)
    rowptr, col, eid, val, _ = csr_weighted(edge_index, weight, n, False, self_loop_mode)
    A = scipy_weighted(rowptr, col, val, n)
    if self_loop_mode == 1:
        deg = np.asarray(A.sum(1)).ravel()
        dis = np.where(deg == 0, 0.0, 1.0 / np.sqrt(np.where(deg == 0, 1.0, deg)))
    else:
        lens = np.diff(rowptr)
        dis = np.where(lens > 0, 1.0 / np.sqrt(np.maximum(lens, 1)), 0.0)
    Ahat = A.multiply(dis[:, None]).multiply(dis[None, :]).tocsr()
    y, u = Ahat @ t, Ahat.T @ g
    ddis = np.zeros(n)
    if self_loop_mode == 1:
        nz = dis != 0
        ddis[nz] = ((g * y).sum(1)[nz] + (t * u).sum(1)[nz]) / dis[nz]
    src, dst = np.asarray(edge_index[0]), np.asarray(edge_index[1])
    out = np.zeros(src.size)
    loop_grad = np.zeros(n)
    for c in range(n):
        for j in range(rowptr[c], rowptr[c + 1]):
            r = col[j]
            d = dis[c] * dis[r] * (g[c] @ t[r]) - 0.5 * dis[c] ** 3 * ddis[c]
            if self_loop_mode == 1 and r == c:
                loop_grad[c] = d
            elif eid[j] >= 0:
                out[eid[j]] += d
    if self_loop_mode == 1:
        loops = src == dst
        out[loops] += loop_grad[src[loops]]
    return out
