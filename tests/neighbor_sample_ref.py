"""numpy restatement of the device neighbour sampler (sgformer_b200/csrc/sample.cu, DESIGN.md §4.15): the counter-based draws,
Floyd's algorithm, first-appearance relabelling in (hop, frontier position, slot) order and the (target, slot)-ordered edge list.
`brute_force` states the same semantics the slow, obvious way (set of taken positions, dict of seen nodes) for the CPU tests."""
import numpy as np

M1, M2 = np.uint64(0xff51afd7ed558ccd), np.uint64(0xc4ceb9fe1a85ec53)
PHI, C2 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xC2B2AE3D27D4EB4F)


def fmix64(x):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(33)); x = x * M1
        x = x ^ (x >> np.uint64(33)); x = x * M2
        x = x ^ (x >> np.uint64(33))
    return x


def draw(seed, hop, v, d):
    """The 64-bit draw d of hop `hop` at target v (vectorised over v and d)."""
    v = np.asarray(v, dtype=np.int64).astype(np.uint64)
    d = np.asarray(d, dtype=np.int64).astype(np.uint64)
    with np.errstate(over="ignore"):
        h = fmix64(np.uint64(seed) ^ (v * PHI))
        return fmix64(h ^ (((np.uint64(hop) << np.uint64(32)) | d) * C2))


def uniform_below(h, m):
    """Integer in [0, m) from the high 32 bits of h: ((h >> 32) * m) >> 32."""
    return ((np.asarray(h, dtype=np.uint64) >> np.uint64(32)) * np.asarray(m, dtype=np.uint64)) >> np.uint64(32)


def row_positions(seed, hop, v, deg, k, width):
    """Sorted entry positions row v (degree deg) takes at hop `hop` (scalar version)."""
    if k < 0 or deg <= k:
        return list(range(min(deg, width)))
    taken = []
    for d in range(k):
        j = deg - k + d
        t = int(uniform_below(draw(seed, hop, v, d), j + 1))
        taken.append(j if t in taken else t)
    return sorted(taken)


def hop_positions(seed, hop, vs, degs, k):
    """Vectorised Floyd for rows with deg > k: [rows, k] sorted positions."""
    vs, degs = np.asarray(vs, dtype=np.int64), np.asarray(degs, dtype=np.int64)
    S = np.empty((vs.size, k), dtype=np.int64)
    for d in range(k):
        j = degs - k + d
        t = uniform_below(draw(seed, hop, vs, d), j + 1).astype(np.int64)
        hit = (S[:, :d] == t[:, None]).any(1) if d else np.zeros(vs.size, dtype=bool)
        S[:, d] = np.where(hit, j, t)
    return np.sort(S, axis=1)


def sample(rowptr, col, seeds, num_neighbors, seed, capacity=None):
    """-> (idx int64 [b] global ids in local order, edge_index int64 [2, e] (source local, target local) in (target, slot) order,
    need = largest row met by a k = -1 hop).  rowptr / col: the parent CSR (rows = targets, sorted entries)."""
    rowptr, col = np.asarray(rowptr, dtype=np.int64), np.asarray(col, dtype=np.int64)
    n = rowptr.size - 1
    local = np.full(n, -1, dtype=np.int64)
    seeds = np.asarray(seeds, dtype=np.int64)
    local[seeds] = np.arange(seeds.size)
    idx = [seeds]
    frontier, f0 = seeds, 0
    nn = seeds.size
    src_l, dst_l, need = [], [], 0
    for hop, k in enumerate(num_neighbors):
        width = k if k >= 0 else capacity
        degs = rowptr[frontier + 1] - rowptr[frontier]
        pos = [None] * frontier.size
        if k >= 0:
            big = np.nonzero(degs > k)[0]
            if big.size:
                P = hop_positions(seed, hop, frontier[big], degs[big], k)
                for r, i in enumerate(big):
                    pos[i] = P[r]
        else:
            need = max(need, int(degs.max()) if degs.size else 0)
        for i in range(frontier.size):
            if pos[i] is None:
                pos[i] = np.arange(min(int(degs[i]), width))
        cnt = np.array([p.size for p in pos], dtype=np.int64)
        flat_pos = np.concatenate(pos) if frontier.size else np.zeros(0, np.int64)
        rows = np.repeat(np.arange(frontier.size), cnt)
        cand = col[rowptr[frontier[rows]] + flat_pos] if rows.size else np.zeros(0, np.int64)
        # first appearance in (frontier position, slot) order among the nodes not seen yet
        unseen = local[cand] < 0
        _, first = np.unique(cand[unseen], return_index=True)
        new = cand[unseen][np.sort(first)]
        local[new] = nn + np.arange(new.size)
        idx.append(new)
        src_l.append(local[cand])
        dst_l.append(f0 + rows)
        f0, nn = nn, nn + new.size
        frontier = new
    idx = np.concatenate(idx)
    ei = np.stack([np.concatenate(src_l) if src_l else np.zeros(0, np.int64),
                   np.concatenate(dst_l) if dst_l else np.zeros(0, np.int64)]).astype(np.int64)
    return idx, ei, need


def brute_force(edges, n, seeds, num_neighbors, seed, capacity=None):
    """The semantics from the edge list: row v = sources of v's in-edges sorted (duplicates kept); scalar Floyd per row; a
    dict of seen nodes; edges appended per (hop, frontier row, slot)."""
    rows = [sorted(int(s) for s, t in zip(*edges) if t == v) for v in range(n)]
    seen = {int(s): i for i, s in enumerate(seeds)}
    order = [int(s) for s in seeds]
    frontier, f0 = list(order), 0
    out = []
    for hop, k in enumerate(num_neighbors):
        width = k if k >= 0 else capacity
        new = []
        for i, v in enumerate(frontier):
            for p in row_positions(seed, hop, v, len(rows[v]), k, width):
                u = rows[v][p]
                if u not in seen:
                    seen[u] = len(order)
                    order.append(u)
                    new.append(u)
                out.append((seen[u], f0 + i))
        f0 += len(frontier)
        frontier = new
    ei = np.array(out, dtype=np.int64).T.reshape(2, -1)
    return np.array(order, dtype=np.int64), ei


def csr_of(edges, n):
    """Parent CSR of an edge list in self_loop_mode 0 (rows = targets, entries = sources sorted, duplicates kept)."""
    src, dst = np.asarray(edges[0], dtype=np.int64), np.asarray(edges[1], dtype=np.int64)
    order = np.lexsort((src, dst))
    rowptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(rowptr, dst + 1, 1)
    return np.cumsum(rowptr), src[order]
