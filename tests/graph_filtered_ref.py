"""numpy restatement of the filtered graph search and of the pruning of appended rows (include/sgpt_b200.h
sgpt_graph_search_filtered / sgpt_graph_prune_append), written from the documented definitions, for tests to compare
against bit for bit.  The unfiltered search, prune and merge are in tests/graph_ref.py."""
import numpy as np

from tests.graph_ref import seed_hash


def search_filtered(table: np.ndarray, graph: np.ndarray, k: int, itopk: int, search_width: int, max_iterations: int,
                    num_seeds: int, seeds=None, seed: int = 0, mask=None, id_base: int = 0):
    """sgpt_graph_search_filtered: the walk of `search` without a mask, then the best k of the allowed positions of V
    (mask None, bool [n] shared, or bool [nq, n] per query).  Returns (scores fp32 [nq, k], global ids int64 [nq, k],
    visited int32 [nq])."""
    nq, n = table.shape
    out_s = np.full((nq, k), -np.inf, dtype=np.float32)
    out_i = np.full((nq, k), -1, dtype=np.int64)
    visited = np.zeros(nq, dtype=np.int32)
    for q in range(nq):
        if seeds is not None:
            S = [int(x) for x in seeds[q][:num_seeds] if 0 <= x < n]
        else:
            S = [seed_hash(seed, q, j) % n for j in range(num_seeds)]
        V = set(S)
        B = sorted((-float(table[q, x]), x, False) for x in V)[:itopk]
        for _ in range(max_iterations):
            P = [e[1] for e in B if not e[2]][:search_width]
            if not P:
                break
            B = [(e[0], e[1], True) if e[1] in P else e for e in B]
            new = {int(e) for p in P for e in graph[p] if 0 <= e < n and int(e) not in V}
            V |= new
            B = sorted(B + [(-float(table[q, x]), x, False) for x in new])[:itopk]
        allow = None if mask is None else (mask[q] if np.ndim(mask) == 2 else mask)
        res = sorted((-float(table[q, x]), x) for x in V if allow is None or allow[x])[:k]
        for r, (_, x) in enumerate(res):
            out_s[q, r] = np.float32(table[q, x]) + np.float32(0)  # -0 is returned as +0
            out_i[q, r] = id_base + x
        visited[q] = len(V)
    return out_s, out_i, visited


def prune_append(graph, knn_new: np.ndarray, degree: int) -> np.ndarray:
    """sgpt_graph_prune_append: rows a = n_old + r with list L = knn_new[r] (local positions); entries outside
    [0, n_old + m), equal to a, or repeating an earlier entry are empty; list(b) = graph[b] for b < n_old, else
    knn_new[b - n_old]; d_i = #{j < i : L[j] valid and L[i] in list(L[j])[0 .. i-1]}; the valid entries by (d_i, i), cut
    to degree, padded with -1.  graph int32 [n_old, degree] (None when n_old = 0)."""
    knn_new = np.asarray(knn_new, dtype=np.int64)
    m, K = knn_new.shape
    n_old = 0 if graph is None else len(graph)
    n = n_old + m
    out = np.full((m, degree), -1, dtype=np.int32)
    idx = np.arange(K)
    for r in range(m):
        a, L = n_old + r, knn_new[r]
        valid, seen = np.zeros(K, dtype=bool), set()
        for i in range(K):
            x = int(L[i])
            valid[i] = 0 <= x < n and x != a and x not in seen
            seen.add(x)
        lists = np.full((K, K), -2, dtype=np.int64)  # [j, p]: list(L[j]) (old rows: degree entries), -2 past its end
        for j in np.nonzero(valid)[0]:
            b = int(L[j])
            row = graph[b] if b < n_old else knn_new[b - n_old]
            lists[j, :len(row)] = row
        eq = lists[:, :, None] == L[None, None, :]  # [j, p, i]
        pos = np.where(eq.any(1), eq.argmax(1), K)  # [j, i]: first position of L[i] in list(L[j])
        hit = valid[:, None] & valid[None, :] & (idx[:, None] < idx[None, :]) & (pos < idx[None, :])
        d = hit.sum(0)
        order = sorted((int(d[i]), i) for i in range(K) if valid[i])[:degree]
        out[r, :len(order)] = [L[i] for _, i in order]
    return out
