"""numpy restatement of the graph index (include/sgpt_b200.h sgpt_graph_prune / sgpt_graph_search and
sgpt_b200.graph.merge_reverse / self_knn), written from the documented definitions, for tests to compare against bit for
bit."""
import numpy as np

M32 = 0xFFFFFFFF


def prune(knn: np.ndarray, degree: int) -> np.ndarray:
    """Rank-based detour pruning.  Entries outside [0, n), equal to the row, or repeating an earlier entry are empty;
    d_i = #{j < i : entry j valid and knn[a][i] in knn[knn[a][j]][0 .. i-1]}; the valid entries by (d_i, i), cut to
    degree, padded with -1."""
    knn = np.asarray(knn, dtype=np.int64)
    n, K = knn.shape
    # first[b, v]: the first position of v in row b (K when absent); entries outside [0, n) never match a valid entry
    first = np.full((n, n), K, dtype=np.int64)
    for p in range(K - 1, -1, -1):
        col = knn[:, p]
        ok = (col >= 0) & (col < n)
        first[np.nonzero(ok)[0], col[ok]] = p
    out = np.full((n, degree), -1, dtype=np.int32)
    idx = np.arange(K)
    for a in range(n):
        row = knn[a]
        valid = (row >= 0) & (row < n) & (row != a)
        seen = set()
        for i in range(K):
            if valid[i]:
                if int(row[i]) in seen:
                    valid[i] = False
                seen.add(int(row[i]))
        safe = np.where(valid, row, 0)
        pos = first[safe[:, None], safe[None, :]]  # [j, i]: first position of entry i in the list of entry j
        hit = valid[:, None] & valid[None, :] & (idx[:, None] < idx[None, :]) & (pos < idx[None, :])
        d = hit.sum(0)
        order = sorted((int(d[i]), i) for i in range(K) if valid[i])[:degree]
        out[a, :len(order)] = [row[i] for _, i in order]
    return out


def merge(pruned: np.ndarray) -> np.ndarray:
    """F[a] = the first degree / 2 entries; R[b] = every a with b in F[a] by (rank of b in F[a], a), cut to degree / 2;
    final[a] = F[a], R[a], the rest of a's list, repeats and -1 skipped, cut to degree, padded with -1."""
    n, degree = pruned.shape
    half = degree // 2
    rev = [[] for _ in range(n)]
    for a in range(n):
        for r in range(half):
            b = int(pruned[a, r])
            if b >= 0:
                rev[b].append((r, a))
    out = np.full((n, degree), -1, dtype=np.int32)
    for a in range(n):
        R = [x for _, x in sorted(rev[a])[:half]]
        row = []
        for x in list(pruned[a, :half]) + R + list(pruned[a, half:]):
            x = int(x)
            if x >= 0 and x not in row:
                row.append(x)
        row = row[:degree]
        out[a, :len(row)] = row
    return out


def self_knn(table: np.ndarray, K: int, allowed=None, id_base: int = 0) -> np.ndarray:
    """sgpt_b200.graph.self_knn from table fp32 [n, n] (table[a, x] = the exact search's score of row a's stored vector
    against position x): the exact top-(K + 1) of the allowed positions by (score descending, position ascending), tail
    -1; then row a's own id removed, or the last entry dropped when a is not among them.  Global ids int64 [n, K]."""
    n = table.shape[0]
    cand = np.arange(n) if allowed is None else np.nonzero(allowed)[0]
    out = np.full((n, K), -1, dtype=np.int64)
    for a in range(n):
        top = cand[np.lexsort((cand, -table[a, cand].astype(np.float64)))][:K + 1].tolist()  # -0 == +0
        top = [x for x in top if x != a][:K]
        out[a, :len(top)] = np.asarray(top, dtype=np.int64) + id_base
    return out


def score_table(score_block, nq: int, n: int, id_base: int = 0, block: int = 4096) -> np.ndarray:
    """The table fp32 [nq, n] that drives `search`, from a top-m scorer of at most `block` candidates per call:
    score_block(global ids int64 [m]) -> (scores [nq, m], global ids [nq, m]) in any order.  A candidate's score does not
    depend on the other candidates, so blocks of ids give the table of one call over all n.  Every position must come
    back exactly once per query; NaN counts as -1."""
    table = np.full((nq, n), np.nan, dtype=np.float32)
    seen = np.zeros((nq, n), dtype=np.int64)
    rows = np.arange(nq)[:, None]
    for c in range(0, n, block):
        m = min(block, n - c)
        s, i = score_block(np.arange(c, c + m, dtype=np.int64) + id_base)
        i = np.asarray(i, dtype=np.int64) - id_base
        if i.shape != (nq, m) or not ((i >= c) & (i < c + m)).all():
            raise AssertionError(f"block [{c}, {c + m}) came back with ids outside it")
        table[rows, i] = np.asarray(s, dtype=np.float32)
        np.add.at(seen, (np.broadcast_to(rows, i.shape), i), 1)
    if not (seen == 1).all():
        raise AssertionError("a position was scored more or less than once")
    return np.where(np.isnan(table), np.float32(-1), table)


def seed_hash(seed: int, q: int, j: int) -> int:
    x = (seed + 0x9E3779B1 * q + 0x85EBCA77 * j) & M32
    x ^= x >> 16
    x = (x * 0x85EBCA6B) & M32
    x ^= x >> 13
    x = (x * 0xC2B2AE35) & M32
    x ^= x >> 16
    return x


def search(table: np.ndarray, graph: np.ndarray, k: int, itopk: int, search_width: int, max_iterations: int,
           num_seeds: int, seeds=None, seed: int = 0, mask=None, id_base: int = 0):
    """The documented beam search over a score table fp32 [nq, n] (table[q, x] = s(q, x)).  Returns (scores fp32
    [nq, k], global ids int64 [nq, k], visited int32 [nq])."""
    nq, n = table.shape
    out_s = np.full((nq, k), -np.inf, dtype=np.float32)
    out_i = np.full((nq, k), -1, dtype=np.int64)
    visited = np.zeros(nq, dtype=np.int32)
    for q in range(nq):
        def entry(x):
            return (-float(table[q, x]), x, False)  # key order: score descending (-0 == +0), position ascending

        if seeds is not None:
            S = [int(x) for x in seeds[q][:num_seeds] if 0 <= x < n]
        else:
            S = [seed_hash(seed, q, j) % n for j in range(num_seeds)]
        V, new = set(), []
        for x in S:
            if x not in V:
                V.add(x)
                new.append(x)
        B = sorted(entry(x) for x in new)[:itopk]
        for _ in range(max_iterations):
            P = [e[1] for e in B if not e[2]][:search_width]
            if not P:
                break
            B = [(e[0], e[1], True) if e[1] in P else e for e in B]
            new = []
            for p in P:
                for e in graph[p]:
                    e = int(e)
                    if 0 <= e < n and e not in V:
                        V.add(e)
                        new.append(e)
            B = sorted(B + [entry(x) for x in new])[:itopk]
        res = [e for e in B if mask is None or mask[e[1]]][:k]
        for r, (_, x, _) in enumerate(res):
            out_s[q, r] = np.float32(table[q, x]) + np.float32(0)  # -0 is returned as +0
            out_i[q, r] = id_base + x
        visited[q] = len(V)
    return out_s, out_i, visited
