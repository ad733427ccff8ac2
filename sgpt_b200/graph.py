"""Graph index over a corpus shard: a fixed-degree, pruned k-NN graph searched by a beam search (CAGRA-style).

Every document keeps ``degree`` out-edges to other documents of the shard.  ``GraphIndex.build`` takes each row's exact
k-NN list (``CorpusShard.search`` of the shard's own stored rows), prunes it with rank-based detour counting
(``sgpt_graph_prune``) and merges in reverse edges so that documents that are nobody's near neighbour stay reachable.
A search (``sgpt_graph_search``, one CTA per query, one launch per batch) starts from ``num_seeds`` entry points, keeps the
``itopk`` best documents seen so far and repeatedly expands the best ``search_width`` of them that it has not expanded
yet, until all are expanded or ``max_iterations`` steps have run.  What a query costs grows with the rows it visits
rather than with n.

The rows are the shard's own: scores are ``sgpt_rerank``'s, bit for bit (for int8 shards, the exact search's bits), and
the top-k keeps the exact search's order (score descending, ties by ascending id).  The result is approximate: a document
the walk never reaches is not returned.  Deleted documents are still walked through, never returned.

``search(..., allow=)`` filters by a boolean mask, shared or one row per query (``sgpt_graph_search_filtered``): the walk
does not see the filter, and a query is answered with the best k allowed documents among those its walk visited, or by
the exact filtered search where the walk visited fewer than k allowed ones.  ``add()`` appends documents to the shard
and links them into the graph: their exact k-NN lists over the grown shard are pruned against the graph
(``sgpt_graph_prune_append``) and the reverse edges of all rows are merged again.  The forward lists of the old rows are
never revised, so ``build`` over n rows and ``add`` of m is not ``build`` over n + m: rebuild after heavy growth.
Documents added to the shard directly (``CorpusShard.add``) are not in the graph, and a search then raises.

Not supported: binary shards and indexes spread over several GPUs.
"""
from __future__ import annotations

import json
import os
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from .index import CorpusShard, _check_allow, _check_score_function
from .ivf import _rows_f32

FORMAT = "sgpt_b200.GraphIndex/1"
_KNN_WS_BYTES = 2 << 30   # search workspace of one block of k-NN queries
_MERGE_ROWS = 1 << 20     # rows per block of the duplicate removal in _merge
_VISITED_SLOTS = 16384    # visited-table slots the default max_iterations stays within (64 KB of shared memory)


def _check_degree(degree: int, K: int) -> None:
    if degree < 16 or degree > 128 or degree % 16 != 0:
        raise ValueError(f"degree={degree} must be a multiple of 16 in [16, 128]")
    if not degree <= K <= 256:
        raise ValueError(f"k-NN lists of {K} entries: need degree={degree} <= K <= 256")


def self_knn(shard: CorpusShard, K: int, score_function: str = "cos_sim",
             rows: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Each row's K nearest other rows by the exact search of its stored row (int8 rows dequantized): global ids int64
    [n, K], best first.  The search asks for K + 1 and drops the row's own id (or, where ties keep it out of the list,
    the last entry).  Deleted documents are not neighbours.  Query blocks are sized so that the search workspace stays
    around 2 GB.  ``rows``: local positions int64 [r] whose lists to compute (default: every row), giving [r, K]; their
    neighbours are still searched among all n rows."""
    n, dev, lib = shard.n, shard.device, _lib.lib()
    block = 1 << 16
    while block > 1 and lib.sgpt_search_workspace_bytes(block, n, K + 1) > _KNN_WS_BYTES:
        block //= 2
    which = None if rows is None else torch.as_tensor(rows).to(dev, torch.int64).reshape(-1)
    total = n if which is None else which.numel()
    out = torch.empty((total, K), dtype=torch.int64, device=dev)
    for a in range(0, total, block):
        pos = torch.arange(a, min(a + block, n), device=dev) if which is None else which[a:a + block]
        rows = shard.vectors.index_select(0, pos) if shard.dtype == "bf16" else _rows_f32(shard, pos)
        ids = shard.search(rows, K + 1, score_function)[1]
        own = (ids == (pos + shard.id_base)[:, None]).to(torch.int8)
        order = torch.sort(own, dim=1, stable=True)[1]  # the own id, if present, moves to the end
        out[a:a + len(pos)] = torch.gather(ids, 1, order)[:, :K]
    return out


def prune(knn: torch.Tensor, degree: int) -> torch.Tensor:
    """``sgpt_graph_prune`` of local positions int32 [n, K] (device): int32 [n, degree], -1 padded."""
    knn = knn.to(torch.int32).contiguous()
    n, K = knn.shape
    _check_degree(degree, K)
    out = torch.empty((n, degree), dtype=torch.int32, device=knn.device)
    with torch.cuda.device(knn.device):
        rc = _lib.lib().sgpt_graph_prune(knn.data_ptr(), n, K, degree, out.data_ptr(), _lib.current_stream())
    _lib.check(rc, "sgpt_graph_prune")
    return out


def prune_append(graph: torch.Tensor, knn: torch.Tensor, degree: int) -> torch.Tensor:
    """``sgpt_graph_prune_append``: the detour pruning of m rows appended after the n_old rows of ``graph`` (int32
    [n_old, degree], device), from their lists ``knn`` (local positions int32 [m, K], device): int32 [m, degree], -1
    padded.  An old position's list is its graph row, a new one's its knn row."""
    knn = knn.to(torch.int32).contiguous()
    graph = graph.to(knn.device, torch.int32).contiguous()
    m, K = knn.shape
    _check_degree(degree, K)
    out = torch.empty((m, degree), dtype=torch.int32, device=knn.device)
    with torch.cuda.device(knn.device):
        rc = _lib.lib().sgpt_graph_prune_append(_lib.ptr(graph) if graph.shape[0] else None, graph.shape[0], degree,
                                                knn.data_ptr(), m, K, out.data_ptr(), _lib.current_stream())
    _lib.check(rc, "sgpt_graph_prune_append")
    return out


def merge_reverse(pruned: torch.Tensor) -> torch.Tensor:
    """The reverse-edge merge of pruned lists int32 [n, degree] (-1 = empty): half = degree / 2, F[a] = the first half
    entries of a's list, R[b] = every a with b in F[a] ordered by (rank of b in F[a], a) and cut to half; the result is
    F[a], then R[a], then the rest of a's pruned list, repeats skipped, cut to degree and padded with -1.  Every sort key
    is unique, so the result is deterministic."""
    n, degree = pruned.shape
    half, dev = degree // 2, pruned.device
    F = pruned[:, :half].long()
    a = torch.arange(n, device=dev).repeat_interleave(half)
    r = torch.arange(half, device=dev).repeat(n)
    b = F.reshape(-1)
    ok = b >= 0
    a, r, b = a[ok], r[ok], b[ok]
    order = torch.sort((b * half + r) * n + a)[1]
    a, b = a[order], b[order]
    rank = torch.arange(len(b), device=dev) - torch.searchsorted(b, b)
    keep = rank < half
    R = torch.full((n, half), -1, dtype=torch.int64, device=dev)
    R[b[keep], rank[keep]] = a[keep]
    del a, r, b, order, rank, keep
    out = torch.empty((n, degree), dtype=torch.int32, device=dev)
    for s in range(0, n, _MERGE_ROWS):
        v = torch.cat([F[s:s + _MERGE_ROWS], R[s:s + _MERGE_ROWS], pruned[s:s + _MERGE_ROWS, half:].long()], 1)
        W = v.shape[1]
        pos = torch.arange(W, device=dev)
        valid = v >= 0
        sk, idx = torch.sort(torch.where(valid, v * W + pos, torch.iinfo(torch.int64).max), dim=1)
        val = sk // W
        dup = torch.zeros_like(valid)
        dup.scatter_(1, idx[:, 1:], (val[:, 1:] == val[:, :-1]) & (sk[:, 1:] != torch.iinfo(torch.int64).max))
        kept = valid & ~dup
        order = torch.sort((~kept).long() * W + pos, dim=1)[1][:, :degree]
        row = torch.gather(v, 1, order)
        out[s:s + _MERGE_ROWS] = torch.where(torch.gather(kept, 1, order), row, -1).to(torch.int32)
    return out


def default_max_iterations(itopk: int, search_width: int, degree: int, num_seeds: int) -> int:
    """2 itopk / search_width steps, cut so that the visited table stays within 16384 slots (64 KB of shared memory)."""
    cap = (_VISITED_SLOTS // 2 - num_seeds) // (search_width * degree)
    return max(1, min(2 * itopk // search_width, cap))


class GraphIndex:
    """Pruned k-NN graph over the rows of one ``CorpusShard`` (bf16 or int8).  Made by ``build``, ``from_knn`` or
    ``load``; ``graph`` int32 [n, degree] holds local positions, -1 = no edge.

    ``pruned`` (int32 [n, degree], host memory, or None) keeps the pruned lists before the reverse-edge merge and
    ``intermediate_degree`` the length K of the k-NN lists they came from; ``add`` needs both.  ``build`` and
    ``from_knn`` set them, ``save`` / ``load`` keep them; an index made from a bare graph can search but not add."""

    def __init__(self, shard: CorpusShard, graph: torch.Tensor, score_function: str):
        _check_score_function(score_function)
        if shard.dtype not in ("bf16", "int8"):
            raise ValueError(f"graph indexes are built over bf16 or int8 shards, not {shard.dtype!r}")
        self.shard, self.score_function = shard, score_function
        self.graph = graph.to(shard.device, torch.int32).contiguous()
        self.n, self.degree = self.graph.shape
        self.dim, self.id_base, self.device = shard.dim, shard.id_base, shard.device
        self.pruned: Optional[torch.Tensor] = None
        self.intermediate_degree: Optional[int] = None

    # ---- construction -------------------------------------------------------------------------------------------
    @classmethod
    def build(cls, shard: CorpusShard, degree: int = 32, intermediate_degree: int = 64,
              score_function: str = "cos_sim") -> "GraphIndex":
        """Exact k-NN lists of ``intermediate_degree`` entries (``self_knn``), then ``from_knn``.  The same shard gives
        the same graph."""
        _check_score_function(score_function)
        _check_degree(int(degree), int(intermediate_degree))
        return cls.from_knn(shard, self_knn(shard, int(intermediate_degree), score_function), degree, score_function)

    @classmethod
    def from_knn(cls, shard: CorpusShard, knn_ids: torch.Tensor, degree: int = 32,
                 score_function: str = "cos_sim") -> "GraphIndex":
        """The graph of caller-supplied neighbour lists: global ids int64 [n, K], best first (for example
        ``IVFIndex.search`` of the rows where an exact self-search is too slow).  Ids outside the shard and a row's own
        id are empty entries.  ``prune`` (detour pruning to ``degree``), then ``merge_reverse``."""
        knn = torch.as_tensor(knn_ids).to(shard.device, torch.int64)
        if knn.dim() != 2 or knn.shape[0] != shard.n:
            raise ValueError(f"knn_ids must be [n={shard.n}, K], got {tuple(knn.shape)}")
        _check_degree(int(degree), knn.shape[1])
        local = knn - shard.id_base
        local = torch.where((local >= 0) & (local < shard.n), local, -1)
        pruned = prune(local, int(degree))
        index = cls(shard, merge_reverse(pruned), score_function)
        index.pruned, index.intermediate_degree = pruned.cpu(), int(knn.shape[1])
        return index

    # ---- search -------------------------------------------------------------------------------------------------
    def _check_in_sync(self) -> None:
        if self.shard.n != self.n:
            raise ValueError(f"the shard holds {self.shard.n} documents but the graph was built over {self.n}; rows "
                             "added later are not in the graph: build it again")

    def search(self, queries: torch.Tensor, k: int, itopk: int = 64, search_width: int = 1,
               max_iterations: Optional[int] = None, num_seeds: Optional[int] = None,
               seeds: Optional[torch.Tensor] = None, seed: int = 0, return_visited: bool = False,
               allow: Optional[torch.Tensor] = None):
        """Top-k of fp32/bf16 queries [Q, D] by beam search: (scores fp32 [Q, k] descending, global ids int64 [Q, k]),
        tail (-inf, -1), and with ``return_visited`` the rows each query scored (int32 [Q]).

        ``seeds``: global ids [Q, s] of the entry points (ids outside the shard are skipped); otherwise ``num_seeds``
        hashed positions (default itopk) from ``seed``.  ``max_iterations`` defaults to ``default_max_iterations``:
        2 itopk / search_width steps, cut so the visited table stays within 64 KB of shared memory.

        ``allow``: boolean device tensor [n] (all queries) or [Q, n] (one row per query), indexed by global id -
        id_base as in ``CorpusShard.search``: only those documents may be returned (deleted ones never are).  The walk
        does not see the filter, so a query's result is the top-k of the allowed documents its walk visited (scores as
        without a filter).  A query whose walk visited fewer than k allowed documents is answered instead by the exact
        ``CorpusShard.search(allow=)`` of that query, so every query gets k results whenever k allowed documents exist;
        on an int8 shard those rows carry the same score bits as the walk would, on a bf16 shard the exact search's
        tensor-core scores, within fp32 rounding of ``sgpt_rerank``'s.  Finding those queries costs one host
        synchronisation per filtered search.  A filter also lowers recall: the walk spends its steps on documents the
        filter then drops (README, graph filter tables).  ``return_visited`` reports the walk's visited count for every
        query, fallback or not."""
        self._check_in_sync()
        k, itopk, search_width = int(k), int(itopk), int(search_width)
        if allow is not None:
            allow = _check_allow(allow, self.device, self.n, queries.shape[0])
        local = None
        if seeds is not None:
            s = torch.as_tensor(seeds).to(self.device, torch.int64)
            if s.dim() != 2 or s.shape[0] != queries.shape[0]:
                raise ValueError(f"seeds must be [Q={queries.shape[0]}, s], got {tuple(s.shape)}")
            s = s - self.id_base
            local = torch.where((s >= 0) & (s < self.n), s, -1).to(torch.int32).contiguous()
            num_seeds = s.shape[1]
        num_seeds = itopk if num_seeds is None else int(num_seeds)
        if max_iterations is None:
            max_iterations = default_max_iterations(itopk, search_width, self.degree, num_seeds)
        qb, q_scale, c_scale = self.shard._queries(queries, self.score_function)
        nq = qb.shape[0]
        mask, pitch = self.shard._mask(allow, nq)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        visited = torch.empty(nq, dtype=torch.int32, device=self.device) if return_visited else None
        args = (self.shard._dtype_id(), qb.data_ptr(), self.shard.vectors.data_ptr(), _lib.ptr(q_scale), c_scale, nq,
                self.n, self.dim, self.id_base, self.graph.data_ptr(), self.degree, _lib.ptr(local), num_seeds,
                int(seed) & 0xFFFFFFFF, itopk, search_width, int(max_iterations), k, _lib.ptr(mask))
        with torch.cuda.device(self.device):
            if allow is None:
                rc = _lib.lib().sgpt_graph_search(*args, out_s.data_ptr(), out_i.data_ptr(), _lib.ptr(visited),
                                                  _lib.current_stream())
            else:
                rc = _lib.lib().sgpt_graph_search_filtered(*args, pitch, out_s.data_ptr(), out_i.data_ptr(),
                                                           _lib.ptr(visited), _lib.current_stream())
        _lib.check(rc, "sgpt_graph_search_filtered" if allow is not None else "sgpt_graph_search")
        if allow is not None and nq > 0:
            short = (out_i[:, -1] < 0).nonzero().flatten()  # the host synchronisation
            if short.numel():
                rows_allow = allow.index_select(0, short) if allow.dim() == 2 else allow
                s, i = self.shard.search(queries.to(self.device).index_select(0, short), k, self.score_function,
                                         allow=rows_allow)
                out_s[short], out_i[short] = s, i
        return (out_s, out_i, visited) if return_visited else (out_s, out_i)

    # ---- growth -------------------------------------------------------------------------------------------------
    def add(self, emb: torch.Tensor) -> None:
        """Append fp32/bf16 embeddings [m, D] to the index's shard (``CorpusShard.add``) as documents id_base + n ..
        id_base + n + m - 1, and link them into the graph.

        Each new row's exact k-NN list of ``intermediate_degree`` entries over the grown shard (``self_knn``: its own
        id dropped, deleted documents excluded) is pruned against the graph (``prune_append``); the pruned lists of old
        and new rows are then merged again (``merge_reverse``, all n + m rows).  Old rows gain edges to new rows only
        through the reverse-edge half; their forward lists are never revised, so ``build`` over n rows and ``add`` of m
        is not ``build`` over n + m.  Rebuild after heavy growth.  Everything is checked before the shard changes: the
        shape, int32 ids, the shard's capacity, a graph in step with the shard, and pruned lists on the index (an index
        made from a bare graph, or loaded from a directory without them, cannot add)."""
        m = int(emb.shape[0])
        if emb.dim() != 2 or emb.shape[1] != self.dim:
            raise ValueError(f"add: embeddings must be [m, {self.dim}], got {tuple(emb.shape)}")
        if self.id_base + self.n + m >= 2 ** 31:
            raise ValueError(f"add: global ids must fit in int32 (id_base + n + m = {self.id_base + self.n + m} >= 2^31)")
        if self.n + m > self.shard.capacity:
            raise ValueError(f"add: shard capacity {self.shard.capacity} exceeded ({self.n} + {m})")
        self._check_in_sync()
        if self.pruned is None or self.intermediate_degree is None:
            raise ValueError("add: this index holds no pruned lists (made from a bare graph or loaded from a directory "
                             "without them): build it again with GraphIndex.build or GraphIndex.from_knn")
        if m == 0:
            return
        n = self.n
        self.shard.add(emb)
        knn = self_knn(self.shard, self.intermediate_degree, self.score_function,
                       rows=torch.arange(n, n + m, device=self.device)) - self.id_base
        knn = torch.where((knn >= 0) & (knn < n + m), knn, -1)
        pruned = torch.cat([self.pruned, prune_append(self.graph, knn, self.degree).cpu()])
        self.graph = merge_reverse(pruned.to(self.device))
        self.pruned, self.n = pruned, n + m

    @property
    def nbytes(self) -> int:
        """Device bytes of the graph (4 degree per document); the rows are the shard's."""
        return 4 * self.graph.numel()

    # ---- persistence --------------------------------------------------------------------------------------------
    def save(self, path: str) -> None:
        """One directory: graph.npy (int32 [n, degree]), pruned.npy (int32 [n, degree], when the index holds its pruned
        lists) and meta.json.  The shard is saved on its own."""
        os.makedirs(path, exist_ok=True)
        np.save(os.path.join(path, "graph.npy"), self.graph.cpu().numpy())
        meta = {"format": FORMAT, "n": self.n, "degree": self.degree, "dim": self.dim, "dtype": self.shard.dtype,
                "id_base": self.id_base, "score_function": self.score_function}
        if self.pruned is not None:
            np.save(os.path.join(path, "pruned.npy"), self.pruned.numpy())
            meta.update(pruned="pruned.npy", intermediate_degree=self.intermediate_degree)
        with open(os.path.join(path, "meta.json"), "w") as f:
            json.dump(meta, f)

    @classmethod
    def load(cls, path: str, shard: CorpusShard) -> "GraphIndex":
        """Reload a graph written by ``save`` over ``shard`` (identical search bits).  The files are checked against
        meta.json and the shard (n, dim, dtype, id_base) on the host before anything is allocated on the device."""
        with open(os.path.join(path, "meta.json")) as f:
            meta = json.load(f)
        if meta.get("format") != FORMAT:
            raise ValueError(f"{path}: not a GraphIndex directory ({meta})")
        _check_score_function(meta["score_function"])
        n, degree = int(meta["n"]), int(meta["degree"])
        want = (shard.n, shard.dim, shard.dtype, shard.id_base)
        have = (n, int(meta["dim"]), meta["dtype"], int(meta["id_base"]))
        if have != want:
            raise ValueError(f"{path}: the graph was built over (n, dim, dtype, id_base) = {have}, the shard holds {want}")
        g = np.load(os.path.join(path, "graph.npy"), mmap_mode="r")
        if g.shape != (n, degree) or g.dtype != np.int32 or degree < 1:
            raise ValueError(f"{path}: graph {g.shape}/{g.dtype} does not match meta {meta} (expected int32 [{n}, "
                             f"{degree}])")
        g = np.array(g)
        if g.size and (int(g.min()) < -1 or int(g.max()) >= n):
            raise ValueError(f"{path}: graph entries must lie in [-1, n={n})")
        pruned = None
        if meta.get("pruned") is not None:  # directories written without pruned lists load as a graph that cannot add
            K = int(meta.get("intermediate_degree", -1))
            if not degree <= K <= 256:
                raise ValueError(f"{path}: intermediate_degree={K} outside [degree={degree}, 256]")
            pruned = np.load(os.path.join(path, meta["pruned"]), mmap_mode="r")
            if pruned.shape != (n, degree) or pruned.dtype != np.int32:
                raise ValueError(f"{path}: pruned lists {pruned.shape}/{pruned.dtype} do not match meta {meta} "
                                 f"(expected int32 [{n}, {degree}])")
            pruned = np.array(pruned)
            if pruned.size and (int(pruned.min()) < -1 or int(pruned.max()) >= n):
                raise ValueError(f"{path}: pruned entries must lie in [-1, n={n})")
        index = cls(shard, torch.from_numpy(g), meta["score_function"])
        if pruned is not None:
            index.pruned, index.intermediate_degree = torch.from_numpy(pruned), K
        return index
