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

Not supported: ``allow=`` filters, ``add()`` to a built graph (documents added to the shard later are not in the graph,
and a search then raises), binary shards and indexes spread over several GPUs.
"""
from __future__ import annotations

import json
import os
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from .index import CorpusShard, _check_score_function
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


def self_knn(shard: CorpusShard, K: int, score_function: str = "cos_sim") -> torch.Tensor:
    """Each row's K nearest other rows by the exact search of its stored row (int8 rows dequantized): global ids int64
    [n, K], best first.  The search asks for K + 1 and drops the row's own id (or, where ties keep it out of the list,
    the last entry).  Deleted documents are not neighbours.  Query blocks are sized so that the search workspace stays
    around 2 GB."""
    n, dev, lib = shard.n, shard.device, _lib.lib()
    block = 1 << 16
    while block > 1 and lib.sgpt_search_workspace_bytes(block, n, K + 1) > _KNN_WS_BYTES:
        block //= 2
    out = torch.empty((n, K), dtype=torch.int64, device=dev)
    for a in range(0, n, block):
        pos = torch.arange(a, min(a + block, n), device=dev)
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
    ``load``; ``graph`` int32 [n, degree] holds local positions, -1 = no edge."""

    def __init__(self, shard: CorpusShard, graph: torch.Tensor, score_function: str):
        _check_score_function(score_function)
        if shard.dtype not in ("bf16", "int8"):
            raise ValueError(f"graph indexes are built over bf16 or int8 shards, not {shard.dtype!r}")
        self.shard, self.score_function = shard, score_function
        self.graph = graph.to(shard.device, torch.int32).contiguous()
        self.n, self.degree = self.graph.shape
        self.dim, self.id_base, self.device = shard.dim, shard.id_base, shard.device

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
        return cls(shard, merge_reverse(prune(local, int(degree))), score_function)

    # ---- search -------------------------------------------------------------------------------------------------
    def search(self, queries: torch.Tensor, k: int, itopk: int = 64, search_width: int = 1,
               max_iterations: Optional[int] = None, num_seeds: Optional[int] = None,
               seeds: Optional[torch.Tensor] = None, seed: int = 0, return_visited: bool = False):
        """Top-k of fp32/bf16 queries [Q, D] by beam search: (scores fp32 [Q, k] descending, global ids int64 [Q, k]),
        tail (-inf, -1), and with ``return_visited`` the rows each query scored (int32 [Q]).

        ``seeds``: global ids [Q, s] of the entry points (ids outside the shard are skipped); otherwise ``num_seeds``
        hashed positions (default itopk) from ``seed``.  ``max_iterations`` defaults to ``default_max_iterations``:
        2 itopk / search_width steps, cut so the visited table stays within 64 KB of shared memory."""
        if self.shard.n != self.n:
            raise ValueError(f"the shard holds {self.shard.n} documents but the graph was built over {self.n}; rows "
                             "added later are not in the graph: build it again")
        k, itopk, search_width = int(k), int(itopk), int(search_width)
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
        mask, _ = self.shard._mask(None, nq)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        visited = torch.empty(nq, dtype=torch.int32, device=self.device) if return_visited else None
        with torch.cuda.device(self.device):
            rc = _lib.lib().sgpt_graph_search(
                self.shard._dtype_id(), qb.data_ptr(), self.shard.vectors.data_ptr(), _lib.ptr(q_scale), c_scale, nq,
                self.n, self.dim, self.id_base, self.graph.data_ptr(), self.degree, _lib.ptr(local), num_seeds,
                int(seed) & 0xFFFFFFFF, itopk, search_width, int(max_iterations), k, _lib.ptr(mask), out_s.data_ptr(),
                out_i.data_ptr(), _lib.ptr(visited), _lib.current_stream())
        _lib.check(rc, "sgpt_graph_search")
        return (out_s, out_i, visited) if return_visited else (out_s, out_i)

    @property
    def nbytes(self) -> int:
        """Device bytes of the graph (4 degree per document); the rows are the shard's."""
        return 4 * self.graph.numel()

    # ---- persistence --------------------------------------------------------------------------------------------
    def save(self, path: str) -> None:
        """One directory: graph.npy (int32 [n, degree]) and meta.json.  The shard is saved on its own."""
        os.makedirs(path, exist_ok=True)
        np.save(os.path.join(path, "graph.npy"), self.graph.cpu().numpy())
        with open(os.path.join(path, "meta.json"), "w") as f:
            json.dump({"format": FORMAT, "n": self.n, "degree": self.degree, "dim": self.dim, "dtype": self.shard.dtype,
                       "id_base": self.id_base, "score_function": self.score_function}, f)

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
        return cls(shard, torch.from_numpy(g), meta["score_function"])
