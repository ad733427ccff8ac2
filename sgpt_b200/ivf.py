"""Inverted-file (IVF) index over a corpus shard: k-means lists, and a search that scans only each query's nearest lists.

The index splits the documents into ``nlist`` lists around k-means centroids and stores them list by list.  A query
probes the ``nprobe`` centroids with the highest score (the exact search over the centroids: score descending, ties by
ascending list id) and scans only the documents of those lists, with one grouped wgmma pass per probed list shared by
every query that probes it (include/sgpt_b200.h ``sgpt_ivf_search``).

The search is exact relative to its lists: ``IVFIndex.search`` returns exactly what ``CorpusShard.search`` returns over
the undeleted documents of the probed lists — the same scores of the same stored rows, the same order and tie rule on
global ids, the tail (-inf, -1) when fewer than k documents are probed.  ``nprobe == nlist`` is the exact search.
Recall against the full exact search depends on the clustering only.

``IVFIndex.range_search`` is the threshold counterpart (``sgpt_ivf_range_search``): exactly ``CorpusShard.range_search``
over the undeleted documents of the probed lists.  ``paraphrase_mining_embeddings`` and ``community_detection``
(mining.py) run over an index with the stored rows themselves as queries.
"""
from __future__ import annotations

import json
import os
from typing import Optional, Tuple, Union

import numpy as np
import torch

from . import _lib
from .index import (CorpusShard, _bit_slice, _check_allow, _check_score_function, _grown_range, _mask_rows,
                    unpack_mask)

FORMAT = "sgpt_b200.IVFIndex/1"
_ASSIGN_BYTES = 256 << 20  # score matrix of one assignment batch (dense search over the centroids)


def _rows_f32(shard: CorpusShard, pos: torch.Tensor) -> torch.Tensor:
    """fp32 rows of the shard at positions `pos` as stored (int8: dequantized with the per-row scale)."""
    v = shard.vectors.index_select(0, pos).float()
    if shard.dtype == "int8":
        v.mul_(shard.scales.index_select(0, pos)[:, None])
    return v


def _assign(cshard: CorpusShard, x: torch.Tensor, score_function: str) -> torch.Tensor:
    """Best centroid of every row of x (exact search, k = 1), int64 [m] on the device."""
    step = max(1, min(65536, _ASSIGN_BYTES // (4 * max(cshard.n, 1))))
    out = [cshard.search(x[i:i + step], 1, score_function)[1][:, 0] for i in range(0, x.shape[0], step)]
    return torch.cat(out) if out else torch.empty(0, dtype=torch.int64, device=x.device)


def _assign_rows(cshard: CorpusShard, shard: CorpusShard, score_function: str) -> torch.Tensor:
    """Best centroid of every stored row of `shard` (dequantized), in batches of ~256 MB of fp32 rows: int64 [n]."""
    n, D, dev = shard.n, shard.dim, shard.device
    bs = max(1, min(65536, _ASSIGN_BYTES // (4 * D)))
    return torch.cat([_assign(cshard, _rows_f32(shard, torch.arange(i, min(i + bs, n), device=dev)), score_function)
                      for i in range(0, n, bs)])


def _kmeans(x: torch.Tensor, nlist: int, n_iter: int, g: torch.Generator, score_function: str) -> torch.Tensor:
    """Coarse k-means of ``IVFIndex.build`` (and ``IVFPQIndex.train``) over the training rows x fp32 [T, D] (device,
    already normalized for cos_sim): centroids fp32 [nlist, D] on x's device.  Starts from x[:nlist]; assignment is the
    exact search (k = 1) against the centroids as a bf16 shard, the update is the mean of the assigned rows summed in fp64
    on the host in row order (no atomics), an empty list is re-seeded with a row drawn from `g`, and for cos_sim the
    centroids are normalized (spherical k-means)."""
    T, D = x.shape
    dev, cos = x.device, score_function == "cos_sim"
    cent = x[:nlist].clone()
    step = max(1, (64 << 20) // (8 * D))  # rows per host transfer of the update
    for _ in range(int(n_iter)):
        a = _assign(CorpusShard.from_embeddings(cent, device=dev), x, score_function).cpu()
        sums = torch.zeros(nlist, D, dtype=torch.float64)
        for i in range(0, T, step):  # index_add_ on the host adds the rows in order: reproducible bits
            sums.index_add_(0, a[i:i + step], x[i:i + step].cpu().double())
        counts = torch.bincount(a, minlength=nlist)
        new = sums / counts.clamp(min=1)[:, None].double()
        empty = (counts == 0).nonzero().flatten()
        if len(empty):
            new[empty] = x[torch.randint(T, (len(empty),), generator=g).to(dev)].double().cpu()
        if cos:
            new = torch.nn.functional.normalize(new, dim=1)
        cent = new.float().to(dev)
    return cent


def _merge_lists(offsets: torch.Tensor, lists: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Destinations of an append to list-ordered storage (``IVFIndex.add``, ``IVFPQIndex.add``): the n old positions
    (offsets int64 [nlist + 1], device) and m new rows whose lists are `lists` int64 [m].  Every list keeps its rows in
    their order, followed by its new rows in input order.  Returns (new offsets, old_dest int64 [n], new_dest int64 [m])."""
    nlist, dev = offsets.numel() - 1, offsets.device
    n, m = int(offsets[-1]), lists.numel()
    added = torch.bincount(lists, minlength=nlist)
    shift = torch.cumsum(added, 0) - added  # new rows inserted before list l
    sizes = offsets[1:] - offsets[:-1]
    new_offsets = offsets.clone()
    new_offsets[1:] += torch.cumsum(added, 0)
    # destinations: old position p of list l -> p + shift[l]; new rows after their list's old rows, in input order
    old_list = torch.repeat_interleave(torch.arange(nlist, device=dev), sizes, output_size=n)
    old_dest = torch.arange(n, device=dev) + shift[old_list]
    order = torch.sort(lists, stable=True).indices
    rank = torch.arange(m, device=dev) - shift[lists[order]]  # place inside the list's new rows
    new_dest = torch.empty(m, dtype=torch.int64, device=dev)
    new_dest[order] = new_offsets[lists[order]] + sizes[lists[order]] + rank
    return new_offsets, old_dest, new_dest


class IVFIndex:
    """IVF index on one GPU.  Built by ``IVFIndex.build`` or ``IVFIndex.load``.

    ``shard`` is a ``CorpusShard`` of the rows in list order whose ids are the positions (0 .. n-1); list l is positions
    ``offsets[l] .. offsets[l+1]`` and ``ids[pos]`` (int32) the global id of position pos.  ``centroids`` fp32
    [nlist, D] are searched as a bf16 shard to choose the probes.  Deletions live in the inner shard's bitmap."""

    def __init__(self, shard: CorpusShard, centroids: torch.Tensor, offsets: torch.Tensor, ids: torch.Tensor,
                 id_base: int, score_function: str):
        _check_score_function(score_function)
        self.score_function, self.id_base = score_function, int(id_base)
        self.device = shard.device
        self.centroids = centroids.to(self.device, torch.float32).contiguous()
        self.nlist, self.dim, self.dtype = self.centroids.shape[0], shard.dim, shard.dtype
        self._cshard = CorpusShard.from_embeddings(self.centroids, device=self.device)
        self._set_lists(shard, offsets, ids)

    def _set_lists(self, shard: CorpusShard, offsets: torch.Tensor, ids: torch.Tensor) -> None:
        """The list-ordered rows and their layout (``build``, ``load``, ``add``)."""
        self.shard, self.n = shard, shard.n
        self.offsets = offsets.to(self.device, torch.int64).contiguous()
        self.ids = ids.to(self.device, torch.int32).contiguous()
        self.list_sizes = (self.offsets[1:] - self.offsets[:-1]).cpu()
        self.max_list_len = int(self.list_sizes.max()) if self.nlist else 0
        # position of every global id (ids are a permutation of id_base .. id_base + n - 1)
        self._pos = torch.empty(self.n, dtype=torch.int64, device=self.device)
        self._pos[self.ids.long() - self.id_base] = torch.arange(self.n, device=self.device)
        self._ws: Optional[torch.Tensor] = None

    # ---- construction -------------------------------------------------------------------------------------------
    @classmethod
    def build(cls, source: Union[CorpusShard, torch.Tensor], nlist: int, score_function: str = "cos_sim",
              dtype: Optional[str] = None, n_iter: int = 10, train_size: Optional[int] = None, seed: int = 0,
              device=None) -> "IVFIndex":
        """k-means lists over ``source`` (a ``CorpusShard``, or fp32/bf16 embeddings [n, D] stored as a ``dtype`` shard
        first, "bf16" by default; a shard's own dtype is kept) and a list-ordered copy of its stored rows.

        k-means runs on ``train_size`` rows (default min(n, 64 nlist)) drawn with ``seed``: assignment is the library's
        exact search (k = 1) against the centroids as a bf16 shard, the update is the mean of the assigned rows summed in
        fp64 on the host in row order (no atomics), and an empty list is re-seeded with a row drawn from the same seeded
        generator.  For cos_sim the training rows are normalized first (spherical k-means).  The same inputs and seed give
        bit-identical centroids, offsets and ids on the same device.  Every row then goes to its best centroid; the rows
        keep their stored bits (a source shard's rows and scales are copied, not re-quantized), so scores equal the
        source's.  A source shard's deletions carry over.

        Peak device memory: the source plus the index (rows, scales, int32 ids, centroids), plus one batch of dequantized
        rows and its centroid scores (~256 MB) during the assignment."""
        _check_score_function(score_function)
        if isinstance(source, CorpusShard):
            if dtype is not None and dtype != source.dtype:
                raise ValueError(f"dtype {dtype!r} differs from the source shard's {source.dtype!r}")
            src = source
        else:
            src = CorpusShard.from_embeddings(torch.as_tensor(source), device=device, dtype=dtype or "bf16")
        n, D, dev = src.n, src.dim, src.device
        nlist = int(nlist)
        if not 1 <= nlist <= n:
            raise ValueError(f"nlist={nlist} must lie in [1, n={n}]")
        if src.id_base < 0 or src.id_base + n >= 2 ** 31:
            raise ValueError("global ids must fit in int32 (id_base + n < 2^31)")
        cos = score_function == "cos_sim"
        g = torch.Generator().manual_seed(int(seed))
        T = min(n, int(train_size) if train_size is not None else 64 * nlist)
        if T < nlist:
            raise ValueError(f"train_size={T} is below nlist={nlist}")
        sample = torch.randperm(n, generator=g)[:T].to(dev)
        x = _rows_f32(src, sample)
        if cos:
            x = torch.nn.functional.normalize(x, dim=1)
        cent = _kmeans(x, nlist, n_iter, g, score_function)
        del x
        assign = _assign_rows(CorpusShard.from_embeddings(cent, device=dev), src, score_function)
        perm = torch.sort(assign, stable=True).indices
        offsets = torch.zeros(nlist + 1, dtype=torch.int64, device=dev)
        torch.cumsum(torch.bincount(assign, minlength=nlist), 0, out=offsets[1:])
        inner = CorpusShard(D, n, device=dev, dtype=src.dtype)
        torch.index_select(src.vectors[:n], 0, perm, out=inner.vectors[:n])
        if src.dtype == "int8":
            torch.index_select(src.scales[:n], 0, perm, out=inner.scales[:n])
            torch.index_select(src.cos_scales[:n], 0, perm, out=inner.cos_scales[:n])
        else:
            torch.index_select(src.inv_norms[:n], 0, perm, out=inner.inv_norms[:n])
        inner.n = n
        if src._deleted["any"]:
            deleted = unpack_mask(_bit_slice(src._deleted["words"], src._deleted_at, n), n)
            inner.remove(deleted[perm].nonzero().flatten())
        return cls(inner, cent, offsets, (perm + src.id_base).to(torch.int32), src.id_base, score_function)

    # ---- search -------------------------------------------------------------------------------------------------
    def probe(self, queries: torch.Tensor, nprobe: int) -> torch.Tensor:
        """The ``nprobe`` lists each query scans: int32 [Q, nprobe], best centroid first (score descending, ties by
        ascending list id), from the exact search over the centroids."""
        if not 1 <= int(nprobe) <= self.nlist:
            raise ValueError(f"nprobe={nprobe} must lie in [1, nlist={self.nlist}]")
        return self._cshard.search(queries.to(self.device), int(nprobe), self.score_function)[1].to(torch.int32)

    def search(self, queries: torch.Tensor, k: int, nprobe: int,
               allow: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Top-k of the undeleted documents in each query's ``nprobe`` probed lists, for fp32/bf16 queries [Q, D]:
        (scores fp32 [Q, k] descending, global ids int64 [Q, k]), tail (-inf, -1) when fewer than k are probed.  Scores,
        order and ties are those of ``CorpusShard.search`` on the same stored rows.

        ``allow``: boolean device tensor [n] (all queries) or [Q, n] (one row per query), indexed by global id - id_base
        as in ``CorpusShard.search``: only those documents may be returned.  The probes do not depend on the filter —
        they are still the ``nprobe`` nearest centroids — so a selective filter can return fewer than k documents even
        where the whole index holds more.  The result is exactly ``CorpusShard.search(allow=allow & probed)``."""
        if not 1 <= int(k) <= 4096:
            raise ValueError(f"k={k} must lie in [1, 4096]")
        probes = self.probe(queries, nprobe)
        qb, q_scale, c_scale = self.shard._queries(queries, self.score_function)
        return self._search_rows(qb, q_scale, c_scale, probes, int(k), self._list_mask(allow, qb.shape[0]))

    def range_search(self, queries: torch.Tensor, threshold: float, nprobe: int,
                     allow: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Every undeleted document of each query's ``nprobe`` probed lists whose score is >= threshold, for fp32/bf16
        queries [Q, D]: (offsets int64 [Q+1], scores fp32 [E], global ids int64 [E]) on the device, query q's documents at
        offsets[q] .. offsets[q+1] in ascending id order.  Queries are converted and scored as in ``search``; a NaN score
        counts as -1.  The output buffer starts and grows once as in ``CorpusShard.range_search``.

        ``allow`` as in ``search`` (boolean [n] or [Q, n], indexed by global id - id_base); the probes ignore it.  The
        result is exactly ``CorpusShard.range_search(allow=allow & probed)`` of the source documents, deleted ones left
        out: the same offsets, scores and ids."""
        if threshold != threshold:
            raise ValueError("threshold is NaN")
        probes = self.probe(queries, nprobe)
        qb, q_scale, c_scale = self.shard._queries(queries, self.score_function)
        return self._range_rows(qb, q_scale, c_scale, probes, threshold, self._list_mask(allow, qb.shape[0]))

    # ---- the calls behind search / range_search, on query rows in the shard's format --------------------------------
    def _workspace(self, need: int, what: str) -> torch.Tensor:
        if need < 0:
            raise ValueError(f"{what} rejects these arguments: {_lib.lib().sgpt_last_error().decode()}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def _list_mask(self, allow: Optional[torch.Tensor], nq: int) -> Tuple[Optional[torch.Tensor], int]:
        """(bitmap, pitch) over list positions: `allow` (document order) permuted to list order with one gather, then
        packed with the deletions ANDed in (``CorpusShard._mask``)."""
        if allow is None:
            return self.shard._mask(None, nq)
        allow = _check_allow(allow, self.device, self.n, nq)
        return self.shard._mask(allow.index_select(-1, self.ids - self.id_base), nq)

    def _search_rows(self, qb, q_scale, c_scale, probes, k: int, mask) -> Tuple[torch.Tensor, torch.Tensor]:
        """sgpt_ivf_search (shared or no bitmap) or sgpt_ivf_search_masked (per-query bitmaps) of prepared rows."""
        nq, nprobe = qb.shape[0], probes.shape[1]
        dt, lib = self.shard._dtype_id(), _lib.lib()
        ws = self._workspace(lib.sgpt_ivf_search_workspace_bytes(dt, nq, self.nlist, nprobe, self.max_list_len,
                                                                 self.dim), "sgpt_ivf_search")
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            if mask[1] == 0:
                rc = lib.sgpt_ivf_search(dt, qb.data_ptr(), self.shard.vectors.data_ptr(), _lib.ptr(q_scale), c_scale,
                                         nq, self.n, self.dim, self.offsets.data_ptr(), self.nlist, self.max_list_len,
                                         self.ids.data_ptr(), probes.data_ptr(), nprobe, k, _lib.ptr(mask[0]),
                                         out_s.data_ptr(), out_i.data_ptr(), ws.data_ptr(), ws.numel(),
                                         _lib.current_stream())
            else:
                rc = lib.sgpt_ivf_search_masked(dt, qb.data_ptr(), self.shard.vectors.data_ptr(), _lib.ptr(q_scale),
                                                c_scale, nq, self.n, self.dim, self.offsets.data_ptr(), self.nlist,
                                                self.max_list_len, self.ids.data_ptr(), probes.data_ptr(), nprobe, k,
                                                _lib.ptr(mask[0]), mask[1], out_s.data_ptr(), out_i.data_ptr(),
                                                ws.data_ptr(), ws.numel(), _lib.current_stream())
        _lib.check(rc, "sgpt_ivf_search")
        return out_s, out_i

    def _range_call(self, qb, q_scale, c_scale, probes, threshold: float, mask, counts: torch.Tensor, cap: int,
                    out_s: Optional[torch.Tensor], out_i: Optional[torch.Tensor]) -> None:
        """One sgpt_ivf_range_search of prepared rows: counts int64 [Q] always, the entries of the queries that fit into
        `cap` into out_s / out_i in the entry point's order (probe order, then list position)."""
        nq, nprobe = qb.shape[0], probes.shape[1]
        dt, lib = self.shard._dtype_id(), _lib.lib()
        ws = self._workspace(lib.sgpt_ivf_range_search_workspace_bytes(dt, nq, self.nlist, nprobe, self.max_list_len,
                                                                       self.dim), "sgpt_ivf_range_search")
        with torch.cuda.device(self.device):
            rc = lib.sgpt_ivf_range_search(dt, qb.data_ptr(), self.shard.vectors.data_ptr(), _lib.ptr(q_scale), c_scale,
                                           nq, self.n, self.dim, self.offsets.data_ptr(), self.nlist, self.max_list_len,
                                           self.ids.data_ptr(), probes.data_ptr(), nprobe, float(threshold),
                                           _lib.ptr(mask[0]), mask[1], counts.data_ptr(), cap, _lib.ptr(out_s),
                                           _lib.ptr(out_i), ws.data_ptr(), ws.numel(), _lib.current_stream())
        _lib.check(rc, "sgpt_ivf_range_search")

    def _range_rows(self, qb, q_scale, c_scale, probes, threshold: float, mask, capacity: Optional[int] = None
                    ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """``_range_call`` through the grow-once buffer of ``CorpusShard._range``, then every query's entries sorted by
        global id with one device sort of the unique keys q * 2^31 + id."""
        nq = qb.shape[0]

        def run(first, counts, cap, out_s, out_i):
            self._range_call(qb[first:], None if q_scale is None else q_scale[first:], c_scale, probes[first:],
                             threshold, _mask_rows(mask, first), counts, cap, out_s, out_i)

        offsets, s, ids = _grown_range(nq, self.device, run, capacity)
        q = torch.repeat_interleave(torch.arange(nq, device=self.device), offsets[1:] - offsets[:-1],
                                    output_size=s.numel())
        o = torch.sort(q * (1 << 31) + ids).indices
        return offsets, s[o], ids[o]

    # ---- the index's own rows as queries (mining) -------------------------------------------------------------------
    def _undeleted(self) -> Optional[torch.Tensor]:
        """Positions of the undeleted rows, ascending (int64), or None when nothing is deleted."""
        if self.shard.n_deleted == 0:
            return None
        deleted = unpack_mask(_bit_slice(self.shard._deleted["words"], self.shard._deleted_at, self.n), self.n)
        return (~deleted).nonzero().flatten()

    def _stored_blocks(self, rows: int):
        """The undeleted positions in position (= list) order, in blocks of at most `rows`: slices when nothing is
        deleted, else int64 position tensors."""
        keep = self._undeleted()
        total = self.n if keep is None else keep.numel()
        for a in range(0, total, rows):
            b = min(a + rows, total)
            yield slice(a, b) if keep is None else keep[a:b]

    def _stored_queries(self, pos, nprobe: int):
        """Stored rows at positions `pos` (a slice or an int64 tensor) as queries, with no re-quantization: (rows,
        q_scale, c_scale, probes).  bf16 rows take their inv_norms (cos_sim) or no scale (dot); int8 rows their cos_scales
        (cos_sim) or scales (dot).  The probes are those of the stored row (dequantized for int8).  A slice is a view of
        the shard's rows, passed to the kernels as it is."""
        sh, cos = self.shard, self.score_function == "cos_sim"
        if isinstance(pos, slice):
            take, idx = (lambda t: t[pos]), torch.arange(pos.start, pos.stop, device=self.device)
        else:
            take, idx = (lambda t: t.index_select(0, pos)), pos
        if sh.dtype == "int8":
            scales = sh.cos_scales if cos else sh.scales
            q_scale, c_scale = take(scales), scales.data_ptr()
        else:
            q_scale, c_scale = (take(sh.inv_norms), sh.inv_norms.data_ptr()) if cos else (None, None)
        return take(sh.vectors), q_scale, c_scale, self.probe(_rows_f32(sh, idx), nprobe)

    def add(self, emb: torch.Tensor) -> None:
        """Append fp32/bf16 embeddings [m, D] as documents id_base + n .. id_base + n + m - 1 (as ``CorpusShard.add``).

        The rows are stored as ``CorpusShard.add`` stores them for the index's dtype, and each goes to the list of its
        best centroid — the assignment of ``build``'s final pass, on the stored row.  Every list keeps its rows in their
        order, followed by its new rows in input order; deletions stay with their documents and new rows start
        undeleted.  The centroids are never retrained, so after heavy growth or drift of the data rebuild the index.

        The inner shard is rebuilt out of place: peak device memory is the old index plus the new one plus the m rows
        staged in the index's format (and one assignment batch, as in ``build``)."""
        m = int(emb.shape[0])
        if emb.dim() != 2 or emb.shape[1] != self.dim:
            raise ValueError(f"add: embeddings must be [m, {self.dim}], got {tuple(emb.shape)}")
        if self.id_base + self.n + m >= 2 ** 31:
            raise ValueError(f"add: global ids must fit in int32 (id_base + n + m = {self.id_base + self.n + m} >= 2^31)")
        if m == 0:
            return
        n, dev, old = self.n, self.device, self.shard
        new = CorpusShard.from_embeddings(emb.to(dev), device=dev, dtype=self.dtype)
        lists = _assign_rows(self._cshard, new, self.score_function)
        offsets, old_dest, new_dest = _merge_lists(self.offsets, lists)
        inner = CorpusShard(self.dim, n + m, device=dev, dtype=self.dtype)
        fields = ("vectors", "scales", "cos_scales") if self.dtype == "int8" else ("vectors", "inv_norms")
        for f in fields:
            dst = getattr(inner, f)[:n + m]
            dst.index_copy_(0, old_dest, getattr(old, f)[:n])
            dst.index_copy_(0, new_dest, getattr(new, f)[:m])
        inner.n = n + m
        ids = torch.empty(n + m, dtype=torch.int32, device=dev)
        ids[old_dest] = self.ids
        ids[new_dest] = torch.arange(self.id_base + n, self.id_base + n + m, dtype=torch.int32, device=dev)
        if old._deleted["any"]:
            deleted = unpack_mask(_bit_slice(old._deleted["words"], old._deleted_at, n), n)
            inner.remove(old_dest[deleted])
        del new
        self._set_lists(inner, offsets, ids)

    def remove(self, ids) -> None:
        """Delete documents by global id: no search returns them afterwards."""
        ids = torch.as_tensor(ids, dtype=torch.int64).to(self.device).reshape(-1)
        if ids.numel() == 0:
            return
        local = ids - self.id_base
        if bool(((local < 0) | (local >= self.n)).any()):
            raise ValueError(f"remove: ids must lie in [{self.id_base}, {self.id_base + self.n})")
        self.shard.remove(self._pos[local])

    @property
    def n_deleted(self) -> int:
        return self.shard.n_deleted

    # ---- persistence --------------------------------------------------------------------------------------------
    def save(self, path: str) -> None:
        """One directory: the inner shard (``shard/``, deletions included) plus centroids.npy (fp32 [nlist, D]),
        offsets.npy (int64 [nlist + 1]), ids.npy (int32 [n]) and meta.json."""
        os.makedirs(path, exist_ok=True)
        self.shard.save(os.path.join(path, "shard"))
        np.save(os.path.join(path, "centroids.npy"), self.centroids.cpu().numpy())
        np.save(os.path.join(path, "offsets.npy"), self.offsets.cpu().numpy())
        np.save(os.path.join(path, "ids.npy"), self.ids.cpu().numpy())
        with open(os.path.join(path, "meta.json"), "w") as f:
            json.dump({"format": FORMAT, "dtype": self.dtype, "dim": self.dim, "n": self.n, "nlist": self.nlist,
                       "id_base": self.id_base, "score_function": self.score_function, "shard": "shard"}, f)

    @classmethod
    def load(cls, path: str, device="cuda:0") -> "IVFIndex":
        """Reload an index written by ``save`` (identical search bits).  Shapes, offset monotonicity and the id range
        are checked on the host before anything is allocated on the device."""
        with open(os.path.join(path, "meta.json")) as f:
            meta = json.load(f)
        if meta.get("format") != FORMAT:
            raise ValueError(f"{path}: not an IVFIndex directory ({meta})")
        n, dim, nlist, id_base = int(meta["n"]), int(meta["dim"]), int(meta["nlist"]), int(meta["id_base"])
        _check_score_function(meta["score_function"])
        cent = np.load(os.path.join(path, "centroids.npy"))
        offsets = np.load(os.path.join(path, "offsets.npy"))
        ids = np.load(os.path.join(path, "ids.npy"))
        if nlist < 1 or cent.shape != (nlist, dim) or cent.dtype != np.float32:
            raise ValueError(f"{path}: centroids {cent.shape}/{cent.dtype} do not match meta {meta}")
        if offsets.shape != (nlist + 1,) or offsets.dtype != np.int64:
            raise ValueError(f"{path}: offsets {offsets.shape}/{offsets.dtype} do not match meta {meta}")
        if offsets[0] != 0 or offsets[-1] != n or bool((np.diff(offsets) < 0).any()):
            raise ValueError(f"{path}: offsets must rise monotonically from 0 to n={n}")
        if ids.shape != (n,) or ids.dtype != np.int32:
            raise ValueError(f"{path}: ids {ids.shape}/{ids.dtype} do not match meta {meta}")
        if n and (int(ids.min()) < id_base or int(ids.max()) >= id_base + n or len(np.unique(ids)) != n):
            raise ValueError(f"{path}: ids must be a permutation of [{id_base}, {id_base + n})")
        shard_dir = os.path.join(path, meta.get("shard", "shard"))
        with open(os.path.join(shard_dir, "meta.json")) as f:
            smeta = json.load(f)
        if (int(smeta.get("n", -1)), int(smeta.get("dim", -1)), smeta.get("dtype")) != (n, dim, meta["dtype"]):
            raise ValueError(f"{path}: inner shard {smeta} does not match meta {meta}")
        shard = CorpusShard.load(shard_dir, device=device)
        return cls(shard, torch.from_numpy(cent), torch.from_numpy(offsets), torch.from_numpy(ids), id_base,
                   meta["score_function"])
