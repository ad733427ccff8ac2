"""IVF-PQ index: the IVF lists of ``IVFIndex`` with every document stored as m product-quantization codes of 8 or 4 bits.

A document costs m nbits / 8 bytes of codes plus its int32 id and its int32 position in the id -> position map
(m nbits / 8 + 8 bytes and a deletion bit) instead of its full row: 104 bytes for a 768-dim document at m = 96 with 8-bit
codes (56 with 4-bit codes) against 1536 in bf16.  With 4-bit codes (``nbits=4``, 16 codewords per subspace) a
subspace's lookup table is 16 fp32 words, which a warp reads without bank conflicts, and the same bytes hold twice as
many subspaces.  A query probes
its ``nprobe`` nearest lists (``IVFIndex.probe``'s rule), and the scan scores every document of those lists from the
query's lookup tables (include/sgpt_b200.h, IVF-PQ search): m shared-memory lookups per document instead of a D-long dot
product.  The scores are approximations (asymmetric distance computation, ADC); ``search(..., refine=shard)`` re-ranks
the PQ pass's best ``k_refine`` documents with their exact scores from a ``CorpusShard`` holding the same documents.
``search(..., allow=)`` takes a boolean filter, shared ([n]) or per query ([Q, n]), as every other search does: the scan
skips the positions it does not allow, so the refine pass re-ranks allowed documents only.

Not supported: range search, paraphrase mining / community detection over an IVF-PQ index, code
sizes other than 4 and 8 bits, OPQ rotations, fp16 tables and indexes spread over several GPUs.
"""
from __future__ import annotations

import json
import os
from typing import Optional, Tuple, Union

import numpy as np
import torch

from . import _lib
from .index import CorpusShard, _allow_mask, _bit_slice, _check_allow, _check_score_function, pack_mask, unpack_mask
from .ivf import _assign, _kmeans, _list_order, _merge_lists, _rows_f32

FORMAT = "sgpt_b200.IVFPQIndex/1"
NBITS = 8                 # the default code width
_NBITS = (4, 8)           # the supported code widths
_BATCH_BYTES = 256 << 20  # fp32 rows per encoding batch
_QUERY_BLOCK = 1024       # queries per table / scan call with 8-bit codes (the tables take m KB per query), and with a
                          # per-query filter at either width (packing a block's filter takes 8 bytes per bit on the way)


def _check_pq_shape(D: int, m: int, nbits: int = NBITS) -> None:
    if nbits not in _NBITS:
        raise ValueError(f"nbits={nbits} is not supported (only 4- and 8-bit codes are)")
    if D % 8 != 0:
        raise ValueError(f"embedding dimension {D} must be a multiple of 8")
    if m < 16 or m % 16 != 0 or D % m != 0:
        raise ValueError(f"m={m} must be a positive multiple of 16 that divides D={D}")
    if nbits == 4 and m % 32 != 0:
        raise ValueError(f"m={m} must be a multiple of 32 for nbits=4")


def _pack_codes(codes: torch.Tensor, nbits: int) -> torch.Tensor:
    """Code rows [T, m] (values < 2^nbits) as stored: uint8 [T, m nbits / 8].  4-bit: byte i = code[2i] | code[2i+1]
    << 4 (include/sgpt_b200.h)."""
    if nbits == 8:
        return codes.to(torch.uint8)
    return (codes[:, 0::2] | (codes[:, 1::2] << 4)).to(torch.uint8)


def _nearest_codewords(r: torch.Tensor, codebooks: torch.Tensor) -> torch.Tensor:
    """code[i][j] = argmin_c sum_t (r[i, j dsub + t] - B[j][c][t])^2 over the K codewords of codebooks [m, K, dsub],
    ties to the lowest c: d = 0, then for t ascending e = r - B, d = d + e * e, every operation one fp32 rounding (no
    fused multiply-add, no GEMM), so a row's codes do not depend on the rows encoded with it and numpy restates them
    exactly.  Row blocks of ~64 MB of distances.  int64 [T, m]."""
    m, K, dsub = codebooks.shape
    T = r.shape[0]
    rows = max(1, (64 << 20) // (4 * K * m))
    out = torch.empty((T, m), dtype=torch.int64, device=r.device)
    for i in range(0, T, rows):
        x = r[i:i + rows].view(-1, m, dsub)
        d = torch.zeros((x.shape[0], m, K), dtype=torch.float32, device=r.device)
        for t in range(dsub):
            diff = x[:, :, t, None] - codebooks[None, :, :, t]
            d += diff * diff
        out[i:i + rows] = d.argmin(-1)
    return out


def _train_codebooks(r: torch.Tensor, m: int, n_iter: int, g: torch.Generator, nbits: int = NBITS) -> torch.Tensor:
    """One K-centroid k-means (K = 2^nbits) per subspace over the training residuals r fp32 [T, D] (device): codebooks
    fp32 [m, K, dsub].  Starts from r[:K]; the update is the mean of the assigned sub-vectors summed in fp64 on the host
    in row order, and an empty cell is re-seeded with a sub-vector of a row drawn from `g`."""
    T, D = r.shape
    K = 1 << nbits
    dsub, dev = D // m, r.device
    cb = r[:K].view(K, m, dsub).transpose(0, 1).contiguous()
    step = max(1, (64 << 20) // (8 * D))  # rows per host transfer of the update
    cell = torch.arange(m)[None, :] * K
    for _ in range(int(n_iter)):
        a = _nearest_codewords(r, cb).cpu()
        sums = torch.zeros(m * K, dsub, dtype=torch.float64)
        for i in range(0, T, step):  # index_add_ on the host adds the rows in order: reproducible bits
            sums.index_add_(0, (a[i:i + step] + cell).flatten(), r[i:i + step].cpu().double().view(-1, dsub))
        counts = torch.bincount((a + cell).flatten(), minlength=m * K)
        new = (sums / counts.clamp(min=1)[:, None].double()).view(m, K, dsub)
        empty = (counts == 0).nonzero().flatten()
        if len(empty):
            rows = r[torch.randint(T, (len(empty),), generator=g).to(dev)].cpu().double().view(-1, m, dsub)
            j = empty // K
            new[j, empty % K] = rows[torch.arange(len(empty)), j]
        cb = new.float().to(dev)
    return cb


class IVFPQIndex:
    """IVF-PQ index on one GPU.  Made by ``train`` (empty) + ``add``, ``build`` or ``load``.

    ``centroids`` fp32 [nlist, D] (searched as a bf16 shard to choose the probes), ``codebooks`` fp32 [m, K, D / m]
    with K = 2^nbits codewords per subspace (``nbits`` 8 or 4, read from the codebooks' shape), ``codes`` uint8
    [n, m nbits / 8] in list order (list l is positions ``offsets[l] .. offsets[l+1]``; 4-bit codes two per byte, the
    even subspace in the low nibble), ``ids`` int32 [n] the global id of each position, and the deleted positions as a
    bitmap."""

    def __init__(self, centroids: torch.Tensor, codebooks: torch.Tensor, codes: torch.Tensor, offsets: torch.Tensor,
                 ids: torch.Tensor, deleted: Optional[torch.Tensor], id_base: int, score_function: str, device):
        _check_score_function(score_function)
        self.score_function, self.id_base = score_function, int(id_base)
        self.device = torch.device(device)
        self.centroids = centroids.to(self.device, torch.float32).contiguous()
        self.codebooks = codebooks.to(self.device, torch.float32).contiguous()
        self.nlist, self.dim = self.centroids.shape
        self.m, K = self.codebooks.shape[0], self.codebooks.shape[1]
        if K not in (1 << b for b in _NBITS):
            raise ValueError(f"codebooks hold {K} codewords per subspace (16 or 256 are supported)")
        self.nbits = K.bit_length() - 1
        _check_pq_shape(self.dim, self.m, self.nbits)
        self._cshard = CorpusShard.from_embeddings(self.centroids, device=self.device)
        self._ws: Optional[torch.Tensor] = None
        self._set_lists(codes, offsets, ids, deleted)

    def _set_lists(self, codes: torch.Tensor, offsets: torch.Tensor, ids: torch.Tensor,
                   deleted: Optional[torch.Tensor]) -> None:
        """The list-ordered codes and their layout (``__init__``, ``add``); `deleted`: int32 words of the deleted
        positions or None."""
        self.codes = codes.to(self.device, torch.uint8).contiguous()
        self.n = self.codes.shape[0]
        self.offsets = offsets.to(self.device, torch.int64).contiguous()
        self.ids = ids.to(self.device, torch.int32).contiguous()
        self.list_sizes = (self.offsets[1:] - self.offsets[:-1]).cpu()
        self.max_list_len = int(self.list_sizes.max()) if self.nlist else 0
        # position of every global id (ids are a permutation of id_base .. id_base + n - 1), int32
        self._pos = torch.empty(self.n, dtype=torch.int32, device=self.device)
        self._pos[self.ids.long() - self.id_base] = torch.arange(self.n, dtype=torch.int32, device=self.device)
        self._deleted = deleted.to(self.device, torch.int32).contiguous() if deleted is not None else None

    # ---- construction -------------------------------------------------------------------------------------------
    @classmethod
    def train(cls, sample: torch.Tensor, nlist: int, m: int, score_function: str = "cos_sim", n_iter: int = 10,
              seed: int = 0, device=None, id_base: int = 0, nbits: int = NBITS) -> "IVFPQIndex":
        """An empty index (n = 0, documents will be numbered from ``id_base``) trained on the fp32/bf16 rows ``sample``
        [T, D]: T >= 2^nbits and T >= nlist.

        The rows (normalized for cos_sim) are shuffled with ``seed``; the coarse centroids are ``IVFIndex.build``'s
        k-means over them, and the codebooks one 2^nbits-centroid k-means per subspace over the residuals to each row's
        centroid (``_train_codebooks``), ``n_iter`` iterations each.  ``nbits``: 8 (256 codewords, m bytes of codes per
        document) or 4 (16 codewords, m / 2 bytes; m % 32 == 0).  The same inputs and seed give bit-identical centroids
        and codebooks on the same device."""
        _check_score_function(score_function)
        x = torch.as_tensor(sample)
        dev = torch.device(device) if device is not None else x.device
        if x.dim() != 2:
            raise ValueError(f"sample must be [T, D], got {tuple(x.shape)}")
        T, D = x.shape
        nlist, m, nbits = int(nlist), int(m), int(nbits)
        _check_pq_shape(D, m, nbits)
        K = 1 << nbits
        if nlist < 1 or T < max(K, nlist):
            raise ValueError(f"a sample of {T} rows is too small: it needs at least {K} and nlist={nlist} rows")
        if id_base < 0:
            raise ValueError("id_base must be >= 0")
        g = torch.Generator().manual_seed(int(seed))
        x = x.to(dev).float()[torch.randperm(T, generator=g).to(dev)]  # (a copy: the sample is only read)
        if score_function == "cos_sim":
            x = torch.nn.functional.normalize(x, dim=1)
        cent = _kmeans(x, nlist, n_iter, g, score_function)
        lists = _assign(CorpusShard.from_embeddings(cent, device=dev), x, score_function)
        x -= cent[lists]
        codebooks = _train_codebooks(x, m, n_iter, g, nbits)
        del x
        empty = torch.zeros(nlist + 1, dtype=torch.int64)
        return cls(cent, codebooks, torch.empty((0, m * nbits // 8), dtype=torch.uint8), empty,
                   torch.empty(0, dtype=torch.int32), None, id_base, score_function, dev)

    @classmethod
    def build(cls, source: Union[CorpusShard, torch.Tensor], nlist: int, m: int, score_function: str = "cos_sim",
              n_iter: int = 10, train_size: Optional[int] = None, seed: int = 0, device=None,
              nbits: int = NBITS) -> "IVFPQIndex":
        """``train`` (with ``nbits``) on ``train_size`` rows of ``source`` (default min(n, max(64 nlist, 256))), drawn as
        ``torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:train_size]``, then ``add`` of all its rows in
        batches.  ``source``: a ``CorpusShard`` (its stored rows; an int8 shard's dequantized with their scales, its
        id_base and deletions carry over) or fp32/bf16 embeddings [n, D] (ids from 0)."""
        if isinstance(source, CorpusShard):
            if source.dtype == "binary":
                raise ValueError("IVF-PQ indexes are not built from binary shards (dtype 'binary'): use bf16 or int8")
            src = source
        else:
            src = CorpusShard.from_embeddings(torch.as_tensor(source).float(), device=device)
        n, dev = src.n, src.device
        T = min(n, int(train_size) if train_size is not None else max(64 * int(nlist), 256))
        sample = torch.randperm(n, generator=torch.Generator().manual_seed(int(seed)))[:T].to(dev)
        index = cls.train(_rows_f32(src, sample), nlist, m, score_function, n_iter, seed, dev, src.id_base, nbits)
        bs = max(1, _BATCH_BYTES // (4 * src.dim))
        for i in range(0, n, bs):
            index.add(_rows_f32(src, torch.arange(i, min(i + bs, n), device=dev)))
        if src._deleted["any"]:
            deleted = unpack_mask(_bit_slice(src._deleted["words"], src._deleted_at, n), n)
            index.remove(deleted.nonzero().flatten() + src.id_base)
        return index

    def add(self, emb: torch.Tensor) -> None:
        """Append fp32/bf16 embeddings [b, D] as documents id_base + n .. id_base + n + b - 1.

        In batches of ~256 MB of fp32 rows: each row x goes to the list of its best centroid, the exact search (k = 1)
        against the centroid shard with x itself as the query, i.e. the assignment ``IVFIndex.add`` makes for a bf16
        index, whose stored row is x rounded to bf16 as the search rounds its queries.  The residual of x~ (x normalized
        for cos_sim) to that centroid is encoded with the nearest codeword of every subspace.  The codes, offsets and ids
        are then rebuilt out of place with ``IVFIndex.add``'s list order: every list keeps its rows, followed by its new
        rows in input order; deletions stay with their documents.  The centroids and codebooks are never retrained.
        ``emb`` is only read."""
        b = int(emb.shape[0])
        if emb.dim() != 2 or emb.shape[1] != self.dim:
            raise ValueError(f"add: embeddings must be [b, {self.dim}], got {tuple(emb.shape)}")
        if self.id_base + self.n + b >= 2 ** 31:
            raise ValueError(f"add: global ids must fit in int32 (id_base + n + b = {self.id_base + self.n + b} >= 2^31)")
        if b == 0:
            return
        dev, n = self.device, self.n
        bs = max(1, _BATCH_BYTES // (4 * self.dim))
        lists = torch.empty(b, dtype=torch.int64, device=dev)
        row_bytes = self.m * self.nbits // 8
        codes = torch.empty((b, row_bytes), dtype=torch.uint8, device=dev)
        for i in range(0, b, bs):
            x = emb[i:i + bs].to(dev).float()  # (may be a view of emb: nothing below writes into it)
            lists[i:i + bs] = _assign(self._cshard, x, self.score_function)
            if self.score_function == "cos_sim":
                x = torch.nn.functional.normalize(x, dim=1)
            r = x - self.centroids[lists[i:i + bs]]
            codes[i:i + bs] = _pack_codes(_nearest_codewords(r, self.codebooks), self.nbits)
            del x, r
        offsets, old_dest, new_dest = _merge_lists(self.offsets, lists)
        all_codes = torch.empty((n + b, row_bytes), dtype=torch.uint8, device=dev)
        all_codes.index_copy_(0, old_dest, self.codes)
        all_codes.index_copy_(0, new_dest, codes)
        ids = torch.empty(n + b, dtype=torch.int32, device=dev)
        ids[old_dest] = self.ids
        ids[new_dest] = torch.arange(self.id_base + n, self.id_base + n + b, dtype=torch.int32, device=dev)
        deleted = None
        if self._deleted is not None:
            bits = torch.zeros(n + b, dtype=torch.bool, device=dev)
            bits[old_dest] = unpack_mask(self._deleted, n)
            deleted = pack_mask(bits)
        del codes
        self._set_lists(all_codes, offsets, ids, deleted)

    # ---- search -------------------------------------------------------------------------------------------------
    def probe(self, queries: torch.Tensor, nprobe: int) -> torch.Tensor:
        """The ``nprobe`` lists each query scans: int32 [Q, nprobe], best centroid first (``IVFIndex.probe``'s rule)."""
        if not 1 <= int(nprobe) <= self.nlist:
            raise ValueError(f"nprobe={nprobe} must lie in [1, nlist={self.nlist}]")
        return self._cshard.search(queries.to(self.device), int(nprobe), self.score_function)[1].to(torch.int32)

    def tables(self, queries: torch.Tensor, probes: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """``sgpt_pq_tables_nbits`` of fp32/bf16 queries [Q, D] (normalized here for cos_sim) and their probes: (lut fp32
        [Q, m, 2^nbits], base fp32 [Q, nprobe])."""
        q = queries.to(self.device).float()
        if self.score_function == "cos_sim":
            q = torch.nn.functional.normalize(q, dim=1)
        q = q.contiguous()
        nq, nprobe = q.shape[0], probes.shape[1]
        lut = torch.empty((nq, self.m, 1 << self.nbits), dtype=torch.float32, device=self.device)
        base = torch.empty((nq, nprobe), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            rc = _lib.lib().sgpt_pq_tables_nbits(q.data_ptr(), self.codebooks.data_ptr(), self.centroids.data_ptr(),
                                                 probes.data_ptr(), nq, self.dim, self.m, self.nbits, self.nlist, nprobe,
                                                 lut.data_ptr(), base.data_ptr(), _lib.current_stream())
        _lib.check(rc, "sgpt_pq_tables_nbits")
        return lut, base

    def _list_mask(self, allow: Optional[torch.Tensor], nq: int) -> Tuple[Optional[torch.Tensor], int]:
        """(bitmap, pitch) over list positions of a search of nq queries: `allow` (document order, boolean [n] or
        [nq, n], or None) permuted to list order (``_list_order``) and packed with the deletions ANDed in."""
        return _allow_mask(_list_order(allow, self.ids, self.id_base, nq), self._deleted, self.device, self.n, nq)

    def scan(self, lut: torch.Tensor, base: torch.Tensor, probes: torch.Tensor, k: int,
             mask: Optional[Tuple[Optional[torch.Tensor], int]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """``sgpt_ivfpq_search_masked`` of prepared tables: the top-k by ADC score of the allowed probed documents.
        ``mask``: (bitmap int32, pitch in words) over list positions, as ``_list_mask`` makes it (deletions already
        cleared); None allows every undeleted document."""
        if mask is None:
            mask = self._list_mask(None, probes.shape[0])
        nq, nprobe = probes.shape
        out_s = torch.full((nq, k), -float("inf"), dtype=torch.float32, device=self.device)
        out_i = torch.full((nq, k), -1, dtype=torch.int64, device=self.device)
        if self.n == 0 or nq == 0:
            return out_s, out_i
        lib = _lib.lib()
        need = lib.sgpt_ivfpq_search_workspace_bytes(nq, self.nlist, nprobe, self.max_list_len, self.m)
        if need < 0:
            raise ValueError(f"sgpt_ivfpq_search rejects these arguments: {lib.sgpt_last_error().decode()}")
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            rc = lib.sgpt_ivfpq_search_masked(lut.data_ptr(), base.data_ptr(), self.codes.data_ptr(), nq, self.n,
                                              self.m, self.nbits, self.offsets.data_ptr(), self.nlist, self.max_list_len,
                                              self.ids.data_ptr(), probes.data_ptr(), nprobe, k, _lib.ptr(mask[0]),
                                              mask[1], out_s.data_ptr(), out_i.data_ptr(), self._ws.data_ptr(),
                                              self._ws.numel(), _lib.current_stream())
        _lib.check(rc, "sgpt_ivfpq_search_masked")
        return out_s, out_i

    def search(self, queries: torch.Tensor, k: int, nprobe: int, refine: Optional[CorpusShard] = None,
               k_refine: Optional[int] = None, allow: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Top-k of the undeleted documents in each query's ``nprobe`` probed lists by ADC score, for fp32/bf16 queries
        [Q, D]: (scores fp32 [Q, k] descending, global ids int64 [Q, k]), ties by ascending id, tail (-inf, -1).

        ``allow``: boolean device tensor [n] (all queries) or [Q, n] (one row per query), indexed by global id - id_base
        as in ``CorpusShard.search``: only those documents may be returned.  The result is the top-k by ADC score of the
        allowed, undeleted documents in each query's probed lists.  The probes do not depend on the filter (they are
        still the ``nprobe`` nearest centroids), so a selective filter can return fewer than k documents even where the
        whole index holds more; nothing falls back to an exact search.

        ``refine``: a ``CorpusShard`` holding the same documents (same id_base and n, e.g. the source of ``build``).  The
        PQ pass then selects ``k_refine`` candidates (default min(4096, 10 k)) and the result is the top-k of their exact
        scores in the shard (``sgpt_rerank``: the bits of ``refine.search``).  The shard's own deletions are not
        consulted: delete documents through the index (``remove``), which leaves them out of the candidates.  With
        ``allow`` the candidates are allowed documents only, so a refined filtered search re-ranks only those."""
        k = int(k)
        if not 1 <= k <= 4096:
            raise ValueError(f"k={k} must lie in [1, 4096]")
        kk = k
        if refine is not None:
            kk = min(4096, 10 * k) if k_refine is None else int(k_refine)
            if not k <= kk <= 4096:
                raise ValueError(f"k_refine={kk} must lie in [k={k}, 4096]")
            if refine.dtype == "binary":
                raise ValueError("refine must be a bf16 or int8 shard: a binary shard (dtype 'binary') holds no exact "
                                 "scores")
            if (refine.id_base, refine.n, refine.dim) != (self.id_base, self.n, self.dim):
                raise ValueError(f"refine shard (id_base={refine.id_base}, n={refine.n}, dim={refine.dim}) does not hold "
                                 f"the index's documents (id_base={self.id_base}, n={self.n}, dim={self.dim})")
        nq = queries.shape[0]
        if allow is not None:
            allow = _check_allow(allow, self.device, self.n, nq)
        per_query = allow is not None and allow.dim() == 2
        mask = None if per_query else self._list_mask(allow, nq)
        queries = queries.to(self.device)
        outs = []
        # the same table bytes per call: 16x the queries with 4-bit codes, unless a per-query filter is packed per block
        block = _QUERY_BLOCK if per_query else _QUERY_BLOCK * (256 >> self.nbits)
        for a in range(0, max(nq, 1), block):
            q = queries[a:a + block]
            if per_query:
                mask = self._list_mask(allow[a:a + block], q.shape[0])
            probes = self.probe(q, nprobe)
            s, i = self.scan(*self.tables(q, probes), probes, kk, mask)
            outs.append((s, i) if refine is None else rerank(refine, q, i, k, self.score_function))
        return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])

    # ---- deletions ------------------------------------------------------------------------------------------------
    def remove(self, ids) -> None:
        """Delete documents by global id: no search returns them afterwards."""
        ids = torch.as_tensor(ids, dtype=torch.int64).to(self.device).reshape(-1)
        if ids.numel() == 0:
            return
        local = ids - self.id_base
        if bool(((local < 0) | (local >= self.n)).any()):
            raise ValueError(f"remove: ids must lie in [{self.id_base}, {self.id_base + self.n})")
        bits = torch.zeros(self.n, dtype=torch.bool, device=self.device) if self._deleted is None else unpack_mask(
            self._deleted, self.n)
        bits[self._pos[local].long()] = True
        self._deleted = pack_mask(bits)

    @property
    def n_deleted(self) -> int:
        return 0 if self._deleted is None else int(unpack_mask(self._deleted, self.n).sum())

    @property
    def nbytes(self) -> int:
        """Device bytes of the index: per document m nbits / 8 bytes of codes, an int32 id and an int32 position
        (m nbits / 8 + 8) plus the deletion bitmap, and the centroids (fp32 and their bf16 shard), codebooks and
        offsets."""
        per_doc = self.codes.numel() + 4 * self.ids.numel() + 4 * self._pos.numel()
        deleted = 0 if self._deleted is None else 4 * self._deleted.numel()
        cs = self._cshard
        fixed = (4 * self.centroids.numel() + 4 * self.codebooks.numel() + 8 * self.offsets.numel() +
                 cs.vectors.numel() * 2 + 4 * cs.inv_norms.numel())
        return per_doc + deleted + fixed

    # ---- persistence --------------------------------------------------------------------------------------------
    def save(self, path: str) -> None:
        """One directory: centroids.npy (fp32 [nlist, D]), codebooks.npy (fp32 [m, 2^nbits, D / m]), codes.npy (uint8
        [n, m nbits / 8]), offsets.npy (int64 [nlist + 1]), ids.npy (int32 [n]), deleted.npy (uint32 [ceil(n / 32)], bit j set =
        position j deleted) and meta.json."""
        os.makedirs(path, exist_ok=True)
        np.save(os.path.join(path, "centroids.npy"), self.centroids.cpu().numpy())
        np.save(os.path.join(path, "codebooks.npy"), self.codebooks.cpu().numpy())
        np.save(os.path.join(path, "codes.npy"), self.codes.cpu().numpy())
        np.save(os.path.join(path, "offsets.npy"), self.offsets.cpu().numpy())
        np.save(os.path.join(path, "ids.npy"), self.ids.cpu().numpy())
        words = np.zeros((self.n + 31) // 32, np.uint32)
        if self._deleted is not None:
            words = self._deleted[:len(words)].cpu().numpy().view(np.uint32)
        np.save(os.path.join(path, "deleted.npy"), words)
        with open(os.path.join(path, "meta.json"), "w") as f:
            json.dump({"format": FORMAT, "dim": self.dim, "m": self.m, "nbits": self.nbits, "n": self.n, "nlist": self.nlist,
                       "id_base": self.id_base, "score_function": self.score_function}, f)

    @classmethod
    def load(cls, path: str, device="cuda:0") -> "IVFPQIndex":
        """Reload an index written by ``save`` (identical search bits).  Every shape and dtype, the offset monotonicity
        and the id permutation are checked on the host before anything is allocated on the device."""
        with open(os.path.join(path, "meta.json")) as f:
            meta = json.load(f)
        if meta.get("format") != FORMAT:
            raise ValueError(f"{path}: not an IVFPQIndex directory ({meta})")
        nbits = meta.get("nbits", -1)
        if not isinstance(nbits, int) or nbits not in _NBITS:
            raise ValueError(f"{path}: nbits={nbits} (only 4- and 8-bit codes are supported)")
        n, dim, m = int(meta["n"]), int(meta["dim"]), int(meta["m"])
        nlist, id_base = int(meta["nlist"]), int(meta["id_base"])
        _check_score_function(meta["score_function"])
        _check_pq_shape(dim, m, nbits)
        arrays = {name: np.load(os.path.join(path, name + ".npy"))
                  for name in ("centroids", "codebooks", "codes", "offsets", "ids", "deleted")}
        want = {"centroids": ((nlist, dim), np.float32), "codebooks": ((m, 1 << nbits, dim // m), np.float32),
                "codes": ((n, m * nbits // 8), np.uint8), "offsets": ((nlist + 1,), np.int64), "ids": ((n,), np.int32),
                "deleted": (((n + 31) // 32,), np.uint32)}
        if nlist < 1:
            raise ValueError(f"{path}: nlist={nlist} must be positive")
        for name, (shape, dtype) in want.items():
            a = arrays[name]
            if a.shape != shape or a.dtype != dtype:
                raise ValueError(f"{path}: {name} {a.shape}/{a.dtype} do not match meta {meta} (expected {shape}/"
                                 f"{np.dtype(dtype)})")
        offsets, ids = arrays["offsets"], arrays["ids"]
        if offsets[0] != 0 or offsets[-1] != n or bool((np.diff(offsets) < 0).any()):
            raise ValueError(f"{path}: offsets must rise monotonically from 0 to n={n}")
        if n and (int(ids.min()) < id_base or int(ids.max()) >= id_base + n or len(np.unique(ids)) != n):
            raise ValueError(f"{path}: ids must be a permutation of [{id_base}, {id_base + n})")
        if id_base < 0 or id_base + n >= 2 ** 31:
            raise ValueError(f"{path}: global ids must fit in int32 (id_base={id_base}, n={n})")
        deleted = arrays["deleted"].copy()
        if n % 32:
            deleted[-1] &= np.uint32((1 << (n % 32)) - 1)  # bits past n are not deletions
        words = torch.from_numpy(deleted.view(np.int32).copy()) if deleted.any() else None
        return cls(torch.from_numpy(arrays["centroids"]), torch.from_numpy(arrays["codebooks"]),
                   torch.from_numpy(arrays["codes"]), torch.from_numpy(offsets), torch.from_numpy(ids), words, id_base,
                   meta["score_function"], device)


def rerank(shard: CorpusShard, queries: torch.Tensor, cand_ids: torch.Tensor, k: int, score_function: str = "cos_sim"
           ) -> Tuple[torch.Tensor, torch.Tensor]:
    """``sgpt_rerank``: the top-k of the exact scores of each query's candidates (global ids int64 [Q, kc]; ids < 0 or
    outside the shard are empty slots, a query's ids must be distinct) in ``shard``, with ``shard.search``'s query
    conversion, score bits and tie rule; tail (-inf, -1).  The shard's deletions are not consulted.  bf16 and int8
    shards only: a binary shard's candidates are rescored with the float query by ``CorpusShard.rerank_binary``."""
    if shard.dtype == "binary":
        raise ValueError("rerank takes bf16 or int8 shards; a binary shard (dtype 'binary') is rescored with "
                         "CorpusShard.rerank_binary")
    qb, q_scale, c_scale = shard._queries(queries, score_function)
    cand = cand_ids.to(shard.device, torch.int64).contiguous()
    nq, kc = cand.shape
    lib = _lib.lib()
    need = lib.sgpt_rerank_workspace_bytes(nq, kc)
    if need < 0:
        raise ValueError(f"sgpt_rerank rejects these arguments: {lib.sgpt_last_error().decode()}")
    ws = torch.empty(need, dtype=torch.uint8, device=shard.device)
    out_s = torch.empty((nq, k), dtype=torch.float32, device=shard.device)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=shard.device)
    with torch.cuda.device(shard.device):
        rc = lib.sgpt_rerank(shard._dtype_id(), qb.data_ptr(), shard.vectors.data_ptr(), _lib.ptr(q_scale), c_scale, nq,
                             shard.n, shard.dim, shard.id_base, cand.data_ptr(), kc, int(k), out_s.data_ptr(),
                             out_i.data_ptr(), ws.data_ptr(), ws.numel(), _lib.current_stream())
    _lib.check(rc, "sgpt_rerank")
    return out_s, out_i
