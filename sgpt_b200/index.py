"""Corpus shard in HBM + exact top-k search over it (rows S1–S3 of SURVEY.md §8a).

A shard holds the embeddings of a contiguous range of documents as a bf16 matrix [n, D] (read once per search at
HBM speed) plus fp32 1/||row|| of the STORED rows, so cosine scores are exactly ``cos_sim`` of the stored vectors
(sentence_transformers/util.py:24-43) and dot scores are exactly ``dot_score`` (:46-63).

An int8 shard (``dtype="int8"``) holds int8 rows [n, D] with a per-row scale and cos-scale instead: half the bytes per
document, so twice the documents per GPU and half the HBM traffic per search.  Queries are quantized the same way, and
scores are those of the dequantized vectors (include/sgpt_b200.h, int8 corpus shards).

Every search takes an optional document filter ``allow=`` (a boolean device tensor [n] shared by all queries, or [Q, n]
with one row per query), and ``CorpusShard.remove`` deletes documents from a built shard.  Both become one document
bitmap per search (``pack_mask``; include/sgpt_b200.h, masked searches): the result is exactly the search over the
allowed, undeleted documents.

A binary shard (``dtype="binary"``) holds the sign bits of every document, D / 8 bytes (sentence-transformers'
``quantize_embeddings(..., precision="ubinary")``), searched exactly by their integer scores: s = D - 2 hamming for
"dot", s / D for "cos_sim" (include/sgpt_b200.h, binary corpus shards).  ``search(..., rescore=kc)`` rescores the best kc
by the float query, ``refine=shard`` with the exact scores of a bf16 / int8 shard of the same documents.
"""
from __future__ import annotations

import json
import math
import os
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib

SCORE_FUNCTIONS = ("cos_sim", "dot")
SHARD_DTYPES = ("bf16", "int8", "binary")


def _check_score_function(score_function: str) -> None:
    if score_function not in SCORE_FUNCTIONS:
        # same message as biencoder/beir/custommodels/exact_search.py:46-51
        raise ValueError(
            "score function: {} must be either (cos_sim) for cosine similarity or (dot) for dot product".format(
                score_function))


def resolve_score_function(score_function) -> str:
    """"cos_sim" / "dot", or the reference's ``cos_sim`` / ``dot_score`` callables recognised by name."""
    if callable(score_function):
        score_function = {"cos_sim": "cos_sim", "pytorch_cos_sim": "cos_sim", "dot_score": "dot"}.get(
            getattr(score_function, "__name__", ""), None)
    _check_score_function(score_function)
    return score_function


def to_bf16_rows(x: torch.Tensor) -> torch.Tensor:
    """fp32 [n, D] (device) -> bf16 [n, D] (round-to-nearest-even) with the library's conversion kernel."""
    x = x.contiguous()
    assert x.dtype == torch.float32 and x.is_cuda and x.numel() % 4 == 0
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().sgpt_f32_to_bf16(x.data_ptr(), out.data_ptr(), x.numel(), _lib.current_stream()))
    return out


def quantize_rows_i8(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """fp32 or bf16 [n, D] (device) -> (int8 [n, D], scale fp32 [n], cos_scale fp32 [n]) with the library's quantizer."""
    if x.dtype != torch.bfloat16:
        x = x.float()
    x = x.contiguous()
    n, D = x.shape
    q = torch.empty((n, D), dtype=torch.int8, device=x.device)
    scale = torch.empty(n, dtype=torch.float32, device=x.device)
    cos_scale = torch.empty(n, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().sgpt_quantize_rows_i8(x.data_ptr(), int(x.dtype == torch.bfloat16), q.data_ptr(),
                                                    scale.data_ptr(), cos_scale.data_ptr(), n, D, _lib.current_stream()),
                   "sgpt_quantize_rows_i8")
    return q, scale, cos_scale


def quantize_rows_b1(x: torch.Tensor, thresholds: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 or bf16 [n, D] (device) -> (sign bits uint8 [n, D / 8] in np.packbits order, popcounts int32 [n]) with the
    library's quantizer: bit j is x_j > thresholds[j] (None: 0), strict, NaN -> 0."""
    if x.dtype != torch.bfloat16:
        x = x.float()
    x = x.contiguous()
    n, D = x.shape
    bits = torch.empty((n, D // 8), dtype=torch.uint8, device=x.device)
    popc = torch.empty(n, dtype=torch.int32, device=x.device)
    t = None if thresholds is None else thresholds.to(x.device, torch.float32).contiguous()
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().sgpt_quantize_rows_b1(x.data_ptr(), int(x.dtype == torch.bfloat16), _lib.ptr(t),
                                                    bits.data_ptr(), popc.data_ptr(), n, D, _lib.current_stream()),
                   "sgpt_quantize_rows_b1")
    return bits, popc


def binary_thresholds(sample: torch.Tensor) -> torch.Tensor:
    """Per-dimension thresholds of a binary shard from a sample of embeddings [m, D]: the lower median of every
    dimension, fp32 [D].  Mean-pooled GPT embeddings are anisotropic (a large common offset), so with zero thresholds
    some bits may hardly vary; median thresholds split every dimension of the sample in half."""
    sample = torch.as_tensor(sample)
    if sample.dim() != 2 or sample.shape[0] == 0:
        raise ValueError(f"binary_thresholds needs a sample [m, D] with m >= 1, got {tuple(sample.shape)}")
    return sample.float().median(dim=0).values.contiguous()  # torch.median: the lower of the two middle values


_POPC8 = [bin(i).count("1") for i in range(256)]


def _popcounts(bits: torch.Tensor) -> torch.Tensor:
    """Number of set bits of every packed row, uint8 [n, B] -> int32 [n] (loading stored bits)."""
    lut = torch.tensor(_POPC8, dtype=torch.int32, device=bits.device)
    out = torch.empty(bits.shape[0], dtype=torch.int32, device=bits.device)
    step = max(1, (16 << 20) // max(1, bits.shape[1]))
    for i in range(0, bits.shape[0], step):
        out[i:i + step] = lut[bits[i:i + step].long()].sum(1, dtype=torch.int32)
    return out


def _b1_cos(scores: torch.Tensor, dim: int) -> torch.Tensor:
    """cos_sim of the +-1 vectors from the sign dot products s: s / D, one correctly rounded fp32 division per score
    (a tensor divisor: torch turns division by a Python scalar into a multiplication by its reciprocal)."""
    return scores / torch.full((), float(dim), dtype=torch.float32, device=scores.device)


def _b1_threshold(threshold: float, score_function: str, dim: int) -> float:
    """A range-search threshold on the shard's scores -> the threshold on s: for cos_sim the smallest integer s0 with
    fl(s0 / D) >= threshold (fl(s / D) is monotone in s), D + 1 when no s qualifies.  -inf admits every document
    (-D), +inf none (D + 1); NaN is passed on for the library to reject."""
    if score_function != "cos_sim" or math.isnan(threshold):
        return float(threshold)
    if math.isinf(threshold):
        return float(-dim if threshold < 0 else dim + 1)
    t, d = np.float32(threshold), np.float32(dim)
    s0 = min(max(math.ceil(float(threshold) * dim), -dim), dim + 1)
    while s0 > -dim and np.float32(s0 - 1) / d >= t:
        s0 -= 1
    while s0 <= dim and np.float32(s0) / d < t:
        s0 += 1
    return float(s0)


def row_inv_norms(x_bf16: torch.Tensor) -> torch.Tensor:
    n, D = x_bf16.shape
    out = torch.empty(n, dtype=torch.float32, device=x_bf16.device)
    with torch.cuda.device(x_bf16.device):
        _lib.check(_lib.lib().sgpt_row_inv_norms(x_bf16.data_ptr(), out.data_ptr(), n, D, _lib.current_stream()))
    return out


def pack_mask(allow: torch.Tensor) -> torch.Tensor:
    """Boolean [..., n] -> the library's document bitmap, int32 [..., ceil(n / 32)] (the bits of uint32 words): bit
    j % 32 of word j // 32 is allow[..., j]; the bits past n are 0."""
    n = allow.shape[-1]
    words = (n + 31) // 32
    bits = torch.zeros((*allow.shape[:-1], words * 32), dtype=torch.int64, device=allow.device)
    bits[..., :n] = allow.to(torch.bool)
    w = (bits.view(*allow.shape[:-1], words, 32) << torch.arange(32, device=allow.device)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def unpack_mask(words: torch.Tensor, n: int) -> torch.Tensor:
    """Inverse of ``pack_mask``: int32 [..., W] -> boolean [..., n] (n <= 32 W)."""
    w = words.to(torch.int64) & 0xFFFFFFFF
    bits = (w.unsqueeze(-1) >> torch.arange(32, device=words.device)) & 1
    return bits.reshape(*words.shape[:-1], -1)[..., :n].to(torch.bool)


def _bit_slice(words: torch.Tensor, start: int, n: int) -> torch.Tensor:
    """Bits [start, start + n) of a bitmap (int32 words, at least one word beyond the last one read) as a bitmap of
    their own (bit 0 = bit `start`); the bits past n are whatever follows in `words`."""
    w0, r, nw = start // 32, start % 32, (n + 31) // 32
    if r == 0:
        return words[w0:w0 + nw]
    w = words[w0:w0 + nw + 1].to(torch.int64) & 0xFFFFFFFF
    s = ((w[:-1] >> r) | (w[1:] << (32 - r))) & 0xFFFFFFFF
    return torch.where(s >= 2 ** 31, s - 2 ** 32, s).to(torch.int32)


def _check_allow(allow, device, n: int, nq: int) -> torch.Tensor:
    """`allow` of a search of nq queries over n documents as a device tensor: boolean [n] or [nq, n], else ValueError."""
    allow = torch.as_tensor(allow, device=device)
    if allow.dtype != torch.bool or allow.shape not in ((n,), (nq, n)):
        raise ValueError(f"allow must be a boolean tensor [{n}] or [{nq}, {n}], got {allow.dtype} {tuple(allow.shape)}")
    return allow


def _allow_mask(allow: Optional[torch.Tensor], deleted: Optional[torch.Tensor], device, n: int, nq: int
                ) -> Tuple[Optional[torch.Tensor], int]:
    """(bitmap, pitch in words) of a search of nq queries over n documents: `allow` (bool [n] or [nq, n], or None)
    packed with the `deleted` bits (int32 words, or None) cleared; (None, 0) when every document is allowed."""
    if allow is None:
        return (None, 0) if deleted is None else (torch.bitwise_not(deleted).contiguous(), 0)
    m = pack_mask(_check_allow(allow, device, n, nq))
    if deleted is not None:
        m = m & torch.bitwise_not(deleted)
    return m.contiguous(), (m.shape[1] if m.dim() == 2 and n > 0 else 0)


def _mask_rows(mask: Tuple[Optional[torch.Tensor], int], first: int) -> Tuple[Optional[torch.Tensor], int]:
    """The (bitmap, pitch) of a search's queries first .. : per-query bitmaps lose their first rows, a shared one stays."""
    return (mask[0][first:], mask[1]) if mask[1] > 0 else mask


def _grown_range(nq: int, device, run, capacity: Optional[int] = None
                 ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """A range search in CSR form whose output buffer starts at `capacity` entries (default max(4096, 64 nq)) and grows
    once.  ``run(first, counts, cap, out_s, out_i)`` runs the queries first .. nq - 1 into buffers of cap entries, writing
    counts int64 [nq - first] always and the entries of the queries that fit (a prefix).  Returns (offsets int64 [nq+1],
    scores, ids) in the order `run` writes them."""
    cap = max(4096, 64 * nq) if capacity is None else max(1, int(capacity))
    counts = torch.empty(nq, dtype=torch.int64, device=device)
    out_s = torch.empty(cap, dtype=torch.float32, device=device)
    out_i = torch.empty(cap, dtype=torch.int64, device=device)
    run(0, counts, cap, out_s, out_i)
    offsets = torch.zeros(nq + 1, dtype=torch.int64, device=device)
    torch.cumsum(counts, 0, out=offsets[1:])
    total = int(offsets[-1])
    if total > cap:
        # the queries that fitted are a prefix: grow the buffer and run the others once more into its tail
        first = int(torch.searchsorted(offsets[1:], cap, right=True))
        done = int(offsets[first])
        grown_s = torch.empty(total, dtype=torch.float32, device=device)
        grown_i = torch.empty(total, dtype=torch.int64, device=device)
        grown_s[:done].copy_(out_s[:done])
        grown_i[:done].copy_(out_i[:done])
        rest = torch.empty(nq - first, dtype=torch.int64, device=device)
        run(first, rest, total - done, grown_s[done:], grown_i[done:])
        out_s, out_i = grown_s, grown_i
    return offsets, out_s[:total], out_i[:total]


def _check_dtype(dtype: str, dim: int) -> None:
    if dtype not in SHARD_DTYPES:
        raise ValueError(f"shard dtype {dtype!r} must be one of {SHARD_DTYPES}")
    if dtype == "binary":
        if dim % 128 != 0 or not 0 < dim <= 65536:
            raise ValueError(f"binary shards need a positive embedding dimension that is a multiple of 128, at most "
                             f"65536 (got {dim})")
        return
    if dim % (16 if dtype == "int8" else 8) != 0:
        raise ValueError(f"embedding dimension must be a multiple of {16 if dtype == 'int8' else 8} for {dtype} shards")
    if dtype == "int8" and dim > 65536:
        raise ValueError("int8 shards hold at most 65536 dimensions")


class CorpusShard:
    """Documents [id_base, id_base + n) of a corpus, resident in the HBM of one GPU.

    ``dtype="bf16"``: ``vectors`` bf16 [capacity, D] and ``inv_norms`` fp32.  ``dtype="int8"``: ``vectors`` int8
    [capacity, D], ``scales`` and ``cos_scales`` fp32 (include/sgpt_b200.h, int8 corpus shards).  ``dtype="binary"``:
    ``vectors`` uint8 [capacity, D / 8] (sign bits in np.packbits order), ``popcounts`` int32 and the ``thresholds``
    fp32 [D] that documents and queries are quantized with (``thresholds=None``: zeros, ST's "ubinary"; see
    ``binary_thresholds``).

    Deleted documents (``remove``) are bits of a device bitmap int32 [capacity / 32 + 1] that the shard and its views
    share (``_deleted``: the words and whether any bit was ever set; ``_deleted_at``: the bit of this shard's row 0).
    Every search leaves them out; ids never change."""

    def __init__(self, dim: int, capacity: int, device="cuda:0", id_base: int = 0, dtype: str = "bf16",
                 thresholds: Optional[torch.Tensor] = None):
        _check_dtype(dtype, dim)
        if thresholds is not None and dtype != "binary":
            raise ValueError(f"thresholds apply to binary shards only (dtype {dtype!r})")
        self.dim, self.capacity, self.id_base, self.dtype = int(dim), int(capacity), int(id_base), dtype
        self.device = torch.device(device)
        if dtype == "binary":
            t = torch.zeros(self.dim) if thresholds is None else torch.as_tensor(thresholds)
            if t.shape != (self.dim,):
                raise ValueError(f"thresholds must be [{self.dim}], got {tuple(t.shape)}")
            self.thresholds = t.to(self.device, torch.float32).contiguous()
            self.vectors = torch.empty((self.capacity, self.dim // 8), dtype=torch.uint8, device=self.device)
            self.popcounts = torch.empty(self.capacity, dtype=torch.int32, device=self.device)
        elif dtype == "int8":
            self.vectors = torch.empty((self.capacity, self.dim), dtype=torch.int8, device=self.device)
            self.scales = torch.empty(self.capacity, dtype=torch.float32, device=self.device)
            self.cos_scales = torch.empty(self.capacity, dtype=torch.float32, device=self.device)
        else:
            self.vectors = torch.empty((self.capacity, self.dim), dtype=torch.bfloat16, device=self.device)
            self.inv_norms = torch.empty(self.capacity, dtype=torch.float32, device=self.device)
        self.n = 0
        self._ws: Optional[torch.Tensor] = None
        self._deleted = {"words": torch.zeros(self.capacity // 32 + 2, dtype=torch.int32, device=self.device),
                         "any": False}
        self._deleted_at = 0

    @classmethod
    def from_embeddings(cls, emb: torch.Tensor, device=None, id_base: int = 0, dtype: str = "bf16",
                        thresholds: Optional[torch.Tensor] = None) -> "CorpusShard":
        device = device or emb.device
        shard = cls(emb.shape[1], emb.shape[0], device=device, id_base=id_base, dtype=dtype, thresholds=thresholds)
        shard.add(emb)
        return shard

    @classmethod
    def from_packed_bits(cls, bits, device="cuda:0", id_base: int = 0, thresholds: Optional[torch.Tensor] = None,
                         capacity: Optional[int] = None) -> "CorpusShard":
        """A binary shard of sign bits as stored by sentence-transformers' ``quantize_embeddings(...,
        precision="ubinary")`` (``np.packbits(x > 0, axis=-1)``): uint8 [n, D / 8], numpy or torch, taken as they are.
        ``thresholds`` [D] are those the queries are quantized with (None: zeros, what "ubinary" used)."""
        b = torch.as_tensor(np.ascontiguousarray(bits) if isinstance(bits, np.ndarray) else bits)
        if b.dim() != 2 or b.dtype != torch.uint8:
            raise ValueError(f"packed bits must be uint8 [n, D / 8], got {b.dtype} {tuple(b.shape)}")
        n = b.shape[0]
        shard = cls(8 * b.shape[1], max(n, capacity or n), device=device, id_base=id_base, dtype="binary",
                    thresholds=thresholds)
        shard.vectors[:n].copy_(b)
        shard.popcounts[:n].copy_(_popcounts(shard.vectors[:n]))
        shard.n = n
        return shard

    def add(self, emb: torch.Tensor) -> None:
        """Append fp32 (or bf16) embeddings [m, D]; a bf16 shard stores them bf16-rounded, an int8 shard quantized."""
        m = emb.shape[0]
        if self.n + m > self.capacity:
            raise ValueError(f"shard capacity {self.capacity} exceeded ({self.n} + {m})")
        emb = emb.to(self.device)
        if self.dtype == "binary":
            bits, popc = quantize_rows_b1(emb, self.thresholds)
            self.vectors[self.n:self.n + m].copy_(bits)
            self.popcounts[self.n:self.n + m].copy_(popc)
            self.n += m
            return
        if self.dtype == "int8":
            q, scale, cos_scale = quantize_rows_i8(emb)
            self.vectors[self.n:self.n + m].copy_(q)
            self.scales[self.n:self.n + m].copy_(scale)
            self.cos_scales[self.n:self.n + m].copy_(cos_scale)
            self.n += m
            return
        rows = emb if emb.dtype == torch.bfloat16 else to_bf16_rows(emb.float())
        self.vectors[self.n:self.n + m].copy_(rows)
        self.inv_norms[self.n:self.n + m].copy_(row_inv_norms(self.vectors[self.n:self.n + m]))
        self.n += m

    def stored(self) -> torch.Tensor:
        return self.vectors[:self.n]

    # ---- persistence (replaces the pickle-per-chunk embedding cache of BDR:311-323, 336-342) ----------------------
    def save(self, path: str) -> None:
        """Write the shard as ``path/{vectors.npy, <scales>, meta.json}``; one directory per rank for a sharded corpus.
        bf16: vectors.npy holds the bf16 bit patterns as uint16, inv_norms.npy the fp32 1/||row||.  int8: vectors.npy
        holds the int8 rows, scales.npy fp32 [n, 2] the (scale, cos_scale) of every row.  binary: vectors.npy holds the
        bits uint8 [n, D / 8], thresholds.npy fp32 [D]; the popcounts are recomputed at load."""
        os.makedirs(path, exist_ok=True)
        if self.dtype == "binary":
            np.save(os.path.join(path, "vectors.npy"), self.stored().cpu().numpy())
            np.save(os.path.join(path, "thresholds.npy"), self.thresholds.cpu().numpy())
        elif self.dtype == "int8":
            np.save(os.path.join(path, "vectors.npy"), self.stored().cpu().numpy())
            np.save(os.path.join(path, "scales.npy"),
                    torch.stack([self.scales[:self.n], self.cos_scales[:self.n]], 1).cpu().numpy())
        else:
            np.save(os.path.join(path, "vectors.npy"), self.stored().view(torch.int16).cpu().numpy().view(np.uint16))
            np.save(os.path.join(path, "inv_norms.npy"), self.inv_norms[:self.n].cpu().numpy())
        # deleted.npy: uint32 [ceil(n / 32)], bit j % 32 of word j // 32 set = document j deleted
        deleted = _bit_slice(self._deleted["words"], self._deleted_at, self.n) & pack_mask(
            torch.ones(self.n, dtype=torch.bool, device=self.device))
        np.save(os.path.join(path, "deleted.npy"), deleted.cpu().numpy().view(np.uint32))
        with open(os.path.join(path, "meta.json"), "w") as f:
            json.dump({"format": "sgpt_b200.CorpusShard/1", "dtype": self.dtype, "dim": self.dim, "n": self.n,
                       "id_base": self.id_base, "deleted": "deleted.npy"}, f)

    @classmethod
    def load(cls, path: str, device="cuda:0", capacity: Optional[int] = None) -> "CorpusShard":
        """Reload a shard written by ``save`` (bit-identical vectors and scales, so identical search results).  The
        files are checked against meta.json before anything is allocated on the device."""
        with open(os.path.join(path, "meta.json")) as f:
            meta = json.load(f)
        if meta.get("format") != "sgpt_b200.CorpusShard/1":
            raise ValueError(f"{path}: not a CorpusShard directory ({meta})")
        dtype = meta.get("dtype")
        if dtype not in SHARD_DTYPES:
            raise ValueError(f"{path}: unknown shard dtype {dtype!r} (expected one of {SHARD_DTYPES})")
        n, dim = int(meta["n"]), int(meta["dim"])
        vec = np.load(os.path.join(path, "vectors.npy"), mmap_mode="r")
        if dtype == "binary":
            thr = np.load(os.path.join(path, "thresholds.npy"))
            if (dim % 128 != 0 or vec.shape != (n, dim // 8) or vec.dtype != np.uint8 or thr.shape != (dim,)
                    or thr.dtype != np.float32):
                raise ValueError(f"{path}: array shapes {vec.shape}/{thr.shape} do not match meta {meta}")
        elif dtype == "int8":
            sc = np.load(os.path.join(path, "scales.npy"))
            if vec.shape != (n, dim) or vec.dtype != np.int8 or sc.shape != (n, 2) or sc.dtype != np.float32:
                raise ValueError(f"{path}: array shapes {vec.shape}/{sc.shape} do not match meta {meta}")
        else:
            inv = np.load(os.path.join(path, "inv_norms.npy"))
            if vec.shape != (n, dim) or vec.dtype != np.uint16 or inv.shape != (n,):
                raise ValueError(f"{path}: array shapes {vec.shape}/{inv.shape} do not match meta {meta}")
        deleted = None
        if meta.get("deleted") is not None:  # directories written before deletions existed have none
            deleted = np.load(os.path.join(path, meta["deleted"]))
            if deleted.shape != ((n + 31) // 32,) or deleted.dtype != np.uint32:
                raise ValueError(f"{path}: deletion bitmap {deleted.shape}/{deleted.dtype} does not match meta {meta} "
                                 f"(expected uint32 [{(n + 31) // 32}])")
        shard = cls(dim, max(n, capacity or n), device=device, id_base=int(meta["id_base"]), dtype=dtype,
                    thresholds=torch.from_numpy(thr) if dtype == "binary" else None)
        if dtype == "binary":
            shard.vectors[:n].copy_(torch.from_numpy(np.array(vec)))
            shard.popcounts[:n].copy_(_popcounts(shard.vectors[:n]))
        elif dtype == "int8":
            shard.vectors[:n].copy_(torch.from_numpy(np.array(vec)))
            shard.scales[:n].copy_(torch.from_numpy(np.ascontiguousarray(sc[:, 0])))
            shard.cos_scales[:n].copy_(torch.from_numpy(np.ascontiguousarray(sc[:, 1])))
        else:
            shard.vectors[:n].copy_(torch.from_numpy(np.array(vec).view(np.int16)).view(torch.bfloat16))
            shard.inv_norms[:n].copy_(torch.from_numpy(inv))
        shard.n = n
        if deleted is not None and deleted.any():
            # (bits past n are dropped: rows added later start undeleted)
            words = torch.from_numpy(deleted.view(np.int32).copy()).to(shard.device)
            shard._deleted["words"][:len(deleted)].copy_(words & pack_mask(torch.ones(n, dtype=torch.bool,
                                                                                      device=shard.device)))
            shard._deleted["any"] = True
        return shard

    # ---- deletions -------------------------------------------------------------------------------------------------
    def remove(self, ids) -> None:
        """Delete documents by global id (id_base .. id_base + n - 1): no search, range search or gather returns them
        afterwards.  Ids never change (there is no compaction); deleting a document twice is allowed.  A view shares
        the deletions of the shard it was taken from."""
        ids = torch.as_tensor(ids, dtype=torch.int64).to(self.device).reshape(-1)
        if ids.numel() == 0:
            return
        local = ids - self.id_base
        if bool(((local < 0) | (local >= self.n)).any()):
            raise ValueError(f"remove: ids must lie in [{self.id_base}, {self.id_base + self.n})")
        words = self._deleted["words"]
        bits = unpack_mask(words, words.numel() * 32)
        bits[local + self._deleted_at] = True
        words.copy_(pack_mask(bits))
        self._deleted["any"] = True

    @property
    def n_deleted(self) -> int:
        """Number of deleted documents among this shard's n."""
        if not self._deleted["any"] or self.n == 0:
            return 0
        return int(unpack_mask(_bit_slice(self._deleted["words"], self._deleted_at, self.n), self.n).sum())

    def _mask(self, allow: Optional[torch.Tensor], nq: int) -> Tuple[Optional[torch.Tensor], int]:
        """(bitmap, pitch in words) of a search of nq queries: `allow` (bool [n] or [nq, n], or None) without the deleted
        documents; (None, 0) when every document is allowed."""
        deleted = _bit_slice(self._deleted["words"], self._deleted_at, self.n) if self._deleted["any"] else None
        return _allow_mask(allow, deleted, self.device, self.n, nq)

    def _dtype_id(self) -> int:
        """The `dtype` argument of the masked entry points for this shard's format."""
        return {"int8": _lib.DTYPE_I8, "binary": _lib.DTYPE_B1}.get(self.dtype, _lib.DTYPE_BF16)

    def _queries(self, queries: torch.Tensor, score_function: str):
        """Queries -> rows in the shard's format + their scales + the shard's scale pointer.  bf16: bf16 rows, 1/||q||
        of the rounded rows for cos_sim and no scales (None) for dot.  int8: quantized rows, cos_scale (cos_sim) or scale
        (dot) of queries and documents.  binary: the query bits (the shard's thresholds) and the popcounts of queries and
        documents, for either score function (cos_sim divides the scores afterwards, ``_b1_cos``)."""
        _check_score_function(score_function)
        q = queries.to(self.device)
        cos = score_function == "cos_sim"
        if self.dtype == "binary":
            bits, popc = quantize_rows_b1(q, self.thresholds)
            return bits, popc, self.popcounts.data_ptr()
        if self.dtype == "int8":
            q8, scale, cos_scale = quantize_rows_i8(q)
            return q8, (cos_scale if cos else scale), (self.cos_scales if cos else self.scales).data_ptr()
        qb = q.contiguous() if q.dtype == torch.bfloat16 else to_bf16_rows(q.float())
        q_scale = row_inv_norms(qb) if cos else None
        return qb, q_scale, (self.inv_norms.data_ptr() if cos else None)

    def _workspace(self, need: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def _prepare(self, queries: torch.Tensor, k: int, score_function: str):
        """Queries -> rows and scales (``_queries``) + a workspace large enough for this search."""
        qb, q_scale, c_scale = self._queries(queries, score_function)
        self._workspace(_lib.lib().sgpt_search_workspace_bytes(qb.shape[0], self.n, k))
        return qb, q_scale, c_scale

    def search(self, queries: torch.Tensor, k: int, score_function: str = "cos_sim",
               allow: Optional[torch.Tensor] = None, rescore: Optional[int] = None,
               refine: Optional["CorpusShard"] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Exact top-k of this shard for fp32/bf16 queries [Q, D] (device).

        Returns (scores fp32 [Q,k] descending, global ids int64 [Q,k]); when the shard has fewer than k documents the
        tail is (-inf, -1).  Queries are rounded to bf16 (the tensor-core input type); their 1/||q|| is taken from the
        rounded rows so the result equals cos_sim of the stored/rounded vectors evaluated in fp32.  On an int8 shard the
        queries are quantized like the documents, and the scores are those of the dequantized vectors.

        ``allow``: boolean device tensor [n] (all queries) or [Q, n] (one row per query) of the documents that may be
        returned; deleted documents (``remove``) never are.  The result is exactly the search over those documents, with
        the tail (-inf, -1) when fewer than k are allowed.

        Binary shards: the queries are quantized with the shard's thresholds and the scores are the sign dot products s
        (dot) or s / D (cos_sim), exact integers / quotients with many ties (broken by ascending id).  ``rescore=kc``
        (k <= kc <= 4096) takes the best kc documents by s and returns their top-k by the asymmetric score of the float
        query against the +-1 documents (``rerank_binary``; cos_sim: F.normalize(q - t) . s / sqrt(D), t the shard's
        thresholds).  ``refine=shard``: a
        bf16 or int8 shard holding the same documents (same id_base, n and dim) whose exact scores rank the kc candidates
        instead, kc = ``rescore`` or min(4096, 10 k).  Both are ValueErrors on bf16 and int8 shards.
        """
        if rescore is not None or refine is not None:
            return self._rescored(queries, k, score_function, allow, rescore, refine)
        qb, q_scale, c_scale = self._prepare(queries, k, score_function)
        nq = qb.shape[0]
        mask, pitch = self._mask(allow, nq)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            rc = _lib.lib().sgpt_search_masked(self._dtype_id(), qb.data_ptr(), self.vectors.data_ptr(),
                                               _lib.ptr(q_scale), c_scale, nq, self.n, self.dim, k, self.id_base,
                                               _lib.ptr(mask), pitch, out_s.data_ptr(), out_i.data_ptr(),
                                               self._ws.data_ptr(), self._ws.numel(), _lib.current_stream())
        _lib.check(rc, "sgpt_search")
        if self.dtype == "binary" and score_function == "cos_sim":
            out_s = _b1_cos(out_s, self.dim)
        return out_s, out_i

    def _rescored(self, queries: torch.Tensor, k: int, score_function: str, allow, rescore: Optional[int],
                  refine: Optional["CorpusShard"]) -> Tuple[torch.Tensor, torch.Tensor]:
        """``search(..., rescore=, refine=)`` of a binary shard: kc candidates by s, then their top-k rescored."""
        if self.dtype != "binary":
            raise ValueError(f"rescore= and refine= apply to binary shards only (this shard is {self.dtype!r})")
        _check_score_function(score_function)
        kc = int(rescore) if rescore is not None else min(4096, 10 * int(k))
        if not int(k) <= kc <= 4096:
            raise ValueError(f"rescore={kc} must lie in [k={k}, 4096]")
        if refine is not None:
            if not isinstance(refine, CorpusShard) or refine.dtype not in ("bf16", "int8"):
                raise ValueError("refine must be a bf16 or int8 CorpusShard")
            if (refine.id_base, refine.n, refine.dim) != (self.id_base, self.n, self.dim):
                raise ValueError(f"refine shard (id_base={refine.id_base}, n={refine.n}, dim={refine.dim}) does not hold "
                                 f"this shard's documents (id_base={self.id_base}, n={self.n}, dim={self.dim})")
        _, cand = self.search(queries, kc, "dot", allow=allow)
        if refine is not None:
            from .ivfpq import rerank
            return rerank(refine, queries, cand, k, score_function)
        return self.rerank_binary(queries, cand, k, score_function)

    def rerank_binary(self, queries: torch.Tensor, cand_ids: torch.Tensor, k: int, score_function: str = "cos_sim"
                      ) -> Tuple[torch.Tensor, torch.Tensor]:
        """Top-k of the candidates (global ids int64 [Q, kc], < 0 = empty, distinct per query) of a binary shard by the
        asymmetric score of the float queries against the +-1 documents: ``sgpt_rerank`` with SGPT_DTYPE_B1 of the
        query q - t centered on the shard's thresholds t (zero thresholds: q itself, sentence-transformers' rescoring),
        in fp32, F.normalize'd and scaled by fp32(1 / sqrt(D)) for cos_sim.  The centering keeps the query's component
        along a common offset (what median thresholds remove from the bits) out of the score.  Deletions are not
        consulted."""
        if self.dtype != "binary":
            raise ValueError(f"rerank_binary needs a binary shard (this shard is {self.dtype!r})")
        _check_score_function(score_function)
        q = queries.to(self.device).float() - self.thresholds
        q_scale = None
        if score_function == "cos_sim":
            q = torch.nn.functional.normalize(q, dim=1)
            q_scale = torch.full((q.shape[0],), float(np.float32(1.0 / math.sqrt(self.dim))), dtype=torch.float32,
                                 device=self.device)
        q = q.contiguous()
        cand = cand_ids.to(self.device, torch.int64).contiguous()
        nq, kc = cand.shape
        lib = _lib.lib()
        need = lib.sgpt_rerank_workspace_bytes(nq, kc)
        if need < 0:
            raise ValueError(f"sgpt_rerank rejects these arguments: {lib.sgpt_last_error().decode()}")
        ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            rc = lib.sgpt_rerank(_lib.DTYPE_B1, q.data_ptr(), self.vectors.data_ptr(), _lib.ptr(q_scale), None, nq,
                                 self.n, self.dim, self.id_base, cand.data_ptr(), kc, int(k), out_s.data_ptr(),
                                 out_i.data_ptr(), ws.data_ptr(), ws.numel(), _lib.current_stream())
        _lib.check(rc, "sgpt_rerank")
        return out_s, out_i

    def search_packed(self, queries: torch.Tensor, k: int, score_function: str = "cos_sim",
                      allow: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The same search with the result as ONE tensor of packed 8-byte entries, int64 [Q,k] whose low 32 bits are the
        fp32 score and high 32 bits the int32 global id (-inf / -1 = empty): what a rank contributes to the single
        all-gather of a sharded search (SURVEY.md §8e).  Needs id_base + n < 2^31.  ``allow`` as in ``search``."""
        qb, q_scale, c_scale = self._prepare(queries, k, score_function)
        nq = qb.shape[0]
        mask, pitch = self._mask(allow, nq)
        out = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            rc = _lib.lib().sgpt_search_packed_masked(self._dtype_id(), qb.data_ptr(), self.vectors.data_ptr(),
                                                      _lib.ptr(q_scale), c_scale, nq, self.n, self.dim, k, self.id_base,
                                                      _lib.ptr(mask), pitch, out.data_ptr(), self._ws.data_ptr(),
                                                      self._ws.numel(), _lib.current_stream())
        _lib.check(rc, "sgpt_search_packed")
        if self.dtype == "binary" and score_function == "cos_sim":
            halves = out.view(torch.int32).view(nq, k, 2)
            halves[..., 0] = _b1_cos(halves[..., 0].contiguous().view(torch.float32), self.dim).view(torch.int32)
        return out

    def search_gather(self, gather_handle, queries: torch.Tensor, k: int, score_function: str = "cos_sim",
                      exclude_ids: Optional[torch.Tensor] = None, allow: Optional[torch.Tensor] = None
                      ) -> Tuple[torch.Tensor, torch.Tensor]:
        """``sgpt_search_gather`` on this shard (dist.PeerGather): local exact top-k, pushed to every rank of the gather
        context `gather_handle` and merged there.  Returns the merged (scores fp32 [Q,k], ids int64 [Q,k]).  ``allow``
        (as in ``search``) and the deletions filter this rank's documents; every rank passes its own."""
        qb, q_scale, c_scale = self._prepare(queries, k, score_function)
        nq = qb.shape[0]
        mask, pitch = self._mask(allow, nq)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=self.device)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            rc = _lib.lib().sgpt_search_gather_masked(self._dtype_id(), gather_handle, qb.data_ptr(),
                                                      self.vectors.data_ptr(), _lib.ptr(q_scale), c_scale, nq, self.n,
                                                      self.dim, k, self.id_base, _lib.ptr(mask), pitch,
                                                      _lib.ptr(exclude_ids), out_s.data_ptr(), out_i.data_ptr(),
                                                      self._ws.data_ptr(), self._ws.numel(), _lib.current_stream())
        _lib.check(rc, "sgpt_search_gather")
        if self.dtype == "binary" and score_function == "cos_sim":
            out_s = _b1_cos(out_s, self.dim)
        return out_s, out_i

    def view(self, start: int, end: int) -> "CorpusShard":
        """Documents [start, end) of this shard as a shard of their own that shares the vectors; its ids are the
        positions ``start ..`` inside this shard.  (The scales are copied: the kernels read them 16 bytes at a time.)
        The view shares this shard's deletions, in both directions."""
        v = object.__new__(CorpusShard)
        v.dim, v.capacity, v.id_base, v.device, v.dtype = self.dim, end - start, int(start), self.device, self.dtype
        v.vectors = self.vectors[start:end]
        if self.dtype == "binary":
            v.popcounts = self.popcounts[start:end].clone()
            v.thresholds = self.thresholds
        elif self.dtype == "int8":
            v.scales = self.scales[start:end].clone()
            v.cos_scales = self.cos_scales[start:end].clone()
        else:
            v.inv_norms = self.inv_norms[start:end].clone()
        v.n = end - start
        v._ws = None
        v._deleted, v._deleted_at = self._deleted, self._deleted_at + int(start)
        return v

    def _range_call(self, qb: torch.Tensor, q_scale: Optional[torch.Tensor], c_scale: Optional[int], threshold: float,
                    counts: torch.Tensor, cap: int, out_s: Optional[torch.Tensor], out_i: Optional[torch.Tensor],
                    mask: Tuple[Optional[torch.Tensor], int] = (None, 0)) -> None:
        """One sgpt_range_search_masked of the query rows qb, in the shard's format (include/sgpt_b200.h): counts
        int64[Q] always, the entries of the queries that fit into `cap` into out_s / out_i.  mask: (bitmap, pitch) of
        ``_mask`` for these queries."""
        nq = qb.shape[0]
        ws = self._workspace(_lib.lib().sgpt_range_search_workspace_bytes(nq, self.n))
        with torch.cuda.device(self.device):
            rc = _lib.lib().sgpt_range_search_masked(self._dtype_id(), qb.data_ptr(), self.vectors.data_ptr(),
                                                     _lib.ptr(q_scale), c_scale, nq, self.n, self.dim, float(threshold),
                                                     self.id_base, _lib.ptr(mask[0]), mask[1], counts.data_ptr(), cap,
                                                     _lib.ptr(out_s), _lib.ptr(out_i), ws.data_ptr(), ws.numel(),
                                                     _lib.current_stream())
        _lib.check(rc, "sgpt_range_search")

    def _range(self, qb: torch.Tensor, q_scale: Optional[torch.Tensor], c_scale: Optional[int], threshold: float,
               capacity: Optional[int] = None, mask: Tuple[Optional[torch.Tensor], int] = (None, 0)
               ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        def run(first, counts, cap, out_s, out_i):
            self._range_call(qb[first:], None if q_scale is None else q_scale[first:], c_scale, threshold, counts, cap,
                             out_s, out_i, _mask_rows(mask, first))
        return _grown_range(qb.shape[0], self.device, run, capacity)

    def range_search(self, queries: torch.Tensor, threshold: float, score_function: str = "cos_sim",
                     allow: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Every document whose score against a query is >= threshold, for fp32/bf16 queries [Q, D] (device).

        Returns (offsets int64 [Q+1], scores fp32 [E], global ids int64 [E]) on the device: query q's documents are
        entries offsets[q] .. offsets[q+1], in ascending id order.  Queries are converted and scored exactly as in
        ``search``; a NaN score counts as -1.  The output buffer starts at 64 entries per query and grows once, for the
        queries that did not fit.  ``allow`` as in ``search``: only allowed, undeleted documents are counted and returned.
        On a binary shard the scores are those of ``search`` (s, or s / D for cos_sim), so a "dot" threshold D - 2 r is
        the Hamming ball of radius r."""
        qb, q_scale, c_scale = self._queries(queries, score_function)
        if self.dtype != "binary":
            return self._range(qb, q_scale, c_scale, threshold, mask=self._mask(allow, qb.shape[0]))
        offsets, scores, ids = self._range(qb, q_scale, c_scale, _b1_threshold(threshold, score_function, self.dim),
                                           mask=self._mask(allow, qb.shape[0]))
        return offsets, (_b1_cos(scores, self.dim) if score_function == "cos_sim" else scores), ids


def unpack_topk(packed: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Packed entries int64[...] -> (scores fp32[...], ids int64[...]) (host-side convenience for tests and tools)."""
    halves = packed.contiguous().view(torch.int32).view(*packed.shape, 2)
    return halves[..., 0].contiguous().view(torch.float32), halves[..., 1].to(torch.int64)


def merge_topk_packed(packed: torch.Tensor, exclude_ids: Optional[torch.Tensor] = None
                      ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Merge G packed candidate lists per query: int64 [G,Q,k] -> (scores fp32 [Q,k], ids int64 [Q,k]) descending;
    empty slots and ids == exclude_ids[q] (XS:118) are dropped."""
    G, Q, k = packed.shape
    packed = packed.contiguous()
    out_s = torch.empty((Q, k), dtype=torch.float32, device=packed.device)
    out_i = torch.empty((Q, k), dtype=torch.int64, device=packed.device)
    with torch.cuda.device(packed.device):
        rc = _lib.lib().sgpt_topk_merge_packed(packed.data_ptr(), G, Q, k, out_s.data_ptr(), out_i.data_ptr(),
                                               _lib.ptr(exclude_ids), _lib.current_stream())
    _lib.check(rc, "sgpt_topk_merge_packed")
    return out_s, out_i


def merge_topk(scores: torch.Tensor, ids: torch.Tensor, exclude_ids: Optional[torch.Tensor] = None
               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Merge G candidate lists per query: scores fp32 [G,Q,k], ids int64 [G,Q,k] -> ([Q,k], [Q,k]) descending.
    Entries with id < 0, or id == exclude_ids[q] (int64 [Q], the XS:118 self-match rule), are dropped."""
    G, Q, k = scores.shape
    scores, ids = scores.contiguous(), ids.contiguous()
    out_s = torch.empty((Q, k), dtype=torch.float32, device=scores.device)
    out_i = torch.empty((Q, k), dtype=torch.int64, device=scores.device)
    with torch.cuda.device(scores.device):
        rc = _lib.lib().sgpt_topk_merge(scores.data_ptr(), ids.data_ptr(), G, Q, k, out_s.data_ptr(), out_i.data_ptr(),
                                        _lib.ptr(exclude_ids), None, _lib.current_stream())
    _lib.check(rc, "sgpt_topk_merge")
    return out_s, out_i


def semantic_search(query_embeddings: torch.Tensor, corpus_embeddings: Union[torch.Tensor, CorpusShard],
                    query_chunk_size: int = 100, corpus_chunk_size: int = 500000, top_k: int = 10,
                    score_function="cos_sim", device="cuda:0") -> List[List[Dict[str, Union[int, float]]]]:
    """``sentence_transformers.util.semantic_search`` (ST/util.py:197-258) on the fused exact search: for every query
    the ``top_k`` corpus entries as ``{"corpus_id", "score"}`` dicts, best first.  ``score_function`` is "cos_sim" /
    "dot" or the reference's ``cos_sim`` / ``dot_score`` callables (recognised by name); the chunk sizes of the reference
    are accepted and ignored — the kernel streams the whole shard once and needs no score-matrix chunks."""
    del query_chunk_size, corpus_chunk_size
    score_function = resolve_score_function(score_function)
    q = torch.as_tensor(query_embeddings)
    if q.dim() == 1:
        q = q.unsqueeze(0)  # ST/util.py:214-217
    shard = corpus_embeddings if isinstance(corpus_embeddings, CorpusShard) else CorpusShard.from_embeddings(
        torch.as_tensor(corpus_embeddings).to(device))
    if shard.dtype == "binary":
        raise ValueError("semantic_search does not take binary shards (dtype 'binary'): use CorpusShard.search")
    k = min(int(top_k), shard.n)
    scores, ids = shard.search(q.to(shard.device), k, score_function)
    scores, ids = scores.cpu().tolist(), ids.cpu().tolist()
    return [[{"corpus_id": int(i), "score": float(s)} for s, i in zip(srow, irow) if i >= 0]
            for srow, irow in zip(scores, ids)]
