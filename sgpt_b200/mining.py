"""``paraphrase_mining`` and ``community_detection`` of sentence_transformers.util (ST/util.py:101-189, 385-448) on the
library's exact top-k search and range search.

The reference builds the full N x N fp32 score matrix and loops over it in Python.  Here the scores come from the fused
search kernels, which never write a score matrix: paraphrase mining takes each corpus chunk's row top-k on the device
and selects and deduplicates the pairs there with sorts over (score, i, j); community detection counts every row's
documents above the threshold first and fetches the members of the qualifying rows only.  Host work is proportional
to the result.
"""
from __future__ import annotations

from typing import List, Tuple, Union

import torch

from .index import CorpusShard, resolve_score_function

MAX_K = 4096  # the library's top-k limit (include/sgpt_b200.h)
_CANDIDATES_PER_STEP = 1 << 24  # row top-k entries selected per step of paraphrase mining
_MEMBERS_PER_BLOCK = 1 << 26    # community members fetched per range search call


def _as_shard(embeddings: Union[torch.Tensor, CorpusShard]) -> CorpusShard:
    """The embeddings as a shard whose ids are row positions 0 .. N-1."""
    if isinstance(embeddings, CorpusShard):
        if embeddings.n_deleted > 0:
            # deleted rows would still be mined as queries: refuse rather than return pairs of deleted documents
            raise ValueError(f"mining a CorpusShard with deleted documents ({embeddings.n_deleted}) is not supported")
        return embeddings.view(0, embeddings.n)
    emb = torch.as_tensor(embeddings)
    if emb.dim() == 1:
        emb = emb.unsqueeze(0)
    return CorpusShard.from_embeddings(emb if emb.is_cuda else emb.to("cuda:0"))


def _tuple_order(s: torch.Tensor, i: torch.Tensor, j: torch.Tensor, n: int, descending: bool) -> torch.Tensor:
    """Permutation that sorts the (score, i, j) tuples (lexicographic, as Python compares them).  Scores must be free
    of NaN and -0.0 (Python counts -0.0 equal to +0.0; the radix sort would not)."""
    o = torch.argsort(i * n + j, descending=descending, stable=True)
    return o[torch.argsort(s[o], descending=descending, stable=True)]


class PairSelector:
    """The priority queue of ST/util.py:151-174 and the deduplication of :177-188, over candidate tensors on any device.

    A candidate (score, i, j) is admitted when i != j and score > -1 (:152, :168).  Once ``max_pairs`` candidates have
    been admitted, every further admission pops the smallest tuple (:172-174), so the queue ends with the max_pairs - 1
    largest admitted tuples.  The reference compares a newcomer with the last popped score only, so at a tie with
    that score which tuples stay depends on the order in which ``torch.topk(sorted=False)`` delivered them, which is
    unspecified; here the largest tuples stay.  Of (i, j) and (j, i) the smaller tuple survives (it is popped first,
    :179-185).  The result is ordered by score descending, ties by ascending (i, j) (:188 sorts the popped, ascending
    list stably)."""

    def __init__(self, n: int, max_pairs: int, device):
        self.n, self.max_pairs = int(n), int(max_pairs)
        self.admitted = 0
        self.s = torch.empty(0, dtype=torch.float32, device=device)
        self.i = torch.empty(0, dtype=torch.int64, device=device)
        self.j = torch.empty(0, dtype=torch.int64, device=device)

    def add(self, s: torch.Tensor, i: torch.Tensor, j: torch.Tensor) -> None:
        keep = (i != j) & (s > -1)
        self.admitted += int(keep.sum())
        s = torch.cat([self.s, s[keep] + 0.0])  # + 0.0: -0.0 -> +0.0
        i = torch.cat([self.i, i[keep]])
        j = torch.cat([self.j, j[keep]])
        limit = max(self.max_pairs, 0)  # the largest max_pairs of the union contain those of every later union
        if s.numel() > limit:
            o = _tuple_order(s, i, j, self.n, descending=True)[:limit]
            s, i, j = s[o], i[o], j[o]
        self.s, self.i, self.j = s, i, j

    def result(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        s, i, j = self.s, self.i, self.j
        if self.admitted >= self.max_pairs:
            o = _tuple_order(s, i, j, self.n, descending=True)[:max(self.max_pairs - 1, 0)]
            s, i, j = s[o], i[o], j[o]
        # ascending tuple order; the first tuple of every unordered pair survives
        o = _tuple_order(s, i, j, self.n, descending=False)
        s, i, j = s[o], i[o], j[o]
        pair = torch.minimum(i, j) * self.n + torch.maximum(i, j)
        by_pair = torch.argsort(pair, stable=True)
        first = torch.ones_like(by_pair, dtype=torch.bool)
        first[1:] = pair[by_pair[1:]] != pair[by_pair[:-1]]
        keep = torch.sort(by_pair[first]).values
        s, i, j = s[keep], i[keep], j[keep]
        o = torch.argsort(s, descending=True, stable=True)
        return s[o], i[o], j[o]


def paraphrase_mining(model, sentences: List[str], show_progress_bar: bool = False, batch_size: int = 32, *args,
                      **kwargs) -> List[list]:
    """ST/util.py:101-126: encode the sentences with ``model`` (e.g. a SentenceEncoder) and mine them with
    ``paraphrase_mining_embeddings(embeddings, *args, **kwargs)``."""
    embeddings = model.encode(sentences, show_progress_bar=show_progress_bar, batch_size=batch_size,
                              convert_to_tensor=True)
    return paraphrase_mining_embeddings(embeddings, *args, **kwargs)


def paraphrase_mining_embeddings(embeddings: Union[torch.Tensor, CorpusShard], query_chunk_size: int = 5000,
                                 corpus_chunk_size: int = 100000, max_pairs: int = 500000, top_k: int = 100,
                                 score_function="cos_sim") -> List[list]:
    """ST/util.py:129-189: the most similar pairs (i, j) inside one corpus, as ``[[score, i, j], ...]``, best first.

    For every corpus chunk of ``corpus_chunk_size`` documents every row takes its top min(top_k + 1, chunk length)
    documents of the chunk (:148, :155-159), with the library's exact search (ties keep the lowest ids); the chunk size
    therefore changes which candidates exist and is honoured.  ``query_chunk_size`` only bounds the reference's score
    matrix and is ignored.  The candidates go through ``PairSelector`` (:151-188, see there for the tie rule at the
    ``max_pairs`` cut).  ``embeddings`` is a tensor (fp32 / bf16, any device; stored bf16-rounded) or a CorpusShard;
    i and j are row positions.  ``score_function``: "cos_sim" / "dot" or the reference's callables."""
    del query_chunk_size
    name = resolve_score_function(score_function)
    k = int(top_k) + 1  # :148
    if k > MAX_K:
        raise ValueError(f"top_k + 1 = {k} exceeds the library's top-k limit of {MAX_K}")
    shard = _as_shard(embeddings)
    n = shard.n
    selector = PairSelector(n, max_pairs, shard.device)
    rows = shard.stored()
    if k > 0:
        for cs in range(0, n, corpus_chunk_size):
            chunk = shard.view(cs, min(cs + corpus_chunk_size, n))
            kc = min(k, chunk.n)
            step = max(256, _CANDIDATES_PER_STEP // kc // 256 * 256)
            for qs in range(0, n, step):
                qe = min(qs + step, n)
                s, j = chunk.search(rows[qs:qe], kc, name)
                i = torch.arange(qs, qe, device=shard.device).unsqueeze(1).expand(-1, kc)
                selector.add(s.reshape(-1), i.reshape(-1), j.reshape(-1))
    s, i, j = selector.result()
    return [[score, a, b] for score, a, b in zip(s.tolist(), i.tolist(), j.tolist())]


def community_detection(embeddings: Union[torch.Tensor, CorpusShard], threshold: float = 0.75,
                        min_community_size: int = 10, init_max_size: int = 1000) -> List[List[int]]:
    """ST/util.py:385-448 ("fast clustering"): communities of documents whose cosine score against a central row is
    >= threshold, largest first, without overlaps.  ``embeddings`` is a tensor (any device; stored bf16-rounded) or a
    CorpusShard; the ids are row positions.

    Row i qualifies iff at least ``min_community_size`` documents score >= threshold against it (:402-407: the
    min_community_size-th largest score reaches the threshold, ties included).  Its community is all of them (:411-425):
    in (score descending, id ascending) order when there are fewer than init_max_size = min(init_max_size, N) (:396,
    the ``topk`` branch), in ascending id order otherwise (the branch that scans the whole row).  The communities are
    sorted stably by size, largest first (:430), and a community that shares a member with an earlier one is dropped
    (:432-446).  The counts of all rows come from one count-only range search; members are fetched for the qualifying
    rows only, in blocks of bounded size."""
    shard = _as_shard(embeddings)
    n = shard.n
    if min_community_size > n:
        raise ValueError(f"min_community_size={min_community_size} exceeds the number of embeddings ({n})")
    init_max_size = min(init_max_size, n)
    rows, inv = shard.stored(), shard.inv_norms
    cscale = inv.data_ptr()
    counts = torch.empty(n, dtype=torch.int64, device=shard.device)
    shard._range_call(rows, inv, cscale, threshold, counts, 0, None, None)
    central = torch.nonzero(counts >= min_community_size).flatten()
    sizes = counts[central].tolist()
    communities: List[List[int]] = []
    a = 0
    while a < len(sizes):
        b, total = a, 0
        while b < len(sizes) and (b == a or total + sizes[b] <= _MEMBERS_PER_BLOCK):
            total += sizes[b]
            b += 1
        idx = central[a:b]
        offsets, s, ids = shard._range(rows[idx].contiguous(), inv[idx].contiguous(), cscale, threshold, total)
        cnt = offsets[1:] - offsets[:-1]
        seg = torch.repeat_interleave(torch.arange(b - a, device=shard.device), cnt)
        # topk-branch rows: score descending (stable: ties keep the ascending ids); the others keep the id order
        key = torch.where((cnt < init_max_size)[seg], -s + 0.0, torch.zeros_like(s))
        o = torch.argsort(key, stable=True)
        o = o[torch.argsort(seg[o], stable=True)]
        members = ids[o].tolist()
        pos = 0
        for c in sizes[a:b]:
            communities.append(members[pos:pos + c])
            pos += c
        a = b
    communities = sorted(communities, key=len, reverse=True)  # stable, like :430
    unique, taken = [], set()
    for community in communities:
        if not any(idx in taken for idx in community):
            unique.append(community)
            taken.update(community)
    return unique
