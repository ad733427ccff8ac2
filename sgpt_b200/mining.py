"""``paraphrase_mining`` and ``community_detection`` of sentence_transformers.util (ST/util.py:101-189, 385-448) on the
library's exact top-k search and range search.

The reference builds the full N x N fp32 score matrix and loops over it in Python.  Here the scores come from the fused
search kernels, which never write a score matrix: paraphrase mining takes each corpus chunk's row top-k on the device
and selects and deduplicates the pairs there with sorts over (score, i, j); community detection counts every row's
documents above the threshold first and fetches the members of the qualifying rows only.  Host work is proportional
to the result.

Both also take an ``IVFIndex`` with ``nprobe``: every undeleted stored row is a query over the undeleted documents of
its probed lists (the IVF search and IVF range search), so the cost grows with n x nprobe x the list length instead of
n^2, and ``nprobe == nlist`` gives the exact functions' result.
"""
from __future__ import annotations

from typing import List, Optional, Tuple, Union

import torch

from .index import CorpusShard, resolve_score_function
from .ivf import IVFIndex

MAX_K = 4096  # the library's top-k limit (include/sgpt_b200.h)
_CANDIDATES_PER_STEP = 1 << 24  # row top-k entries selected per step of paraphrase mining
_MEMBERS_PER_BLOCK = 1 << 26    # community members fetched per range search call
_COUNT_ROWS = 1 << 16           # stored rows per count-only IVF range pass of community detection


def _as_shard(embeddings: Union[torch.Tensor, CorpusShard]) -> CorpusShard:
    """The embeddings as a shard whose ids are row positions 0 .. N-1."""
    if isinstance(embeddings, CorpusShard):
        if embeddings.dtype == "binary":
            raise ValueError("mining does not take binary shards (dtype 'binary'): use bf16 or int8")
        if embeddings.n_deleted > 0:
            # deleted rows would still be mined as queries: refuse rather than return pairs of deleted documents
            raise ValueError(f"mining a CorpusShard with deleted documents ({embeddings.n_deleted}) is not supported")
        return embeddings.view(0, embeddings.n)
    emb = torch.as_tensor(embeddings)
    if emb.dim() == 1:
        emb = emb.unsqueeze(0)
    return CorpusShard.from_embeddings(emb if emb.is_cuda else emb.to("cuda:0"))


def _check_nprobe(embeddings, nprobe) -> None:
    """`nprobe` goes with an IVFIndex and only with one."""
    if isinstance(embeddings, IVFIndex):
        if nprobe is None:
            raise ValueError("mining an IVFIndex needs nprobe (the lists each row scans)")
    elif nprobe is not None:
        raise ValueError("nprobe applies to an IVFIndex only")


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


def paraphrase_mining_embeddings(embeddings: Union[torch.Tensor, CorpusShard, IVFIndex], query_chunk_size: int = 5000,
                                 corpus_chunk_size: int = 100000, max_pairs: int = 500000, top_k: int = 100,
                                 score_function="cos_sim", nprobe: Optional[int] = None) -> List[list]:
    """ST/util.py:129-189: the most similar pairs (i, j) inside one corpus, as ``[[score, i, j], ...]``, best first.

    For every corpus chunk of ``corpus_chunk_size`` documents every row takes its top min(top_k + 1, chunk length)
    documents of the chunk (:148, :155-159), with the library's exact search (ties keep the lowest ids); the chunk size
    therefore changes which candidates exist and is honoured.  ``query_chunk_size`` only bounds the reference's score
    matrix and is ignored.  The candidates go through ``PairSelector`` (:151-188, see there for the tie rule at the
    ``max_pairs`` cut).  ``embeddings`` is a tensor (fp32 / bf16, any device; stored bf16-rounded) or a CorpusShard;
    i and j are row positions.  ``score_function``: "cos_sim" / "dot" or the reference's callables.

    ``embeddings`` may also be an ``IVFIndex``, with ``nprobe`` (required there, a ValueError with any other input):
    then row i's candidates are its top-(top_k + 1) over the undeleted documents of its ``nprobe`` probed lists (the
    probes of its stored row), i and j are global id - id_base (row positions of the embeddings the index was built
    from), deleted documents are neither rows nor candidates, ``score_function`` must be the index's, and
    ``corpus_chunk_size`` does nothing.  ``nprobe == nlist`` gives the pairs of the exact function with one chunk."""
    del query_chunk_size
    name = resolve_score_function(score_function)
    _check_nprobe(embeddings, nprobe)
    k = int(top_k) + 1  # :148
    if k > MAX_K:
        raise ValueError(f"top_k + 1 = {k} exceeds the library's top-k limit of {MAX_K}")
    if isinstance(embeddings, IVFIndex):
        return _pairs_list(_ivf_pairs(embeddings, max_pairs, k, name, int(nprobe)))
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
    return _pairs_list(selector)


def _pairs_list(selector: PairSelector) -> List[list]:
    s, i, j = selector.result()
    return [[score, a, b] for score, a, b in zip(s.tolist(), i.tolist(), j.tolist())]


def _check_index_score_function(index: IVFIndex, name: str) -> None:
    if name != index.score_function:
        raise ValueError(f"score_function {name!r} differs from the IVFIndex's {index.score_function!r}")


def _ivf_pairs(index: IVFIndex, max_pairs: int, k: int, name: str, nprobe: int) -> PairSelector:
    """The candidates of paraphrase mining over an IVF index, in a PairSelector.

    The rows are the undeleted stored rows, fed in position order, i.e. list order: neighbouring rows probe the same
    lists, so the grouped scan's 128-row pair tiles fill up and every list tile is read once for many rows.  This is what
    makes an IVF self-join cheap.  PairSelector does not depend on the order of its input."""
    _check_index_score_function(index, name)
    selector = PairSelector(index.n, max_pairs, index.device)
    if k <= 0:
        return selector
    step = max(256, _CANDIDATES_PER_STEP // k // 256 * 256)
    mask = index.shard._mask(None, 0)  # the deletions, shared by every row
    for pos in index._stored_blocks(step):
        qb, q_scale, c_scale, probes = index._stored_queries(pos, nprobe)
        s, j = index._search_rows(qb, q_scale, c_scale, probes, k, mask)
        i = (index.ids[pos].long() - index.id_base).unsqueeze(1).expand(-1, k)
        selector.add(s.reshape(-1), i.reshape(-1), (j - index.id_base).reshape(-1))
    return selector


def community_detection(embeddings: Union[torch.Tensor, CorpusShard, IVFIndex], threshold: float = 0.75,
                        min_community_size: int = 10, init_max_size: int = 1000,
                        nprobe: Optional[int] = None) -> List[List[int]]:
    """ST/util.py:385-448 ("fast clustering"): communities of documents whose cosine score against a central row is
    >= threshold, largest first, without overlaps.  ``embeddings`` is a tensor (any device; stored bf16-rounded) or a
    CorpusShard; the ids are row positions.

    Row i qualifies iff at least ``min_community_size`` documents score >= threshold against it (:402-407: the
    min_community_size-th largest score reaches the threshold, ties included).  Its community is all of them (:411-425):
    in (score descending, id ascending) order when there are fewer than init_max_size = min(init_max_size, N) (:396,
    the ``topk`` branch), in ascending id order otherwise (the branch that scans the whole row).  The communities are
    sorted stably by size, largest first (:430), and a community that shares a member with an earlier one is dropped
    (:432-446).  The counts of all rows come from one count-only range search; members are fetched for the qualifying
    rows only, in blocks of bounded size.

    ``embeddings`` may also be a cos_sim ``IVFIndex`` (the reference always scores with cos_sim), with ``nprobe``
    (required there, a ValueError with any other input): then row i's documents are those of its ``nprobe`` probed lists
    (the probes of its stored row) with score >= threshold, counted by count-only IVF range searches over all stored rows
    and fetched for the qualifying rows only.  The ids are global id - id_base (row positions of the embeddings the
    index was built from), N is the index's n, and deleted documents are neither central rows nor members.
    ``nprobe == nlist`` gives the communities of the exact function."""
    _check_nprobe(embeddings, nprobe)
    if isinstance(embeddings, IVFIndex):
        return _ivf_communities(embeddings, threshold, min_community_size, init_max_size, int(nprobe))
    shard = _as_shard(embeddings)
    n = shard.n
    if min_community_size > n:
        raise ValueError(f"min_community_size={min_community_size} exceeds the number of embeddings ({n})")
    rows, inv = shard.stored(), shard.inv_norms
    cscale = inv.data_ptr()
    counts = torch.empty(n, dtype=torch.int64, device=shard.device)
    shard._range_call(rows, inv, cscale, threshold, counts, 0, None, None)
    central = torch.nonzero(counts >= min_community_size).flatten()

    def fetch(idx, total):
        return shard._range(rows[idx].contiguous(), inv[idx].contiguous(), cscale, threshold, total)
    return _communities(central, counts[central].tolist(), fetch, min(init_max_size, n), shard.device)


def _ivf_communities(index: IVFIndex, threshold: float, min_community_size: int, init_max_size: int,
                     nprobe: int) -> List[List[int]]:
    """community_detection over an IVF index: counts from count-only IVF range searches over the undeleted stored rows
    in position (= list) order, so that neighbouring rows probe the same lists; then the members of the central rows."""
    _check_index_score_function(index, "cos_sim")
    n, dev = index.n, index.device
    if min_community_size > n:
        raise ValueError(f"min_community_size={min_community_size} exceeds the number of embeddings ({n})")
    mask = index.shard._mask(None, 0)  # the deletions
    by_pos = torch.zeros(n, dtype=torch.int64, device=dev)  # deleted rows keep count 0
    alive = torch.zeros(n, dtype=torch.bool, device=dev)
    for pos in index._stored_blocks(_COUNT_ROWS):
        qb, q_scale, c_scale, probes = index._stored_queries(pos, nprobe)
        counts = torch.empty(qb.shape[0], dtype=torch.int64, device=dev)
        index._range_call(qb, q_scale, c_scale, probes, threshold, mask, counts, 0, None, None)
        by_pos[pos] = counts
        alive[pos] = True
    # id order, so that the central rows come in ascending id as in the exact function
    local = index.ids.long() - index.id_base
    counts = torch.empty_like(by_pos).index_copy_(0, local, by_pos)
    alive = torch.empty_like(alive).index_copy_(0, local, alive)
    central = torch.nonzero((counts >= min_community_size) & alive).flatten()

    def fetch(idx, total):
        qb, q_scale, c_scale, probes = index._stored_queries(index._pos[idx], nprobe)
        offsets, s, ids = index._range_rows(qb, q_scale, c_scale, probes, threshold, mask, total)
        return offsets, s, ids - index.id_base
    return _communities(central, counts[central].tolist(), fetch, min(init_max_size, n), dev)


def _communities(central: torch.Tensor, sizes: List[int], fetch, init_max_size: int, device) -> List[List[int]]:
    """The communities of the central rows (ascending id) with member counts `sizes`: ``fetch(idx, total)`` returns the
    range search of central[idx] in CSR form (each row's members in ascending id, total entries), in blocks of at most
    _MEMBERS_PER_BLOCK members; then the reference's member order, size order and de-duplication (:411-446)."""
    communities: List[List[int]] = []
    a = 0
    while a < len(sizes):
        b, total = a, 0
        while b < len(sizes) and (b == a or total + sizes[b] <= _MEMBERS_PER_BLOCK):
            total += sizes[b]
            b += 1
        offsets, s, ids = fetch(central[a:b], total)
        cnt = offsets[1:] - offsets[:-1]
        seg = torch.repeat_interleave(torch.arange(b - a, device=device), cnt)
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
