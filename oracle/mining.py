"""Oracle: paraphrase mining and community detection (test infra only).

Restates sentence_transformers/util.py:129-189 (paraphrase_mining_embeddings) and :385-448 (community_detection) of
biencoder/nli_msmarco/sentence-transformers on a dense score matrix, with a deterministic tie rule wherever the
reference leaves one open: every top-k is ``topk_ids`` (score descending, id ascending), and at the ``max_pairs`` cut
the largest (score, i, j) tuples stay (the reference keeps whichever tied tuples ``torch.topk(sorted=False)`` delivered
first).  ``rule="arrival"`` runs the reference's own admission rule instead, for candidate sets without ties at the cut.
"""
from __future__ import annotations

import heapq
from typing import Iterable, List, Tuple

import torch

from .search import _as_2d, cos_sim, topk_ids


def mine_pairs(candidates: Iterable[Tuple[float, int, int]], max_pairs: int, rule: str = "tuple") -> List[list]:
    """util.py:151-188 over candidates (score, i, j) in arrival order."""
    pairs: list = []  # min-heap of (score, i, j), the reference's PriorityQueue (:151)
    min_score, min_entry = -1, None  # :152
    num_added = 0
    for score, i, j in candidates:
        if i == j:
            continue
        if rule == "arrival":
            admit = score > min_score  # :168
        else:
            admit = score > -1 and (min_entry is None or (score, i, j) > min_entry)
        if admit:
            heapq.heappush(pairs, (score, i, j))  # :169
            num_added += 1
            if num_added >= max_pairs:  # :172-174
                min_entry = heapq.heappop(pairs)
                min_score = min_entry[0]
    added_pairs, pairs_list = set(), []
    while pairs:  # :179-185: ascending tuples, the first of each unordered pair stays
        score, i, j = heapq.heappop(pairs)
        key = (min(i, j), max(i, j))
        if key[0] != key[1] and key not in added_pairs:
            added_pairs.add(key)
            pairs_list.append([score, i, j])
    return sorted(pairs_list, key=lambda x: x[0], reverse=True)  # :188


def paraphrase_mining_embeddings(embeddings, query_chunk_size: int = 5000, corpus_chunk_size: int = 100000,
                                 max_pairs: int = 500000, top_k: int = 100, score_function=cos_sim,
                                 rule: str = "tuple") -> List[list]:
    """util.py:129-189: per (corpus chunk, query chunk) the row top-min(top_k + 1, chunk) (:148, :155-159), candidates
    in that order (:163-170), then ``mine_pairs``."""
    emb = _as_2d(embeddings)
    k = top_k + 1
    candidates = []
    for cs in range(0, len(emb), corpus_chunk_size):
        for qs in range(0, len(emb), query_chunk_size):
            scores = score_function(emb[qs:qs + query_chunk_size], emb[cs:cs + corpus_chunk_size])
            vals, idx = topk_ids(scores, min(k, scores.shape[1]))
            for r, (vrow, irow) in enumerate(zip(vals.tolist(), idx.tolist())):
                candidates.extend((v, qs + r, cs + c) for v, c in zip(vrow, irow))
    return mine_pairs(candidates, max_pairs, rule)


def community_detection(embeddings, threshold: float = 0.75, min_community_size: int = 10,
                        init_max_size: int = 1000) -> List[List[int]]:
    """util.py:385-448 with ``topk_ids`` for both top-k calls."""
    emb = _as_2d(embeddings)
    if min_community_size > len(emb):
        raise ValueError("min_community_size exceeds the number of embeddings")  # torch.topk fails there (:402)
    init_max_size = min(init_max_size, len(emb))  # :396
    cos_scores = cos_sim(emb, emb)  # :399
    top_k_values, _ = topk_ids(cos_scores, min_community_size)  # :402
    extracted = []
    for i in range(len(top_k_values)):
        if top_k_values[i][-1] >= threshold:  # :407
            new_cluster = []
            top_val_large, top_idx_large = topk_ids(cos_scores[i:i + 1], init_max_size)  # :411
            top_val_large, top_idx_large = top_val_large[0].tolist(), top_idx_large[0].tolist()
            if top_val_large[-1] < threshold:  # :415-420
                for idx, val in zip(top_idx_large, top_val_large):
                    if val < threshold:
                        break
                    new_cluster.append(idx)
            else:  # :421-425
                for idx, val in enumerate(cos_scores[i].tolist()):
                    if val >= threshold:
                        new_cluster.append(idx)
            extracted.append(new_cluster)
    extracted = sorted(extracted, key=lambda x: len(x), reverse=True)  # :430
    unique, taken = [], set()
    for community in extracted:  # :436-446
        if not any(idx in taken for idx in community):
            unique.append(community)
            taken.update(community)
    return unique
