"""Generate tests/golden/mining.npz by running the REFERENCE's paraphrase_mining_embeddings and community_detection.

    python tests/golden/make_mining.py          # needs /root/reference; writes mining.npz here

The reference's own ``sentence_transformers/util.py`` is loaded by file path with the two dead ``huggingface_hub``
imports stubbed (make_golden.py load_reference_util).  Both datasets are rounded to bf16 values before the reference
sees them, so the library stores exactly the same vectors.  fp32 accumulation orders differ between the two sides by
about 1e-7 at D = 64, so every decision the result depends on must have a margin of at least 1e-5: the threshold
against every score, each row's top-k cut, the ``max_pairs`` cut, and the order of the scores the output lists.  A
seed whose data misses a margin is replaced by the next one.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.golden.make_golden import load_reference_util  # noqa: E402

MARGIN = 1e-5
N, D = 600, 64


def bf16(x):
    return x.to(torch.bfloat16).float()


def planted(seed):
    """Clusters of 5 .. 80 noisy copies of random centres plus background documents, shuffled."""
    g = torch.Generator().manual_seed(seed)
    sizes = [80, 60, 45, 33, 25, 18, 12, 9, 7, 5]
    rows = []
    for s in sizes:
        c = torch.randn(D, generator=g)
        rows.append(c + 0.35 * torch.randn(s, D, generator=g))
    rows.append(torch.randn(N - sum(sizes), D, generator=g))
    x = torch.cat(rows)
    return bf16(x[torch.randperm(N, generator=g)])


def gap_threshold(scores, target):
    """A threshold near `target` in the middle of a gap of at least 2 MARGIN between sorted scores."""
    v = np.unique(scores.numpy().astype(np.float64).ravel())
    mid = (v[1:] + v[:-1]) / 2
    ok = (v[1:] - v[:-1]) >= 2 * MARGIN
    cand = mid[ok]
    return float(np.float32(cand[np.argmin(np.abs(cand - target))]))


def communities_case(util, seed):
    x = planted(seed)
    cos = util.cos_sim(x, x)
    t = gap_threshold(cos, 0.8)
    cnt = (cos >= t).sum(1)
    min_size, init_max = 6, 16
    assert ((cnt >= min_size) & (cnt < init_max)).any() and (cnt >= init_max).any(), "both branches must occur"
    assert (cos - t).abs().min().item() >= MARGIN
    # members of the topk branch are ordered by score: distinct scores in every such row
    for i in torch.nonzero((cnt >= min_size) & (cnt < init_max)).flatten().tolist():
        v = torch.sort(cos[i][cos[i] >= t], descending=True).values.double()
        if len(v) > 1 and (v[:-1] - v[1:]).min().item() < MARGIN:
            return None
    out = util.community_detection(x, threshold=t, min_community_size=min_size, init_max_size=init_max)
    assert len(out) >= 3
    return dict(x=x, threshold=t, min_size=min_size, init_max=init_max, communities=out)


def pair_margins_ok(util, x, chunk, top_k, max_pairs):
    """The max_pairs cut, the row top-k cuts that reach the kept scores and the order of the kept pairs all clear
    MARGIN.  (A row cut below the lowest kept score decides nothing: neither of its two candidates is kept.)"""
    cands, row_cuts = [], []
    for cs in range(0, N, chunk):
        sc = util.cos_sim(x, x[cs:cs + chunk]).double()
        k = min(top_k + 1, sc.shape[1])
        if k < sc.shape[1]:
            v = torch.sort(sc, dim=1, descending=True).values
            row_cuts += list(zip(v[:, k - 1].tolist(), v[:, k].tolist()))
        top = torch.topk(sc, k, dim=1)
        for r in range(N):
            for s, c in zip(top.values[r].tolist(), top.indices[r].tolist()):
                if r != cs + c and s > -1:
                    cands.append((s, r, cs + c))
    cands.sort(reverse=True)
    assert len(cands) > max_pairs, "the max_pairs cap must bite"
    key = [(min(i, j), max(i, j)) for _, i, j in cands]
    c = max_pairs - 1  # entries kept
    if key[c - 1] == key[c]:  # a pair's two orientations straddle the cut: the pair must stand apart from both sides
        if cands[c - 2][0] - cands[c - 1][0] < MARGIN or cands[c][0] - cands[c + 1][0] < MARGIN:
            return False
    elif cands[c - 1][0] - cands[c][0] < MARGIN:
        return False
    lowest = cands[c - 1][0]
    if any(a - b < MARGIN and a > lowest - MARGIN for a, b in row_cuts):
        return False
    kept = {}
    for s, i, j in cands[:c]:
        kept.setdefault((min(i, j), max(i, j)), s)
    v = np.sort(np.array(list(kept.values())))
    return bool(len(v) < 2 or np.diff(v).min() >= MARGIN)


def pairs_case(util, seed):
    x = planted(seed)
    chunk, top_k, max_pairs = 250, 5, 60
    if not pair_margins_ok(util, x, chunk, top_k, max_pairs):
        return None
    out = util.paraphrase_mining_embeddings(x, query_chunk_size=97, corpus_chunk_size=chunk, max_pairs=max_pairs,
                                            top_k=top_k)
    assert len(out) >= 20
    return dict(x=x, chunk=chunk, top_k=top_k, max_pairs=max_pairs, pairs=out)


def first_seed(make, util, start):
    for seed in range(start, start + 200):
        case = make(util, seed)
        if case is not None:
            return seed, case
    raise RuntimeError("no seed clears the margins")


if __name__ == "__main__":
    torch.set_num_threads(8)
    util = load_reference_util()
    cseed, cc = first_seed(communities_case, util, 100)
    pseed, pc = first_seed(pairs_case, util, 200)
    comm = cc["communities"]
    pairs = np.array(pc["pairs"], dtype=np.float64)
    np.savez_compressed(
        os.path.join(HERE, "mining.npz"),
        comm_x=cc["x"].numpy(), comm_seed=np.int32(cseed), comm_threshold=np.float32(cc["threshold"]),
        comm_min_size=np.int32(cc["min_size"]), comm_init_max=np.int32(cc["init_max"]),
        comm_sizes=np.array([len(c) for c in comm], np.int64), comm_members=np.array(sum(comm, []), np.int64),
        pairs_x=pc["x"].numpy(), pairs_seed=np.int32(pseed), pairs_chunk=np.int32(pc["chunk"]),
        pairs_top_k=np.int32(pc["top_k"]), pairs_max_pairs=np.int32(pc["max_pairs"]),
        pairs_scores=pairs[:, 0].astype(np.float32), pairs_ij=pairs[:, 1:].astype(np.int64))
    print("communities: seed", cseed, "threshold", cc["threshold"], "sizes", [len(c) for c in comm])
    print("pairs: seed", pseed, len(pc["pairs"]), "pairs")
