"""CPU checks of paraphrase mining and community detection: the oracle against the reference's own results
(tests/golden/mining.npz, tests/golden/make_mining.py), the device-independent pair selection of sgpt_b200/mining.py
against the reference's priority-queue loop, and the host side of sgpt_range_search (argument rejections, workspace
plan)."""
import os

import numpy as np
import pytest
import torch

from oracle import mining as omining
from tests.conftest import GOLDEN


@pytest.fixture(scope="module")
def fx():
    return np.load(os.path.join(GOLDEN, "mining.npz"))


def fixture_communities(fx):
    sizes = fx["comm_sizes"].tolist()
    members = fx["comm_members"].tolist()
    out, pos = [], 0
    for s in sizes:
        out.append(members[pos:pos + s])
        pos += s
    return out


def fixture_pairs(fx):
    return [[float(s), int(i), int(j)] for s, (i, j) in zip(fx["pairs_scores"].tolist(), fx["pairs_ij"].tolist())]


def test_oracle_community_detection_equals_reference(fx):
    got = omining.community_detection(torch.from_numpy(fx["comm_x"]), threshold=float(fx["comm_threshold"]),
                                      min_community_size=int(fx["comm_min_size"]),
                                      init_max_size=int(fx["comm_init_max"]))
    assert got == fixture_communities(fx)


def test_oracle_paraphrase_mining_equals_reference(fx):
    got = omining.paraphrase_mining_embeddings(torch.from_numpy(fx["pairs_x"]), query_chunk_size=97,
                                               corpus_chunk_size=int(fx["pairs_chunk"]),
                                               max_pairs=int(fx["pairs_max_pairs"]), top_k=int(fx["pairs_top_k"]))
    want = fixture_pairs(fx)
    assert [p[1:] for p in got] == [p[1:] for p in want]
    assert [np.float32(p[0]) for p in got] == [np.float32(p[0]) for p in want]


def _select(chunks, n, max_pairs):
    from sgpt_b200.mining import PairSelector

    sel = PairSelector(n, max_pairs, "cpu")
    for s, i, j in chunks:
        sel.add(s, i, j)
    s, i, j = sel.result()
    return [[a, b, c] for a, b, c in zip(s.tolist(), i.tolist(), j.tolist())]


def _candidates(g, n, m, values=None):
    """m candidates (score, i, j) as float32 / int64 tensors: i == j, scores <= -1 and both orientations of a pair
    included; `values` draws the scores from a small set (ties everywhere)."""
    i = torch.randint(0, n, (m,), generator=g)
    j = torch.randint(0, n, (m,), generator=g)
    j[::17] = i[::17]
    flip = torch.arange(m) % 5 == 1  # the reversed orientation of the previous candidate
    i[flip], j[flip] = j.roll(1)[flip], i.roll(1)[flip]
    if values is None:
        s = torch.rand(m, generator=g) * 2.2 - 1.1
    else:
        s = torch.tensor(values)[torch.randint(0, len(values), (m,), generator=g)]
    return s.float(), i, j


def _split(s, i, j, parts):
    bounds = np.linspace(0, len(s), parts + 1).astype(int)
    return [(s[a:b], i[a:b], j[a:b]) for a, b in zip(bounds[:-1], bounds[1:])]


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("max_pairs", [1, 2, 50, 400, 5000])
def test_pair_selection_equals_priority_queue_without_ties(seed, max_pairs):
    """Distinct random scores: the reference's admission rule (score > last popped score) and the largest-tuples rule
    agree, and the device code equals both whatever the chunking."""
    g = torch.Generator().manual_seed(seed)
    n = 300
    s, i, j = _candidates(g, n, 2000)
    cands = list(zip(s.tolist(), i.tolist(), j.tolist()))
    want = omining.mine_pairs(cands, max_pairs, rule="arrival")
    assert want == omining.mine_pairs(cands, max_pairs, rule="tuple")
    for parts in (1, 3, 7):
        assert _select(_split(s, i, j, parts), n, max_pairs) == want


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("max_pairs", [2, 10, 37, 400])
def test_pair_selection_keeps_the_largest_tuples_on_ties(seed, max_pairs):
    """Scores from five values (+0.0 and -0.0 among them, which Python counts equal): the cut falls inside a tie, where
    the device code keeps the largest (score, i, j) tuples."""
    g = torch.Generator().manual_seed(100 + seed)
    n = 40
    s, i, j = _candidates(g, n, 1500, values=[-1.0, -0.5, -0.0, 0.0, 0.25, 0.75])
    cands = list(zip(s.tolist(), i.tolist(), j.tolist()))
    want = omining.mine_pairs(cands, max_pairs, rule="tuple")
    for parts in (1, 4):
        got = _select(_split(s, i, j, parts), n, max_pairs)
        assert [p[1:] for p in got] == [p[1:] for p in want]
        assert [p[0] == q[0] for p, q in zip(got, want)] == [True] * len(want)


def _range_call(nq=4, n=1000, D=64, threshold=0.5, cap=10, counts=True, outs=True, ws_bytes=1 << 40):
    from sgpt_b200 import _lib

    dummy = np.zeros(64, dtype=np.int64)
    p = dummy.ctypes.data
    return _lib.lib().sgpt_range_search(p, p, None, None, nq, n, D, threshold, 0, p if counts else None, cap,
                                        p if outs else None, p if outs else None, p, ws_bytes, None)


@pytest.mark.parametrize("change,message", [
    (dict(threshold=float("nan")), b"threshold is NaN"),
    (dict(D=60), b"D=60 must be a positive multiple of 8"),
    (dict(n=1 << 31), b"outside [0, 2^31)"),
    (dict(n=-1), b"outside [0, 2^31)"),
    (dict(nq=-1), b"bad sizes nq=-1"),
    (dict(cap=-1), b"bad sizes nq=4 cap=-1"),
    (dict(counts=False), b"null out_counts"),
    (dict(outs=False), b"null out_scores / out_ids with cap=10"),
    (dict(ws_bytes=1000), b"workspace too small"),
])
def test_range_search_rejects_bad_arguments(change, message):
    """sgpt_range_search validates before any kernel launch: SGPT_ERR_INVALID and a message naming the problem."""
    from sgpt_b200 import _lib

    assert _range_call(**change) == 1
    assert message in _lib.lib().sgpt_last_error()


def test_range_search_count_only_needs_no_entry_buffers():
    """cap = 0 writes no entries, so null out_scores / out_ids are accepted (nq = 0 returns before any CUDA call)."""
    assert _range_call(nq=0, cap=0, outs=False, counts=False) == 0


def test_range_search_workspace_covers_every_query_block():
    """Batches above 256 queries run in blocks that reuse one workspace; the last block may hold <= 128 queries and take
    the single-CTA list layout, so the size for nq must cover every block size that can occur (no GPU needed: the SM
    count falls back to 132)."""
    from sgpt_b200 import _lib

    ws = _lib.lib().sgpt_range_search_workspace_bytes
    for n in (1, 255, 257, 100_000, 1_000_000):
        for nq in (1, 128, 129, 200, 256, 257, 300, 385, 600, 5000):
            need = ws(nq, n)
            blocks = {min(256, nq)} | ({nq % 256} if nq > 256 and nq % 256 else set())
            for nb in blocks:
                assert need >= ws(nb, n), (nq, nb, n)
    # the candidate lists dominate: ~8 bytes per (query, document), as the two-pass search
    assert 0.9 < ws(256, 1_000_000) / (256 * 1_000_000 * 8) < 1.2
    assert ws(0, 1000) > 0
