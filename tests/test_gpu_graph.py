"""GPU tests of the graph index: sgpt_graph_prune and GraphIndex.build against the numpy restatement (tests/graph_ref.py)
bit for bit, sgpt_graph_search against the restatement driven by sgpt_rerank's full score table (ids, score bits and
visited counts), the complete-graph case, deletions, repeat launches, save / load, and recall on low-dimensional data."""
import numpy as np
import pytest
import torch

from tests import graph_ref

pytestmark = pytest.mark.gpu


def _overlapping_lists(n, K, g):
    """Random k-NN lists with heavy overlap: row a draws K distinct rows of its block of 3 K rows, so neighbours share
    most of their lists; sprinkled with -1, out-of-range entries, repeats and the row itself."""
    knn = np.empty((n, K), dtype=np.int64)
    for a in range(n):
        lo = min(max(0, a - 3 * K // 2), n - 3 * K)
        knn[a] = lo + g.permutation(3 * K)[:K]
    knn[g.random((n, K)) < 0.03] = -1
    knn[g.random((n, K)) < 0.02] = n + 7
    rep = g.random((n, K)) < 0.02
    knn[:, 1:][rep[:, 1:]] = knn[:, :-1][rep[:, 1:]]
    knn[::9, 2] = np.arange(0, n, 9)
    return knn


@pytest.mark.parametrize("K,degree", [(64, 16), (64, 32), (64, 64), (128, 16), (128, 32), (128, 64)])
def test_prune_equals_the_restatement(K, degree):
    from sgpt_b200.graph import prune

    g = np.random.default_rng(K + degree)
    n = 700
    knn = _overlapping_lists(n, K, g)
    got = prune(torch.from_numpy(knn).cuda(), degree).cpu().numpy()
    assert np.array_equal(got, graph_ref.prune(knn, degree))


def _shard(n, D, dtype, seed, id_base=0, capacity=None):
    from sgpt_b200 import CorpusShard

    g = torch.Generator().manual_seed(seed)
    # rows near a 16-dimensional subspace: a graph over them is well connected
    x = torch.randn(n, 16, generator=g) @ torch.randn(16, D, generator=g) + 0.3 * torch.randn(n, D, generator=g)
    q = x[torch.randint(n, (24,), generator=g)] + 0.5 * torch.randn(24, D, generator=g)
    shard = CorpusShard(D, capacity or n, dtype=dtype, id_base=id_base)
    shard.add(x.cuda())
    return shard, q.cuda()


def test_build_equals_restated_prune_and_merge_and_repeats():
    from sgpt_b200 import GraphIndex
    from sgpt_b200.graph import self_knn

    shard, _ = _shard(1500, 64, "bf16", 1, id_base=40)
    knn = self_knn(shard, 64, "cos_sim")
    own = torch.arange(1500, device="cuda")[:, None] + 40
    assert not (knn == own).any()
    want = graph_ref.merge(graph_ref.prune((knn - 40).cpu().numpy(), 32))
    a = GraphIndex.build(shard, degree=32, intermediate_degree=64)
    b = GraphIndex.build(shard, degree=32, intermediate_degree=64)
    assert np.array_equal(a.graph.cpu().numpy(), want)
    assert torch.equal(a.graph, b.graph)


def _table(shard, q, sf):
    """s(q, x) for every position: sgpt_rerank with every id as a candidate and k = kc = n."""
    from sgpt_b200.ivfpq import rerank

    n = shard.n
    cand = (torch.arange(n, device="cuda") + shard.id_base).repeat(q.shape[0], 1)
    s, i = rerank(shard, q, cand, n, sf)
    t = torch.empty_like(s)
    t.scatter_(1, i - shard.id_base, s)
    return t.cpu().numpy()


SEARCH_CASES = [
    # dtype, D, sf, caller seeds, search_width, itopk, k, max_iterations
    ("bf16", 768, "cos_sim", False, 1, 64, 10, 60),
    ("bf16", 768, "cos_sim", False, 1, 64, 10, 3),
    ("bf16", 776, "dot", True, 2, 64, 64, 40),
    ("bf16", 4096, "cos_sim", False, 4, 32, 32, 20),
    ("int8", 784, "cos_sim", True, 3, 96, 96, 30),
    ("int8", 784, "dot", False, 1, 64, 20, 5),
]


@pytest.mark.parametrize("dtype,D,sf,caller_seeds,sw,itopk,k,iters", SEARCH_CASES)
def test_search_equals_the_restatement(dtype, D, sf, caller_seeds, sw, itopk, k, iters):
    from sgpt_b200 import GraphIndex

    n = 1200 if D == 4096 else 3000
    shard, q = _shard(n, D, dtype, D + sw, id_base=7)
    index = GraphIndex.build(shard, degree=32, intermediate_degree=64, score_function=sf)
    table = _table(shard, q, sf)
    g = torch.Generator().manual_seed(k)
    seeds = torch.randint(-3, n + 3, (q.shape[0], 24), generator=g) + 7 if caller_seeds else None
    kw = dict(itopk=itopk, search_width=sw, max_iterations=iters, return_visited=True)
    if caller_seeds:
        s, i, v = index.search(q, k, seeds=seeds.cuda(), **kw)
        ws, wi, wv = graph_ref.search(table, index.graph.cpu().numpy(), k, itopk, sw, iters, 24,
                                      seeds=(seeds - 7).numpy(), id_base=7)
    else:
        s, i, v = index.search(q, k, num_seeds=40, seed=5, **kw)
        ws, wi, wv = graph_ref.search(table, index.graph.cpu().numpy(), k, itopk, sw, iters, 40, seed=5, id_base=7)
    assert np.array_equal(i.cpu().numpy(), wi)
    assert np.array_equal(s.cpu().numpy().view(np.uint32), ws.view(np.uint32))
    assert np.array_equal(v.cpu().numpy(), wv)
    ok = i.cpu().numpy() >= 0
    rows = np.nonzero(ok)
    assert np.array_equal(s.cpu().numpy()[ok], table[rows[0], i.cpu().numpy()[ok] - 7] + np.float32(0))
    s2, i2, v2 = index.search(q, k, seeds=None if seeds is None else seeds.cuda(),
                              **(dict(num_seeds=40, seed=5) if seeds is None else {}), **kw)
    assert torch.equal(i, i2) and torch.equal(s.view(torch.int32), s2.view(torch.int32)) and torch.equal(v, v2)


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_complete_graph_returns_the_exact_top_k(dtype):
    from sgpt_b200 import GraphIndex
    from sgpt_b200.ivfpq import rerank

    n, k = 300, 100
    shard, q = _shard(n, 256, dtype, 3, id_base=11)
    full = torch.tensor([[(x + 1 + j) % n for j in range(n - 1)] for x in range(n)], dtype=torch.int32)
    index = GraphIndex(shard, full, "cos_sim")  # one expansion visits everything
    s, i, v = index.search(q, k, itopk=320, num_seeds=1, max_iterations=3, return_visited=True)
    assert (v == n).all()
    cand = (torch.arange(n, device="cuda") + 11).repeat(q.shape[0], 1)
    ws, wi = rerank(shard, q, cand, k, "cos_sim")
    assert torch.equal(i, wi) and torch.equal(s.view(torch.int32), ws.view(torch.int32))


def test_deleted_documents_are_walked_but_never_returned():
    from sgpt_b200 import GraphIndex
    from sgpt_b200.index import unpack_mask

    shard, q = _shard(3000, 128, "bf16", 8)
    index = GraphIndex.build(shard)
    shard.remove(torch.arange(0, 3000, 3))
    s, i, v = index.search(q, 30, itopk=64, num_seeds=64, seed=1, max_iterations=50, return_visited=True)
    assert ((i % 3 != 0) | (i < 0)).all() and (i >= 0).sum() > 0.9 * i.numel()
    mask = ~unpack_mask(shard._deleted["words"], 3000).cpu().numpy()
    ws, wi, wv = graph_ref.search(_table(shard, q, "cos_sim"), index.graph.cpu().numpy(), 30, 64, 1, 50, 64, seed=1,
                                  mask=mask)
    assert np.array_equal(i.cpu().numpy(), wi) and np.array_equal(s.cpu().numpy(), ws)
    assert np.array_equal(v.cpu().numpy(), wv)


def test_save_load_round_trip(tmp_path):
    from sgpt_b200 import GraphIndex

    shard, q = _shard(2000, 64, "int8", 4, id_base=3, capacity=2001)
    index = GraphIndex.build(shard, degree=16, intermediate_degree=32, score_function="dot")
    index.save(str(tmp_path / "g"))
    back = GraphIndex.load(str(tmp_path / "g"), shard)
    assert torch.equal(back.graph, index.graph) and back.score_function == "dot" and back.nbytes == 2000 * 16 * 4
    a, b = index.search(q, 10), back.search(q, 10)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    shard.add(torch.randn(1, 64).cuda())
    with pytest.raises(ValueError, match="built over 2000"):
        index.search(q, 10)


def test_recall_on_low_intrinsic_dimension_rows():
    """100 k rows G z + 0.1 eps (z ~ N(0, I_16), G a fixed 768 x 16 matrix), 200 queries from the same law, itopk 128,
    hashed seeds and default iterations: recall@10 against the exact search must be >= 0.95 (measured: 1.0000 on an
    H100 SXM)."""
    from sgpt_b200 import CorpusShard, GraphIndex

    g = torch.Generator(device="cuda").manual_seed(0)
    G = torch.randn(768, 16, generator=g, device="cuda")
    x = torch.randn(100_200, 16, generator=g, device="cuda") @ G.T
    x += 0.1 * torch.randn(x.shape, generator=g, device="cuda")
    shard = CorpusShard.from_embeddings(x[:100_000])
    q = x[100_000:]
    index = GraphIndex.build(shard)
    _, exact = shard.search(q, 10)
    _, got = index.search(q, 10, itopk=128)
    hit = sum(len(set(a) & set(b)) for a, b in zip(got.tolist(), exact.tolist()))
    recall = hit / exact.numel()
    print(f"graph recall@10 = {recall:.4f}")
    assert recall >= 0.95
