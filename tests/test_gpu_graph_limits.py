"""GPU tests of the graph index at the limits of its kernels, bit for bit against the numpy restatement
(tests/graph_ref.py).

- sgpt_graph_prune at K up to 256 (a half-full id -> rank map) and degree up to 128, with degenerate rows and tiny n.
- merge_reverse and from_knn at degrees 16, 64 and 128 with hub rows whose reverse lists are cut.
- GraphIndex.build at degree 128 from 256-entry lists, and self_knn on duplicate-heavy rows with deletions.
- sgpt_graph_search at every degree, the widest step (search_width x degree = 512), itopk = 512, num_seeds = 512, both
  32768-slot visited tables, thousands of queries, ids at the top of the int32 range, the warp scorer's D edges, and
  tie-heavy, NaN, +-inf, all-zero and tiny inputs.

Every search runs once into outputs prefilled with NaN and a sentinel and is compared with the restatement driven by
sgpt_rerank's score table (ids, score bits and visited counts); GraphIndex.search must then return the same bits."""
import numpy as np
import pytest
import torch

from tests import graph_ref

pytestmark = pytest.mark.gpu

SENTINEL = -7  # never an id, a position or a visited count
TOP = 2 ** 31  # global ids must stay below it


def _lib():
    from sgpt_b200 import _lib

    return _lib


# ---- prune ----------------------------------------------------------------------------------------------------------
def _lists(n, K, g, hub=5):
    """k-NN lists with heavy overlap (row a draws K distinct rows of a window of 3 K rows), sprinkled with -1,
    out-of-range entries, repeats and the row itself; a hub id at the head of most lists; and the degenerate rows: all
    -1, every entry the row itself, one id K times."""
    knn = np.empty((n, K), dtype=np.int64)
    for a in range(n):
        lo = min(max(0, a - 3 * K // 2), n - 3 * K)
        knn[a] = lo + g.permutation(3 * K)[:K]
    knn[g.random((n, K)) < 0.03] = -1
    knn[g.random((n, K)) < 0.02] = n + 7
    rep = g.random((n, K)) < 0.02
    knn[:, 1:][rep[:, 1:]] = knn[:, :-1][rep[:, 1:]]
    knn[::9, 2] = np.arange(0, n, 9)
    knn[g.random(n) < 0.8, 0] = hub
    knn[10] = -1
    knn[11] = 11
    knn[12] = 13
    return knn


def _check_prune(knn, degree):
    from sgpt_b200.graph import prune

    n, K = knn.shape
    lib = _lib()
    d = torch.from_numpy(knn).to("cuda", torch.int32).contiguous()
    out = torch.full((n, degree), SENTINEL, dtype=torch.int32, device="cuda")
    lib.check(lib.lib().sgpt_graph_prune(d.data_ptr(), n, K, degree, out.data_ptr(), lib.current_stream()),
              "sgpt_graph_prune")
    want = graph_ref.prune(knn, degree)
    assert np.array_equal(out.cpu().numpy(), want)
    assert torch.equal(prune(d, degree), out)
    return want


PRUNE_CASES = [(K, d) for K in (16, 100, 128, 256) for d in (16, 48, 128) if d <= K]


@pytest.mark.parametrize("K,degree", PRUNE_CASES, ids=[f"K{K}-degree{d}" for K, d in PRUNE_CASES])
def test_prune_at_every_list_length_and_degree(K, degree):
    g = np.random.default_rng(1000 * K + degree)
    n = 2003 + 3 * K
    knn = _lists(n, K, g)
    want = _check_prune(knn, degree)
    assert (want[10] == -1).all() and (want[11] == -1).all() and want[12].tolist() == [13] + [-1] * (degree - 1)
    assert (want[:, 0] == 5).sum() > n // 2  # the hub heads most pruned lists


@pytest.mark.parametrize("n,K,degree", [(1, 16, 16), (2, 100, 48), (3, 256, 128), (37, 256, 128), (90, 128, 16)])
def test_prune_with_fewer_rows_than_entries(n, K, degree):
    g = np.random.default_rng(n + K)
    knn = g.integers(-3, 3 * n + 3, (n, K))  # most entries outside [0, n)
    _check_prune(knn, degree)


# ---- merge_reverse, from_knn, build, self_knn ---------------------------------------------------------------------
def _pruned_with_hubs(n, degree, g):
    """Pruned-shaped lists int32 [n, degree]: distinct entries, a -1 tail of random length and a few -1 holes; hubs 0, 1
    and 2 in the first half of most lists at every rank, so each hub has far more than degree / 2 in-edges."""
    half = degree // 2
    out = np.full((n, degree), -1, dtype=np.int32)
    for a in range(n):
        m = int(g.integers(degree // 4, degree + 1))
        row = g.choice(np.arange(3, n), m, replace=False)
        for h in (0, 1, 2):
            if g.random() < 0.7:
                row[int(g.integers(0, min(m, half)))] = h
        out[a, :m] = row
    out[g.random((n, degree)) < 0.02] = -1
    return out


@pytest.mark.parametrize("degree", [16, 64, 128])
def test_merge_reverse_cuts_the_reverse_lists_of_hubs(degree):
    from sgpt_b200.graph import merge_reverse

    g = np.random.default_rng(degree)
    n = 2500
    pruned = _pruned_with_hubs(n, degree, g)
    for h in (0, 1, 2):
        assert (pruned[:, :degree // 2] == h).sum() > 4 * degree
    got = merge_reverse(torch.from_numpy(pruned).cuda())
    assert np.array_equal(got.cpu().numpy(), graph_ref.merge(pruned))
    assert torch.equal(merge_reverse(torch.from_numpy(pruned).cuda()), got)


def _rows(n, D, g):
    """Rows near a 16-dimensional subspace (a graph over them is well connected), fp32 on the host."""
    return torch.randn(n, 16, generator=g) @ torch.randn(16, D, generator=g) + 0.3 * torch.randn(n, D, generator=g)


def _shard(x, dtype, id_base=0):
    from sgpt_b200 import CorpusShard

    return CorpusShard.from_embeddings(x.cuda(), dtype=dtype, id_base=id_base)


@pytest.mark.parametrize("degree,K", [(16, 40), (64, 100), (128, 160)])
def test_from_knn_equals_restated_prune_and_merge(degree, K):
    from sgpt_b200 import GraphIndex

    g = np.random.default_rng(degree + K)
    n, base = 2200, 1000
    shard = _shard(_rows(n, 32, torch.Generator().manual_seed(K)), "bf16", id_base=base)
    ids = _lists(n, K, g) + base  # -1 and n + 7 become ids outside the shard
    ids[g.random((n, K)) < 0.01] = 3
    local = np.where((ids >= base) & (ids < base + n), ids - base, -1)
    pruned = graph_ref.prune(local, degree)
    assert (pruned[:, :degree // 2] == 5).sum() > 4 * degree  # the hub heads most pruned lists: its R is cut
    want = graph_ref.merge(pruned)
    a = GraphIndex.from_knn(shard, torch.from_numpy(ids), degree)
    assert np.array_equal(a.graph.cpu().numpy(), want)
    assert torch.equal(GraphIndex.from_knn(shard, torch.from_numpy(ids), degree).graph, a.graph)


def _self_table(shard, sf):
    """The exact search's score of every stored row (int8 dequantized, as self_knn queries them) against every
    position: fp32 [n, n] (n <= 4096)."""
    from sgpt_b200.ivf import _rows_f32

    n, base = shard.n, shard.id_base
    pos = torch.arange(n, device="cuda")
    rows = shard.vectors[:n] if shard.dtype == "bf16" else _rows_f32(shard, pos)
    s, i = shard.search(rows, n, sf)
    assert (i >= base).all()
    t = torch.full((n, n), float("nan"), device="cuda")
    t.scatter_(1, i - base, s)
    return t.cpu().numpy()


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_build_at_degree_128_from_256_entry_lists(dtype):
    from sgpt_b200 import GraphIndex
    from sgpt_b200.graph import self_knn

    n, base = 2600, 3
    shard = _shard(_rows(n, 64, torch.Generator().manual_seed(2)), dtype, id_base=base)
    knn = self_knn(shard, 256, "cos_sim")
    assert np.array_equal(knn.cpu().numpy(), graph_ref.self_knn(_self_table(shard, "cos_sim"), 256, id_base=base))
    want = graph_ref.merge(graph_ref.prune((knn - base).cpu().numpy(), 128))
    a = GraphIndex.build(shard, degree=128, intermediate_degree=256)
    assert np.array_equal(a.graph.cpu().numpy(), want)
    assert torch.equal(GraphIndex.build(shard, degree=128, intermediate_degree=256).graph, a.graph)


@pytest.mark.parametrize("dtype,sf", [("bf16", "cos_sim"), ("int8", "dot"), ("bf16", "dot")])
def test_self_knn_on_duplicate_heavy_rows(dtype, sf):
    """Rows drawn from 5 distinct integer vectors (about 300 copies each, far more than K + 1 = 65) and a few unique
    rows: the top-(K + 1) cut and the own-id removal fall inside ties, broken by ascending id.  Every 7th row is
    deleted."""
    from sgpt_b200.graph import self_knn

    g = torch.Generator().manual_seed(5)
    n, K, D, base = 1500, 64, 48, 20
    basis = torch.randint(-4, 5, (5, D), generator=g).float()
    x = basis[torch.randint(5, (n,), generator=g)]
    x[::50] = torch.randint(-4, 5, (n // 50, D), generator=g).float()
    shard = _shard(x, dtype, id_base=base)
    table = _self_table(shard, sf)
    shard.remove(torch.arange(base, base + n, 7))
    allowed = np.ones(n, dtype=bool)
    allowed[::7] = False
    want = graph_ref.self_knn(table, K, allowed, id_base=base)
    got = self_knn(shard, K, sf).cpu().numpy()
    assert np.array_equal(got, want)
    assert ((want - base) % 7 != 0).all()
    # the (K + 1)-th score ties with scores outside the list for most rows
    kth = np.array([np.sort(table[a, allowed])[::-1][K] for a in range(n)])
    assert ((table[:, allowed] == kth[:, None]).sum(1) > K + 1).mean() > 0.9


# ---- search ---------------------------------------------------------------------------------------------------------
def _table(shard, q, sf):
    """s(q, x) for every position: sgpt_rerank's bits, scored in blocks of at most 4096 candidates."""
    from sgpt_b200.ivfpq import rerank

    def block(ids):
        cand = torch.from_numpy(ids).cuda().repeat(q.shape[0], 1)
        s, i = rerank(shard, q, cand, len(ids), sf)
        return s.cpu().numpy(), i.cpu().numpy()

    return graph_ref.score_table(block, q.shape[0], shard.n, shard.id_base)


def _random_graph(n, degree, g, junk=True):
    """Uniform random edges int32 [n, degree].  With junk, the rows a search must step over: every 30th row all -1,
    every 30th (from 10) ids outside [0, n), every 30th (from 20) the row itself, and 2 % empty entries elsewhere."""
    graph = g.integers(0, n, (n, degree)).astype(np.int64)
    if junk:
        graph[g.random((n, degree)) < 0.02] = -1
        graph[0::30] = -1
        bad = np.array([n, n + 5, TOP - 1, -2, -1000])
        graph[10::30] = bad[g.integers(0, len(bad), graph[10::30].shape)]
        graph[20::30] = np.arange(20, n, 30)[:, None]
    return torch.from_numpy(graph.astype(np.int32))


def _launch(index, q, k, itopk, sw, iters, num_seeds=None, seeds=None, seed=0):
    """sgpt_graph_search with GraphIndex.search's arguments into outputs prefilled with NaN and SENTINEL; then
    GraphIndex.search must return the same bits.  Returns numpy (scores, ids, visited) of the first launch."""
    lib = _lib()
    shard = index.shard
    local = None
    if seeds is not None:
        s = seeds.to("cuda", torch.int64) - index.id_base
        local = torch.where((s >= 0) & (s < index.n), s, -1).to(torch.int32).contiguous()
        num_seeds = seeds.shape[1]
    qb, q_scale, c_scale = shard._queries(q, index.score_function)
    nq = qb.shape[0]
    mask, _ = shard._mask(None, nq)
    out_s = torch.full((nq, k), float("nan"), device="cuda")
    out_i = torch.full((nq, k), SENTINEL, dtype=torch.int64, device="cuda")
    out_v = torch.full((nq,), SENTINEL, dtype=torch.int32, device="cuda")
    rc = lib.lib().sgpt_graph_search(shard._dtype_id(), qb.data_ptr(), shard.vectors.data_ptr(), lib.ptr(q_scale),
                                     c_scale, nq, index.n, index.dim, index.id_base, index.graph.data_ptr(),
                                     index.degree, lib.ptr(local), num_seeds, seed, itopk, sw, iters, k, lib.ptr(mask),
                                     out_s.data_ptr(), out_i.data_ptr(), out_v.data_ptr(), lib.current_stream())
    lib.check(rc, "sgpt_graph_search")
    kw = dict(itopk=itopk, search_width=sw, max_iterations=iters, return_visited=True)
    if seeds is not None:
        kw.update(seeds=seeds)
    else:
        kw.update(num_seeds=num_seeds, seed=seed)
    s2, i2, v2 = index.search(q, k, **kw)
    assert torch.equal(out_i, i2) and torch.equal(out_s.view(torch.int32), s2.view(torch.int32))
    assert torch.equal(out_v, v2)
    return out_s.cpu().numpy(), out_i.cpu().numpy(), out_v.cpu().numpy()


def _check(index, q, table, k, itopk, sw, iters, num_seeds=None, seeds=None, seed=0, allowed=None, rows=None):
    """_launch, then every query of `rows` (default: all; table holds their rows) against graph_ref.search: ids, score
    bits and visited counts.  Returns the launch's (scores, ids, visited) and the restatement's."""
    s, i, v = _launch(index, q, k, itopk, sw, iters, num_seeds, seeds, seed)
    n, base = index.n, index.id_base
    if seeds is not None:
        kw = dict(seeds=seeds.cpu().numpy()[rows if rows is not None else slice(None)] - base)
        num_seeds = seeds.shape[1]
    elif rows is not None:  # the hash takes the query's row in the launch, not its row in the table
        kw = dict(seeds=np.array([[graph_ref.seed_hash(seed, int(r), j) % n for j in range(num_seeds)] for r in rows]))
    else:
        kw = dict(seed=seed)
    rows = np.arange(q.shape[0]) if rows is None else rows
    want = graph_ref.search(table, index.graph.cpu().numpy(), k, itopk, sw, iters, num_seeds, mask=allowed,
                            id_base=base, **kw)
    assert np.array_equal(i[rows], want[1])
    assert np.array_equal(s[rows].view(np.uint32), want[0].view(np.uint32))
    assert np.array_equal(v[rows], want[2])
    return (s, i, v), want


def _queries(x, nq, g):
    return x[torch.randint(x.shape[0], (nq,), generator=g)] + 0.5 * torch.randn(nq, x.shape[1], generator=g)


SEARCH_CASES = [
    # dtype, D, score function, degree (40: hand-built, else GraphIndex.build), search_width, itopk, k,
    # max_iterations, seeds ("hash" / "caller"), num_seeds, id_base
    ("bf16", 8, "dot", 16, 8, 512, 512, 20, "hash", 512, 0),
    ("bf16", 8, "cos_sim", 128, 4, 512, 1, 31, "caller", 512, 0),
    ("bf16", 24, "cos_sim", 40, 8, 480, 480, 30, "caller", 512, 0),
    ("bf16", 24, "dot", 64, 8, 512, 1, 31, "hash", 512, TOP - 3000),
    ("bf16", 776, "dot", 128, 4, 480, 100, 20, "hash", 64, 0),
    ("bf16", 776, "cos_sim", 16, 8, 64, 10, 100, "hash", 64, 0),
    ("int8", 16, "cos_sim", 64, 8, 480, 480, 31, "hash", 512, 0),
    ("int8", 16, "dot", 40, 8, 512, 512, 40, "hash", 300, 0),
    ("int8", 48, "cos_sim", 16, 8, 512, 1, 50, "caller", 512, 0),
    ("int8", 48, "dot", 128, 4, 512, 512, 31, "caller", 512, TOP - 3000),
    ("int8", 784, "cos_sim", 40, 8, 96, 20, 40, "hash", 128, 0),
    ("int8", 784, "dot", 64, 2, 480, 100, 100, "hash", 96, 0),
]


def _case_id(c):
    dtype, D, sf, degree, sw, itopk, k, iters, how, ns, base = c
    return (f"{dtype}-D{D}-{sf}-degree{degree}{'hand' if degree == 40 else ''}-sw{sw}-itopk{itopk}-k{k}-it{iters}-"
            f"{how}{ns}" + ("-top_ids" if base else ""))


@pytest.mark.parametrize("case", SEARCH_CASES, ids=[_case_id(c) for c in SEARCH_CASES])
def test_search_at_the_limits(case):
    from sgpt_b200 import GraphIndex

    dtype, D, sf, degree, sw, itopk, k, iters, how, ns, base = case
    assert 2 * (ns + iters * sw * degree) <= 32768 and sw * degree <= 512
    n = 3000
    g = torch.Generator().manual_seed(D + degree + sw)
    x = _rows(n, D, g)
    q = _queries(x, 24, g)
    shard = _shard(x, dtype, id_base=base)
    if degree == 40:
        index = GraphIndex(shard, _random_graph(n, degree, np.random.default_rng(D)), sf)
    else:
        index = GraphIndex.build(shard, degree=degree, intermediate_degree=min(256, 2 * degree), score_function=sf)
    seeds = torch.randint(-3, n + 3, (24, ns), generator=g) + base if how == "caller" else None
    (s, i, v), _ = _check(index, q, _table(shard, q, sf), k, itopk, sw, iters, num_seeds=ns, seeds=seeds, seed=D)
    assert (i >= base).all() and (i < base + n).all()  # n = 3000 rows fill every beam


@pytest.mark.parametrize("num_seeds,sw,degree,iters", [(512, 8, 64, 31), (64, 1, 32, 510)],
                         ids=["seeds512-sw8-degree64-it31", "seeds64-sw1-degree32-it510"])
def test_largest_visited_tables(num_seeds, sw, degree, iters):
    """2 (num_seeds + max_iterations search_width degree) = 32768 slots (128 KB of shared memory).  A random graph over
    200k rows makes nearly every candidate new, so the table really fills to about half."""
    from sgpt_b200 import GraphIndex

    bound = num_seeds + iters * sw * degree
    assert 2 * bound == 32768
    n = 200_003
    g = torch.Generator().manual_seed(degree)
    x = torch.randn(n, 64, generator=g)
    q = torch.randn(6, 64, generator=g)
    shard = _shard(x, "bf16")
    index = GraphIndex(shard, _random_graph(n, degree, np.random.default_rng(iters), junk=False), "dot")
    (_, _, v), _ = _check(index, q, _table(shard, q, "dot"), 100, 512, sw, iters, num_seeds=num_seeds, seed=9)
    assert (v <= bound).all() and (v > 0.9 * bound).all(), v


def test_thousands_of_queries_with_hashed_seeds():
    """3000 queries in one launch: the seed hash sees q > 2^11.  A stride of queries (and the rows around 2^11) against
    the restatement, every query for repeatability."""
    from sgpt_b200 import GraphIndex

    n = 5000
    g = torch.Generator().manual_seed(11)
    x = _rows(n, 64, g)
    q = _queries(x, 3000, g)
    shard = _shard(x, "bf16", id_base=17)
    index = GraphIndex.build(shard, degree=32, intermediate_degree=64)
    rows = np.unique(np.r_[0:3000:97, 2047, 2048, 2049, 2999])
    _check(index, q, _table(shard, q[torch.from_numpy(rows)], "cos_sim"), 10, 64, 2, 40, num_seeds=64,
           seed=0xDEADBEEF, rows=rows)


@pytest.mark.parametrize("n", [1, 7, 200])
def test_fewer_rows_than_itopk_and_seeds(n):
    """n < itopk = 256 < num_seeds = 512 hashed seeds: the seeds repeat, B keeps empty slots, the output ends in
    (-inf, -1), and every row is expanded long before max_iterations (the search stops early)."""
    from sgpt_b200 import GraphIndex

    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, 32, generator=g)
    q = torch.randn(5, 32, generator=g)
    shard = _shard(x, "bf16", id_base=5)
    index = GraphIndex(shard, _random_graph(n, 16, np.random.default_rng(n), junk=False), "cos_sim")
    (s, i, v), _ = _check(index, q, _table(shard, q, "cos_sim"), 256, 256, 1, 900, num_seeds=512, seed=3)
    assert (v == n).all()
    assert (i[:, :n] >= 5).all() and (i[:, n:] == -1).all() and (s[:, n:] == -np.inf).all()


def _awkward(kind, n, D, nq, g):
    """(rows, queries) fp32 on the host for the awkward-data searches."""
    if kind == "ties":  # integer rows from 6 distinct vectors: most scores tie
        basis = torch.randint(-3, 4, (6, D), generator=g).float()
        x = basis[torch.randint(6, (n,), generator=g)]
        return x, basis[torch.randint(6, (nq,), generator=g)] + torch.randint(-1, 2, (nq, D), generator=g).float()
    x = _rows(n, D, g)
    q = _queries(x, nq, g)
    if kind == "nan":  # whole NaN rows and rows with one NaN: score -1
        x[torch.randperm(n, generator=g)[:n // 10]] = float("nan")
        x[torch.randperm(n, generator=g)[:n // 20], 3] = float("nan")
    elif kind == "inf":  # one +inf or -inf entry: scores +-inf under dot
        r = torch.randperm(n, generator=g)[:n // 5]
        x[r, torch.randint(D, (len(r),), generator=g)] = torch.where(torch.rand(len(r), generator=g) < 0.5, 1.0,
                                                                     -1.0) * float("inf")
    elif kind == "zero":  # all-zero queries: every score 0
        q.zero_()
    return x, q


AWKWARD_CASES = [
    # kind, dtype, score function, n, itopk, k, search_width, max_iterations, built graph
    ("ties", "bf16", "dot", 2000, 128, 100, 4, 40, True),
    ("ties", "int8", "cos_sim", 2001, 64, 10, 8, 30, False),
    ("nan", "bf16", "cos_sim", 3001, 96, 50, 2, 40, False),
    ("nan", "int8", "dot", 3001, 64, 64, 4, 30, False),
    ("inf", "bf16", "dot", 100, 128, 128, 2, 60, False),
    ("inf", "bf16", "dot", 3001, 64, 64, 4, 30, False),
    ("zero", "bf16", "cos_sim", 3001, 64, 64, 4, 30, False),
    ("zero", "int8", "dot", 1001, 96, 30, 1, 100, False),
]


@pytest.mark.parametrize("case", AWKWARD_CASES, ids=[f"{c[0]}-{c[1]}-{c[2]}-n{c[3]}" for c in AWKWARD_CASES])
def test_search_on_awkward_data(case):
    from sgpt_b200 import GraphIndex

    kind, dtype, sf, n, itopk, k, sw, iters, built = case
    g = torch.Generator().manual_seed(n + itopk)
    x, q = _awkward(kind, n, 32, 16, g)
    shard = _shard(x, dtype, id_base=40)
    if built:
        index = GraphIndex.build(shard, degree=32, intermediate_degree=64, score_function=sf)
    else:
        index = GraphIndex(shard, _random_graph(n, 32, np.random.default_rng(n)), sf)
    table = _table(shard, q, sf)
    (s, i, v), (ws, wi, wv) = _check(index, q, table, k, itopk, sw, iters, num_seeds=64, seed=n)
    ok = i >= 0
    if kind == "ties":  # the k cut falls inside a run of equal scores for most queries
        kth = ws[:, -1]
        assert ((table == kth[:, None]).sum(1) > (ws == kth[:, None]).sum(1)).mean() > 0.5
    elif kind == "nan":
        assert (table == -1).sum() >= 16 * (n // 10)
    elif kind == "inf":
        assert np.isposinf(s).any() and (np.isneginf(s) & ok).any() == (n < itopk)
    elif kind == "zero":
        assert (s[ok].view(np.uint32) == 0).all() and ok.all()


def test_deletions_leave_fewer_than_k_allowed_in_the_beam():
    """All but every 41st row and the last row deleted, n = 3001 (not a multiple of 32): B holds fewer than k allowed
    rows, so every output ends in (-inf, -1).  Query 0 is the last row, which every query is seeded with, so the mask
    bit past the last full word is read."""
    from sgpt_b200 import GraphIndex

    n, base = 3001, 9
    g = torch.Generator().manual_seed(41)
    x = _rows(n, 64, g)
    q = _queries(x, 16, g)
    q[0] = x[n - 1]
    shard = _shard(x, "bf16", id_base=base)
    index = GraphIndex(shard, _random_graph(n, 32, np.random.default_rng(41)), "cos_sim")
    table = _table(shard, q, "cos_sim")
    allowed = np.zeros(n, dtype=bool)
    allowed[::41] = True
    allowed[n - 1] = True
    shard.remove(torch.from_numpy(np.nonzero(~allowed)[0] + base))
    seeds = torch.randint(0, n, (16, 64), generator=g) + base
    seeds[:, 0] = base + n - 1
    (s, i, v), _ = _check(index, q, table, 20, 64, 2, 40, seeds=seeds, allowed=allowed)
    got = i >= 0
    assert (got.sum(1) < 20).all() and i[0, 0] == base + n - 1
    assert (s[~got] == -np.inf).all()
