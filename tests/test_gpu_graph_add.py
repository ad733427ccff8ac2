"""GPU tests of GraphIndex.add: sgpt_graph_prune_append against the numpy restatement
(tests/graph_filtered_ref.prune_append), the graph after one and two adds against graph_ref.merge of the old pruned
lists and the restated appended ones, bit for bit, m = 0, save / load / add, and recall of queries near the added rows
next to a rebuild."""
import numpy as np
import pytest
import torch

from tests import graph_filtered_ref, graph_ref
from tests.test_gpu_graph import _overlapping_lists, _shard

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n_old,m,K,degree", [(0, 500, 64, 32), (600, 300, 64, 16), (700, 40, 128, 64),
                                              (600, 200, 256, 128)])
def test_prune_append_equals_the_restatement(n_old, m, K, degree):
    from sgpt_b200.graph import prune, prune_append

    g = np.random.default_rng(n_old + m + K)
    knn = _overlapping_lists(n_old + m, K, g)
    graph = graph_ref.prune(knn[:n_old], degree) if n_old else np.zeros((0, degree), np.int32)
    graph[g.random(graph.shape) < 0.05] = -1
    new = knn[n_old:]
    got = prune_append(torch.from_numpy(graph).cuda(), torch.from_numpy(new).cuda(), degree).cpu().numpy()
    assert np.array_equal(got, graph_filtered_ref.prune_append(graph if n_old else None, new, degree))
    if n_old == 0:
        assert np.array_equal(got, prune(torch.from_numpy(new).cuda(), degree).cpu().numpy())


def _restated_add(index, before_graph, before_pruned, n, m):
    """The graph and pruned lists an add of rows n .. n + m - 1 must give, from the index's k-NN lists of those rows."""
    from sgpt_b200.graph import self_knn

    K = index.intermediate_degree
    knn = self_knn(index.shard, K, index.score_function, rows=torch.arange(n, n + m, device="cuda"))
    own = torch.arange(n, n + m, device="cuda")[:, None] + index.id_base
    assert not (knn == own).any()
    assert torch.equal(knn, self_knn(index.shard, K, index.score_function)[n:])
    local = (knn - index.id_base).cpu().numpy()
    local[local < 0] = -1
    pruned = np.concatenate([before_pruned, graph_filtered_ref.prune_append(before_graph, local, index.degree)])
    return graph_ref.merge(pruned), pruned


@pytest.mark.parametrize("dtype,sf,id_base", [("bf16", "cos_sim", 0), ("int8", "dot", 1234)])
def test_add_equals_restated_prune_append_and_merge(dtype, sf, id_base):
    from sgpt_b200 import GraphIndex

    n0, m1, m2 = 1500, 250, 120
    shard, _ = _shard(n0, 64, dtype, 5, id_base=id_base, capacity=n0 + m1 + m2)
    index = GraphIndex.build(shard, degree=32, intermediate_degree=64, score_function=sf)
    shard.remove(torch.arange(0, n0, 11) + id_base)  # deleted documents are nobody's new neighbour
    g = torch.Generator().manual_seed(6)
    for m in (m1, m2):
        n = index.n
        before_graph, before_pruned = index.graph.cpu().numpy(), index.pruned.numpy()
        x = torch.randn(m, 16, generator=g) @ torch.randn(16, 64, generator=g) + 0.3 * torch.randn(m, 64, generator=g)
        index.add(x.cuda())
        assert index.n == shard.n == n + m
        want_graph, want_pruned = _restated_add(index, before_graph, before_pruned, n, m)
        assert np.array_equal(index.pruned.numpy(), want_pruned)
        assert np.array_equal(index.graph.cpu().numpy(), want_graph)
        assert index.nbytes == 4 * (n + m) * 32 and index.pruned.device.type == "cpu"
        assert np.array_equal(index.pruned.numpy()[:n], before_pruned)  # the old forward lists are never revised
        assert torch.equal(index.graph, torch.from_numpy(graph_ref.merge(index.pruned.numpy())).cuda())
    s, i = index.search(torch.randn(8, 64).cuda(), 10)
    assert (i >= 0).all()


def test_add_of_nothing_changes_nothing():
    from sgpt_b200 import GraphIndex

    shard, q = _shard(800, 64, "bf16", 7, capacity=900)
    index = GraphIndex.build(shard, degree=16, intermediate_degree=32)
    graph, pruned = index.graph.clone(), index.pruned.clone()
    index.add(torch.empty(0, 64).cuda())
    assert index.n == shard.n == 800
    assert torch.equal(index.graph, graph) and torch.equal(index.pruned, pruned)


def test_save_load_add_search_matches_the_index_in_memory(tmp_path):
    from sgpt_b200 import CorpusShard, GraphIndex

    shard, q = _shard(1200, 64, "int8", 8, id_base=40, capacity=1400)
    index = GraphIndex.build(shard, degree=16, intermediate_degree=48, score_function="cos_sim")
    index.save(str(tmp_path / "g"))
    shard.save(str(tmp_path / "s"))
    shard2 = CorpusShard.load(str(tmp_path / "s"), capacity=1400)
    back = GraphIndex.load(str(tmp_path / "g"), shard2)
    assert back.intermediate_degree == 48 and torch.equal(back.pruned, index.pruned)
    x = torch.randn(150, 64, generator=torch.Generator().manual_seed(9)).cuda()
    index.add(x)
    back.add(x)
    assert torch.equal(back.graph, index.graph) and torch.equal(back.pruned, index.pruned)
    a = index.search(q, 10, return_visited=True)
    b = back.search(q, 10, return_visited=True)
    assert all(torch.equal(u.view(torch.int32) if u.dtype == torch.float32 else u,
                           w.view(torch.int32) if w.dtype == torch.float32 else w) for u, w in zip(a, b))


def test_recall_of_added_rows_next_to_a_rebuild():
    """The 100 k low-dimensional rows of test_gpu_graph.test_recall_on_low_intrinsic_dimension_rows: build on the first
    90 k and add the last 10 k, or build on all 100 k; 200 queries drawn near the added rows, itopk 128, recall@10 against
    the exact search must be >= 0.98 for the grown graph (measured: 1.0000 for both graphs on an H100 SXM)."""
    from sgpt_b200 import CorpusShard, GraphIndex

    g = torch.Generator(device="cuda").manual_seed(0)
    G = torch.randn(768, 16, generator=g, device="cuda")
    x = torch.randn(100_000, 16, generator=g, device="cuda") @ G.T
    x += 0.1 * torch.randn(x.shape, generator=g, device="cuda")
    q = x[90_000 + torch.randint(10_000, (200,), generator=g, device="cuda")]
    q = q + 0.1 * torch.randn(q.shape, generator=g, device="cuda")
    shard = CorpusShard(768, 100_000)
    shard.add(x[:90_000])
    grown = GraphIndex.build(shard)
    grown.add(x[90_000:])
    full = GraphIndex.build(CorpusShard.from_embeddings(x))
    _, exact = shard.search(q, 10)
    recall = {}
    for name, index in (("add", grown), ("build", full)):
        _, got = index.search(q, 10, itopk=128)
        recall[name] = sum(len(set(a) & set(b)) for a, b in zip(got.tolist(), exact.tolist())) / exact.numel()
    print(f"recall@10 near the added rows: build 90k + add 10k {recall['add']:.4f}, build 100k {recall['build']:.4f}")
    assert recall["add"] >= 0.98
