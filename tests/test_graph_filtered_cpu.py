"""CPU checks of the filtered graph search and of GraphIndex.add: every host-side rejection of
sgpt_graph_search_filtered and sgpt_graph_prune_append (before any CUDA call, dummy host pointers that are never
dereferenced) with their inclusive limits, the Python rejections of search(allow=) and add() before anything changes,
the pruned-list checks of GraphIndex.load (before any device allocation), and the numpy restatements on small cases."""
import json

import numpy as np
import pytest
import torch

from tests import graph_filtered_ref, graph_ref
from tests.test_graph_cpu import P, SEARCH, SEARCH_REJECTIONS, _Reached, _Shard, _case_id, _write_graph


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


# ---- sgpt_graph_search_filtered ---------------------------------------------------------------------------------------
def _filtered(mask=None, pitch=0, **kw):
    a = dict(SEARCH, **kw)
    return _lib().sgpt_graph_search_filtered(a["dtype"], a["Q"], a["C"], None, None, a["nq"], a["n"], a["D"],
                                             a["id_base"], a["graph"], a["degree"], None, a["num_seeds"], 0, a["itopk"],
                                             a["search_width"], a["max_iterations"], a["k"], mask, pitch, a["out_s"],
                                             a["out_i"], None, None)


MASK_REJECTIONS = [  # n = 1000: ceil(n / 32) = 32 words
    (dict(mask=P, pitch=-1), b"negative mask pitch -1"),
    (dict(mask=None, pitch=-4), b"negative mask pitch -4"),
    (dict(mask=P, pitch=1), b"mask pitch 1 words is below ceil(n / 32) = 32"),
    (dict(mask=P, pitch=31), b"mask pitch 31 words is below ceil(n / 32) = 32"),
    (dict(mask=None, pitch=32), b"mask pitch 32 without a mask"),
    (dict(mask=None, n=33, pitch=2), b"mask pitch 2 without a mask"),
]


@pytest.mark.parametrize("bad,msg", SEARCH_REJECTIONS + MASK_REJECTIONS,
                         ids=[_case_id(b) for b, _ in SEARCH_REJECTIONS + MASK_REJECTIONS])
def test_graph_search_filtered_rejects_bad_arguments(bad, msg):
    assert _filtered(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_graph_search_filtered:"), err


def test_graph_search_filtered_limits_are_inclusive():
    """The largest visited tables, the widest step, itopk = k = 512, and every legal mask form (none, shared, pitch of
    exactly ceil(n / 32) words and wider) pass the checks; nq = 0 returns before any CUDA call."""
    assert _filtered(nq=0, max_iterations=510) == 0, _lib().sgpt_last_error()
    assert _filtered(nq=0, search_width=8, degree=64, num_seeds=512, max_iterations=31) == 0, _lib().sgpt_last_error()
    assert _filtered(nq=0, itopk=512, k=512, num_seeds=512, max_iterations=1) == 0, _lib().sgpt_last_error()
    for mask, pitch in ((None, 0), (P, 0), (P, 32), (P, 33), (P, 1 << 40)):
        assert _filtered(nq=0, mask=mask, pitch=pitch) == 0, _lib().sgpt_last_error()
    assert _filtered(nq=0, n=33, mask=P, pitch=2) == 0, _lib().sgpt_last_error()


# ---- sgpt_graph_prune_append -------------------------------------------------------------------------------------------
APPEND = dict(graph=P, n_old=100, degree=32, knn=P, m=50, K=64, out=P)


def _append(**kw):
    a = dict(APPEND, **kw)
    return _lib().sgpt_graph_prune_append(a["graph"], a["n_old"], a["degree"], a["knn"], a["m"], a["K"], a["out"],
                                          None)


APPEND_REJECTIONS = [
    (dict(n_old=-1), b"n_old=-1 and m=50 must be non-negative"),
    (dict(m=-1), b"n_old=100 and m=-1 must be non-negative"),
    (dict(n_old=(1 << 31) - 50), b"with n_old + m < 2^31"),
    (dict(n_old=0, m=1 << 31), b"with n_old + m < 2^31"),
    (dict(degree=0), b"degree=0 must be a multiple of 16"),
    (dict(degree=24), b"degree=24 must be a multiple of 16"),
    (dict(degree=144, K=200), b"degree=144 must be a multiple of 16"),
    (dict(K=16), b"K=16 outside [degree=32, 256]"),
    (dict(K=257), b"K=257 outside [degree=32, 256]"),
    (dict(graph=None), b"null input graph with n_old=100"),
    (dict(knn=None), b"null input knn"),
    (dict(out=None), b"null output"),
]


@pytest.mark.parametrize("bad,msg", APPEND_REJECTIONS, ids=[_case_id(b) for b, _ in APPEND_REJECTIONS])
def test_graph_prune_append_rejects_bad_arguments(bad, msg):
    assert _append(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_graph_prune_append:"), err


def test_graph_prune_append_limits_are_inclusive():
    """m = 0 returns before any CUDA call, also with n_old + m = 2^31 - 1, degree 16 / 128 and K = degree / 256; a null
    graph is legal with n_old = 0."""
    assert _append(m=0, n_old=(1 << 31) - 1) == 0, _lib().sgpt_last_error()
    assert _append(m=0, degree=16, K=16) == 0, _lib().sgpt_last_error()
    assert _append(m=0, degree=128, K=256) == 0, _lib().sgpt_last_error()
    assert _append(m=0, n_old=0, graph=None) == 0, _lib().sgpt_last_error()


# ---- GraphIndex.search(allow=) and add(): Python rejections before anything changes ---------------------------------
class _FakeShard:
    """What search / add read of a shard before they reach the device; add() on it records the call."""
    dtype, dim, id_base, device = "bf16", 32, 100, torch.device("cpu")

    def __init__(self, n=40, capacity=50):
        self.n, self.capacity, self.added = n, capacity, []

    def add(self, emb):
        self.added.append(emb)


def _index(n=40, capacity=50, shard_n=None, pruned=True, id_base=100):
    from sgpt_b200 import GraphIndex

    shard = _FakeShard(n if shard_n is None else shard_n, capacity)
    shard.id_base = id_base
    index = GraphIndex.__new__(GraphIndex)  # no device graph needed for the checks
    index.shard, index.score_function = shard, "cos_sim"
    index.n, index.degree, index.dim, index.id_base, index.device = n, 16, 32, id_base, torch.device("cpu")
    index.pruned = torch.zeros((n, 16), dtype=torch.int32) if pruned else None
    index.intermediate_degree = 32 if pruned else None
    return index


@pytest.mark.parametrize("allow", [torch.ones(39, dtype=torch.bool), torch.ones(40, dtype=torch.int32),
                                   torch.ones(4, 40, dtype=torch.bool), torch.ones(3, 41, dtype=torch.bool),
                                   torch.ones(1, 3, 40, dtype=torch.bool)],
                         ids=["n-1", "int32", "Q+1 rows", "n+1 cols", "3-d"])
def test_search_rejects_bad_allow(allow):
    with pytest.raises(ValueError, match="allow must be a boolean tensor"):
        _index().search(torch.zeros(3, 32), 5, allow=allow)


def test_search_allow_on_an_out_of_sync_graph_raises():
    with pytest.raises(ValueError, match="built over 40"):
        _index(shard_n=41).search(torch.zeros(3, 32), 5, allow=torch.ones(40, dtype=torch.bool))


@pytest.mark.parametrize("case", ["shape_1d", "shape_dim", "ids", "capacity", "sync", "no_pruned", "no_pruned_m0"])
def test_add_rejects_before_the_shard_changes(case):
    emb = torch.zeros(5, 32)
    kw, msg = {}, None
    if case == "shape_1d":
        emb, msg = torch.zeros(32), "embeddings must be"
    elif case == "shape_dim":
        emb, msg = torch.zeros(5, 31), "embeddings must be"
    elif case == "ids":
        kw, msg = dict(id_base=(1 << 31) - 44, capacity=100), "must fit in int32"
    elif case == "capacity":
        emb, msg = torch.zeros(11, 32), r"capacity 50 exceeded \(40 \+ 11\)"
    elif case == "sync":
        kw, msg = dict(shard_n=41), "built over 40"
    elif case == "no_pruned":
        kw, msg = dict(pruned=False), "no pruned lists"
    else:
        emb, kw, msg = torch.zeros(0, 32), dict(pruned=False), "no pruned lists"
    index = _index(**kw)
    with pytest.raises(ValueError, match=msg):
        index.add(emb)
    assert index.shard.added == [] and index.n == 40


def test_add_limits_are_inclusive():
    """Exactly filling the capacity and the int32 id range passes the checks (m = 0 stops there; m > 0 reaches
    shard.add)."""
    _index(capacity=45, id_base=(1 << 31) - 46).add(torch.zeros(0, 32))

    class _Stop(Exception):
        pass

    index = _index(capacity=45, id_base=(1 << 31) - 46)

    def stop(emb):
        raise _Stop()

    index.shard.add = stop
    with pytest.raises(_Stop):
        index.add(torch.zeros(5, 32))


# ---- GraphIndex.load of pruned lists -----------------------------------------------------------------------------------
def _write_pruned(path, pruned=None, K=32, **meta_over):
    _write_graph(path, **meta_over)
    meta = json.loads((path / "meta.json").read_text())
    meta.update(pruned="pruned.npy", intermediate_degree=K)
    (path / "meta.json").write_text(json.dumps(meta))
    np.save(path / "pruned.npy", np.tile(np.arange(16, dtype=np.int32), (40, 1)) if pruned is None else pruned)


BAD_PRUNED = {
    "shape": (dict(pruned=np.zeros((40, 32), np.int32)), "pruned lists .* do not match meta"),
    "rows": (dict(pruned=np.zeros((39, 16), np.int32)), "pruned lists .* do not match meta"),
    "dtype": (dict(pruned=np.zeros((40, 16), np.int64)), "pruned lists .* do not match meta"),
    "entry_below": (dict(pruned=np.full((40, 16), -2, np.int32)), r"pruned entries must lie in \[-1, n=40\)"),
    "entry_above": (dict(pruned=np.full((40, 16), 40, np.int32)), r"pruned entries must lie in \[-1, n=40\)"),
    "K_below": (dict(K=15), r"intermediate_degree=15 outside \[degree=16, 256\]"),
    "K_above": (dict(K=257), r"intermediate_degree=257 outside \[degree=16, 256\]"),
}


@pytest.mark.parametrize("name", sorted(BAD_PRUNED))
def test_graph_load_rejects_bad_pruned_lists_before_allocating(tmp_path, monkeypatch, name):
    from sgpt_b200 import GraphIndex

    def no_alloc(*a, **k):
        raise AssertionError("the index was constructed before the files were checked")

    kw, msg = BAD_PRUNED[name]
    _write_pruned(tmp_path / name, **kw)
    monkeypatch.setattr(GraphIndex, "__init__", no_alloc)
    monkeypatch.setattr(torch, "empty", no_alloc)
    monkeypatch.setattr(torch, "zeros", no_alloc)
    with pytest.raises(ValueError, match=msg):
        GraphIndex.load(str(tmp_path / name), _Shard())


@pytest.mark.parametrize("K", [16, 256])
def test_graph_load_keeps_consistent_pruned_lists(tmp_path, monkeypatch, K):
    """With pruned lists the index is still made by cls(shard, graph, score_function), and then holds them."""
    from sgpt_b200 import GraphIndex

    def init(self, shard, graph, score_function):
        self.graph = graph

    want = np.tile(np.arange(-1, 15, dtype=np.int32), (40, 1))
    _write_pruned(tmp_path / "ok", pruned=want, K=K)
    monkeypatch.setattr(GraphIndex, "__init__", init)
    index = GraphIndex.load(str(tmp_path / "ok"), _Shard())
    assert index.intermediate_degree == K and np.array_equal(index.pruned.numpy(), want)
    assert index.pruned.dtype == torch.int32 and index.pruned.device.type == "cpu"


def test_graph_load_without_pruned_lists_is_unchanged(tmp_path, monkeypatch):
    from sgpt_b200 import GraphIndex

    def stop(self, shard, graph, score_function):
        raise _Reached()

    _write_graph(tmp_path / "old")
    monkeypatch.setattr(GraphIndex, "__init__", stop)
    with pytest.raises(_Reached):
        GraphIndex.load(str(tmp_path / "old"), _Shard())


# ---- the restatements ------------------------------------------------------------------------------------------------
def test_restated_prune_append_of_no_old_rows_is_prune():
    g = np.random.default_rng(5)
    n, K = 120, 32
    knn = np.stack([g.permutation(n)[:K] for _ in range(n)]).astype(np.int64)
    knn[g.random((n, K)) < 0.05] = -1
    knn[g.random((n, K)) < 0.05] = n + 3
    knn[::7, 3] = np.arange(0, n, 7)
    for degree in (16, 32):
        assert np.array_equal(graph_filtered_ref.prune_append(None, knn, degree), graph_ref.prune(knn, degree))


def test_restated_prune_append_on_a_hand_worked_case():
    # old rows 0..3 with graph rows of degree 2; new rows 4 and 5 (n = 6).
    graph = np.array([[1, 2], [2, 3], [3, 0], [0, -1]], np.int32)
    # row 4: L = [1, 2, 3, 4, 9]: 4 is the row itself and 9 lies outside [0, 6): both empty.
    #   d(2) = 1 (graph[1] holds 2 at 0 < 1); d(3) = 2 (graph[1] holds 3 at 1 < 2, graph[2] at 0 < 2); d(1) = 0
    # row 5: L = [4, 0, 4, 1]: the second 4 repeats the first.  list(4) = knn row of 4 = [1, 2, 3, 4, 9]:
    #   d(0) = 0 (4's list holds no 0); d(1) = 2 (4's list holds 1 at 0 < 3, and so does 0's graph row)
    knn = np.array([[1, 2, 3, 4, 9], [4, 0, 4, 1, -1]], np.int64)
    got = graph_filtered_ref.prune_append(graph, knn, 4)
    assert got[0].tolist() == [1, 2, 3, -1]
    assert got[1].tolist() == [4, 0, 1, -1]
    assert graph_filtered_ref.prune_append(graph, knn, 2)[0].tolist() == [1, 2]


def test_restated_filtered_search_walks_as_the_unfiltered_one():
    g = np.random.default_rng(6)
    nq, n = 4, 200
    table = g.standard_normal((nq, n)).astype(np.float32)
    graph = g.integers(-1, n, (n, 8)).astype(np.int32)
    # |V| <= 5 + 6 x 2 x 8 = 101 <= itopk: B keeps all of V, and the unfiltered top-128 lists V in key order
    kw = dict(k=10, itopk=128, search_width=2, max_iterations=6, num_seeds=5, seed=3, id_base=50)
    s, i, v = graph_ref.search(table, graph, **kw)
    fs, fi, fv = graph_filtered_ref.search_filtered(table, graph, **kw)
    assert np.array_equal(v, fv) and np.array_equal(i, fi) and np.array_equal(s.view(np.uint32), fs.view(np.uint32))
    for mask in (np.ones(n, bool), np.ones((nq, n), bool)):
        ms, mi, mv = graph_filtered_ref.search_filtered(table, graph, mask=mask, **kw)
        assert np.array_equal(mi, i) and np.array_equal(mv, v)
    # a per-query mask allowing only odd positions for query 0 and nothing for query 1
    mask = np.ones((nq, n), bool)
    mask[0, ::2] = False
    mask[1] = False
    ms, mi, mv = graph_filtered_ref.search_filtered(table, graph, mask=mask, **kw)
    assert np.array_equal(mv, v) and (mi[1] == -1).all() and np.isneginf(ms[1]).all()
    V = graph_ref.search(table, graph, **dict(kw, k=128))[1][0]
    V = V[V >= 0] - 50
    assert len(V) == v[0]
    odd = V[V % 2 == 1][:10]
    assert np.array_equal(mi[0][:len(odd)] - 50, odd) and (mi[0][len(odd):] == -1).all()
