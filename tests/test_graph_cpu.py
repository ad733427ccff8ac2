"""CPU checks of the graph index: every host-side rejection of sgpt_graph_prune and sgpt_graph_search (before any CUDA
call, dummy host pointers that are never dereferenced), the file checks of GraphIndex.load (before any device
allocation), and the numpy restatement (tests/graph_ref.py) on cases whose answer is known."""
import json

import numpy as np
import pytest
import torch

from tests import graph_ref

HOST = np.zeros(4096, dtype=np.int64)
P = (HOST.ctypes.data + 15) & ~15  # dummy 16-byte aligned host pointer, never dereferenced
PTR_ARGS = {"knn", "out", "Q", "C", "graph", "out_s", "out_i"}


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


def _case_id(bad):
    return ",".join(f"{k}=P+{v - P}" if k in PTR_ARGS and v is not None else f"{k}={v}" for k, v in bad.items())


# ---- sgpt_graph_prune -------------------------------------------------------------------------------------------------
PRUNE = dict(knn=P, n=100, K=64, degree=32, out=P)


def _prune(**kw):
    a = dict(PRUNE, **kw)
    return _lib().sgpt_graph_prune(a["knn"], a["n"], a["K"], a["degree"], a["out"], None)


PRUNE_REJECTIONS = [
    (dict(n=-1), b"n=-1 outside"),
    (dict(n=1 << 31), b"n=2147483648 outside"),
    (dict(degree=0), b"degree=0 must be a multiple of 16"),
    (dict(degree=24), b"degree=24 must be a multiple of 16"),
    (dict(degree=144, K=200), b"degree=144 must be a multiple of 16"),
    (dict(K=16), b"K=16 outside [degree=32, 256]"),
    (dict(K=257), b"K=257 outside [degree=32, 256]"),
    (dict(knn=None), b"null input"),
    (dict(out=None), b"null output"),
]


@pytest.mark.parametrize("bad,msg", PRUNE_REJECTIONS, ids=[_case_id(b) for b, _ in PRUNE_REJECTIONS])
def test_graph_prune_rejects_bad_arguments(bad, msg):
    assert _prune(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_graph_prune"), err


def test_graph_prune_legal_empty_call_passes():
    assert _prune(n=0) == 0, _lib().sgpt_last_error()


# ---- sgpt_graph_search ------------------------------------------------------------------------------------------------
SEARCH = dict(dtype=0, Q=P, C=P, nq=3, n=1000, D=64, id_base=0, graph=P, degree=32, num_seeds=64, itopk=64,
              search_width=1, max_iterations=100, k=10, out_s=P, out_i=P)


def _search(**kw):
    a = dict(SEARCH, **kw)
    return _lib().sgpt_graph_search(a["dtype"], a["Q"], a["C"], None, None, a["nq"], a["n"], a["D"], a["id_base"],
                                    a["graph"], a["degree"], None, a["num_seeds"], 0, a["itopk"], a["search_width"],
                                    a["max_iterations"], a["k"], None, a["out_s"], a["out_i"], None, None)


SEARCH_REJECTIONS = [
    (dict(dtype=3), b"must be bf16 (0) or int8 (1)"),
    (dict(dtype=2), b"must be bf16 (0) or int8 (1)"),
    (dict(nq=-1), b"bad query count"),
    (dict(D=60), b"positive multiple of 8"),
    (dict(D=0), b"positive multiple of 8"),
    (dict(dtype=1, D=72), b"positive multiple of 16"),
    (dict(dtype=1, D=65552), b"at most 65536"),
    (dict(n=0), b"corpus size n=0 outside [1, 2^31)"),
    (dict(n=1 << 31), b"corpus size n=2147483648"),
    (dict(id_base=-1), b"must fit in int32"),
    (dict(id_base=(1 << 31) - 999), b"must fit in int32"),
    (dict(itopk=16, k=10), b"itopk=16 must be a multiple of 32"),
    (dict(itopk=48), b"itopk=48 must be a multiple of 32"),
    (dict(itopk=544), b"itopk=544 must be a multiple of 32"),
    (dict(k=0), b"k=0 outside [1, itopk=64]"),
    (dict(k=65), b"k=65 outside [1, itopk=64]"),
    (dict(degree=0), b"degree=0 must be positive"),
    (dict(search_width=0), b"search_width=0 outside [1, 8]"),
    (dict(search_width=9), b"search_width=9 outside [1, 8]"),
    (dict(search_width=8, degree=65, max_iterations=1), b"exceeds 512 candidates per step"),
    (dict(num_seeds=0), b"num_seeds=0 outside [1, 512]"),
    (dict(num_seeds=513), b"num_seeds=513 outside [1, 512]"),
    (dict(max_iterations=0), b"max_iterations=0 must be positive"),
    (dict(max_iterations=511), b"exceeds 32768"),
    (dict(num_seeds=512, degree=64, search_width=8, max_iterations=32), b"exceeds 32768"),
    (dict(Q=None), b"null input"),
    (dict(C=None), b"null input"),
    (dict(graph=None), b"null input"),
    (dict(Q=P + 8), b"16-byte aligned"),
    (dict(C=P + 2), b"16-byte aligned"),
    (dict(out_s=None), b"null output"),
    (dict(out_i=None), b"null output"),
]


@pytest.mark.parametrize("bad,msg", SEARCH_REJECTIONS, ids=[_case_id(b) for b, _ in SEARCH_REJECTIONS])
def test_graph_search_rejects_bad_arguments(bad, msg):
    assert _search(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_graph_search"), err


def test_graph_search_limits_are_inclusive():
    """The largest legal visited tables (2 (64 + 510 x 32) = 32768 and 2 (512 + 31 x 8 x 64) = 32768 slots), the widest
    step and the largest itopk pass the checks; nq = 0 returns before any CUDA call."""
    assert _search(nq=0, max_iterations=510) == 0, _lib().sgpt_last_error()
    assert _search(nq=0, search_width=8, degree=64, num_seeds=512, max_iterations=31) == 0, _lib().sgpt_last_error()
    assert _search(nq=0, itopk=512, k=512, num_seeds=512, max_iterations=1) == 0, _lib().sgpt_last_error()


# ---- GraphIndex.load ----------------------------------------------------------------------------------------------
class _Shard:
    """What load reads of a shard (no device memory)."""
    n, dim, dtype, id_base = 40, 32, "bf16", 100


def _write_graph(path, graph=None, **meta_over):
    path.mkdir()
    meta = {"format": "sgpt_b200.GraphIndex/1", "n": 40, "degree": 16, "dim": 32, "dtype": "bf16", "id_base": 100,
            "score_function": "cos_sim"}
    meta.update(meta_over)
    (path / "meta.json").write_text(json.dumps(meta))
    g = np.tile(np.arange(16, dtype=np.int32), (40, 1)) if graph is None else graph
    np.save(path / "graph.npy", g)


BAD_GRAPHS = {
    "format": (dict(format="sgpt_b200.IVFIndex/1"), "not a GraphIndex"),
    "score_function": (dict(score_function="l2"), "score function"),
    "n": (dict(n=41), "was built over"),
    "dim": (dict(dim=64), "was built over"),
    "dtype": (dict(dtype="int8"), "was built over"),
    "id_base": (dict(id_base=0), "was built over"),
    "degree": (dict(degree=32), "does not match meta"),
    "graph_shape": (dict(graph=np.zeros((39, 16), np.int32)), "does not match meta"),
    "graph_dtype": (dict(graph=np.zeros((40, 16), np.int64)), "does not match meta"),
    "entry_below": (dict(graph=np.full((40, 16), -2, np.int32)), r"\[-1, n=40\)"),
    "entry_above": (dict(graph=np.full((40, 16), 40, np.int32)), r"\[-1, n=40\)"),
}


@pytest.mark.parametrize("name", sorted(BAD_GRAPHS))
def test_graph_load_rejects_bad_files_before_allocating(tmp_path, monkeypatch, name):
    from sgpt_b200 import GraphIndex

    def no_alloc(*a, **k):
        raise AssertionError("the index was constructed before the files were checked")

    kw, msg = BAD_GRAPHS[name]
    kw = dict(kw)
    _write_graph(tmp_path / name, kw.pop("graph", None), **kw)
    monkeypatch.setattr(GraphIndex, "__init__", no_alloc)
    monkeypatch.setattr(torch, "empty", no_alloc)
    monkeypatch.setattr(torch, "zeros", no_alloc)
    with pytest.raises(ValueError, match=msg):
        GraphIndex.load(str(tmp_path / name), _Shard())


class _Reached(Exception):
    pass


def test_graph_load_reaches_the_device_only_with_consistent_files(tmp_path, monkeypatch):
    from sgpt_b200 import GraphIndex

    def stop(self, shard, graph, score_function):
        assert graph.dtype == torch.int32 and tuple(graph.shape) == (40, 16) and score_function == "cos_sim"
        raise _Reached()

    _write_graph(tmp_path / "ok")
    monkeypatch.setattr(GraphIndex, "__init__", stop)
    with pytest.raises(_Reached):
        GraphIndex.load(str(tmp_path / "ok"), _Shard())


def test_graph_build_rejects_bad_degrees():
    from sgpt_b200.graph import _check_degree

    for degree, K in ((24, 64), (0, 64), (144, 200), (32, 16), (32, 257)):
        with pytest.raises(ValueError):
            _check_degree(degree, K)


# ---- the restatement ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seeds", [False, True])
def test_restated_search_on_a_complete_graph_is_the_exact_top_k(seeds):
    """With every position linked to every other and itopk >= n, one expansion visits everything: the output is the
    exact top-k (score descending, ties by ascending id), repeated scores included."""
    g = np.random.default_rng(1)
    nq, n, k = 5, 60, 20
    table = g.integers(-6, 7, (nq, n)).astype(np.float32)  # many ties
    table[:, 7] = -0.0
    graph = np.array([[y for y in range(n) if y != x] for x in range(n)], dtype=np.int32)
    sd = g.integers(0, n, (nq, 3)) if seeds else None
    s, i, v = graph_ref.search(table, graph, k, itopk=64, search_width=1, max_iterations=2, num_seeds=3, seeds=sd,
                               id_base=1000)
    for q in range(nq):
        order = np.lexsort((np.arange(n), -table[q].astype(np.float64)))[:k]
        assert np.array_equal(i[q], order + 1000)
        assert np.array_equal(s[q], table[q, order] + np.float32(0))
    assert (v == n).all()


def test_restated_search_mask_and_tail():
    g = np.random.default_rng(2)
    n = 40
    table = g.standard_normal((2, n)).astype(np.float32)
    graph = np.array([[y for y in range(n) if y != x] for x in range(n)], dtype=np.int32)
    mask = np.zeros(n, dtype=bool)
    mask[::5] = True
    s, i, _ = graph_ref.search(table, graph, 12, itopk=64, search_width=2, max_iterations=3, num_seeds=1, mask=mask)
    assert (i[:, :8] % 5 == 0).all() and (i[:, 8:] == -1).all() and np.isinf(s[:, 8:]).all()


def test_restated_prune_and_merge_on_a_hand_worked_case():
    # row 0: [1, 2, 3]; row 1 lists 2 first, so 2 is a detour of 1 for row 0 (d = 1); 3 is in row 1 at position 1 < 2
    # and in row 2 at position 0 < 2 (d = 2).  Row 3 repeats 0 and lists itself: both are empty.
    knn = np.array([[1, 2, 3], [2, 3, 0], [3, 0, 1], [0, 3, 0], ], dtype=np.int64)
    pruned = graph_ref.prune(knn, 3)
    assert pruned[0].tolist() == [1, 2, 3]
    d = {a: pruned[a].tolist() for a in range(4)}
    assert d[3] == [0, -1, -1]
    knn = np.array([[1, 2, 3, 4], [2, 4, 0, 5], [4, 5, 0, 1], [5, 0, 1, 2], [0, 1, 2, 3], [0, 1, 2, 9]], np.int64)
    # row 0: d(1) = 0; d(2) = 1 (row 1 holds 2 at 0 < 1); d(3) = 0 (rows 1 and 2 hold no 3 before position 2);
    # d(4) = 2 (rows 1 and 2 hold 4 before position 3, row 3 does not)
    assert graph_ref.prune(knn, 4)[0].tolist() == [1, 3, 2, 4]
    assert graph_ref.prune(knn, 3)[0].tolist() == [1, 3, 2]
    assert graph_ref.prune(knn, 4)[5].tolist() == [0, 1, 2, -1]
    merged = graph_ref.merge(np.array([[1, 2, -1, -1], [0, 2, 3, -1], [0, 1, -1, -1], [2, 1, 0, -1]], np.int32))
    # F = first 2; R[0] = {1 (rank 0), 2 (rank 0)} -> [1, 2]; R[2] = {0 (rank 1), 1 (rank 1), 3 (rank 0)} -> [3, 0]
    assert merged[0].tolist() == [1, 2, -1, -1]
    assert merged[2].tolist() == [0, 1, 3, -1]
    assert merged[3].tolist() == [2, 1, 0, -1]


def test_seed_hash_is_32_bit():
    vals = {graph_ref.seed_hash(s, q, j) for s in (0, 7) for q in range(20) for j in range(50)}
    assert len(vals) == 2000 and max(vals) < 2 ** 32


def test_restated_self_knn_ties_own_id_and_deletions():
    # rows 0-4 are copies of one vector (all score 3 against each other), row 5 is another (score 1 against the copies,
    # 5 against itself); position 2 is deleted
    t = np.array([[3, 3, 3, 3, 3, 1]] * 5 + [[1, 1, 1, 1, 1, 5]], dtype=np.float32)
    t[0, 5] = -0.0  # -0 ties with +0, broken by position
    allowed = np.array([True, True, False, True, True, True])
    got = graph_ref.self_knn(t, 2, allowed, id_base=100)
    # top-3 of row 0 over {0, 1, 3, 4, 5}: 0, 1, 3 -> own id 0 removed
    assert got[0].tolist() == [101, 103]
    # row 2 is deleted, so it is absent from its own top-3 {0, 1, 3}: the last entry is dropped
    assert got[2].tolist() == [100, 101]
    # row 5: its own id first, then the copies by position
    assert got[5].tolist() == [100, 101]
    full = graph_ref.self_knn(t, 4, None)
    assert full[4].tolist() == [0, 1, 2, 3]  # the row is the 5th of its ties: removed from the top-5
    few = graph_ref.self_knn(t, 5, np.array([True, False, False, False, False, True]))
    assert few[0].tolist() == [5, -1, -1, -1, -1]  # fewer than K + 1 allowed: tail -1


def test_score_table_from_blocks_of_top_k():
    g = np.random.default_rng(3)
    nq, n, base = 3, 30, 50
    want = g.integers(-3, 4, (nq, n)).astype(np.float32)
    want[1, 4] = np.nan
    want[2, 9] = -np.inf

    def top_m(ids, shift=0):
        s = want[:, ids - base]
        order = np.lexsort((np.broadcast_to(ids, s.shape), -np.nan_to_num(s, nan=-1)), axis=-1)
        return np.take_along_axis(s, order, 1), ids[order] + shift

    got = graph_ref.score_table(top_m, nq, n, id_base=base, block=7)
    assert np.array_equal(got, np.where(np.isnan(want), np.float32(-1), want))
    with pytest.raises(AssertionError, match="outside"):
        graph_ref.score_table(lambda ids: top_m(ids, 1), nq, n, id_base=base, block=7)
    with pytest.raises(AssertionError, match="more or less than once"):
        graph_ref.score_table(lambda ids: (want[:, ids - base], np.broadcast_to(ids[:1], (nq, len(ids)))), nq, n,
                              id_base=base, block=7)
