"""CPU-only checks of the host side: the C-ABI library loads and exports every symbol include/sgpt_b200.h declares,
ragged packing, reference token rules, error behaviour, shard ranges, and the 2-rank gloo path of the sharded search."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "sgpt_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sgpt_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from sgpt_b200 import _lib

    assert os.path.exists(_lib.LIB_PATH), "build the library first: python -c 'import __graft_entry__ as g; g.build()'"
    declared = _header_functions()
    assert len(declared) >= 18
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(handle, name), f"{name} declared in include/sgpt_b200.h but not exported"
    assert sorted(_lib.exported_symbols()) == declared, "ctypes signature table out of sync with the header"
    lib = _lib.lib()
    assert lib.sgpt_abi_version() == _lib.ABI_VERSION == 3
    # argument validation happens before any CUDA call, so it is checkable without a GPU
    assert lib.sgpt_linear(None, 8, None, 8, None, None, 8, None, 4, 4, 7, 0, None) == 1  # K % 8 != 0
    assert b"multiples of 8" in lib.sgpt_last_error()
    assert lib.sgpt_topk(None, 4, 1, 8, 3, 0, None, None, None, None) == 1  # lds < n


def test_search_workspace_plan_is_consistent_across_query_blocks():
    """Host logic of the fused search (csrc/search.cu make_plan / sgpt_search_workspace_bytes; no GPU needed — the SM count
    falls back to the H100's 132): batches above 256 queries are processed in blocks that REUSE one workspace, whose last block may be
    small enough for the single-CTA plan with its different list layout, so the size for nq queries must cover every block
    size that can occur; small shards take the dense path (nq x n fp32 scores)."""
    from sgpt_b200 import _lib

    ws = _lib.lib().sgpt_search_workspace_bytes
    n, k = 1_000_000, 1001
    for nq in (129, 200, 256, 300, 1000, 5000):
        need = ws(nq, n, k)
        blocks = {min(256, nq)} | ({nq % 256} if nq > 256 and nq % 256 else set())
        for nb in blocks:
            assert need >= ws(nb, n, k), (nq, nb)
    assert ws(128, n, k) >= ws(7, n, k) > 0
    # two-pass lists are worst-case sized: ~8 bytes per (query, document)
    assert 0.9 < ws(128, n, k) / (128 * n * 8) < 1.2
    # below two corpus tiles per SM (67 584 documents at 132 SMs): dense scores, 4 bytes per (query, document)
    assert ws(16, 50_000, k) == 16 * 50_000 * 4 + 256
    assert ws(16, 80_000, k) > 16 * 80_000 * 4 + 256


def test_missing_library_fails_loudly(monkeypatch):
    from sgpt_b200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libsgpt_b200.so")
    with pytest.raises(RuntimeError, match="no CPU or PyTorch fallback"):
        _lib.lib()


def test_encoder_refuses_cpu_device():
    from sgpt_b200 import ModelConfig
    from sgpt_b200.encoder import Encoder

    with pytest.raises(RuntimeError, match="no CPU path"):
        Encoder(ModelConfig(n_layer=1, d_model=64, n_head=1, d_ff=256, vocab=10, max_pos=8), {}, device="cpu")


def test_pack_ragged_right_and_left_padding():
    from sgpt_b200.encoder import pack_ragged

    ids = np.array([[5, 6, 7, 0], [9, 0, 0, 0], [1, 2, 3, 4]])
    mask = np.array([[1, 1, 1, 0], [1, 0, 0, 0], [1, 1, 1, 1]])
    p, pos, cu, mx = pack_ragged(ids, mask)
    assert p.tolist() == [5, 6, 7, 9, 1, 2, 3, 4] and pos.tolist() == [0, 1, 2, 0, 0, 1, 2, 3]
    assert cu.tolist() == [0, 3, 4, 8] and mx == 4
    # left padding keeps the PADDED index (pooling weights / position ids are functions of it)
    p, pos, cu, mx = pack_ragged(np.array([[0, 0, 8, 9]]), np.array([[0, 0, 1, 1]]))
    assert p.tolist() == [8, 9] and pos.tolist() == [2, 3]
    with pytest.raises(ValueError, match="contiguous"):
        pack_ragged(np.array([[1, 2, 3]]), np.array([[1, 0, 1]]))
    # an empty row is legal (the reference would divide 0/0 there)
    p, pos, cu, mx = pack_ragged(np.array([[1, 2], [3, 4]]), np.array([[0, 0], [1, 1]]))
    assert cu.tolist() == [0, 0, 2]


def test_shard_range_covers_corpus():
    from sgpt_b200.dist import shard_range

    for n, g in [(10, 3), (1000001, 8), (5, 8), (0, 2)]:
        spans = [shard_range(n, r, g) for r in range(g)]
        assert spans[0][0] == 0 and spans[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


def test_score_function_error_matches_reference():
    from sgpt_b200.index import _check_score_function

    with pytest.raises(ValueError, match=r"score function: euclid must be either \(cos_sim\)"):
        _check_score_function("euclid")


def test_reference_token_rules():
    """beir_dense_retriever.py:164-201: newline->space, truncation to maxseqlen(-2 with specb), brackets with mask 1,
    right padding, ValueError on empty text."""
    from sgpt_b200 import embedder
    from tests.helpers import ToyTokenizer

    tok = ToyTokenizer()
    e = object.__new__(embedder.CustomEmbedder)
    e.tokenizer, e.max_token_len, e.specb, e.pad_id = tok, 5 - 2, True, tok.pad_token_id
    e.bos_token_q, e.eos_token_q = tok.encode("["), tok.encode("]")
    e.bos_token_d, e.eos_token_d = tok.encode("{"), tok.encode("}")
    ids, mask = e.tokenize_batch(["a b\nc d e f", "x"], is_query=True)
    assert ids.shape == (2, 5) and ids[0, 0] == 58 and ids[0, 4] == 60 and mask[0].tolist() == [1] * 5
    assert ids[1, :3].tolist() == [58, tok.encode("x")[0], 60] and mask[1].tolist() == [1, 1, 1, 0, 0]
    assert ids[1, 3] == tok.pad_token_id
    assert ids[0, 1:4].tolist() == tok.encode("a b c")  # newline replaced, truncated to 3
    d_ids, _ = e.tokenize_batch(["x"], is_query=False)
    assert d_ids[0].tolist() == [90, tok.encode("x")[0], 92]
    with pytest.raises(ValueError, match="Empty items"):
        e.tokenize_batch(["   "], is_query=True)


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        sys.path.insert(0, ROOT)
        from oracle import search as osearch
        from sgpt_b200.dist import shard_range, sharded_search

        g = torch.Generator().manual_seed(5)
        queries, corpus = torch.randn(6, 16, generator=g), torch.randn(203, 16, generator=g)
        lo, hi = shard_range(len(corpus), rank, world)
        k = 12

        class CpuShard:  # stands in for CorpusShard: same contract, oracle arithmetic
            def search(self, qe, k, score_function):
                sc = osearch.cos_sim(qe, corpus[lo:hi])
                s, i = osearch.topk_ids(sc, k)
                pad = k - s.shape[1]
                if pad > 0:
                    s = torch.cat([s, torch.full((len(s), pad), float("-inf"))], 1)
                    i = torch.cat([i, torch.full((len(i), pad), -1 - lo, dtype=i.dtype)], 1)
                return s.contiguous(), (i + lo).contiguous()

        def cpu_merge(gs, gi, exclude):
            G, Q, kk = gs.shape
            s = gs.permute(1, 0, 2).reshape(Q, G * kk).clone()
            i = gi.permute(1, 0, 2).reshape(Q, G * kk)
            s[i < 0] = float("-inf")
            if exclude is not None:
                s[i == exclude[:, None]] = float("-inf")
            order = torch.argsort(-s, dim=1, stable=True)[:, :kk]
            return torch.gather(s, 1, order), torch.gather(i, 1, order)

        exclude = torch.tensor([7, -1, -1, 150, -1, -1])
        s, i = sharded_search(queries, CpuShard(), k, exclude_ids=exclude, merge=cpu_merge)
        full = osearch.cos_sim(queries, corpus)
        for qi in range(len(queries)):
            full[qi, exclude[qi]] = float("-inf") if exclude[qi] >= 0 else full[qi, exclude[qi]]
        es, ei = osearch.topk_ids(full, k)
        q.put((rank, bool(torch.equal(i, ei)), float((s - es).abs().max())))
    finally:
        dist.destroy_process_group()


def test_sharded_search_two_ranks_gloo():
    """N>1 path on CPU: 2 gloo ranks, each scanning its row range, all-gather of per-shard top-k, merge == global."""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in procs]
    [p.join(60) for p in procs]
    for rank, same_ids, err in res:
        assert same_ids and err < 1e-6, (rank, same_ids, err)


def _toy_embed(text, dim=16):
    """Deterministic text -> vector (stands in for the GPU encoder in the CPU tests)."""
    import zlib

    g = torch.Generator().manual_seed(zlib.crc32(text.encode()))
    return torch.randn(dim, generator=g)


class _StubEmbedder:
    device = torch.device("cpu")

    def __init__(self):
        self.corpus_calls = []

    def encode_queries(self, queries, batch_size, **kw):
        return torch.stack([_toy_embed(t) for _, t in queries])

    def encode_corpus(self, corpus, batch_size, batch_num="", **kw):
        self.corpus_calls.append((batch_num, [cid for cid, _ in corpus]))
        return torch.stack([_toy_embed((d["title"] + " " + d["text"]).strip()) for _, d in corpus])


def _toy_corpus(n=57):
    corpus = {f"d{i}": {"title": f"t{i}", "text": "w " * (1 + (i * 7) % 23)} for i in range(n)}
    queries = {"q0": "t3 " + "w " * 22, "d5": "some query", "q2": "another"}
    queries["q0"] = (corpus["d3"]["title"] + " " + corpus["d3"]["text"]).strip()  # exact duplicate of d3 -> top hit
    return corpus, queries


class _CpuShard:  # CorpusShard contract on CPU tensors with the oracle's arithmetic
    def __init__(self, dim, capacity):
        self.rows = []

    def add(self, emb):
        self.rows.append(emb.float())

    def search(self, qe, k, score_function):
        from oracle import search as osearch

        c = torch.cat(self.rows) if self.rows else torch.zeros(0, qe.shape[1])
        sc = osearch.SCORE_FUNCTIONS[score_function](qe, c) if len(c) else torch.zeros(len(qe), 0)
        s, i = osearch.topk_ids(sc, min(k, sc.shape[1])) if sc.shape[1] else (sc, sc.long())
        pad = k - s.shape[1]
        s = torch.cat([s, torch.full((len(s), pad), float("-inf"))], 1)
        i = torch.cat([i, torch.full((len(i), pad), -1, dtype=torch.int64)], 1)
        return s.contiguous(), i.contiguous()


def _cpu_merge(gs, gi, exclude):
    G, Q, kk = gs.shape
    s = gs.permute(1, 0, 2).reshape(Q, G * kk).clone()
    i = gi.permute(1, 0, 2).reshape(Q, G * kk)
    s[i < 0] = float("-inf")
    if exclude is not None:
        s[i == exclude[:, None]] = float("-inf")
    order = torch.argsort(-s, dim=1, stable=True)[:, :kk]
    s, i = torch.gather(s, 1, order), torch.gather(i, 1, order)
    return s, torch.where(torch.isinf(s), torch.full_like(i, -1), i)


def _expected_results(corpus, queries, top_k):
    """The reference algorithm on one process: oracle.search.search_embeddings over the length-sorted corpus."""
    out = {}
    cids = list(corpus)
    cemb = torch.stack([_toy_embed((corpus[c]["title"] + " " + corpus[c]["text"]).strip()) for c in cids])
    for qid, text in queries.items():
        sc = torch.nn.functional.cosine_similarity(_toy_embed(text)[None], cemb)
        ranked = [(float(s), c) for s, c in sorted(zip(sc.tolist(), cids), reverse=True) if c != qid][:top_k + 1]
        out[qid] = {c: s for s, c in ranked}
    return out


def _sharded_dres_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        sys.path.insert(0, ROOT)
        from sgpt_b200.dist import ShardedDenseRetrievalExactSearch

        corpus, queries = _toy_corpus()
        emb = _StubEmbedder()
        dres = ShardedDenseRetrievalExactSearch(emb, batch_size=8, corpus_chunk_size=10, shard_factory=_CpuShard,
                                                merge=_cpu_merge)
        res = dres.search(corpus, queries, top_k=5, score_function="cos_sim")
        q.put((rank, res, emb.corpus_calls))
    finally:
        dist.destroy_process_group()


def test_sharded_dres_two_ranks_gloo_matches_single_process():
    """End-to-end multi-rank DRES on CPU (gloo, 2 ranks, stub embedder): the corpus is dealt i mod G over the ranks after
    the length sort, each rank encodes only its share, and both ranks return the single-process result."""
    import torch.multiprocessing as mp

    corpus, queries = _toy_corpus()
    want = _expected_results(corpus, queries, 5)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_sharded_dres_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda t: t[0])
    [p.join(60) for p in procs]
    seen = []
    for rank, got, calls in res:
        assert set(got) == set(want)
        for qid in want:
            assert set(got[qid]) == set(want[qid]), (rank, qid)
            assert "d5" not in got["d5"]  # self match dropped (XS:118)
            for cid, s in want[qid].items():
                assert abs(got[qid][cid] - s) < 1e-5
        assert max(got["q0"], key=got["q0"].get) == "d3"
        assert all(len(ids) <= 10 for _, ids in calls) and [b for b, _ in calls] == [f"{rank}_{i}" for i in range(len(calls))]
        seen.append([c for _, ids in calls for c in ids])
    assert abs(len(seen[0]) - len(seen[1])) <= 1 and sorted(seen[0] + seen[1]) == sorted(corpus)  # disjoint cover
    # single process (no process group): same class, same answer
    from sgpt_b200.dist import ShardedDenseRetrievalExactSearch

    solo = ShardedDenseRetrievalExactSearch(_StubEmbedder(), corpus_chunk_size=10, shard_factory=_CpuShard,
                                            merge=_cpu_merge).search(corpus, queries, 5, "cos_sim")
    assert {k: set(v) for k, v in solo.items()} == {k: set(v) for k, v in want.items()}
