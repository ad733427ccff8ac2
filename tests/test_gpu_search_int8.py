"""int8 corpus shards: the quantizer, the int8 similarity GEMM and every search on top of it, bit for bit.

The quantizer is compared with a torch fp32 restatement of the contract in include/sgpt_b200.h (int8 corpus shards).
Scores are exact: the s32 dot product is exact on the device and in an fp64 matmul of the same integers, both sides round
it to fp32 once and multiply by the two scales in the same order.  The search tests reuse the tie-heavy small-integer
corpora of test_gpu_search_exact.py (|x| <= 8, D = 64: valid int8 rows) with power-of-two scales, so their fp64 reference
is exact too and every result must equal the exact top-k (score descending, ties by ascending id) under torch.equal.
Every case also checks that a second launch returns the same bits."""
import math

import pytest
import torch

from tests.test_gpu_search_exact import _equal, _plan, _reference, corpus, two_pass_n

pytestmark = pytest.mark.gpu

NAN = float("nan")


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def quant_ref(x):
    """The quantization contract in torch fp32 arithmetic (CPU): x fp32/bf16 [n, D] -> (int8, scale, cos_scale)."""
    x = x.float().cpu()
    amax = x.abs().amax(1)
    bad = ~torch.isfinite(x).all(1)
    zero = (amax == 0) & ~bad
    m = torch.full_like(amax, 127.0) / amax
    q = torch.round(x * m[:, None]).clamp(-127, 127)  # torch.round: half to even, like rint
    q[bad | zero] = 0
    q = q.to(torch.int8)
    scale = amax / torch.full_like(amax, 127.0)
    ss = (q.long() ** 2).sum(1)
    cos = scale / torch.clamp(scale * torch.sqrt(ss.float()), min=1e-12)
    scale[zero], cos[zero] = 0.0, 0.0
    scale[bad], cos[bad] = NAN, NAN
    return q, scale, cos


def quantize(x):
    from sgpt_b200.index import quantize_rows_i8

    return quantize_rows_i8(x.cuda())


def _bits_equal(a, b):
    return torch.equal(a.cpu().contiguous().view(torch.int32), b.cpu().contiguous().view(torch.int32))


def _quant_rows(D, g):
    x = torch.randn(40, D, generator=g) * torch.logspace(-3, 3, 40)[:, None]
    x[1] = 0.0
    x[2, D // 3] = NAN
    x[3, -1] = math.inf
    x[4, 0] = -math.inf
    x[5] = 0.0
    x[5, 7] = -1e-30  # tiny amax, one nonzero element
    # amax 127 (m = 1) and 254 (m = 0.5): products land exactly on .5 and must round half to even
    x[6] = torch.arange(D).float() % 9 - 4.5
    x[6, 0] = 127.0
    x[7] = (torch.arange(D).float() % 13) * 2 - 11
    x[7, 1] = -254.0
    x[8] = 1.0  # every element equal to amax
    return x


@pytest.mark.parametrize("D", [16, 768, 784, 4096])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_quantizer_bit_exact(D, dtype):
    g = torch.Generator().manual_seed(D)
    x = _quant_rows(D, g)
    if dtype == "bf16":
        x = x.to(torch.bfloat16)
    want = quant_ref(x)
    got = quantize(x)
    assert torch.equal(got[0].cpu(), want[0]), "int8 rows differ"
    for name, a, b in (("scale", got[1], want[1]), ("cos_scale", got[2], want[2])):
        assert _bits_equal(a, b), f"{name}: got {a.cpu()[:10]}, want {b[:10]}"
    assert torch.isnan(got[1][2]) and torch.isnan(got[2][3]) and float(got[1][1]) == 0.0
    assert got[0][6].cpu()[1:9].tolist() == [-4, -2, -2, 0, 0, 2, 2, 4]  # x.5 -> even
    again = quantize(x)
    assert torch.equal(got[0], again[0]) and _bits_equal(got[1], again[1]) and _bits_equal(got[2], again[2]), \
        "a second launch returned different bits"


def _scores_i8(Q, C, qs, cs):
    L, lib = _lib()
    nq, n, D = Q.shape[0], C.shape[0], Q.shape[1]
    lds = n + 3
    out = torch.full((nq, lds), 7.0, dtype=torch.float32, device="cuda")
    L.check(lib.sgpt_scores_i8(Q.data_ptr(), C.data_ptr(), L.ptr(qs), L.ptr(cs), out.data_ptr(), lds, nq, n, D,
                               L.current_stream()), "sgpt_scores_i8")
    return out.cpu()


@pytest.mark.parametrize("D", [16, 112, 128, 784])
@pytest.mark.parametrize("nq,n", [(1, 77), (77, 1000), (300, 2333)])
def test_scores_i8_exact(D, nq, n):
    """Full int8 range (-128 included), ragged n and nq, K tails; NaN scales give -1; the pad columns keep their bits."""
    g = torch.Generator().manual_seed(D * 1000 + nq)
    Q = torch.randint(-128, 128, (nq, D), generator=g, dtype=torch.int8)
    C = torch.randint(-128, 128, (n, D), generator=g, dtype=torch.int8)
    qs = torch.rand(nq, generator=g) + 0.01
    cs = torch.rand(n, generator=g) + 0.01
    qs[nq // 2] = NAN
    cs[n // 3] = NAN
    dot = (Q.double() @ C.double().T).float()  # exact integers, rounded once to fp32
    for a, b in ((None, None), (qs, cs)):
        want = dot.clone()
        if a is not None:
            want = want * a[:, None] * b[None, :]
        want = torch.where(torch.isnan(want), torch.full_like(want, -1.0), want)
        got = _scores_i8(Q.cuda(), C.cuda(), None if a is None else a.cuda(), None if b is None else b.cuda())
        assert _bits_equal(got[:, :n], want), f"D={D} nq={nq} n={n}: max diff {(got[:, :n] - want).abs().max()}"
        assert (got[:, n:] == 7.0).all()
        again = _scores_i8(Q.cuda(), C.cuda(), None if a is None else a.cuda(), None if b is None else b.cuda())
        assert _bits_equal(got, again)
    if nq > 1:
        assert (got[nq // 2, :n] == -1).all() and (got[:, n // 3] == -1).all()


def _rows_of_larger_buffer(Q):
    """Q as the first rows of a buffer twice its size whose other rows differ: a query block taken at the wrong row
    step reads other queries (and stays inside the allocation) instead of the right ones."""
    buf = torch.cat([Q, -Q.flip(0)])
    return buf[:Q.shape[0]]


def _search_i8(Q, C, k, id_base=0, q_scale=None, c_scale=None, packed=False):
    L, lib = _lib()
    nq, n, D = Q.shape[0], C.shape[0], Q.shape[1]
    ws = torch.empty(lib.sgpt_search_workspace_bytes(nq, n, k), dtype=torch.uint8, device="cuda")
    qs, cs = L.ptr(q_scale), L.ptr(c_scale)
    if packed:
        from sgpt_b200.index import unpack_topk

        out = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        L.check(lib.sgpt_search_packed_i8(Q.data_ptr(), C.data_ptr(), qs, cs, nq, n, D, k, id_base, out.data_ptr(),
                                          ws.data_ptr(), ws.numel(), L.current_stream()), "sgpt_search_packed_i8")
        return unpack_topk(out.cpu())
    s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_search_i8(Q.data_ptr(), C.data_ptr(), qs, cs, nq, n, D, k, id_base, s.data_ptr(), i.data_ptr(),
                               ws.data_ptr(), ws.numel(), L.current_stream()), "sgpt_search_i8")
    return s.cpu(), i.cpu()


def _run_case(kind, nq, n, k, id_base, seed, scales=False):
    g = torch.Generator().manual_seed(seed)
    Qf, Cf = corpus(kind, nq, n, k, g)
    Q, C = _rows_of_larger_buffer(Qf.to(torch.int8).cuda()), Cf.to(torch.int8).cuda()
    qs = cs = None
    if scales:  # powers of two keep every score exact
        qs = (2.0 ** torch.randint(-1, 2, (nq,), generator=g).float()).cuda()
        cs = (2.0 ** torch.randint(-1, 3, (n,), generator=g).float()).cuda()
    want = _reference(Qf, Cf, k, id_base, qs, cs)
    what = f"{kind} nq={nq} n={n} k={k} id_base={id_base} ({_plan(nq, n, k)})"
    got = _search_i8(Q, C, k, id_base, qs, cs)
    _equal(f"sgpt_search_i8 {what}", got, want)
    again = _search_i8(Q, C, k, id_base, qs, cs)
    assert _bits_equal(got[0], again[0]) and torch.equal(got[1], again[1]), f"{what}: a second search differs"
    if id_base + n < 2 ** 31:
        _equal(f"sgpt_search_packed_i8 {what}", _search_i8(Q, C, k, id_base, qs, cs, packed=True), want)
    return Q, C, want


@pytest.mark.parametrize("kind", ["random", "identical", "negative"])
@pytest.mark.parametrize("n_name", ["dense", "dense-uncached", "two-pass"])
def test_search_i8_plans_bit_exact(kind, n_name):
    n = {"dense": 20000, "dense-uncached": 60000, "two-pass": two_pass_n(77)}[n_name]
    for j, (nq, k) in enumerate([(1, 1), (37, 10), (129, 1001), (37, 1025)]):
        _run_case(kind, nq, n, k, id_base=(0, 7)[j % 2], seed=j, scales=j % 2 == 1)


@pytest.mark.parametrize("kind", ["k_sampled", "k_unsampled", "negative"])
@pytest.mark.parametrize("k_hi", [None, "1", "k"])
@pytest.mark.parametrize("front", [None, "1"])
def test_search_i8_two_pass_thresholds_bit_exact(kind, k_hi, front, monkeypatch):
    """The two-pass plan at its admission edges under every SGPT_SEARCH_K_HI x SGPT_FRONT_SELECT setting; the last tile
    is ragged and sampled."""
    if front:
        monkeypatch.setenv("SGPT_FRONT_SELECT", front)
    n = two_pass_n(77)
    for j, (nq, k) in enumerate([(1, 1), (37, 10), (128, 1001), (257, 1025)]):
        if k_hi:
            monkeypatch.setenv("SGPT_SEARCH_K_HI", str(k) if k_hi == "k" else k_hi)
        assert _plan(nq, n, k) == "two-pass"
        _run_case(kind, nq, n, k, id_base=(0, 7, 2 ** 31 - 1 - n, 3)[j], seed=100 + j)


@pytest.mark.parametrize("nq", [1, 37, 128, 129, 256, 257, 300])
def test_search_i8_query_blocks_bit_exact(nq):
    """CTA pairs above 128 queries and query blocks of 256 above 256 (the per-block query step is D bytes per row)."""
    n = two_pass_n(77)
    _run_case("random", nq, n, 1001, id_base=2 ** 31 - 1 - n, seed=nq, scales=True)
    _run_case("random", nq, 20000, 10, id_base=3, seed=nq + 1)


@pytest.mark.parametrize("n_name", ["dense", "two-pass"])
def test_search_i8_shards_merged_equal_whole(n_name):
    from sgpt_b200.index import merge_topk_packed
    from tests.test_gpu_topk import pack

    n = {"dense": 20000, "two-pass": 2 * two_pass_n(77)}[n_name]
    nq, k, id_base = 37, 1001, 5
    Q, C, want = _run_case("random", nq, n, k, id_base, seed=3)
    cut = n // 2
    parts = [_search_i8(Q, C[:cut], k, id_base), _search_i8(Q, C[cut:], k, id_base + cut)]
    P = torch.stack([pack(s, i) for s, i in parts]).cuda()
    s, i = merge_topk_packed(P)
    _equal(f"two int8 shards merged ({n_name})", (s.cpu(), i.cpu()), want)


def _range_i8(Q, C, threshold, id_base, cap, qs=None, cs=None):
    L, lib = _lib()
    nq, n, D = Q.shape[0], C.shape[0], Q.shape[1]
    ws = torch.empty(lib.sgpt_range_search_workspace_bytes(nq, n), dtype=torch.uint8, device="cuda")
    counts = torch.full((nq,), -5, dtype=torch.int64, device="cuda")
    out_s = torch.full((max(cap, 1),), 9.0, dtype=torch.float32, device="cuda")
    out_i = torch.full((max(cap, 1),), -9, dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_range_search_i8(Q.data_ptr(), C.data_ptr(), L.ptr(qs), L.ptr(cs), nq, n, D, float(threshold), id_base,
                                     counts.data_ptr(), cap, out_s.data_ptr(), out_i.data_ptr(), ws.data_ptr(), ws.numel(),
                                     L.current_stream()), "sgpt_range_search_i8")
    return counts.cpu(), out_s.cpu(), out_i.cpu()


@pytest.mark.parametrize("nq", [1, 37, 300])
@pytest.mark.parametrize("threshold", [-1e9, -3.0, 6.0, 40.0])
def test_range_search_i8_bit_exact(nq, threshold):
    """Every document with score >= threshold in ascending id order; cap 0 (counts only), tight (a query straddles it)
    and ample; a NaN document scale scores -1."""
    g = torch.Generator().manual_seed(nq)
    n, id_base = 5000, 11
    Qf, Cf = corpus("random", nq, n, 10, g)
    cs = (2.0 ** torch.randint(-1, 2, (n,), generator=g).float())
    cs[::97] = NAN
    sc = (Qf.double() @ Cf.double().T) * cs.double()[None, :]
    sc = torch.nan_to_num(sc, nan=-1.0)
    keep = sc >= threshold
    counts = keep.sum(1)
    total = int(counts.sum())
    Q, C = _rows_of_larger_buffer(Qf.to(torch.int8).cuda()), Cf.to(torch.int8).cuda()
    off = torch.cumsum(counts, 0) - counts
    for cap in sorted({0, total // 2, total + 100}):
        got_c, got_s, got_i = _range_i8(Q, C, threshold, id_base, cap, None, cs.cuda())
        assert torch.equal(got_c, counts), "counts differ"
        for q in range(nq):
            a, c = int(off[q]), int(counts[q])
            if a + c > cap:
                continue
            cols = keep[q].nonzero().flatten()
            assert torch.equal(got_i[a:a + c], cols + id_base), f"query {q} ids (cap {cap})"
            assert torch.equal(got_s[a:a + c].double(), sc[q, cols]), f"query {q} scores (cap {cap})"
        fitted = int((off + counts <= cap).sum())
        if cap > 0:
            last = int((off + counts)[:fitted].max()) if fitted else 0
            assert (got_i[last:cap] == -9).all(), "slots past the fitted queries were written"
        again = _range_i8(Q, C, threshold, id_base, cap, None, cs.cuda())
        assert torch.equal(again[0], got_c) and _bits_equal(again[1], got_s) and torch.equal(again[2], got_i), \
            "a second launch returned different bits"


def _continuous(nq, n, D, g):
    Q = torch.randn(nq, D, generator=g)
    C = torch.randn(n, D, generator=g)
    C[::50] = Q[torch.arange(0, n, 50) % nq] + 0.3 * C[::50]
    return Q.cuda(), C.cuda()


@pytest.mark.parametrize("score_function", ["cos_sim", "dot"])
def test_corpus_shard_int8_matches_entry_points(score_function, tmp_path):
    """CorpusShard(dtype="int8"): search, search_packed, range_search and view equal the raw entry points on the shard's
    own int8 rows and the quantized queries; save/load is bit-identical; a bf16 shard's stored rows convert."""
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import unpack_topk

    g = torch.Generator().manual_seed(7)
    Qd, Cd = _continuous(37, 30000, 784, g)
    shard = CorpusShard.from_embeddings(Cd, device="cuda:0", id_base=100, dtype="int8")
    q8, qsc, qcs = quantize(Qd)
    c8, csc, ccs = quantize(Cd)
    assert torch.equal(shard.stored(), c8) and _bits_equal(shard.scales, csc) and _bits_equal(shard.cos_scales, ccs)
    qs, cs = (qcs, ccs) if score_function == "cos_sim" else (qsc, csc)
    k = 100
    L, lib = _lib()
    ws = torch.empty(lib.sgpt_search_workspace_bytes(37, shard.n, k), dtype=torch.uint8, device="cuda")
    s = torch.empty((37, k), dtype=torch.float32, device="cuda")
    i = torch.empty((37, k), dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_search_i8(q8.data_ptr(), c8.data_ptr(), qs.data_ptr(), cs.data_ptr(), 37, shard.n, 784, k, 100,
                               s.data_ptr(), i.data_ptr(), ws.data_ptr(), ws.numel(), L.current_stream()))
    gs, gi = shard.search(Qd, k, score_function)
    assert _bits_equal(gs, s) and torch.equal(gi, i)
    ps, pi = unpack_topk(shard.search_packed(Qd, k, score_function).cpu())
    assert _bits_equal(ps, s) and torch.equal(pi, i.cpu())
    # range search: the threshold at the 10th best score of query 0
    thr = float(s[0, 9])
    off, rs, ri = shard.range_search(Qd, thr, score_function)
    counts, out_s, out_i = _range_i8(q8, c8, thr, 100, 10 ** 6, qs, cs)
    assert torch.equal((off[1:] - off[:-1]).cpu(), counts) and int(counts[0]) >= 10
    assert _bits_equal(rs, out_s[:int(off[-1])]) and torch.equal(ri.cpu(), out_i[:int(off[-1])])
    # a view searches its rows with ids = positions inside the shard
    v = shard.view(1001, 9001)
    vs, vi = v.search(Qd, k, score_function)
    want = _search_i8(q8, c8[1001:9001].contiguous(), k, 1001, qs, cs[1001:9001].contiguous())
    assert _bits_equal(vs, want[0]) and torch.equal(vi.cpu(), want[1])
    # save / load
    shard.save(str(tmp_path / "s"))
    back = CorpusShard.load(str(tmp_path / "s"), device="cuda:0")
    assert back.dtype == "int8" and back.id_base == 100 and back.n == shard.n
    assert torch.equal(back.stored(), shard.stored()) and _bits_equal(back.scales[:back.n], shard.scales[:shard.n])
    assert _bits_equal(back.cos_scales[:back.n], shard.cos_scales[:shard.n])
    bs, bi = back.search(Qd, k, score_function)
    assert _bits_equal(bs, gs) and torch.equal(bi, gi)
    # converting a saved bf16 shard
    b16 = CorpusShard.from_embeddings(Cd, device="cuda:0")
    conv = CorpusShard.from_embeddings(b16.stored(), dtype="int8")
    assert torch.equal(conv.stored(), quantize(b16.stored())[0])


@pytest.mark.parametrize("score_function", ["cos_sim", "dot"])
def test_int8_search_continuous_vs_fp64_dequantized(score_function):
    """On continuous data the ids equal an fp64 top-k of the dequantized stored vectors and queries, ids within a few
    ulps of the cut compared as sets; scores within fp32 rounding."""
    from sgpt_b200 import CorpusShard

    g = torch.Generator().manual_seed(11)
    Qd, Cd = _continuous(129, 200000, 768, g)
    shard = CorpusShard.from_embeddings(Cd, device="cuda:0", dtype="int8")
    k = 1001
    s, i = shard.search(Qd, k, score_function)
    s, i = s.cpu(), i.cpu()
    q8, qsc, qcs = quantize(Qd)
    cos = score_function == "cos_sim"
    qs = (qcs if cos else qsc).double()
    cs = (shard.cos_scales if cos else shard.scales)[:shard.n].double()
    full = (q8.double() @ shard.stored().double().T) * qs[:, None] * cs[None, :]
    ws_, wi = (t.cpu() for t in torch.topk(full, k, dim=1))
    tol = 4e-7 * float(full.abs().max())
    for q in range(0, 129, 8):
        fq = full[q].cpu()
        cut = float(ws_[q, -1])
        got = set(i[q].tolist())
        safe = {int(j) for j, v in zip(wi[q].tolist(), ws_[q].tolist()) if v > cut + 2 * tol}
        assert safe <= got, f"query {q}: {len(safe - got)} ids clearly above the cut missing"
        assert all(float(fq[j]) >= cut - 2 * tol for j in got)
        assert (s[q].double() - fq[i[q]]).abs().max() <= tol


def test_int8_shard_through_semantic_search_sharded_search_and_sharded_dres():
    from sgpt_b200 import CorpusShard, semantic_search
    from sgpt_b200.dist import PeerGather, ShardedDenseRetrievalExactSearch, sharded_search

    g = torch.Generator().manual_seed(5)
    Qd, Cd = _continuous(20, 3000, 256, g)
    shard = CorpusShard.from_embeddings(Cd, device="cuda:0", id_base=0, dtype="int8")
    s, i = shard.search(Qd, 10, "cos_sim")
    hits = semantic_search(Qd, shard, top_k=10)
    assert [[h["corpus_id"] for h in row] for row in hits] == i.cpu().tolist()
    assert [[h["score"] for h in row] for row in hits] == s.cpu().tolist()
    ss, si = sharded_search(Qd, shard, 10, "cos_sim")
    assert torch.equal(si, i) and _bits_equal(ss, s)
    # excluding each query's best hit: the other ten of its top 11, then an empty slot
    ex = i[:, 0].clone()
    ss, si = sharded_search(Qd, shard, 11, "cos_sim", exclude_ids=ex)
    s11, i11 = shard.search(Qd, 11, "cos_sim")
    assert torch.equal(si[:, :10], i11[:, 1:]) and _bits_equal(ss[:, :10], s11[:, 1:]) and (si[:, 10] == -1).all()
    # PeerGather at world size 1: sgpt_search_gather_i8 equals sgpt_search_i8
    pg = PeerGather(20, 10, "cuda:0")
    try:
        gs, gi = pg.search(shard, Qd, 10, "cos_sim")
        gs2, gi2 = pg.search(shard, Qd, 10, "cos_sim")
    finally:
        pg.close()
    assert _bits_equal(gs, s) and torch.equal(gi, i) and _bits_equal(gs2, s) and torch.equal(gi2, i)

    class Emb:
        device = torch.device("cuda:0")

        def encode_queries(self, queries, batch_size, **kw):
            return Qd[[int(q[1:]) for q, _ in queries]]

        def encode_corpus(self, docs, batch_size, **kw):
            return Cd[[int(c[1:]) for c, _ in docs]]

    corpus_ = {f"d{j}": {"title": "", "text": "x" * (j % 17)} for j in range(Cd.shape[0])}
    queries = {f"q{j}": "q" for j in range(Qd.shape[0])}
    res = ShardedDenseRetrievalExactSearch(Emb(), shard_dtype="int8").search(corpus_, queries, 10, "cos_sim")
    for q in range(20):
        assert res[f"q{q}"] == {f"d{int(j)}": float(v) for v, j in zip(s11[q], i11[q])}, q
