"""The masked (filtered) searches and CorpusShard deletions, bit for bit on integer data.

The corpora are the tie-heavy small-integer ones of test_gpu_search_exact.py (every device score exact, bf16 and int8
alike), and the reference is the exact top-k (tests/helpers.py topk_reference) with the masked documents removed:
each result must equal it under torch.equal, on every plan (dense, dense-uncached, two-pass), under every
SGPT_SEARCH_K_HI x SGPT_FRONT_SELECT setting, across 256-query blocks, for bf16 and int8 shards.  A mask of all ones
must return exactly the bits of the unmasked entry point, and every case checks that a second launch returns the same
bits."""
import math

import pytest
import torch

from tests.helpers import topk_reference
from tests.test_gpu_search_exact import D, TILE, _equal, _plan, _stride, corpus, two_pass_n

pytestmark = pytest.mark.gpu

N_PLANS = {"dense": 20000, "dense-uncached": 60000, "two-pass": None}


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _n(plan):
    return N_PLANS[plan] or two_pass_n(77)


def _pack(allow):
    from sgpt_b200.index import pack_mask

    return pack_mask(allow.cuda()).contiguous()


def _operands(Qf, Cf, dtype):
    if dtype == "int8":  # |x| <= 8: valid int8 rows, and the s32 dot products are the same integers
        return Qf.to(torch.int8).cuda(), Cf.to(torch.int8).cuda()
    return Qf.to(torch.bfloat16).cuda(), Cf.to(torch.bfloat16).cuda()


def _search(Q, C, k, dtype, words=None, pitch=0, id_base=0, packed=False, masked=True):
    """The masked entry point (masked=False: the unmasked one of the same dtype)."""
    L, lib = _lib()
    nq, n, D = Q.shape[0], C.shape[0], Q.shape[1]
    dt = L.DTYPE_I8 if dtype == "int8" else L.DTYPE_BF16
    ws = torch.empty(lib.sgpt_search_workspace_bytes(nq, n, k), dtype=torch.uint8, device="cuda")
    st = L.current_stream()
    if packed:
        from sgpt_b200.index import unpack_topk

        out = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        if masked:
            rc = lib.sgpt_search_packed_masked(dt, Q.data_ptr(), C.data_ptr(), None, None, nq, n, D, k, id_base,
                                               L.ptr(words), pitch, out.data_ptr(), ws.data_ptr(), ws.numel(), st)
        else:
            fn = lib.sgpt_search_packed_i8 if dtype == "int8" else lib.sgpt_search_packed
            rc = fn(Q.data_ptr(), C.data_ptr(), None, None, nq, n, D, k, id_base, out.data_ptr(), ws.data_ptr(),
                    ws.numel(), st)
        L.check(rc, "packed search")
        return unpack_topk(out.cpu())
    s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    if masked:
        rc = lib.sgpt_search_masked(dt, Q.data_ptr(), C.data_ptr(), None, None, nq, n, D, k, id_base, L.ptr(words),
                                    pitch, s.data_ptr(), i.data_ptr(), ws.data_ptr(), ws.numel(), st)
    else:
        fn = lib.sgpt_search_i8 if dtype == "int8" else lib.sgpt_search
        rc = fn(Q.data_ptr(), C.data_ptr(), None, None, nq, n, D, k, id_base, s.data_ptr(), i.data_ptr(), ws.data_ptr(),
                ws.numel(), st)
    L.check(rc, "search")
    return s.cpu(), i.cpu()


def _scores(Qf, Cf):
    sc = Qf.double() @ Cf.double().T
    return torch.nan_to_num(sc, nan=-1.0, posinf=math.inf, neginf=-math.inf)


def _reference(sc, allow, k, id_base=0):
    """Exact top-k of the allowed documents: allow bool [n] or [nq, n]."""
    ids = torch.arange(sc.shape[1], dtype=torch.int64).expand_as(sc) + id_base
    ids = torch.where(allow.expand_as(sc), ids, torch.full_like(ids, -1))
    return topk_reference(sc, ids, k)


def _sampled_tiles(n):
    s = _stride(n)
    t = torch.arange(n) // TILE
    return (t % s) == 0


def make_allow(kind, nq, n, k, g):
    """bool [n] (shared) or [nq, n] (per query) for a mask kind."""
    def frac(p, shape=(n,)):
        return torch.rand(shape, generator=g) < p

    def exactly(m):
        a = torch.zeros(n, dtype=torch.bool)
        a[torch.randperm(n, generator=g)[:m]] = True
        return a

    if kind == "ones":
        return torch.ones(n, dtype=torch.bool)
    if kind == "zeros":
        return torch.zeros(n, dtype=torch.bool)
    if kind == "fewer_than_k":
        return exactly(k - 1)
    if kind == "exactly_k":
        return exactly(k)
    if kind in ("sampled_only", "unsampled_only"):
        # (on the dense plans the tiles are only a pattern; on the two-pass plan unsampled_only leaves pass A without a
        # single allowed maximum, so tau must admit every allowed document)
        sampled = _sampled_tiles(n)
        return frac(0.5) & (sampled if kind == "sampled_only" else ~sampled)
    if kind == "p50":
        return frac(0.5)
    if kind == "p1":
        return frac(0.01)
    if kind == "p001":
        return frac(0.0001)
    if kind == "per_query":  # a different mask per query, at different densities
        p = torch.tensor([1.0, 0.5, 0.01, 0.0, 0.2, 0.0001, 0.9])[torch.arange(nq) % 7]
        return torch.rand((nq, n), generator=g) < p[:, None]
    if kind == "low_ids_masked":  # ties at the cut whose lowest ids are masked: the lowest ALLOWED ids must win
        a = frac(0.5)
        a[:n // 3] = False
        return a
    raise ValueError(kind)


KINDS = ["ones", "zeros", "fewer_than_k", "exactly_k", "sampled_only", "unsampled_only", "p50", "p1", "p001",
         "per_query", "low_ids_masked"]


def _run(kind, dtype, nq, n, k, seed, corpus_kind="random", id_base=0, check_packed=True):
    g = torch.Generator().manual_seed(seed)
    Qf, Cf = corpus("identical" if kind == "low_ids_masked" else corpus_kind, nq, n, k, g)
    Q, C = _operands(Qf, Cf, dtype)
    allow = make_allow(kind, nq, n, k, g)
    words = _pack(allow)
    pitch = words.shape[1] if allow.dim() == 2 else 0
    want = _reference(_scores(Qf, Cf), allow, k, id_base)
    what = f"{kind} {dtype} nq={nq} n={n} k={k} ({_plan(nq, n, k)})"
    got = _search(Q, C, k, dtype, words, pitch, id_base)
    _equal(what, got, want)
    again = _search(Q, C, k, dtype, words, pitch, id_base)
    assert torch.equal(got[0].view(torch.int32), again[0].view(torch.int32)) and torch.equal(got[1], again[1]), \
        f"{what}: a second search returned different bits"
    if check_packed:
        _equal(f"packed {what}", _search(Q, C, k, dtype, words, pitch, id_base, packed=True), want)
    if kind == "ones":
        plain = _search(Q, C, k, dtype, id_base=id_base, masked=False)
        assert torch.equal(got[0].view(torch.int32), plain[0].view(torch.int32)) and torch.equal(got[1], plain[1]), \
            f"{what}: an all-ones mask differs from the unmasked entry point"
        nomask = _search(Q, C, k, dtype, None, 0, id_base)
        assert torch.equal(got[0].view(torch.int32), nomask[0].view(torch.int32)) and torch.equal(got[1], nomask[1])
    return Qf, Cf, Q, C, allow, want


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("plan", ["dense", "dense-uncached", "two-pass"])
@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_masked_search_bit_exact(kind, plan, dtype):
    n = _n(plan)
    for j, (nq, k) in enumerate([(1, 1), (37, 10), (129, 1001), (37, 1025)]):
        assert _plan(nq, n, k) == plan
        _run(kind, dtype, nq, n, k, seed=1000 * j + KINDS.index(kind), id_base=(0, 7)[j % 2])


@pytest.mark.parametrize("kind", ["p1", "fewer_than_k", "unsampled_only", "per_query", "low_ids_masked"])
@pytest.mark.parametrize("k_hi", [None, "1", "k"])
@pytest.mark.parametrize("front", [None, "1"])
def test_masked_two_pass_settings_bit_exact(kind, k_hi, front, monkeypatch):
    """Every split of the candidate lists (SGPT_SEARCH_K_HI unset / 1 / k) with the front-list kernel off and on: under a
    selective mask the front parts often hold fewer than k entries and the back parts answer."""
    if front:
        monkeypatch.setenv("SGPT_FRONT_SELECT", front)
    n = two_pass_n(77)
    for j, (nq, k) in enumerate([(1, 1), (37, 10), (128, 1001), (257, 1025)]):
        if k_hi:
            monkeypatch.setenv("SGPT_SEARCH_K_HI", str(k) if k_hi == "k" else k_hi)
        _run(kind, ("bf16", "int8")[j % 2], nq, n, k, seed=77 + j, check_packed=False)


@pytest.mark.parametrize("nq", [1, 37, 128, 129, 255, 256, 257, 300])
def test_masked_query_blocks_bit_exact(nq):
    """CTA pairs above 128 queries and 256-query blocks: per-query bitmaps must follow their queries into each block."""
    n = two_pass_n(77)
    _run("per_query", "bf16", nq, n, 1001, seed=nq)
    _run("per_query", "int8", nq, 20000, 10, seed=nq + 1)


@pytest.mark.parametrize("plan", ["dense", "two-pass"])
def test_shared_mask_equals_the_same_mask_per_query(plan):
    """Pitch 0 against the same bitmap repeated per query, at a pitch with spare words; bits past n (inside the last
    word and in the spare words) are set and must be ignored."""
    n, nq, k = _n(plan) - 5, 40, 1001
    g = torch.Generator().manual_seed(5)
    Qf, Cf = corpus("random", nq, n, k, g)
    Q, C = _operands(Qf, Cf, "bf16")
    allow = torch.rand(n, generator=g) < 0.3
    shared = _pack(allow)
    W = shared.numel()
    assert n % 32 != 0
    shared_dirty = shared.clone()
    shared_dirty[-1] |= torch.tensor(-1 << (n % 32), dtype=torch.int32, device="cuda")  # bits n .. 32 W - 1
    per = torch.full((nq, W + 3), -1, dtype=torch.int32, device="cuda")
    per[:, :W] = shared_dirty
    want = _reference(_scores(Qf, Cf), allow, k)
    a = _search(Q, C, k, "bf16", shared, 0)
    _equal("shared", a, want)
    _equal("shared, bits past n", _search(Q, C, k, "bf16", shared_dirty, 0), want)
    _equal("per query, pitch W + 3", _search(Q, C, k, "bf16", per, W + 3), want)


def _range(Q, C, thr, words, pitch, cap, dtype="bf16", id_base=0):
    L, lib = _lib()
    nq, n, D = Q.shape[0], C.shape[0], Q.shape[1]
    dt = L.DTYPE_I8 if dtype == "int8" else L.DTYPE_BF16
    ws = torch.empty(lib.sgpt_range_search_workspace_bytes(nq, n), dtype=torch.uint8, device="cuda")
    counts = torch.full((nq,), -7, dtype=torch.int64, device="cuda")
    s = torch.full((max(cap, 1),), 7.0, dtype=torch.float32, device="cuda")
    i = torch.full((max(cap, 1),), -7, dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_range_search_masked(dt, Q.data_ptr(), C.data_ptr(), None, None, nq, n, D, float(thr), id_base,
                                         L.ptr(words), pitch, counts.data_ptr(), cap, s.data_ptr(), i.data_ptr(),
                                         ws.data_ptr(), ws.numel(), L.current_stream()), "sgpt_range_search_masked")
    return counts.cpu(), s.cpu(), i.cpu()


@pytest.mark.parametrize("kind", ["ones", "zeros", "p50", "p1", "per_query", "unsampled_only"])
@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_masked_range_search_bit_exact(kind, dtype):
    """Counts and CSR entries (ascending id) of the allowed documents only; with `cap` below the total only the queries
    that fit are written and the rest of both buffers keeps its bits."""
    n, nq = 20000, 300
    g = torch.Generator().manual_seed(11)
    Qf, Cf = corpus("random", nq, n, 10, g)
    Q, C = _operands(Qf, Cf, dtype)
    allow = make_allow(kind, nq, n, 10, g)
    words = _pack(allow)
    pitch = words.shape[1] if allow.dim() == 2 else 0
    sc = _scores(Qf, Cf)
    thr = 12.0
    hit = (sc >= thr) & allow.expand_as(sc)
    want_counts = hit.sum(1)
    total = int(want_counts.sum())
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), want_counts.cumsum(0)])
    for cap in (total, total // 2, 0):
        counts, s, i = _range(Q, C, thr, words, pitch, cap, dtype, id_base=3)
        assert torch.equal(counts, want_counts), f"{kind} {dtype}: counts differ"
        fit_end = 0  # the queries that fit are a prefix; their entries end here
        for q in range(nq):
            a, b = int(offsets[q]), int(offsets[q + 1])
            if b > cap:
                break
            fit_end = b
            docs = hit[q].nonzero().flatten()
            assert torch.equal(i[a:b], docs + 3), f"{kind} {dtype} cap={cap} query {q}: ids differ"
            assert torch.equal(s[a:b].double(), sc[q, docs]), f"{kind} {dtype} cap={cap} query {q}: scores differ"
        assert (i[fit_end:cap] == -7).all() and (s[fit_end:cap] == 7.0).all(), f"{kind} {dtype} cap={cap}: overwritten"


@pytest.mark.parametrize("plan", ["dense", "two-pass"])
def test_masked_halves_merge_and_gather_equal_whole_search(plan):
    """Two masked half shards merged with merge_topk_packed equal the whole masked search, and so does PeerGather at
    world size 1 over a CorpusShard whose deletions are the masked documents."""
    from sgpt_b200 import CorpusShard
    from sgpt_b200.dist import PeerGather
    from sgpt_b200.index import merge_topk_packed

    n = _n(plan) * 2
    nq, k, id_base = 37, 1001, 5
    g = torch.Generator().manual_seed(3)
    Qf, Cf = corpus("random", nq, n, k, g)
    Q, C = _operands(Qf, Cf, "bf16")
    allow = torch.rand(n, generator=g) < 0.2
    want = _reference(_scores(Qf, Cf), allow, k, id_base)
    whole = _search(Q, C, k, "bf16", _pack(allow), 0, id_base)
    _equal("whole", whole, want)
    h = n // 2 + 13  # (an unaligned cut: the second half's bitmap starts mid-word)
    from tests.test_gpu_topk import pack

    parts = []
    for a, b in ((0, h), (h, n)):
        parts.append(pack(*_search(Q, C[a:b], k, "bf16", _pack(allow[a:b]), 0, id_base + a, packed=True)))
    s, i = merge_topk_packed(torch.stack(parts).cuda())
    _equal("merge_topk_packed of two masked halves", (s.cpu(), i.cpu()), want)
    shard = CorpusShard.from_embeddings(C, device="cuda:0", id_base=id_base)
    shard.remove((~allow).nonzero().flatten() + id_base)
    pg = PeerGather(nq, k, "cuda:0")
    try:
        s, i = pg.search(shard, Q, k, "dot")
        _equal("PeerGather world 1 with deletions", (s.cpu(), i.cpu()), want)
    finally:
        pg.close()


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_corpus_shard_remove_equals_a_rebuilt_shard(dtype, tmp_path):
    """remove() then search equals a shard built without the removed rows, after mapping its ids back; allow= combines
    with the deletions; add() after remove() appends allowed rows; save / load keep the deletions."""
    from sgpt_b200 import CorpusShard

    n, nq, k, id_base = 20000, 50, 100, 1000
    g = torch.Generator().manual_seed(21)
    Qf, Cf = corpus("random", nq, n + 300, k, g)
    Q = Qf.cuda()
    shard = CorpusShard(D, n + 300, device="cuda:0", id_base=id_base, dtype=dtype)
    shard.add(Cf[:n].cuda())
    gone = torch.randperm(n, generator=g)[:n // 3]
    shard.remove(gone + id_base)
    shard.remove(gone[:10] + id_base)  # twice is allowed
    assert shard.n_deleted == len(gone)
    keep = torch.ones(n, dtype=torch.bool)
    keep[gone] = False
    kept_rows = keep.nonzero().flatten()
    rebuilt = CorpusShard.from_embeddings(Cf[:n][keep].cuda(), device="cuda:0", dtype=dtype)
    for fn in ("dot", "cos_sim"):
        s, i = shard.search(Q, k, fn)
        rs, ri = rebuilt.search(Q, k, fn)
        ri = torch.where(ri >= 0, kept_rows.cuda()[ri.clamp(min=0)] + id_base, ri)
        # the rebuilt shard orders ties by its own (monotone) ids, so the mapped ids are in the same order
        assert torch.equal(s.view(torch.int32), rs.view(torch.int32)) and torch.equal(i, ri), f"{dtype} {fn}"
        packed = shard.search_packed(Q, k, fn)
        from sgpt_b200.index import unpack_topk

        ps, pi = unpack_topk(packed)
        assert torch.equal(ps.view(torch.int32), s.view(torch.int32)) and torch.equal(pi, i)
    # allow= on top of the deletions, per query
    allow = torch.rand((nq, n), generator=g) < 0.5
    s, i = shard.search(Q, k, "dot", allow=allow.cuda())
    sc = _scores(Qf, Cf[:n]) if dtype == "bf16" else None
    if sc is not None:
        _equal("allow & ~deleted", (s.cpu(), i.cpu()), _reference(sc, allow & keep, k, id_base))
    # range search honours the deletions
    off, rs_, ri_ = shard.range_search(Q, 12.0, "dot")
    assert not torch.isin(ri_.cpu(), gone + id_base).any()
    # add() after remove(): the new rows are allowed
    shard.add(Cf[n:].cuda())
    assert shard.n_deleted == len(gone)
    s2, i2 = shard.search(Q, k, "dot")
    assert not torch.isin(i2.cpu(), gone + id_base).any()
    # save / load keeps the deletions bit for bit
    shard.save(str(tmp_path / "s"))
    back = CorpusShard.load(str(tmp_path / "s"), device="cuda:0")
    assert back.n_deleted == len(gone)
    s3, i3 = back.search(Q, k, "dot")
    assert torch.equal(s3.view(torch.int32), s2.view(torch.int32)) and torch.equal(i3, i2)


@pytest.mark.parametrize("start", [0, 33, 64, 100])
def test_views_share_deletions_at_unaligned_starts(start):
    from sgpt_b200 import CorpusShard

    n, nq, k = 20000, 20, 50
    g = torch.Generator().manual_seed(start)
    Qf, Cf = corpus("random", nq, n, k, g)
    shard = CorpusShard.from_embeddings(Cf.cuda(), device="cuda:0")
    gone = torch.randperm(n, generator=g)[:5000]
    shard.remove(gone)
    end = n - 77
    v = shard.view(start, end)
    keep = torch.ones(n, dtype=torch.bool)
    keep[gone] = False
    assert v.n_deleted == int((~keep[start:end]).sum())
    s, i = v.search(Qf.cuda(), k, "dot")
    _equal(f"view({start}, {end})", (s.cpu(), i.cpu()), _reference(_scores(Qf, Cf[start:end]), keep[start:end], k, start))
    v.remove([start + 1])  # removal through the view reaches the parent
    keep[start + 1] = False
    s, i = shard.search(Qf.cuda(), k, "dot")
    _equal("parent after a removal through the view", (s.cpu(), i.cpu()), _reference(_scores(Qf, Cf), keep, k))


def test_semantic_search_and_mining_on_a_shard_with_deletions():
    from sgpt_b200 import CorpusShard, community_detection, paraphrase_mining_embeddings, semantic_search

    n, nq = 3000, 4
    g = torch.Generator().manual_seed(9)
    Qf, Cf = corpus("random", nq, n, 10, g)
    shard = CorpusShard.from_embeddings(Cf.cuda(), device="cuda:0")
    shard.remove(torch.arange(0, n, 2))
    hits = semantic_search(Qf.cuda(), shard, top_k=20, score_function="dot")
    keep = torch.arange(n) % 2 == 1
    ws, wi = _reference(_scores(Qf, Cf), keep, 20)
    for q in range(nq):
        assert [h["corpus_id"] for h in hits[q]] == wi[q].tolist()
        assert [h["score"] for h in hits[q]] == ws[q].tolist()
    with pytest.raises(ValueError, match="deleted documents"):
        paraphrase_mining_embeddings(shard)
    with pytest.raises(ValueError, match="deleted documents"):
        community_detection(shard)
