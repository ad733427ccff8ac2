"""The filtered IVF-PQ search (sgpt_ivfpq_search_masked, IVFPQIndex.search(allow=)) bit for bit.

Kernel: small-integer lookup tables and bases with random codes, so every ADC sum is exact; the result must equal the
numpy restatement in tests/ivfpq_filtered_ref.py under np.array_equal, for both code widths in both table modes (whole
table: 8-bit m = 96, 4-bit m = 128; chunked: 8-bit m = 192, 4-bit m = 288), across the 256-query block, with shared
and per-query bitmaps at the exact and a padded pitch, n not a multiple of 32 with the bits past n set, and the tile-group
split of one query's long lists.

Index: a shared filter must equal the unfiltered search of a copy with the disallowed documents removed, and a per-query
filter row q the one-query search with that row; with deletions, after add(), after save/load, with id_base > 0 and
across the Python block of 1024 queries.  Refine re-ranks only allowed candidates."""
import functools

import numpy as np
import pytest
import torch

from tests import ivfpq_filtered_ref as ref
from tests.helpers import planted_corpus

pytestmark = pytest.mark.gpu

SIZES = [0, 1, 256, 257, 1500, 0, 5, 1, 700, 37, 0, 230, 2, 13]  # n = 3002: not a multiple of 32
ID_BASE = 1000
MODES = [(8, 96), (8, 192), (4, 128), (4, 288)]  # (nbits, m): whole table, chunked, for each width
MODE_IDS = ["8bit-whole", "8bit-chunked", "4bit-whole", "4bit-chunked"]


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


@functools.lru_cache(maxsize=None)
def _case(nbits, m, nq, seed, sizes=tuple(SIZES), nprobe=5):
    """Integer tables, random codes, a shuffled id layout with a few negative doc_ids, distinct probes (some skipped)
    and the restated ADC scores [nq, n] (host arrays)."""
    from sgpt_b200.ivfpq import _pack_codes

    g = torch.Generator().manual_seed(seed)
    offsets = torch.zeros(len(sizes) + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.tensor(sizes, dtype=torch.int64), 0)
    n, nlist = int(offsets[-1]), len(sizes)
    ids = (torch.randperm(n, generator=g) + ID_BASE).to(torch.int32)
    ids[::97] = -1
    lut = torch.randint(-8, 9, (nq, m, 1 << nbits), generator=g).float()
    base = torch.randint(-20, 21, (nq, nprobe), generator=g).float()
    codes = _pack_codes(torch.randint(0, 1 << nbits, (n, m), generator=g), nbits)
    probes = torch.stack([torch.randperm(nlist, generator=g)[:nprobe] for _ in range(nq)]).to(torch.int32)
    probes[::5, 0] = -1
    sc = ref.adc_scores(lut.numpy(), base.numpy(), codes.numpy(), nbits, offsets.numpy(), probes.numpy())
    return lut, base, codes, offsets, ids, probes, sc


def _call(case, k, mask=None, pitch=0, nbits=8, masked=True):
    """sgpt_ivfpq_search_masked (or, masked=False, sgpt_ivfpq_search_nbits with the shared mask) into outputs prefilled
    with NaN / a sentinel: host (scores, ids)."""
    L, lib = _lib()
    lut, base, codes, offsets, ids, probes = case[:6]
    nq, nprobe = probes.shape
    nlist, n = offsets.numel() - 1, codes.shape[0]
    m = lut.shape[1]
    max_len = int((offsets[1:] - offsets[:-1]).max())
    d = [t.cuda().contiguous() for t in (lut, base, codes, offsets, ids, probes)]
    md = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask).view(np.int32)).cuda()
    need = lib.sgpt_ivfpq_search_workspace_bytes(nq, nlist, nprobe, max_len, m)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    s = torch.full((nq, k), float("nan"), device="cuda")
    i = torch.full((nq, k), -7, dtype=torch.int64, device="cuda")
    args = (d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), nq, n, m, nbits, d[3].data_ptr(), nlist, max_len,
            d[4].data_ptr(), d[5].data_ptr(), nprobe, k, L.ptr(md))
    tail = (s.data_ptr(), i.data_ptr(), ws.data_ptr(), ws.numel(), L.current_stream())
    if masked:
        L.check(lib.sgpt_ivfpq_search_masked(*args, pitch, *tail), "sgpt_ivfpq_search_masked")
    else:
        assert pitch == 0
        L.check(lib.sgpt_ivfpq_search_nbits(*args, *tail), "sgpt_ivfpq_search_nbits")
    return s.cpu().numpy(), i.cpu().numpy()


def _bitmaps(nq, n, pitch, share, seed):
    """Random per-query bitmaps uint32 [nq, pitch] (pitch >= ceil(n / 32)) with every bit at or past n set, and the bool
    [nq, n] they allow."""
    allow = np.random.default_rng(seed).random((nq, n)) < share
    bits = np.ones((nq, pitch * 32), dtype=np.uint64)
    bits[:, :n] = allow
    words = (bits.reshape(nq, pitch, 32) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32)
    return words, allow


def _assert_equal(what, got, want):
    """Ids and score bits equal."""
    (s, i), (ws_, wi) = got, want
    diff = (i != wi) | (s.view(np.uint32) != ws_.view(np.uint32))
    if diff.any():
        q, j = np.argwhere(diff)[0]
        raise AssertionError(f"{what}: query {q} rank {j}: got ({s[q, j]}, {i[q, j]}), want ({ws_[q, j]}, {wi[q, j]}); "
                             f"{int(diff.any(1).sum())} of {s.shape[0]} queries differ")


# ---- kernel --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nbits,m", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("nq", [1, 7, 256, 300])
@pytest.mark.parametrize("k", [1, 10, 1001])
def test_per_query_bitmaps_equal_the_restatement(nbits, m, nq, k):
    case = _case(nbits, m, nq, seed=nbits * 1000 + m + nq)
    n = case[2].shape[0]
    W = (n + 31) // 32
    words, allow = _bitmaps(nq, n, W, 0.4, seed=nq * 7 + k)
    got = _call(case, k, words, W, nbits)
    _assert_equal(f"nbits={nbits} m={m} nq={nq} k={k}", got, ref.search(case[6], case[4].numpy(), allow, k))


@pytest.mark.parametrize("nbits,m", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("form", ["shared", "exact", "padded"])
def test_every_pitch_equals_the_restatement(nbits, m, form):
    """Pitch 0 (one bitmap), ceil(n / 32) and ceil(n / 32) + 5 whose padding words are all ones; 300 queries."""
    nq, k = 300, 100
    case = _case(nbits, m, nq, seed=nbits * 1000 + m + nq)
    n = case[2].shape[0]
    W = (n + 31) // 32
    pitch = {"shared": 0, "exact": W, "padded": W + 5}[form]
    words, allow = _bitmaps(1 if pitch == 0 else nq, n, max(pitch, W), 0.3, seed=len(form))
    if pitch == 0:
        allow = np.repeat(allow, nq, axis=0)
    assert np.array_equal(ref.allowed(words, pitch, nq, n), allow)
    got = _call(case, k, words, pitch, nbits)
    _assert_equal(f"nbits={nbits} m={m} {form}", got, ref.search(case[6], case[4].numpy(), allow, k))


@pytest.mark.parametrize("nbits,m", MODES, ids=MODE_IDS)
def test_tile_groups_of_one_query_with_a_per_query_bitmap(nbits, m):
    """One query, two probes of lists of 40 and 23 tiles of 256 documents: the scan splits each list over many CTAs,
    each of which reads the query's bitmap."""
    sizes = (10240, 3, 5877, 1, 300)
    case = _case(nbits, m, 1, seed=77 + m, sizes=sizes, nprobe=2)
    lut, base, codes, offsets, ids, _, _ = case
    probes = torch.tensor([[2, 0]], dtype=torch.int32)
    sc = ref.adc_scores(lut.numpy(), base.numpy(), codes.numpy(), nbits, offsets.numpy(), probes.numpy())
    case = (lut, base, codes, offsets, ids, probes, sc)
    n = codes.shape[0]
    W = (n + 31) // 32
    for share in (0.5, 0.01):
        words, allow = _bitmaps(1, n, W + 1, share, seed=int(share * 100))
        for k in (10, 1001):
            got = _call(case, k, words, W + 1, nbits)
            _assert_equal(f"tile groups share={share} k={k}", got, ref.search(sc, ids.numpy(), allow, k))


@pytest.mark.parametrize("nbits,m", MODES, ids=MODE_IDS)
def test_equivalences(nbits, m):
    """All-ones per-query bitmaps equal the unmasked call; row q of a per-query call equals a one-query call with that
    row shared; an all-zero bitmap gives the empty tail; a second launch gives the same bits."""
    nq, k = 300, 64
    case = _case(nbits, m, nq, seed=nbits * 1000 + m + nq)
    n = case[2].shape[0]
    W = (n + 31) // 32
    plain = _call(case, k, nbits=nbits, masked=False)
    ones = np.full((nq, W + 2), 0xFFFFFFFF, dtype=np.uint32)
    _assert_equal("all ones", _call(case, k, ones, W + 2, nbits), plain)
    _assert_equal("null mask", _call(case, k, None, 0, nbits), plain)
    words, allow = _bitmaps(nq, n, W, 0.2, seed=5)
    got = _call(case, k, words, W, nbits)
    for q in (0, 1, 255, 256, 299):
        one = (case[0][q:q + 1], case[1][q:q + 1]) + case[2:5] + (case[5][q:q + 1],)
        row = _call(one, k, words[q], 0, nbits)
        _assert_equal(f"row {q}", (got[0][q:q + 1], got[1][q:q + 1]), row)
        shared_old = _call(one, k, words[q], 0, nbits, masked=False)
        _assert_equal(f"row {q} through sgpt_ivfpq_search_nbits", row, shared_old)
    zero = np.zeros((nq, W), dtype=np.uint32)
    s, i = _call(case, k, zero, W, nbits)
    assert (i == -1).all() and (s == -np.inf).all()
    again = _call(case, k, words, W, nbits)
    assert np.array_equal(got[0].view(np.uint32), again[0].view(np.uint32)) and np.array_equal(got[1], again[1])


# ---- IVFPQIndex ----------------------------------------------------------------------------------------------------
N, DIM, NQ, NLIST = 8000, 64, 150, 32
INDEXES = [("bf16", "cos_sim", 8), ("int8", "cos_sim", 4), ("bf16", "dot", 4), ("int8", "dot", 8)]


@pytest.fixture(scope="module", params=INDEXES, ids=[f"{d}-{s}-{b}bit" for d, s, b in INDEXES])
def saved(request, tmp_path_factory):
    """(source shard, saved index directory, queries, score function): every test loads its own copy."""
    from sgpt_b200 import CorpusShard, IVFPQIndex

    dtype, sf, nbits = request.param
    q, c = planted_corpus(N, DIM, NQ, seed=4)
    src = CorpusShard.from_embeddings(c.cuda(), dtype=dtype, id_base=500)
    index = IVFPQIndex.build(src, NLIST, 16 if nbits == 8 else 32, score_function=sf, n_iter=3, seed=2, nbits=nbits)
    path = str(tmp_path_factory.mktemp("ivfpq") / "index")
    index.save(path)
    return src, path, q.cuda(), sf


def _load(path):
    from sgpt_b200 import IVFPQIndex

    return IVFPQIndex.load(path, device="cuda:0")


def _same(what, a, b):
    assert torch.equal(a[1], b[1]), what
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)), what


def _allow(n, share, seed, rows=None):
    g = torch.Generator().manual_seed(seed)
    shape = (n,) if rows is None else (rows, n)
    return (torch.rand(shape, generator=g) < share).cuda()


@pytest.mark.parametrize("share", [0.5, 0.05])
def test_shared_filter_equals_removing_the_disallowed(saved, share):
    src, path, q, sf = saved
    index, copy = _load(path), _load(path)
    removed = torch.arange(500, 500 + N, 17, device="cuda")
    index.remove(removed)
    copy.remove(removed)
    a = _allow(N, share, seed=int(share * 100))
    copy.remove((~a).nonzero().flatten() + 500)
    for nprobe, k in ((4, 10), (NLIST, 100)):
        got = index.search(q, k, nprobe, allow=a)
        _same(f"nprobe={nprobe} k={k}", got, copy.search(q, k, nprobe))
        assert not torch.isin(got[1], (~a).nonzero().flatten() + 500).any()
        assert not torch.isin(got[1], removed).any()


def test_per_query_rows_equal_one_query_searches_across_blocks(saved):
    """1100 queries: with 8-bit codes two Python blocks of 1024, each packing its own rows of the filter."""
    src, path, q, sf = saved
    index = _load(path)
    index.remove(torch.arange(503, 500 + N, 29, device="cuda"))
    qq = q[torch.arange(1100, device="cuda") % NQ]
    a = _allow(N, 0.3, seed=1, rows=1100)
    got = index.search(qq, 20, 6, allow=a)
    for r in (0, 1, 1023, 1024, 1099):
        _same(f"row {r}", (got[0][r:r + 1], got[1][r:r + 1]), index.search(qq[r:r + 1], 20, 6, allow=a[r]))
    # all-ones rows are the unfiltered search
    _same("all ones", index.search(qq, 20, 6, allow=torch.ones(1100, N, dtype=torch.bool, device="cuda")),
          index.search(qq, 20, 6))


def test_filter_after_add_and_after_save_load(saved, tmp_path):
    src, path, q, sf = saved
    index, copy = _load(path), _load(path)
    extra = torch.randn(1500, DIM, generator=torch.Generator().manual_seed(3)).cuda()
    index.add(extra)
    copy.add(extra)
    n = N + 1500
    a = _allow(n, 0.4, seed=7)
    a[N:N + 700] = True
    copy.remove((~a).nonzero().flatten() + 500)
    got = index.search(q, 30, 8, allow=a)
    _same("after add", got, copy.search(q, 30, 8))
    index.save(str(tmp_path / "grown"))
    back = _load(str(tmp_path / "grown"))
    _same("after save/load", back.search(q, 30, 8, allow=a), got)
    rows = _allow(n, 0.4, seed=8, rows=NQ)
    _same("per query after save/load", back.search(q, 30, 8, allow=rows), index.search(q, 30, 8, allow=rows))


def test_refine_reranks_only_allowed_candidates(saved):
    from sgpt_b200.ivfpq import rerank

    src, path, q, sf = saved
    index = _load(path)
    for a in (_allow(N, 0.2, seed=11), _allow(N, 0.2, seed=12, rows=NQ)):
        got = index.search(q, 10, 8, refine=src, k_refine=100, allow=a)
        cand = index.search(q, 100, 8, allow=a)[1]
        _same("refine", got, rerank(src, q, cand, 10, sf))
        disallowed = ~a if a.dim() == 2 else (~a).expand(NQ, N)
        bad = torch.stack([torch.isin(got[1][r], disallowed[r].nonzero().flatten() + 500).any() for r in range(NQ)])
        assert not bad.any()


def test_refine_over_every_allowed_document_equals_the_exact_filtered_search(saved):
    """Every list probed and k_refine above the allowed count: the refined result is the exact search over the allowed
    documents.  Bit for bit on int8 shards (sgpt_rerank's score is the exact search's there)."""
    src, path, q, sf = saved
    if src.dtype != "int8":
        pytest.skip("sgpt_rerank equals the exact search's bits on int8 shards (bf16: within fp32 rounding)")
    index = _load(path)
    for a in (_allow(N, 0.03, seed=21), _allow(N, 0.03, seed=22, rows=NQ)):
        assert int(a.sum(-1).max()) <= 4096
        got = index.search(q, 50, NLIST, refine=src, k_refine=4096, allow=a)
        _same("exact filtered", got, src.search(q, 50, sf, allow=a))
