"""The fused search (sgpt_search, sgpt_search_packed) bit for bit on integer data.

Queries and documents hold small integers (|x| <= 8), exact in bf16; with D = 64 every dot product and every partial sum
is an integer below 2^24, so the fp32 accumulation is exact in any order, and the scales are powers of two.  Every device
score then equals the fp64 reference, and the result must equal the exact top-k (tests/helpers.py topk_reference: score
descending, ties by ascending id) under torch.equal.  Integer data gives as many exact ties as wanted.

Which plan a shard takes follows csrc/search.cu make_plan: fewer than two 256-document tiles per SM -> dense scores plus
the selection kernel (cached in shared memory up to the limit of test_gpu_topk.cache_limit, uncached beyond); otherwise
the two-pass filter, whose pass A samples the tiles 0, s, 2s, ... with s = max(8, ceil(tiles / SMs)).  The plan is read
back from sgpt_search_workspace_bytes (the dense plan needs exactly nq x padded(n) x 4 + 256 bytes)."""
import math

import pytest
import torch

from tests.helpers import topk_reference
from tests.test_gpu_topk import cache_limit

pytestmark = pytest.mark.gpu

TILE = 256  # csrc/gemm_api.h kSimBN: documents per corpus tile
D = 64


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stride(n):
    tiles = -(-n // TILE)
    return max(8, -(-tiles // _sms()))


def two_pass_n(ragged):
    """A shard size on the two-pass plan whose last tile is sampled and holds `ragged` documents (0 = full)."""
    tiles = 2 * _sms() + 1
    while (tiles - 1) % _stride(tiles * TILE) != 0:
        tiles += 1
    return (tiles - 1) * TILE + (ragged or TILE)


def _plan(nq, n, k):
    _, lib = _lib()
    nb = min(nq, 256) if nq <= 256 else 256
    dense = lib.sgpt_search_workspace_bytes(nb, n, k) == nb * ((n + 3) // 4 * 4) * 4 + 256
    if not dense:
        return "two-pass"
    return "dense" if (n + 31) // 32 * 32 <= cache_limit(k) else "dense-uncached"


def _search(Q, C, k, id_base=0, q_scale=None, c_scale=None, packed=False):
    L, lib = _lib()
    nq, n, D = Q.shape[0], C.shape[0], Q.shape[1]
    ws = torch.empty(lib.sgpt_search_workspace_bytes(nq, n, k), dtype=torch.uint8, device="cuda")
    qs, cs = L.ptr(q_scale), L.ptr(c_scale)
    if packed:
        from sgpt_b200.index import unpack_topk

        out = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        L.check(lib.sgpt_search_packed(Q.data_ptr(), C.data_ptr(), qs, cs, nq, n, D, k, id_base, out.data_ptr(),
                                       ws.data_ptr(), ws.numel(), L.current_stream()), "sgpt_search_packed")
        s, i = unpack_topk(out.cpu())
        return s, i
    s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_search(Q.data_ptr(), C.data_ptr(), qs, cs, nq, n, D, k, id_base, s.data_ptr(), i.data_ptr(),
                            ws.data_ptr(), ws.numel(), L.current_stream()), "sgpt_search")
    return s.cpu(), i.cpu()


def _reference(Q, C, k, id_base=0, q_scale=None, c_scale=None, exclude=None):
    sc = Q.double().cpu() @ C.double().cpu().T
    if q_scale is not None:
        sc = sc * q_scale.double().cpu()[:, None]
    if c_scale is not None:
        sc = sc * c_scale.double().cpu()[None, :]
    sc = torch.nan_to_num(sc, nan=-1.0, posinf=math.inf, neginf=-math.inf)  # XS:99: NaN -> -1
    ids = torch.arange(C.shape[0], dtype=torch.int64).expand_as(sc) + id_base
    return topk_reference(sc, ids, k, exclude)


def _equal(what, got, want):
    s, i = got
    ws_, wi = want
    bad = ((i != wi) | (s.double() != ws_)).any(dim=1).nonzero()
    if len(bad):
        q = int(bad[0])
        j = int(((i[q] != wi[q]) | (s[q].double() != ws_[q])).nonzero()[0])
        raise AssertionError(f"{what}: query {q} rank {j}: got ({float(s[q, j])}, {int(i[q, j])}), want "
                             f"({float(ws_[q, j])}, {int(wi[q, j])}); {len(bad)} of {s.shape[0]} queries differ")


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g).float()


def planted_weights(D):
    """(a, b): queries carry a in coordinate 0 and the planted documents are (b, 0, ..., 0), so a planted document scores
    a * b >= D, strictly above the D - 1 that any other document of the k_sampled / k_unsampled corpora can reach.  Both
    are exact in bf16 and int8 up to D = 8128: (8, 8) at D <= 64, else a power of two a <= 64 with b = ceil(D / a)."""
    if D <= 64:
        return 8, 8
    a = min(64, 1 << math.ceil(math.log2(D) / 2))
    return a, -(-D // a)


def corpus(kind, nq, n, k, g, D=D):
    """(Q, C) fp32 with small-integer entries (NaN rows for 'nan_rows')."""
    if kind == "random":  # scores in a few hundred values: ties everywhere
        return _ints((nq, D), -2, 2, g), _ints((n, D), -2, 2, g)
    if kind == "identical":  # every document equal: the ids must be id_base .. id_base + k - 1
        return _ints((nq, D), -8, 8, g), _ints((1, D), -8, 8, g).expand(n, D).contiguous()
    if kind in ("k_sampled", "k_unsampled"):
        # every query: coordinate 0 = a, the others in {-1, 0, 1}.  Documents: coordinate 0 <= 0, others in {-1, 0, 1}
        # -> scores <= D - 1; k special documents (b, 0, ..., 0) score exactly a * b >= D (planted_weights), each in its
        # own 4-document block, inside the sampled tiles (then the admission threshold tau equals the k-th best score:
        # `x >= tau` decides at equality) or outside them
        a, b = planted_weights(D)
        Q = _ints((nq, D), -1, 1, g)
        Q[:, 0] = a
        C = _ints((n, D), -1, 1, g)
        C[:, 0] = _ints((n,), -8, 0, g)
        s = _stride(n)
        tiles = [t for t in range(-(-n // TILE)) if (t % s == 0) == (kind == "k_sampled")]
        blocks = [t * TILE + 4 * b + (t % 4) for t in tiles for b in range(TILE // 4) if t * TILE + 4 * b + 3 < n]
        assert len(blocks) >= k
        pick = torch.tensor(blocks)[torch.randperm(len(blocks), generator=g)[:k]]
        C[pick] = 0.0
        C[pick, 0] = float(b)
        return Q, C
    if kind == "negative":  # every score <= -1: zero-filled columns past n would score 0 and win if not masked
        return _ints((nq, D), 1, 3, g), _ints((n, D), -3, -1, g)
    if kind == "nan_rows":
        # queries: coordinate 0 = 1, the others in [1, 2]; documents score <= -2, except that every other document above
        # the NaN rows is (-1, 0, ..., 0) and scores exactly -1.  The NaN rows score -1 (XS:99) and have the lowest ids,
        # the cut falls inside the -1 group, so tau <= -1 and the NaN mapping of the filter decides the result
        Q = _ints((nq, D), 1, 2, g)
        Q[:, 0] = 1
        C = _ints((n, D), -2, -1, g)
        C[300::2] = 0.0
        C[300::2, 0] = -1.0
        C[:300:3] = float("nan")
        return Q, C
    raise ValueError(kind)


def _run_case(kind, nq, n, k, id_base, seed, scales=False, check_packed=True):
    g = torch.Generator().manual_seed(seed)
    Qf, Cf = corpus(kind, nq, n, k, g)
    Q, C = Qf.to(torch.bfloat16).cuda(), Cf.to(torch.bfloat16).cuda()
    qs = cs = None
    if scales:  # powers of two keep every score exact
        qs = (2.0 ** torch.randint(-1, 2, (nq,), generator=g).float()).cuda()
        cs = (2.0 ** torch.randint(-1, 3, (n,), generator=g).float()).cuda()
    want = _reference(Qf, Cf, k, id_base, qs, cs)
    what = f"{kind} nq={nq} n={n} k={k} id_base={id_base} ({_plan(nq, n, k)})"
    got = _search(Q, C, k, id_base, qs, cs)
    _equal(f"sgpt_search {what}", got, want)
    again = _search(Q, C, k, id_base, qs, cs)
    assert torch.equal(got[0].view(torch.int32), again[0].view(torch.int32)) and torch.equal(got[1], again[1]), \
        f"{what}: a second search returned different bits"
    if check_packed and id_base + n < 2 ** 31:
        _equal(f"sgpt_search_packed {what}", _search(Q, C, k, id_base, qs, cs, packed=True), want)
    return Q, C, qs, cs, want


def test_plans_are_the_intended_ones():
    assert _plan(37, 20000, 1001) == "dense"
    assert _plan(37, 60000, 1001) == "dense-uncached"
    assert _plan(37, two_pass_n(77), 1001) == "two-pass"
    assert _plan(300, two_pass_n(77), 1001) == "two-pass"


@pytest.mark.parametrize("kind", ["random", "identical", "negative"])
@pytest.mark.parametrize("n_name", ["dense", "dense-uncached", "two-pass"])
def test_search_plans_bit_exact(kind, n_name):
    """Every plan on tie-heavy integer corpora, with and without power-of-two scales; the dense plan also against
    sgpt_scores + sgpt_topk."""
    n = {"dense": 20000, "dense-uncached": 60000, "two-pass": two_pass_n(77)}[n_name]
    for j, (nq, k) in enumerate([(1, 1), (37, 10), (129, 1001), (37, 1025)]):
        Q, C, qs, cs, want = _run_case(kind, nq, n, k, id_base=(0, 7)[j % 2], seed=j, scales=j % 2 == 1)
        if n_name == "dense":
            L, lib = _lib()
            sc = torch.empty((nq, n), dtype=torch.float32, device="cuda")
            L.check(lib.sgpt_scores(Q.data_ptr(), C.data_ptr(), L.ptr(qs), L.ptr(cs), sc.data_ptr(), n, nq, n, D,
                                    L.current_stream()))
            s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
            i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
            ws = torch.empty(256, dtype=torch.uint8, device="cuda")
            L.check(lib.sgpt_topk(sc.data_ptr(), n, nq, n, k, (0, 7)[j % 2], s.data_ptr(), i.data_ptr(), ws.data_ptr(),
                                  L.current_stream()))
            _equal(f"sgpt_scores + sgpt_topk {kind} nq={nq} k={k}", (s.cpu(), i.cpu()), want)


@pytest.mark.parametrize("kind", ["k_sampled", "k_unsampled", "nan_rows", "negative"])
@pytest.mark.parametrize("k_hi", [None, "1", "k"])
@pytest.mark.parametrize("front", [None, "1"])
def test_two_pass_thresholds_bit_exact(kind, k_hi, front, monkeypatch):
    """The two-pass plan at its admission edges, under every split of its candidate lists: SGPT_SEARCH_K_HI unset, 1
    (front parts nearly empty: the back parts are read) or k (no split), and the front-list kernel (SGPT_FRONT_SELECT=1)
    off or on.  The last tile is ragged and sampled."""
    if front:
        monkeypatch.setenv("SGPT_FRONT_SELECT", front)
    n = two_pass_n(77)
    for j, (nq, k) in enumerate([(1, 1), (37, 10), (128, 1001), (257, 1025)]):
        if k_hi:
            monkeypatch.setenv("SGPT_SEARCH_K_HI", str(k) if k_hi == "k" else k_hi)
        assert _plan(nq, n, k) == "two-pass"
        _run_case(kind, nq, n, k, id_base=(0, 7, 2 ** 31 - 1 - n, 3)[j], seed=100 + j)


@pytest.mark.parametrize("nq", [1, 37, 128, 129, 256, 257, 300])
def test_query_blocks_bit_exact(nq):
    """CTA pairs above 128 queries, query blocks of 256 above 256; the packed output at the largest legal id_base."""
    n = two_pass_n(77)
    _run_case("random", nq, n, 1001, id_base=2 ** 31 - 1 - n, seed=nq)


@pytest.mark.parametrize("parts", [2, 4])
@pytest.mark.parametrize("n_name", ["dense", "two-pass"])
def test_shards_and_merge_equal_whole_search(parts, n_name):
    """Split the corpus into shards, search each, merge (fp32 lists and packed lists): bit for bit the whole-shard search.
    With exclude_ids: bit for bit the exact top k of the shards' lists without the excluded id (ties resolve to the lowest
    ids, so the replacement of an excluded entry may be a shard's (k+1)-th, which no list holds).  The same search through
    PeerGather at world size 1."""
    from sgpt_b200.dist import PeerGather
    from sgpt_b200.index import merge_topk, merge_topk_packed

    n = {"dense": 20000, "two-pass": 4 * two_pass_n(77)}[n_name]
    nq, k, id_base = 37, 1001, 5
    g = torch.Generator().manual_seed(parts)
    Qf, Cf = corpus("random", nq, n, k, g)
    Q, C = Qf.to(torch.bfloat16).cuda(), Cf.to(torch.bfloat16).cuda()
    whole = _search(Q, C, k, id_base)
    _equal("whole", whole, _reference(Qf, Cf, k, id_base))
    cuts = [n * p // parts for p in range(parts + 1)]
    res, packed = [], []
    for a, b in zip(cuts[:-1], cuts[1:]):
        res.append(_search(Q, C[a:b], k, id_base + a))
        s, i = res[-1]
        from tests.test_gpu_topk import pack

        packed.append(pack(s, i))
    S, I, P = torch.stack([r[0] for r in res]).cuda(), torch.stack([r[1] for r in res]).cuda(), torch.stack(packed).cuda()
    ex = whole[1][:, torch.arange(nq) % 5 * 200].diagonal().clone()  # an id at rank 0, 200, .., 800 of the whole result
    ex[::7] = -1
    ex[3] = 10 ** 9  # absent
    for exclude in (None, ex):
        want = whole if exclude is None else topk_reference(S.permute(1, 0, 2).reshape(nq, -1).cpu(),
                                                            I.permute(1, 0, 2).reshape(nq, -1).cpu(), k, exclude)
        exd = None if exclude is None else exclude.cuda()
        s, i = merge_topk(S, I, exd)
        _equal(f"merge_topk of {parts} shards exclude={exclude is not None}", (s.cpu(), i.cpu()), want)
        s, i = merge_topk_packed(P, exd)
        _equal(f"merge_topk_packed of {parts} shards exclude={exclude is not None}", (s.cpu(), i.cpu()), want)
    from sgpt_b200 import CorpusShard

    shard = CorpusShard.from_embeddings(C, device="cuda:0", id_base=id_base)
    pg = PeerGather(nq, k, "cuda:0")
    try:
        s, i = pg.search(shard, Q, k, "dot")
        _equal("PeerGather world 1", (s.cpu(), i.cpu()), whole)
    finally:
        pg.close()
