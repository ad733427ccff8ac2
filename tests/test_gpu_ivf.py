"""The IVF search (sgpt_ivf_search, IVFIndex) bit for bit.

Entry point: queries and documents hold small integers (|x| <= 2, D = 64), exact in bf16 and int8, so every dot product is
an exact integer and the scales are powers of two: each device score equals the fp64 reference, and the result must equal
the exact top-k over the probed documents (tests/helpers.py topk_reference: score descending, ties by ascending GLOBAL
id) under torch.equal.  The list layouts are made by hand: empty lists, one-document lists, lists of exactly 256 and 257
documents, a list spanning many tiles and badly unbalanced sizes; global ids are a shuffled range, so list order, position
order and id order all differ.

IVFIndex: continuous planted data; the search must equal CorpusShard.search restricted (allow=) to the probed documents
of the source shard, bit for bit."""
import math

import pytest
import torch

from tests.helpers import planted_corpus, topk_reference

pytestmark = pytest.mark.gpu

D = 64
SIZES = [0, 1, 256, 257, 3000, 0, 5, 1, 700, 37, 0, 1200, 2, 513]  # hand-made lists (6 + 4 + 1 ... tiles)
ID_BASE = 1000


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _layout(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    offsets = torch.zeros(len(sizes) + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.tensor(sizes, dtype=torch.int64), 0)
    n = int(offsets[-1])
    ids = (torch.randperm(n, generator=g) + ID_BASE).to(torch.int32)
    return offsets, ids


def _probes(nq, nlist, nprobe, g, skipped=True):
    """Distinct random probes per query; with `skipped`, about one query in five has one entry out of range."""
    p = torch.stack([torch.randperm(nlist, generator=g)[:nprobe] for _ in range(nq)]).to(torch.int32)
    if skipped:
        for q in range(0, nq, 5):
            p[q, int(torch.randint(nprobe, (1,), generator=g))] = -1 if q % 2 else nlist + 3
    return p


def _ivf(dtype, Q, C, q_scale, c_scale, offsets, ids, probes, k, mask=None):
    L, lib = _lib()
    nq, nprobe = probes.shape
    D = Q.shape[1]
    nlist = offsets.numel() - 1
    max_len = int((offsets[1:] - offsets[:-1]).max())
    dt = L.DTYPE_I8 if dtype == "int8" else L.DTYPE_BF16
    Qd = Q.to(torch.int8 if dtype == "int8" else torch.bfloat16).cuda()
    Cd = C.to(torch.int8 if dtype == "int8" else torch.bfloat16).cuda()
    qs = None if q_scale is None else q_scale.cuda()
    cs = None if c_scale is None else c_scale.cuda()
    off, idd, pr = offsets.cuda(), ids.cuda(), probes.cuda()
    m = None if mask is None else mask.cuda()
    need = lib.sgpt_ivf_search_workspace_bytes(dt, nq, nlist, nprobe, max_len, D)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_ivf_search(dt, Qd.data_ptr(), Cd.data_ptr(), L.ptr(qs), L.ptr(cs), nq, C.shape[0], D,
                                off.data_ptr(), nlist, max_len, idd.data_ptr(), pr.data_ptr(), nprobe, k, L.ptr(m),
                                s.data_ptr(), i.data_ptr(), ws.data_ptr(), ws.numel(), L.current_stream()),
            "sgpt_ivf_search")
    return s.cpu(), i.cpu()


def _reference(Q, C, q_scale, c_scale, offsets, ids, probes, k, deleted=None):
    sc = Q.double() @ C.double().T
    if q_scale is not None:
        sc = sc * q_scale.double()[:, None]
    if c_scale is not None:
        sc = sc * c_scale.double()[None, :]
    sc = torch.nan_to_num(sc, nan=-1.0, posinf=math.inf, neginf=-math.inf)
    nq, n = sc.shape
    nlist = offsets.numel() - 1
    list_of = torch.repeat_interleave(torch.arange(nlist), offsets[1:] - offsets[:-1])  # list of each position
    probed = torch.zeros(nq, nlist + 1, dtype=torch.bool)
    p = probes.long().clone()
    p[(p < 0) | (p >= nlist)] = nlist  # skipped
    probed.scatter_(1, p, True)
    keep = probed[:, :nlist].gather(1, list_of.expand(nq, n))
    if deleted is not None:
        keep &= ~deleted
    gid = torch.where(keep, ids.long().expand(nq, n), torch.full((nq, n), -1, dtype=torch.int64))
    return topk_reference(sc, gid, k)


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


def _data(nq, g, sizes=SIZES, D=D):
    offsets, ids = _layout(sizes, int(torch.randint(1 << 30, (1,), generator=g)))
    n = int(offsets[-1])
    return _ints((nq, D), -2, 2, g), _ints((n, D), -2, 2, g), offsets, ids


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("nq", [1, 7, 128, 129, 300])
@pytest.mark.parametrize("k", [1, 10, 1001, 4096])
@pytest.mark.parametrize("nprobe", [1, 3, len(SIZES)])
def test_ivf_entry_point_equals_exact_topk_of_probed_lists(dtype, nq, k, nprobe):
    g = torch.Generator().manual_seed(nq * 7919 + k * 31 + nprobe)
    Q, C, offsets, ids = _data(nq, g)
    probes = _probes(nq, len(SIZES), nprobe, g)
    got = _ivf(dtype, Q, C, None, None, offsets, ids, probes, k)
    _equal(f"{dtype} nq={nq} k={k} nprobe={nprobe}", got, _reference(Q, C, None, None, offsets, ids, probes, k))


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_ivf_scales_nan_rows_and_a_second_launch(dtype):
    """Power-of-two query and document scales (exact), a NaN document scale (score -1), and identical bits from a
    second launch."""
    g = torch.Generator().manual_seed(5)
    nq, k = 129, 1001
    Q, C, offsets, ids = _data(nq, g)
    n = C.shape[0]
    q_scale = 2.0 ** _ints((nq,), -2, 2, g)
    c_scale = 2.0 ** _ints((n,), -3, 1, g)
    c_scale[::97] = float("nan")
    probes = _probes(nq, len(SIZES), 4, g)
    got = _ivf(dtype, Q, C, q_scale, c_scale, offsets, ids, probes, k)
    _equal(dtype, got, _reference(Q, C, q_scale, c_scale, offsets, ids, probes, k))
    again = _ivf(dtype, Q, C, q_scale, c_scale, offsets, ids, probes, k)
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1])


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("frac", [0.0, 0.3, 1.0])
def test_ivf_deletions_never_appear(dtype, frac):
    from sgpt_b200.index import pack_mask

    g = torch.Generator().manual_seed(int(frac * 10) + 1)
    nq, k = 64, 300
    Q, C, offsets, ids = _data(nq, g)
    n = C.shape[0]
    deleted = torch.rand(n, generator=g) < frac
    deleted[int(offsets[4]):int(offsets[5])] = True  # the long list entirely
    probes = _probes(nq, len(SIZES), 5, g)
    got = _ivf(dtype, Q, C, None, None, offsets, ids, probes, k, mask=pack_mask(~deleted))
    want = _reference(Q, C, None, None, offsets, ids, probes, k, deleted=deleted)
    _equal(f"{dtype} deleted {frac}", got, want)
    assert not torch.isin(got[1], ids[deleted].long()).any()


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_ivf_fewer_probed_documents_than_k(dtype):
    """Tails of (-inf, -1): single small lists, every probe skipped, and probes of empty lists only."""
    g = torch.Generator().manual_seed(3)
    nq = 9
    Q, C, offsets, ids = _data(nq, g)
    probes = torch.tensor([[6, 7], [1, 12], [0, 5], [-1, 99], [10, 0], [7, -4], [12, 1], [6, 10], [5, 0]],
                          dtype=torch.int32)
    got = _ivf(dtype, Q, C, None, None, offsets, ids, probes, 10)
    want = _reference(Q, C, None, None, offsets, ids, probes, 10)
    _equal(dtype, got, want)
    assert (got[1][3] == -1).all() and (got[0][3] == -math.inf).all()


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_ivf_unbalanced_lists(dtype):
    """One list holds almost everything, many hold one or no document; every query probes the big list."""
    g = torch.Generator().manual_seed(11)
    sizes = [9000] + [1, 0, 2] * 30
    nq, k = 200, 1001
    Q, C, offsets, ids = _data(nq, g, sizes)
    probes = _probes(nq, len(sizes), 8, g, skipped=False)
    probes[:, 0] = 0
    probes[:, 1:] = torch.where(probes[:, 1:] == 0, torch.full_like(probes[:, 1:], -1), probes[:, 1:])
    _equal(dtype, _ivf(dtype, Q, C, None, None, offsets, ids, probes, k),
           _reference(Q, C, None, None, offsets, ids, probes, k))


# ---- IVFIndex on continuous data ---------------------------------------------------------------------------------
N, DIM, NQ, NLIST = 20000, 64, 150, 48


def _planted():
    return planted_corpus(N, DIM, NQ, seed=1)


def _probed_allow(index, probes):
    """allow [Q, n] over the SOURCE shard's documents: those in a probed list."""
    pos = index._pos.cpu()  # global id - id_base -> position
    list_of_pos = torch.searchsorted(index.offsets.cpu(), torch.arange(index.n), right=True) - 1
    list_of_doc = list_of_pos[pos]
    probed = torch.zeros(probes.shape[0], index.nlist, dtype=torch.bool)
    probed.scatter_(1, probes.long().cpu(), True)
    return probed.gather(1, list_of_doc.expand(probes.shape[0], -1)).cuda()


@pytest.fixture(scope="module", params=[("bf16", "cos_sim"), ("int8", "cos_sim"), ("bf16", "dot")],
                ids=["bf16-cos", "int8-cos", "bf16-dot"])
def built(request):
    from sgpt_b200 import CorpusShard, IVFIndex

    dtype, sf = request.param
    q, c = _planted()
    src = CorpusShard.from_embeddings(c.cuda(), dtype=dtype, id_base=500)
    index = IVFIndex.build(src, NLIST, score_function=sf, n_iter=6, seed=3)
    return src, index, q.cuda(), sf


@pytest.mark.parametrize("nprobe", [1, 4, 17])
@pytest.mark.parametrize("k", [10, 100])
def test_index_search_equals_exact_search_of_probed_documents(built, nprobe, k):
    src, index, q, sf = built
    got = index.search(q, k, nprobe)
    probes = index.probe(q, nprobe)
    want = src.search(q, k, sf, allow=_probed_allow(index, probes))
    assert torch.equal(got[1], want[1]) and torch.equal(got[0], want[0])


def test_index_full_probe_equals_unmasked_exact_search(built):
    src, index, q, sf = built
    got = index.search(q, 100, NLIST)
    want = src.search(q, 100, sf)
    assert torch.equal(got[1], want[1]) and torch.equal(got[0], want[0])


def test_index_scores_grow_with_nprobe(built):
    src, index, q, sf = built
    prev = None
    for nprobe in (1, 2, 3, 5, 8, 13, NLIST):
        s, _ = index.search(q, 50, nprobe)
        if prev is not None:
            assert (s >= prev).all(), nprobe
        prev = s


def test_index_build_is_reproducible_and_lists_cover_the_corpus(built):
    from sgpt_b200 import IVFIndex

    src, index, q, sf = built
    again = IVFIndex.build(src, NLIST, score_function=sf, n_iter=6, seed=3)
    assert torch.equal(index.centroids, again.centroids)
    assert torch.equal(index.offsets, again.offsets) and torch.equal(index.ids, again.ids)
    assert int(index.list_sizes.sum()) == N and index.list_sizes.numel() == NLIST
    assert torch.equal(torch.sort(index.ids.long()).values, torch.arange(N, device="cuda") + 500)


def test_index_save_load_round_trip(built, tmp_path):
    from sgpt_b200 import IVFIndex

    src, index, q, sf = built
    index.save(str(tmp_path / "ivf"))
    back = IVFIndex.load(str(tmp_path / "ivf"), device="cuda:0")
    for nprobe in (1, 6):
        a, b = index.search(q, 64, nprobe), back.search(q, 64, nprobe)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_index_remove_and_source_deletions():
    from sgpt_b200 import CorpusShard, IVFIndex

    q, c = _planted()
    q = q.cuda()
    src = CorpusShard.from_embeddings(c.cuda(), dtype="int8", id_base=7)
    src.remove(torch.arange(7, 7 + N, 13))  # deletions of the source carry over
    index = IVFIndex.build(src, NLIST, n_iter=4, seed=0)
    assert index.n_deleted == src.n_deleted
    top = index.search(q, 10, 6)[1]
    gone = torch.unique(top[:, :3].flatten())
    index.remove(gone)
    src.remove(gone)
    got = index.search(q, 10, 6)
    assert not torch.isin(got[1], gone).any()
    want = src.search(q, 10, "cos_sim", allow=_probed_allow(index, index.probe(q, 6)))
    assert torch.equal(got[1], want[1]) and torch.equal(got[0], want[0])
