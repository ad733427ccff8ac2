"""Filtered IVF search (sgpt_ivf_search_masked, IVFIndex.search(allow=)) and IVFIndex.add, bit for bit.

Entry point: the tie-heavy integer data and hand-made list layouts of test_gpu_ivf.py; the result must equal the fp64
top-k over the probed AND allowed positions under torch.equal, for a shared bitmap and one bitmap per query (pitch
ceil(n/32) and ceil(n/32) + 3, garbage in the bits past n and in the padding words).  Per-query rows differ across the
256-query block boundary, so a block that read the first block's bitmaps would fail.

IVFIndex: continuous planted data; search(allow=a) must equal CorpusShard.search(allow=a & probed), also after add()."""
import math

import pytest
import torch

from tests.test_gpu_ivf import SIZES, _data, _equal, _ints, _ivf, _planted, _probed_allow, _probes, _reference

pytestmark = pytest.mark.gpu


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _ivf_masked(dtype, Q, C, offsets, ids, probes, k, mask, pitch, q_scale=None, c_scale=None):
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
    m = None if mask is None else mask.cuda().contiguous()
    need = lib.sgpt_ivf_search_workspace_bytes(dt, nq, nlist, nprobe, max_len, D)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_ivf_search_masked(dt, Qd.data_ptr(), Cd.data_ptr(), L.ptr(qs), L.ptr(cs), nq, C.shape[0], D,
                                       off.data_ptr(), nlist, max_len, idd.data_ptr(), pr.data_ptr(), nprobe, k,
                                       L.ptr(m), pitch, s.data_ptr(), i.data_ptr(), ws.data_ptr(), ws.numel(),
                                       L.current_stream()),
            "sgpt_ivf_search_masked")
    return s.cpu(), i.cpu()


def _words(allowed, extra, g):
    """allowed bool [n] (shared, pitch 0) or [nq, n] (pitch ceil(n/32) + extra) -> (bitmap, pitch), with every bit past n
    set and the `extra` padding words random: none of them may matter."""
    from sgpt_b200.index import pack_mask

    n = allowed.shape[-1]
    w = pack_mask(allowed)
    if n % 32:
        w[..., -1] |= torch.tensor(-(1 << (n % 32)), dtype=torch.int32)  # bits n % 32 .. 31 of the last word
    if allowed.dim() == 1:
        return w, 0
    pad = torch.randint(-(1 << 31), 1 << 31, (allowed.shape[0], extra), generator=g, dtype=torch.int64).to(torch.int32)
    w = torch.cat([w, pad], 1)
    return w, w.shape[1]


DENSITIES = [0.01, 0.3, 1.0, 0.0, 0.9, 0.05]  # per query row, cycled (a random 1 % mask, all ones, all zeros, ...)


def _allowed(nq, n, per_query, g):
    if not per_query:
        return torch.rand(n, generator=g) < 0.4
    dens = torch.tensor([DENSITIES[(q * 5 + q // 7) % len(DENSITIES)] for q in range(nq)])
    return torch.rand(nq, n, generator=g) < dens[:, None]


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("nq", [1, 129, 300])
@pytest.mark.parametrize("k", [1, 1001, 4096])
@pytest.mark.parametrize("nprobe", [1, len(SIZES)])
@pytest.mark.parametrize("kind", ["shared", "pitch", "pitch+3"])
def test_ivf_masked_equals_exact_topk_of_probed_allowed_rows(dtype, nq, k, nprobe, kind):
    g = torch.Generator().manual_seed(nq * 7919 + k * 31 + nprobe * 3 + len(kind))
    Q, C, offsets, ids = _data(nq, g)
    n = C.shape[0]
    probes = _probes(nq, len(SIZES), nprobe, g)
    allowed = _allowed(nq, n, kind != "shared", g)
    mask, pitch = _words(allowed, 3 if kind == "pitch+3" else 0, g)
    got = _ivf_masked(dtype, Q, C, offsets, ids, probes, k, mask, pitch)
    want = _reference(Q, C, None, None, offsets, ids, probes, k, deleted=~allowed)
    _equal(f"{dtype} nq={nq} k={k} nprobe={nprobe} {kind}", got, want)


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("per_query", [False, True])
def test_ivf_masked_all_zero_masks_and_fewer_allowed_than_k(dtype, per_query):
    """Every row masked (the whole result is the (-inf, -1) tail), and masks that allow fewer than k probed rows."""
    g = torch.Generator().manual_seed(17 + per_query)
    nq, k = 40, 1001
    Q, C, offsets, ids = _data(nq, g)
    n = C.shape[0]
    probes = _probes(nq, len(SIZES), len(SIZES), g, skipped=False)
    for allowed in (torch.zeros(n, dtype=torch.bool), torch.rand(n, generator=g) < 0.05):
        if per_query:
            allowed = allowed.expand(nq, n).clone()
        mask, pitch = _words(allowed, 1, g)
        got = _ivf_masked(dtype, Q, C, offsets, ids, probes, k, mask, pitch)
        _equal(dtype, got, _reference(Q, C, None, None, offsets, ids, probes, k, deleted=~allowed))
        if not allowed.any():
            assert (got[1] == -1).all() and (got[0] == -math.inf).all()
        assert not torch.isin(got[1], ids[~allowed.reshape(-1, n)[0]].long()).any()


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("per_query", [False, True])
def test_ivf_masked_keeps_one_row_of_a_257_row_list(dtype, per_query):
    """Only one row of the 257-row list (list 3) is allowed; per query it is a different row, the last one included."""
    g = torch.Generator().manual_seed(23)
    nq, k = 7, 10
    Q, C, offsets, ids = _data(nq, g)
    n = C.shape[0]
    b = int(offsets[3])
    assert int(offsets[4]) - b == 257
    probes = torch.full((nq, 2), -1, dtype=torch.int32)
    probes[:, 0] = 3
    rows = [256, 0, 31, 32, 33, 255, 128]
    allowed = torch.zeros(nq, n, dtype=torch.bool)
    for q, r in enumerate(rows):
        allowed[q, b + (r if per_query else 256)] = True
    if not per_query:
        allowed = allowed[0]
    mask, pitch = _words(allowed, 2, g)
    got = _ivf_masked(dtype, Q, C, offsets, ids, probes, k, mask, pitch)
    _equal(dtype, got, _reference(Q, C, None, None, offsets, ids, probes, k, deleted=~allowed))
    for q, r in enumerate(rows):
        assert int(got[1][q, 0]) == int(ids[b + (r if per_query else 256)]) and (got[1][q, 1:] == -1).all()


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_ivf_masked_all_ones_is_bit_identical_to_the_unmasked_search(dtype):
    """NULL mask, all-ones shared and all-ones per-query bitmaps give sgpt_ivf_search's bits, with scales and NaN rows;
    per-query rows that are all equal give the shared-mask result; a second launch gives the same bits."""
    from sgpt_b200.index import pack_mask

    g = torch.Generator().manual_seed(29)
    nq, k = 300, 1001
    Q, C, offsets, ids = _data(nq, g)
    n = C.shape[0]
    q_scale = 2.0 ** _ints((nq,), -2, 2, g)
    c_scale = 2.0 ** _ints((n,), -3, 1, g)
    c_scale[::97] = float("nan")
    probes = _probes(nq, len(SIZES), 5, g)
    base = _ivf(dtype, Q, C, q_scale, c_scale, offsets, ids, probes, k)
    ones = torch.ones(n, dtype=torch.bool)
    for mask, pitch in ((None, 0), _words(ones, 0, g), _words(ones.expand(nq, n), 0, g), _words(ones.expand(nq, n), 5, g)):
        got = _ivf_masked(dtype, Q, C, offsets, ids, probes, k, mask, pitch, q_scale, c_scale)
        assert torch.equal(got[0], base[0]) and torch.equal(got[1], base[1]), pitch
    some = torch.rand(n, generator=g) < 0.5
    shared = _ivf(dtype, Q, C, q_scale, c_scale, offsets, ids, probes, k, mask=pack_mask(some))
    m, pitch = _words(some.expand(nq, n), 1, g)
    per_query = _ivf_masked(dtype, Q, C, offsets, ids, probes, k, m, pitch, q_scale, c_scale)
    assert torch.equal(per_query[0], shared[0]) and torch.equal(per_query[1], shared[1])
    again = _ivf_masked(dtype, Q, C, offsets, ids, probes, k, m, pitch, q_scale, c_scale)
    assert torch.equal(per_query[0], again[0]) and torch.equal(per_query[1], again[1])
    _equal(dtype, per_query, _reference(Q, C, q_scale, c_scale, offsets, ids, probes, k, deleted=~some))


# ---- IVFIndex ----------------------------------------------------------------------------------------------------
N, DIM, NQ, NLIST = 20000, 64, 150, 48
ADD = N // 4
FIXTURES = [("bf16", "cos_sim"), ("int8", "cos_sim"), ("bf16", "dot")]
FIXTURE_IDS = ["bf16-cos", "int8-cos", "bf16-dot"]


def _extra_rows(seed=7):
    """ADD more rows: fresh random rows and near-copies of existing documents (some land in every list)."""
    q, c = _planted()
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(ADD, DIM, generator=g)
    x[::3] = c[torch.randint(N, (len(x[::3]),), generator=g)] + 0.1 * x[::3]
    return x


def _source(dtype, id_base=500, extra=ADD):
    from sgpt_b200 import CorpusShard

    q, c = _planted()
    src = CorpusShard(DIM, N + extra, device="cuda:0", id_base=id_base, dtype=dtype)
    src.add(c.cuda())
    return src, q.cuda()


def _same(a, b):
    return torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.fixture(scope="module", params=FIXTURES, ids=FIXTURE_IDS)
def built(request):
    from sgpt_b200 import IVFIndex

    dtype, sf = request.param
    src, q = _source(dtype)
    return src, IVFIndex.build(src, NLIST, score_function=sf, n_iter=6, seed=3), q, sf


def _allow_rows(n, nq, seed):
    g = torch.Generator().manual_seed(seed)
    dens = torch.tensor([(0.01, 0.5, 1.0, 0.0, 0.2)[q % 5] for q in range(nq)])
    return (torch.rand(nq, n, generator=g) < dens[:, None]).cuda()


@pytest.mark.parametrize("nprobe", [1, 6, NLIST])
@pytest.mark.parametrize("k", [10, 100])
def test_index_search_allow_equals_exact_search_of_probed_allowed_documents(built, nprobe, k):
    src, index, q, sf = built
    probed = _probed_allow(index, index.probe(q, nprobe))
    shared = torch.rand(index.n, generator=torch.Generator().manual_seed(k)).cuda() < 0.5
    for allow in (shared, _allow_rows(index.n, q.shape[0], nprobe + k)):
        got = index.search(q, k, nprobe, allow=allow)
        assert _same(got, src.search(q, k, sf, allow=allow & probed))
    ones = torch.ones(index.n, dtype=torch.bool, device="cuda")
    assert _same(index.search(q, k, nprobe, allow=ones), index.search(q, k, nprobe))
    assert _same(index.search(q, k, nprobe, allow=ones.expand(q.shape[0], -1)), index.search(q, k, nprobe))


def test_index_search_rejects_bad_allow(built):
    src, index, q, sf = built
    n, nq = index.n, q.shape[0]
    for bad in (torch.ones(n + 1, dtype=torch.bool), torch.ones(nq + 1, n, dtype=torch.bool),
                torch.ones(n, dtype=torch.float32), torch.ones(nq, n, dtype=torch.int32), torch.ones(1, 1, n).bool()):
        with pytest.raises(ValueError, match="allow must be a boolean tensor"):
            index.search(q, 10, 4, allow=bad.cuda())


def test_index_allow_combines_with_remove():
    from sgpt_b200 import IVFIndex

    src, q = _source("int8", id_base=11)
    index = IVFIndex.build(src, NLIST, n_iter=4, seed=1)
    gone = torch.unique(index.search(q, 10, 6)[1][:, :2].flatten())
    index.remove(gone)
    src.remove(gone)
    probed = _probed_allow(index, index.probe(q, 6))
    for allow in (torch.rand(N).cuda() < 0.7, _allow_rows(N, q.shape[0], 5)):
        got = index.search(q, 10, 6, allow=allow)
        assert not torch.isin(got[1], gone).any()
        assert _same(got, src.search(q, 10, "cos_sim", allow=allow & probed))


# ---- add ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=FIXTURES, ids=FIXTURE_IDS)
def grown(request):
    """(src with the extra rows appended, the index before add (a saved copy), the index after add, queries, sf)."""
    from sgpt_b200 import IVFIndex

    dtype, sf = request.param
    src, q = _source(dtype)
    index = IVFIndex.build(src, NLIST, score_function=sf, n_iter=6, seed=3)
    before = (index.offsets.clone(), index.ids.clone())
    x = _extra_rows()
    index.add(x.cuda())
    src.add(x.cuda())
    return src, before, index, q, sf


@pytest.mark.parametrize("nprobe", [1, 6, NLIST])
def test_add_then_search_equals_exact_search_of_probed_documents(grown, nprobe):
    src, before, index, q, sf = grown
    assert index.n == N + ADD and src.n == N + ADD
    probed = _probed_allow(index, index.probe(q, nprobe))
    assert _same(index.search(q, 100, nprobe), src.search(q, 100, sf, allow=probed))
    allow = _allow_rows(index.n, q.shape[0], nprobe)
    assert _same(index.search(q, 100, nprobe, allow=allow), src.search(q, 100, sf, allow=allow & probed))


def test_add_layout(grown):
    """New rows sit in the list of their best centroid after the list's old rows, in input order; ids continue the
    range; the old rows keep their order; sizes, offsets and the id -> position map agree."""
    from sgpt_b200.ivf import _rows_f32

    src, (old_off, old_ids), index, q, sf = grown
    off, ids = index.offsets.cpu(), index.ids.cpu()
    old_off, old_ids = old_off.cpu(), old_ids.cpu()
    sizes = off[1:] - off[:-1]
    assert torch.equal(index.list_sizes, sizes) and index.max_list_len == int(sizes.max())
    assert int(off[0]) == 0 and int(off[-1]) == N + ADD
    assert torch.equal(torch.sort(ids.long()).values, torch.arange(N + ADD) + 500)
    assert torch.equal(index._pos.cpu()[ids.long() - 500], torch.arange(N + ADD))
    list_of_pos = torch.repeat_interleave(torch.arange(NLIST), sizes)
    new_pos = index._pos[torch.arange(N, N + ADD, device="cuda")]
    want = index.probe(_rows_f32(index.shard, new_pos), 1)[:, 0].long().cpu()
    assert torch.equal(list_of_pos[new_pos.cpu()], want)
    for l in range(NLIST):
        a, b, old = int(off[l]), int(off[l + 1]), int(old_off[l + 1] - old_off[l])
        assert torch.equal(ids[a:a + old], old_ids[int(old_off[l]):int(old_off[l + 1])]), l
        tail = ids[a + old:b].long()
        assert bool((tail >= 500 + N).all()) and bool((tail[1:] > tail[:-1]).all()), l  # input order


def test_add_survives_save_load(grown, tmp_path):
    from sgpt_b200 import IVFIndex

    src, before, index, q, sf = grown
    index.save(str(tmp_path / "ivf"))
    back = IVFIndex.load(str(tmp_path / "ivf"), device="cuda:0")
    assert torch.equal(back.offsets, index.offsets) and torch.equal(back.ids, index.ids)
    allow = _allow_rows(index.n, q.shape[0], 3)
    for nprobe in (1, 6):
        assert _same(index.search(q, 64, nprobe), back.search(q, 64, nprobe))
        assert _same(index.search(q, 64, nprobe, allow=allow), back.search(q, 64, nprobe, allow=allow))


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_add_with_removals_before_and_after(dtype):
    from sgpt_b200 import IVFIndex

    src, q = _source(dtype, id_base=3)
    index = IVFIndex.build(src, NLIST, n_iter=4, seed=2)
    early = torch.unique(index.search(q, 10, 6)[1][:, :2].flatten())
    index.remove(early)
    src.remove(early)
    x = _extra_rows(seed=9).cuda()
    index.add(x)
    src.add(x)
    assert index.n_deleted == src.n_deleted == early.numel()
    top = index.search(q, 10, 6)[1]
    late = torch.unique(top[top >= 3 + N])[:50]  # added documents
    assert late.numel() > 0
    index.remove(late)
    src.remove(late)
    assert index.n_deleted == src.n_deleted
    got = index.search(q, 10, 6)
    assert not torch.isin(got[1], torch.cat([early, late])).any()
    assert _same(got, src.search(q, 10, "cos_sim", allow=_probed_allow(index, index.probe(q, 6))))


def test_add_zero_rows_and_id_overflow_change_nothing():
    from sgpt_b200 import IVFIndex

    base = 2 ** 31 - N - 11  # room for 10 more ids: id_base + n must stay below 2^31
    src, q = _source("bf16", id_base=base)
    index = IVFIndex.build(src, NLIST, n_iter=3, seed=4)
    shard, offsets, ids = index.shard, index.offsets.clone(), index.ids.clone()
    want = index.search(q, 20, 5)

    def unchanged():
        assert index.n == N and index.shard is shard and shard.n == N
        assert torch.equal(index.offsets, offsets) and torch.equal(index.ids, ids)
        assert _same(index.search(q, 20, 5), want)

    index.add(torch.empty(0, DIM, device="cuda"))
    unchanged()
    with pytest.raises(ValueError, match="2\\^31"):
        index.add(torch.randn(11, DIM, device="cuda"))
    unchanged()
    index.add(torch.randn(10, DIM, device="cuda"))
    assert index.n == N + 10 and int(index.ids.max()) == 2 ** 31 - 2 and int(index.offsets[-1]) == N + 10
