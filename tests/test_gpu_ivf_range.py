"""The IVF range search (sgpt_ivf_range_search, IVFIndex.range_search) and mining over an IVFIndex, bit for bit.

Entry point: the tie-heavy integer data and hand-made list layouts of tests/test_gpu_ivf.py, where every score is exact,
against an fp64 restatement of the contract in include/sgpt_b200.h: per query, its probes in the given order, each
probe's allowed, id >= 0 positions in list order with score >= threshold (NaN as -1), written at the running offset if
the query fits `cap`; the rest of the buffers keeps its sentinels.

IVFIndex: continuous planted data; the range search must equal CorpusShard.range_search(allow=allow & probed) of the
source shard under torch.equal.  Mining over an index: at nprobe = nlist, +-1 data where cos = dot / 64 is exact, it
equals the exact functions; at nprobe < nlist it equals a reference built from the exact masked searches of the inner
shard with per-query masks "probed & undeleted"."""
import math

import pytest
import torch

from tests.helpers import planted_corpus
from tests.test_gpu_ivf import SIZES, _data, _ints, _probed_allow, _probes

pytestmark = pytest.mark.gpu

D = 64
SENT_S, SENT_I = 12345.0, -99


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _ivf_range(dtype, Q, C, q_scale, c_scale, offsets, ids, probes, threshold, cap, mask=None, pitch=0):
    """(counts, scores, ids) of sgpt_ivf_range_search on sentinel-filled buffers; a second launch must give the same."""
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
    need = lib.sgpt_ivf_range_search_workspace_bytes(dt, nq, nlist, nprobe, max_len, D)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    counts = torch.full((nq,), -7, dtype=torch.int64, device="cuda")
    s = torch.full((max(cap, 1),), SENT_S, dtype=torch.float32, device="cuda")
    i = torch.full((max(cap, 1),), SENT_I, dtype=torch.int64, device="cuda")
    out = []
    for _ in range(2):
        L.check(lib.sgpt_ivf_range_search(dt, Qd.data_ptr(), Cd.data_ptr(), L.ptr(qs), L.ptr(cs), nq, C.shape[0], D,
                                          off.data_ptr(), nlist, max_len, idd.data_ptr(), pr.data_ptr(), nprobe,
                                          float(threshold), L.ptr(m), pitch, counts.data_ptr(), cap, s.data_ptr(),
                                          i.data_ptr(), ws.data_ptr(), ws.numel(), L.current_stream()),
                "sgpt_ivf_range_search")
        out.append((counts.cpu().clone(), s.cpu().clone(), i.cpu().clone()))
    assert all(torch.equal(a, b) for a, b in zip(out[0], out[1])), "second launch differs"
    return out[0]


def _scores(Q, C, q_scale, c_scale):
    sc = Q.double() @ C.double().T
    if q_scale is not None:
        sc = sc * q_scale.double()[:, None]
    if c_scale is not None:
        sc = sc * c_scale.double()[None, :]
    return torch.nan_to_num(sc, nan=-1.0, posinf=math.inf, neginf=-math.inf)


def _reference(sc, offsets, ids, probes, threshold, cap, allowed=None):
    """The contract: allowed bool [nq, n] over positions (None: all)."""
    nq, n = sc.shape
    nlist = offsets.numel() - 1
    counts = torch.zeros(nq, dtype=torch.int64)
    s = torch.full((max(cap, 1),), SENT_S, dtype=torch.float32)
    i = torch.full((max(cap, 1),), SENT_I, dtype=torch.int64)
    off = 0
    for q in range(nq):
        pos = [torch.arange(int(offsets[l]), int(offsets[l + 1])) for l in probes[q].tolist() if 0 <= l < nlist]
        pos = torch.cat(pos) if pos else torch.zeros(0, dtype=torch.int64)
        keep = (sc[q, pos] >= threshold) & (ids[pos] >= 0)
        if allowed is not None:
            keep &= allowed[q, pos]
        pos = pos[keep]
        c = pos.numel()
        counts[q] = c
        if off + c <= cap:
            s[off:off + c] = sc[q, pos].float()
            i[off:off + c] = ids[pos].long()
        off += c
    return counts, s, i


def _check(got, want, what):
    for name, a, b in zip(("counts", "scores", "ids"), got, want):
        if not torch.equal(a, b):
            bad = int((a != b).nonzero()[0][0])
            raise AssertionError(f"{what}: {name}[{bad}] = {a[bad].item()}, want {b[bad].item()}")


def _present_threshold(sc, offsets, probes):
    """A score that occurs among query 0's probed positions (the median one): documents exactly at it count."""
    nlist = offsets.numel() - 1
    pos = torch.cat([torch.arange(int(offsets[l]), int(offsets[l + 1])) for l in probes[0].tolist() if 0 <= l < nlist]
                    + [torch.zeros(1, dtype=torch.int64)])
    return float(torch.sort(sc[0, pos]).values[pos.numel() // 2])


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("nq", [1, 129, 300])
@pytest.mark.parametrize("nprobe", [1, 4, len(SIZES)])
@pytest.mark.parametrize("which", ["present", "-inf", "above"])
def test_ivf_range_entry_point_equals_contract(dtype, nq, nprobe, which):
    """Every list shape of SIZES (empty, 1, 256, 257, 3000 rows ...), skipped probes, nq across the 256-query block."""
    g = torch.Generator().manual_seed(nq * 131 + nprobe * 7 + len(which))
    Q, C, offsets, ids = _data(nq, g)
    probes = _probes(nq, len(SIZES), nprobe, g)
    sc = _scores(Q, C, None, None)
    t = {"present": _present_threshold(sc, offsets, probes), "-inf": -math.inf, "above": 1e9}[which]
    want = _reference(sc, offsets, ids, probes, t, 0)
    total = int(want[0].sum())
    got = _ivf_range(dtype, Q, C, None, None, offsets, ids, probes, t, total)
    _check(got, _reference(sc, offsets, ids, probes, t, total), f"{dtype} nq={nq} nprobe={nprobe} t={t}")
    if which == "above":
        assert total == 0


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_ivf_range_cap_cuts(dtype):
    """cap 0 (counts only), a cut inside the first query, inside a later query (past the 256-query block), exactly at a
    query's end, and one entry short of the total: the queries that fit are written, the rest keeps its sentinels."""
    g = torch.Generator().manual_seed(17)
    nq = 300
    Q, C, offsets, ids = _data(nq, g)
    probes = _probes(nq, len(SIZES), 3, g)
    sc = _scores(Q, C, None, None)
    t = _present_threshold(sc, offsets, probes)
    counts = _reference(sc, offsets, ids, probes, t, 0)[0]
    ends = torch.cumsum(counts, 0)
    first = int(torch.nonzero(counts > 1)[0])
    later = int(torch.nonzero((counts > 1) & (torch.arange(nq) > 260))[0])
    for cap in (0, int(ends[first]) - int(counts[first]) // 2, int(ends[later]) - 1, int(ends[200]), int(ends[-1]) - 1,
                int(ends[-1])):
        got = _ivf_range(dtype, Q, C, None, None, offsets, ids, probes, t, cap)
        _check(got, _reference(sc, offsets, ids, probes, t, cap), f"{dtype} cap={cap}")


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_ivf_range_scales_and_nan_rows(dtype):
    """Power-of-two scales (exact) and NaN document scales: a NaN score counts as -1, admitted at thresholds <= -1."""
    g = torch.Generator().manual_seed(5)
    nq = 129
    Q, C, offsets, ids = _data(nq, g)
    n = C.shape[0]
    q_scale = 2.0 ** _ints((nq,), -2, 2, g)
    c_scale = 2.0 ** _ints((n,), -3, 1, g)
    c_scale[::97] = float("nan")
    probes = _probes(nq, len(SIZES), 5, g)
    sc = _scores(Q, C, q_scale, c_scale)
    for t in (-1.0, -0.5, _present_threshold(sc, offsets, probes)):
        total = int(_reference(sc, offsets, ids, probes, t, 0)[0].sum())
        got = _ivf_range(dtype, Q, C, q_scale, c_scale, offsets, ids, probes, t, total)
        _check(got, _reference(sc, offsets, ids, probes, t, total), f"{dtype} t={t}")
        if t == -1.0:
            assert (got[1] == -1.0).any()


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("form", ["deleted", "shared", "per_query", "per_query_pad", "all_zero", "per_query_zero"])
def test_ivf_range_masks(dtype, form):
    """Deletions (a shared bitmap), shared and per-query filters (pitch ceil(n/32) and + 3, rows that differ across the
    256-query boundary), all-zero masks, and ids < 0 in doc_ids (never counted)."""
    from sgpt_b200.index import pack_mask

    g = torch.Generator().manual_seed(len(form) * 13 + (dtype == "int8"))
    nq = 300
    Q, C, offsets, ids = _data(nq, g)
    n = C.shape[0]
    ids = ids.clone()
    ids[::101] = -1
    probes = _probes(nq, len(SIZES), 4, g)
    sc = _scores(Q, C, None, None)
    t = _present_threshold(sc, offsets, probes)
    words = (n + 31) // 32
    if form in ("deleted", "shared", "all_zero"):
        allow = torch.rand(n, generator=g) < (0.0 if form == "all_zero" else 0.6 if form == "shared" else 0.8)
        mask, pitch, allowed = pack_mask(allow), 0, allow.expand(nq, n)
    else:
        allow = torch.rand(nq, n, generator=g) < 0.5
        if form == "per_query_zero":
            allow[::3] = False
        pitch = words + (3 if form == "per_query_pad" else 0)
        mask = torch.zeros(nq, pitch, dtype=torch.int32)
        mask[:, :words] = pack_mask(allow)
        if pitch > words:
            mask[:, words:] = -1  # garbage past the bitmap
        allowed = allow
    total = int(_reference(sc, offsets, ids, probes, t, 0, allowed)[0].sum())
    got = _ivf_range(dtype, Q, C, None, None, offsets, ids, probes, t, total, mask.contiguous(), pitch)
    _check(got, _reference(sc, offsets, ids, probes, t, total, allowed), f"{dtype} {form}")
    if form == "all_zero":
        assert int(got[0].sum()) == 0


# ---- IVFIndex.range_search on continuous data ----------------------------------------------------------------------
N, DIM, NQ, NLIST = 20000, 64, 150, 48


def _threshold(src, q, sf, rank):
    return float(src.search(q, rank + 1, sf)[0][:, rank].median())


@pytest.fixture(scope="module", params=[("bf16", "cos_sim"), ("int8", "cos_sim"), ("bf16", "dot")],
                ids=["bf16-cos", "int8-cos", "bf16-dot"])
def built(request):
    from sgpt_b200 import CorpusShard, IVFIndex

    dtype, sf = request.param
    q, c = planted_corpus(N, DIM, NQ, seed=2)
    src = CorpusShard.from_embeddings(c.cuda(), dtype=dtype, id_base=300)
    index = IVFIndex.build(src, NLIST, score_function=sf, n_iter=6, seed=1)
    return src, index, q.cuda(), sf


def _equal_csr(got, want, what):
    for name, a, b in zip(("offsets", "scores", "ids"), got, want):
        assert torch.equal(a, b), f"{what}: {name} differ"


@pytest.mark.parametrize("nprobe", [1, 5, NLIST])
@pytest.mark.parametrize("rank", [10, 400])
def test_index_range_search_equals_exact_range_search_of_probed_documents(built, nprobe, rank):
    """rank 400: about 400 documents per query at nprobe = nlist, past the 64 per query the buffer starts with, so
    the buffer grows once."""
    src, index, q, sf = built
    t = _threshold(src, q, sf, rank)
    got = index.range_search(q, t, nprobe)
    want = src.range_search(q, t, sf, allow=_probed_allow(index, index.probe(q, nprobe)))
    _equal_csr(got, want, f"nprobe={nprobe} rank={rank}")
    if nprobe == NLIST:
        _equal_csr(got, src.range_search(q, t, sf), "full probe")


@pytest.mark.parametrize("shape", ["shared", "per_query"])
def test_index_range_search_with_allow(built, shape):
    src, index, q, sf = built
    g = torch.Generator(device="cuda").manual_seed(4)
    allow = torch.rand((N,) if shape == "shared" else (NQ, N), generator=g, device="cuda") < 0.4
    t = _threshold(src, q, sf, 50)
    got = index.range_search(q, t, 6, allow=allow)
    want = src.range_search(q, t, sf, allow=allow & _probed_allow(index, index.probe(q, 6)))
    _equal_csr(got, want, shape)


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_index_range_search_after_remove_and_add(dtype):
    from sgpt_b200 import CorpusShard, IVFIndex

    q, c = planted_corpus(N, DIM, NQ, seed=3)
    q, c = q.cuda(), c.cuda()
    extra = c[:3000] + 0.05 * torch.randn(3000, DIM, generator=torch.Generator().manual_seed(1)).cuda()
    src = CorpusShard(DIM, N + 3000, device="cuda:0", dtype=dtype, id_base=11)
    src.add(c)
    index = IVFIndex.build(src, NLIST, n_iter=4, seed=0)
    t = _threshold(src, q, "cos_sim", 30)
    gone = torch.unique(index.range_search(q, t, 4)[2][::7])
    index.remove(gone)
    src.remove(gone)
    _equal_csr(index.range_search(q, t, 4), src.range_search(q, t, allow=_probed_allow(index, index.probe(q, 4))),
               "after remove")
    index.add(extra)
    src.add(extra)
    got = index.range_search(q, t, 4)
    _equal_csr(got, src.range_search(q, t, allow=_probed_allow(index, index.probe(q, 4))), "after add")
    assert not torch.isin(got[2], gone).any()
    assert (got[2] >= 11 + N).any()  # added documents are found


# ---- mining over an IVFIndex ---------------------------------------------------------------------------------------
def _pm_data(n=3000, clusters=100, flip=0.1, seed=0):
    """+-1 rows (cos = dot / 64, exact): noisy copies of cluster centres, so that both functions have work to do."""
    g = torch.Generator().manual_seed(seed)
    centres = torch.where(torch.rand(clusters, D, generator=g) < 0.5, -1.0, 1.0)
    x = centres[torch.randint(clusters, (n,), generator=g)]
    x = torch.where(torch.rand(n, D, generator=g) < flip, -x, x)
    return x.cuda()


def test_ivf_mining_at_full_probe_equals_exact_functions():
    from sgpt_b200 import IVFIndex, community_detection, paraphrase_mining_embeddings

    x = _pm_data()
    n = x.shape[0]
    index = IVFIndex.build(x, 16, n_iter=4, seed=0)
    for top_k, max_pairs in ((20, 2000), (5, 500000)):
        want = paraphrase_mining_embeddings(x, corpus_chunk_size=n, top_k=top_k, max_pairs=max_pairs)
        got = paraphrase_mining_embeddings(index, top_k=top_k, max_pairs=max_pairs, nprobe=16)
        assert got == want, top_k
    for threshold, size, init in ((0.5, 10, 25), (0.75, 3, 1000)):
        want = community_detection(x, threshold=threshold, min_community_size=size, init_max_size=init)
        got = community_detection(index, threshold=threshold, min_community_size=size, init_max_size=init, nprobe=16)
        assert len(want) > 0 and got == want, threshold


def _stored(index, keep):
    sh, cos = index.shard, index.score_function == "cos_sim"
    if sh.dtype == "int8":
        scales = sh.cos_scales if cos else sh.scales
        return sh.vectors[keep], scales[keep], scales.data_ptr()
    return sh.vectors[keep], (sh.inv_norms[keep] if cos else None), (sh.inv_norms.data_ptr() if cos else None)


def _reference_mining(index, nprobe, top_k, max_pairs, threshold, size, init):
    """Paraphrase pairs and communities from the exact masked searches of the inner shard, the stored rows as queries
    and per-query masks "probed & undeleted" (positions), then PairSelector / the community ordering."""
    from sgpt_b200 import _lib as L
    from sgpt_b200.index import _bit_slice, unpack_mask
    from sgpt_b200.ivf import _rows_f32
    from sgpt_b200.mining import PairSelector, _communities, _pairs_list

    sh, n, base = index.shard, index.n, index.id_base
    deleted = unpack_mask(_bit_slice(sh._deleted["words"], sh._deleted_at, n), n)
    keep = (~deleted).nonzero().flatten()
    qb, q_scale, c_scale = _stored(index, keep)
    probes = index.probe(_rows_f32(sh, keep), nprobe).long()
    list_of = torch.repeat_interleave(torch.arange(index.nlist, device="cuda"), index.offsets[1:] - index.offsets[:-1])
    probed = torch.zeros(keep.numel(), index.nlist, dtype=torch.bool, device="cuda").scatter_(1, probes, True)
    mask = sh._mask(probed[:, list_of], keep.numel())
    gid = index.ids.long() - base  # position -> id
    k = top_k + 1
    nq = keep.numel()
    lib = L.lib()
    ws = sh._workspace(lib.sgpt_search_workspace_bytes(nq, n, k))
    s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    j = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_search_masked(sh._dtype_id(), qb.data_ptr(), sh.vectors.data_ptr(), L.ptr(q_scale), c_scale, nq, n,
                                   index.dim, k, 0, L.ptr(mask[0]), mask[1], s.data_ptr(), j.data_ptr(), ws.data_ptr(),
                                   ws.numel(), L.current_stream()))
    sel = PairSelector(n, max_pairs, "cuda")
    jj = torch.where(j >= 0, gid[j.clamp(min=0)], -1)
    sel.add(s.reshape(-1), gid[keep].unsqueeze(1).expand(-1, k).reshape(-1), jj.reshape(-1))
    pairs = _pairs_list(sel)

    def by_id(offsets, s, pos):
        q = torch.repeat_interleave(torch.arange(offsets.numel() - 1, device="cuda"), offsets[1:] - offsets[:-1])
        ids = gid[pos]
        o = torch.sort(q * (1 << 31) + ids).indices
        return offsets, s[o], ids[o]

    offsets, rs, rpos = sh._range(qb, q_scale, c_scale, threshold, mask=mask)
    counts = torch.zeros(n, dtype=torch.int64, device="cuda")
    counts[gid[keep]] = offsets[1:] - offsets[:-1]
    alive = torch.zeros(n, dtype=torch.bool, device="cuda")
    alive[gid[keep]] = True
    central = torch.nonzero((counts >= size) & alive).flatten()
    row_of_id = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    row_of_id[gid[keep]] = torch.arange(nq, device="cuda")

    def fetch(idx, total):
        rows = row_of_id[idx]
        sub = (mask[0][rows], mask[1])
        return by_id(*sh._range(qb[rows], None if q_scale is None else q_scale[rows], c_scale, threshold, total, sub))
    comms = _communities(central, counts[central].tolist(), fetch, min(init, n), "cuda")
    return pairs, comms


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
@pytest.mark.parametrize("deletions", [False, True])
def test_ivf_mining_equals_reference_of_probed_lists(dtype, deletions, monkeypatch):
    """nprobe < nlist.  Small steps and blocks force several query blocks, count passes and member fetches."""
    from sgpt_b200 import IVFIndex, community_detection, mining, paraphrase_mining_embeddings

    x = _pm_data(n=4000, clusters=60, flip=0.12, seed=1 + deletions)
    index = IVFIndex.build(x.float() + 0.01 * torch.randn(x.shape, generator=torch.Generator(device="cuda").manual_seed(2),
                                                          device="cuda"), 24, dtype=dtype, n_iter=4, seed=1)
    gone = torch.arange(0, 4000, 9, device="cuda")
    if deletions:
        index.remove(gone)
    monkeypatch.setattr(mining, "_CANDIDATES_PER_STEP", 1)  # 256 rows per step
    monkeypatch.setattr(mining, "_COUNT_ROWS", 700)
    monkeypatch.setattr(mining, "_MEMBERS_PER_BLOCK", 900)
    nprobe, top_k, max_pairs, threshold, size, init = 3, 8, 5000, 0.6, 5, 40
    pairs = paraphrase_mining_embeddings(index, top_k=top_k, max_pairs=max_pairs, nprobe=nprobe)
    comms = community_detection(index, threshold=threshold, min_community_size=size, init_max_size=init, nprobe=nprobe)
    want_pairs, want_comms = _reference_mining(index, nprobe, top_k, max_pairs, threshold, size, init)
    assert len(pairs) > 100 and pairs == want_pairs
    assert len(comms) > 5 and comms == want_comms
    if deletions:
        dead = set(gone.tolist())
        assert not any(a in dead or b in dead for _, a, b in pairs)
        assert not any(m in dead for c in comms for m in c)
