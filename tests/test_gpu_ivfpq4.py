"""The 4-bit IVF-PQ search (sgpt_pq_tables_nbits, sgpt_ivfpq_search_nbits, IVFPQIndex(nbits=4)) bit for bit.

Scan + select: small-integer 16-entry lookup tables and bases with random nibbles, so every ADC sum is an exact integer
with many ties; the result must equal the exact top-k over the fp64 sums (tests/helpers.py topk_reference) under
torch.equal, on the hand-made list layouts of test_gpu_ivfpq.py and with m on both sides of the whole-table limit
(m <= 256: the whole table in shared memory; above it 128-subspace chunks).  With continuous tables the device scores
must equal a numpy restatement of the documented sum order; one-hot tables pin the nibble order.  With nbits = 8 the
_nbits entry points must equal their 8-bit twins bit for bit.

IVFPQIndex(nbits=4): planted data; the search must equal an oracle built from the index's own centroids, codebooks,
codes and device tables, and the refine pass the exact re-rank of the PQ pass's candidates."""
import math

import numpy as np
import pytest
import torch

from tests.helpers import planted_corpus, topk_reference
from tests.test_gpu_ivfpq import SIZES, _base_per_pos, _clustered, _equal, _keep, _layout, _probes

pytestmark = pytest.mark.gpu


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _pack(codes):
    """[n, m] codes < 16 -> uint8 [n, m / 2]: byte i = code[2i] | code[2i+1] << 4."""
    from sgpt_b200.ivfpq import _pack_codes

    return _pack_codes(codes.long(), 4)


def _unpack(packed):
    p = packed.long()
    return torch.stack([p & 15, p >> 4], -1).reshape(p.shape[0], -1)


def _search(lut, base, codes, offsets, ids, probes, k, mask=None, nbits=4):
    """sgpt_ivfpq_search_nbits of unpacked codes [n, m] (packed here for nbits = 4)."""
    L, lib = _lib()
    nq, nprobe = probes.shape
    m = codes.shape[1]
    stored = _pack(codes) if nbits == 4 else codes.to(torch.uint8)
    nlist = offsets.numel() - 1
    max_len = int((offsets[1:] - offsets[:-1]).max())
    d = [t.cuda().contiguous() for t in (lut, base, stored, offsets, ids, probes)]
    md = None if mask is None else mask.cuda()
    need = lib.sgpt_ivfpq_search_workspace_bytes(nq, nlist, nprobe, max_len, m)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    L.check(lib.sgpt_ivfpq_search_nbits(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), nq, codes.shape[0], m, nbits,
                                        d[3].data_ptr(), nlist, max_len, d[4].data_ptr(), d[5].data_ptr(), nprobe, k,
                                        L.ptr(md), s.data_ptr(), i.data_ptr(), ws.data_ptr(), ws.numel(),
                                        L.current_stream()), "sgpt_ivfpq_search_nbits")
    return s.cpu(), i.cpu()


def _adc_f64(lut, codes):
    """sum_j lut[q, j, codes[pos, j]] in fp64 on the device: [nq, n] (exact for integer tables)."""
    lut, codes = lut.cuda().double(), codes.cuda().long()
    out = torch.zeros(lut.shape[0], codes.shape[0], dtype=torch.float64, device="cuda")
    for j in range(codes.shape[1]):
        out += lut[:, j, :][:, codes[:, j]]
    return out.cpu()


def _adc_restated(lut, base, codes, offsets, probes):
    """The documented order in numpy from unpacked codes: acc = 0; acc += lut[q][j][code[j]] for j ascending (fp32);
    score = fixnan(acc + base[q][p]); NaN where no probe covers the position.  [nq, n] float32."""
    lut, base, codes = lut.numpy(), base.numpy(), codes.numpy().astype(np.int64)
    nq, m = lut.shape[0], codes.shape[1]
    n = codes.shape[0]
    nlist = offsets.numel() - 1
    list_of = np.repeat(np.arange(nlist), (offsets[1:] - offsets[:-1]).numpy())
    out = np.full((nq, n), np.nan, dtype=np.float32)
    for q in range(nq):
        acc = np.zeros(n, dtype=np.float32)
        for j in range(m):
            acc = acc + lut[q, j][codes[:, j]]
        for p, l in enumerate(probes[q].tolist()):
            if 0 <= l < nlist:
                sel = list_of == l
                s = acc[sel] + base[q, p]
                out[q, sel] = np.where(np.isnan(s), np.float32(-1), s)
    return out


def _exact_case(nq, m, seed, sizes=SIZES, nprobe=5, deleted_frac=0.0):
    g = torch.Generator().manual_seed(seed)
    offsets, ids = _layout(sizes, g)
    n = int(offsets[-1])
    lut = torch.randint(-8, 9, (nq, m, 16), generator=g).float()
    base = torch.randint(-20, 21, (nq, nprobe), generator=g).float()
    codes = torch.randint(0, 16, (n, m), generator=g)
    probes = _probes(nq, len(sizes), nprobe, g)
    deleted = torch.rand(n, generator=g) < deleted_frac
    return lut, base, codes, offsets, ids, probes, deleted


# m = 32, 96, 256: the whole table in shared memory; 288 (a partial second chunk) and 2048 (D = 4096): chunked
@pytest.mark.parametrize("m", [32, 96, 256, 288, 2048])
@pytest.mark.parametrize("nq", [1, 7, 256, 300])
@pytest.mark.parametrize("k", [1, 10, 1001, 4096])
def test_scan_select_equals_exact_topk_of_integer_sums(m, nq, k):
    from sgpt_b200.index import pack_mask

    lut, base, codes, offsets, ids, probes, deleted = _exact_case(nq, m, seed=m * 131 + nq * 7 + k, deleted_frac=0.2)
    got = _search(lut, base, codes, offsets, ids, probes, k, mask=pack_mask(~deleted))
    sc = _adc_f64(lut, codes) + _base_per_pos(base, offsets, probes)
    _equal(f"m={m} nq={nq} k={k}", got, topk_reference(sc, _keep(offsets, ids, probes, deleted), k))
    assert not torch.isin(got[1], ids[deleted].long()).any()


@pytest.mark.parametrize("m", [96, 512])
def test_scan_unbalanced_lists_negative_ids_and_a_second_launch(m):
    sizes = [9000] + [1, 0, 2] * 30
    lut, base, codes, offsets, ids, probes, _ = _exact_case(200, m, seed=11 + m, sizes=sizes, nprobe=8)
    probes[:, 1:] = torch.where(probes[:, 1:] == 0, torch.full_like(probes[:, 1:], -1), probes[:, 1:])
    probes[:, 0] = 0
    ids[::101] = -1
    got = _search(lut, base, codes, offsets, ids, probes, 1001)
    sc = _adc_f64(lut, codes) + _base_per_pos(base, offsets, probes)
    _equal("unbalanced", got, topk_reference(sc, _keep(offsets, ids, probes), 1001))
    again = _search(lut, base, codes, offsets, ids, probes, 1001)
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1])


def test_scan_fewer_probed_documents_than_k():
    lut, base, codes, offsets, ids, _, _ = _exact_case(9, 32, seed=3, nprobe=2)
    probes = torch.tensor([[6, 7], [1, 12], [0, 5], [-1, 99], [10, 0], [7, -4], [12, 1], [6, 10], [5, 0]],
                          dtype=torch.int32)
    got = _search(lut, base, codes, offsets, ids, probes, 10)
    sc = _adc_f64(lut, codes) + _base_per_pos(base, offsets, probes)
    _equal("tails", got, topk_reference(sc, _keep(offsets, ids, probes), 10))
    assert (got[1][3] == -1).all() and (got[0][3] == -math.inf).all()


@pytest.mark.parametrize("m", [96, 256, 512, 2048])
def test_scan_reproduces_the_documented_sum_order(m):
    """Continuous tables and bases (NaN in a few table entries): every device score equals the numpy restatement, on
    the whole-table path (96, 256) and the chunked path (512, 2048), whose partial sums carry across chunks."""
    g = torch.Generator().manual_seed(m)
    nq, nprobe, k = 7, 6, 500
    offsets, ids = _layout(SIZES, g)
    n = int(offsets[-1])
    lut = torch.randn(nq, m, 16, generator=g)
    lut[0, 3, :7] = float("nan")
    base = torch.randn(nq, nprobe, generator=g) * 3
    codes = torch.randint(0, 16, (n, m), generator=g)
    probes = _probes(nq, len(SIZES), nprobe, g)
    s, i = _search(lut, base, codes, offsets, ids, probes, k)
    want = _adc_restated(lut, base, codes, offsets, probes)
    gid = _keep(offsets, ids, probes)
    _equal(f"restated m={m}", (s, i), topk_reference(torch.from_numpy(want).double().nan_to_num(-7.0), gid, k))


@pytest.mark.parametrize("m", [64, 512])
def test_nibble_order_on_the_device(m):
    """One-hot tables: lut[q][j][c] = 1 for c = pattern[q][j], else 0.  One document per query holds the pattern
    (score m), another the pattern with the two nibbles of every byte swapped, another with the bytes of every 16-byte
    unit reversed.  A wrong nibble or byte order scores the decoys higher than the pattern."""
    g = torch.Generator().manual_seed(m)
    nq, n = 12, 3000
    offsets = torch.tensor([0, n], dtype=torch.int64)
    ids = torch.arange(n, dtype=torch.int32)
    pattern = torch.randint(0, 16, (nq, m), generator=g)
    pattern[:, 1::2] = (pattern[:, 0::2] + 1 + torch.randint(0, 15, (nq, m // 2), generator=g)) % 16  # pairs differ
    codes = torch.randint(0, 16, (n, m), generator=g)
    codes[0::3][:nq] = pattern
    codes[1::3][:nq] = pattern.view(nq, m // 2, 2).flip(-1).reshape(nq, m)
    codes[2::3][:nq] = pattern.view(nq, m // 32, 16, 2).flip(2).reshape(nq, m)
    lut = torch.zeros(nq, m, 16)
    lut.scatter_(2, pattern[:, :, None], 1.0)
    base = torch.zeros(nq, 1)
    probes = torch.zeros(nq, 1, dtype=torch.int32)
    s, i = _search(lut, base, codes, offsets, ids, probes, 5)
    assert torch.equal(i[:, 0], torch.arange(nq) * 3) and (s[:, 0] == m).all()
    assert (s[:, 1] < m).all()
    sc = _adc_f64(lut, codes)
    _equal("one-hot", (s, i), topk_reference(sc, ids.long().expand(nq, n), 5))


def _tables(q, cb, cent, probes, nbits):
    L, lib = _lib()
    nq, D = q.shape
    m, K, _ = cb.shape
    nprobe = probes.shape[1]
    lut = torch.empty((nq, m, K), device="cuda")
    base = torch.empty((nq, nprobe), device="cuda")
    qd, cbd, cd, pd = q.cuda(), cb.cuda(), cent.cuda(), probes.cuda()
    L.check(lib.sgpt_pq_tables_nbits(qd.data_ptr(), cbd.data_ptr(), cd.data_ptr(), pd.data_ptr(), nq, D, m, nbits,
                                     cent.shape[0], nprobe, lut.data_ptr(), base.data_ptr(), L.current_stream()),
            "sgpt_pq_tables_nbits")
    return lut.cpu(), base.cpu()


@pytest.mark.parametrize("D,m", [(768, 96), (4096, 2048), (256, 32)])
def test_tables_within_the_fma_chain_bound_and_skipped_probes(D, m):
    g = torch.Generator().manual_seed(D + m)
    nq, nlist, nprobe = 33, 40, 9
    dsub = D // m
    q = torch.nn.functional.normalize(torch.randn(nq, D, generator=g), dim=1)
    cb = torch.randn(m, 16, dsub, generator=g)
    cent = torch.randn(nlist, D, generator=g)
    probes = _probes(nq, nlist, nprobe, g)
    lut, base = _tables(q, cb, cent, probes, 4)
    qs = q.double().view(nq, m, dsub)
    want = torch.einsum("qjt,jct->qjc", qs, cb.double())
    absum = torch.einsum("qjt,jct->qjc", qs.abs(), cb.double().abs())
    assert ((lut.double() - want).abs() <= dsub * 2.0 ** -23 * absum + 1e-30).all()
    ok = (probes >= 0) & (probes < nlist)
    pc = cent.double()[probes.long().clamp(0, nlist - 1)]
    wb = torch.einsum("qd,qpd->qp", q.double(), pc)
    bb = torch.einsum("qd,qpd->qp", q.double().abs(), pc.abs())
    assert ((base.double() - wb).abs()[ok] <= D * 2.0 ** -23 * bb[ok]).all()
    assert (base[~ok] == 0).all()


def test_8_bit_through_the_nbits_entry_points_equals_the_twins():
    """nbits = 8: sgpt_pq_tables_nbits and sgpt_ivfpq_search_nbits give the bits of sgpt_pq_tables and
    sgpt_ivfpq_search, on the whole-table (m = 96) and the chunked (m = 512) path."""
    L, lib = _lib()
    for m in (96, 512):
        g = torch.Generator().manual_seed(m + 1)
        D, nq, nlist, nprobe, k = 1536, 37, len(SIZES), 5, 300
        q = torch.randn(nq, D, generator=g).cuda()
        cb = torch.randn(m, 256, D // m, generator=g).cuda()
        cent = torch.randn(nlist, D, generator=g).cuda()
        probes = _probes(nq, nlist, nprobe, g).cuda()
        outs = []
        for fn in ("twin", "nbits"):
            lut = torch.empty((nq, m, 256), device="cuda")
            base = torch.empty((nq, nprobe), device="cuda")
            args = [q.data_ptr(), cb.data_ptr(), cent.data_ptr(), probes.data_ptr(), nq, D, m]
            tail = [nlist, nprobe, lut.data_ptr(), base.data_ptr(), L.current_stream()]
            rc = (lib.sgpt_pq_tables(*args, *tail) if fn == "twin" else lib.sgpt_pq_tables_nbits(*args, 8, *tail))
            L.check(rc, fn)
            outs.append((lut.cpu(), base.cpu()))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        lut, base = outs[0]
        offsets, ids = _layout(SIZES, g)
        codes = torch.randint(0, 256, (int(offsets[-1]), m), generator=g)
        got = _search(lut, base, codes, offsets, ids, probes.cpu(), k, nbits=8)
        from tests.test_gpu_ivfpq import _ivfpq

        want = _ivfpq(lut, base, codes.to(torch.uint8), offsets, ids, probes.cpu(), k)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


# ---- IVFPQIndex(nbits=4) on planted data --------------------------------------------------------------------------------
N, DIM, NQ, NLIST, M = 20000, 64, 150, 48, 32


def _oracle(index, q, k, nprobe, removed=None):
    """Top-k over the index's own (unpacked) codes, scored from the index's device tables in the documented order."""
    probes = index.probe(q, nprobe)
    lut, base = index.tables(q, probes)
    offsets, ids = index.offsets.cpu(), index.ids.cpu()
    want = _adc_restated(lut.cpu(), base.cpu(), _unpack(index.codes.cpu()), offsets, probes.cpu())
    deleted = None if removed is None else torch.isin(ids.long(), removed.cpu())
    gid = _keep(offsets, ids, probes.cpu(), deleted)
    return topk_reference(torch.from_numpy(want).double().nan_to_num(-7.0), gid, k)


@pytest.fixture(scope="module", params=[("bf16", "cos_sim"), ("int8", "cos_sim"), ("bf16", "dot")],
                ids=["bf16-cos", "int8-cos", "bf16-dot"])
def built(request):
    from sgpt_b200 import CorpusShard, IVFPQIndex

    dtype, sf = request.param
    q, c = planted_corpus(N, DIM, NQ, seed=1)
    src = CorpusShard.from_embeddings(c.cuda(), dtype=dtype, id_base=500)
    index = IVFPQIndex.build(src, NLIST, M, score_function=sf, n_iter=4, seed=3, nbits=4)
    return src, index, q.cuda(), sf


@pytest.mark.parametrize("nprobe", [1, 8, NLIST])
@pytest.mark.parametrize("k", [10, 100])
def test_index_search_equals_oracle_from_its_own_tables(built, nprobe, k):
    src, index, q, sf = built
    assert index.nbits == 4 and tuple(index.codes.shape) == (N, M // 2)
    assert tuple(index.codebooks.shape) == (M, 16, DIM // M)
    got = index.search(q, k, nprobe)
    _equal(f"nprobe={nprobe} k={k}", (got[0].cpu(), got[1].cpu()), _oracle(index, q, k, nprobe))


def test_index_build_equals_train_plus_chunked_add(built):
    from sgpt_b200 import IVFPQIndex
    from sgpt_b200.ivf import _rows_f32
    from sgpt_b200.ivfpq import _nearest_codewords

    src, index, q, sf = built
    T = min(N, max(64 * NLIST, 256))
    sample = torch.randperm(N, generator=torch.Generator().manual_seed(3))[:T].cuda()
    other = IVFPQIndex.train(_rows_f32(src, sample), NLIST, M, sf, n_iter=4, seed=3, id_base=500, nbits=4)
    rows = _rows_f32(src, torch.arange(N, device="cuda"))
    other.add(rows[:7000])
    other.add(rows[7000:])
    for a in ("centroids", "codebooks", "codes", "offsets", "ids"):
        assert torch.equal(getattr(index, a), getattr(other, a)), a
    a, b = index.search(q, 50, 6), other.search(q, 50, 6)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert index.nbytes >= N * (M // 2 + 8) and index.nbytes - N * (M // 2 + 8) < N // 8 + (1 << 20)
    # the stored nibbles are the encoder's codes of the residuals
    pos = index._pos[torch.arange(0, N, 97, device="cuda")].long()
    x = rows[torch.arange(0, N, 97, device="cuda")]
    if sf == "cos_sim":
        x = torch.nn.functional.normalize(x, dim=1)
    lists = torch.searchsorted(index.offsets, pos, right=True) - 1
    want = _nearest_codewords(x - index.centroids[lists], index.codebooks)
    assert torch.equal(_unpack(index.codes[pos]), want)


def test_index_save_load_round_trip(built, tmp_path):
    import json

    from sgpt_b200 import IVFPQIndex

    src, index, q, sf = built
    index.save(str(tmp_path / "pq4"))
    assert json.loads((tmp_path / "pq4" / "meta.json").read_text())["nbits"] == 4
    assert np.load(tmp_path / "pq4" / "codes.npy").shape == (N, M // 2)
    back = IVFPQIndex.load(str(tmp_path / "pq4"), device="cuda:0")
    assert back.nbits == 4 and torch.equal(back.codes, index.codes)
    for nprobe in (1, 6):
        a, b = index.search(q, 64, nprobe), back.search(q, 64, nprobe)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("k", [10, 40])
def test_index_refine_equals_rerank_of_the_pq_candidates(built, k):
    from sgpt_b200.ivfpq import rerank

    src, index, q, sf = built
    kr = 10 * k
    got = index.search(q, k, 8, refine=src, k_refine=kr)
    cand = index.search(q, kr, 8)[1]
    want = rerank(src, q, cand, k, sf)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_index_refine_recall_on_planted_clusters(dtype):
    """4-bit codes at m = 64 take the bytes of the 8-bit test's m = 32 (test_gpu_ivfpq.py)."""
    from sgpt_b200 import CorpusShard, IVFPQIndex

    q, c = _clustered(N, 128, NLIST, 200, seed=5)
    src = CorpusShard.from_embeddings(c.cuda(), dtype=dtype)
    index = IVFPQIndex.build(src, NLIST, 64, n_iter=6, seed=0, nbits=4)
    q = q.cuda()
    got = index.search(q, 10, 8, refine=src)[1]
    exact = src.search(q, 10)[1]
    recall = float(torch.stack([torch.isin(exact[r], got[r]).float().mean() for r in range(q.shape[0])]).mean())
    print(f"recall@10 with refine at nprobe=8 ({dtype}, cos_sim, 20000 x 128, nlist 48, m 64, 4-bit): {recall:.4f}")
    assert recall >= 0.9  # measured 0.9545 (bf16) and 0.9560 (int8) on an H100


def test_index_remove_and_source_deletions():
    from sgpt_b200 import CorpusShard, IVFPQIndex

    q, c = planted_corpus(N, DIM, NQ, seed=1)
    q = q.cuda()
    src = CorpusShard.from_embeddings(c.cuda(), dtype="int8", id_base=7)
    src.remove(torch.arange(7, 7 + N, 13))  # deletions of the source carry over
    index = IVFPQIndex.build(src, NLIST, M, n_iter=3, seed=0, nbits=4)
    assert index.n_deleted == src.n_deleted
    top = index.search(q, 10, 6)[1]
    gone = torch.unique(top[:, :3].flatten())
    index.remove(gone)
    removed = torch.cat([gone, torch.arange(7, 7 + N, 13, device="cuda")])
    got = index.search(q, 10, 6)
    assert not torch.isin(got[1], removed).any()
    _equal("removed", (got[0].cpu(), got[1].cpu()), _oracle(index, q, 10, 6, removed))
    index.add(torch.randn(3000, DIM, generator=torch.Generator().manual_seed(8)).cuda())
    assert index.n_deleted == removed.numel()
    got = index.search(q, 10, 6)
    assert not torch.isin(got[1], removed).any()
    _equal("removed after add", (got[0].cpu(), got[1].cpu()), _oracle(index, q, 10, 6, removed))


@pytest.mark.parametrize("sf", ["cos_sim", "dot"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_index_add_leaves_its_input_unchanged(sf, dtype):
    from sgpt_b200 import IVFPQIndex

    q, c = _clustered(4000, 64, 16, 4, seed=2)
    trained = IVFPQIndex.train(c.cuda(), 16, 32, score_function=sf, n_iter=2, seed=1, nbits=4)
    emb = c.cuda().to(dtype)
    before = emb.clone()
    trained.add(emb)
    assert torch.equal(emb, before)
    other = IVFPQIndex.train(c.cuda(), 16, 32, score_function=sf, n_iter=2, seed=1, nbits=4)
    other.add(before.clone())
    assert torch.equal(trained.codes, other.codes) and torch.equal(trained.ids, other.ids)
