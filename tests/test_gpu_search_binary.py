"""Binary corpus shards on the GPU, bit for bit against numpy / exact references: the sign-bit quantizer, the single-bit
wgmma search (dense and two-pass plans, ragged last k-block, both score functions, tie-heavy by construction), filters
and deletions, the packed merge, range search, rescoring with the float query, refine, persistence, and a recall
property of median thresholds and rescoring on offset data."""
import numpy as np
import pytest
import torch

from tests import binary_ref as ref
from tests.helpers import topk_reference

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _signs(bits):
    """uint8 [n, B] (device) -> fp32 +-1 [n, 8 B] in dimension order (np.unpackbits order)."""
    sh = torch.arange(7, -1, -1, device=bits.device)
    b = (bits.long().unsqueeze(-1) >> sh) & 1
    return (b.reshape(bits.shape[0], -1).float() * 2 - 1)


def _sign_dot(qbits, dbits):
    """Exact s for every pair: a +-1 fp32 matmul (every partial sum an integer below 2^24), fp32 [nq, n]."""
    return _signs(qbits) @ _signs(dbits).T


def _ref_topk(s, k, allow=None):
    """Top-k by (score desc, id asc) of a device score matrix; disallowed entries absent; tail (-inf, -1)."""
    s = s.clone()
    if allow is not None:
        s[~allow.expand_as(s)] = -float("inf")
    vals, idx = torch.sort(s, dim=1, descending=True, stable=True)
    kk = min(k, s.shape[1])
    out_s = torch.full((s.shape[0], k), -float("inf"), device=s.device)
    out_i = torch.full((s.shape[0], k), -1, dtype=torch.int64, device=s.device)
    out_s[:, :kk], out_i[:, :kk] = vals[:, :kk], idx[:, :kk]
    absent = out_s == -float("inf")
    out_i[absent] = -1
    return out_s, out_i


def _data(n, nq, D, seed, offset=0.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = torch.randn(n, D, device=DEV, generator=g) + offset
    q = torch.randn(nq, D, device=DEV, generator=g) + offset
    return c, q


def _expect(shard, q, k, score_function, allow=None):
    from sgpt_b200.index import quantize_rows_b1

    qbits, _ = quantize_rows_b1(q, shard.thresholds)
    s = _sign_dot(qbits, shard.stored())
    es, ei = _ref_topk(s, k, allow)
    if score_function == "cos_sim":
        es = es / torch.full((), float(shard.dim), device=DEV)
    return es, ei + shard.id_base * (ei >= 0)


# ---- quantizer --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [128, 768, 4096])
@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("thresholds", ["zero", "random"])
def test_quantizer_matches_packbits(D, bf16, thresholds):
    from sgpt_b200.index import quantize_rows_b1

    g = torch.Generator(device=DEV).manual_seed(D)
    x = torch.randn(37, D, device=DEV, generator=g)
    t = None if thresholds == "zero" else torch.randn(D, device=DEV, generator=g).to(torch.bfloat16).float()
    tt = torch.zeros(D, device=DEV) if t is None else t
    x[0] = tt                       # every value equal to its threshold: all 0
    x[1, ::3] = float("nan")        # NaN -> 0
    x[2] = 0.0
    x[3] = -0.0
    x[4, 1::2] = tt[1::2]           # half equal, half NaN
    x[4, ::2] = float("nan")
    x[5] = tt + 1.0                 # all 1
    if bf16:
        x = x.to(torch.bfloat16)
    bits, popc = quantize_rows_b1(x, t)
    want = ref.pack(x.float().cpu().numpy(), None if t is None else t.cpu().numpy())
    assert np.array_equal(bits.cpu().numpy(), want)
    assert np.array_equal(popc.cpu().numpy(), ref.popcounts(want))
    assert int(popc[0]) == 0 and int(popc[5]) == D
    # twice: the same bits
    bits2, _ = quantize_rows_b1(x, t)
    assert torch.equal(bits, bits2)


# ---- search -----------------------------------------------------------------------------------------------------------
CASES = [  # (D, n, nq, k)
    (128, 1, 7, 10),          # n < k
    (128, 255, 1, 1),
    (768, 256, 129, 10),
    (1152, 257, 300, 1001),   # ragged last k-block (144 bytes = 128 + 16)
    (4096, 3000, 128, 4096),
    (768, 3000, 256, 10),
    (1152, 3000, 7, 1001),
    (768, 200_000, 129, 10),  # two-pass plan
    (1152, 200_000, 300, 100),
    (4096, 200_000, 1, 1001),
]


@pytest.mark.parametrize("D,n,nq,k", CASES)
@pytest.mark.parametrize("score_function", ["dot", "cos_sim"])
def test_search_matches_exact_sign_dot(D, n, nq, k, score_function):
    from sgpt_b200 import CorpusShard

    c, q = _data(n, nq, D, seed=D + n + nq)
    shard = CorpusShard.from_embeddings(c, device=DEV, id_base=5, dtype="binary")
    s, i = shard.search(q, k, score_function)
    es, ei = _expect(shard, q, k, score_function)
    assert torch.equal(i, ei)
    assert torch.equal(s, es)


def test_ties_at_the_cut_go_to_the_lowest_ids():
    from sgpt_b200 import CorpusShard

    D, n = 256, 5000
    c, q = _data(n, 4, D, seed=1)
    c[1000:] = c[0]  # 4000 identical documents
    q[:] = c[0]
    shard = CorpusShard.from_embeddings(c, device=DEV, dtype="binary")
    s, i = shard.search(q, 100, "dot")
    assert torch.all(s == D)
    want = torch.cat([torch.tensor([0]), torch.arange(1000, 1099)]).to(DEV)
    assert torch.equal(i, want.expand(4, -1))


@pytest.mark.parametrize("n", [3000, 200_000])
def test_allow_and_remove_equal_the_search_over_the_rest(n):
    from sgpt_b200 import CorpusShard

    D, nq, k = 768, 129, 50
    c, q = _data(n, nq, D, seed=7)
    shard = CorpusShard.from_embeddings(c, device=DEV, dtype="binary")
    g = torch.Generator(device=DEV).manual_seed(3)
    shared = torch.rand(n, device=DEV, generator=g) < 0.3
    per_q = torch.rand(nq, n, device=DEV, generator=g) < 0.05
    for allow in (shared, per_q):
        s, i = shard.search(q, k, "cos_sim", allow=allow)
        es, ei = _expect(shard, q, k, "cos_sim", allow=allow)
        assert torch.equal(i, ei) and torch.equal(s, es)
    gone = torch.arange(0, n, 3, device=DEV)
    shard.remove(gone)
    keep = torch.ones(n, dtype=torch.bool, device=DEV)
    keep[gone] = False
    s, i = shard.search(q, k, "dot", allow=shared)
    es, ei = _expect(shard, q, k, "dot", allow=shared & keep)
    assert torch.equal(i, ei) and torch.equal(s, es)


def test_packed_views_merge_to_the_whole_shard():
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import merge_topk_packed

    D, n, nq, k = 1152, 9000, 33, 64
    c, q = _data(n, nq, D, seed=11)
    shard = CorpusShard.from_embeddings(c, device=DEV, dtype="binary")
    for sf in ("dot", "cos_sim"):
        parts = [shard.view(0, 4096).search_packed(q, k, sf), shard.view(4096, n).search_packed(q, k, sf)]
        s, i = merge_topk_packed(torch.stack(parts))
        ws, wi = shard.search(q, k, sf)
        assert torch.equal(i, wi) and torch.equal(s, ws)


@pytest.mark.parametrize("score_function", ["dot", "cos_sim"])
def test_range_search_equals_the_numpy_sets(score_function):
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import quantize_rows_b1

    D, n, nq = 768, 20_000, 9
    c, q = _data(n, nq, D, seed=5)
    c[::500] = q[torch.arange(40, device=DEV) % nq] + 0.3 * c[::500]
    shard = CorpusShard.from_embeddings(c, device=DEV, dtype="binary")
    qbits, _ = quantize_rows_b1(q)
    s = _sign_dot(qbits, shard.stored()).cpu().numpy().astype(np.int64)
    score = s.astype(np.float32) if score_function == "dot" else ref.cos_of(s, D)
    thr = 200.0 if score_function == "dot" else float(ref.cos_of(np.array([200]), D)[0]) - 1e-7
    off, sc, ids = shard.range_search(q, thr, score_function)
    off, sc, ids = off.cpu().numpy(), sc.cpu().numpy(), ids.cpu().numpy()
    for j in range(nq):
        want = np.nonzero(score[j] >= np.float32(thr))[0]
        assert np.array_equal(ids[off[j]:off[j + 1]], want)
        assert np.array_equal(sc[off[j]:off[j + 1]], score[j][want])
    assert off[-1] > nq  # the planted documents are found


# ---- rescoring --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [128, 1152, 4096])
@pytest.mark.parametrize("score_function", ["dot", "cos_sim"])
def test_rescore_equals_the_numpy_restatement(D, score_function):
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import binary_thresholds

    n, nq, k, kc = 5000, 6, 10, 100
    c, q = _data(n, nq, D, seed=D, offset=0.25)
    thr = None if D == 128 else binary_thresholds(c[:1000])
    shard = CorpusShard.from_embeddings(c, device=DEV, dtype="binary", thresholds=thr)
    _, cand = shard.search(q, kc, "dot")
    s, i = shard.search(q, k, score_function, rescore=kc)
    qf = q.float() - shard.thresholds
    qs = None
    if score_function == "cos_sim":
        qf = torch.nn.functional.normalize(qf, dim=1)
        qs = np.full(nq * kc, ref.inv_sqrt_dim(D), np.float32)
    cand_np = cand.cpu().numpy()
    rows = shard.stored().cpu().numpy()[cand_np.reshape(-1)]
    asym = ref.asym_scores(np.repeat(qf.cpu().numpy(), kc, axis=0), rows, qs).reshape(nq, kc)
    es, ei = topk_reference(torch.from_numpy(asym), torch.from_numpy(cand_np), k)
    assert torch.equal(i.cpu(), ei)
    assert np.array_equal(s.cpu().numpy(), es.numpy().astype(np.float32))


@pytest.mark.parametrize("refine_dtype", ["bf16", "int8"])
def test_refine_equals_rerank_of_the_candidates(refine_dtype):
    from sgpt_b200 import CorpusShard
    from sgpt_b200.ivfpq import rerank

    D, n, nq, k = 768, 20_000, 17, 10
    c, q = _data(n, nq, D, seed=23)
    shard = CorpusShard.from_embeddings(c, device=DEV, id_base=100, dtype="binary")
    exact = CorpusShard.from_embeddings(c, device=DEV, id_base=100, dtype=refine_dtype)
    for sf in ("cos_sim", "dot"):
        _, cand = shard.search(q, 100, "dot")
        s, i = shard.search(q, k, sf, refine=exact)
        ws, wi = rerank(exact, q, cand, k, sf)
        assert torch.equal(i, wi) and torch.equal(s, ws)
    with pytest.raises(ValueError, match="does not hold"):
        shard.search(q, k, refine=CorpusShard.from_embeddings(c[:100], device=DEV))


# ---- persistence ------------------------------------------------------------------------------------------------------
def test_save_load_and_packed_bits_round_trips(tmp_path):
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import binary_thresholds

    D, n, nq, k = 768, 3000, 8, 20
    c, q = _data(n, nq, D, seed=31, offset=0.5)
    thr = binary_thresholds(c[:500])
    shard = CorpusShard.from_embeddings(c, device=DEV, id_base=7, dtype="binary", thresholds=thr)
    shard.remove([7, 100])
    want = shard.search(q, k, "cos_sim")
    shard.save(str(tmp_path / "s"))
    back = CorpusShard.load(str(tmp_path / "s"), device=DEV)
    assert back.dtype == "binary" and torch.equal(back.stored(), shard.stored())
    assert torch.equal(back.popcounts[:n], shard.popcounts[:n]) and torch.equal(back.thresholds, shard.thresholds)
    got = back.search(q, k, "cos_sim")
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    # sentence-transformers' "ubinary": np.packbits(x > 0)
    ub = np.packbits(c.cpu().numpy() > 0, axis=-1)
    st = CorpusShard.from_packed_bits(ub, device=DEV)
    mine = CorpusShard.from_embeddings(c, device=DEV, dtype="binary")
    assert torch.equal(st.stored(), mine.stored()) and torch.equal(st.popcounts[:n], mine.popcounts[:n])
    for sf in ("dot", "cos_sim"):
        a, b = st.search(q, k, sf), mine.search(q, k, sf)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ---- recall property --------------------------------------------------------------------------------------------------
def test_median_thresholds_and_rescoring_recall_more_on_offset_clusters():
    """Planted clusters under a large common offset (anisotropic embeddings): zero thresholds see mostly the offset's
    sign, median thresholds split every dimension, and rescoring with the float query (centered on the thresholds)
    recalls more than the bits."""
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import binary_thresholds

    D, n, nq, k = 768, 50_000, 64, 10
    g = torch.Generator(device=DEV).manual_seed(0)
    offset = 3.0 * torch.rand(D, device=DEV, generator=g) + 1.0
    centers = torch.randn(nq, D, device=DEV, generator=g)
    c = torch.randn(n, D, device=DEV, generator=g)
    members = torch.arange(nq * 50, device=DEV)
    c[members] = centers[members % nq] + 0.8 * torch.randn(len(members), D, device=DEV, generator=g)
    q = centers + 0.8 * torch.randn(nq, D, device=DEV, generator=g)
    c, q = c + offset, q + offset
    exact = CorpusShard.from_embeddings(c, device=DEV)
    _, truth = exact.search(q, k, "cos_sim")

    def recall(ids):
        return sum(len(set(a) & set(b)) for a, b in zip(ids.tolist(), truth.tolist())) / truth.numel()

    zero = CorpusShard.from_embeddings(c, device=DEV, dtype="binary")
    med = CorpusShard.from_embeddings(c, device=DEV, dtype="binary", thresholds=binary_thresholds(c[:5000]))
    r_zero = recall(zero.search(q, k, "cos_sim")[1])
    r_med = recall(med.search(q, k, "cos_sim")[1])
    r_rescore = recall(med.search(q, k, "cos_sim", rescore=100)[1])
    print(f"recall@{k}: zero thresholds {r_zero:.3f}, median {r_med:.3f}, median + rescore {r_rescore:.3f}")
    assert r_med > r_zero
    assert r_rescore > r_med


def test_range_search_takes_infinite_cos_thresholds():
    """-inf admits every (undeleted) document, +inf none, as on bf16 and int8 shards."""
    from sgpt_b200 import CorpusShard

    D, n, nq = 256, 1000, 3
    c, q = _data(n, nq, D, seed=41)
    shard = CorpusShard.from_embeddings(c, device=DEV, dtype="binary")
    shard.remove([5])
    off, sc, ids = shard.range_search(q, float("-inf"), "cos_sim")
    assert off.tolist() == [0, n - 1, 2 * (n - 1), 3 * (n - 1)]
    want = torch.cat([torch.arange(5), torch.arange(6, n)]).to(DEV)
    assert all(torch.equal(ids[off[j]:off[j + 1]], want) for j in range(nq))
    off, _, _ = shard.range_search(q, float("inf"), "cos_sim")
    assert int(off[-1]) == 0
