"""Range search (sgpt_range_search, CorpusShard.range_search), paraphrase mining and community detection on the GPU.

Range search bit for bit: queries and documents hold small integers (|x| <= 8) and D = 64, the scales are powers of two,
so every device score equals the fp64 reference exactly (as tests/test_gpu_search_exact.py) and the CSR result must
equal the reference's under torch.equal, including documents exactly at the threshold.  Mining is compared with the
reference's own results (tests/golden/mining.npz) and, on tie-heavy +-1 data where cos = dot / 64 is exact, with the
oracle (oracle/mining.py) exactly."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import mining as omining
from oracle import search as osearch
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu

TILE = 256  # csrc/gemm_api.h kSimBN
D = 64
SENT_S, SENT_I = 12345.0, -99  # sentinels of the entry buffers


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def big_n():
    """More tiles than twice the SM count, the last one ragged."""
    return (2 * torch.cuda.get_device_properties(0).multi_processor_count + 3) * TILE + 77


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g).float()


def _pow2(m, g):
    return torch.pow(2.0, torch.randint(-3, 4, (m,), generator=g).float())


def device_range(Q, C, threshold, cap, id_base=0, q_scale=None, c_scale=None):
    L, lib = _lib()
    nq, n, D = Q.shape[0], C.shape[0], Q.shape[1]
    Qd, Cd = Q.to(torch.bfloat16).cuda(), C.to(torch.bfloat16).cuda()
    qs = None if q_scale is None else q_scale.cuda()
    cs = None if c_scale is None else c_scale.cuda()
    ws = torch.empty(lib.sgpt_range_search_workspace_bytes(nq, n), dtype=torch.uint8, device="cuda")
    counts = torch.full((nq,), -7, dtype=torch.int64, device="cuda")
    s = torch.full((max(cap, 1),), SENT_S, dtype=torch.float32, device="cuda")
    i = torch.full((max(cap, 1),), SENT_I, dtype=torch.int64, device="cuda")
    out = []
    for _ in range(2):  # a second launch must return the same bits
        L.check(lib.sgpt_range_search(Qd.data_ptr(), Cd.data_ptr(), L.ptr(qs), L.ptr(cs), nq, n, D, float(threshold),
                                      id_base, counts.data_ptr(), cap, s.data_ptr(), i.data_ptr(), ws.data_ptr(),
                                      ws.numel(), L.current_stream()), "sgpt_range_search")
        out.append((counts.cpu().clone(), s.cpu().clone(), i.cpu().clone()))
    assert all(torch.equal(a, b) for a, b in zip(out[0], out[1])), "second launch differs"
    return out[0]


def reference_scores(Q, C, q_scale=None, c_scale=None):
    sc = Q.double() @ C.double().T
    if q_scale is not None:
        sc = sc * q_scale.double()[:, None]
    if c_scale is not None:
        sc = sc * c_scale.double()[None, :]
    return torch.nan_to_num(sc, nan=-1.0, posinf=math.inf, neginf=-math.inf)  # XS:99


def reference_range(sc, threshold, cap, id_base=0):
    """(counts, entry buffers with sentinels) of the contract in include/sgpt_b200.h."""
    mask = sc >= threshold
    counts = mask.sum(1)
    s = torch.full((max(cap, 1),), SENT_S, dtype=torch.float32)
    i = torch.full((max(cap, 1),), SENT_I, dtype=torch.int64)
    off = 0
    for q in range(sc.shape[0]):
        c = int(counts[q])
        if off + c <= cap:
            cols = torch.nonzero(mask[q]).flatten()
            s[off:off + c] = sc[q, cols].float()
            i[off:off + c] = cols + id_base
        off += c
    return counts, s, i


def check_range(got, want, what):
    for name, a, b in zip(("counts", "scores", "ids"), got, want):
        if not torch.equal(a, b):
            bad = int((a != b).nonzero()[0][0])
            raise AssertionError(f"{what}: {name}[{bad}] = {a[bad].item()}, want {b[bad].item()}")


def exact_data(nq, n, g, nan_rows=False):
    Q, C = _ints((nq, D), -8, 8, g), _ints((n, D), -8, 8, g)
    if n > 3:
        C[n // 3] = C[n // 2]  # identical documents
    if nan_rows:
        C[::7] = float("nan")
    return Q, C, _pow2(nq, g), _pow2(n, g)


@pytest.mark.parametrize("nq", [1, 128, 129, 256, 257, 600])
@pytest.mark.parametrize("n", [1, 255, 256, 257, "big"])
def test_range_search_bit_exact(n, nq):
    """The threshold is a score that occurs (query 0's 37th best): documents exactly at it are included."""
    n = big_n() if n == "big" else n
    g = torch.Generator().manual_seed(1000 * nq + n % 1000)
    Q, C, qs, cs = exact_data(nq, n, g)
    sc = reference_scores(Q, C, qs, cs)
    t = float(torch.sort(sc[0], descending=True).values[min(n, 37) - 1])
    assert (sc == t).sum() >= 1
    total = int((sc >= t).sum())
    got = device_range(Q, C, t, total, q_scale=qs, c_scale=cs)
    check_range(got, reference_range(sc, t, total), f"n={n} nq={nq} t={t}")


@pytest.mark.parametrize("case", ["above_all", "below_all", "nan_rows", "dot_at_zero"])
def test_range_search_threshold_extremes_and_nan_rows(case):
    """Above every score nothing is admitted; below every score (and below -1) everything, NaN rows as -1."""
    g = torch.Generator().manual_seed(7)
    nq, n = 129, 1000
    Q, C, qs, cs = exact_data(nq, n, g, nan_rows=case in ("nan_rows", "below_all"))
    if case == "dot_at_zero":
        qs = cs = None
    sc = reference_scores(Q, C, qs, cs)
    t = {"above_all": float(sc.max()) + 1, "below_all": -math.inf, "nan_rows": -1.0, "dot_at_zero": 0.0}[case]
    total = int((sc >= t).sum())
    got = device_range(Q, C, t, total, id_base=0, q_scale=qs, c_scale=cs)
    check_range(got, reference_range(sc, t, total), case)
    if case == "below_all":
        assert int(got[0].sum()) == nq * n


@pytest.mark.parametrize("cap", ["zero", "mid", "exact", "large"])
def test_range_search_cap_and_id_base(cap):
    """cap = 0 only counts; a cap inside a query writes exactly the queries that fit (a prefix) and leaves every other
    slot of both buffers untouched; ids are offset by id_base."""
    g = torch.Generator().manual_seed(11)
    nq, n, id_base = 300, big_n(), 5_000_000_000
    Q, C, qs, cs = exact_data(nq, n, g)
    sc = reference_scores(Q, C, qs, cs)
    t = float(torch.quantile(sc[0].float(), 0.995))
    counts = (sc >= t).sum(1)
    total = int(counts.sum())
    off = torch.cumsum(counts, 0)
    q_cut = int((off < total // 2).sum())  # query q_cut straddles total // 2
    c = {"zero": 0, "mid": int(off[q_cut]) - 1, "exact": total, "large": total + 1000}[cap]
    if cap == "mid":
        assert int(off[q_cut]) - int(counts[q_cut]) < c  # the cut falls inside query q_cut
    got = device_range(Q, C, t, c, id_base=id_base, q_scale=qs, c_scale=cs)
    check_range(got, reference_range(sc, t, c, id_base), f"cap={cap}")


def test_corpus_shard_range_search_continuous():
    """Continuous bf16 data through the Python surface (the first buffer is too small, so it grows once): every document
    above threshold + 1e-5 of the fp64 cosine of the stored vectors is present, none below threshold - 1e-5, and the
    scores agree within 1e-5; each query's ids ascend."""
    from sgpt_b200 import CorpusShard

    g = torch.Generator().manual_seed(3)
    n, nq, dim, t = 70_000, 300, 128, 0.2
    C = torch.randn(n, dim, generator=g)
    Q = torch.randn(nq, dim, generator=g)
    C[:5000] += 1.5 * Q[torch.arange(5000) % nq]
    shard = CorpusShard.from_embeddings(C.cuda())
    off, s, ids = shard.range_search(Q.cuda(), t)
    off, s, ids = off.cpu(), s.cpu(), ids.cpu()
    assert off[0] == 0 and off[-1] == len(s) == len(ids) and int(off[-1]) > 64 * nq
    Cb, Qb = C.to(torch.bfloat16).double(), Q.to(torch.bfloat16).double()
    ref = (Qb / Qb.norm(dim=1, keepdim=True)) @ (Cb / Cb.norm(dim=1, keepdim=True)).T
    for q in range(nq):
        a, b = int(off[q]), int(off[q + 1])
        row = ids[a:b]
        assert torch.all(row[1:] > row[:-1])
        assert (s[a:b].double() - ref[q, row]).abs().max().item() < 1e-5 if b > a else True
        sure = torch.nonzero(ref[q] >= t + 1e-5).flatten()
        assert torch.isin(sure, row).all(), f"query {q}: a document above the threshold is missing"
        assert (ref[q, row] >= t - 1e-5).all(), f"query {q}: a document below the threshold is present"


# ---- mining -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def fx():
    return np.load(os.path.join(GOLDEN, "mining.npz"))


def test_community_detection_equals_reference_fixture(fx):
    from sgpt_b200 import community_detection
    from tests.test_mining_cpu import fixture_communities

    got = community_detection(torch.from_numpy(fx["comm_x"]).cuda(), threshold=float(fx["comm_threshold"]),
                              min_community_size=int(fx["comm_min_size"]), init_max_size=int(fx["comm_init_max"]))
    assert got == fixture_communities(fx)


def test_paraphrase_mining_equals_reference_fixture(fx):
    """Identical pairs in identical order, scores within 1e-6.  A pair is compared unordered: which of (i, j) and (j, i)
    survives (the smaller tuple, util.py:179-185) is decided by the last bit of two roundings of the same cosine."""
    from sgpt_b200 import paraphrase_mining_embeddings
    from tests.test_mining_cpu import fixture_pairs

    got = paraphrase_mining_embeddings(torch.from_numpy(fx["pairs_x"]), query_chunk_size=97,
                                       corpus_chunk_size=int(fx["pairs_chunk"]), max_pairs=int(fx["pairs_max_pairs"]),
                                       top_k=int(fx["pairs_top_k"]))
    want = fixture_pairs(fx)
    assert [sorted(p[1:]) for p in got] == [sorted(p[1:]) for p in want]
    assert max(abs(a[0] - b[0]) for a, b in zip(got, want)) < 1e-6


def pm1_data(n, seed):
    """+-1 vectors, D = 64 (|x| = 8, cos = dot / 64 exactly): clusters of near-duplicates (a few signs flipped)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 2, (n, D), generator=g).float() * 2 - 1
    centres = x[: n // 10].clone()
    for r in range(n // 10, n // 2):
        v = centres[int(torch.randint(0, len(centres), (1,), generator=g))].clone()
        flip = torch.randint(0, D, (int(torch.randint(0, 6, (1,), generator=g)),), generator=g)
        v[flip] *= -1
        x[r] = v
    return x[torch.randperm(n, generator=g)]


@pytest.mark.parametrize("score_function", ["cos_sim", "dot"])
@pytest.mark.parametrize("chunk,top_k,max_pairs", [(128, 7, 100), (1000, 3, 5000), (77, 20, 37)])
def test_paraphrase_mining_equals_oracle_on_ties(score_function, chunk, top_k, max_pairs):
    from sgpt_b200 import paraphrase_mining_embeddings

    x = pm1_data(300, seed=chunk + top_k)
    fn = osearch.cos_sim if score_function == "cos_sim" else osearch.dot_score
    want = omining.paraphrase_mining_embeddings(x, corpus_chunk_size=chunk, max_pairs=max_pairs, top_k=top_k,
                                                score_function=fn)
    got = paraphrase_mining_embeddings(x.cuda(), corpus_chunk_size=chunk, max_pairs=max_pairs, top_k=top_k,
                                       score_function=fn if chunk == 77 else score_function)
    assert got == want


@pytest.mark.parametrize("threshold,min_size,init_max", [(40 / 64, 3, 8), (52 / 64, 2, 1000), (0.0, 5, 200)])
def test_community_detection_equals_oracle_on_ties(threshold, min_size, init_max):
    """Thresholds equal to occurring scores; both member orders (init_max between the community sizes)."""
    from sgpt_b200 import CorpusShard, community_detection

    x = pm1_data(400, seed=min_size)
    want = omining.community_detection(x, threshold, min_size, init_max)
    assert community_detection(x.cuda(), threshold, min_size, init_max) == want
    assert community_detection(CorpusShard.from_embeddings(x.cuda(), id_base=10), threshold, min_size, init_max) == want
    with pytest.raises(ValueError):
        community_detection(x.cuda(), threshold, 401, init_max)


class IdTokenizer:
    """Texts are space-separated token ids."""
    pad_token_id = 299
    model_max_length = 64

    def tokenize(self, text):
        return text.split()

    def convert_tokens_to_ids(self, tokens):
        return [int(t) for t in tokens]

    def encode(self, text, add_special_tokens=False):
        return [int(t) for t in text.split()]


def test_paraphrase_mining_through_the_encoder():
    from sgpt_b200 import SentenceEncoder, paraphrase_mining, paraphrase_mining_embeddings

    g = torch.Generator().manual_seed(5)
    base = [torch.randint(0, 299, (int(torch.randint(3, 20, (1,), generator=g)),), generator=g).tolist()
            for _ in range(20)]
    sents = [" ".join(map(str, b)) for b in base] + [" ".join(map(str, b[:-1])) for b in base[:20]]
    model = SentenceEncoder.from_pretrained(os.path.join(GOLDEN, "st_tiny"), tokenizer=IdTokenizer(), batch_capacity=8)
    got = paraphrase_mining(model, sents, batch_size=8, top_k=5, max_pairs=50)
    want = paraphrase_mining_embeddings(model.encode(sents, batch_size=8, convert_to_tensor=True), top_k=5,
                                        max_pairs=50)
    assert got == want and len(got) > 10
    model.encoder.close()
