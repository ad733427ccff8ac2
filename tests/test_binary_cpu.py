"""CPU checks of binary corpus shards: the numpy restatements (tests/binary_ref.py) against hand-made cases, and every
rejection of sgpt_quantize_rows_b1 and of SGPT_DTYPE_B1 before any CUDA call or device allocation."""
import json

import numpy as np
import pytest

from tests import binary_ref as ref

N_PTR = np.zeros(64, dtype=np.int64)
P = N_PTR.ctypes.data  # dummy host pointer, never dereferenced (16-byte aligned: numpy aligns its buffers)
B1 = 3


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


# ---- numpy restatements ---------------------------------------------------------------------------------------------
def test_pack_is_packbits_order_with_strict_compare():
    x = np.zeros((1, 16), np.float32)
    x[0, 0] = 1.0          # dimension 0 -> bit 7 of byte 0
    x[0, 9] = 0.5          # dimension 9 -> bit 6 of byte 1
    x[0, 15] = 2.0         # dimension 15 -> bit 0 of byte 1
    x[0, 3] = np.nan       # NaN -> 0
    x[0, 4] = -0.0         # -0 > 0 is false
    assert ref.pack(x).tolist() == [[0b10000000, 0b01000001]]
    t = np.zeros(16, np.float32)
    t[0], t[9] = 1.0, 0.25  # x == t gives 0, x > t gives 1
    assert ref.pack(x, t).tolist() == [[0b00000000, 0b01000001]]
    assert ref.popcounts(ref.pack(x)).tolist() == [3]


def test_sign_dot_and_cosine_by_hand():
    D = 128
    q = np.ones((1, D), np.float32)
    d = np.ones((3, D), np.float32)
    d[1, :10] = -1   # hamming 10
    d[2] = -1        # hamming D
    s = ref.sign_dot(ref.pack(q), ref.pack(d))
    assert s.tolist() == [[D, D - 20, -D]]
    pm = ref.signs(ref.pack(q)).astype(np.int64) @ ref.signs(ref.pack(d)).astype(np.int64).T
    assert np.array_equal(s, pm)  # the +-1 dot product
    c = ref.cos_of(s, D)
    assert c.dtype == np.float32 and c.tolist() == [[1.0, np.float32(108) / np.float32(128), -1.0]]
    D = 768
    assert ref.cos_of(np.array([1]), D)[0] == np.float32(1) / np.float32(768)


def test_asymmetric_order_by_hand():
    """With small-integer queries every partial sum is exact, so the fixed order equals the exact sum; a cancellation
    case shows that the order matters and that the restatement takes lane 0's order first."""
    rng = np.random.default_rng(0)
    D = 256
    q = rng.integers(-4, 5, size=(5, D)).astype(np.float32)
    bits = ref.pack(rng.standard_normal((5, D)))
    want = (q.astype(np.float64) * ref.signs(bits)).sum(1)
    assert np.array_equal(ref.asym_scores(q, bits), want.astype(np.float32))
    # lane 0 holds dimensions 0..127, lane 1 dimensions 128..255: 1e8 + 1 - 1e8 in lane 0 rounds the 1 away
    q = np.zeros((1, D), np.float32)
    q[0, 0], q[0, 1], q[0, 2] = 1e8, 1.0, -1e8
    bits = ref.pack(np.ones((1, D), np.float32))
    assert ref.asym_scores(q, bits)[0] == 0.0
    assert ref.asym_scores(q, bits, q_scale=np.array([0.5], np.float32))[0] == 0.0
    q[0, 2] = 1e8
    bits = ref.pack(np.where(np.arange(D) == 2, -1.0, 1.0)[None, :].astype(np.float32))
    assert ref.asym_scores(q, bits)[0] == 0.0
    assert ref.inv_sqrt_dim(768) == np.float32(1 / np.sqrt(768.0))


def test_cos_threshold_maps_to_the_smallest_qualifying_sign_dot():
    from sgpt_b200.index import _b1_threshold

    for D in (128, 768, 1152, 4096):
        s = np.arange(-D, D + 1)
        c = ref.cos_of(s, D)
        for t in (-2.0, -1.0, -0.3, 0.0, 1e-9, 0.1, 0.5, float(c[D + 17]), 0.999, 1.0, 1.5):
            s0 = _b1_threshold(t, "cos_sim", D)
            assert np.array_equal(s >= s0, c >= np.float32(t)), (D, t)
    assert _b1_threshold(0.25, "dot", 768) == 0.25
    # non-finite thresholds: -inf admits everything, +inf nothing, NaN goes on to the library (which rejects it)
    assert _b1_threshold(float("-inf"), "cos_sim", 768) == -768.0
    assert _b1_threshold(float("inf"), "cos_sim", 768) == 769.0
    assert np.isnan(_b1_threshold(float("nan"), "cos_sim", 768))
    assert _b1_threshold(float("-inf"), "dot", 768) == float("-inf")


# ---- C ABI rejections -----------------------------------------------------------------------------------------------
def _quant(D=128, n=4, x=P, bits=P, popc=P, thr=None):
    return _lib().sgpt_quantize_rows_b1(x, 0, thr, bits, popc, n, D, None)


@pytest.mark.parametrize("D", [0, 64, 200, 65536 + 128])
def test_quantizer_rejects_bad_dims(D):
    assert _quant(D=D) == 1
    assert f"D={D} must be a positive multiple of 128, at most 65536".encode() in _lib().sgpt_last_error()


def test_quantizer_rejects_null_and_unaligned_pointers():
    assert _quant(popc=None) == 1 and b"null" in _lib().sgpt_last_error()
    assert _quant(bits=None) == 1 and b"null" in _lib().sgpt_last_error()
    assert _quant(x=P + 4) == 1 and b"aligned" in _lib().sgpt_last_error()
    assert _quant(bits=P + 8) == 1 and b"aligned" in _lib().sgpt_last_error()
    assert _quant(n=0, D=65536) == 0, _lib().sgpt_last_error()  # no rows: nothing to do
    assert _quant(n=-1) == 1


def _call(name, D=128, n=100, nq=3, k=10, q=P, c=P, qs=P, cs=P, mask=None, pitch=0, dtype=B1):
    lib = _lib()
    if name == "sgpt_search_masked":
        return lib.sgpt_search_masked(dtype, q, c, qs, cs, nq, n, D, k, 0, mask, pitch, P, P, P, 1 << 40, None)
    if name == "sgpt_search_packed_masked":
        return lib.sgpt_search_packed_masked(dtype, q, c, qs, cs, nq, n, D, k, 0, mask, pitch, P, P, 1 << 40, None)
    if name == "sgpt_range_search_masked":
        return lib.sgpt_range_search_masked(dtype, q, c, qs, cs, nq, n, D, 0.5, 0, mask, pitch, P, 10, P, P, P, 1 << 40,
                                            None)
    if name == "sgpt_search_gather_masked":
        return lib.sgpt_search_gather_masked(dtype, None, q, c, qs, cs, nq, n, D, k, 0, mask, pitch, None, P, P, P,
                                             1 << 40, None)
    raise ValueError(name)


SEARCHES = ["sgpt_search_masked", "sgpt_search_packed_masked", "sgpt_range_search_masked"]


@pytest.mark.parametrize("name", SEARCHES)
@pytest.mark.parametrize("D", [0, 64, 136, 65536 + 128])
def test_binary_searches_reject_bad_dims(name, D):
    assert _call(name, D=D) == 1
    assert f"binary D={D} must be a positive multiple of 128, at most 65536".encode() in _lib().sgpt_last_error()


@pytest.mark.parametrize("name", SEARCHES)
def test_binary_searches_reject_null_popcounts_and_unaligned_rows(name):
    for kw in ({"qs": None}, {"cs": None}):
        assert _call(name, **kw) == 1
        assert b"popcounts" in _lib().sgpt_last_error()
    for kw in ({"q": P + 4}, {"c": P + 8}, {"cs": P + 4}):
        assert _call(name, **kw) == 1
        assert b"16-byte aligned" in _lib().sgpt_last_error()


@pytest.mark.parametrize("name", SEARCHES)
def test_binary_searches_with_no_queries_pass_every_legal_mask_form(name):
    for mask, pitch in ((None, 0), (P, 0), (P, 4), (P, 1000)):
        assert _call(name, nq=0, mask=mask, pitch=pitch, q=None, c=None, qs=None, cs=None) == 0, _lib().sgpt_last_error()


def test_binary_gather_checks_its_operands_after_the_context():
    assert _call("sgpt_search_gather_masked") == 1
    assert b"null gather context" in _lib().sgpt_last_error()


def test_ivf_entry_points_reject_the_binary_dtype():
    lib = _lib()
    assert lib.sgpt_ivf_search_workspace_bytes(B1, 4, 8, 2, 100, 128) == -1
    assert lib.sgpt_ivf_search(B1, P, P, None, None, 4, 100, 128, P, 8, 100, P, P, 2, 10, None, P, P, P, 1 << 40,
                               None) == 1
    assert b"unknown shard dtype 3" in lib.sgpt_last_error()


def test_rerank_takes_the_binary_dtype_with_its_own_dim_rule():
    lib = _lib()
    assert lib.sgpt_rerank(B1, P, P, None, None, 2, 100, 200, 0, P, 10, 5, P, P, P, 1 << 40, None) == 1
    assert b"binary D=200 must be a positive multiple of 128" in lib.sgpt_last_error()
    assert lib.sgpt_rerank(B1, P, P, None, None, 0, 100, 256, 0, P, 10, 5, P, P, P, 1 << 40, None) == 0, \
        lib.sgpt_last_error()
    assert lib.sgpt_rerank(4, P, P, None, None, 0, 100, 256, 0, P, 10, 5, P, P, P, 1 << 40, None) == 1
    assert b"unknown shard dtype 4" in lib.sgpt_last_error()


# ---- Python layer -----------------------------------------------------------------------------------------------------
def test_corpus_shard_binary_dims_and_options():
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import SHARD_DTYPES

    assert "binary" in SHARD_DTYPES
    for D in (64, 200, 65536 + 128):
        with pytest.raises(ValueError, match="multiple of 128"):
            CorpusShard(D, 10, device="cpu", dtype="binary")
    with pytest.raises(ValueError, match="binary shards only"):
        CorpusShard(128, 10, device="cpu", dtype="int8", thresholds=np.zeros(128, np.float32))
    with pytest.raises(ValueError, match="thresholds must be"):
        CorpusShard(128, 10, device="cpu", dtype="binary", thresholds=np.zeros(64, np.float32))
    s = CorpusShard(256, 10, device="cpu", dtype="binary")
    assert s.vectors.shape == (10, 32) and str(s.vectors.dtype) == "torch.uint8"
    assert s.popcounts.shape == (10,) and s.thresholds.shape == (256,) and float(s.thresholds.abs().sum()) == 0.0
    assert s._dtype_id() == B1


def test_rescore_and_refine_are_rejected_on_other_dtypes():
    import torch

    from sgpt_b200 import CorpusShard

    s = CorpusShard(128, 10, device="cpu", dtype="bf16")
    for kw in ({"rescore": 20}, {"refine": s}):
        with pytest.raises(ValueError, match="binary shards only"):
            s.search(torch.zeros(1, 128), 5, **kw)


def test_exact_rerank_and_ivfpq_refine_reject_binary_shards():
    """ivfpq.rerank reads Q as rows of the shard's format, which for a binary shard would not be the fp32 rows
    sgpt_rerank's SGPT_DTYPE_B1 reads: both it and IVFPQIndex.search(refine=) refuse a binary shard before any CUDA
    call."""
    import torch

    from sgpt_b200 import CorpusShard
    from sgpt_b200.ivfpq import IVFPQIndex, rerank

    s = CorpusShard(128, 10, device="cpu", dtype="binary")
    with pytest.raises(ValueError, match="binary"):
        rerank(s, torch.zeros(2, 128), torch.zeros(2, 5, dtype=torch.int64), 3)
    index = object.__new__(IVFPQIndex)
    index.id_base, index.n, index.dim = s.id_base, s.n, s.dim
    with pytest.raises(ValueError, match="binary"):
        index.search(torch.zeros(2, 128), 3, 1, refine=s)


def test_binary_thresholds_are_the_lower_median():
    import torch

    from sgpt_b200.index import binary_thresholds

    x = torch.tensor([[1.0, 4.0], [3.0, 2.0], [2.0, 8.0], [10.0, 6.0]])
    assert binary_thresholds(x).tolist() == [2.0, 4.0]
    with pytest.raises(ValueError):
        binary_thresholds(torch.zeros(0, 4))


def test_out_of_scope_paths_reject_binary_shards():
    import torch

    from sgpt_b200 import CorpusShard
    from sgpt_b200.dist import ShardedDenseRetrievalExactSearch
    from sgpt_b200.index import semantic_search
    from sgpt_b200.ivf import IVFIndex
    from sgpt_b200.ivfpq import IVFPQIndex
    from sgpt_b200.mining import paraphrase_mining_embeddings

    s = CorpusShard(128, 10, device="cpu", dtype="binary")
    with pytest.raises(ValueError, match="binary"):
        IVFIndex.build(s, 4)
    with pytest.raises(ValueError, match="binary"):
        IVFIndex.build(torch.zeros(10, 128), 4, dtype="binary")
    with pytest.raises(ValueError, match="binary"):
        IVFPQIndex.build(s, 4, 16)
    with pytest.raises(ValueError, match="binary"):
        paraphrase_mining_embeddings(s)
    with pytest.raises(ValueError, match="binary"):
        ShardedDenseRetrievalExactSearch(None, shard_dtype="binary")
    with pytest.raises(ValueError, match="binary"):
        semantic_search(torch.zeros(1, 128), s)


def _write(path, meta, vectors, thresholds=None):
    path.mkdir()
    (path / "meta.json").write_text(json.dumps(meta))
    np.save(path / "vectors.npy", vectors)
    if thresholds is not None:
        np.save(path / "thresholds.npy", thresholds)


def test_corpus_shard_load_rejects_mismatched_bits_and_thresholds(tmp_path, monkeypatch):
    """CorpusShard.load checks the bit rows and the thresholds against meta.json before it allocates on the device."""
    import torch

    from sgpt_b200 import CorpusShard

    def no_alloc(*a, **k):
        raise AssertionError("device memory allocated before the files were checked")

    monkeypatch.setattr(torch, "empty", no_alloc)
    monkeypatch.setattr(torch, "zeros", no_alloc)
    meta = {"format": "sgpt_b200.CorpusShard/1", "dtype": "binary", "dim": 256, "n": 3, "id_base": 0}
    cases = {
        "rows": (np.zeros((4, 32), np.uint8), np.zeros(256, np.float32)),
        "width": (np.zeros((3, 16), np.uint8), np.zeros(256, np.float32)),
        "unpacked": (np.zeros((3, 256), np.uint8), np.zeros(256, np.float32)),
        "dtype": (np.zeros((3, 32), np.int8), np.zeros(256, np.float32)),
        "thr_len": (np.zeros((3, 32), np.uint8), np.zeros(128, np.float32)),
        "thr_dtype": (np.zeros((3, 32), np.uint8), np.zeros(256, np.float64)),
    }
    for name, (vec, thr) in cases.items():
        _write(tmp_path / name, meta, vec, thr)
        with pytest.raises(ValueError, match="do not match meta"):
            CorpusShard.load(str(tmp_path / name), device="cuda:0")
    bad = dict(meta, dim=200)
    _write(tmp_path / "dim", bad, np.zeros((3, 25), np.uint8), np.zeros(200, np.float32))
    with pytest.raises(ValueError, match="do not match meta"):
        CorpusShard.load(str(tmp_path / "dim"), device="cuda:0")
