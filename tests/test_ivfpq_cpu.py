"""CPU checks of the IVF-PQ entry points: every host-side rejection of sgpt_pq_tables, sgpt_ivfpq_search and sgpt_rerank
(before any CUDA call, dummy host pointers that are never dereferenced), the workspace queries, and the file checks of
IVFPQIndex.load (before any device allocation)."""
import json

import numpy as np
import pytest
import torch

HOST = np.zeros(4096, dtype=np.int64)
P = (HOST.ctypes.data + 15) & ~15  # dummy 16-byte aligned host pointer, never dereferenced
PTR_ARGS = {"Q", "C", "cb", "cent", "lut", "base", "codes", "offsets", "ids", "probes", "cand", "out_s", "out_i", "ws",
            "lut_out", "base_out"}


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


def _case_id(bad):
    return ",".join(f"{k}=P+{v - P}" if k in PTR_ARGS and v is not None else f"{k}={v}" for k, v in bad.items())


# ---- sgpt_pq_tables ---------------------------------------------------------------------------------------------------
TABLES = dict(Q=P, cb=P, cent=P, probes=P, nq=3, D=64, m=16, nlist=4, nprobe=2, lut_out=P, base_out=P)


def _tables(**kw):
    a = dict(TABLES, **kw)
    return _lib().sgpt_pq_tables(a["Q"], a["cb"], a["cent"], a["probes"], a["nq"], a["D"], a["m"], a["nlist"],
                                 a["nprobe"], a["lut_out"], a["base_out"], None)


TABLE_REJECTIONS = [
    (dict(nq=-1), b"bad query count"),
    (dict(D=60), b"positive multiple of 8"),
    (dict(D=0), b"positive multiple of 8"),
    (dict(m=8), b"m=8 must be a positive multiple of 16"),
    (dict(m=24), b"m=24 must be a positive multiple of 16"),
    (dict(m=8192, D=8192), b"at most 4096"),
    (dict(D=80, m=32), b"D=80 is not a multiple of m=32"),
    (dict(nlist=0, nprobe=1), b"nlist=0 must be positive"),
    (dict(nprobe=0), b"nprobe=0 outside [1, nlist=4]"),
    (dict(nprobe=5), b"nprobe=5 outside [1, nlist=4]"),
    (dict(Q=None), b"null input"),
    (dict(cb=None), b"null input"),
    (dict(cent=None), b"null input"),
    (dict(probes=None), b"null input"),
    (dict(lut_out=None), b"null output"),
    (dict(base_out=None), b"null output"),
]


@pytest.mark.parametrize("bad,msg", TABLE_REJECTIONS, ids=[_case_id(b) for b, _ in TABLE_REJECTIONS])
def test_pq_tables_rejects_bad_arguments(bad, msg):
    assert _tables(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_pq_tables"), err


def test_pq_tables_legal_empty_call_passes():
    assert _tables(nq=0) == 0, _lib().sgpt_last_error()


# ---- sgpt_ivfpq_search ------------------------------------------------------------------------------------------------
SEARCH = dict(lut=P, base=P, codes=P, nq=3, n=100, m=16, offsets=P, nlist=4, max_list_len=50, ids=P, probes=P, nprobe=2,
              k=10, out_s=P, out_i=P, ws=P, ws_bytes=1 << 40)


def _search(**kw):
    a = dict(SEARCH, **kw)
    return _lib().sgpt_ivfpq_search(a["lut"], a["base"], a["codes"], a["nq"], a["n"], a["m"], a["offsets"], a["nlist"],
                                    a["max_list_len"], a["ids"], a["probes"], a["nprobe"], a["k"], None, a["out_s"],
                                    a["out_i"], a["ws"], a["ws_bytes"], None)


# the rejections of sgpt_ivf_search (tests/test_ivf_cpu.py) that apply, with the same wording, plus the m rules
SEARCH_REJECTIONS = [
    (dict(nq=-1), b"bad query count"),
    (dict(m=0), b"m=0 must be a positive multiple of 16"),
    (dict(m=40), b"m=40 must be a positive multiple of 16"),
    (dict(m=4112), b"at most 4096"),
    (dict(nlist=0, nprobe=1), b"nlist=0 must be positive"),
    (dict(nprobe=0), b"nprobe=0 outside [1, nlist=4]"),
    (dict(nprobe=5), b"nprobe=5 outside [1, nlist=4]"),
    (dict(k=0), b"k=0 outside [1, 4096]"),
    (dict(k=4097), b"k=4097 outside [1, 4096]"),
    (dict(n=-1, max_list_len=0), b"corpus size n=-1"),
    (dict(n=1 << 31), b"corpus size n=2147483648"),
    (dict(max_list_len=-1), b"max_list_len=-1 outside"),
    (dict(max_list_len=101), b"max_list_len=101 exceeds n=100"),
    (dict(n=1 << 22, nlist=4096, nprobe=4096, max_list_len=1 << 20), b"2^32-entry selection space"),
    (dict(nq=256, nlist=1 << 24, nprobe=1 << 24, max_list_len=1), b"pairs per block"),
    (dict(lut=None), b"null input"),
    (dict(base=None), b"null input"),
    (dict(codes=None), b"null input"),
    (dict(offsets=None), b"null input"),
    (dict(ids=None), b"null input"),
    (dict(probes=None), b"null input"),
    (dict(lut=P + 4), b"16-byte aligned"),
    (dict(codes=P + 8), b"16-byte aligned"),
    (dict(out_s=None), b"null output"),
    (dict(out_i=None), b"null output"),
    (dict(ws=None), b"workspace too small"),
    (dict(ws_bytes=100), b"workspace too small"),
]


@pytest.mark.parametrize("bad,msg", SEARCH_REJECTIONS, ids=[_case_id(b) for b, _ in SEARCH_REJECTIONS])
def test_ivfpq_search_rejects_bad_arguments(bad, msg):
    assert _search(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_ivfpq_search"), err


@pytest.mark.parametrize("m", [16, 96, 512])
def test_ivfpq_workspace_is_exact_and_legal_calls_pass(m):
    lib = _lib()
    need = lib.sgpt_ivfpq_search_workspace_bytes(0, 4, 2, 50, m)
    assert need > 0
    assert _search(m=m, nq=0, ws_bytes=need) == 0, lib.sgpt_last_error()
    assert _search(m=m, nq=0, ws_bytes=need - 1) == 1
    assert b"workspace too small" in lib.sgpt_last_error()
    # blocks of 256 queries reuse the workspace: 256 and 1000 queries need the same
    a, b, c = (lib.sgpt_ivfpq_search_workspace_bytes(nq, 4, 2, 50, m) for nq in (7, 256, 1000))
    assert need < a < b == c
    # (score, id) slots of every pair's list: 256 queries x 2 probes x 50 entries x 8 bytes at least
    assert b >= 256 * 2 * 50 * 8


def test_ivfpq_workspace_query_rejects_what_the_search_rejects():
    lib = _lib()
    for args in ((-1, 4, 2, 50, 16), (3, 4, 5, 50, 16), (3, 0, 1, 50, 16), (3, 4, 2, -1, 16), (3, 4, 2, 50, 8),
                 (3, 4, 2, 50, 40), (3, 4, 2, 50, 8192)):
        assert lib.sgpt_ivfpq_search_workspace_bytes(*args) == -1, args


# ---- sgpt_rerank --------------------------------------------------------------------------------------------------
RERANK = dict(dtype=0, Q=P, C=P, nq=3, n=100, D=64, id_base=0, cand=P, kc=40, k=10, out_s=P, out_i=P, ws=P,
              ws_bytes=1 << 40)


def _rerank(**kw):
    a = dict(RERANK, **kw)
    return _lib().sgpt_rerank(a["dtype"], a["Q"], a["C"], None, None, a["nq"], a["n"], a["D"], a["id_base"], a["cand"],
                              a["kc"], a["k"], a["out_s"], a["out_i"], a["ws"], a["ws_bytes"], None)


RERANK_REJECTIONS = [
    (dict(dtype=-1), b"unknown shard dtype"),
    (dict(dtype=2), b"unknown shard dtype"),
    (dict(nq=-1), b"bad query count"),
    (dict(kc=0), b"kc=0 outside"),
    (dict(kc=(1 << 24) + 1), b"kc=16777217 outside"),
    (dict(D=60), b"positive multiple of 8"),
    (dict(D=0), b"positive multiple of 8"),
    (dict(dtype=1, D=72), b"positive multiple of 16"),
    (dict(dtype=1, D=65552), b"at most 65536"),
    (dict(n=-1), b"corpus size n=-1"),
    (dict(n=1 << 31), b"corpus size n=2147483648"),
    (dict(id_base=-1), b"must fit in int32"),
    (dict(id_base=(1 << 31) - 50), b"must fit in int32"),
    (dict(k=0), b"k=0 outside [1, 4096]"),
    (dict(k=4097), b"k=4097 outside [1, 4096]"),
    (dict(Q=None), b"null input"),
    (dict(C=None), b"null input"),
    (dict(cand=None), b"null input"),
    (dict(Q=P + 8), b"16-byte aligned"),
    (dict(C=P + 2), b"16-byte aligned"),
    (dict(out_s=None), b"null output"),
    (dict(out_i=None), b"null output"),
    (dict(ws=None), b"workspace too small"),
    (dict(ws_bytes=100), b"workspace too small"),
]


@pytest.mark.parametrize("bad,msg", RERANK_REJECTIONS, ids=[_case_id(b) for b, _ in RERANK_REJECTIONS])
def test_rerank_rejects_bad_arguments(bad, msg):
    assert _rerank(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_rerank"), err


def test_rerank_workspace_is_exact():
    lib = _lib()
    need = lib.sgpt_rerank_workspace_bytes(3, 40)
    assert need >= 3 * 40 * 8
    assert lib.sgpt_rerank_workspace_bytes(7, 40) > need
    assert _rerank(nq=0, ws_bytes=lib.sgpt_rerank_workspace_bytes(0, 40)) == 0, lib.sgpt_last_error()
    assert _rerank(nq=0, ws_bytes=lib.sgpt_rerank_workspace_bytes(0, 40) - 1) == 1
    assert b"workspace too small" in lib.sgpt_last_error()
    for args in ((-1, 40), (3, 0), (3, (1 << 24) + 1)):
        assert lib.sgpt_rerank_workspace_bytes(*args) == -1, args


# ---- IVFPQIndex.load ----------------------------------------------------------------------------------------------
def _write_index(path, n=40, dim=32, m=16, nlist=3, **over):
    path.mkdir()
    meta = {"format": "sgpt_b200.IVFPQIndex/1", "dim": dim, "m": m, "nbits": 8, "n": n, "nlist": nlist, "id_base": 100,
            "score_function": "cos_sim"}
    meta.update(over.pop("meta", {}))
    (path / "meta.json").write_text(json.dumps(meta))
    arrays = {"centroids": np.zeros((nlist, dim), np.float32), "codebooks": np.zeros((m, 256, dim // m), np.float32),
              "codes": np.zeros((n, m), np.uint8), "offsets": np.array([0, 10, 25, n], np.int64),
              "ids": np.arange(n, dtype=np.int32)[::-1] + 100, "deleted": np.zeros((n + 31) // 32, np.uint32)}
    arrays.update(over)
    for name, a in arrays.items():
        np.save(path / f"{name}.npy", a)


BAD_INDEXES = {
    "format": (dict(meta={"format": "sgpt_b200.IVFIndex/1"}), "not an IVFPQIndex"),
    "nbits": (dict(meta={"nbits": 4}), "nbits"),
    "m_rule": (dict(meta={"m": 8}), "multiple of 16"),
    "score_function": (dict(meta={"score_function": "l2"}), "score function"),
    "centroid_shape": (dict(centroids=np.zeros((2, 32), np.float32)), "centroids"),
    "centroid_dtype": (dict(centroids=np.zeros((3, 32), np.float64)), "centroids"),
    "codebook_shape": (dict(codebooks=np.zeros((16, 255, 2), np.float32)), "codebooks"),
    "codebook_dtype": (dict(codebooks=np.zeros((16, 256, 2), np.float16)), "codebooks"),
    "codes_shape": (dict(codes=np.zeros((40, 32), np.uint8)), "codes"),
    "codes_dtype": (dict(codes=np.zeros((40, 16), np.int8)), "codes"),
    "offsets_shape": (dict(offsets=np.array([0, 10, 40], np.int64)), "offsets"),
    "offsets_dtype": (dict(offsets=np.array([0, 10, 25, 40], np.int32)), "offsets"),
    "offsets_not_monotone": (dict(offsets=np.array([0, 30, 25, 40], np.int64)), "monotonically"),
    "offsets_start": (dict(offsets=np.array([1, 10, 25, 40], np.int64)), "monotonically"),
    "offsets_end": (dict(offsets=np.array([0, 10, 25, 39], np.int64)), "offsets"),
    "ids_shape": (dict(ids=np.arange(39, dtype=np.int32) + 100), "ids"),
    "ids_dtype": (dict(ids=np.arange(40, dtype=np.int64) + 100), "ids"),
    "ids_below": (dict(ids=np.arange(40, dtype=np.int32) + 99), "permutation"),
    "ids_above": (dict(ids=np.arange(40, dtype=np.int32) + 101), "permutation"),
    "ids_duplicate": (dict(ids=np.r_[np.arange(39), 0].astype(np.int32) + 100), "permutation"),
    "deleted_shape": (dict(deleted=np.zeros(3, np.uint32)), "deleted"),
    "deleted_dtype": (dict(deleted=np.zeros(2, np.int64)), "deleted"),
}


class _Reached(Exception):
    pass


@pytest.mark.parametrize("name", sorted(BAD_INDEXES))
def test_ivfpq_load_rejects_bad_files_before_allocating(tmp_path, monkeypatch, name):
    from sgpt_b200 import IVFPQIndex

    def no_alloc(*a, **k):
        raise AssertionError("the index was constructed before the files were checked")

    kw, msg = BAD_INDEXES[name]
    _write_index(tmp_path / name, **kw)
    monkeypatch.setattr(IVFPQIndex, "__init__", no_alloc)
    monkeypatch.setattr(torch, "empty", no_alloc)
    monkeypatch.setattr(torch, "zeros", no_alloc)
    with pytest.raises(ValueError, match=msg):
        IVFPQIndex.load(str(tmp_path / name), device="cuda:0")


def test_ivfpq_load_reaches_the_device_only_with_consistent_files(tmp_path, monkeypatch):
    """The well-formed directory passes every check: the next step is constructing the index on the device."""
    from sgpt_b200 import IVFPQIndex

    def stop(self, centroids, codebooks, codes, offsets, ids, deleted, *rest):
        assert codes.dtype == torch.uint8 and tuple(codes.shape) == (40, 16) and deleted is None
        raise _Reached()

    _write_index(tmp_path / "ok")
    monkeypatch.setattr(IVFPQIndex, "__init__", stop)
    with pytest.raises(_Reached):
        IVFPQIndex.load(str(tmp_path / "ok"), device="cuda:0")


def test_ivfpq_train_rejects_bad_shapes_and_small_samples():
    from sgpt_b200 import IVFPQIndex

    with pytest.raises(ValueError, match="multiple of 16"):
        IVFPQIndex.train(torch.zeros(300, 64), 4, 24, device="cpu")
    with pytest.raises(ValueError, match="multiple of 16"):
        IVFPQIndex.train(torch.zeros(300, 48), 4, 32, device="cpu")
    with pytest.raises(ValueError, match="too small"):
        IVFPQIndex.train(torch.zeros(255, 64), 4, 16, device="cpu")
    with pytest.raises(ValueError, match="too small"):
        IVFPQIndex.train(torch.zeros(300, 64), 301, 16, device="cpu")


# ---- the encoder's codeword definition ----------------------------------------------------------------------------
def _codes_restated(r, cb):
    """include/sgpt_b200.h: code[j] = argmin_c of d = 0; for t ascending: e = r_t - B_t, d = d + e * e (fp32, each
    operation rounded on its own), ties to the lowest c (np.argmin returns the first minimum)."""
    m, _, dsub = cb.shape
    x = r.reshape(r.shape[0], m, dsub).astype(np.float32)
    d = np.zeros((r.shape[0], m, 256), dtype=np.float32)
    for t in range(dsub):
        e = (x[:, :, t, None] - cb[None, :, :, t]).astype(np.float32)
        d = (d + (e * e).astype(np.float32)).astype(np.float32)
    return d.argmin(-1)


@pytest.mark.parametrize("m,D", [(16, 64), (32, 256), (16, 16)])
def test_nearest_codewords_matches_the_documented_definition(m, D):
    """The encoder (CPU here; the GPU test file repeats it on the device) against a numpy restatement, with duplicated
    codewords so that exact ties occur and must go to the lowest index."""
    from sgpt_b200.ivfpq import _nearest_codewords

    g = torch.Generator().manual_seed(m + D)
    cb = torch.randn(m, 256, D // m, generator=g)
    cb[:, 200:] = cb[:, 10:66]  # codewords 200.. repeat 10..65: a tie must pick the lower index
    r = torch.randn(700, D, generator=g)
    r[:50] = cb[:, 200].reshape(1, -1).expand(50, -1)  # rows sitting exactly on a duplicated codeword
    got = _nearest_codewords(r, cb).numpy()
    want = _codes_restated(r.numpy(), cb.numpy())
    assert np.array_equal(got, want)
    assert (got[:50] == 10).all() and not (got >= 200).any()
