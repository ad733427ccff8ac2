"""CPU checks of the IVF search: every host-side rejection of sgpt_ivf_search (before any CUDA call, dummy host pointers
that are never dereferenced), the workspace query, and the file checks of IVFIndex.load (before any device allocation)."""
import json

import numpy as np
import pytest
import torch

HOST = np.zeros(4096, dtype=np.int64)
P = (HOST.ctypes.data + 15) & ~15  # dummy 16-byte aligned host pointer, never dereferenced


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


BASE = dict(dtype=0, Q=P, C=P, nq=3, n=100, D=64, offsets=P, nlist=4, max_list_len=50, ids=P, probes=P, nprobe=2, k=10,
            out_s=P, out_i=P, ws=P, ws_bytes=1 << 40)


def _call(**kw):
    a = dict(BASE, **kw)
    return _lib().sgpt_ivf_search(a["dtype"], a["Q"], a["C"], None, None, a["nq"], a["n"], a["D"], a["offsets"],
                                  a["nlist"], a["max_list_len"], a["ids"], a["probes"], a["nprobe"], a["k"], None,
                                  a["out_s"], a["out_i"], a["ws"], a["ws_bytes"], None)


REJECTIONS = [
    (dict(dtype=-1), b"unknown shard dtype"),
    (dict(dtype=2), b"unknown shard dtype"),
    (dict(nq=-1), b"bad query count"),
    (dict(D=60), b"positive multiple of 8"),
    (dict(D=0), b"positive multiple of 8"),
    (dict(dtype=1, D=72), b"positive multiple of 16"),
    (dict(dtype=1, D=65552, n=10, max_list_len=10), b"at most 65536"),
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
    (dict(Q=None), b"null input"),
    (dict(C=None), b"null input"),
    (dict(offsets=None), b"null input"),
    (dict(ids=None), b"null input"),
    (dict(probes=None), b"null input"),
    (dict(out_s=None), b"null output"),
    (dict(out_i=None), b"null output"),
    (dict(Q=P + 8), b"16-byte aligned"),
    (dict(ws=None), b"workspace too small"),
    (dict(ws_bytes=100), b"workspace too small"),
]


PTR_ARGS = {"Q", "C", "offsets", "ids", "probes", "out_s", "out_i", "ws"}


def _case_id(bad):
    """Test id of a rejection.  A pointer is named by its offset from P: the address itself changes from run to run."""
    return ",".join(f"{k}=P+{v - P}" if k in PTR_ARGS and v is not None else f"{k}={v}" for k, v in bad.items())


@pytest.mark.parametrize("bad,msg", REJECTIONS, ids=[_case_id(b) for b, _ in REJECTIONS])
def test_ivf_search_rejects_bad_arguments(bad, msg):
    """Each rejection returns SGPT_ERR_INVALID with its message, before any CUDA call (no GPU needed)."""
    assert _call(**bad) == 1
    assert msg in _lib().sgpt_last_error(), _lib().sgpt_last_error()


@pytest.mark.parametrize("dtype,D", [(0, 64), (1, 64), (0, 8), (1, 4096)])
def test_ivf_workspace_is_exact_and_legal_calls_pass(dtype, D):
    """The workspace query's size is the least the search accepts; nq = 0 returns SGPT_OK without touching the device."""
    lib = _lib()
    need = lib.sgpt_ivf_search_workspace_bytes(dtype, 0, 4, 2, 50, D)
    assert need > 0
    assert _call(dtype=dtype, D=D, nq=0, ws_bytes=need) == 0, lib.sgpt_last_error()
    assert _call(dtype=dtype, D=D, nq=0, ws_bytes=need - 1) == 1
    assert b"workspace too small" in lib.sgpt_last_error()
    # a larger batch needs more (query blocks of 256 reuse it: 256 and 1000 queries need the same)
    a, b, c = (lib.sgpt_ivf_search_workspace_bytes(dtype, nq, 4, 2, 50, D) for nq in (7, 256, 1000))
    assert need < a < b == c
    # int8 rows take half the bytes of bf16 rows in the gathered query block
    if dtype == 0:
        assert lib.sgpt_ivf_search_workspace_bytes(1, 256, 4, 2, 50, D) < b


def test_ivf_workspace_query_rejects_what_the_search_rejects():
    lib = _lib()
    for args in ((2, 3, 4, 2, 50, 64), (0, -1, 4, 2, 50, 64), (0, 3, 4, 5, 50, 64), (0, 3, 0, 1, 50, 64),
                 (0, 3, 4, 2, -1, 64), (0, 3, 4, 2, 50, 60), (1, 3, 4, 2, 50, 72)):
        assert lib.sgpt_ivf_search_workspace_bytes(*args) == -1, args


# ---- IVFIndex.load -----------------------------------------------------------------------------------------------
def _write_index(path, n=40, dim=32, nlist=3, centroids=None, offsets=None, ids=None, shard_n=None):
    path.mkdir()
    meta = {"format": "sgpt_b200.IVFIndex/1", "dtype": "int8", "dim": dim, "n": n, "nlist": nlist, "id_base": 100,
            "score_function": "cos_sim", "shard": "shard"}
    (path / "meta.json").write_text(json.dumps(meta))
    np.save(path / "centroids.npy", np.zeros((nlist, dim), np.float32) if centroids is None else centroids)
    np.save(path / "offsets.npy", np.array([0, 10, 25, n], np.int64) if offsets is None else offsets)
    np.save(path / "ids.npy", (np.arange(n, dtype=np.int32)[::-1] + 100) if ids is None else ids)
    sd = path / "shard"
    sd.mkdir()
    sn = n if shard_n is None else shard_n
    (sd / "meta.json").write_text(json.dumps({"format": "sgpt_b200.CorpusShard/1", "dtype": "int8", "dim": dim, "n": sn,
                                              "id_base": 0, "deleted": "deleted.npy"}))
    np.save(sd / "vectors.npy", np.zeros((sn, dim), np.int8))
    np.save(sd / "scales.npy", np.zeros((sn, 2), np.float32))
    np.save(sd / "deleted.npy", np.zeros((sn + 31) // 32, np.uint32))


BAD_INDEXES = {
    "centroid_shape": (dict(centroids=np.zeros((2, 32), np.float32)), "centroids"),
    "centroid_dtype": (dict(centroids=np.zeros((3, 32), np.float64)), "centroids"),
    "offsets_shape": (dict(offsets=np.array([0, 10, 40], np.int64)), "offsets"),
    "offsets_dtype": (dict(offsets=np.array([0, 10, 25, 40], np.int32)), "offsets"),
    "offsets_not_monotone": (dict(offsets=np.array([0, 30, 25, 40], np.int64)), "monotonically"),
    "offsets_start": (dict(offsets=np.array([1, 10, 25, 40], np.int64)), "monotonically"),
    "offsets_end": (dict(offsets=np.array([0, 10, 25, 39], np.int64)), "monotonically"),
    "ids_shape": (dict(ids=np.arange(39, dtype=np.int32) + 100), "ids"),
    "ids_dtype": (dict(ids=np.arange(40, dtype=np.int64) + 100), "ids"),
    "ids_below": (dict(ids=np.arange(40, dtype=np.int32) + 99), "permutation"),
    "ids_above": (dict(ids=np.arange(40, dtype=np.int32) + 101), "permutation"),
    "ids_duplicate": (dict(ids=np.r_[np.arange(39), 0].astype(np.int32) + 100), "permutation"),
    "shard_size": (dict(shard_n=41), "inner shard"),
}


@pytest.mark.parametrize("name", sorted(BAD_INDEXES))
def test_ivf_load_rejects_bad_files_before_allocating(tmp_path, monkeypatch, name):
    from sgpt_b200 import IVFIndex

    def no_alloc(*a, **k):
        raise AssertionError("device memory allocated before the files were checked")

    kw, msg = BAD_INDEXES[name]
    _write_index(tmp_path / name, **kw)
    monkeypatch.setattr(torch, "empty", no_alloc)
    monkeypatch.setattr(torch, "zeros", no_alloc)
    with pytest.raises(ValueError, match=msg):
        IVFIndex.load(str(tmp_path / name), device="cuda:0")


def test_ivf_load_reaches_the_device_only_with_consistent_files(tmp_path, monkeypatch):
    """The well-formed directory passes every check: the first device allocation is the inner shard's."""
    from sgpt_b200 import IVFIndex

    class Reached(Exception):
        pass

    def stop(*a, **k):
        raise Reached()

    _write_index(tmp_path / "ok")
    monkeypatch.setattr(torch, "empty", stop)
    with pytest.raises(Reached):
        IVFIndex.load(str(tmp_path / "ok"), device="cuda:0")
