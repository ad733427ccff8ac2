"""CPU checks of the int8 shard entry points and of CorpusShard's int8 format: every rejection happens before any CUDA
call or device allocation."""
import json

import numpy as np
import pytest

N_PTR = np.zeros(64, dtype=np.int64)
P = N_PTR.ctypes.data  # dummy host pointer, never dereferenced


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


def _call(name, D=64, n=100, nq=1, k=10, id_base=0, out=P, ws_bytes=1 << 40):
    lib = _lib()
    if name == "sgpt_search_i8":
        return lib.sgpt_search_i8(P, P, None, None, nq, n, D, k, id_base, out, out, P, ws_bytes, None)
    if name == "sgpt_search_packed_i8":
        return lib.sgpt_search_packed_i8(P, P, None, None, nq, n, D, k, id_base, out, P, ws_bytes, None)
    if name == "sgpt_range_search_i8":
        return lib.sgpt_range_search_i8(P, P, None, None, nq, n, D, 0.5, id_base, out, 10, out, out, P, ws_bytes, None)
    if name == "sgpt_scores_i8":
        return lib.sgpt_scores_i8(P, P, None, None, out, n, nq, n, D, None)
    if name == "sgpt_quantize_rows_i8":
        return lib.sgpt_quantize_rows_i8(P, 0, out, out, out, n, D, None)
    raise ValueError(name)


ALL = ["sgpt_search_i8", "sgpt_search_packed_i8", "sgpt_range_search_i8", "sgpt_scores_i8", "sgpt_quantize_rows_i8"]


@pytest.mark.parametrize("name", ALL)
@pytest.mark.parametrize("D", [0, 8, 60, 65536 + 16])
def test_int8_entry_points_reject_bad_dims(name, D):
    """D % 16 == 0 (TMA row pitch of int8 rows) and D <= 65536 (no s32 overflow)."""
    assert _call(name, D=D) == 1  # SGPT_ERR_INVALID
    assert f"D={D} must be a positive multiple of 16, at most 65536".encode() in _lib().sgpt_last_error()


@pytest.mark.parametrize("name", ALL)
def test_int8_entry_points_reject_null_outputs(name):
    assert _call(name, out=None) == 1
    assert b"null" in _lib().sgpt_last_error()


@pytest.mark.parametrize("name", ["sgpt_search_i8", "sgpt_search_packed_i8", "sgpt_range_search_i8"])
def test_int8_searches_reject_a_short_workspace(name):
    assert _call(name, ws_bytes=16) == 1
    assert b"workspace too small" in _lib().sgpt_last_error()


def test_int8_packed_search_rejects_ids_beyond_31_bits():
    n = 1000
    assert _call("sgpt_search_packed_i8", n=n, id_base=(1 << 31) - n) == 1
    assert b"global ids must fit 31 bits" in _lib().sgpt_last_error()
    assert _call("sgpt_search_packed_i8", n=n, id_base=(1 << 31) - n - 1, nq=0) == 0  # largest legal id_base


def test_int8_entry_points_accept_the_largest_dim_with_no_work():
    for name in ("sgpt_scores_i8", "sgpt_quantize_rows_i8"):
        assert _call(name, D=65536, n=0) == 0, _lib().sgpt_last_error()


def test_gather_i8_rejects_a_null_context():
    lib = _lib()
    assert lib.sgpt_search_gather_i8(None, P, P, None, None, 1, 100, 64, 10, 0, None, P, P, P, 1 << 40, None) == 1
    assert b"null gather context" in lib.sgpt_last_error()


def test_corpus_shard_rejects_unknown_dtype_and_ragged_int8_dims():
    from sgpt_b200 import CorpusShard

    with pytest.raises(ValueError, match="shard dtype 'fp8'"):
        CorpusShard(64, 10, device="cpu", dtype="fp8")
    with pytest.raises(ValueError, match="multiple of 16 for int8"):
        CorpusShard(72, 10, device="cpu", dtype="int8")


def _write(path, meta, vectors, scales=None):
    path.mkdir()
    (path / "meta.json").write_text(json.dumps(meta))
    np.save(path / "vectors.npy", vectors)
    if scales is not None:
        np.save(path / "scales.npy", scales)


def test_corpus_shard_load_rejects_unknown_dtype_and_mismatched_scales(tmp_path, monkeypatch):
    """CorpusShard.load checks the directory against meta.json before it allocates anything on the device."""
    import torch

    from sgpt_b200 import CorpusShard

    def no_alloc(*a, **k):
        raise AssertionError("device memory allocated before the files were checked")

    monkeypatch.setattr(torch, "empty", no_alloc)
    meta = {"format": "sgpt_b200.CorpusShard/1", "dtype": "fp8", "dim": 32, "n": 3, "id_base": 0}
    _write(tmp_path / "a", meta, np.zeros((3, 32), np.int8), np.zeros((3, 2), np.float32))
    with pytest.raises(ValueError, match="unknown shard dtype 'fp8'"):
        CorpusShard.load(str(tmp_path / "a"), device="cuda:0")
    meta["dtype"] = "int8"
    for name, scales in (("b", np.zeros((4, 2), np.float32)), ("c", np.zeros((3,), np.float32)),
                         ("d", np.zeros((3, 2), np.float64))):
        _write(tmp_path / name, meta, np.zeros((3, 32), np.int8), scales)
        with pytest.raises(ValueError, match="do not match meta"):
            CorpusShard.load(str(tmp_path / name), device="cuda:0")
    _write(tmp_path / "e", meta, np.zeros((3, 32), np.uint16), np.zeros((3, 2), np.float32))
    with pytest.raises(ValueError, match="do not match meta"):
        CorpusShard.load(str(tmp_path / "e"), device="cuda:0")
