"""CPU checks of the masked (filtered) searches and of CorpusShard's deletion bitmap: the argument rejections of the four
masked entry points (before any CUDA call), the deletion checks of CorpusShard.load (before any device allocation), and
the bitmap packing against a NumPy restatement of the format in include/sgpt_b200.h."""
import json

import numpy as np
import pytest
import torch

HOST = np.zeros(4096, dtype=np.int64)
P = HOST.ctypes.data  # dummy host pointer, never dereferenced


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


def _call(name, mask=P, pitch=0, dtype=0, n=100, nq=3, D=64, k=10):
    lib = _lib()
    if name == "sgpt_search_masked":
        return lib.sgpt_search_masked(dtype, P, P, None, None, nq, n, D, k, 0, mask, pitch, P, P, P, 1 << 40, None)
    if name == "sgpt_search_packed_masked":
        return lib.sgpt_search_packed_masked(dtype, P, P, None, None, nq, n, D, k, 0, mask, pitch, P, P, 1 << 40, None)
    if name == "sgpt_range_search_masked":
        return lib.sgpt_range_search_masked(dtype, P, P, None, None, nq, n, D, 0.5, 0, mask, pitch, P, 10, P, P, P,
                                            1 << 40, None)
    if name == "sgpt_search_gather_masked":
        # a null gather context is rejected first; a fake non-null one is never reached by the mask checks below
        return lib.sgpt_search_gather_masked(dtype, None, P, P, None, None, nq, n, D, k, 0, mask, pitch, None, P, P, P,
                                             1 << 40, None)
    raise ValueError(name)


SEARCHES = ["sgpt_search_masked", "sgpt_search_packed_masked", "sgpt_range_search_masked"]


@pytest.mark.parametrize("name", SEARCHES)
@pytest.mark.parametrize("n,pitch", [(100, 1), (100, 3), (32, -1), (33, 1), (0, -5)])
def test_masked_entry_points_reject_bad_pitches(name, n, pitch):
    """0 < pitch < ceil(n / 32) and negative pitches are rejected with SGPT_ERR_INVALID."""
    assert _call(name, n=n, pitch=pitch) == 1
    assert b"mask pitch" in _lib().sgpt_last_error()


@pytest.mark.parametrize("name", SEARCHES)
def test_masked_entry_points_reject_a_pitch_without_a_mask(name):
    assert _call(name, mask=None, pitch=4) == 1
    assert b"without a mask" in _lib().sgpt_last_error()


@pytest.mark.parametrize("name", SEARCHES)
@pytest.mark.parametrize("dtype", [-1, 2])
def test_masked_entry_points_reject_unknown_dtypes(name, dtype):
    assert _call(name, dtype=dtype) == 1
    assert b"unknown shard dtype" in _lib().sgpt_last_error()


@pytest.mark.parametrize("name", SEARCHES)
@pytest.mark.parametrize("dtype", [0, 1])
def test_masked_entry_points_accept_legal_masks_with_no_work(name, dtype):
    """nq = 0: every legal mask form passes the checks and returns SGPT_OK without touching the device."""
    for mask, pitch in ((None, 0), (P, 0), (P, 4), (P, 1000)):
        assert _call(name, mask=mask, pitch=pitch, dtype=dtype, nq=0) == 0, _lib().sgpt_last_error()


def test_masked_entry_points_keep_the_unmasked_checks():
    assert _call("sgpt_search_masked", dtype=1, D=60) == 1
    assert b"multiple of 16" in _lib().sgpt_last_error()
    assert _call("sgpt_search_masked", k=0) == 1
    assert _call("sgpt_search_gather_masked") == 1
    assert b"null gather context" in _lib().sgpt_last_error()


def _np_pack(allow):
    """NumPy restatement: bit j % 32 of little-endian uint32 word j // 32 = allow[..., j]."""
    a = np.asarray(allow, dtype=bool)
    n = a.shape[-1]
    padded = np.zeros(a.shape[:-1] + (-(-n // 32) * 32,), dtype=bool)
    padded[..., :n] = a
    return np.packbits(padded, axis=-1, bitorder="little").view("<u4")


@pytest.mark.parametrize("shape", [(0,), (1,), (31,), (32,), (33,), (1000,), (3, 77), (5, 64)])
def test_pack_mask_matches_numpy(shape):
    from sgpt_b200.index import pack_mask, unpack_mask

    g = torch.Generator().manual_seed(sum(shape))
    allow = torch.rand(shape, generator=g) < 0.5
    got = pack_mask(allow)
    want = _np_pack(allow.numpy())
    assert got.dtype == torch.int32
    assert np.array_equal(got.numpy().view(np.uint32), want)
    assert torch.equal(unpack_mask(got, shape[-1]), allow)
    ones = pack_mask(torch.ones(shape, dtype=torch.bool))
    assert np.array_equal(ones.numpy().view(np.uint32), _np_pack(np.ones(shape, dtype=bool)))  # bits past n are 0


@pytest.mark.parametrize("start", [0, 1, 31, 32, 45, 64, 100])
def test_bit_slice_shifts_a_bitmap(start):
    """A view's bitmap: bits [start, start + n) of the parent's, with bit 0 = the view's first row."""
    from sgpt_b200.index import _bit_slice, pack_mask, unpack_mask

    g = torch.Generator().manual_seed(start)
    bits = torch.rand(320, generator=g) < 0.3
    words = torch.cat([pack_mask(bits), torch.zeros(2, dtype=torch.int32)])
    for n in (0, 1, 40, 320 - start):
        assert torch.equal(unpack_mask(_bit_slice(words, start, n), n), bits[start:start + n]), n


def _write(path, meta, deleted):
    path.mkdir()
    (path / "meta.json").write_text(json.dumps(meta))
    np.save(path / "vectors.npy", np.zeros((meta["n"], meta["dim"]), np.int8))
    np.save(path / "scales.npy", np.zeros((meta["n"], 2), np.float32))
    np.save(path / "deleted.npy", deleted)


def test_corpus_shard_load_rejects_a_bad_deletion_bitmap(tmp_path, monkeypatch):
    """A deletion bitmap of the wrong length or type is rejected before anything is allocated on the device."""
    from sgpt_b200 import CorpusShard

    def no_alloc(*a, **k):
        raise AssertionError("device memory allocated before the files were checked")

    monkeypatch.setattr(torch, "empty", no_alloc)
    monkeypatch.setattr(torch, "zeros", no_alloc)
    meta = {"format": "sgpt_b200.CorpusShard/1", "dtype": "int8", "dim": 32, "n": 40, "id_base": 0,
            "deleted": "deleted.npy"}
    for name, bad in (("a", np.zeros(1, np.uint32)), ("b", np.zeros(3, np.uint32)), ("c", np.zeros(2, np.int64)),
                      ("d", np.zeros((2, 1), np.uint32))):
        _write(tmp_path / name, meta, bad)
        with pytest.raises(ValueError, match="deletion bitmap"):
            CorpusShard.load(str(tmp_path / name), device="cuda:0")


def test_corpus_shard_remove_and_mask_on_the_host(tmp_path):
    """The deletion bookkeeping is plain tensor code: on a CPU-resident shard object, remove / n_deleted / views /
    the search mask and the saved bitmap follow the format (no library call is made)."""
    from sgpt_b200.index import CorpusShard, unpack_mask

    shard = CorpusShard(32, 100, device="cpu", id_base=1000, dtype="int8")
    shard.n = 100
    assert shard.n_deleted == 0 and shard._mask(None, 4) == (None, 0)
    shard.remove([1000, 1037, 1099, 1037])
    assert shard.n_deleted == 3
    m, pitch = shard._mask(None, 4)
    assert pitch == 0 and torch.equal(~unpack_mask(m, 100), torch.isin(torch.arange(100), torch.tensor([0, 37, 99])))
    with pytest.raises(ValueError, match="ids must lie in"):
        shard.remove([999])
    v = shard.view(33, 90)  # unaligned start: the view's bit 0 is the parent's bit 33
    assert v.n_deleted == 1
    v.remove([40])  # the view's ids are positions in the parent
    assert shard.n_deleted == 4
    allow = torch.zeros(4, 57, dtype=torch.bool)
    allow[:, 4] = allow[:, 7] = True
    allow[2, 10] = True
    m, pitch = v._mask(allow, 4)
    assert pitch == 2 and m.shape == (4, 2)
    got = unpack_mask(m, 57)
    want = allow.clone()
    want[:, 4] = want[:, 7] = False  # parent rows 37 and 40 are deleted
    assert torch.equal(got, want)
    with pytest.raises(ValueError, match="boolean tensor"):
        v._mask(torch.ones(56, dtype=torch.bool), 4)
