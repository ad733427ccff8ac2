"""CPU checks of the code-width entry points sgpt_pq_tables_nbits and sgpt_ivfpq_search_nbits (every host-side rejection,
before any CUDA call, with dummy host pointers that are never dereferenced), the workspace query for a 4-bit call, the
16-codeword encoder, the nibble packing and the 4-bit file checks of IVFPQIndex.load (before any device allocation)."""
import numpy as np
import pytest
import torch

from tests.test_ivfpq_cpu import P, _case_id, _write_index

M4 = 32


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


# ---- sgpt_pq_tables_nbits -------------------------------------------------------------------------------------------
TABLES = dict(Q=P, cb=P, cent=P, probes=P, nq=3, D=64, m=M4, nbits=4, nlist=4, nprobe=2, lut_out=P, base_out=P)


def _tables(**kw):
    a = dict(TABLES, **kw)
    return _lib().sgpt_pq_tables_nbits(a["Q"], a["cb"], a["cent"], a["probes"], a["nq"], a["D"], a["m"], a["nbits"],
                                       a["nlist"], a["nprobe"], a["lut_out"], a["base_out"], None)


TABLE_REJECTIONS = [
    (dict(nq=-1), b"bad query count"),
    (dict(D=60), b"positive multiple of 8"),
    (dict(m=8), b"m=8 must be a positive multiple of 16"),
    (dict(m=8192, D=8192), b"at most 4096"),
    (dict(nbits=0), b"nbits=0 must be 4 or 8"),
    (dict(nbits=2), b"nbits=2 must be 4 or 8"),
    (dict(nbits=16), b"nbits=16 must be 4 or 8"),
    (dict(m=16), b"m=16 must be a multiple of 32 for 4-bit codes"),
    (dict(m=48, D=96), b"m=48 must be a multiple of 32 for 4-bit codes"),
    (dict(D=96, m=64), b"D=96 is not a multiple of m=64"),
    (dict(nlist=0, nprobe=1), b"nlist=0 must be positive"),
    (dict(nprobe=5), b"nprobe=5 outside [1, nlist=4]"),
    (dict(Q=None), b"null input"),
    (dict(cb=None), b"null input"),
    (dict(lut_out=None), b"null output"),
    (dict(base_out=None), b"null output"),
]


@pytest.mark.parametrize("bad,msg", TABLE_REJECTIONS, ids=[_case_id(b) for b, _ in TABLE_REJECTIONS])
def test_pq_tables_nbits_rejects_bad_arguments(bad, msg):
    assert _tables(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_pq_tables_nbits:"), err


@pytest.mark.parametrize("nbits,m", [(4, 32), (8, 16), (4, 2048)])
def test_pq_tables_nbits_legal_empty_calls_pass(nbits, m):
    assert _tables(nq=0, nbits=nbits, m=m, D=4096) == 0, _lib().sgpt_last_error()


def test_pq_tables_8_bit_twin_keeps_its_name_and_rules():
    """sgpt_pq_tables is the 8-bit call: m = 16 passes and its errors carry its own name."""
    lib = _lib()
    assert lib.sgpt_pq_tables(P, P, P, P, 0, 64, 16, 4, 2, P, P, None) == 0
    assert lib.sgpt_pq_tables(P, P, P, P, 3, 64, 24, 4, 2, P, P, None) == 1
    assert lib.sgpt_last_error().startswith(b"sgpt_pq_tables:")


# ---- sgpt_ivfpq_search_nbits ----------------------------------------------------------------------------------------
SEARCH = dict(lut=P, base=P, codes=P, nq=3, n=100, m=M4, nbits=4, offsets=P, nlist=4, max_list_len=50, ids=P, probes=P,
              nprobe=2, k=10, out_s=P, out_i=P, ws=P, ws_bytes=1 << 40)


def _search(**kw):
    a = dict(SEARCH, **kw)
    return _lib().sgpt_ivfpq_search_nbits(a["lut"], a["base"], a["codes"], a["nq"], a["n"], a["m"], a["nbits"],
                                          a["offsets"], a["nlist"], a["max_list_len"], a["ids"], a["probes"],
                                          a["nprobe"], a["k"], None, a["out_s"], a["out_i"], a["ws"], a["ws_bytes"],
                                          None)


SEARCH_REJECTIONS = [
    (dict(nq=-1), b"bad query count"),
    (dict(m=0), b"m=0 must be a positive multiple of 16"),
    (dict(m=4128), b"at most 4096"),
    (dict(nbits=0), b"nbits=0 must be 4 or 8"),
    (dict(nbits=5), b"nbits=5 must be 4 or 8"),
    (dict(nbits=-8), b"nbits=-8 must be 4 or 8"),
    (dict(m=16), b"m=16 must be a multiple of 32 for 4-bit codes"),
    (dict(m=4080), b"m=4080 must be a multiple of 32 for 4-bit codes"),
    (dict(nlist=0, nprobe=1), b"nlist=0 must be positive"),
    (dict(nprobe=0), b"nprobe=0 outside [1, nlist=4]"),
    (dict(k=0), b"k=0 outside [1, 4096]"),
    (dict(k=4097), b"k=4097 outside [1, 4096]"),
    (dict(n=-1, max_list_len=0), b"corpus size n=-1"),
    (dict(max_list_len=101), b"max_list_len=101 exceeds n=100"),
    (dict(n=1 << 22, nlist=4096, nprobe=4096, max_list_len=1 << 20), b"2^32-entry selection space"),
    (dict(lut=None), b"null input"),
    (dict(codes=None), b"null input"),
    (dict(ids=None), b"null input"),
    (dict(lut=P + 4), b"16-byte aligned"),
    (dict(codes=P + 8), b"16-byte aligned"),
    (dict(out_s=None), b"null output"),
    (dict(out_i=None), b"null output"),
    (dict(ws=None), b"workspace too small"),
    (dict(ws_bytes=100), b"workspace too small"),
]


@pytest.mark.parametrize("bad,msg", SEARCH_REJECTIONS, ids=[_case_id(b) for b, _ in SEARCH_REJECTIONS])
def test_ivfpq_search_nbits_rejects_bad_arguments(bad, msg):
    assert _search(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_ivfpq_search_nbits:"), err


@pytest.mark.parametrize("m", [32, 96, 256, 288, 2048])
def test_workspace_query_covers_a_4_bit_call(m):
    """The workspace does not depend on the code width: the 8-bit query sizes a 4-bit call exactly."""
    lib = _lib()
    need = lib.sgpt_ivfpq_search_workspace_bytes(0, 4, 2, 50, m)
    assert need > 0
    assert _search(m=m, nq=0, ws_bytes=need) == 0, lib.sgpt_last_error()
    assert _search(m=m, nq=0, ws_bytes=need - 1) == 1
    assert b"workspace too small" in lib.sgpt_last_error()
    assert _search(m=m, nbits=8, nq=0, ws_bytes=need) == 0, lib.sgpt_last_error()


def test_ivfpq_search_8_bit_twin_keeps_its_name_and_rules():
    lib = _lib()
    a = dict(SEARCH, m=16)
    args = (a["lut"], a["base"], a["codes"], 0, a["n"], 16, a["offsets"], a["nlist"], a["max_list_len"], a["ids"],
            a["probes"], a["nprobe"], a["k"], None, a["out_s"], a["out_i"], a["ws"], a["ws_bytes"], None)
    assert lib.sgpt_ivfpq_search(*args) == 0, lib.sgpt_last_error()
    assert lib.sgpt_ivfpq_search(*args[:12], 0, *args[13:]) == 1
    assert lib.sgpt_last_error().startswith(b"sgpt_ivfpq_search:")


# ---- the encoder and the packing --------------------------------------------------------------------------------------
def _codes_restated(r, cb):
    """include/sgpt_b200.h: code[j] = argmin_c over the K codewords of d = 0; for t ascending: e = r_t - B_t,
    d = d + e * e (fp32, each operation rounded on its own), ties to the lowest c (np.argmin returns the first)."""
    m, K, dsub = cb.shape
    x = r.reshape(r.shape[0], m, dsub).astype(np.float32)
    d = np.zeros((r.shape[0], m, K), dtype=np.float32)
    for t in range(dsub):
        e = (x[:, :, t, None] - cb[None, :, :, t]).astype(np.float32)
        d = (d + (e * e).astype(np.float32)).astype(np.float32)
    return d.argmin(-1)


@pytest.mark.parametrize("m,D", [(32, 64), (32, 256), (64, 64)])
def test_nearest_codewords_with_16_codewords_matches_the_documented_definition(m, D):
    from sgpt_b200.ivfpq import _nearest_codewords

    g = torch.Generator().manual_seed(m * 3 + D)
    cb = torch.randn(m, 16, D // m, generator=g)
    cb[:, 12:] = cb[:, 3:7]  # codewords 12..15 repeat 3..6: a tie must pick the lower index
    r = torch.randn(900, D, generator=g)
    r[:40] = cb[:, 13].reshape(1, -1).expand(40, -1)  # rows sitting exactly on a duplicated codeword
    got = _nearest_codewords(r, cb).numpy()
    want = _codes_restated(r.numpy(), cb.numpy())
    assert np.array_equal(got, want)
    assert (got[:40] == 4).all() and not (got >= 12).any() and got.max() < 16


def _pack_restated(codes):
    """include/sgpt_b200.h: code j of a row is in byte j >> 1, the low nibble for even j, the high nibble for odd j."""
    T, m = codes.shape
    out = np.zeros((T, m // 2), np.uint8)
    for j in range(m):
        out[:, j >> 1] |= (codes[:, j].astype(np.uint8) << (4 * (j & 1))).astype(np.uint8)
    return out


def test_nibble_packing_matches_the_documented_layout():
    from sgpt_b200.ivfpq import _pack_codes

    g = torch.Generator().manual_seed(1)
    codes = torch.randint(0, 16, (300, 64), generator=g)
    got = _pack_codes(codes, 4).numpy()
    assert got.dtype == np.uint8 and got.shape == (300, 32)
    assert np.array_equal(got, _pack_restated(codes.numpy()))
    # unpacking restores every code; the 8-bit width stores the codes as they are
    assert np.array_equal(np.stack([got & 15, got >> 4], -1).reshape(300, 64), codes.numpy())
    c8 = torch.randint(0, 256, (5, 16), generator=g)
    assert torch.equal(_pack_codes(c8, 8), c8.to(torch.uint8))


# ---- IVFPQIndex.load of 4-bit directories ------------------------------------------------------------------------------
def _write4(path, m=M4, dim=64, n=40, nlist=3, **over):
    arrays = {"codebooks": np.zeros((m, 16, dim // m), np.float32), "codes": np.zeros((n, m // 2), np.uint8),
              "centroids": np.zeros((nlist, dim), np.float32)}
    arrays.update(over.pop("arrays", {}))
    meta = {"nbits": 4, "m": m, "dim": dim}
    meta.update(over.pop("meta", {}))
    _write_index(path, n=n, dim=dim, m=m, nlist=nlist, meta=meta, **arrays)


BAD_4BIT = {
    "nbits_3": (dict(meta={"nbits": 3}), "nbits"),
    "nbits_16": (dict(meta={"nbits": 16}), "nbits"),
    "nbits_text": (dict(meta={"nbits": "4"}), "nbits"),
    "m_not_32": (dict(m=16, dim=64, arrays={"codebooks": np.zeros((16, 16, 4), np.float32),
                                             "codes": np.zeros((40, 8), np.uint8)}), "multiple of 32"),
    "code_width_8bit": (dict(arrays={"codes": np.zeros((40, 32), np.uint8)}), "codes"),
    "code_width_short": (dict(arrays={"codes": np.zeros((40, 15), np.uint8)}), "codes"),
    "codebook_K_256": (dict(arrays={"codebooks": np.zeros((32, 256, 2), np.float32)}), "codebooks"),
    "codebook_K_8": (dict(arrays={"codebooks": np.zeros((32, 8, 2), np.float32)}), "codebooks"),
    "codebook_dsub": (dict(arrays={"codebooks": np.zeros((32, 16, 4), np.float32)}), "codebooks"),
    "eight_bit_meta_4bit_files": (dict(meta={"nbits": 8}), "codebooks"),
}


@pytest.mark.parametrize("name", sorted(BAD_4BIT))
def test_load_rejects_bad_4_bit_directories_before_allocating(tmp_path, monkeypatch, name):
    from sgpt_b200 import IVFPQIndex

    def no_alloc(*a, **k):
        raise AssertionError("the index was constructed before the files were checked")

    kw, msg = BAD_4BIT[name]
    _write4(tmp_path / name, **kw)
    monkeypatch.setattr(IVFPQIndex, "__init__", no_alloc)
    monkeypatch.setattr(torch, "empty", no_alloc)
    monkeypatch.setattr(torch, "zeros", no_alloc)
    with pytest.raises(ValueError, match=msg):
        IVFPQIndex.load(str(tmp_path / name), device="cuda:0")


def test_load_reaches_the_device_with_a_consistent_4_bit_directory(tmp_path, monkeypatch):
    from sgpt_b200 import IVFPQIndex

    class Reached(Exception):
        pass

    def stop(self, centroids, codebooks, codes, *rest):
        assert tuple(codebooks.shape) == (M4, 16, 2) and tuple(codes.shape) == (40, M4 // 2)
        raise Reached()

    _write4(tmp_path / "ok")
    monkeypatch.setattr(IVFPQIndex, "__init__", stop)
    with pytest.raises(Reached):
        IVFPQIndex.load(str(tmp_path / "ok"), device="cuda:0")


def test_train_rejects_bad_4_bit_shapes():
    from sgpt_b200 import IVFPQIndex

    with pytest.raises(ValueError, match="multiple of 32"):
        IVFPQIndex.train(torch.zeros(300, 64), 4, 16, device="cpu", nbits=4)
    with pytest.raises(ValueError, match="nbits=6"):
        IVFPQIndex.train(torch.zeros(300, 64), 4, 32, device="cpu", nbits=6)
    with pytest.raises(ValueError, match="too small"):
        IVFPQIndex.train(torch.zeros(15, 64), 4, 32, device="cpu", nbits=4)
