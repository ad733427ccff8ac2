"""CPU checks of the filtered IVF-PQ search: every host-side rejection of sgpt_ivfpq_search_masked (before any CUDA call,
dummy host pointers that are never dereferenced), the allow= checks of IVFPQIndex.search before any device work, the
list-order packing of a filter with deletions against numpy, and the restatement in tests/ivfpq_filtered_ref.py on a
hand-worked case."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import ivfpq_filtered_ref as ref
from tests.test_ivfpq_cpu import P, PTR_ARGS, SEARCH_REJECTIONS


def _case_id(bad):
    return ",".join(f"{k}=P+{v - P}" if k in PTR_ARGS | {"mask"} and v is not None else f"{k}={v}"
                    for k, v in bad.items())


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


# ---- sgpt_ivfpq_search_masked ---------------------------------------------------------------------------------------
MASKED = dict(lut=P, base=P, codes=P, nq=3, n=100, m=16, nbits=8, offsets=P, nlist=4, max_list_len=50, ids=P, probes=P,
              nprobe=2, k=10, mask=None, pitch=0, out_s=P, out_i=P, ws=P, ws_bytes=1 << 40)


def _masked(**kw):
    a = dict(MASKED, **kw)
    return _lib().sgpt_ivfpq_search_masked(a["lut"], a["base"], a["codes"], a["nq"], a["n"], a["m"], a["nbits"],
                                           a["offsets"], a["nlist"], a["max_list_len"], a["ids"], a["probes"],
                                           a["nprobe"], a["k"], a["mask"], a["pitch"], a["out_s"], a["out_i"], a["ws"],
                                           a["ws_bytes"], None)


# sgpt_ivfpq_search_nbits's rejections with the same wording, then the three mask rules of sgpt_ivf_search_masked
MASKED_REJECTIONS = SEARCH_REJECTIONS + [
    (dict(nbits=5), b"nbits=5 must be 4 or 8"),
    (dict(nbits=4, m=48), b"m=48 must be a multiple of 32 for 4-bit codes"),
    (dict(mask=P, pitch=-1), b"negative mask pitch -1"),
    (dict(mask=P, pitch=3), b"mask pitch 3 words is below ceil(n / 32) = 4"),
    (dict(mask=P, pitch=1, n=33, max_list_len=33), b"mask pitch 1 words is below ceil(n / 32) = 2"),
    (dict(mask=None, pitch=4), b"mask pitch 4 without a mask"),
]


@pytest.mark.parametrize("bad,msg", MASKED_REJECTIONS, ids=[_case_id(b) for b, _ in MASKED_REJECTIONS])
def test_ivfpq_search_masked_rejects_bad_arguments(bad, msg):
    assert _masked(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_ivfpq_search_masked:"), err


@pytest.mark.parametrize("nbits,m", [(8, 16), (4, 32), (4, 512)])
@pytest.mark.parametrize("mask,pitch", [(None, 0), (P, 0), (P, 4), (P, 9)], ids=["null", "shared", "exact", "padded"])
def test_ivfpq_search_masked_accepts_every_mask_form(nbits, m, mask, pitch):
    """nq = 0 makes no CUDA call: every legal mask form passes the checks, with the workspace of the unmasked search."""
    lib = _lib()
    need = lib.sgpt_ivfpq_search_workspace_bytes(0, 4, 2, 50, m)
    assert _masked(nq=0, m=m, nbits=nbits, mask=mask, pitch=pitch, ws_bytes=need) == 0, lib.sgpt_last_error()
    assert _masked(nq=0, m=m, nbits=nbits, mask=mask, pitch=pitch, ws_bytes=need - 1) == 1
    assert lib.sgpt_last_error().startswith(b"sgpt_ivfpq_search_masked: workspace too small")


# ---- IVFPQIndex: allow= ---------------------------------------------------------------------------------------------
def _host_index(n=70, id_base=9, deleted=(), seed=0):
    """An object with the fields IVFPQIndex.search and _list_mask read, on the CPU: a shuffled id -> position layout and
    deletions by position; any device work (probe, tables, scan) fails the test."""
    from sgpt_b200.index import pack_mask

    g = torch.Generator().manual_seed(seed)
    ids = (torch.randperm(n, generator=g) + id_base).to(torch.int32)
    bits = torch.zeros(n, dtype=torch.bool)
    bits[list(deleted)] = True

    def device_work(*a, **k):
        raise AssertionError("device work before the allow= checks")

    return SimpleNamespace(device=torch.device("cpu"), n=n, id_base=id_base, ids=ids,
                           _deleted=pack_mask(bits) if len(deleted) else None, probe=device_work, tables=device_work,
                           scan=device_work)


BAD_ALLOW = [
    (torch.ones(70, dtype=torch.uint8), "uint8 [70]"),
    (torch.ones(70, dtype=torch.int64), "int64 [70]"),
    (torch.ones(70), "float [70]"),
    (torch.ones(69, dtype=torch.bool), "bool [69]"),
    (torch.ones(71, dtype=torch.bool), "bool [71]"),
    (torch.ones(4, 70, dtype=torch.bool), "bool [4, 70] for 3 queries"),
    (torch.ones(2, 70, dtype=torch.bool), "bool [2, 70] for 3 queries"),
    (torch.ones(3, 69, dtype=torch.bool), "bool [3, 69]"),
    (torch.ones(1, 3, 70, dtype=torch.bool), "bool [1, 3, 70]"),
    (torch.tensor(True), "bool scalar"),
]


@pytest.mark.parametrize("allow", [a for a, _ in BAD_ALLOW], ids=[i for _, i in BAD_ALLOW])
def test_search_rejects_bad_allow_before_device_work(allow):
    from sgpt_b200 import IVFPQIndex

    index = _host_index()
    with pytest.raises(ValueError, match=r"allow must be a boolean tensor \[70\] or \[3, 70\]"):
        IVFPQIndex.search(index, torch.zeros(3, 16), 10, 2, allow=allow)
    with pytest.raises(ValueError, match="allow must be a boolean tensor"):
        IVFPQIndex._list_mask(index, allow, 3)


def _want_bits(index, allow):
    """numpy: bit p of row q = allow[q][ids[p] - id_base] and position p not deleted."""
    ids = index.ids.numpy().astype(np.int64) - index.id_base
    a = np.atleast_2d(allow.numpy())[:, ids]
    if index._deleted is not None:
        deleted = ref.allowed(index._deleted.numpy(), 0, 1, index.n)[0]
        a = a & ~deleted
    return a


@pytest.mark.parametrize("n", [1, 31, 32, 70, 97])
@pytest.mark.parametrize("deleted", [(), (0, 5, 30), "all"], ids=["none", "some", "all"])
@pytest.mark.parametrize("nq", [0, 1, 3])
def test_list_mask_packs_the_filter_in_list_order_with_deletions(n, deleted, nq):
    from sgpt_b200 import IVFPQIndex

    deleted = tuple(range(n)) if deleted == "all" else tuple(d for d in deleted if d < n)
    index = _host_index(n=n, deleted=deleted, seed=n)
    g = torch.Generator().manual_seed(n + nq)
    W = (n + 31) // 32
    # shared
    allow = torch.rand(n, generator=g) < 0.5
    mask, pitch = IVFPQIndex._list_mask(index, allow, nq)
    assert pitch == 0 and mask.dtype == torch.int32 and mask.shape == (W,) and mask.is_contiguous()
    assert np.array_equal(ref.allowed(mask.numpy(), 0, 1, n)[0], _want_bits(index, allow)[0])
    # per query: one row of ceil(n / 32) words each
    allow = torch.rand(nq, n, generator=g) < 0.5
    mask, pitch = IVFPQIndex._list_mask(index, allow, nq)
    assert pitch == W and mask.shape == (nq, W) and mask.is_contiguous()
    assert np.array_equal(ref.allowed(mask.numpy(), pitch, nq, n), _want_bits(index, allow))
    # no filter: the deletions alone, or no bitmap at all
    mask, pitch = IVFPQIndex._list_mask(index, None, nq)
    if not deleted:
        assert mask is None and pitch == 0
    else:
        assert pitch == 0 and np.array_equal(ref.allowed(mask.numpy(), 0, 1, n)[0],
                                             _want_bits(index, torch.ones(n, dtype=torch.bool))[0])


def test_list_mask_of_an_empty_index_is_shared():
    """n = 0: a [Q, 0] filter has no words, so it is passed as pitch 0 (the search makes no call then)."""
    from sgpt_b200 import IVFPQIndex

    index = _host_index(n=0)
    mask, pitch = IVFPQIndex._list_mask(index, torch.ones(3, 0, dtype=torch.bool), 3)
    assert pitch == 0 and mask.shape == (3, 0)


# ---- the restatement ------------------------------------------------------------------------------------------------
def test_restatement_on_a_hand_worked_case():
    """Two lists [0, 3) and [3, 5); 4-bit codes, m = 2 (one byte per document).  Query 0 probes both lists and its
    bitmap allows positions 0, 1, 3 and 4; query 1 probes list 1 only (and a skipped probe) with every bit set."""
    lut = np.zeros((2, 2, 16))
    lut[:, 0, :] = np.arange(16)
    lut[:, 1, :] = 100 * np.arange(16)
    codes = np.array([[0x21], [0x12], [0x03], [0x21], [0x00]], dtype=np.uint8)  # (code0, code1) = (1,2) (2,1) (3,0) ...
    offsets = np.array([0, 3, 5])
    probes = np.array([[0, 1], [1, -1]])
    base = np.array([[0.0, 1000.0], [5.0, 7.0]])
    ids = np.array([10, 11, 12, 13, -1])
    sc = ref.adc_scores(lut, base, codes, 4, offsets, probes)
    assert np.array_equal(sc[0], [201.0, 102.0, 3.0, 1201.0, 1000.0])
    assert np.isnan(sc[1, :3]).all() and np.array_equal(sc[1, 3:], [206.0, 5.0])
    mask = np.array([0b11011, -1], dtype=np.int64).astype(np.uint32)  # bits past n = 5 set in row 1
    allow = ref.allowed(mask, 1, 2, 5)
    assert np.array_equal(allow, [[True, True, False, True, True], [True] * 5])
    s, i = ref.search(sc, ids, allow, 4)
    assert i.tolist() == [[13, 10, 11, -1], [13, -1, -1, -1]]  # id -1 (position 4) is never returned
    assert s.tolist() == [[1201.0, 201.0, 102.0, -np.inf], [206.0, -np.inf, -np.inf, -np.inf]]
