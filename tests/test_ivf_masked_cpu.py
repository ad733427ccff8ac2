"""CPU checks of sgpt_ivf_search_masked: its mask rejections (the rules of the masked shard searches) and every rejection
of sgpt_ivf_search, all before any CUDA call, with dummy host pointers that are never dereferenced."""
import pytest

from tests.test_ivf_cpu import BASE, P, REJECTIONS, _call, _case_id, _lib


def _call_masked(mask=None, pitch=0, **kw):
    a = dict(BASE, **kw)
    return _lib().sgpt_ivf_search_masked(a["dtype"], a["Q"], a["C"], None, None, a["nq"], a["n"], a["D"], a["offsets"],
                                         a["nlist"], a["max_list_len"], a["ids"], a["probes"], a["nprobe"], a["k"],
                                         mask, pitch, a["out_s"], a["out_i"], a["ws"], a["ws_bytes"], None)


# BASE has n = 100 rows: ceil(n / 32) = 4 words
MASK_REJECTIONS = [
    (dict(mask=P, pitch=-1), b"negative mask pitch -1"),
    (dict(mask=None, pitch=-4), b"negative mask pitch -4"),
    (dict(mask=P, pitch=1), b"mask pitch 1 words is below ceil(n / 32) = 4"),
    (dict(mask=P, pitch=3), b"mask pitch 3 words is below ceil(n / 32) = 4"),
    (dict(mask=None, pitch=4), b"mask pitch 4 without a mask"),
    (dict(mask=None, pitch=100), b"mask pitch 100 without a mask"),
]


@pytest.mark.parametrize("bad,msg", MASK_REJECTIONS, ids=[f"mask={'P' if b['mask'] else None},pitch={b['pitch']}"
                                                          for b, _ in MASK_REJECTIONS])
def test_ivf_masked_rejects_bad_masks(bad, msg):
    assert _call_masked(**bad) == 1
    err = _lib().sgpt_last_error()
    assert msg in err and err.startswith(b"sgpt_ivf_search_masked"), err


@pytest.mark.parametrize("mask,pitch", [(None, 0), (P, 0), (P, 4), (P, 5), (P, 1 << 40)],
                         ids=["null", "shared", "pitch=words", "pitch=words+1", "pitch=2^40"])
def test_ivf_masked_accepts_the_three_pitch_rules(mask, pitch):
    """pitch 0 with or without a bitmap, and pitch >= ceil(n/32) with one: legal (nq = 0 touches no device memory)."""
    lib = _lib()
    need = lib.sgpt_ivf_search_workspace_bytes(0, 0, 4, 2, 50, 64)
    assert _call_masked(mask, pitch, nq=0, ws_bytes=need) == 0, lib.sgpt_last_error()


def test_ivf_masked_pitch_rules_follow_n():
    """ceil(n / 32) counts a partial last word: n = 97 needs 4 words, n = 96 three; n = 0 needs none."""
    need = _lib().sgpt_ivf_search_workspace_bytes(0, 0, 4, 2, 0, 64)
    assert _call_masked(P, 3, nq=0, n=97, max_list_len=0, ws_bytes=need) == 1
    assert _call_masked(P, 4, nq=0, n=97, max_list_len=0, ws_bytes=need) == 0
    assert _call_masked(P, 3, nq=0, n=96, max_list_len=0, ws_bytes=need) == 0
    assert _call_masked(P, 1, nq=0, n=0, max_list_len=0, ws_bytes=need) == 0


@pytest.mark.parametrize("bad,msg", REJECTIONS, ids=[_case_id(b) for b, _ in REJECTIONS])
def test_ivf_masked_makes_every_rejection_of_the_unmasked_search(bad, msg):
    """Each sgpt_ivf_search rejection, with a valid mask (none, shared and per query), is also the masked call's."""
    assert _call(**bad) == 1
    for mask, pitch in ((None, 0), (P, 0), (P, 4)):
        assert _call_masked(mask, pitch, **bad) == 1
        err = _lib().sgpt_last_error()
        assert msg in err and err.startswith(b"sgpt_ivf_search_masked"), err
