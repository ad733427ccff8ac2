"""CPU checks of sgpt_ivf_range_search: every host-side rejection (before any CUDA call, dummy host pointers that are
never dereferenced), the workspace query, and the argument errors of mining over an IVFIndex that need no device."""
import math

import pytest

from tests.test_ivf_cpu import BASE, P, REJECTIONS, _case_id, _lib


def _call_range(mask=None, pitch=0, threshold=0.5, counts=P, cap=10, **kw):
    a = dict(BASE, **kw)
    return _lib().sgpt_ivf_range_search(a["dtype"], a["Q"], a["C"], None, None, a["nq"], a["n"], a["D"], a["offsets"],
                                        a["nlist"], a["max_list_len"], a["ids"], a["probes"], a["nprobe"], threshold,
                                        mask, pitch, counts, cap, a["out_s"], a["out_i"], a["ws"], a["ws_bytes"], None)


# sgpt_ivf_search's rejections other than k (out_s / out_i are checked with cap below; the workspace has its own size)
SHARED = [(b, m) for b, m in REJECTIONS if "k" not in b and "out_s" not in b and "out_i" not in b]
MASK_REJECTIONS = [
    (dict(mask=P, pitch=-1), b"negative mask pitch -1"),
    (dict(mask=P, pitch=3), b"mask pitch 3 words is below ceil(n / 32) = 4"),
    (dict(mask=None, pitch=4), b"mask pitch 4 without a mask"),
]
OWN = [
    (dict(threshold=math.nan), b"threshold is NaN"),
    (dict(cap=-1), b"cap=-1 is negative"),
    (dict(counts=None), b"null out_counts"),
    (dict(counts=None, cap=0), b"null out_counts"),
    (dict(out_s=None), b"null out_scores / out_ids with cap=10"),
    (dict(out_i=None), b"null out_scores / out_ids with cap=10"),
    (dict(out_s=None, out_i=None, cap=1), b"null out_scores / out_ids with cap=1"),
]


def _id(bad):
    return _case_id({k: v for k, v in bad.items() if k not in ("mask", "pitch", "threshold", "counts", "cap")}) + "".join(
        f",{k}={'P' if k in ('mask', 'counts') and v is not None else v}" for k, v in bad.items()
        if k in ("mask", "pitch", "threshold", "counts", "cap"))


@pytest.mark.parametrize("bad,msg", SHARED + MASK_REJECTIONS + OWN, ids=[_id(b) for b, _ in SHARED + MASK_REJECTIONS + OWN])
def test_ivf_range_rejects_bad_arguments(bad, msg):
    """Each rejection returns SGPT_ERR_INVALID with its message, named after the range entry point, before any CUDA
    call; every mask form (none, shared, per query) is rejected alike."""
    for mask, pitch in ((None, 0), (P, 0), (P, 4)):
        kw = dict(dict(mask=mask, pitch=pitch), **bad)
        assert _call_range(**kw) == 1, kw
        err = _lib().sgpt_last_error()
        assert msg in err and err.startswith(b"sgpt_ivf_range_search"), err


def test_ivf_range_ignores_k_rules_and_accepts_cap_zero_without_outputs():
    """k has no part in the range search; cap = 0 only counts, so null out_scores / out_ids are legal (nq = 0 touches
    no device memory)."""
    need = _lib().sgpt_ivf_range_search_workspace_bytes(0, 0, 4, 2, 50, 64)
    assert _call_range(nq=0, ws_bytes=need, cap=0, out_s=None, out_i=None) == 0, _lib().sgpt_last_error()
    assert _call_range(nq=0, ws_bytes=need, threshold=-math.inf) == 0
    assert _call_range(nq=0, ws_bytes=need, threshold=math.inf) == 0


@pytest.mark.parametrize("dtype,D", [(0, 64), (1, 64), (0, 8), (1, 4096)])
def test_ivf_range_workspace_is_exact(dtype, D):
    """The workspace query's size is the least the range search accepts, and it holds the top-k search's workspace."""
    lib = _lib()
    for nq in (0, 7, 300):
        need = lib.sgpt_ivf_range_search_workspace_bytes(dtype, nq, 4, 2, 50, D)
        assert need > lib.sgpt_ivf_search_workspace_bytes(dtype, nq, 4, 2, 50, D) > 0
        if nq == 0:
            assert _call_range(dtype=dtype, D=D, nq=0, ws_bytes=need) == 0, lib.sgpt_last_error()
        assert _call_range(dtype=dtype, D=D, nq=nq, ws_bytes=need - 1) == 1
        assert b"workspace too small" in lib.sgpt_last_error()
    assert _call_range(ws=None, nq=0, ws_bytes=1 << 40) == 1


def test_ivf_range_workspace_query_rejects_what_the_search_rejects():
    lib = _lib()
    for args in ((2, 3, 4, 2, 50, 64), (0, -1, 4, 2, 50, 64), (0, 3, 4, 5, 50, 64), (0, 3, 0, 1, 50, 64),
                 (0, 3, 4, 0, 50, 64), (0, 3, 4, 2, -1, 64), (0, 3, 4, 2, 50, 60), (1, 3, 4, 2, 50, 72),
                 (0, 3, 4, 2, 1 << 31, 64), (0, 3, 4096, 4096, 1 << 20, 64)):
        assert lib.sgpt_ivf_range_search_workspace_bytes(*args) == -1, args
        assert lib.sgpt_ivf_search_workspace_bytes(*args) == -1, args


# ---- mining arguments ---------------------------------------------------------------------------------------------
def _fake_index(score_function):
    """An IVFIndex with nothing but its score function: the argument checks run before any device work."""
    from sgpt_b200 import IVFIndex

    index = object.__new__(IVFIndex)
    index.score_function = score_function
    return index


@pytest.mark.parametrize("fn", ["paraphrase_mining_embeddings", "community_detection"])
def test_mining_nprobe_only_with_an_index(fn):
    import torch

    from sgpt_b200 import mining

    f = getattr(mining, fn)
    with pytest.raises(ValueError, match="needs nprobe"):
        f(_fake_index("cos_sim"))
    with pytest.raises(ValueError, match="nprobe applies to an IVFIndex only"):
        f(torch.zeros(4, 8), nprobe=2)


def test_mining_score_function_must_be_the_index_s():
    from sgpt_b200 import mining

    with pytest.raises(ValueError, match="differs from the IVFIndex's 'dot'"):
        mining.paraphrase_mining_embeddings(_fake_index("dot"), nprobe=1)
    with pytest.raises(ValueError, match="differs from the IVFIndex's 'cos_sim'"):
        mining.paraphrase_mining_embeddings(_fake_index("cos_sim"), nprobe=1, score_function="dot")
    with pytest.raises(ValueError, match="differs from the IVFIndex's 'dot'"):
        mining.community_detection(_fake_index("dot"), nprobe=1)
