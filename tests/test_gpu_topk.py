"""The top-k selection kernels bit for bit against an exact reference (tests/helpers.py topk_reference), through the C ABI:
sgpt_topk on dense rows, sgpt_topk_merge on fp32 + int64 lists and sgpt_topk_merge_packed on sorted packed lists.

The reference is exact: the kernels take the score values the test builds and return a subset of them, so scores are
compared with torch.equal and ids exactly, with no tolerance.  Most distributions are tie-heavy on purpose: the contract
(include/sgpt_b200.h) is that the k winners are the first k entries in (score descending, id ascending) order, so the
result may not depend on which of several equal scores a kernel happens to meet first.

Shapes come from the launcher's arithmetic in csrc/topk.cu (launch_topk_select): a dense row is cached in shared memory
when its 32-padded length fits the dynamic shared memory left after the sort buffers (12 bytes per slot of KP, the power
of two >= k) and the first-digit buffer (kSubCap keys); longer rows take the uncached path over global memory."""
import numpy as np
import pytest
import torch

from tests.helpers import topk_reference

pytestmark = pytest.mark.gpu

SUB_CAP = 8192          # csrc/topk.cu kSubCap
SUB_PAIRS = SUB_CAP // 2  # fast-path short list capacity
MAX_FLAT_LISTS = 1024   # csrc/topk.cu kMaxFlatLists
DYN_MAX = 208 * 1024    # csrc/topk.cu launch_topk_select kDynMax
SENT_S, SENT_I = 12345.5, -77  # rows of the output buffers past nq must keep these


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _kp(k):
    kp = 2
    while kp < k:
        kp *= 2
    return kp


def cache_limit(k):
    """Longest dense row that is still cached in shared memory (pad32(n) <= room)."""
    room = (DYN_MAX - 12 * _kp(k) - 4 * SUB_CAP) // 4
    return room // 32 * 32


def _outs(nq, k):
    s = torch.full((nq + 2, k), SENT_S, dtype=torch.float32, device="cuda")
    i = torch.full((nq + 2, k), SENT_I, dtype=torch.int64, device="cuda")
    return s, i


def _check(what, run, nq, want_s, want_i):
    """run(out_s, out_i) twice: equal to the reference, identical bits the second time, rows past nq untouched."""
    got = []
    for _ in range(2):
        s, i = _outs(nq, want_s.shape[1])
        run(s, i)
        torch.cuda.synchronize()
        got.append((s.cpu(), i.cpu()))
    (s, i), (s2, i2) = got
    assert torch.equal(s[nq:], torch.full_like(s[nq:], SENT_S)) and torch.equal(i[nq:], torch.full_like(i[nq:], SENT_I)), \
        f"{what}: rows past nq were written"
    s, i = s[:nq], i[:nq]
    bad = ((i != want_i) | (s.double() != want_s)).any(dim=1).nonzero()
    if len(bad):
        q = int(bad[0])
        j = int(((i[q] != want_i[q]) | (s[q].double() != want_s[q])).nonzero()[0])
        raise AssertionError(f"{what}: query {q} rank {j}: got ({float(s[q, j])}, {int(i[q, j])}), want "
                             f"({float(want_s[q, j])}, {int(want_i[q, j])}); {len(bad)} queries differ")
    assert torch.equal(s.view(torch.int32), s2[:nq].view(torch.int32)) and torch.equal(i, i2[:nq]), \
        f"{what}: a second launch returned different bits"


# ---------------------------------------------------------------------------------------------------------------------
# score distributions of a dense row
DISTS = ["continuous", "ties40", "equal", "one_digit", "band", "ascending", "descending", "mixed"]


def _scores(dist, nq, n, k, g):
    if dist == "continuous":
        return torch.randn(nq, n, generator=g)
    if dist == "ties40":  # 40 distinct values: the cut falls inside a tie group
        return torch.randint(0, 40, (nq, n), generator=g).float() * 0.25 - 5.0
    if dist == "equal":
        return torch.full((nq, n), 0.75)
    if dist == "one_digit":  # one 11-bit first radix digit: the first-digit group exceeds kSubCap for n > 8192
        return 1.0 + torch.rand(nq, n, generator=g) * 1e-4
    if dist == "band":
        # more than SUB_PAIRS equal keys above the rest: the sampled pivot's short list overflows, so the radix fallback
        # runs, with its first-digit compaction (the band is one digit group smaller than kSubCap)
        x = torch.randn(nq, n, generator=g) * 0.1
        m = min(n, SUB_PAIRS + 700 + k // 4)
        for q in range(nq):
            x[q, torch.randperm(n, generator=g)[:m]] = 2.0
        return x
    if dist in ("ascending", "descending"):  # adversarial for the strided pivot sample
        x = torch.randint(0, max(2, n // 3), (nq, n), generator=g).float().sort(dim=1).values
        return x if dist == "ascending" else x.flip(1)
    if dist == "mixed":
        vals = torch.tensor([float("-inf"), float("inf"), -3.5, -1.0, -0.0, 0.0, 2.5, -1e-30])
        return vals[torch.randint(0, len(vals), (nq, n), generator=g)]
    raise ValueError(dist)


def _dense_case(k, dist, n, nq, id_base, seed):
    L, lib = _lib()
    g = torch.Generator().manual_seed(seed)
    x = _scores(dist, nq, n, k, g)
    lds = n + 5
    buf = torch.full((nq, lds), float("inf"))  # pad columns: +inf and NaN would win if they were read
    buf[:, n + 1::2] = float("nan")
    buf[:, :n] = x
    xd = buf.cuda()
    ws = torch.empty(256, dtype=torch.uint8, device="cuda")
    ids = torch.arange(n, dtype=torch.int64).expand(nq, n) + id_base
    want_s, want_i = topk_reference(x, ids, k)

    def run(s, i):
        L.check(lib.sgpt_topk(xd.data_ptr(), lds, nq, n, k, id_base, s.data_ptr(), i.data_ptr(), ws.data_ptr(),
                              L.current_stream()), "sgpt_topk")

    path = "empty" if n == 0 else ("cached" if ((n + 31) // 32 * 32) <= cache_limit(k) else "uncached")
    _check(f"sgpt_topk {dist} k={k} n={n} nq={nq} id_base={id_base} ({path})", run, nq, want_s, want_i)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("k", [1, 2, 31, 32, 33, 1001, 1024, 1025, 2048, 4096])
def test_topk_dense_rows_bit_exact(k, dist):
    """sgpt_topk over every path of topk_select_kernel.  Row lengths: empty, 1, around k (fewer valid entries than k
    fills the tail with (-inf, -1)), around SUB_PAIRS = 4096 (up to it the short list holds every key, no pivot sample),
    8193, either side of the shared-memory cache limit (cached: sampled pivot + compaction or the radix fallback over
    shared memory; one past it: the radix passes over global memory), and 60 000 (uncached).  k = 1025 .. 4096 sorts
    with the shared-memory bitonic loop (KP > 1024 threads).  Ties at the cut must resolve to the lowest ids."""
    lim = cache_limit(k)
    ns = sorted({0, 1, max(0, k - 1), k, k + 1, 4096, 4097, 8193, lim - 1, lim, lim + 1, 60000})
    if dist in ("continuous", "ascending", "descending", "mixed") and k not in (1, 33, 1025, 4096):
        ns = [n for n in ns if n in (k + 1, 8193, lim, 60000)]  # the rest of the grid runs on the tie-heavy data
    for j, n in enumerate(ns):
        nq = (3, 1, 130)[j % 3] if n <= 10000 else (3, 1)[j % 2]
        _dense_case(k, dist, n, nq, id_base=(0, 1 << 40)[j % 2], seed=1000 * k + j)


def test_topk_dense_130_queries_uncached_ties():
    """130 queries of 60 000 tied scores each: the uncached radix path, the straddling tie at the cut in every row."""
    _dense_case(1001, "ties40", 60000, 130, id_base=1 << 40, seed=5)
    _dense_case(1025, "equal", 41000, 130, id_base=0, seed=6)


# ---------------------------------------------------------------------------------------------------------------------
# sgpt_topk_merge: G lists of fp32 scores + int64 ids per query
def _merge_lists(G, nq, k, g, empty_frac=0.2):
    """Unsorted lists with tie-heavy scores, unique ids per query beyond 2^31 and empty slots (id -1) interspersed."""
    s = (torch.randint(0, 12, (G, nq, k), generator=g).float() * 0.5 - 2.0)
    s[torch.rand(G, nq, k, generator=g) < 0.05] = -0.0
    ids = torch.empty(G, nq, k, dtype=torch.int64)
    for q in range(nq):
        ids[:, q, :] = (torch.randperm(G * k * 4, generator=g)[:G * k] * 977 + (1 << 33)).view(G, k)
    ids[torch.rand(G, nq, k, generator=g) < empty_frac] = -1
    return s, ids


def _exclude_for(ids, g, how):
    G, nq, k = ids.shape
    ex = torch.full((nq,), -1, dtype=torch.int64)
    for q in range(nq):
        valid = ids[:, q][ids[:, q] >= 0]
        if how == "present" and len(valid):
            ex[q] = valid[torch.randint(0, len(valid), (1,), generator=g)]
        elif how == "absent":
            ex[q] = 5  # never an id of these lists
    return ex


@pytest.mark.parametrize("G,k", [(1, 1), (1, 1001), (2, 33), (2, 1001), (4, 32), (4, 4096), (17, 1025), (17, 2),
                                 (1025, 10), (1025, 33)])
@pytest.mark.parametrize("exclude", [None, "present", "absent", "minus_one"])
def test_topk_merge_bit_exact(G, k, exclude):
    """sgpt_topk_merge (generic kernel): G = 1025 > kMaxFlatLists takes the per-list loop of for_each_elem and the
    uncached path.  Equal scores across lists, ids beyond 2^31, -0.0 and +0.0 in the same lists, exclude_ids present in a
    list / absent / -1 / NULL."""
    L, lib = _lib()
    g = torch.Generator().manual_seed(G * 7919 + k)
    nq = 3 if G * k < 20000 else 2
    s, ids = _merge_lists(G, nq, k, g)
    ex = None if exclude is None else _exclude_for(ids, g, exclude)
    want_s, want_i = topk_reference(s.permute(1, 0, 2).reshape(nq, G * k), ids.permute(1, 0, 2).reshape(nq, G * k), k, ex)
    sd, idd = s.cuda(), ids.cuda()
    exd = None if ex is None else ex.cuda()

    def run(os_, oi):
        L.check(lib.sgpt_topk_merge(sd.data_ptr(), idd.data_ptr(), G, nq, k, os_.data_ptr(), oi.data_ptr(), L.ptr(exd),
                                    None, L.current_stream()), "sgpt_topk_merge")

    _check(f"sgpt_topk_merge G={G} k={k} exclude={exclude}", run, nq, want_s, want_i)


# ---------------------------------------------------------------------------------------------------------------------
# sgpt_topk_merge_packed: sorted packed lists
def pack(scores, ids):
    """(fp32 scores, int ids) -> packed int64 entries: low 32 bits the score's bits, high 32 bits the int32 id."""
    bits = scores.float().contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return (ids.to(torch.int64) << 32) | bits


def _sorted_packed_lists(G, nq, k, g, max_id=(1 << 31) - 2):
    """Sorted lists (score descending, id ascending, empty tail) with ids unique across the lists of a query; empty tails of
    different lengths, one query with every list empty."""
    s_all = torch.full((G, nq, k), float("-inf"))
    i_all = torch.full((G, nq, k), -1, dtype=torch.int64)
    for q in range(nq):
        if q == nq - 1 and nq > 2:
            continue  # all lists of this query empty
        pool = torch.randperm(min(max_id + 1, G * k * 8), generator=g)[:G * k]
        pool = max_id - pool  # ids up to 2^31 - 2
        for h in range(G):
            m = int(torch.randint(0, k + 1, (1,), generator=g)) if h % 2 else k - h
            m = max(0, m)
            sc = torch.randint(0, 6, (m,), generator=g).float() - 2.0
            idv = pool[h * k:h * k + m]
            order = np.lexsort((idv.numpy(), -sc.numpy()))
            s_all[h, q, :m], i_all[h, q, :m] = sc[order], idv[order]
    return s_all, i_all


@pytest.mark.parametrize("G,k", [(1, 1), (1, 100), (2, 1), (2, 1001), (3, 33), (3, 1025), (3, 4096), (4, 1001),
                                 (9, 128)])
def test_topk_merge_packed_both_kernels_bit_exact(G, k):
    """sgpt_topk_merge_packed: G = 1..3 lists that fit 200 KiB of shared memory go to the rank-merge kernel
    (merge_sorted_kernel), more lists to the generic selection kernel.  The same data is run both ways, by appending
    all-empty lists up to at least 4, and both must equal the reference.  The excluded id sits at position 0 of a list, in
    its middle, at its last entry (typically ranked at or beyond k in the merge), is absent, or -1."""
    L, lib = _lib()
    g = torch.Generator().manual_seed(31 * G + k)
    nq = 7
    s, ids = _sorted_packed_lists(G, nq, k, g)
    ex = torch.full((nq,), -1, dtype=torch.int64)
    for q in range(nq):
        row = ids[q % G, q]
        m = int((row >= 0).sum())
        if m:
            ex[q] = row[[0, m // 2, m - 1, 0, 0, 0, 0][q]] if q < 3 else (-1 if q == 3 else (1 << 31) - 1)
    packed = pack(s, ids)
    flat = lambda t: t.permute(1, 0, 2).reshape(nq, -1)  # noqa: E731
    results = []
    for exclude in (None, ex):
        want_s, want_i = topk_reference(flat(s), flat(ids), k, exclude)
        exd = None if exclude is None else exclude.cuda()
        for G2 in sorted({G, max(G + 1, 4)}):
            pk = torch.cat([packed, pack(torch.full((G2 - G, nq, k), float("-inf")),
                                         torch.full((G2 - G, nq, k), -1, dtype=torch.int64))]).cuda()

            def run(os_, oi):
                L.check(lib.sgpt_topk_merge_packed(pk.data_ptr(), G2, nq, k, os_.data_ptr(), oi.data_ptr(), L.ptr(exd),
                                                   L.current_stream()), "sgpt_topk_merge_packed")

            kernel = "rank-merge" if G2 <= 3 and G2 * k * 8 <= 200 * 1024 else "generic"
            _check(f"sgpt_topk_merge_packed G={G2} ({kernel}) k={k} exclude={exclude is not None}", run, nq, want_s, want_i)
            results.append(kernel)
    assert "generic" in results
