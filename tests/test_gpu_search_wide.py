"""Every corpus search bit for bit at real embedding widths: many k-blocks, a ragged last k-block, bf16 and int8.

The D = 64 suites run exactly one k-block per tile (one partial one for int8).  Here the widths are those where the
similarity GEMM (csrc/gemm.cuh gemm_bf16_tn_kernel) goes wrong: a single partial k-block (bf16 D = 8 .. 56, int8 D = 16),
a ragged last k-block after many full ones (bf16 D % 64 != 0, int8 D % 128 != 0), the ring wrapping inside one tile
(D = 320 at BN = 128), and the widths the served models produce (768 .. 4096: 12 to 64 k-blocks per tile), on every
search entry point and on the BN = 256 instantiations (filter, sample maxima, IVF rows) as well as the BN = 128 scores.

Exact data at any D: bf16 entries are small integers (|x| <= 2), so at D = 4096 every partial sum stays below 2^24 and
the fp32 accumulation is exact in any order; scales are powers of two.  One int8 corpus takes the full range (-128
included) at D >= 2048, where the dot products exceed 2^24: its reference is the exact integer dot rounded once to fp32,
then multiplied by the scales in the documented order, the kernel's cvt.rn.f32.s32 rounding included.  References are
fp64 matmuls on the device (exact for these integers: torch only checks) and the exact top-k of tests/helpers.py
topk_reference (score descending, ties by ascending id).  Every case also checks that a second launch returns the same
bits.  sgpt_row_inv_norms and one continuous search per dtype are held to error bounds of the kernels' fp32 order."""
import math

import pytest
import torch

from tests.helpers import tensor_core_sum_bound, topk_reference
from tests.test_gpu_ivf import SIZES, _data as _ivf_data, _ivf, _probes
from tests.test_gpu_ivf import _reference as _ivf_reference
from tests.test_gpu_ivf_masked import _ivf_masked, _words
from tests.test_gpu_ivf_range import _check as _ivf_range_check
from tests.test_gpu_ivf_range import _ivf_range, _present_threshold
from tests.test_gpu_ivf_range import _reference as _ivf_range_reference
from tests.test_gpu_ivf_range import _scores as _ivf_scores
from tests.test_gpu_mining import big_n, check_range, device_range, reference_range
from tests.test_gpu_search_exact import _equal, _plan, _search, corpus, two_pass_n
from tests.test_gpu_search_int8 import _bits_equal, _range_i8, _scores_i8, _search_i8
from tests.test_gpu_search_masked import _pack, make_allow
from tests.test_gpu_search_masked import _range as _range_masked
from tests.test_gpu_search_masked import _search as _search_masked

pytestmark = pytest.mark.gpu

BF16_WIDTHS = [8, 56, 128, 200, 320, 768, 776, 2048, 4096]
I8_WIDTHS = [16, 144, 784, 4096, 4112]
# per family: one single partial k-block, one ragged multi-k-block width, and the served widths
SEARCH_WIDTHS = [("bf16", 56), ("bf16", 776), ("bf16", 4096), ("int8", 16), ("int8", 784), ("int8", 4112)]
IVF_WIDTHS = [("bf16", 56), ("bf16", 776), ("bf16", 4096), ("int8", 16), ("int8", 784), ("int8", 4096)]
PLAN_N = {"dense": 20000, "dense-uncached": 60000, "two-pass": None}
U = 2.0 ** -24  # fp32 unit roundoff (round to nearest)


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _n(plan):
    return PLAN_N[plan] or two_pass_n(77)


def _ints(shape, lo, hi, g, dtype):
    """Uniform integers in [lo, hi] drawn on the device, as `dtype` ("bf16" or "int8")."""
    x = torch.randint(lo, hi + 1, shape, generator=g, device="cuda", dtype=torch.int16)
    return x.to(torch.int8 if dtype == "int8" else torch.bfloat16)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _pow2(m, g, lo=-1, hi=2):
    return 2.0 ** torch.randint(lo, hi + 1, (m,), generator=g, device="cuda").float()


def _dot64(Q, C, q_scale=None, c_scale=None):
    """fp64 scores on the device (exact for the integer operands here), NaN -> -1 as the kernels (XS:99)."""
    sc = Q.double() @ C.double().T
    if q_scale is not None:
        sc = sc * q_scale.double()[:, None]
    if c_scale is not None:
        sc = sc * c_scale.double()[None, :]
    return torch.nan_to_num(sc, nan=-1.0, posinf=math.inf, neginf=-math.inf)


def _topk64(sc, k, id_base=0, allow=None):
    """topk_reference for ids id_base + column on the device: a stable descending sort keeps tied columns, and so tied
    ids, in ascending order.  allow: bool [n] or [nq, n] (None: all); the tail is (-inf, -1)."""
    nq, n = sc.shape
    key = sc + 0.0  # -0.0 -> +0.0: equal scores must be equal keys
    ids = (torch.arange(n, device=sc.device) + id_base).expand(nq, n)
    if allow is not None:
        a = allow.to(sc.device).expand(nq, n)
        key = torch.where(a, key, torch.full_like(key, -math.inf))
        ids = torch.where(a, ids, torch.full_like(ids, -1))
    if n < k:
        key = torch.cat([key, torch.full((nq, k - n), -math.inf, dtype=key.dtype, device=key.device)], 1)
        ids = torch.cat([ids, torch.full((nq, k - n), -1, dtype=ids.dtype, device=ids.device)], 1)
    s, order = torch.sort(key, dim=1, descending=True, stable=True)
    s, i = s[:, :k], ids.gather(1, order[:, :k])
    s = torch.where(i < 0, torch.full_like(s, -math.inf), s)
    return s.cpu(), i.cpu()


def test_device_topk_reference_equals_helpers():
    """The device top-k reference is tests/helpers.py topk_reference, ties, -0.0, masks and short rows included."""
    g = torch.Generator().manual_seed(0)
    sc = torch.randint(-3, 4, (37, 700), generator=g).double()
    sc[:, ::5] = -0.0
    allow = torch.rand(37, 700, generator=g) < 0.3
    allow[3] = False
    for a, k in ((None, 50), (allow, 300), (allow[0], 1001)):
        ids = (torch.arange(700) + 11).expand(37, 700)
        if a is not None:
            ids = torch.where(a.expand(37, 700), ids, torch.full_like(ids, -1))
        want = topk_reference(sc, ids, k)
        got = _topk64(sc.cuda(), k, 11, None if a is None else a.cuda())
        assert torch.equal(got[1], want[1]) and torch.equal(got[0], want[0]), k


# ---- sgpt_row_inv_norms ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [8, 64, 776, 4096])
def test_row_inv_norms_fp64_bound(D):
    """1 / max(||x||, 1e-12) against fp64.  The kernel squares bf16 values exactly in fp32, adds each 8-element chunk in a
    tree (3 roundings), each lane's chunks in a chain (ceil(D / 256) roundings), the 32 lanes in a tree (5), then takes
    IEEE sqrt and divide: with m = 8 + ceil(D / 256) roundings of a sum of non-negative terms the relative error is at
    most m u / 2 + 2 u (+ O(u^2)).  A zero row is exactly 1.0f / 1e-12f, and so is a row holding a NaN (fmaxf returns the
    non-NaN operand; the row's scores are NaN regardless and map to -1).  n % 8 != 0: the last CTA is partial."""
    L, lib = _lib()
    n = 1003
    g = torch.Generator().manual_seed(D)
    x = torch.randn(n, D, generator=g) * 2.0 ** torch.randint(-20, 21, (n, 1), generator=g).float()
    x[1] = 0.0
    x[2] = 1.0
    x[5, D // 2] = float("nan")
    x[7] = 2.0 ** -40  # squares near 2^-80: normal in fp32
    xb = x.to(torch.bfloat16).cuda()
    out = torch.full((n + 4,), 7.0, dtype=torch.float32, device="cuda")
    L.check(lib.sgpt_row_inv_norms(xb.data_ptr(), out.data_ptr(), n, D, L.current_stream()), "sgpt_row_inv_norms")
    got = out.cpu()
    assert (got[n:] == 7.0).all(), "wrote past n"
    tiny = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(1e-12, dtype=torch.float32)
    assert _bits_equal(got[1:2], tiny.reshape(1)) and _bits_equal(got[5:6], tiny.reshape(1))
    ok = torch.ones(n, dtype=torch.bool)
    ok[[1, 5]] = False
    ref = 1.0 / torch.sqrt((xb.double() ** 2).sum(1)).cpu()
    m = 8 + -(-D // 256)
    rel = (m / 2 + 2) * U * 1.001
    err = (got[:n].double() - ref).abs() / ref
    assert (err[ok] <= rel).all(), f"D={D}: relative error {float(err[ok].max())} > {rel}"
    again = out.clone()
    L.check(lib.sgpt_row_inv_norms(xb.data_ptr(), again.data_ptr(), n, D, L.current_stream()))
    assert _bits_equal(out, again)


# ---- sgpt_scores / sgpt_scores_i8 --------------------------------------------------------------------------------
def _scores_bf16(Q, C, qs, cs):
    L, lib = _lib()
    nq, n, D = Q.shape[0], C.shape[0], Q.shape[1]
    lds = n + 5
    out = torch.full((nq, lds), 7.0, dtype=torch.float32, device="cuda")
    L.check(lib.sgpt_scores(Q.data_ptr(), C.data_ptr(), L.ptr(qs), L.ptr(cs), out.data_ptr(), lds, nq, n, D,
                            L.current_stream()), "sgpt_scores")
    return out.cpu()


@pytest.mark.parametrize("D", BF16_WIDTHS)
def test_scores_bf16_bit_exact(D):
    """nq 1 / 129 / 300, n = 777 (a ragged last tile), power-of-two scales with a NaN query and a NaN document scale
    (-1); the pad columns keep their sentinel bits."""
    g = _gen(D)
    n = 777
    C = _ints((n, D), -2, 2, g, "bf16")
    for nq in (1, 129, 300):
        Q = _ints((nq, D), -2, 2, g, "bf16")
        qs = cs = None
        if nq > 1:
            qs, cs = _pow2(nq, g), _pow2(n, g)
            qs[nq // 2] = float("nan")
            cs[n // 3] = float("nan")
        want = _dot64(Q, C, qs, cs).float().cpu()
        got = _scores_bf16(Q, C, qs, cs)
        what = f"D={D} nq={nq}"
        assert _bits_equal(got[:, :n], want), f"{what}: max diff {float((got[:, :n] - want).abs().max())}"
        assert (got[:, n:] == 7.0).all(), f"{what}: pad columns written"
        assert _bits_equal(got, _scores_bf16(Q, C, qs, cs)), f"{what}: a second launch differs"


@pytest.mark.parametrize("D", I8_WIDTHS)
def test_scores_i8_bit_exact(D):
    """Full int8 range (-128 included).  The first queries repeat the first documents and one query and one document
    are all -128, so at D >= 2048 some dot products exceed 2^24 and their one rounding to fp32 is checked.  Continuous
    scales (dot * q_scale * c_scale in that order), NaN scales -> -1, pad columns kept."""
    g = _gen(D + 1)
    n = 777
    C = _ints((n, D), -128, 127, g, "int8")
    C[9] = -128
    for nq in (1, 129, 300):
        Q = _ints((nq, D), -128, 127, g, "int8")
        Q[:8] = C[:min(nq, 8)]  # sum of squares: about 5461 D
        if nq > 1:
            Q[-1] = -128
        dot64 = Q.double() @ C.double().T  # exact integers
        dot = dot64.float().cpu()  # rounded once
        if D >= 2048 and nq > 1:
            assert (dot64.abs() > 2 ** 24).any() and (dot64.float().double() != dot64).any()
        qs = torch.rand(nq, generator=g, device="cuda") + 0.01
        cs = torch.rand(n, generator=g, device="cuda") + 0.01
        qs[nq // 2] = float("nan")
        cs[n // 3] = float("nan")
        for a, b in ((None, None), (qs, cs)):
            want = dot.clone() if a is None else dot * a.cpu()[:, None] * b.cpu()[None, :]
            want = torch.where(torch.isnan(want), torch.full_like(want, -1.0), want)
            got = _scores_i8(Q, C, a, b)
            what = f"D={D} nq={nq} scales={a is not None}"
            assert _bits_equal(got[:, :n], want), f"{what}: max diff {float((got[:, :n] - want).abs().max())}"
            assert (got[:, n:] == 7.0).all(), f"{what}: pad columns written"
            assert _bits_equal(got, _scores_i8(Q, C, a, b)), f"{what}: a second launch differs"


# ---- sgpt_search / sgpt_search_packed and the _i8 twins, every plan -------------------------------------------------
CASES = {"dense": [(1, 1), (129, 1001), (257, 10)],
         "dense-uncached": [(1, 1001), (129, 1001), (257, 1001)],
         "two-pass": [(1, 1), (129, 1001), (257, 1001)]}


def _run(dtype, Q, C, k, id_base, qs, cs, want, what):
    """The search and its packed twin against `want`; a second launch returns the same bits."""
    fn = _search_i8 if dtype == "int8" else _search
    got = fn(Q, C, k, id_base, qs, cs)
    _equal(what, got, want)
    again = fn(Q, C, k, id_base, qs, cs)
    assert _bits_equal(got[0], again[0]) and torch.equal(got[1], again[1]), f"{what}: a second search differs"
    if id_base + C.shape[0] < 2 ** 31:
        _equal(f"{what} packed", fn(Q, C, k, id_base, qs, cs, packed=True), want)


@pytest.mark.parametrize("dtype,D", SEARCH_WIDTHS)
@pytest.mark.parametrize("plan", ["dense", "dense-uncached", "two-pass"])
def test_search_plans_bit_exact(dtype, D, plan):
    """Tie-heavy integer corpora on each plan; nq = 129 (CTA pairs) and 257 (query blocks), power-of-two scales, and
    the packed output at the largest legal id_base."""
    n = _n(plan)
    g = _gen(D * 10 + len(plan))
    C = _ints((n, D), -2, 2, g, dtype)
    Qall = _ints((257, D), -2, 2, g, dtype)
    cs = _pow2(n, g)
    for j, (nq, k) in enumerate(CASES[plan]):
        assert _plan(nq, n, k) == plan, (nq, n, k)
        Q = Qall[:nq]
        qs = _pow2(nq, g) if j > 0 else None
        c = cs if j > 0 else None
        id_base = 2 ** 31 - 1 - n if nq == 257 else 7 * j
        want = _topk64(_dot64(Q, C, qs, c), k, id_base)
        _run(dtype, Q, C, k, id_base, qs, c, want, f"{dtype} D={D} {plan} nq={nq} k={k}")


@pytest.mark.parametrize("dtype,D,kind", [(dt, D, kind) for dt, D in (("bf16", 200), ("bf16", 776), ("int8", 144),
                                                                      ("int8", 784))
                                          for kind in ("k_sampled", "k_unsampled", "nan_rows", "negative")
                                          if not (dt == "int8" and kind == "nan_rows")])  # int8 rows hold no NaN
def test_two_pass_thresholds_bit_exact(dtype, D, kind):
    """The two-pass plan at its admission edges: k planted documents strictly above all others inside or outside the
    sampled tiles (tau equals the k-th best score), NaN rows at the cut (bf16), all scores negative."""
    n = two_pass_n(77)
    for j, (nq, k) in enumerate([(1, 1), (129, 1001), (257, 1025)]):
        assert _plan(nq, n, k) == "two-pass"
        g = torch.Generator().manual_seed(D + 10 * j)
        Qf, Cf = corpus(kind, nq, n, k, g, D=D)
        Q, C = Qf.cuda(), Cf.cuda()
        want = _topk64(_dot64(Q, C), k, j)
        dt = torch.int8 if dtype == "int8" else torch.bfloat16
        _run(dtype, Q.to(dt), C.to(dt), k, j, None, None, want, f"{dtype} D={D} {kind} nq={nq} k={k}")


# ---- range search -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,D", SEARCH_WIDTHS)
def test_range_search_bit_exact(dtype, D):
    """sgpt_range_search(_i8) over a ragged shard of more than two tiles per SM: the threshold is a score that occurs
    (query 0's 37th best), so documents exactly at it are admitted."""
    nq, n, id_base = 129, big_n(), 5
    g = _gen(D * 7 + 3)
    Q, C = _ints((nq, D), -2, 2, g, dtype), _ints((n, D), -2, 2, g, dtype)
    qs, cs = _pow2(nq, g), _pow2(n, g)
    sc = _dot64(Q, C, qs, cs)
    t = float(torch.sort(sc[0], descending=True).values[36])
    total = int((sc >= t).sum())
    want = reference_range(sc.cpu(), t, total, id_base)
    what = f"{dtype} D={D} t={t}"
    if dtype == "bf16":
        check_range(device_range(Q, C, t, total, id_base, qs, cs), want, what)
        return
    got = _range_i8(Q, C, t, id_base, total, qs, cs)
    assert torch.equal(got[0], want[0]), f"{what}: counts differ"
    assert _bits_equal(got[1][:total], want[1][:total]) and torch.equal(got[2][:total], want[2][:total]), what
    again = _range_i8(Q, C, t, id_base, total, qs, cs)
    assert torch.equal(again[0], got[0]) and _bits_equal(again[1], got[1]) and torch.equal(again[2], got[2]), \
        f"{what}: a second launch differs"


# ---- masked search and masked range search ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype,D", SEARCH_WIDTHS)
@pytest.mark.parametrize("plan", ["dense", "two-pass"])
def test_masked_search_and_range_bit_exact(dtype, D, plan):
    """sgpt_search_masked (and its packed twin) and sgpt_range_search_masked with one shared bitmap (nq = 257) and one
    bitmap per query (nq = 129)."""
    n = _n(plan)
    g = torch.Generator().manual_seed(D + len(plan))
    gd = _gen(D + len(plan))
    C = _ints((n, D), -2, 2, gd, dtype)
    for nq, kind in ((257, "p50"), (129, "per_query")):
        k = 1001
        assert _plan(nq, n, k) == plan
        Q = _ints((nq, D), -2, 2, gd, dtype)
        allow = make_allow(kind, nq, n, k, g)
        words = _pack(allow)
        pitch = words.shape[1] if allow.dim() == 2 else 0
        sc = _dot64(Q, C)
        allow_d = allow.cuda()
        what = f"{dtype} D={D} {plan} nq={nq} {kind}"
        want = _topk64(sc, k, 3, allow_d)
        got = _search_masked(Q, C, k, dtype, words, pitch, id_base=3)
        _equal(what, got, want)
        again = _search_masked(Q, C, k, dtype, words, pitch, id_base=3)
        assert _bits_equal(got[0], again[0]) and torch.equal(got[1], again[1]), f"{what}: a second search differs"
        _equal(f"{what} packed", _search_masked(Q, C, k, dtype, words, pitch, id_base=3, packed=True), want)
        # range: the threshold is query 0's 37th best allowed score
        masked = torch.where(allow_d.expand_as(sc), sc, torch.full_like(sc, -math.inf))
        t = float(torch.sort(masked[0], descending=True).values[36])
        total = int((masked >= t).sum())
        counts, s, i = reference_range(masked.cpu(), t, total, 3)
        got = _range_masked(Q, C, t, words, pitch, total, dtype, id_base=3)
        assert torch.equal(got[0], counts), f"{what} range: counts differ"
        assert _bits_equal(got[1][:total], s[:total]) and torch.equal(got[2][:total], i[:total]), f"{what} range"


# ---- IVF: search, masked search, range search ------------------------------------------------------------------
def _ivf_operands(dtype, D, nq, seed, nan_rows=False):
    """The hand-made list layout of tests/test_gpu_ivf.py SIZES (empty lists, 256 and 257 rows, one list over many
    tiles) at width D, with power-of-two scales; nan_rows: NaN rows (bf16) or NaN document scales (int8)."""
    g = torch.Generator().manual_seed(seed)
    Q, C, offsets, ids = _ivf_data(nq, g, D=D)
    n = C.shape[0]
    qs, cs = 2.0 ** _ivf_ints((nq,), -2, 2, g), 2.0 ** _ivf_ints((n,), -3, 1, g)
    if nan_rows:
        if dtype == "bf16":
            C[::97] = float("nan")
        else:
            cs[::97] = float("nan")
    return g, Q, C, qs, cs, offsets, ids


def _ivf_ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g).float()


@pytest.mark.parametrize("dtype,D", IVF_WIDTHS)
def test_ivf_search_bit_exact(dtype, D):
    """nq = 300 probing every list (two 256-query blocks), and nq = 129 with skipped probes, NaN rows and scales; the
    gathered query rows are D * 2 (bf16) or D (int8) bytes long."""
    nl = len(SIZES)
    for nq, nprobe, skipped, k in ((300, nl, False, 1001), (129, 4, True, 10), (129, nl, True, 1)):
        g, Q, C, qs, cs, offsets, ids = _ivf_operands(dtype, D, nq, D + nq + k, nan_rows=skipped)
        probes = _probes(nq, nl, nprobe, g, skipped=skipped)
        if not skipped:
            qs = cs = None
        want = _ivf_reference(Q, C, qs, cs, offsets, ids, probes, k)
        what = f"{dtype} D={D} nq={nq} nprobe={nprobe} k={k}"
        got = _ivf(dtype, Q, C, qs, cs, offsets, ids, probes, k)
        _equal(what, got, want)
        again = _ivf(dtype, Q, C, qs, cs, offsets, ids, probes, k)
        assert _bits_equal(got[0], again[0]) and torch.equal(got[1], again[1]), f"{what}: a second launch differs"


@pytest.mark.parametrize("dtype,D", IVF_WIDTHS)
def test_ivf_masked_bit_exact(dtype, D):
    """sgpt_ivf_search_masked with one shared bitmap and one bitmap per query (pitch ceil(n/32) + 3), nq = 300."""
    nl = len(SIZES)
    for nq, per_query in ((300, True), (129, False)):
        g, Q, C, qs, cs, offsets, ids = _ivf_operands(dtype, D, nq, D + 2 * nq)
        n = C.shape[0]
        probes = _probes(nq, nl, nl, g)
        allowed = torch.rand((nq, n) if per_query else (n,), generator=g) < 0.4
        mask, pitch = _words(allowed, 3, g)
        k = 1001
        want = _ivf_reference(Q, C, None, None, offsets, ids, probes, k, deleted=~allowed)
        what = f"{dtype} D={D} nq={nq} per_query={per_query}"
        got = _ivf_masked(dtype, Q, C, offsets, ids, probes, k, mask, pitch)
        _equal(what, got, want)
        again = _ivf_masked(dtype, Q, C, offsets, ids, probes, k, mask, pitch)
        assert _bits_equal(got[0], again[0]) and torch.equal(got[1], again[1]), f"{what}: a second launch differs"


@pytest.mark.parametrize("dtype,D", IVF_WIDTHS)
def test_ivf_range_bit_exact(dtype, D):
    """sgpt_ivf_range_search at a threshold that occurs (documents at it are admitted), nq = 300 over every list with
    skipped probes, scales and NaN rows (the wrapper checks a second launch)."""
    nl = len(SIZES)
    nq = 300
    g, Q, C, qs, cs, offsets, ids = _ivf_operands(dtype, D, nq, D + 5, nan_rows=True)
    probes = _probes(nq, nl, nl, g)
    sc = _ivf_scores(Q, C, qs, cs)
    t = _present_threshold(sc, offsets, probes)
    total = int(_ivf_range_reference(sc, offsets, ids, probes, t, 0)[0].sum())
    got = _ivf_range(dtype, Q, C, qs, cs, offsets, ids, probes, t, total)
    _ivf_range_check(got, _ivf_range_reference(sc, offsets, ids, probes, t, total), f"{dtype} D={D} t={t}")


# ---- continuous data through CorpusShard.search ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "int8"])
def test_shard_search_continuous_within_fp32_bound(dtype):
    """cos_sim at D = 4096 on Gaussian data.  Reference: the fp64 score of the stored rows with the stored fp32 scales.
    bf16: the device score is fl(fl(dot) * q_scale * c_scale) with dot summed on the tensor cores, so it lies within
    tensor_core_sum_bound(sum |q c|, D) * q_scale * c_scale + 3 u |score| of the reference.  int8: the integer dot is
    exact and rounded once, then scaled twice: within 3 u |score|.  Every returned score lies within its bound, and no
    unreturned document's reference exceeds the k-th returned score by more than its own bound."""
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import quantize_rows_i8, row_inv_norms, to_bf16_rows

    D, n, nq, k = 4096, 30000, 64, 100
    g = _gen(41)
    q = torch.randn(nq, D, generator=g, device="cuda")
    c = torch.randn(n, D, generator=g, device="cuda")
    c[::50] = q[torch.arange(0, n, 50, device="cuda") // 50 % nq] + 0.5 * c[::50]  # near-duplicates at the top
    shard = CorpusShard.from_embeddings(c, dtype=dtype, id_base=9)
    s, i = shard.search(q, k, "cos_sim")
    stored = shard.vectors[:n].double()
    if dtype == "int8":
        q8, _, qcos = quantize_rows_i8(q)
        ref = (q8.double() @ stored.T) * qcos.double()[:, None] * shard.cos_scales[:n].double()[None, :]
        bound = 3 * U * ref.abs() * 1.001
    else:
        qb = to_bf16_rows(q)
        qs, cs = row_inv_norms(qb).double(), shard.inv_norms[:n].double()
        ref = (qb.double() @ stored.T) * qs[:, None] * cs[None, :]
        abs_sum = qb.double().abs() @ stored.abs().T
        bound = (tensor_core_sum_bound(abs_sum, D) + D * 2.0 ** -52 * abs_sum) * qs[:, None] * cs[None, :] \
            + 3 * U * ref.abs() * 1.001
    assert (i >= 9).all() and (i < 9 + n).all()
    assert all(len(set(r)) == k for r in i.tolist()), "an id returned twice"
    cols = i - 9
    r, b = ref.gather(1, cols), bound.gather(1, cols)
    err = (s.double() - r).abs()
    assert (err <= b).all(), f"{dtype}: returned score off by {float(err.max())}, bound {float(b[err > b].min())}"
    out = torch.ones_like(ref, dtype=torch.bool)
    out.scatter_(1, cols, False)
    kth = s[:, -1].double()[:, None]
    beat = out & (ref > kth + bound)
    assert not beat.any(), f"{dtype}: {int(beat.sum())} unreturned documents beat the k-th score beyond the bound"
