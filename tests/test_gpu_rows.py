"""The encoder's row kernels through the C ABI, each against a plain fp64 (or exact) restatement of its contract in
include/sgpt_b200.h, evaluated on exactly the values the kernel reads: the token(+position) embedding gather, LayerNorm
on every width dispatch path (the 16-byte bf16 kernels, the `layernorm_kernel` instances for d % 8 == 4 and d > 8192,
and the gathered LayerNorm of the LM head), the log-prob rows and segment sums of the cross-encoder, the fp32 <-> bf16
conversions and the stand-alone L2 normalisation.  Where the kernel's arithmetic is exact the comparison is bit for bit;
elsewhere the tolerance is an error bound of the kernel's fp32 arithmetic, per element."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # unit roundoff of fp32
FLT_MAX = float(np.finfo(np.float32).max)
BF16 = torch.bfloat16


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def ulp_bf16(v):
    """Spacing of the bf16 numbers at |v| (fp64 tensor): 2^(e-7) for 2^e <= |v| < 2^(e+1), 2^-133 below 2^-126."""
    _, e = torch.frexp(v.abs())  # v = m 2^e, 0.5 <= m < 1
    return torch.where(v == 0, torch.full_like(v, 2.0 ** -133),
                       torch.ldexp(torch.ones_like(v), (e - 8).clamp(min=-133)))


def bits16(t):
    return t.contiguous().view(torch.int16)


# --------------------------------------------------------------------------------------------------------------------
# F1: embedding gather
# --------------------------------------------------------------------------------------------------------------------
# T * d/8 above the grid cap of the grid-stride loop (132 SMs x 16 CTAs x 256 threads = 540672 vectors) for d = 8 and
# d = 4104; a small row count besides
@pytest.mark.parametrize("T,d", [(600_000, 8), (1100, 4104), (37, 64)])
@pytest.mark.parametrize("with_wpe", [True, False])
def test_embed_tokens_bit_exact(T, d, with_wpe):
    L, lib = _lib()
    vocab, max_pos = 1000, 300
    g = torch.Generator(device="cuda").manual_seed(T + d)
    wte = (torch.randn(vocab, d, generator=g, device="cuda") * 0.5).to(BF16)
    wpe = (torch.randn(max_pos, d, generator=g, device="cuda") * 0.3).to(BF16)  # same scale: the adds round
    ids = torch.randint(0, vocab, (T,), generator=g, device="cuda", dtype=torch.int32)
    pos = torch.randint(0, max_pos, (T,), generator=g, device="cuda", dtype=torch.int32)
    ids[0], ids[-1], pos[0], pos[-1] = 0, vocab - 1, max_pos - 1, 0
    out = torch.full((T + 1, d), 7.0, dtype=BF16, device="cuda")
    L.check(lib.sgpt_embed_tokens(ids.data_ptr(), pos.data_ptr() if with_wpe else None, wte.data_ptr(),
                                  wpe.data_ptr() if with_wpe else None, out.data_ptr(), T, d, vocab, max_pos,
                                  L.current_stream()), "sgpt_embed_tokens")
    want = wte[ids.long()].float()
    if with_wpe:
        want = want + wpe[pos.long()].float()  # fp32 add, then one round-to-nearest-even to bf16
    assert torch.equal(bits16(out[:T]), bits16(want.to(BF16)))
    assert bool((out[T] == 7.0).all())  # nothing written past the last row


def test_embed_tokens_empty_clamped_and_rejected():
    L, lib = _lib()
    vocab, max_pos, d = 50, 20, 16
    g = torch.Generator(device="cuda").manual_seed(5)
    wte = torch.randn(vocab, d, generator=g, device="cuda").to(BF16)
    wpe = torch.randn(max_pos, d, generator=g, device="cuda").to(BF16)
    out = torch.full((4, d), 7.0, dtype=BF16, device="cuda")
    dummy = torch.zeros(1, dtype=torch.int32, device="cuda")
    L.check(lib.sgpt_embed_tokens(dummy.data_ptr(), dummy.data_ptr(), wte.data_ptr(), wpe.data_ptr(), out.data_ptr(),
                                  0, d, vocab, max_pos, L.current_stream()))
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())  # T = 0 writes nothing
    # out-of-range ids and positions are clamped to the table, never read out of bounds
    ids = torch.tensor([-5, vocab, vocab + 100, -2 ** 31], dtype=torch.int32, device="cuda")
    pos = torch.tensor([max_pos, -1, 2 ** 31 - 1, 3], dtype=torch.int32, device="cuda")
    L.check(lib.sgpt_embed_tokens(ids.data_ptr(), pos.data_ptr(), wte.data_ptr(), wpe.data_ptr(), out.data_ptr(), 4,
                                  d, vocab, max_pos, L.current_stream()))
    ci = ids.long().clamp(0, vocab - 1)
    cp = pos.long().clamp(0, max_pos - 1)
    assert torch.equal(bits16(out), bits16((wte[ci].float() + wpe[cp].float()).to(BF16)))
    assert lib.sgpt_embed_tokens(ids.data_ptr(), None, wte.data_ptr(), wpe.data_ptr(), out.data_ptr(), 4, d, vocab,
                                 max_pos, L.current_stream()) == 1  # wpe without pos
    assert lib.sgpt_embed_tokens(ids.data_ptr(), None, wte.data_ptr(), None, out.data_ptr(), 4, 12, vocab, max_pos,
                                 L.current_stream()) == 1  # d % 8 != 0


# --------------------------------------------------------------------------------------------------------------------
# F2/F7: LayerNorm
# --------------------------------------------------------------------------------------------------------------------
CONSTANTS = (300.0, -3.140625, 0.0, 0.00146484375, 20000.0, -7.5, 96.5, 1.75)  # none a power of two


def ln_rows(T, d, seed):
    """bf16 rows: random (with an outlier feature); every 4th row a large common offset with a small spread
    (512 + noise); rows 2, 6, 10, ... constant (variance 0).  A one-pass E[x^2] - E[x]^2 variance breaks on the last two
    kinds, and a LayerNorm without eps divides by zero on the constant rows."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, d, generator=g) * 2.5 + 0.4
    x[:, min(3, d - 1)] += 30.0
    x[1::4] = 512.0 + 8.0 * torch.randn(x[1::4].shape, generator=g)
    const_rows = list(range(2, T, 4))[:len(CONSTANTS)]
    for r, c in zip(const_rows, CONSTANTS):
        x[r] = c
    return x.to(BF16), const_rows


def ln_reference(xb, gamma, beta, eps):
    """fp64 LayerNorm of the widened bf16 rows, and the per-element bound: one bf16 rounding of the fp32 result
    (ulp_bf16 of the exact value, twice the rounding error) plus the fp32 error of the statistics: 2^-20 relative on the
    normalised value and beta, and a mean off by 2^-20 of the row's mean magnitude, amplified by rstd."""
    x = xb.double()
    mu = x.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mu) ** 2).mean(1, keepdim=True) + eps)
    xh = (x - mu) * rstd
    g, b = gamma.double(), beta.double()
    want = xh * g + b
    tol = ulp_bf16(want) + 2.0 ** -20 * ((xh * g).abs() + b.abs() + g.abs() * rstd * x.abs().mean(1, keepdim=True))
    return want, tol


def ln_params(d, seed):
    g = torch.Generator().manual_seed(seed)
    return 1.0 + 0.3 * torch.randn(d, generator=g), 0.05 * torch.randn(d, generator=g)


def check_ln(got, xb, gamma, beta, eps, const_rows, d):
    want, tol = ln_reference(xb, gamma, beta, eps)
    got = got.double()
    err = (got - want).abs()
    bad = ~(err <= tol)
    assert not bool(bad.any()), (f"{int(bad.sum())} elements out of bound, first at "
                                 f"{[int(i) for i in bad.nonzero()[0]]}: got {got[bad][0].item()} want {want[bad][0].item()}")
    if d & (d - 1) == 0:  # 1/d is exact: the mean of a constant row is exact, so the row is exactly bf16(beta)
        for r in const_rows:
            assert torch.equal(bits16(got[r].to(BF16)), bits16(beta.to(BF16))), r


# d % 8 == 4 (layernorm_kernel <32,8>, <128,8>, <256,16>), d > 8192 (<128,8> is never reached there: <256,16>), and the
# 16-byte bf16 kernels (64, 768, 1024, 4096, 5120, 8192) held to the same bound
@pytest.mark.parametrize("d", [4, 20, 772, 1028, 4100, 8200, 16384, 64, 768, 1024, 4096, 5120, 8192])
@pytest.mark.parametrize("in_place", [False, True])
def test_layernorm_fp64_bound(d, in_place):
    L, lib = _lib()
    T = 37 if d > 4096 else 301
    xb, const_rows = ln_rows(T, d, seed=d)
    gamma, beta = ln_params(d, seed=d + 1)
    eps = 1e-5
    xd = xb.cuda()
    yd = xd if in_place else torch.full((T + 1, d), 7.0, dtype=BF16, device="cuda")
    gd, bd = gamma.cuda(), beta.cuda()
    L.check(lib.sgpt_layernorm(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), yd.data_ptr(), T, d, eps,
                               L.current_stream()), "sgpt_layernorm")
    check_ln(yd[:T].cpu(), xb, gamma, beta, eps, const_rows, d)
    if not in_place:
        assert bool((yd[T] == 7.0).all())  # nothing written past the last row


def test_layernorm_rejects_widths():
    L, lib = _lib()
    x = torch.zeros(2, 16388, dtype=BF16, device="cuda")
    p = torch.ones(16388, device="cuda")
    assert lib.sgpt_layernorm(x.data_ptr(), p.data_ptr(), p.data_ptr(), x.data_ptr(), 2, 16388, 1e-5,
                              L.current_stream()) == 3  # SGPT_ERR_UNSUPPORTED: no row kernel holds 16388 elements
    assert lib.sgpt_layernorm(x.data_ptr(), p.data_ptr(), p.data_ptr(), x.data_ptr(), 2, 6, 1e-5,
                              L.current_stream()) == 1  # d % 4 != 0
    assert lib.sgpt_layernorm_gather(x.data_ptr(), None, p.data_ptr(), p.data_ptr(), x.data_ptr(), 2, 16, 1e-5,
                                     L.current_stream()) == 1  # no row indices


# widths on each side of the SGPT_ROW_DISPATCH boundaries (d4 = 256 / 257, 1024 / 1025) and the extremes; M below and
# above T, with repeated, unordered row indices
@pytest.mark.parametrize("d", [4, 1024, 1028, 4096, 4100, 16384])
@pytest.mark.parametrize("M", [37, 517])
def test_layernorm_gather_fp64_bound(d, M):
    L, lib = _lib()
    T = 300 if d <= 4100 else 40
    xb, const_rows = ln_rows(T, d, seed=3 * d + M)
    gamma, beta = ln_params(d, seed=d + 7)
    g = torch.Generator().manual_seed(M)
    rows = torch.randint(0, T, (M,), generator=g, dtype=torch.int32)
    rows[:4] = torch.tensor([T - 1, 0, T - 1, const_rows[0]], dtype=torch.int32)
    eps = 1e-5
    xd, rd = xb.cuda(), rows.cuda()
    yd = torch.full((M + 1, d), 7.0, dtype=BF16, device="cuda")
    gd, bd = gamma.cuda(), beta.cuda()
    L.check(lib.sgpt_layernorm_gather(xd.data_ptr(), rd.data_ptr(), gd.data_ptr(), bd.data_ptr(), yd.data_ptr(), M, d,
                                      eps, L.current_stream()), "sgpt_layernorm_gather")
    sel = xb[rows.long()]
    check_ln(yd[:M].cpu(), sel, gamma, beta, eps, [3], d)
    assert bool((yd[M] == 7.0).all())  # the row after M stays unwritten
    assert torch.equal(xd.cpu(), xb)  # the input is only read


# --------------------------------------------------------------------------------------------------------------------
# Log-prob rows of the cross-encoder
# --------------------------------------------------------------------------------------------------------------------
def _logprob_rows(M, V, lds, seed):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(M, lds, generator=g) * 4
    logits[:, V:] = float("nan")  # padding columns: never read
    logits[0, :V] = 3.0                      # all equal: greedy 0, logprob -log(V)
    logits[1, :V] = -FLT_MAX                 # all -FLT_MAX: greedy 0
    logits[2, :V] = float("-inf")            # all -inf: greedy 0, logprob NaN (as torch.log_softmax)
    logits[3, V - 1] = logits[3, :V].max() + 1  # maximum in the last valid column
    if V > 3:
        logits[4, 1] = logits[4, 3] = logits[4, :V].max() + 2  # tie: the lowest index wins
        logits[5, 0] = float("nan")          # NaN is never the greedy token
        logits[5, 2] = logits[5, 1:V].max() + 1
    logits[6, :V] = float("nan")             # nothing but NaN: greedy 0
    tgt = torch.randint(0, V, (M,), generator=g, dtype=torch.int32)
    return logits, tgt


@pytest.mark.parametrize("V", [1, 255, 256, 257, 50257])
def test_token_logprobs_fp64(V):
    L, lib = _lib()
    M = 20
    lds = V + 5
    logits, tgt = _logprob_rows(M, V, lds, seed=V)
    bias = torch.randn(V, generator=torch.Generator().manual_seed(V + 1))
    for b, with_greedy in ((None, True), (bias, True), (bias, False)):
        ld, td = logits.cuda(), tgt.cuda()
        bd = None if b is None else b.cuda()
        lp = torch.full((M,), 7.0, device="cuda")
        gr = torch.full((M,), -7, dtype=torch.int32, device="cuda")
        L.check(lib.sgpt_token_logprobs(ld.data_ptr(), lds, M, V, L.ptr(bd), td.data_ptr(), lp.data_ptr(),
                                        gr.data_ptr() if with_greedy else None, L.current_stream()),
                "sgpt_token_logprobs")
        z32 = logits[:, :V] + (0.0 if b is None else b)  # the fp32 sum the kernel forms
        z = z32.double()
        want = torch.log_softmax(z, -1).gather(1, tgt.long()[:, None])[:, 0]
        got = lp.cpu().double()
        # kernel: (z_t - mx) - logf(sum_v expf(z_v - mx)); each expf within 2 ulps, the positive terms summed in
        # ceil(V / 256) + 13 adds per row, one rounding each for the subtractions and logf
        z_nonan = torch.where(torch.isnan(z), float("-inf"), z)
        mx = z_nonan.max(1).values
        zt = z.gather(1, tgt.long()[:, None])[:, 0]
        logt = torch.logsumexp(z, -1) - mx
        tol = U * ((zt - mx).abs() + want.abs()) + 2 * U * logt.abs() + ((V + 255) // 256 + 20) * 2 * U
        nan_want = torch.isnan(want)
        assert torch.equal(torch.isnan(got), nan_want), (V, b is None)
        assert bool(((got - want).abs() <= tol)[~nan_want].all()), (V, float((got - want).abs()[~nan_want].max()))
        if with_greedy:
            greedy_want = z_nonan.argmax(-1)  # lowest index of the largest non-NaN value; 0 for the all-NaN row
            assert torch.equal(gr.cpu().long(), greedy_want), (V, gr.cpu().tolist()[:8], greedy_want.tolist()[:8])
        else:
            assert bool((gr == -7).all())
        assert torch.equal(ld.cpu().view(torch.int32), logits.view(torch.int32))  # only read


def test_segment_sum_sequential_fp32_bits():
    L, lib = _lib()
    rs = np.random.RandomState(4)
    R = 300
    lens = rs.randint(0, 60, R)
    lens[::7] = 0  # empty segments
    lens[5] = lens[200] = 100_000
    off = np.zeros(R + 1, dtype=np.int32)
    np.cumsum(lens, out=off[1:])
    x = (rs.randn(int(off[-1])) * 3).astype(np.float32)
    want = np.zeros(R, dtype=np.float32)
    for r in range(R):
        if lens[r]:
            want[r] = np.cumsum(x[off[r]:off[r + 1]], dtype=np.float32)[-1]  # sequential fp32 sum in index order
    xd, od = torch.from_numpy(x).cuda(), torch.from_numpy(off).cuda()
    out = torch.full((R + 1,), 7.0, device="cuda")
    L.check(lib.sgpt_segment_sum(xd.data_ptr(), od.data_ptr(), R, out.data_ptr(), L.current_stream()))
    got = out.cpu().numpy()
    assert np.array_equal(got[:R].view(np.int32), want.view(np.int32))
    assert got[R] == 7.0


# --------------------------------------------------------------------------------------------------------------------
# Conversions and the stand-alone L2 normalisation
# --------------------------------------------------------------------------------------------------------------------
def test_f32_to_bf16_round_to_nearest_even():
    L, lib = _lib()
    rs = np.random.RandomState(6)
    b16 = rs.randint(0, 1 << 16, 200_000).astype(np.uint32)
    special = np.array([0x00000000, 0x80000000, 0x7f800000, 0xff800000,  # +-0, +-inf
                        0x7f7fffff, 0xff7fffff,                         # +-FLT_MAX: above the bf16 range, round to inf
                        0x7f7f7fff, 0x7f7f8000, 0x7f7e8000,             # just below / at the overflow tie, even tie
                        0x00000001, 0x80000001, 0x00008000, 0x00018000, 0x007f8000, 0x007fffff,  # subnormals, ties
                        0x3f808000, 0x3f818000, 0x3f80c000, 0x3f804000], dtype=np.uint32)
    bits = np.concatenate([
        rs.randint(0, 1 << 32, 1 << 20, dtype=np.uint64).astype(np.uint32),  # any pattern
        (b16 << 16) | 0x8000,  # exact ties between two bf16 neighbours, odd and even
        (b16 << 16) | 0x7fff, (b16 << 16) | 0x8001,  # one fp32 ulp either side of a tie
        rs.randint(0, 1 << 23, 4096).astype(np.uint32),  # subnormals
        special])
    bits = np.concatenate([bits, np.zeros((-len(bits)) % 4, dtype=np.uint32)])
    x = torch.from_numpy(bits.view(np.float32).copy())
    y = torch.empty(len(bits), dtype=BF16, device="cuda")
    xd = x.cuda()
    L.check(lib.sgpt_f32_to_bf16(xd.data_ptr(), y.data_ptr(), len(bits), L.current_stream()))
    got = y.cpu()
    want = x.to(BF16)
    nan = torch.isnan(x)
    assert bool(torch.isnan(got[nan]).all())  # NaN stays NaN (payload unspecified)
    assert torch.equal(bits16(got)[~nan], bits16(want)[~nan])


def test_bf16_to_f32_every_pattern():
    L, lib = _lib()
    pat = torch.arange(1 << 16, dtype=torch.int32)
    x = pat.to(torch.int16).view(BF16).cuda()  # every bf16 bit pattern, NaNs included
    y = torch.empty(1 << 16, device="cuda")
    L.check(lib.sgpt_bf16_to_f32(x.data_ptr(), y.data_ptr(), 1 << 16, L.current_stream()))
    assert torch.equal(y.cpu().view(torch.int32), pat << 16)  # exact widening, bit for bit


@pytest.mark.parametrize("B", [1, 13])
@pytest.mark.parametrize("d", [1, 33, 4097])
def test_normalize_rows_fp64(B, d):
    L, lib = _lib()
    g = torch.Generator().manual_seed(B * d)
    x = torch.randn(B, d, generator=g) * 3
    x[0] = 0.0  # stays 0
    if B > 2:
        x[1] *= 1e-20  # norm below 1e-12: divided by 1e-12
        x[2] *= 1e15  # large, but its squares stay finite in fp32
    xd = x.cuda()
    L.check(lib.sgpt_normalize_rows(xd.data_ptr(), B, d, L.current_stream()))
    xx = x.double()
    want = xx / xx.norm(dim=1, keepdim=True).clamp(min=1e-12)
    # per lane ceil(d/32) fmaf, a 5-level shuffle tree, sqrtf, the division and the scaling
    tol = want.abs() * ((d + 31) // 32 + 16) * U
    got = xd.cpu().double()
    assert bool(((got - want).abs() <= tol).all()), float((got - want).abs().max())
    assert bool((got[0] == 0).all())
