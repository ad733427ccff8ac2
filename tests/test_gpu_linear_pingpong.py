"""sgpt_linear and sgpt_linear_qkv_rotary bit for bit at the work-unit edges of the ping-pong linear GEMM: odd tile counts
per CTA (one consumer warpgroup takes one tile more than the other), fewer tiles than SMs, M and N tails, one k-block,
banded rasterisation, split-K 2 and 4, and the GPT-J rotary projection.

The operands are small integers, so every accumulator is exact in fp32 whatever the summation order, and the reference
is the epilogue's own arithmetic in torch fp32: acc + bias, then bf16 round-to-nearest-even.  The reduce-add cases keep
every partial sum an integer of at most 256 in magnitude (exact in bf16), so the L2's bf16 adds are exact in any order.
The rotary table holds multiples of 1/8, which makes both products of a rotated pair exact.  gelu_new uses the hardware
tanh approximation, which torch does not have: it is held to one bf16 unit in the last place plus that
approximation's error."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


@pytest.fixture
def gemm_env():
    keys = ("SGPT_GEMM_SPLITK", "SGPT_GEMM_BAND")
    old = {k: os.environ.get(k) for k in keys}
    yield os.environ
    for k, v in old.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def _ints(shape, lo, hi, g, p_zero=0.0):
    t = torch.randint(lo, hi + 1, shape, generator=g).float()
    if p_zero > 0:
        t = t * (torch.rand(shape, generator=g) >= p_zero)
    return t


def _gelu_new_f32(x):
    k0, k1 = 0.7978845608028654, 0.044715
    return 0.5 * x * (1.0 + torch.tanh(k0 * (x + k1 * x * x * x)))


def _ulp_bf16(x):
    """one bf16 unit in the last place of each element of x (float32)"""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _run_linear(epi, x, w, bias, out):
    L, lib = _lib()
    M, K = x.shape
    N = w.shape[0]
    code = {"bf16": L.EPI_BF16, "gelu": L.EPI_GELU_BF16, "resid": L.EPI_RESID_BF16}[epi]
    xd, wd = x.to(torch.bfloat16).cuda(), w.to(torch.bfloat16).cuda()
    bd = bias.cuda() if bias is not None else None
    od = out.cuda()
    L.check(lib.sgpt_linear(xd.data_ptr(), K, wd.data_ptr(), K, L.ptr(bd), od.data_ptr(), N,
                            od.data_ptr() if epi == "resid" else None, M, N, K, code, L.current_stream()),
            f"sgpt_linear {epi} M={M} N={N} K={K}")
    torch.cuda.synchronize()
    return od.cpu()


# (M, N, K, band): 19 x 15 = 285 tiles (two or three per CTA: odd counts on some CTAs, each consumer's tile sequence
# wraps the ring); 6 tiles (one per CTA, fewer tiles than SMs) with M and N tails; one k-block; 135 tiles in bands of 3
# (M-fastest order, last band lower)
SHAPES = [(2432, 1920, 256, 0), (300, 200, 512, 0), (1000, 392, 64, 0), (1920, 1152, 128, 3)]


@pytest.mark.parametrize("M,N,K,band", SHAPES)
@pytest.mark.parametrize("with_bias", [True, False])
def test_bias_epilogue_bits(M, N, K, band, with_bias, gemm_env):
    gemm_env["SGPT_GEMM_BAND"] = str(band)
    g = torch.Generator().manual_seed(M + N + K)
    x, w = _ints((M, K), -3, 3, g), _ints((N, K), -3, 3, g)
    bias = torch.randn(N, generator=g) * 8 if with_bias else None
    got = _run_linear("bf16", x, w, bias, torch.full((M, N), float("nan"), dtype=torch.bfloat16))
    acc = x @ w.T  # exact: |acc| <= 9 K < 2^24
    want = (acc + bias if with_bias else acc + 0.0).to(torch.bfloat16)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
        f"M={M} N={N} K={K}: {int((got.view(torch.int16) != want.view(torch.int16)).sum())} elements differ"


@pytest.mark.parametrize("M,N,K,band", SHAPES[:2])
def test_gelu_epilogue(M, N, K, band, gemm_env):
    gemm_env["SGPT_GEMM_BAND"] = str(band)
    g = torch.Generator().manual_seed(M * 3 + N)
    x, w = _ints((M, K), -2, 2, g, 0.8), _ints((N, K), -2, 2, g, 0.8)
    bias = torch.randn(N, generator=g)
    got = _run_linear("gelu", x, w, bias, torch.full((M, N), float("nan"), dtype=torch.bfloat16)).float()
    pre = x @ w.T + bias
    want = _gelu_new_f32(pre)
    # one bf16 ulp, and tanh.approx.f32's absolute error of 2^-11 scaled by 0.5 |pre|
    err = (got - want).abs()
    assert bool((err <= _ulp_bf16(want) + 2.0 ** -11 * pre.abs() + 2.0 ** -20).all()), float(err.max())


@pytest.mark.parametrize("M,N,K,split", [(1000, 768, 2048, 2), (300, 392, 4096, 4), (2432, 640, 2048, 2)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_residual_epilogue_bits(M, N, K, split, with_bias, gemm_env):
    """reduce-add into the residual stream, unsplit and split into `split` K slices: exact, so both are bit-identical"""
    g = torch.Generator().manual_seed(M + K + split)
    x, w = _ints((M, K), -1, 1, g, 0.9), _ints((N, K), -1, 1, g, 0.9)
    bias = _ints((N,), -8, 8, g) if with_bias else None
    r0 = _ints((M, N), -16, 16, g).to(torch.bfloat16)
    acc = x @ w.T
    pre = acc + bias if with_bias else acc + 0.0
    slices = [x[:, s:s + K // split] @ w[:, s:s + K // split].T for s in range(0, K, K // split)]
    assert max(float(pre.abs().max()), float((r0.float() + pre).abs().max()),
               max(float(p.abs().max()) for p in slices)) <= 256, "operands outside the exact regime"
    want = (r0.float() + pre).to(torch.bfloat16)
    for setting in ("0", str(split)):
        gemm_env["SGPT_GEMM_SPLITK"] = setting
        got = _run_linear("resid", x, w, bias, r0.clone())
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
            f"split {setting}: {int((got.view(torch.int16) != want.view(torch.int16)).sum())} elements differ"


@pytest.mark.parametrize("M,d,hd,rd", [(700, 256, 64, 32), (2500, 512, 128, 64)])
def test_rotary_epilogue_bits(M, d, hd, rd):
    L, lib = _lib()
    g = torch.Generator().manual_seed(M + d)
    max_pos = 600
    x, w = _ints((M, d), -3, 3, g), _ints((3 * d, d), -3, 3, g)
    cos_sin = _ints((max_pos, rd // 2, 2), -8, 8, g) / 8
    pos = torch.randint(-5, max_pos + 5, (M,), generator=g, dtype=torch.int32)  # clamped into the table by the kernel
    out = torch.full((M, 3 * d), float("nan"), dtype=torch.bfloat16, device="cuda")
    xd, wd = x.to(torch.bfloat16).cuda(), w.to(torch.bfloat16).cuda()
    pd, csd = pos.cuda(), cos_sin.cuda()
    L.check(lib.sgpt_linear_qkv_rotary(xd.data_ptr(), d, wd.data_ptr(), out.data_ptr(), pd.data_ptr(), csd.data_ptr(), M,
                                       d, hd, rd, max_pos, L.current_stream()), "sgpt_linear_qkv_rotary")
    torch.cuda.synchronize()
    y = x @ w.T  # exact
    want = y.clone()
    cs = cos_sin[pos.clamp(0, max_pos - 1).long()]  # [M, rd/2, 2]
    for h in range(2 * d // hd):  # q and k heads
        base = h * hd
        e, od = y[:, base:base + rd:2], y[:, base + 1:base + rd:2]
        c, s = cs[..., 0], cs[..., 1]
        want[:, base:base + rd:2] = e * c - od * s
        want[:, base + 1:base + rd:2] = od * c + e * s
    want = want.to(torch.bfloat16)
    got = out.cpu()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
        f"{int((got.view(torch.int16) != want.view(torch.int16)).sum())} elements differ"
