"""The linear-layer GEMM's two-CTA clusters bit for bit: each cluster computes a pair of vertically adjacent M-tiles and
multicasts the weight tile they share.  The cases are an odd M-tile count (the last pair's second CTA computes rows that
lie wholly past M and must still take part in every load and barrier), M below one tile, and more pair units than
clusters that fit on the GPU at once (every cluster walks several units and wraps its ring), in N-fastest and banded
order, for the bias, reduce-add and fp8 epilogues.  Two launches on the same operands must also return the same bits.

As in test_gpu_linear_pingpong.py, the operands are small integers: every accumulator is exact in fp32 whatever the
summation order, so the reference is the epilogue's own arithmetic in torch fp32 (acc + bias, then bf16
round-to-nearest-even) and nothing but the right rows and columns of the right k-blocks can match it."""
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


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g).float()


def _bits(t):
    return t.view(torch.int16)


def _linear(epi, x, w, bias, out):
    L, lib = _lib()
    M, K = x.shape
    N = w.shape[0]
    code = {"bf16": L.EPI_BF16, "resid": L.EPI_RESID_BF16}[epi]
    xd, wd = x.to(torch.bfloat16).cuda(), w.to(torch.bfloat16).cuda()
    bd = bias.cuda() if bias is not None else None
    od = out.cuda()
    L.check(lib.sgpt_linear(xd.data_ptr(), K, wd.data_ptr(), K, L.ptr(bd), od.data_ptr(), N,
                            od.data_ptr() if epi == "resid" else None, M, N, K, code, L.current_stream()),
            f"sgpt_linear {epi} M={M} N={N} K={K}")
    torch.cuda.synchronize()
    return od.cpu()


# (M, N, K, band): 9 M-tiles, the last one a single row; 5 whole M-tiles (the last pair's second tile wholly past M);
# M < 128 with an N tail; 32 x 18 tiles = 288 pair units, several per cluster, N-fastest and in bands of 3 pairs with
# the last band lower
SHAPES = [(1025, 392, 320, 0), (640, 256, 64, 0), (77, 200, 512, 0), (4096, 2304, 256, 0), (4096, 2304, 256, 3)]


@pytest.mark.parametrize("M,N,K,band", SHAPES)
def test_bias_epilogue_bits(M, N, K, band, gemm_env):
    gemm_env["SGPT_GEMM_BAND"] = str(band)
    g = torch.Generator().manual_seed(M + 7 * N + K)
    x, w = _ints((M, K), -3, 3, g), _ints((N, K), -3, 3, g)
    bias = torch.randn(N, generator=g) * 8
    got = _linear("bf16", x, w, bias, torch.full((M, N), float("nan"), dtype=torch.bfloat16))
    want = (x @ w.T + bias).to(torch.bfloat16)  # x @ w.T exact: |acc| <= 9 K < 2^24
    diff = _bits(got) != _bits(want)
    assert not bool(diff.any()), f"M={M} N={N} K={K} band={band}: {int(diff.sum())} elements differ"


@pytest.mark.parametrize("M,N,K,split", [(1025, 392, 2048, 1), (1025, 392, 2048, 2), (77, 768, 4096, 4)])
def test_residual_epilogue_bits(M, N, K, split, gemm_env):
    gemm_env["SGPT_GEMM_SPLITK"] = str(split)
    g = torch.Generator().manual_seed(M + N + K + split)
    # |x w| <= 1 per product and 128 nonzero products per row keep |acc + bias| + |resid| <= 208: every partial sum
    # and every sum of them is an integer exact in bf16, so the L2's adds are exact in any order
    x, w = _ints((M, K), -1, 1, g), _ints((N, K), -1, 1, g)
    x[:, 128:] = 0
    bias = _ints((N,), -16, 16, g)
    resid = _ints((M, N), -64, 64, g).to(torch.bfloat16)
    got = _linear("resid", x, w, bias, resid.clone())
    want = (resid.float() + (x @ w.T + bias)).to(torch.bfloat16)
    diff = _bits(got) != _bits(want)
    assert not bool(diff.any()), f"M={M} N={N} K={K} split={split}: {int(diff.sum())} elements differ"


@pytest.mark.parametrize("M,N,K", [(1025, 392, 320), (77, 200, 512), (4096, 2304, 256)])
def test_fp8_bias_epilogue_bits(M, N, K):
    L, lib = _lib()
    g = torch.Generator().manual_seed(3 * M + N + K)
    x, w = _ints((M, K), -4, 4, g), _ints((N, K), -4, 4, g)  # exact in e4m3
    bias = torch.randn(N, generator=g) * 8
    xq = x.to(torch.float8_e4m3fn).view(torch.uint8).cuda()
    wq = w.to(torch.float8_e4m3fn).view(torch.uint8).cuda()
    xs, ws = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
    od = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
    L.check(lib.sgpt_linear_fp8(xq.data_ptr(), K, xs.data_ptr(), wq.data_ptr(), K, ws.data_ptr(), bias.cuda().data_ptr(),
                                od.data_ptr(), N, None, M, N, K, L.EPI_BF16, L.current_stream()),
            f"sgpt_linear_fp8 M={M} N={N} K={K}")
    torch.cuda.synchronize()
    want = (x @ w.T + bias).to(torch.bfloat16)  # |acc| <= 16 K < 2^24: exact, and the scales are 1
    diff = _bits(od.cpu()) != _bits(want)
    assert not bool(diff.any()), f"M={M} N={N} K={K}: {int(diff.sum())} elements differ"


def test_two_launches_same_bits():
    """Real-valued operands at an SGPT-125M shape with an odd M-tile count: the k order of every tile is fixed, so two
    launches agree bit for bit."""
    g = torch.Generator().manual_seed(11)
    M, N, K = 4865, 2304, 768  # 39 M-tiles
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) * 0.02
    bias = torch.randn(N, generator=g) * 0.1
    nan = torch.full((M, N), float("nan"), dtype=torch.bfloat16)
    a = _linear("bf16", x, w, bias, nan.clone())
    b = _linear("bf16", x, w, bias, nan.clone())
    assert bool(torch.isfinite(a.float()).all())
    assert torch.equal(_bits(a), _bits(b))
