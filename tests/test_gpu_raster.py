"""Tile rasterisation of the linear-layer GEMM (gemm.cuh TileMap::band): the order in which the persistent CTAs visit the
output tiles changes which operand tiles are live in the L2, never the arithmetic of a tile.  sgpt_linear through the C ABI
with SGPT_GEMM_BAND forced to 0 (N fastest) / 3 / 8 (banded M-fastest; 3 leaves a lower last band) must give bit-identical
outputs, and they must equal fp64 torch arithmetic on the same inputs within bf16 rounding (HF:gpt_neo:342-350 nn.Linear)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture
def band_env():
    old = {k: os.environ.get(k) for k in ("SGPT_GEMM_BAND",)}
    yield
    for k, v in old.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


@pytest.mark.parametrize("M,K,N,epi", [(2700, 256, 1304, "bf16"), (5000, 512, 768, "gelu"), (1290, 1024, 520, "resid"),
                                       (40000, 768, 2304, "bf16")])
def test_linear_is_independent_of_the_tile_order(M, K, N, epi, band_env):
    from sgpt_b200 import _lib as L

    lib = L.lib()
    g = torch.Generator().manual_seed(M + K + N)
    x = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    b = torch.randn(N, generator=g)
    r0 = (torch.randn(M, N, generator=g) * 2).to(torch.bfloat16)
    acc = x.double() @ w.double().T + b.double()
    if epi == "gelu":  # gelu_new, HF:activations NewGELUActivation
        want = 0.5 * acc * (1.0 + torch.tanh(0.7978845608028654 * (acc + 0.044715 * acc ** 3)))
    elif epi == "resid":
        want = r0.double() + acc
    else:
        want = acc
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    code = {"bf16": L.EPI_BF16, "gelu": L.EPI_GELU_BF16, "resid": L.EPI_RESID_BF16}[epi]
    results = {}
    for setting in ("0", "3", "8"):
        os.environ["SGPT_GEMM_BAND"] = setting
        out = r0.clone().cuda() if epi == "resid" else torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
        L.check(lib.sgpt_linear(xd.data_ptr(), K, wd.data_ptr(), K, bd.data_ptr(), out.data_ptr(), N,
                                out.data_ptr() if epi == "resid" else None, M, N, K, code, L.current_stream()))
        torch.cuda.synchronize()
        results[setting] = out.cpu()
    assert torch.equal(results["0"], results["3"]) and torch.equal(results["0"], results["8"])
    err = (results["8"].double() - want).abs()
    assert bool((err <= 0.02 + 0.01 * want.abs()).all()), float(err.max())
    # run to run: the same tile order again gives the same bits (several tiles per CTA: the epilogue of one tile and the
    # operand loads of the next overlap)
    os.environ["SGPT_GEMM_BAND"] = "0"
    for _ in range(2):
        out = r0.clone().cuda() if epi == "resid" else torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
        L.check(lib.sgpt_linear(xd.data_ptr(), K, wd.data_ptr(), K, bd.data_ptr(), out.data_ptr(), N,
                                out.data_ptr() if epi == "resid" else None, M, N, K, code, L.current_stream()))
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), results["0"])
