"""Split-K of the residual (reduce-add) linear layers: out = resid + x W^T + b (HF:gpt_neo:342,348 — the attention
out-projection and the MLP c_proj added onto the residual stream) must not depend on how many K slices a tile is computed
in, beyond the rounding of the extra adds.  sgpt_linear through the C ABI with SGPT_GEMM_SPLITK forced to 0 / 2 / 3 / 4
(read per call) and in its automatic setting, against fp64 torch arithmetic on the CPU from the same inputs."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


@pytest.fixture
def splitk_env():
    old = os.environ.get("SGPT_GEMM_SPLITK")
    yield
    if old is None:
        os.environ.pop("SGPT_GEMM_SPLITK", None)
    else:
        os.environ["SGPT_GEMM_SPLITK"] = old


@pytest.mark.parametrize("M,K,N", [(300, 2048, 768), (1000, 3072, 768), (129, 4096, 320), (2500, 8192, 2048)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_residual_linear_is_independent_of_the_k_split(M, K, N, with_bias, splitk_env):
    L, lib = _lib()
    g = torch.Generator().manual_seed(M + K + N)
    x = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    b = torch.randn(N, generator=g) if with_bias else None
    r0 = (torch.randn(M, N, generator=g) * 2).to(torch.bfloat16)
    want = r0.double() + x.double() @ w.double().T + (b.double() if with_bias else 0.0)
    xd, wd = x.cuda(), w.cuda()
    bd = b.cuda() if with_bias else None
    results = {}
    for setting in ("0", "2", "3", "4", None):
        if setting is None:
            os.environ.pop("SGPT_GEMM_SPLITK", None)
        else:
            os.environ["SGPT_GEMM_SPLITK"] = setting
        out = r0.clone().cuda()
        L.check(lib.sgpt_linear(xd.data_ptr(), K, wd.data_ptr(), K, bd.data_ptr() if with_bias else None, out.data_ptr(),
                                N, out.data_ptr(), M, N, K, L.EPI_RESID_BF16, L.current_stream()))
        torch.cuda.synchronize()
        results[setting] = out.cpu().double()
    # each extra slice rounds the running bf16 sum once more
    tol = 0.1 + 0.03 * want.abs()
    for setting, got in results.items():
        err = (got - want).abs()
        assert bool((err <= tol).all()), (setting, float(err.max()))
    # the split really happened for the long-K shapes: results of "0" and "2" differ in the last bits somewhere, or are equal
    # when the slice would be shorter than 16 k-blocks (K = 2048 / 3: unsplit)
    if K // 64 // 2 >= 16:
        assert not torch.equal(results["0"], results["2"])
