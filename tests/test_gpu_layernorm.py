"""LayerNorm pass over the bf16 residual stream (HF:gpt_neo/modeling_gpt_neo.py:332,344 `self.ln_1` / `self.ln_2` =
nn.LayerNorm(hidden_size, eps)) through the C ABI, every kernel instance the width dispatch can pick — persistent groups
with gamma / beta in registers (default) and the one-row-per-group kernels (SGPT_LN_PERSIST=0 is read at first use, so
those are reached through widths without a persistent instance) — against torch.nn.functional.layer_norm in fp64 on
the same bf16 inputs, to one bf16 rounding of the output.  Also in place (BLOOM's embedding LayerNorm)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


# widths: 768 (<32,3> persistent), 1024 (<32,4> one-row), 2048 / 1536 (<128,2> persistent), 2560 / 4096 (<256,2>
# persistent), 5120 (<256,4> one-row), 64 (tiny); row counts straddle the grid-stride loop (SMs x MINB CTAs x rows) of
# the H100's 132 SMs (2112 / 2113) and of a 148-SM part
@pytest.mark.parametrize("T,d", [(1, 768), (7, 768), (2112, 768), (2113, 768), (2368, 768), (2369 + 8 * 296, 768), (33000, 768), (300, 1024),
                                 (5, 2048), (1777, 2048), (9001, 1536), (3, 4096), (1333, 4096), (2000, 2560),
                                 (700, 5120), (19, 64)])
@pytest.mark.parametrize("in_place", [False, True])
def test_layernorm_bf16_stream_vs_torch(T, d, in_place):
    L, lib = _lib()
    g = torch.Generator().manual_seed(T * 31 + d)
    x = (torch.randn(T, d, generator=g) * 2.5 + 0.4)
    x[:, 3] += 30.0  # an outlier feature, as GPT residual streams have
    xb = x.to(torch.bfloat16)
    gamma = 1.0 + 0.3 * torch.randn(d, generator=g)
    beta = 0.2 * torch.randn(d, generator=g)
    eps = 1e-5
    want = torch.nn.functional.layer_norm(xb.double(), (d,), gamma.double(), beta.double(), eps)
    xd = xb.cuda()
    yd = xd if in_place else torch.full((T + 1, d), 7.0, dtype=torch.bfloat16, device="cuda")
    gd, bd = gamma.cuda(), beta.cuda()
    L.check(lib.sgpt_layernorm_ex(xd.data_ptr(), 1, gd.data_ptr(), bd.data_ptr(), yd.data_ptr(), T, d, eps,
                                  L.current_stream()))
    torch.cuda.synchronize()
    got = yd[:T].cpu().double()
    tol = want.abs() * 2.0 ** -8 + 1e-3  # one bf16 rounding (2^-9 relative) with slack for the fp32 statistics
    err = (got - want).abs()
    assert bool((err <= tol).all()), float((err - tol).max())
    if not in_place:
        assert bool((yd[T] == 7.0).all())  # nothing written past the last row
