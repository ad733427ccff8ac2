"""CPU restatement of the fp8 linear layers of include/sgpt_b200.h (test infrastructure only): the e4m3 row quantization,
and a quantization-aware forward of the three architectures — the oracle forwards (oracle/gpt_neo.py, gptj.py,
bloom.py) with every linear layer replaced by quantize -> dequantized matmul -> scaled epilogue."""
from __future__ import annotations

import numpy as np
import torch

E4M3_MAX = 448.0


def e4m3_grid() -> np.ndarray:
    """Every finite non-negative e4m3 value (bit patterns 0x00..0x7e; 0x7f is NaN), decoded from the format's definition
    (1 sign, 4 exponent bits with bias 7, 3 mantissa bits, subnormals at exponent 0), ascending; index = bit pattern."""
    vals = []
    for b in range(0x7F):
        e, m = b >> 3, b & 7
        vals.append(m / 8.0 * 2.0 ** -6 if e == 0 else (1 + m / 8.0) * 2.0 ** (e - 7))
    return np.array(vals)


def cvt_satfinite_e4m3(x: np.ndarray) -> np.ndarray:
    """cvt.rn.satfinite.e4m3 restated from the format alone: round to the nearest finite e4m3 value, ties to the even
    bit pattern, magnitudes beyond 448 to +-448, NaN to NaN.  Independent of torch's cast, so a test can check that
    torch's float8_e4m3fn cast after a clamp to +-448 is the same map."""
    x = np.asarray(x, dtype=np.float64)
    grid = e4m3_grid()
    a = np.minimum(np.abs(x), E4M3_MAX)
    hi = np.clip(np.searchsorted(grid, a, side="left"), 0, len(grid) - 1)
    lo = np.maximum(hi - 1, 0)
    dlo, dhi = a - grid[lo], grid[hi] - a
    pick_hi = (dhi < dlo) | ((dhi == dlo) & (hi % 2 == 0))
    out = np.where(pick_hi, grid[hi], grid[lo])
    out = np.where(a == grid[hi], grid[hi], out)
    out = np.copysign(out, x)
    return np.where(np.isnan(x), np.nan, out)


def quantize_rows(x: torch.Tensor):
    """Row quantization of include/sgpt_b200.h on bf16-valued rows x [..., K]: returns (q float8_e4m3fn [..., K], scale fp32
    [...]).  inv = min(448 / amax, FLT_MAX) in fp32, q = e4m3(x * inv) (fp32 product; torch's cast after a clamp to
    +-448 is cvt.rn.satfinite), scale = amax / 448; zero rows: q = 0, scale = 0; rows holding NaN / inf: q = 0,
    scale = NaN."""
    x = x.float()
    finite = torch.isfinite(x).all(dim=-1)
    amax = torch.where(finite, x.abs().amax(dim=-1), torch.zeros((), dtype=torch.float32))
    inv = torch.where(amax > 0, torch.clamp(torch.tensor(E4M3_MAX, dtype=torch.float32) / amax,
                                            max=torch.finfo(torch.float32).max), torch.zeros((), dtype=torch.float32))
    y = torch.where(finite[..., None], x * inv[..., None], torch.zeros((), dtype=torch.float32))
    q = y.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    scale = torch.where(finite, amax / torch.tensor(E4M3_MAX, dtype=torch.float32),
                        torch.full_like(amax, float("nan")))
    return q, scale


def linear_fp8(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """The fp8 GEMM's value before bias / activation: ((q_x q_w^T) * s_x[m]) * s_w[n], the dot products in fp64 rounded
    to fp32 (the accumulator), the scales applied in fp32 in that order.  x and w are rounded to bf16 first: the A
    operand and the weight the GPU quantizes are bf16 tensors."""
    qx, sx = quantize_rows(x.to(torch.bfloat16))
    qw, sw = quantize_rows(w.to(torch.bfloat16))
    acc = (qx.double() @ qw.double().T).float()
    return acc * sx[..., None] * sw


class _Fp8Weight:
    """A linear weight as the oracle forwards use it (``x @ w.T``): ``x @ q.T`` evaluates linear_fp8(x, w).  torch's
    matmul returns NotImplemented for an operand that is not a tensor, so Python calls __rmatmul__."""

    def __init__(self, w: torch.Tensor):
        self.w = w

    @property
    def T(self):
        return self

    def __rmatmul__(self, x):
        return linear_fp8(x, self.w)


_EMBEDDINGS = ("wte.weight", "wpe.weight", "word_embeddings.weight")


def fp8_weights(w: dict) -> dict:
    """The state dict with every linear weight (the 2-D weights that are not embedding tables) wrapped as _Fp8Weight."""
    return {k: (_Fp8Weight(v) if (v.dim() == 2 and k not in _EMBEDDINGS) else v) for k, v in w.items()}


def forward_fp8(module, spec, w: dict, input_ids, attention_mask=None):
    """Quantization-aware forward: module.forward (oracle.gpt_neo / gptj / bloom) with fp8 linear layers, quantized at
    the four points of the contract (LayerNorm output, attention output, gelu output; weights per output channel)."""
    return module.forward(spec, fp8_weights(w), input_ids, attention_mask)
