"""sgpt_linear at the edges of its tiles and sgpt_linear_qkv_rotary (GPT-J's fused q/k/v projection with the rotary
embedding in the epilogue), each against fp64 torch arithmetic on the same bf16 inputs, through the C ABI.

Tolerances are built from the arithmetic (tests/helpers.py): the GEMM accumulates in fp32 on the tensor cores
(tensor_core_sum_bound), the epilogue adds in fp32, and every bf16 store rounds with relative error <= u = 2^-8."""
import pytest
import torch

from tests.helpers import (BF16_U, left_padded_positions, rotary_abs_bound, rotary_cos_sin, rotary_reference,
                           tensor_core_sum_bound)

pytestmark = pytest.mark.gpu

U = BF16_U
F32 = 2.0 ** -23  # one fp32 ulp, relative


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))


def _padded(t, ld, fill):
    """t [rows, n] placed in the first n columns of a [rows, ld] buffer whose other columns hold `fill`."""
    buf = torch.full((t.shape[0], ld), fill, dtype=t.dtype)
    buf[:, :t.shape[1]] = t
    return buf


def _check_linear(epi, M, K, N, with_bias, padded, seed):
    """One sgpt_linear call.  With `padded` the row pitches exceed the rows: ldx > K and ldw > K with NaN in the pad
    columns (a read of them would poison the output), ldo > N with a sentinel in the pad columns (must keep its bits)."""
    L, lib = _lib()
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, K, generator=g)).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.1).to(torch.bfloat16)
    bias = torch.randn(N, generator=g) * 0.5 if with_bias else None
    ldx, ldw, ldo = (K + 24, K + 8, N + 40) if padded else (K, K, N)
    sentinel = -12352.0  # exact in bf16 and fp32
    resid = None
    if epi == "resid_bf16":  # in place: out starts as the residual
        resid = (torch.randn(M, N, generator=g) * 2).to(torch.bfloat16)
        out0 = _padded(resid, ldo, sentinel)
    else:  # every element the call must write starts as NaN
        out0 = _padded(torch.full((M, N), float("nan"), dtype=torch.bfloat16), ldo, sentinel)
    dev = "cuda"
    xd, wd = _padded(x, ldx, float("nan")).to(dev), _padded(w, ldw, float("nan")).to(dev)
    bd = bias.to(dev) if with_bias else None
    od = out0.to(dev)
    rd = od if resid is not None else None
    code = {"bf16": L.EPI_BF16, "gelu": L.EPI_GELU_BF16, "resid_bf16": L.EPI_RESID_BF16}[epi]
    L.check(lib.sgpt_linear(xd.data_ptr(), ldx, wd.data_ptr(), ldw, L.ptr(bd), od.data_ptr(), ldo, L.ptr(rd), M, N, K,
                            code, L.current_stream()), f"sgpt_linear {epi} M={M} K={K} N={N}")
    torch.cuda.synchronize()
    what = f"{epi} M={M} K={K} N={N} bias={with_bias} padded={padded}"
    got_full = od.cpu()
    assert torch.equal(got_full[:, N:].view(torch.int16), out0[:, N:].view(torch.int16)), \
        f"{what}: pad columns of out were written"
    got = got_full[:, :N].double()
    assert bool(torch.isfinite(got).all()), f"{what}: output not written or not finite"

    # fp64 reference and its bound
    acc = x.double() @ w.double().T
    e = tensor_core_sum_bound(x.double().abs() @ w.double().abs().T, K)
    pre = acc + (bias.double() if with_bias else 0.0)
    e_pre = e + F32 * pre.abs()  # fp32 bias add
    if epi == "bf16":
        want = pre
        tol = U * want.abs() + (1 + U) * e_pre
    elif epi == "gelu":
        # gelu_new's derivative is at most 1.13 in magnitude; tanh.approx.f32 errs by <= 2^-10 absolute (PTX ISA: max
        # relative error 2^-11 on |tanh| <= 1), i.e. 0.5 |pre| 2^-10 on the result; the cubic and the products are a few
        # fp32 ulps of |pre| (1 + pre^2)
        want = _gelu_new(pre)
        tol = U * want.abs() + (1 + U) * (1.13 * e_pre + 2.0 ** -11 * pre.abs() + 8 * F32 * pre.abs() * (1 + pre * pre))
    else:  # resid_bf16: acc + bias is rounded to bf16, then added to the bf16 residual by the TMA reduce (rounded again)
        want = resid.double() + pre
        tol = U * want.abs() + (1 + U) * (e_pre + U * pre.abs())
    err = (got - want).abs()
    if bool((err > tol).any()):
        m, n = (err > tol).nonzero()[0].tolist()
        raise AssertionError(f"{what}: out[{m},{n}] = {float(got[m, n])}, want {float(want[m, n])} (tol {float(tol[m, n])})")


@pytest.mark.parametrize("epi", ["bf16", "gelu", "resid_bf16"])
@pytest.mark.parametrize("M", [1, 2, 127, 129])
def test_linear_edge_shapes_vs_fp64(epi, M):
    """M around one 128-row tile, K tails below the 64-wide k-block (8, 72 = 64 + 8, 136 = 128 + 8), N column tails inside
    a 64-column output box (8, 136, 200: 200 also takes the per-element bias path for its last chunk), with and without
    bias, tight and padded row pitches."""
    for K in (8, 72, 136):
        for N in (8, 136, 200):
            for with_bias in (True, False):
                for padded in (False, True):
                    _check_linear(epi, M, K, N, with_bias, padded, seed=M * 1009 + K * 31 + N + with_bias + 2 * padded)


# (d_model, head_dim, rotary_dim): GPT-J-6B, rotary_dim == head_dim (twice), the smallest rotary_dim, hd 64 at d 768
ROTARY_GEOMETRIES = [(4096, 256, 64), (1024, 256, 256), (512, 64, 64), (512, 128, 8), (768, 64, 32)]


def _rotary_inputs(M, d, max_pos, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, d, generator=g).to(torch.bfloat16)
    w = (torch.randn(3 * d, d, generator=g) * d ** -0.5).to(torch.bfloat16)
    pos = left_padded_positions(M, max_pos, seed)
    return x, w, pos


@pytest.mark.parametrize("M", [1, 77, 129, 300])
@pytest.mark.parametrize("d,hd,rd", ROTARY_GEOMETRIES)
def test_linear_qkv_rotary_vs_fp64(d, hd, rd, M):
    """qkv = rotary(x w^T) (HF:gptj:98-101 projections, :55-67 + :196-207 rotate_every_two), positions of a left-padded
    batch up to max_pos - 1.  Bound: the fp32 GEMM error of each pre-rotary element (tensor_core_sum_bound) mixed by the
    rotation as |c| e0 + |s| e1, plus two fp32 roundings of the rotation (|y0 c| + |y1 s| <= S_rot), then the bf16 store:
    |got - ref| <= u |ref| + (1 + u) (e_rot + 2^-22 S_rot), S_rot the rotated sum of |x_k w_k|.
    The v columns and the dims past rotary_dim pass through: they must equal sgpt_linear's bias-free output bit for bit
    (same GEMM, same tiles)."""
    L, lib = _lib()
    max_pos = 2048
    x, w, pos = _rotary_inputs(M, d, max_pos, seed=M + d + rd)
    cos_sin = rotary_cos_sin(max_pos, rd)
    dev = "cuda"
    xd, wd, pd, csd = x.to(dev), w.to(dev), pos.to(dev), cos_sin.to(dev)
    out = torch.full((M, 3 * d), float("nan"), dtype=torch.bfloat16, device=dev)
    L.check(lib.sgpt_linear_qkv_rotary(xd.data_ptr(), d, wd.data_ptr(), out.data_ptr(), pd.data_ptr(), csd.data_ptr(), M,
                                       d, hd, rd, max_pos, L.current_stream()), "sgpt_linear_qkv_rotary")
    plain = torch.full((M, 3 * d), float("nan"), dtype=torch.bfloat16, device=dev)
    L.check(lib.sgpt_linear(xd.data_ptr(), d, wd.data_ptr(), d, None, plain.data_ptr(), 3 * d, None, M, 3 * d, d,
                            L.EPI_BF16, L.current_stream()), "sgpt_linear")
    torch.cuda.synchronize()
    got = out.cpu()
    assert bool(torch.isfinite(got).all())
    passthrough = torch.ones(3 * d, dtype=torch.bool)
    passthrough[:2 * d].view(-1, hd)[:, :rd] = False
    assert torch.equal(got[:, passthrough].view(torch.int16), plain.cpu()[:, passthrough].view(torch.int16)), \
        "v columns / non-rotary dims differ from the plain projection"

    xx, ww = x.double().to(dev), w.double().to(dev)
    want = rotary_reference(xx @ ww.T, pos.to(dev), cos_sin, d, hd, rd).cpu()
    s_rot = rotary_abs_bound(xx.abs() @ ww.abs().T, pos.to(dev), cos_sin, d, hd, rd)
    tol = (U * want.abs() + (1 + U) * (tensor_core_sum_bound(s_rot, d) + 2.0 ** -22 * s_rot).cpu())
    err = (got.double() - want).abs()
    if bool((err > tol).any()):
        m, n = (err > tol).nonzero()[0].tolist()
        raise AssertionError(f"{int((err > tol).sum())} elements out of tolerance; first qkv[{m},{n}] (head {n // hd}, dim "
                             f"{n % hd}, pos {int(pos[m])}) = {float(got[m, n])}, want {float(want[m, n])}")
