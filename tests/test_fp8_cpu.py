"""CPU checks of the fp8 linear layers: argument validation of every new entry point (before any CUDA call, so no GPU is
needed), the row quantization of the reference (tests/fp8_ref.py) and Encoder(precision=) validation."""
import ctypes

import numpy as np
import pytest
import torch

from tests import fp8_ref


def _lib():
    from sgpt_b200 import _lib

    return _lib.lib()


_DUMMY = np.zeros(64, dtype=np.int64)
P = _DUMMY.ctypes.data  # 16-byte aligned host memory, never dereferenced: every call below is rejected first


QUANTIZE_REJECTIONS = [
    (4, 24, P, b"K=24 must be a positive multiple of 16"),
    (4, 0, P, b"K=0 must be a positive multiple of 16"),
    (-1, 16, P, b"bad row count"),
    (4, 16, None, b"null argument"),
    (4, 16, P + 8, b"16-byte aligned"),
]


def _quantize_case_id(n, K, x, message):
    """The pointer as an offset from P: P itself is a heap address, which differs from one process to the next."""
    return f"{n}-{K}-{'None' if x is None else f'P+{x - P}'}-{message.decode()}"


@pytest.mark.parametrize("n,K,x,message", QUANTIZE_REJECTIONS, ids=[_quantize_case_id(*c) for c in QUANTIZE_REJECTIONS])
def test_quantize_rows_fp8_rejects_bad_arguments(n, K, x, message):
    lib = _lib()
    assert lib.sgpt_quantize_rows_fp8(x, P, P, n, K, None) == 1
    assert message in lib.sgpt_last_error()


def test_quantize_rows_fp8_empty_is_a_no_op():
    assert _lib().sgpt_quantize_rows_fp8(None, None, None, 0, 16, None) == 0


def _linear(epilogue=0, K=32, ldx=32, ldw=32, xs=P, ws=P, resid=None, out=P, M=4, N=8, ldo=8):
    return _lib().sgpt_linear_fp8(P, ldx, xs, P, ldw, ws, None, out, ldo, resid, M, N, K, epilogue, None)


@pytest.mark.parametrize("kw,message", [
    (dict(K=24, ldx=24, ldw=24), b"multiples of 16"),
    (dict(ldx=40), b"multiples of 16"),
    (dict(ldx=16), b"row pitch smaller than the row"),
    (dict(xs=None), b"null operand or scale"),
    (dict(ws=None), b"null operand or scale"),
    (dict(epilogue=2), b"unknown epilogue 2"),
    (dict(epilogue=100), b"unknown epilogue 100"),
    (dict(epilogue=3, resid=None), b"resid must alias out"),
    (dict(ldo=4), b"ldo must be >= N"),
    (dict(M=-1), b"bad sizes"),
])
def test_linear_fp8_rejects_bad_arguments(kw, message):
    assert _linear(**kw) == 1
    assert message in _lib().sgpt_last_error()


def test_linear_fp8_rejects_split_k(monkeypatch):
    monkeypatch.setenv("SGPT_GEMM_SPLITK", "2")
    assert _linear(epilogue=3, resid=P) == 1
    assert b"split-K is not supported" in _lib().sgpt_last_error()


def test_linear_fp8_empty_is_a_no_op():
    assert _linear(M=0) == 0


@pytest.mark.parametrize("kw,message", [
    (dict(d=40), b"multiples of 16"),
    (dict(xs=None), b"null operand or scale"),
    (dict(ws=None), b"null operand or scale"),
    (dict(head_dim=24), b"bad head_dim 24"),
    (dict(rotary_dim=12), b"rotary_dim 12"),
    (dict(pos=None), b"pos / cos_sin missing"),
])
def test_linear_qkv_rotary_fp8_rejects_bad_arguments(kw, message):
    a = dict(d=64, xs=P, ws=P, head_dim=32, rotary_dim=16, pos=P)
    a.update(kw)
    lib = _lib()
    rc = lib.sgpt_linear_qkv_rotary_fp8(P, a["d"], a["xs"], P, a["ws"], P, a["pos"], P, 4, a["d"], a["head_dim"],
                                        a["rotary_dim"], 64, None)
    assert rc == 1
    assert message in lib.sgpt_last_error()


def _create_fp8(fp8_layers, n_layer=2):
    from sgpt_b200 import _lib as L

    cfg = L.ModelConfigC(arch=L.ARCH_GPT_NEO, n_layer=n_layer, d_model=64, n_head=1, d_ff=256, vocab=10, max_pos=8,
                         window=0, rotary_dim=0, ln_eps=1e-5, max_tokens=16, max_batch=2)
    layers = (L.LayerWeightsC * n_layer)()
    for lw in layers:  # LayerNorm parameters only: the bf16 linear pointers are not read by an fp8 handle
        lw.ln1_g = lw.ln1_b = lw.ln2_g = lw.ln2_b = P
    mw = L.ModelWeightsC(wte=P, wpe=P, lnf_g=P, lnf_b=P, layers=layers)
    handle = ctypes.c_void_p()
    return _lib().sgpt_model_create_fp8(ctypes.byref(cfg), ctypes.byref(mw), fp8_layers, ctypes.byref(handle))


def test_model_create_fp8_rejects_missing_weights():
    from sgpt_b200 import _lib as L

    lib = _lib()
    assert _create_fp8(None) == 1
    assert b"null fp8 layer weights" in lib.sgpt_last_error()
    fl = (L.Fp8LayerWeightsC * 2)()
    for f in fl:
        for name, _ in L.Fp8LayerWeightsC._fields_:
            setattr(f, name, P)
    fl[1].s_fc = None  # one missing scale
    assert _create_fp8(fl) == 1
    assert b"layer 1 has missing weights" in lib.sgpt_last_error()


def test_torch_cast_after_clamp_is_cvt_rn_satfinite():
    """The reference quantizes with torch's float8_e4m3fn cast after a clamp to +-448; this is the cvt.rn.satfinite of the
    kernel: every e4m3 value, every midpoint between neighbours (ties to even), points just off the midpoints, the
    subnormal range, the saturation edge and random magnitudes over the whole range, both signs."""
    grid = fp8_ref.e4m3_grid()
    mids = (grid[1:] + grid[:-1]) / 2
    g = np.random.default_rng(0)
    xs = np.concatenate([grid, mids, np.nextafter(mids.astype(np.float32), np.float32(np.inf)),
                         np.nextafter(mids.astype(np.float32), np.float32(0)),
                         np.linspace(0, 2.0 ** -6, 4097), [447.9, 448, 449, 464, 465, 480, 1e6, 3.4e38],
                         np.exp(g.uniform(np.log(1e-5), np.log(500), 200000))]).astype(np.float32)
    xs = np.concatenate([xs, -xs])
    want = fp8_ref.cvt_satfinite_e4m3(xs.astype(np.float64))
    got = torch.from_numpy(xs).clamp(-448, 448).to(torch.float8_e4m3fn).double().numpy()
    np.testing.assert_array_equal(got, want)
    assert np.isnan(fp8_ref.cvt_satfinite_e4m3(np.array([np.nan]))).all()


def test_quantize_rows_properties():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(64, 768, generator=g) * torch.logspace(-30, 30, 64)[:, None]).to(torch.bfloat16)
    x[3] = 0
    x[5, 7] = float("nan")
    x[6, 0] = float("inf")
    x[7, 1] = -float("inf")
    x[8] = 0
    x[8, 100] = -3.0  # a single non-zero element maps to -448
    q, s = fp8_ref.quantize_rows(x)
    qf = q.float()
    assert qf.abs().max() <= 448
    assert s[3] == 0 and (qf[3] == 0).all()
    assert torch.isnan(s[5:8]).all() and (qf[5:8] == 0).all()
    assert qf[8, 100] == -448 and (qf[8].abs().sum() == 448) and s[8] == torch.tensor(3.0) / 448
    ok = torch.isfinite(s) & (s > 0)
    # the largest magnitude of every row maps to +-448, and the dequantized row is within half an e4m3 ulp (2^-4
    # relative) of x wherever x is a normal e4m3 value after scaling
    assert (qf[ok].abs().amax(dim=1) == 448).all()
    xf, deq = x.float()[ok], (qf * s[:, None])[ok]
    normal = (xf.abs() / s[ok][:, None]) >= 2.0 ** -6
    assert ((deq - xf).abs() <= 2.0 ** -4 * xf.abs() * 1.0001)[normal].all()


def test_quantize_rows_tiny_rows_stay_finite():
    """inv = 448 / amax overflows fp32 for amax below ~1.3e-36 (bf16 reaches 9e-41); it saturates to FLT_MAX, so zeros of
    such a row stay 0 instead of 0 * inf = NaN."""
    x = torch.zeros(1, 16, dtype=torch.bfloat16)
    x[0, 0] = 1e-39
    q, s = fp8_ref.quantize_rows(x)
    assert torch.isfinite(q.float()).all() and (q.float()[0, 1:] == 0).all() and q.float()[0, 0] > 0
    assert torch.isfinite(s).all()


def test_encoder_rejects_unknown_precision():
    from sgpt_b200 import CustomEmbedder, ModelConfig
    from sgpt_b200.cross_encoder import LogLikelihoodScorer
    from sgpt_b200.encoder import Encoder

    cfg = ModelConfig(n_layer=1, d_model=64, n_head=1, d_ff=256, vocab=10, max_pos=8)
    for bad in ("fp16", "int8", "FP8", None):
        with pytest.raises(ValueError, match="precision must be 'bf16' or 'fp8'"):
            Encoder(cfg, {}, device="cuda:0", precision=bad)
    with pytest.raises(ValueError, match="precision must be"):
        LogLikelihoodScorer(cfg, {}, precision="e4m3")
    with pytest.raises(ValueError, match="precision must be"):
        CustomEmbedder(config=cfg, state_dict={}, tokenizer=object(), precision="fp4")


def test_fp8_reference_forward_matches_exact_linear_on_e4m3_data():
    """linear_fp8 on operands that are already e4m3 values times a power of two per row is the exact product."""
    g = torch.Generator().manual_seed(1)
    grid = torch.tensor(fp8_ref.e4m3_grid(), dtype=torch.float32)
    x = grid[torch.randint(0, 127, (8, 64), generator=g)] * torch.sign(torch.randn(8, 64, generator=g))
    w = grid[torch.randint(0, 127, (16, 64), generator=g)] * torch.sign(torch.randn(16, 64, generator=g))
    x[:, 0], w[:, 0] = 448, -448  # amax = 448 per row: scale 1
    want = (x.double() @ w.double().T).float()
    assert torch.equal(fp8_ref.linear_fp8(x, w), want)
