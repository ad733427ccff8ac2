"""Unit parity of the kernels that replace the stand-alone LayerNorm passes (include/sgpt_b200.h "LayerNorm without a
pass of its own"), each against fp64 torch arithmetic on the CPU from the same inputs, called through the C ABI:
sgpt_resid_stats, sgpt_fold_layernorm + sgpt_linear_lnfold (== act(LayerNorm(x) W^T + b), HF:gpt_neo:332-345 + :84-87 /
:304-305), sgpt_linear_resid_ln (== x W^T + b + residual, HF:gpt_neo:342,348, plus the statistics of the result)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))


@pytest.mark.parametrize("T,d", [(5, 128), (77, 192), (1000, 768), (300, 2048)])
def test_resid_stats(T, d):
    L, lib = _lib()
    g = torch.Generator().manual_seed(T + d)
    x = (torch.randn(T, d, generator=g) * 3 + 0.7)
    xd = x.cuda()
    P = (d + 127) // 128
    xb = torch.zeros(T, d, dtype=torch.bfloat16, device="cuda")
    st = torch.full((T, P, 2), float("nan"), device="cuda")
    L.check(lib.sgpt_resid_stats(xd.data_ptr(), xb.data_ptr(), st.data_ptr(), T, d, L.current_stream()))
    assert torch.equal(xb.cpu(), x.to(torch.bfloat16))
    pad = torch.nn.functional.pad(x.double(), (0, P * 128 - d)).view(T, P, 128)
    assert torch.allclose(st[..., 0].cpu().double(), pad.sum(-1), rtol=1e-5, atol=1e-3)
    assert torch.allclose(st[..., 1].cpu().double(), (pad * pad).sum(-1), rtol=1e-5, atol=1e-3)


@pytest.mark.parametrize("M,K,N,gelu", [(77, 128, 384, 0), (300, 768, 2304, 0), (1000, 768, 3072, 1), (130, 192, 576, 1)])
def test_linear_lnfold_equals_layernorm_then_linear(M, K, N, gelu):
    L, lib = _lib()
    g = torch.Generator().manual_seed(M + K + N)
    x = torch.randn(M, K, generator=g) * 2.0 + 0.5          # residual stream rows (non-zero mean)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    gamma, beta = torch.randn(K, generator=g) * 0.1 + 1.0, torch.randn(K, generator=g) * 0.05
    bias = torch.randn(N, generator=g) * 0.1
    eps = 1e-5
    dev = "cuda"
    wf = torch.empty(N, K, dtype=torch.bfloat16, device=dev)
    cs, bf = torch.empty(N, device=dev), torch.empty(N, device=dev)
    wd, gd, bd, biasd = w.to(dev), gamma.to(dev), beta.to(dev), bias.to(dev)
    L.check(lib.sgpt_fold_layernorm(wd.data_ptr(), gd.data_ptr(), bd.data_ptr(), biasd.data_ptr(), wf.data_ptr(),
                                    cs.data_ptr(), bf.data_ptr(), N, K, L.current_stream()))
    torch.cuda.synchronize()
    assert torch.equal(wf.cpu(), (w.float() * gamma).to(torch.bfloat16))
    assert torch.allclose(cs.cpu().double(), wf.cpu().double().sum(1), rtol=1e-5, atol=1e-4)
    assert torch.allclose(bf.cpu().double(), bias.double() + w.double() @ beta.double(), rtol=1e-5, atol=1e-4)
    P = (K + 127) // 128
    xd = x.to(dev)
    xb = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
    st = torch.empty(M, P, 2, device=dev)
    L.check(lib.sgpt_resid_stats(xd.data_ptr(), xb.data_ptr(), st.data_ptr(), M, K, L.current_stream()))
    out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=dev)
    L.check(lib.sgpt_linear_lnfold(xb.data_ptr(), K, wf.data_ptr(), K, bf.data_ptr(), cs.data_ptr(), st.data_ptr(), P, eps,
                                   out.data_ptr(), N, M, N, K, gelu, L.current_stream()), "sgpt_linear_lnfold")
    xx = x.double()
    ln = (xx - xx.mean(1, keepdim=True)) / torch.sqrt(xx.var(1, unbiased=False, keepdim=True) + eps) * gamma.double() + beta.double()
    want = ln @ w.double().T + bias.double()
    if gelu:
        want = _gelu_new(want)
    got = out.cpu().double()
    assert torch.isfinite(got).all()
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    assert err < 0.02 * scale, (err, scale)
    cos = torch.nn.functional.cosine_similarity(got, want, dim=1).min().item()
    assert cos > 1 - 2e-4, cos


@pytest.mark.parametrize("M,K,N,with_bias", [(77, 64, 128, True), (300, 768, 768, True), (1000, 3072, 768, True),
                                             (130, 256, 192, False), (513, 128, 2048, True)])
def test_linear_resid_ln(M, K, N, with_bias):
    L, lib = _lib()
    g = torch.Generator().manual_seed(M * 7 + K + N)
    x = (torch.randn(M, K, generator=g)).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(torch.bfloat16)
    bias = torch.randn(N, generator=g) * 0.1 if with_bias else None
    resid = torch.randn(M, N, generator=g) * 2 + 0.3
    dev = "cuda"
    xd, wd, rd = x.to(dev), w.to(dev), resid.to(dev).clone()
    bd = bias.to(dev) if with_bias else None
    P = (N + 127) // 128
    xb = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=dev)
    st = torch.full((M, P, 2), float("nan"), device=dev)
    L.check(lib.sgpt_linear_resid_ln(xd.data_ptr(), K, wd.data_ptr(), K, L.ptr(bd), rd.data_ptr(), xb.data_ptr(),
                                     st.data_ptr(), M, N, K, L.current_stream()), "sgpt_linear_resid_ln")
    want = resid.double() + x.double() @ w.double().T + (bias.double() if with_bias else 0.0)
    got = rd.cpu()
    assert torch.isfinite(got).all()
    assert (got.double() - want).abs().max().item() < 2e-3 * max(1.0, want.abs().max().item())
    assert torch.equal(xb.cpu(), got.to(torch.bfloat16))  # the bf16 copy is the rounding of exactly what was stored
    pad = torch.nn.functional.pad(got.double(), (0, P * 128 - N)).view(M, P, 128)
    assert torch.allclose(st[..., 0].cpu().double(), pad.sum(-1), rtol=1e-5, atol=2e-3)
    assert torch.allclose(st[..., 1].cpu().double(), (pad * pad).sum(-1), rtol=1e-5, atol=2e-3)
    # a second application accumulates on top (in place) — exercises both buffer parities again
    L.check(lib.sgpt_linear_resid_ln(xd.data_ptr(), K, wd.data_ptr(), K, L.ptr(bd), rd.data_ptr(), xb.data_ptr(),
                                     st.data_ptr(), M, N, K, L.current_stream()))
    want2 = want + x.double() @ w.double().T + (bias.double() if with_bias else 0.0)
    assert (rd.cpu().double() - want2).abs().max().item() < 4e-3 * max(1.0, want2.abs().max().item())


def _lnfold_fp32_bound(x, wf, w, beta, eps):
    """Bound on the fp32 error of act-free sgpt_linear_lnfold arithmetic, y = r acc - r mu c + b', against
    LayerNorm(x) W^T + b in exact arithmetic, for inputs where the bf16 copy of x and the folded weights are exact (x is
    bf16-representable, gamma a power of two).  Terms, each sum bounded by (number of roundings) * 2^-24 * (sum of |terms|):
      - acc = xb W'^T on the tensor cores: tensor_core_sum_bound;
      - column sums c and folded bias b' (one warp per row: K/32 terms per lane, then 5 shuffles): (K/32 + 5) 2^-24;
      - row sums of x and x^2 (8-term trees and 4 shuffles per 128-column group, then P groups): (8 + P) 2^-24, which
        moves mu by d_mu and var by d_var; 1/sqrt(var + eps) by rsqrtf (2 ulp) adds 2^-22, the products around it 2^-23;
      - the two fmas of the epilogue: 2^-23 of the magnitudes they combine.
    Returns the bound [M, N] (fp64) on the device of x."""
    from tests.helpers import tensor_core_sum_bound

    xx, wf, w, beta = x.double(), wf.double(), w.double(), beta.double()
    K = xx.shape[1]
    P = (K + 127) // 128
    mu = xx.mean(1, keepdim=True)
    ex2 = (xx * xx).mean(1, keepdim=True)
    var = ex2 - mu * mu
    r = 1.0 / torch.sqrt(var + eps)
    n_st, n_fold = (8 + P) * 2.0 ** -24, (K / 32 + 5) * 2.0 ** -24
    d_mu = n_st * xx.abs().mean(1, keepdim=True) + 2.0 ** -24 * mu.abs()
    d_var = n_st * ex2 + 2 * mu.abs() * d_mu + 2.0 ** -22 * (ex2 + mu * mu)
    rel_r = 0.5 * d_var / (var + eps) + 2.0 ** -22 + 2.0 ** -23
    a1, c1, b1 = xx.abs() @ wf.abs().T, wf.abs().sum(1), beta.abs() @ w.abs().T
    c = wf.sum(1)
    dev_term = (xx @ wf.T - mu * c).abs()  # |acc - mu c| = |sum_k (x_k - mu) W'_k|
    return (r * (tensor_core_sum_bound(a1, K) + mu.abs() * n_fold * c1 + c.abs() * d_mu) + n_fold * b1
            + rel_r * r * dev_term + 2.0 ** -23 * (r * (a1 + mu.abs() * c1) + b1))


@pytest.mark.parametrize("M", [1, 77, 129, 300])
@pytest.mark.parametrize("d,hd,rd", [(4096, 256, 64), (1024, 256, 256), (512, 128, 8), (768, 64, 32)])
def test_linear_qkv_rotary_lnfold_equals_layernorm_then_rotary_projection(d, hd, rd, M):
    """GPT-J's q/k/v projection with ln_1 folded in (sgpt_fold_layernorm + sgpt_resid_stats +
    sgpt_linear_qkv_rotary_lnfold) against fp64 LayerNorm(x) W^T followed by rotate_every_two on the first rotary_dim dims
    of every q and k head (HF:gptj:400, :98-101, :55-67 + :196-207), positions of a left-padded batch up to max_pos - 1.
    x is drawn in bf16 and gamma from {1/2, 1, 2}, so the bf16 copy of the residual and the folded weights are exact and
    the kernel differs from the reference only by fp32 arithmetic (_lnfold_fp32_bound, mixed by the rotation) and the bf16
    store (u = 2^-8).  v columns and non-rotary dims must equal sgpt_linear_lnfold's output bit for bit."""
    from tests.helpers import (BF16_U, left_padded_positions, rotary_abs_bound, rotary_cos_sin, rotary_reference)

    L, lib = _lib()
    max_pos, eps, dev = 2048, 1e-5, "cuda"
    N = 3 * d
    g = torch.Generator().manual_seed(M * 13 + d + rd)
    x = (torch.randn(M, d, generator=g) * 2.0 + 0.5).to(torch.bfloat16).float()  # residual stream rows, non-zero mean
    w = (torch.randn(N, d, generator=g) * d ** -0.5).to(torch.bfloat16)
    gamma = 2.0 ** torch.randint(-1, 2, (d,), generator=g).float()
    beta = torch.randn(d, generator=g) * 0.05
    pos = left_padded_positions(M, max_pos, seed=M + rd)
    cos_sin = rotary_cos_sin(max_pos, rd)
    wd, gd, bd, xd, pd, csd = w.to(dev), gamma.to(dev), beta.to(dev), x.to(dev), pos.to(dev), cos_sin.to(dev)
    wf = torch.empty(N, d, dtype=torch.bfloat16, device=dev)
    cs, bf = torch.empty(N, device=dev), torch.empty(N, device=dev)
    L.check(lib.sgpt_fold_layernorm(wd.data_ptr(), gd.data_ptr(), bd.data_ptr(), None, wf.data_ptr(), cs.data_ptr(),
                                    bf.data_ptr(), N, d, L.current_stream()), "sgpt_fold_layernorm")
    P = (d + 127) // 128
    xb = torch.empty(M, d, dtype=torch.bfloat16, device=dev)
    st = torch.empty(M, P, 2, device=dev)
    L.check(lib.sgpt_resid_stats(xd.data_ptr(), xb.data_ptr(), st.data_ptr(), M, d, L.current_stream()))
    out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=dev)
    L.check(lib.sgpt_linear_qkv_rotary_lnfold(xb.data_ptr(), d, wf.data_ptr(), bf.data_ptr(), cs.data_ptr(), st.data_ptr(),
                                              P, eps, out.data_ptr(), pd.data_ptr(), csd.data_ptr(), M, d, hd, rd, max_pos,
                                              L.current_stream()), "sgpt_linear_qkv_rotary_lnfold")
    plain = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device=dev)
    L.check(lib.sgpt_linear_lnfold(xb.data_ptr(), d, wf.data_ptr(), d, bf.data_ptr(), cs.data_ptr(), st.data_ptr(), P, eps,
                                   plain.data_ptr(), N, M, N, d, 0, L.current_stream()), "sgpt_linear_lnfold")
    torch.cuda.synchronize()
    assert torch.equal(wf.cpu(), (w.float() * gamma).to(torch.bfloat16))  # exact fold: gamma is a power of two
    got = out.cpu()
    assert bool(torch.isfinite(got).all())
    passthrough = torch.ones(N, dtype=torch.bool)
    passthrough[:2 * d].view(-1, hd)[:, :rd] = False
    assert torch.equal(got[:, passthrough].view(torch.int16), plain.cpu()[:, passthrough].view(torch.int16)), \
        "v columns / non-rotary dims differ from the lnfold projection"

    xx = xd.double()
    ln = (xx - xx.mean(1, keepdim=True)) / torch.sqrt(xx.var(1, unbiased=False, keepdim=True) + eps) * gd.double() + bd.double()
    want = rotary_reference(ln @ wd.double().T, pd, cos_sin, d, hd, rd).cpu()
    e = _lnfold_fp32_bound(xd, wf, wd, bd, eps)
    y_abs = (ln @ wd.double().T).abs()
    e_rot = rotary_abs_bound(e + 2.0 ** -22 * y_abs, pd, cos_sin, d, hd, rd).cpu()
    tol = BF16_U * want.abs() + (1 + BF16_U) * e_rot
    err = (got.double() - want).abs()
    if bool((err > tol).any()):
        m, n = (err > tol).nonzero()[0].tolist()
        raise AssertionError(f"{int((err > tol).sum())} elements out of tolerance; first qkv[{m},{n}] (head {n // hd}, dim "
                             f"{n % hd}, pos {int(pos[m])}) = {float(got[m, n])}, want {float(want[m, n])} "
                             f"(tol {float(tol[m, n])})")


def test_ln_fold_block_flow_matches_reference_fixture(golden_dir, monkeypatch):
    """The opt-in block flow without LayerNorm passes (SGPT_LN_FOLD=1, csrc/model.cu) against the same HF fixture as the
    default flow: pooled embeddings within 1e-3 cosine, all-layer pooling modes, and the two flows agree with each other."""
    import os

    import numpy as np

    from oracle import gpt_neo
    from sgpt_b200 import Encoder
    from tests.helpers import min_row_cosine
    from tests.test_gpu_parity import _cfg_from_spec, _spec_from

    z = np.load(os.path.join(golden_dir, "neo_tiny.npz"))
    spec = _spec_from(z)
    w = gpt_neo.init_weights(spec, seed=int(z["weight_seed"]))
    ids, mask = z["input_ids"], z["attention_mask"]
    outs = {}
    for fold in ("0", "1"):
        monkeypatch.setenv("SGPT_LN_FOLD", fold)
        enc = Encoder(_cfg_from_spec(spec), w, device="cuda:0", max_tokens=4096, max_batch=64)
        outs[fold] = {m: enc.encode_tokens(ids, mask, method=m).cpu() for m in ("weightedmean", "mean", "meanmean", "lasttoken")}
        outs[fold]["mid"] = enc.encode_tokens(ids, mask, method="weightedmean", layer_idx=int(z["mid_layer"])).cpu()
        outs[fold]["norm"] = enc.encode_tokens(ids, mask, method="weightedmean", normalize=True).cpu()
        enc.close()
    assert min_row_cosine(outs["1"]["weightedmean"], z["pooled_weightedmean"]) > 1 - 1e-3
    assert min_row_cosine(outs["1"]["mean"], z["pooled_mean"]) > 1 - 1e-3
    assert min_row_cosine(outs["1"]["mid"], z["pooled_weightedmean_mid"]) > 1 - 1e-3
    for k in outs["0"]:
        assert min_row_cosine(outs["1"][k], outs["0"][k]) > 1 - 2e-4, k
    assert torch.allclose(outs["1"]["norm"].norm(dim=1), torch.ones(len(ids)), atol=1e-5)


@pytest.mark.parametrize("resid_bf16", ["1", "0"])
def test_residual_stream_dtype_flows_match_reference_fixture(golden_dir, monkeypatch, resid_bf16):
    """The residual stream is stored in bf16 by default (what HF does for a bf16 checkpoint) and in fp32 with
    SGPT_RESID_BF16=0: both against the HF fp32 fixture — pooled embeddings within the 1e-3 cosine bar, per-token residual
    tap readable."""
    import os

    import numpy as np

    from oracle import gpt_neo
    from sgpt_b200 import Encoder
    from tests.helpers import min_row_cosine
    from tests.test_gpu_parity import _cfg_from_spec, _spec_from

    z = np.load(os.path.join(golden_dir, "neo_tiny.npz"))
    spec = _spec_from(z)
    w = gpt_neo.init_weights(spec, seed=int(z["weight_seed"]))
    ids, mask = z["input_ids"], z["attention_mask"]
    monkeypatch.setenv("SGPT_RESID_BF16", resid_bf16)
    enc = Encoder(_cfg_from_spec(spec), w, device="cuda:0", max_tokens=4096, max_batch=64)
    for method, key in (("weightedmean", "pooled_weightedmean"), ("mean", "pooled_mean")):
        got = enc.encode_tokens(ids, mask, method=method).cpu()
        assert min_row_cosine(got, z[key]) > 1 - 1e-3, method
    got = enc.encode_tokens(ids, mask, method="weightedmean", layer_idx=int(z["mid_layer"])).cpu()
    assert min_row_cosine(got, z["pooled_weightedmean_mid"]) > 1 - 1e-3
    sp = np.load(os.path.join(golden_dir, "script_pooling_neo_tiny.npz"))
    for method in ("meanmean", "lasttokenmean", "lasttoken"):
        assert min_row_cosine(enc.encode_tokens(ids, mask, method=method).cpu(), sp["pooled_" + method]) > 1 - 1e-3, method
    enc.encode_tokens(ids, mask)
    resid = enc.last_residual().cpu()
    h = gpt_neo.layer_norm(resid, w["ln_f.weight"], w["ln_f.bias"], spec.ln_eps)
    ref = torch.from_numpy(z["hidden_states"][-1])[torch.from_numpy(mask).bool()]
    assert torch.nn.functional.cosine_similarity(h.double(), ref.double(), dim=1).min().item() > 1 - 1e-3
    enc.close()
