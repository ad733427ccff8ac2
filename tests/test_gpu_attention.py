"""sgpt_attention (include/sgpt_b200.h F4) against a plain fp64 reference of the same operation, through the C ABI.

Both kernels are checked against fp64 on their own, not only against each other: impl 0 (tensor cores, mma.sync,
FlashAttention-2 style online softmax) and impl 1 (SIMT).  The reference (`_reference`) states the header's semantics
directly: per sequence, key j is visible to query i iff i - w < j <= i (j <= i for w = 0); logits are scale * q.k plus
slope_h * j when ALiBi slopes are given; softmax over the visible keys; times V.  It runs in torch fp64 on the device,
from the same bf16 q / k / v the kernel reads.

Three kinds of inputs:
  - random q / k / v with realistic logit spreads (`_tolerance` derives the bound);
  - uniform probes: q = 0, so every visible key has weight exactly 1 and the output is the mean of the visible V rows;
    V[key, c] = 1 iff position(key) mod hd == c, so one key too many or too few moves a column by 1 / count;
  - peaked probes: one key per query whose logit exceeds every other by >= 30, so the output is that key's V row.
Every launch also checks the write set (rows past T keep their bits, every valid element is finite) and that a second
launch gives the same bits.
"""
import math

import pytest
import torch

from tests.helpers import BF16_U as U

pytestmark = pytest.mark.gpu

# ragged batch: lengths around the 32 / 64-key tiles and the 64-query tiles, an empty sequence, and a long one
LENS = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 0, 129, 255, 256, 257, 300, 1500]
GUARD_ROWS = 3


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


def _cu(lens):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return cu


def _positions(lens):
    """Index of every packed token inside its own sequence (device int64[T])."""
    return torch.cat([torch.arange(n, dtype=torch.int64) for n in lens]).cuda()


def _run(qkv, lens, H, hd, scale, window, slopes=None, impl=0, max_seqlen=None):
    """One sgpt_attention call into an output with GUARD_ROWS extra rows, everything prefilled with NaN.  Checks the write
    set and that a second launch reproduces the bits; returns out[:T]."""
    L, lib = _lib()
    T = sum(lens)
    cu = torch.tensor(_cu(lens), dtype=torch.int32, device="cuda")
    if max_seqlen is None:
        max_seqlen = max(lens) + 70  # one query tile past the longest sequence: those CTAs must exit without writing
    outs = []
    for _ in range(2):
        out = torch.full((T + GUARD_ROWS, H * hd), float("nan"), dtype=torch.bfloat16, device="cuda")
        L.check(lib.sgpt_attention(qkv.data_ptr(), out.data_ptr(), cu.data_ptr(), len(lens), T, H, hd, scale, window,
                                   max_seqlen, L.ptr(slopes), impl, L.current_stream()), "sgpt_attention")
        torch.cuda.synchronize()
        outs.append(out)
    nan_bits = torch.full((GUARD_ROWS, H * hd), float("nan"), dtype=torch.bfloat16).view(torch.int16)
    assert torch.equal(outs[0][T:].cpu().view(torch.int16), nan_bits), "rows past T were written"
    bad = (~torch.isfinite(outs[0][:T])).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} valid elements not written or not finite, first (token, col) {bad[0].tolist()}"
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), "two launches differ"
    return outs[0][:T]


def _reference(qkv, lens, H, hd, scale, window, slopes=None):
    """fp64 attention over the ragged batch -> (ref, pv): ref = softmax(logits) V and pv = softmax(logits) |V|, both
    [T, H*hd]."""
    T = sum(lens)
    x = qkv.double().view(T, 3, H, hd)
    ref = torch.zeros(T, H, hd, dtype=torch.float64, device=qkv.device)
    pv = torch.zeros_like(ref)
    s0 = 0
    for n in lens:
        if n == 0:
            continue
        i = torch.arange(n, device=qkv.device).unsqueeze(1)
        j = torch.arange(n, device=qkv.device).unsqueeze(0)
        visible = (j <= i) & ((j > i - window) if window > 0 else True)
        for h0 in range(0, H, 8):  # bounds the [heads, n, n] logits at n = 2048
            h1 = min(H, h0 + 8)
            q, k, v = (x[s0:s0 + n, c, h0:h1].transpose(0, 1) for c in range(3))
            logits = scale * (q @ k.transpose(1, 2))
            if slopes is not None:
                logits = logits + slopes[h0:h1].double().view(-1, 1, 1) * j.double()
            p = torch.softmax(logits.masked_fill(~visible, float("-inf")), dim=-1)
            ref[s0:s0 + n, h0:h1] = (p @ v).transpose(0, 1)
            pv[s0:s0 + n, h0:h1] = (p @ v.abs()).transpose(0, 1)
        s0 += n
    return ref.view(T, H * hd), pv.view(T, H * hd)


def _tolerance(ref, pv):
    """Per-element bound for random inputs.  The tensor-core kernel rounds the unnormalised weights P to bf16 before the PV
    product and rounds the output to bf16; the rest is fp32 (the SIMT kernel does not round P, so the bound covers it).
    Each bf16 rounding has relative error <= u = 2^-8.  With ref = sum_j p_j v_j / sum_j p_j:
      - rounding P moves the output by <= u * sum_j p_j |v_j| / sum_j p_j = u * pv;
      - rounding the output adds <= u * |ref| (times 1 + the error above);
      - fp32 logits (q.k as hd/16 + 16 accumulations on the tensor cores, the scale, the ALiBi fma at |logit| < 4096 in the
        exp2 domain, the max subtraction) and exp2 err by an absolute delta <= 2^-11 in the exponent at the logit spreads
        used here; each weight changes by a factor 1 + delta, the output by <= delta * (|ref| + pv).
    |got - ref| <= u |ref| + (u + u^2 + delta) pv + delta |ref| <= (2^-8 + 2^-10) (|ref| + pv)."""
    return (U + 2.0 ** -10) * (ref.abs() + pv)


def _assert_close(got, ref, tol, hd, what):
    err = (got.double() - ref).abs()
    bad = err > tol
    if bool(bad.any()):
        t, c = (bad.nonzero()[0]).tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements out of tolerance; first at token {t} head {c // hd} "
                             f"dim {c % hd}: got {float(got[t, c])} want {float(ref[t, c])} (tol {float(tol[t, c])}); "
                             f"worst excess {float((err - tol).max())}")


def _random_qkv(lens, H, hd, scale, logit_std, seed):
    """q, k ~ N(0, s^2) with scale * s^2 * sqrt(hd) = logit_std (the spread of scale * q.k), v ~ N(0, 1); bf16."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    T = sum(lens)
    x = torch.randn(T, 3, H, hd, generator=g, device="cuda")
    s = math.sqrt(logit_std / (scale * math.sqrt(hd)))
    x[:, :2] *= s
    return x.to(torch.bfloat16).view(T, 3 * H * hd)


def _check_random(lens, H, hd, scale, logit_std, window, impl, seed, slopes=None, max_seqlen=None):
    qkv = _random_qkv(lens, H, hd, scale, logit_std, seed)
    got = _run(qkv, lens, H, hd, scale, window, slopes, impl, max_seqlen)
    ref, pv = _reference(qkv, lens, H, hd, scale, window, slopes)
    _assert_close(got, ref, _tolerance(ref, pv), hd, f"hd={hd} window={window} impl={impl}")
    return qkv, got


# GPT-J / BLOOM style 1/sqrt(hd) with a logit spread of ~2.5 (tests/helpers.py full_size_weights), and GPT-Neo's unscaled
# q.k (scale 1.0) with larger logits
SCALINGS = {"scaled": (None, 2.5), "unscaled": (1.0, 8.0)}


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("window", [0, 1, 17, 64, 256])
@pytest.mark.parametrize("hd", [64, 128, 256])
@pytest.mark.parametrize("scaling", sorted(SCALINGS))
def test_attention_random_vs_fp64(scaling, hd, window, impl):
    scale, logit_std = SCALINGS[scaling]
    scale = scale or 1.0 / math.sqrt(hd)
    _check_random(LENS, 3, hd, scale, logit_std, window, impl, seed=hd * 1000 + window)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("hd", [64, 128, 256])
def test_attention_window_covering_the_sequence_is_causal(hd, impl):
    """A window at least as long as every sequence hides no key: the result is plain causal attention, bit for bit."""
    scale = 1.0 / math.sqrt(hd)
    qkv, causal = _check_random(LENS, 2, hd, scale, 2.5, 0, impl, seed=hd + 7)
    wide = _run(qkv, LENS, 2, hd, scale, max(LENS), impl=impl)
    assert torch.equal(wide.view(torch.int16), causal.view(torch.int16))
    wider = _run(qkv, LENS, 2, hd, scale, 4096, impl=impl)
    assert torch.equal(wider.view(torch.int16), causal.view(torch.int16))


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("window", [0, 1, 17, 64, 256])
@pytest.mark.parametrize("hd", [64, 128, 256])
def test_attention_uniform_probe_counts_visible_keys(hd, window, impl):
    """q = 0 and no ALiBi: every visible key has logit 0 and weight exactly 1 (exp2(0)), so out[i, c] is the number of
    visible keys j with j mod hd == c over the number of visible keys.  The counts and the weights are exact in fp32; the
    normalisation is two fp32 roundings (2^-23) and the output one bf16 rounding (2^-8):
    |got - ref| <= (2^-8 + 2^-20) |ref|, and a zero column must be exactly zero.  A missing or extra key changes the
    column of its residue class by about 1 / (keys in that class) of its value: at least 4 % here (at most 24 keys per
    class), ten times the bound."""
    H = 2
    T = sum(LENS)
    pos = _positions(LENS)
    qkv = torch.zeros(T, 3, H, hd, dtype=torch.bfloat16, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(hd + window)
    qkv[:, 1] = torch.randn(T, H, hd, generator=g, device="cuda").to(torch.bfloat16)  # keys play no role when q = 0
    qkv[:, 2] = torch.nn.functional.one_hot(pos % hd, hd).to(torch.bfloat16).unsqueeze(1)
    got = _run(qkv.view(T, -1), LENS, H, hd, 0.125, window, impl=impl)
    ref, _ = _reference(qkv.view(T, -1), LENS, H, hd, 0.125, window)
    _assert_close(got, ref, (U + 2.0 ** -20) * ref.abs(), hd, f"uniform probe hd={hd} window={window} impl={impl}")


def _peak_codes(p):
    """Three base-16 digits of a position (< 4096) as a 48-dim 0/1 code: two positions share all three digits only if
    equal, so code(i) . code(j) is 3 for i == j and at most 2 otherwise."""
    dig = torch.stack([p % 16, p // 16 % 16, p // 256 % 16], dim=1) + torch.tensor([0, 16, 32], device=p.device)
    return torch.zeros(p.shape[0], 48, device=p.device).scatter_(1, dig, 1.0)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("window", [0, 17, 256])
@pytest.mark.parametrize("where", ["edge", "diagonal", "earlier"])
@pytest.mark.parametrize("hd", [64, 128, 256])
def test_attention_peaked_probe_selects_one_key(hd, where, window, impl):
    """Query i carries A * code(kappa_i) and key j carries code(j) (`_peak_codes`), so scale * q.k is 3 scale A for key
    kappa_i and at most 2 scale A for every other key, with scale A >= 30.  kappa_i is the first visible key (the window
    edge: the running max arrives first), the diagonal (the last key tile: it arrives last) or 70 keys back (an earlier
    key tile followed by tiles of smaller logits).  The peak has weight exactly 1 and the at most 2047 others together
    < 2047 * e^-30 < 2^-32 of it, far below half a bf16 ulp (2^-8) of the result: out[i] must equal V[kappa_i] bit for
    bit."""
    H = 2
    scale = 1.0 / math.sqrt(hd)
    T = sum(LENS)
    pos = _positions(LENS)
    lo = (pos - window + 1).clamp(min=0) if window > 0 else torch.zeros_like(pos)
    kappa = {"edge": lo, "diagonal": pos, "earlier": torch.maximum(lo, pos - 70)}[where]
    amp = float(torch.tensor(32.0 / scale).to(torch.bfloat16))
    g = torch.Generator(device="cuda").manual_seed(hd * 3 + window)
    qkv = torch.zeros(T, 3, H, hd, device="cuda")
    qkv[:, 0, :, :48] = (amp * _peak_codes(kappa)).unsqueeze(1)
    qkv[:, 1, :, :48] = _peak_codes(pos).unsqueeze(1)
    qkv[:, 2] = torch.randn(T, H, hd, generator=g, device="cuda")
    qkv = qkv.to(torch.bfloat16)
    got = _run(qkv.view(T, -1), LENS, H, hd, scale, window, impl=impl)
    seq0 = pos.new_tensor(_cu(LENS)[:-1]).repeat_interleave(torch.tensor(LENS, device="cuda"))
    want = qkv[seq0 + kappa, 2].reshape(T, H * hd)
    mismatch = (got != want).any(dim=1).nonzero()
    assert mismatch.numel() == 0, (f"{mismatch.shape[0]} query rows differ from V[kappa]; first token {int(mismatch[0])} "
                                   f"(position {int(pos[mismatch[0]])}, kappa {int(kappa[mismatch[0]])})")


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("H,hd", [(8, 64), (12, 128), (32, 64)])
def test_attention_alibi_vs_fp64(H, hd, impl):
    """BLOOM ALiBi with the HF slopes (oracle/bloom.py alibi_slopes; 12 heads is not a power of two) on sequences up to
    2048 tokens, where slope * key position reaches ~1700 in the logits: checks the fp32 fma of the bias and the max
    subtraction at that magnitude (the tolerance of `_tolerance` allows for it)."""
    from oracle.bloom import alibi_slopes

    slopes = alibi_slopes(H).float().cuda()
    lens = [1, 33, 129, 700, 2048]
    _check_random(lens, H, hd, 1.0 / math.sqrt(hd), 2.5, 0, impl, seed=H * hd, slopes=slopes)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("window", [0, 256])
def test_attention_bench_shape_vs_fp64(window, impl):
    """The benchmark's shape: 256 sequences of 128 tokens, 12 heads of 64, GPT-Neo's unscaled logits, max_seqlen exactly
    the sequence length.  Every row and head is compared: the fp64 reference runs on the device, so the whole grid costs
    well under a second."""
    _check_random([128] * 256, 12, 64, 1.0, 8.0, window, impl, seed=256 + window, max_seqlen=128)
