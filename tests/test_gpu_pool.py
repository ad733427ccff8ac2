"""sgpt_pool (P1/P2) on both of its paths — ln_f fused into one pass for d <= 1024, row statistics then pooling for
d > 1024, and the plain pooling kernel without ln_f — against one fp64 restatement of the header's contract, for every
mode, with and without ln_f, clamp, normalize and accumulate; its bit-repeatability; and the all-hidden-state modes and
layer_idx of sgpt_encode against the fp64 pool of the exact hidden states the encoder produced."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # unit roundoff of fp32
MEAN, WMEAN, LAST = 0, 1, 2
TABLE = "table"  # WEIGHTEDMEAN with a learnt position-weight table


def _lib():
    from sgpt_b200 import _lib

    return _lib, _lib.lib()


class Batch:
    """A ragged batch on the device: lengths, cu_seqlens, pos (the index in a padded row: left-padded rows start late)."""

    def __init__(self, lens, seed, pad_max=20):
        g = torch.Generator().manual_seed(seed)
        self.lens = torch.as_tensor(lens, dtype=torch.int64)
        self.B = len(lens)
        cu = torch.zeros(self.B + 1, dtype=torch.int64)
        cu[1:] = torch.cumsum(self.lens, 0)
        self.T = int(cu[-1])
        start = torch.randint(0, pad_max + 1, (self.B,), generator=g) * (torch.arange(self.B) % 2)
        self.pos = torch.cat([torch.arange(int(s), int(s) + int(n)) for s, n in zip(start, self.lens)]).to(torch.int32)
        self.cu = cu.to(torch.int32)
        self.seg = torch.repeat_interleave(torch.arange(self.B), self.lens)
        self.pos_d, self.cu_d = self.pos.cuda(), self.cu.cuda()


def token_weights(batch, mode, pw):
    """Weight of every token: pos + 1, the learnt table at min(pos, n - 1), 1, or [token is its sequence's last]."""
    if mode == MEAN:
        return torch.ones(batch.T, dtype=torch.float64)
    if mode == LAST:
        w = torch.zeros(batch.T, dtype=torch.float64)
        w[batch.cu[1:].long()[batch.lens > 0] - 1] = 1.0
        return w
    if pw is not None:
        return pw.double()[batch.pos.long().clamp(max=len(pw) - 1)]
    return batch.pos.double() + 1.0


def pool_reference(x, batch, mode, pw, lnf, eps, clamp):
    """fp64 pool of one hidden state (x: fp64 [T, d] on the device, the values the kernel reads) and a per-element bound
    on the kernel's fp32 error.  Returns (pool [B, d], bound [B, d])."""
    dev = x.device
    w = token_weights(batch, mode, pw).to(dev)
    seg = batch.seg.to(dev)
    lens = batch.lens.to(dev).double()
    B, d = batch.B, x.shape[1]
    if lnf is not None:
        mu = x.mean(1, keepdim=True)
        rstd = 1.0 / torch.sqrt(((x - mu) ** 2).mean(1, keepdim=True) + eps)
        xh = (x - mu) * rstd
        # per row: fp32 mean / rstd within 2^-20 relative (the mean relative to the row's magnitude, amplified by rstd)
        stat_err = 2.0 ** -20 * (xh.abs() + rstd * x.abs().mean(1, keepdim=True))
    else:
        xh, stat_err = x, torch.zeros_like(x)
    # the sums over each sequence as one product with the [B, T] matrix of token weights (no atomics: exact to fp64
    # rounding and the same on every run)
    S = torch.zeros(B, batch.T, dtype=torch.float64, device=dev)
    S[seg, torch.arange(batch.T, device=dev)] = w
    A, absA, statA = S @ xh, S.abs() @ xh.abs(), S.abs() @ stat_err
    W, absW = S.sum(1), S.abs().sum(1)
    # fp32 sums over a sequence: at most len + 8 roundings of partial sums bounded by the absolute sums
    gam = (lens + 8.0)[:, None] * U
    A_err = gam * absA + statA
    W_err = gam[:, 0] * absW
    if lnf is not None:
        g, b = lnf[0].to(dev).double(), lnf[1].to(dev).double()
        num = g * A + b * W[:, None]
        num_err = g.abs() * A_err + b.abs() * W_err[:, None] + 3 * U * ((g * A).abs() + (b * W[:, None]).abs())
    else:
        num, num_err = A, A_err
    floor = float(np.float32(1e-9))  # the kernel's clamp is fmaxf(W, 1e-9f)
    den = W.clamp(min=floor) if clamp else W
    den_err = torch.where(W > floor, W_err, torch.zeros_like(W_err)) if clamp else W_err
    pool = num / den[:, None]
    bound = (num_err + pool.abs() * den_err[:, None]) / den.abs()[:, None] + U * pool.abs()
    return pool, bound


def finish_reference(pool, bound, prev, prev_bound, scale, normalize):
    """out = (prev or 0) + scale * pool, then the optional L2 normalisation of the row; with the bound carried along."""
    o = scale * pool
    ob = abs(scale) * bound + U * o.abs()
    if prev is not None:
        o = o + prev
        ob = ob + prev_bound + U * o.abs()
    if normalize:
        nrm = o.norm(dim=1, keepdim=True)
        d = o.shape[1]
        # ||o~|| differs from ||o|| by at most ||err||_2, plus the fp32 sum of squares over the row
        rel = ob.norm(dim=1, keepdim=True) / nrm + (d / 4 + 64) * U
        on = o / nrm.clamp(min=1e-12)
        ob = ob / nrm.clamp(min=1e-12) + on.abs() * rel + 4 * U * on.abs()  # sqrtf, the division, the scaling
        o = on
    return o, ob


def run_pool(batch, x, x_bf16, mode, pw, lnf, eps, clamp, normalize, accumulate, scale, out):
    L, lib = _lib()
    T, d = batch.T, x.shape[1]
    ws = torch.empty(2 * T + batch.B, device="cuda")
    g, b = (None, None) if lnf is None else (lnf[0], lnf[1])
    L.check(lib.sgpt_pool(x.data_ptr(), x_bf16, batch.pos_d.data_ptr(), batch.cu_d.data_ptr(), L.ptr(g), L.ptr(b), eps,
                          L.ptr(pw), 0 if pw is None else pw.numel(), out.data_ptr(), ws.data_ptr(), batch.B, T, d,
                          WMEAN if mode == TABLE else mode, int(clamp), int(normalize), int(accumulate), scale,
                          L.current_stream()), "sgpt_pool")
    return out


def assert_within(got, want, bound, what):
    err = (got.double() - want).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements out of bound, first at {i}: got {got[i[0], i[1]].item()} "
                             f"want {want[i[0], i[1]].item()} bound {bound[i[0], i[1]].item()}")


# lengths on the fused kernel's 8-warp / 16-row stride, one long sequence, and enough short ones for B > 132
LENS = [1, 7, 8, 9, 16, 17, 300, 2048] + [int(n) for n in torch.randint(1, 25, (140,),
                                                                        generator=torch.Generator().manual_seed(1))]


def hidden_states(T, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(T, d, generator=g, device="cuda") * 1.5 + 0.3
    x[:, min(5, d - 1)] += 12.0  # an outlier feature
    return x


def lnf_params(d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (1.0 + 0.3 * torch.randn(d, generator=g, device="cuda"), 0.05 * torch.randn(d, generator=g, device="cuda"))


def learnt_table(seed):
    """40 learnt weights, some negative; positions past the table read its last entry."""
    g = torch.Generator().manual_seed(seed)
    pw = torch.randn(40, generator=g) * 0.6 + 0.8
    pw[-1] = 1.25
    return pw.cuda()


# d on the fused path (4, 100, 1024) and the two-kernel path (1028 .. 4096), with partial column blocks
@pytest.mark.parametrize("d", [4, 100, 1024, 1028, 1100, 2048, 4096])
@pytest.mark.parametrize("with_lnf", [False, True])
@pytest.mark.parametrize("mode", [MEAN, WMEAN, TABLE, LAST])
def test_pool_fp64_bound(mode, with_lnf, d):
    batch = Batch(LENS, seed=d)
    x32 = hidden_states(batch.T, d, seed=d + 1)
    lnf = lnf_params(d, seed=d + 2) if with_lnf else None
    pw = learnt_table(d) if mode == TABLE else None
    eps = 1e-5
    g = torch.Generator(device="cuda").manual_seed(d + 3)
    prev = torch.randn(batch.B, d, generator=g, device="cuda")
    for x_bf16 in (0, 1):
        x = x32.to(torch.bfloat16) if x_bf16 else x32
        pool, bound = pool_reference(x.double(), batch, mode, pw, lnf, eps, clamp=False)
        pool_c, bound_c = pool_reference(x.double(), batch, mode, pw, lnf, eps, clamp=True)
        for clamp in (0, 1):
            p, pb = (pool_c, bound_c) if clamp else (pool, bound)
            for accumulate in (0, 1):
                for normalize in (0, 1):
                    scale = 0.375 if accumulate else 1.0
                    out = torch.full((batch.B + 1, d), 7.0, device="cuda")
                    out[:batch.B] = prev
                    run_pool(batch, x, x_bf16, mode, pw, lnf, eps, clamp, normalize, accumulate, scale, out)
                    want, wb = finish_reference(p, pb, prev.double() if accumulate else None, 0.0, scale, normalize)
                    assert_within(out[:batch.B], want, wb,
                                  f"x_bf16={x_bf16} clamp={clamp} accumulate={accumulate} normalize={normalize}")
                    assert bool((out[batch.B] == 7.0).all())  # nothing written past row B


@pytest.mark.parametrize("d", [128, 2048])
@pytest.mark.parametrize("with_lnf", [False, True])
def test_pool_zero_learnt_table(d, with_lnf):
    """A table of zeros: W = 0, so the clamped pool is exactly 0 and the unclamped one 0/0 = NaN, as in fp64."""
    batch = Batch([1, 9, 40, 300], seed=2)
    x = hidden_states(batch.T, d, seed=3).to(torch.bfloat16)
    lnf = lnf_params(d, seed=4) if with_lnf else None
    pw = torch.zeros(16, device="cuda")
    for clamp in (0, 1):
        for normalize in (0, 1):
            out = torch.full((batch.B, d), 7.0, device="cuda")
            run_pool(batch, x, 1, TABLE, pw, lnf, 1e-5, clamp, normalize, 0, 1.0, out)
            if clamp:
                assert bool((out == 0).all()), (clamp, normalize)
            else:
                assert bool(torch.isnan(out).all()), (clamp, normalize)


def _launch_all(batch, x, d, with_lnf, normalize):
    lnf = lnf_params(d, seed=9) if with_lnf else None
    out = torch.empty(batch.B, d, device="cuda")
    return run_pool(batch, x, 1, WMEAN, None, lnf, 1e-5, 1, normalize, 0, 1.0, out)


# every path: fused ln_f (1024), two-kernel ln_f (2048, 4096), no ln_f (1024, 4096); normalize on and off
@pytest.mark.parametrize("d,with_lnf", [(1024, True), (2048, True), (4096, True), (1024, False), (4096, False)])
@pytest.mark.parametrize("normalize", [0, 1])
def test_pool_bit_repeatable_and_batch_invariant(d, with_lnf, normalize):
    lens = [int(n) for n in torch.randint(1, 65, (256,), generator=torch.Generator().manual_seed(d))]
    batch = Batch(lens, seed=d, pad_max=0)
    x = hidden_states(batch.T, d, seed=d).to(torch.bfloat16)
    first = _launch_all(batch, x, d, with_lnf, normalize).clone()
    for _ in range(3):
        again = _launch_all(batch, x, d, with_lnf, normalize)
        diff = (again.view(torch.int32) != first.view(torch.int32))
        assert not bool(diff.any()), (f"{int(diff.sum())} elements differ between launches, in rows "
                                      f"{sorted(set(diff.nonzero()[:, 0].tolist()))[:10]}")
    # the same sequences in reverse order, packed the other way round: each sequence's row keeps its bits
    rev = Batch(lens[::-1], seed=d, pad_max=0)
    xr = torch.cat([x[int(batch.cu[b]):int(batch.cu[b + 1])] for b in reversed(range(batch.B))])
    got = _launch_all(rev, xr, d, with_lnf, normalize).flip(0)
    assert torch.equal(got.view(torch.int32), first.view(torch.int32))


# --------------------------------------------------------------------------------------------------------------------
# sgpt_encode: the all-hidden-state modes and layer_idx
# --------------------------------------------------------------------------------------------------------------------
def _encoder(n_layer, d, n_head):
    from oracle import gpt_neo
    from sgpt_b200 import Encoder, ModelConfig

    spec = gpt_neo.NeoSpec(n_layer=n_layer, d_model=d, n_head=n_head, d_ff=4 * d, vocab=500, max_pos=64, window=8)
    w = gpt_neo.init_weights(spec, seed=n_layer + d)
    cfg = ModelConfig(arch="gpt_neo", n_layer=n_layer, d_model=d, n_head=n_head, d_ff=4 * d, vocab=500, max_pos=64,
                      window=8)
    return Encoder(cfg, w, device="cuda:0", max_tokens=4096, max_batch=64), w, spec


# a small GPT-Neo on the fused ln_f path (d = 128), and a depth-1 model on the two-kernel path with d/4 = 272, not a
# multiple of 32
@pytest.mark.parametrize("n_layer,d,n_head", [(2, 128, 2), (1, 1088, 17)])
def test_encode_all_layer_modes_and_layer_idx(n_layer, d, n_head):
    from sgpt_b200.encoder import pack_ragged

    enc, w, spec = _encoder(n_layer, d, n_head)
    g = torch.Generator().manual_seed(d)
    lens = torch.tensor([1, 5, 8, 17, 40, 64, 9, 33])
    S = int(lens.max())
    ids = torch.randint(0, spec.vocab, (len(lens), S), generator=g)
    mask = (torch.arange(S)[None] < lens[:, None]).long()
    _, pos, cu, _ = pack_ragged(ids.numpy(), mask.numpy())
    batch = Batch(lens.tolist(), seed=0)
    batch.pos = torch.from_numpy(pos)  # right-padded rows: the same positions as the encoder's
    lnf = (w["ln_f.weight"].cuda().float(), w["ln_f.bias"].cuda().float())
    eps = spec.ln_eps
    L = n_layer
    hs = []
    for l in range(L + 1):  # hidden state l, bit-identical to the one any other run of this batch produces
        enc.encode_tokens(ids, mask, method="mean", layer_idx=l)
        hs.append(enc.last_residual().double().clone())
    for clamp in (False, True):
        for normalize in (False, True):
            for method, base in (("meanmean", MEAN), ("lasttokenmean", LAST)):
                got = enc.encode_tokens(ids, mask, method=method, clamp=clamp, normalize=normalize)
                o, ob = None, 0.0
                for l in range(L + 1):  # ln_f on hidden state L only; each state scaled by 1/(L+1) and accumulated
                    p, pb = pool_reference(hs[l], batch, base, None, lnf if l == L else None, eps, clamp)
                    pb = pb + U * p.abs()  # the scale is 1/(L+1) rounded to fp32
                    o, ob = finish_reference(p, pb, o, ob, 1.0 / (L + 1), normalize and l == L)
                assert_within(got, o, ob, f"{method} clamp={clamp} normalize={normalize}")
            for l in list(range(L + 1)) + [-1]:
                for method, mode in (("weightedmean", WMEAN), ("lasttoken", LAST)):
                    got = enc.encode_tokens(ids, mask, method=method, layer_idx=l, clamp=clamp, normalize=normalize)
                    ll = L if l == -1 else l
                    p, pb = pool_reference(hs[ll], batch, mode, None, lnf if ll == L else None, eps, clamp)
                    want, wb = finish_reference(p, pb, None, 0.0, 1.0, normalize)
                    assert_within(got, want, wb, f"{method} layer_idx={l} clamp={clamp} normalize={normalize}")
    enc.close()
