"""sgpt_lm_logprobs, the LM head of the cross-encoder scorer, at the LM-head shapes real SGPT-CE models use: GPT-Neo
d 768 / 2560 with the tied vocab-50257 head (its last 128-column tile holds 81 columns), GPT-J d 4096 with an untied
vocab-50400 head and its fp32 bias, BLOOM d 4096 with the tied vocab-250880 head.  Each model has one block, weights drawn
on the device like tests/helpers.full_size_weights, and runs one ragged batch through sgpt_forward.

The reference is layered so that its bound stays tight:
* the LM-head input: the residual stream read back exactly (sgpt_model_read_residual), then sgpt_layernorm_gather on the
  selected rows.  That is the kernel sgpt_lm_logprobs runs, and its row result depends on d only; its accuracy against
  fp64 is held in tests/test_gpu_rows.py;
* the logits: fp64 products of those bf16 rows with the bf16 head, each within tensor_core_sum_bound of |x| @ |W|^T, plus
  one fp32 rounding for the bias add;
* the log-prob: log-sum-exp is 1-Lipschitz in the max norm, so |error| <= eps(target) + max_v eps(v) + the log-softmax
  kernel's own rounding (the term of test_gpu_rows.py::test_token_logprobs_fp64).  Greedy must lie within 2 max_v eps(v)
  of the fp64 maximum, and be the fp64 argmax whenever that is alone in the window.
Every row's log-prob and greedy token must be bit-identical for every rows_per_chunk and every M, since a row's result
does not depend on its chunk or its position."""
import numpy as np
import pytest
import torch

from tests.helpers import full_size_weights, tensor_core_sum_bound

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # unit roundoff of fp32
BF16 = torch.bfloat16
TILE = 128  # columns per tile of the LM-head GEMM (gemm.cu launch_lm_logits)
SLICE = 8192  # head rows per fp64 reference slice: the fp64 head never exists whole (a BLOOM head is 2 GB in bf16)
B, S_FULL, M_FULL = 24, 2048, 300
POISON_IDS = (11, 12)  # the tokens of the two length-1 sequences POISON_SEQS; test_nan_inf_rows makes them NaN / +inf
POISON_SEQS = (5, 17)
SENTINEL = -7.0
GUARD = 4096  # bytes past the workspace size a call is given, which it must leave alone

# preset, seed, untied head with a bias (GPT-J's lm_head)
GEOMETRIES = {
    "neo768": ("sgpt-125m", 31, False),
    "neo2560": ("sgpt-2.7b", 32, False),
    "gptj4096": ("sgpt-5.8b", 33, True),
    "bloom4096": ("sgpt-bloom-7b1", 34, False),
}


def bits(t):
    return t.contiguous().view(torch.int32)


class LMHead:
    """One-block model of a geometry, its batch, M_FULL selected rows with targets, and the fp64 logits of those rows."""

    def __init__(self, name):
        from sgpt_b200 import Encoder, _lib, preset

        self.L, self.lib = _lib, _lib.lib()
        pname, seed, untied = GEOMETRIES[name]
        cfg = preset(pname, n_layer=1)
        self.name, self.cfg, self.d, self.V = name, cfg, cfg.d_model, cfg.vocab
        self.w, _ = full_size_weights(cfg.arch, cfg, seed=seed, host_copy=False)
        self.wte = self.w["word_embeddings.weight" if cfg.arch == "bloom" else "wte.weight"]
        g = torch.Generator(device="cuda").manual_seed(seed + 1000)
        if untied:
            self.W = (torch.randn(self.V, self.d, generator=g, device="cuda") * 0.02).to(BF16)
            self.bias = torch.randn(self.V, generator=g, device="cuda")
        else:
            self.W, self.bias = self.wte, None
        self.Wc = self.W.clone()  # the head of the planted-tie and NaN tests; equal to W outside them

        rs = np.random.RandomState(seed)
        lens = rs.randint(2, 161, B)
        lens[0], lens[1] = 1, S_FULL
        lens[list(POISON_SEQS)] = 1
        cu = np.zeros(B + 1, dtype=np.int32)
        np.cumsum(lens, out=cu[1:])
        T = int(cu[-1])
        ids = rs.randint(0, self.V, T).astype(np.int32)
        ids[np.isin(ids, POISON_IDS)] = 13
        for s, tok in zip(POISON_SEQS, POISON_IDS):
            ids[cu[s]] = tok
        pos = np.concatenate([np.arange(n, dtype=np.int32) for n in lens])
        self.T, self.cu = T, cu
        self.ids, self.pos, self.cu_d = (torch.from_numpy(a).cuda() for a in (ids, pos, cu))
        self.enc = Encoder(cfg, self.w, device="cuda:0", max_tokens=T, max_batch=B)
        assert any(t.data_ptr() == self.wte.data_ptr() for t in self.enc._keep)  # the handle reads this wte

        # rows: the length-1 sequence, the last token of the batch and of the full-length sequence first (the M = 1 and
        # planted-tie cases use them), then unordered rows with repeats, the poisoned sequences' rows among them
        self.poison_rows = [int(cu[s]) for s in POISON_SEQS]
        rows = rs.randint(0, T, M_FULL)
        rows[:3] = [0, T - 1, cu[2] - 1]
        extra = [int(cu[1]), 0, T - 1, cu[2] - 1] + self.poison_rows
        rows[3 + rs.choice(M_FULL - 3, len(extra), replace=False)] = extra
        self.rows = torch.from_numpy(rows.astype(np.int32)).cuda()

        self.forward()
        self.resid = self.enc.last_residual().clone()
        self.xsel = torch.empty(M_FULL, self.d, dtype=BF16, device="cuda")
        gamma, beta = self.w["ln_f.weight"], self.w["ln_f.bias"]
        self.L.check(self.lib.sgpt_layernorm_gather(self.resid.to(BF16).data_ptr(), self.rows.data_ptr(),
                                                    gamma.data_ptr(), beta.data_ptr(), self.xsel.data_ptr(), M_FULL,
                                                    self.d, cfg.ln_eps, self.L.current_stream()),
                     "sgpt_layernorm_gather")
        self.reference()

        # targets: 0, vocab - 1, columns of the last (partial) tile, the greedy column, the rest random
        t = rs.randint(0, self.V, M_FULL)
        last_tile = (self.V - 1) // TILE * TILE
        t[1], t[2], t[3] = 0, self.V - 1, last_tile
        t[4:9] = rs.randint(last_tile, self.V, 5)
        t[9:14] = self.z0[9:14].argmax(1).cpu().numpy()
        if self.bias is not None:
            t[14:19] = (self.z0[14:19] + self.bias.double()).argmax(1).cpu().numpy()
        self.targets = torch.from_numpy(t.astype(np.int32)).cuda()
        self.ws = torch.empty(self.ws_bytes(1024) + GUARD, dtype=torch.uint8, device="cuda")
        self._base = {}

    def reference(self):
        """fp64 logits z0 = xsel @ W^T and, per bias variant, the largest logit error bound of each row."""
        x = self.xsel.double()
        ax = x.abs()
        self.z0 = torch.empty(M_FULL, self.V, dtype=torch.float64, device="cuda")
        self.max_eps = {False: torch.zeros(M_FULL, dtype=torch.float64, device="cuda")}
        if self.bias is not None:
            self.max_eps[True] = torch.zeros_like(self.max_eps[False])
        for s in range(0, self.V, SLICE):
            Ws = self.W[s:s + SLICE].double()
            z = x @ Ws.t()
            e = tensor_core_sum_bound(ax @ Ws.abs().t(), self.d)
            del Ws
            self.z0[:, s:s + SLICE] = z
            self.max_eps[False] = torch.maximum(self.max_eps[False], e.max(1).values)
            if self.bias is not None:
                e = e + U * (z.abs() + self.bias[s:s + SLICE].double().abs() + e)
                self.max_eps[True] = torch.maximum(self.max_eps[True], e.max(1).values)

    def eps_at(self, k, cols, bias, head=None):
        """Logit error bound of rows k (indices into the selected rows) at the columns cols of head (default W)."""
        W = self.W if head is None else head
        x = self.xsel[k].double()
        wt = W[cols].double()
        z = (x * wt).sum(1)
        e = tensor_core_sum_bound((x.abs() * wt.abs()).sum(1), self.d)
        if bias is not None:
            e = e + U * (z.abs() + bias[cols].double().abs() + e)
        return e

    def ws_bytes(self, rpc):
        return self.lib.sgpt_lm_logprobs_workspace_bytes(self.d, self.V, rpc)

    def forward(self):
        self.L.check(self.lib.sgpt_forward(self.enc._handle, self.ids.data_ptr(), self.pos.data_ptr(),
                                           self.cu_d.data_ptr(), B, self.T, S_FULL, self.L.current_stream()),
                     "sgpt_forward")

    def run(self, rows, targets, rpc, head=None, bias=None, greedy=True, handle=None):
        """sgpt_lm_logprobs with a workspace of exactly the size rpc needs; checks that the sentinel past M and the bytes
        past the workspace keep their values.  Returns (log-probs [M], greedy [M] or None) on the device."""
        M = rows.numel()
        need = self.ws_bytes(rpc)
        self.ws[need:need + GUARD].fill_(0xA5)
        lp = torch.full((M + 1,), SENTINEL, device="cuda")
        gr = torch.full((M + 1,), -7, dtype=torch.int32, device="cuda")
        W = self.W if head is None else head
        self.L.check(self.lib.sgpt_lm_logprobs(handle or self.enc._handle, W.data_ptr(), self.L.ptr(bias), self.V,
                                               rows.data_ptr(), targets.data_ptr(), M, lp.data_ptr(),
                                               gr.data_ptr() if greedy else None, self.ws.data_ptr(), need, rpc,
                                               self.L.current_stream()), "sgpt_lm_logprobs")
        assert float(lp[M]) == SENTINEL and int(gr[M]) == -7, "written past M"
        assert bool((self.ws[need:need + GUARD] == 0xA5).all()), "written past the workspace"
        if not greedy:
            assert bool((gr == -7).all())
        return lp[:M], (gr[:M] if greedy else None)

    def base(self, with_bias):
        """The M_FULL rows in one chunk, with the model as built (cached)."""
        if with_bias not in self._base:
            self._base[with_bias] = self.run(self.rows, self.targets, M_FULL, bias=self.bias if with_bias else None)
        return self._base[with_bias]

    def close(self):
        self.enc.close()


def logprob_bound(z, t, eps_t, max_eps, V):
    """fp64 log-prob of the targets t under logits z [n, V], and the bound of a kernel whose logits are each within eps of
    z (eps_t at the target, max_eps the largest of the row)."""
    mx = z.max(1).values
    lse = torch.logsumexp(z, 1)
    zt = z.gather(1, t.long()[:, None])[:, 0]
    want = zt - lse
    # sgpt_token_logprobs' own rounding (test_gpu_rows.py::test_token_logprobs_fp64), on the kernel's logits: each value
    # it scales may be off by eps_t + max_eps from the fp64 one
    slack = eps_t + max_eps
    rnd = (U * ((zt - mx).abs() + want.abs() + 2 * slack) + 2 * U * (lse - mx + max_eps)
           + ((V + 255) // 256 + 20) * 2 * U)
    return want, eps_t + max_eps + rnd


def check_rows(lm, z, t, eps_t, max_eps, lp, gr, what):
    """The log-prob bound and the greedy window of every row; returns the worst error / bound ratio."""
    want, tol = logprob_bound(z, t, eps_t, max_eps, lm.V)
    err = (lp.double() - want).abs()
    bad = ~(err <= tol)
    assert not bool(bad.any()), (f"{lm.name} {what}: {int(bad.sum())} rows out of bound, first row "
                                 f"{int(bad.nonzero()[0])}: got {lp[bad][0].item()} want {want[bad][0].item()} "
                                 f"bound {tol[bad][0].item()}")
    g = gr.long()
    assert bool(((g >= 0) & (g < lm.V)).all())
    mx = z.max(1).values
    window = mx - 2 * max_eps
    assert bool((z.gather(1, g[:, None])[:, 0] >= window).all()), f"{lm.name} {what}: greedy outside the window"
    alone = (z >= window[:, None]).sum(1) == 1
    assert torch.equal(g[alone], z.argmax(1)[alone]), f"{lm.name} {what}: greedy is not the fp64 argmax"
    return float((err / tol).max()), int(alone.sum())


@pytest.fixture(scope="module", params=list(GEOMETRIES))
def lm(request):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m = LMHead(request.param)
    yield m
    print(f"[lm head] {m.name}: peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    m.close()


@pytest.fixture(scope="module")
def neo():
    m = LMHead("neo768")
    yield m
    m.close()


def _bias_variants(lm):
    return (False, True) if lm.bias is not None else (False,)


def test_fp64_bound_and_chunk_invariance(lm):
    lm.forward()
    for with_bias in _bias_variants(lm):
        bias = lm.bias if with_bias else None
        lp, gr = lm.base(with_bias)
        z = lm.z0 + bias.double() if with_bias else lm.z0
        eps_t = lm.eps_at(torch.arange(M_FULL, device="cuda"), lm.targets.long(), bias)
        ratio, alone = check_rows(lm, z, lm.targets, eps_t, lm.max_eps[with_bias], lp, gr, f"bias={with_bias}")
        print(f"[lm head] {lm.name} bias={with_bias}: worst log-prob err/bound {ratio:.3g}, greedy alone in its window "
              f"on {alone}/{M_FULL} rows")
        # the same rows through every chunking, as prefixes of the row list, with and without the greedy output
        for M in (0, 1, 129, M_FULL):
            for rpc in sorted({1, 7, M - 1, M, M + 1, 1024} - {-1, 0}):
                for greedy in ((True, False) if rpc in (7, M) else (True,)):
                    lpc, grc = lm.run(lm.rows[:M], lm.targets[:M], rpc, bias=bias, greedy=greedy)
                    what = f"bias={with_bias} M={M} rows_per_chunk={rpc}"
                    assert torch.equal(bits(lpc), bits(lp[:M])), what
                    if greedy:
                        assert torch.equal(grc, gr[:M]), what


def test_planted_exact_ties(lm):
    """Head rows j1 < j2 both set to bf16(alpha x_k) for the selected row x_k: its logits tie exactly at the maximum, and
    greedy must be j1 wherever the row sits in the batch and its chunk."""
    lm.forward()
    V = lm.V
    last_tile = (V - 1) // TILE * TILE
    pairs = [(TILE - 1, TILE), (0, V - 1), (last_tile + 3, V - 2)]
    for with_bias in _bias_variants(lm):
        for k, (j1, j2) in enumerate(pairs):  # selected rows 0, 1, 2: the length-1 sequence, token T-1, the full one
            x = lm.xsel[k].double()
            z = lm.z0[k].clone()
            bias = None
            if with_bias:
                bias = lm.bias.clone()
                bias[j2] = bias[j1]
                z += bias.double()
            alpha = float((2 * z.abs().max() + 10) / (x @ x))
            p = (alpha * x).to(BF16)
            lm.Wc[j1], lm.Wc[j2] = p, p
            try:
                planted = float(x @ p.double()) + (float(bias[j1]) if with_bias else 0.0)
                z[j1] = z[j2] = planted
                eps_p = lm.eps_at(torch.tensor([k, k], device="cuda"), torch.tensor([j1, j2], device="cuda"), bias,
                                  head=lm.Wc)
                max_eps = torch.maximum(lm.max_eps[with_bias][k], eps_p.max())
                others = torch.ones(V, dtype=torch.bool, device="cuda")
                others[[j1, j2]] = False
                assert planted - 2 * float(max_eps) > float(z[others].max()), "the planted pair is not the maximum"
                # row k first and last of 22 rows, in different chunks of 7
                sel = torch.cat([torch.tensor([k], device="cuda"), torch.arange(3, 23, device="cuda"),
                                 torch.tensor([k], device="cuda")])
                rows, tg = lm.rows[sel], lm.targets[sel].clone()
                tg[0], tg[-1] = j1, j2
                for rpc in (1, 7, 22):
                    lp, gr = lm.run(rows, tg, rpc, head=lm.Wc, bias=bias)
                    what = f"bias={with_bias} pair {(j1, j2)} rows_per_chunk={rpc}"
                    assert int(gr[0]) == j1 and int(gr[-1]) == j1, (what, int(gr[0]), int(gr[-1]))
                    ends = bits(lp[[0, -1]])
                    assert int(ends[0]) == int(ends[1]), (what, float(lp[0]), float(lp[-1]))  # equal logits
                    tt = torch.tensor([j1, j2], dtype=torch.int32, device="cuda")
                    check_rows(lm, z[None].expand(2, V), tt, eps_p, max_eps.expand(2), lp[[0, -1]], gr[[0, -1]], what)
            finally:
                lm.Wc[j1], lm.Wc[j2] = lm.W[j1], lm.W[j2]
    assert torch.equal(lm.Wc.view(torch.int16), lm.W.view(torch.int16))


def test_nan_inf_rows(lm):
    """Two length-1 sequences whose token embeddings hold NaN and +inf: their rows give a NaN log-prob and greedy 0,
    like sgpt_token_logprobs on a row of NaN; every other row keeps its bits."""
    lm.forward()
    want = {b: lm.base(b) for b in _bias_variants(lm)}
    saved = lm.wte[list(POISON_IDS)].clone()
    try:
        lm.wte[POISON_IDS[0]] = float("nan")
        lm.wte[POISON_IDS[1]] = float("inf")
        lm.forward()
        res = lm.enc.last_residual()
        clean = torch.ones(lm.T, dtype=torch.bool, device="cuda")
        clean[lm.poison_rows] = False
        assert not bool(torch.isfinite(res[lm.poison_rows]).any())
        assert torch.equal(bits(res[clean]), bits(lm.resid[clean]))  # the other sequences never see the poisoned rows
        poisoned = torch.isin(lm.rows, torch.tensor(lm.poison_rows, dtype=torch.int32, device="cuda"))
        assert int(poisoned.sum()) >= 2
        for with_bias in _bias_variants(lm):
            lp, gr = lm.run(lm.rows, lm.targets, 7, head=lm.Wc, bias=lm.bias if with_bias else None)
            assert bool(torch.isnan(lp[poisoned]).all()), (lm.name, with_bias, lp[poisoned].tolist())
            assert bool((gr[poisoned] == 0).all()), (lm.name, with_bias, gr[poisoned].tolist())
            wl, wg = want[with_bias]
            assert torch.equal(bits(lp[~poisoned]), bits(wl[~poisoned]))
            assert torch.equal(gr[~poisoned], wg[~poisoned])
    finally:
        lm.wte[list(POISON_IDS)] = saved
        lm.forward()


def test_score_batch_matches_direct_calls(neo):
    """LogLikelihoodScorer.score_batch against sgpt_lm_logprobs on the rows the reference selects: the last len(cont)
    positions of each input (sgptce.py:196-200).  Sums must be the sequential fp32 sums of the direct log-probs bit for
    bit, greedy flags all(greedy == target), and a request whose hidden state is NaN must get a NaN sum."""
    from sgpt_b200.cross_encoder import LogLikelihoodScorer

    lm = neo
    sc = LogLikelihoodScorer(lm.cfg, {**lm.w, "lm_head.weight": lm.Wc}, max_tokens=4096, max_batch=16, rows_per_chunk=7)
    assert sc.lm_head.data_ptr() == lm.Wc.data_ptr()
    rs = np.random.RandomState(8)

    def toks(n):
        t = rs.randint(0, lm.V, n)
        t[np.isin(t, POISON_IDS)] = 13
        return t.tolist()

    in_lens, cont_lens = (1, 40, 300, 7, 2, 100, 64), (1, 40, 12, 3, 1, 33, 20)
    inputs = [toks(n) for n in in_lens]
    conts = [toks(n) for n in cont_lens]
    conts[1][0], conts[2][-1] = 0, lm.V - 1

    def direct(inputs, conts):
        lens = np.array([len(x) for x in inputs])
        cl = np.array([len(c) for c in conts])
        cu = np.concatenate([[0], np.cumsum(lens)])
        rows = np.concatenate([np.arange(cu[b + 1] - cl[b], cu[b + 1]) for b in range(len(inputs))]).astype(np.int32)
        tg = np.concatenate([np.asarray(c) for c in conts]).astype(np.int32)
        off = np.concatenate([[0], np.cumsum(cl)])
        lp, gr = lm.run(torch.from_numpy(rows).cuda(), torch.from_numpy(tg).cuda(), 5, head=sc.lm_head,
                        handle=sc.encoder._handle)  # the residual score_batch's forward left in the scorer's handle
        lp, gr = lp.cpu().numpy(), gr.cpu().numpy()
        sums = np.array([np.cumsum(lp[off[b]:off[b + 1]], dtype=np.float32)[-1] for b in range(len(inputs))],
                        dtype=np.float32)
        flags = [bool((gr[off[b]:off[b + 1]] == tg[off[b]:off[b + 1]]).all()) for b in range(len(inputs))]
        return sums, flags, gr, off

    def check(inputs, conts):
        got, got_flags = sc.score_batch(inputs, conts, return_greedy=True)
        want, want_flags, gr, off = direct(inputs, conts)
        got = got.cpu().numpy()
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan)
        assert np.array_equal(got[~nan].view(np.int32), want[~nan].view(np.int32)), (got, want)
        assert got_flags == want_flags
        return got, got_flags, gr, off

    saved = lm.wte[list(POISON_IDS)].clone()
    try:
        _, flags, gr, off = check(inputs, conts)
        assert not any(flags)
        # request 0 continues with its greedy tokens, request 3 with all but its last
        conts[0] = gr[off[0]:off[1]].tolist()
        conts[3] = gr[off[3]:off[4]].tolist()
        conts[3][-1] = (conts[3][-1] + 1) % lm.V
        # two more requests: one NaN token alone, one NaN token inside the input (every later position is NaN too)
        lm.wte[POISON_IDS[0]] = float("nan")
        inputs += [[POISON_IDS[0]], [7, POISON_IDS[0], 9]]
        conts += [[5], [1, 2]]
        sums, flags, _, _ = check(inputs, conts)
        assert flags[0] and not flags[3], flags
        assert np.isnan(sums[-2:]).all() and not np.isnan(sums[:-2]).any(), sums
        assert flags[-2:] == [False, False]
    finally:
        lm.wte[list(POISON_IDS)] = saved
        sc.close()


def test_rejections(neo):
    """A workspace one byte short, rows_per_chunk <= 0, vocab <= 0 and a workspace that is not 16-byte aligned are
    rejected before any CUDA call; the unaligned workspace with M = 0, so a missing check could not launch anything."""
    lm = neo
    L, lib, h = lm.L, lm.lib, lm.enc._handle
    M, rpc = 3, 7
    need = lm.ws_bytes(rpc)
    rows, tg = lm.rows[:M], lm.targets[:M]
    lp = torch.full((M,), SENTINEL, device="cuda")
    gr = torch.full((M,), -7, dtype=torch.int32, device="cuda")
    ws = lm.ws.data_ptr()
    assert ws % 256 == 0

    def call(vocab=lm.V, m=M, ws_ptr=ws, ws_bytes=need, rows_per_chunk=rpc):
        return lib.sgpt_lm_logprobs(h, lm.W.data_ptr(), None, vocab, rows.data_ptr(), tg.data_ptr(), m, lp.data_ptr(),
                                    gr.data_ptr(), ws_ptr, ws_bytes, rows_per_chunk, L.current_stream())

    assert call(ws_bytes=need - 1) == 1
    assert call(ws_ptr=None) == 1
    for bad in (0, -1):
        assert call(rows_per_chunk=bad, ws_bytes=lm.ws.numel()) == 1
        assert call(vocab=bad, ws_bytes=lm.ws.numel()) == 1
        assert lm.lib.sgpt_lm_logprobs_workspace_bytes(lm.d, lm.V, bad) == 0
    for off in (1, 8):
        assert call(m=0, ws_ptr=ws + off, ws_bytes=need) == 1
        assert b"aligned" in lib.sgpt_last_error()
    torch.cuda.synchronize()
    assert bool((lp == SENTINEL).all()) and bool((gr == -7).all())
    assert call(m=0) == 0 and call(ws_ptr=ws + 16, ws_bytes=need) == 0  # the same arguments are otherwise valid
    assert torch.equal(bits(lp), bits(lm.base(False)[0][:M]))
