"""GPU parity tests (run on an H100: pytest -m gpu).  Everything goes through the C ABI (ctypes -> libsgpt_b200.so).

Bars (BASELINE.json north_star): pooled embeddings within 1e-3 cosine of the reference HF path on the same inputs and
weights; identical top-k document ids vs the oracle evaluated on the same stored (bf16-rounded) vectors, ties at the
cut compared as sets.  Golden fixtures were produced by the reference code itself (tests/golden/make_golden.py).
"""
import os

import numpy as np
import pytest
import torch

from oracle import gpt_neo, pooling, search
from tests.helpers import ToyTokenizer, min_row_cosine, planted_corpus, ragged_batch

pytestmark = pytest.mark.gpu

COS_TOL = 1e-3  # north_star: "within 1e-3 cosine on pooled embeddings"


def _cfg_from_spec(spec):
    from sgpt_b200 import ModelConfig

    return ModelConfig(arch="gpt_neo", n_layer=spec.n_layer, d_model=spec.d_model, n_head=spec.n_head, d_ff=spec.d_ff,
                       vocab=spec.vocab, max_pos=spec.max_pos, window=spec.window, ln_eps=spec.ln_eps,
                       attention_layers=list(spec.attention_layers))


def _spec_from(npz):
    L, d, H, ff, vocab, max_pos, window = [int(x) for x in npz["spec"]]
    return gpt_neo.NeoSpec(n_layer=L, d_model=d, n_head=H, d_ff=ff, vocab=vocab, max_pos=max_pos, window=window)


@pytest.fixture(scope="module")
def tiny_encoder(golden_dir):
    from sgpt_b200 import Encoder

    z = np.load(os.path.join(golden_dir, "neo_tiny.npz"))
    spec = _spec_from(z)
    w = gpt_neo.init_weights(spec, seed=int(z["weight_seed"]))
    enc = Encoder(_cfg_from_spec(spec), w, device="cuda:0", max_tokens=4096, max_batch=64)
    yield z, spec, w, enc
    enc.close()


def test_tiny_model_all_pooling_modes_vs_reference_fixture(tiny_encoder):
    """4-layer model with window 16 < S 48 (local-attention layers active), ragged lengths incl. 1 and S."""
    z, spec, w, enc = tiny_encoder
    ids, mask = z["input_ids"], z["attention_mask"]
    got = enc.encode_tokens(ids, mask, method="weightedmean").cpu()
    assert min_row_cosine(got, z["pooled_weightedmean"]) > 1 - COS_TOL
    assert np.abs(got.numpy() - z["pooled_weightedmean"]).max() < 0.05
    got = enc.encode_tokens(ids, mask, method="mean").cpu()
    assert min_row_cosine(got, z["pooled_mean"]) > 1 - COS_TOL
    # lasttoken: script semantics (BDR:271-282); Pooling.py's argmin variant is wrong on unpadded rows, so compare with
    # the oracle's script variant on the reference hidden states
    hs_last = torch.from_numpy(z["hidden_states"][-1])
    want = pooling.last_token(hs_last, torch.from_numpy(mask).long())
    got = enc.encode_tokens(ids, mask, method="lasttoken").cpu()
    assert min_row_cosine(got, want) > 1 - COS_TOL
    mid = int(z["mid_layer"])
    got = enc.encode_tokens(ids, mask, method="weightedmean", layer_idx=mid).cpu()
    assert min_row_cosine(got, z["pooled_weightedmean_mid"]) > 1 - COS_TOL
    # all-hidden-state modes and script lasttoken vs the EXECUTED reference pooling block (make_script_pooling.py)
    sp = np.load(os.path.join(os.path.dirname(__file__), "golden", "script_pooling_neo_tiny.npz"))
    for method in ("meanmean", "lasttokenmean", "lasttoken", "mean", "weightedmean"):
        got = enc.encode_tokens(ids, mask, method=method).cpu()
        assert min_row_cosine(got, sp["pooled_" + method]) > 1 - COS_TOL, method
    got = enc.encode_tokens(ids, mask, method="meanmean", normalize=True).cpu()
    assert torch.allclose(got.norm(dim=1), torch.ones(len(got)), atol=1e-5)
    assert min_row_cosine(got, sp["pooled_meanmean"]) > 1 - COS_TOL
    # normalize + clamp flags (ST path)
    got = enc.encode_tokens(ids, mask, method="weightedmean", clamp=True, normalize=True).cpu()
    assert torch.allclose(got.norm(dim=1), torch.ones(len(got)), atol=1e-5)
    assert min_row_cosine(got, z["pooled_weightedmean"]) > 1 - COS_TOL


def test_tiny_model_residual_stream_vs_reference_hidden_states(tiny_encoder):
    """Per-token check: the residual stream after all blocks, passed through ln_f on the host, must match HF's
    last hidden state (bf16 activations between kernels bound the error)."""
    z, spec, w, enc = tiny_encoder
    ids, mask = z["input_ids"], z["attention_mask"]
    enc.encode_tokens(ids, mask, method="weightedmean")
    resid = enc.last_residual().cpu()
    h = gpt_neo.layer_norm(resid, w["ln_f.weight"], w["ln_f.bias"], spec.ln_eps)
    ref = torch.from_numpy(z["hidden_states"][-1])[torch.from_numpy(mask).bool()]
    assert h.shape == ref.shape
    cos = torch.nn.functional.cosine_similarity(h.double(), ref.double(), dim=1)
    assert cos.min().item() > 1 - COS_TOL
    assert (h - ref).abs().max().item() < 0.08


def test_bf16_residual_stream_matches_reference_fixture(golden_dir):
    """The residual stream is stored in bf16 (what HF does for a bf16 checkpoint), against the HF fp32 fixture: pooled
    embeddings within the 1e-3 cosine bar, per-token residual tap readable."""
    from sgpt_b200 import Encoder

    z = np.load(os.path.join(golden_dir, "neo_tiny.npz"))
    spec = _spec_from(z)
    w = gpt_neo.init_weights(spec, seed=int(z["weight_seed"]))
    ids, mask = z["input_ids"], z["attention_mask"]
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


def test_left_padded_rows_use_padded_positions(tiny_encoder):
    """Pooling weights / position ids follow the PADDED index (Pooling.py:104-112; HF position_ids = arange(S))."""
    z, spec, w, enc = tiny_encoder
    g = torch.Generator().manual_seed(3)
    S = 24
    ids = torch.randint(0, spec.vocab, (3, S), generator=g)
    mask = torch.zeros(3, S, dtype=torch.long)
    mask[0, 5:] = 1
    mask[1, :] = 1
    mask[2, S - 1:] = 1
    with torch.no_grad():
        hs = gpt_neo.forward(spec, w, ids, mask)
    want = pooling.weighted_mean(hs[-1], mask)
    got = enc.encode_tokens(ids.numpy(), mask.numpy(), method="weightedmean").cpu()
    # row 1 (unpadded) is exact-path; left-padded rows: HF lets pad positions be attended by nothing real (causal+mask),
    # real tokens see only real tokens, so the ragged execution is still exact
    assert min_row_cosine(got, want) > 1 - COS_TOL


def test_config1_sgpt125m_b32_s64_vs_reference_fixture(golden_dir):
    """BASELINE.json configs[0]: SGPT-125M-weightedmean bi-encoder, 32 synthetic sentences, seq_len 64 —
    pooled-embedding + cosine parity vs the reference (HF GPTNeoModel fp32 + Pooling.py)."""
    from sgpt_b200 import CorpusShard, Encoder

    z = np.load(os.path.join(golden_dir, "neo_125m_b32_s64.npz"))
    spec = _spec_from(z)
    w = gpt_neo.init_weights(spec, seed=int(z["weight_seed"]))
    enc = Encoder(_cfg_from_spec(spec), w, device="cuda:0", max_tokens=32 * 64, max_batch=32)
    got = enc.encode_tokens(z["input_ids"], z["attention_mask"], method="weightedmean")
    ref = torch.from_numpy(z["pooled_weightedmean"])
    assert min_row_cosine(got.cpu(), ref) > 1 - COS_TOL
    got_mean = enc.encode_tokens(z["input_ids"], z["attention_mask"], method="mean").cpu()
    assert min_row_cosine(got_mean, z["pooled_mean"]) > 1 - COS_TOL
    mid = int(z["mid_layer"])
    got_mid = enc.encode_tokens(z["input_ids"], z["attention_mask"], method="weightedmean", layer_idx=mid).cpu()
    assert min_row_cosine(got_mid, z["pooled_weightedmean_mid"]) > 1 - COS_TOL
    # cosine parity: pairwise cos_sim of our embeddings vs of the reference embeddings
    ours = search.cos_sim(got.cpu(), got.cpu())
    theirs = search.cos_sim(ref, ref)
    assert (ours - theirs).abs().max().item() < 2e-3
    # and through the device scorer: each embedding's nearest neighbour among the 32 is itself with score ~1
    shard = CorpusShard.from_embeddings(got, device="cuda:0")
    s, i = shard.search(got, 1, "cos_sim")
    assert i.view(-1).cpu().tolist() == list(range(32))
    assert (s.view(-1).cpu() - 1).abs().max().item() < 1e-5
    enc.close()


def test_encode_is_batch_invariant_and_deterministic(tiny_encoder):
    """Size-independent properties: a row's embedding does not depend on its batch mates; repeated calls are bit-equal."""
    z, spec, w, enc = tiny_encoder
    ids, mask = ragged_batch(40, 100, spec.vocab, seed=9)
    a = enc.encode_tokens(ids.numpy(), mask.numpy()).cpu()
    b = enc.encode_tokens(ids.numpy(), mask.numpy()).cpu()
    assert torch.equal(a, b)
    perm = torch.randperm(40, generator=torch.Generator().manual_seed(1))
    c = enc.encode_tokens(ids[perm].numpy(), mask[perm].numpy()).cpu()
    assert torch.allclose(c, a[perm], atol=1e-6)
    solo = enc.encode_tokens(ids[7:8].numpy(), mask[7:8].numpy()).cpu()
    assert torch.allclose(solo[0], a[7], atol=1e-6)


def test_full_size_batch_256x128_properties():
    """BASELINE.json configs[1] shape (SGPT-125M, batch 256, seq_len 128): finite output, permutation equivariance and
    agreement of a few rows with the CPU oracle (full oracle run would take minutes)."""
    from sgpt_b200 import Encoder, preset

    spec = gpt_neo.NeoSpec()
    w = gpt_neo.init_weights(spec, seed=0)
    enc = Encoder(preset("sgpt-125m"), w, device="cuda:0", max_tokens=256 * 128, max_batch=256)
    ids, mask = ragged_batch(256, 128, spec.vocab, seed=1235)
    mask[2:130] = 1  # half of the rows full length
    out = enc.encode_tokens(ids.numpy(), mask.numpy()).cpu()
    assert torch.isfinite(out).all()
    rows = [0, 1, 2, 200]
    with torch.no_grad():
        hs = gpt_neo.forward(spec, w, ids[rows], mask[rows])
    want = pooling.weighted_mean(hs[-1], mask[rows])
    assert min_row_cosine(out[rows], want) > 1 - COS_TOL
    perm = torch.randperm(256, generator=torch.Generator().manual_seed(2))
    out2 = enc.encode_tokens(ids[perm].numpy(), mask[perm].numpy()).cpu()
    again = enc.encode_tokens(ids.numpy(), mask.numpy()).cpu()
    assert torch.equal(again, out), f"non-deterministic: max diff {(again - out).abs().max().item():.3e}"
    assert torch.allclose(out2, out[perm], atol=1e-6), f"batch-order dependent: {(out2 - out[perm]).abs().max().item():.3e}"
    enc.close()


# ------------------------------------------------------------------------------------------------------------------
def _oracle_topk_on_stored(q, c, k, fn):
    """Oracle scores on the bf16-rounded vectors the device stores, fp32 arithmetic."""
    qs, cs = q.to(torch.bfloat16).float(), c.to(torch.bfloat16).float()
    return search.SCORE_FUNCTIONS[fn](qs, cs)


def _assert_same_topk(scores_dev, ids_dev, full, k, id_base=0):
    ids_dev, scores_dev = ids_dev.cpu(), scores_dev.cpu()
    for qi in range(full.shape[0]):
        order = torch.argsort(-full[qi].double(), stable=True)
        want_ids = order[:k]
        got = ids_dev[qi] - id_base
        cut = full[qi, want_ids[-1]].item()
        # ids identical except among scores within 1e-6 (relative to the score scale) of the cut, compared as sets
        tol = 1e-6 * max(1.0, full[qi].abs().max().item())  # fp32 accumulation-order noise scales with |score| (dot)
        safe_want = {int(j) for j in want_ids if full[qi, j].item() > cut + 2 * tol}
        got_set = {int(j) for j in got}
        assert safe_want <= got_set, (qi, len(safe_want - got_set))
        assert all(full[qi, j].item() >= cut - 2 * tol for j in got_set)
        assert (scores_dev[qi] - full[qi, got]).abs().max().item() < 20 * tol
        assert torch.all(scores_dev[qi][:-1] >= scores_dev[qi][1:])  # descending


@pytest.mark.parametrize("nq,n,D,k,fn", [(128, 20000, 768, 1001, "cos_sim"), (16, 5003, 2048, 1001, "dot"),
                                         (1, 3000, 768, 1001, "cos_sim"), (7, 600, 64, 1001, "cos_sim"),
                                         # >= 8 x 132 corpus tiles: the two-pass threshold-filter path; 130 queries =
                                         # two query blocks; ragged last tile (n % 256 != 0)
                                         (130, 320001, 64, 1001, "cos_sim"), (5, 310000, 128, 10, "dot"),
                                         # more than 128 queries: two CTAs per tile scan 256 queries per pass; 300 =
                                         # one 256-query block + a 44-query block on the single-CTA plan; 256 = a full one
                                         (300, 320001, 64, 100, "dot"), (256, 150001, 128, 1001, "cos_sim")])
def test_search_identical_topk_ids(nq, n, D, k, fn):
    from sgpt_b200 import CorpusShard

    q, c = planted_corpus(n, D, nq, seed=4321)
    shard = CorpusShard.from_embeddings(c.cuda(), device="cuda:0", id_base=1000)
    s, i = shard.search(q.cuda(), k, fn)
    full = _oracle_topk_on_stored(q, c, k, fn)
    kk = min(k, n)
    _assert_same_topk(s[:, :kk], i[:, :kk], full, kk, id_base=1000)
    if n < k:
        assert torch.all(i[:, n:] == -1) and torch.all(torch.isinf(s[:, n:]))


def test_search_nan_scores_become_minus_one():
    """XS:99: cos_scores[isnan] = -1."""
    from sgpt_b200 import CorpusShard

    q, c = planted_corpus(500, 64, 4, seed=1)
    c[17] = float("nan")
    shard = CorpusShard.from_embeddings(c.cuda(), device="cuda:0")
    s, i = shard.search(q.cuda(), 500, "cos_sim")
    pos = (i[0] == 17).nonzero().item()
    assert s[0, pos].item() == -1.0


def test_dres_search_matches_oracle_search_loop(tiny_encoder):
    """End to end through the reference's plug-in surface: CustomEmbedder(specb) + DenseRetrievalExactSearch with chunked
    corpus (3 chunks) vs the oracle's restatement of XS:80-134 run on the device-produced embeddings."""
    from sgpt_b200 import CustomEmbedder, DenseRetrievalExactSearch

    z, spec, w, _ = tiny_encoder
    tok = ToyTokenizer(vocab=spec.vocab)
    emb = CustomEmbedder("toy-gpt-neo", batch_size=16, device="cuda:0", method="weightedmean", specb=True, maxseqlen=40,
                         config=_cfg_from_spec(spec), state_dict=w, tokenizer=tok)
    rs = np.random.RandomState(0)
    words = [f"w{i}" for i in range(300)]
    corpus = {f"d{i}": {"title": " ".join(rs.choice(words, 3)), "text": " ".join(rs.choice(words, rs.randint(1, 60)))}
              for i in range(130)}
    queries = {f"q{i}": " ".join(rs.choice(words, rs.randint(1, 12))) for i in range(9)}
    queries["d5"] = corpus["d5"]["text"]  # a query that IS a corpus doc id -> self match must be dropped (XS:118)
    dres = DenseRetrievalExactSearch(emb, batch_size=16, corpus_chunk_size=50)
    top_k = 20
    res = dres.search(corpus, queries, top_k, "cos_sim")
    # oracle loop on the same embeddings and the same (length-sorted) corpus order
    corpus_ids = sorted(corpus, key=lambda k: len(corpus[k].get("title", "") + corpus[k].get("text", "")), reverse=True)
    q_emb = emb.encode_queries([(qid, queries[qid]) for qid in queries], convert_to_tensor=True)
    c_emb = emb.encode_corpus([(cid, corpus[cid]) for cid in corpus_ids], convert_to_tensor=True)
    want = search.search_embeddings(list(queries), q_emb.cpu().to(torch.bfloat16).float(), corpus_ids,
                                    c_emb.cpu().to(torch.bfloat16).float(), top_k, "cos_sim", corpus_chunk_size=50)
    assert set(res) == set(want)
    for qid in queries:
        assert "d5" not in res["d5"]
        got_sorted = sorted(res[qid], key=res[qid].get, reverse=True)
        want_sorted = sorted(want[qid], key=want[qid].get, reverse=True)
        assert len(res[qid]) == len(want[qid]) <= top_k + 1
        assert got_sorted == want_sorted, qid
        assert max(abs(res[qid][c] - want[qid][c]) for c in want[qid]) < 2e-5
    with pytest.raises(ValueError):
        dres.search(corpus, queries, top_k, "euclid")


def test_sentence_encoder_encode_signature(tiny_encoder):
    """ST-path surface: encode() sorts by length internally but returns rows in input order; str in -> 1-D out;
    specb markers are replaced by brackets (models/Transformer.py:131-153)."""
    from sgpt_b200 import SentenceBERTBOSEOS, SentenceEncoder

    z, spec, w, _ = tiny_encoder
    tok = ToyTokenizer(vocab=spec.vocab)
    st = SentenceEncoder(_cfg_from_spec(spec), w, tok, device="cuda:0", max_seq_length=32, batch_capacity=8)
    sents = ["a b c d e f", "x", "hello world this is a test", "q r"]
    e = st.encode(sents, batch_size=2)
    assert isinstance(e, np.ndarray) and e.shape == (4, spec.d_model)
    one = st.encode("x")
    assert one.shape == (spec.d_model,) and np.allclose(one, e[1], atol=1e-6)
    t = st.encode(sents, batch_size=8, convert_to_tensor=True, normalize_embeddings=True)
    assert t.is_cuda and torch.allclose(t.norm(dim=1), torch.ones(4, device=t.device), atol=1e-5)
    wrapped = SentenceBERTBOSEOS(st, specb=True)
    ids, mask = st.tokenize(["[SOS]" + "a b", "{SOS}" + "c"])
    assert ids[0, 0] == 58 and ids[0, 3] == 60 and ids[1, 0] == 90 and ids[1, 2] == 92
    qe = wrapped.encode_queries(["a b"], batch_size=4)
    de = wrapped.encode_corpus([{"title": "a", "text": "b"}], batch_size=4)
    assert qe.shape == de.shape == (1, spec.d_model) and not np.allclose(qe, de)
    st.encoder.close()


# --- GPT-J (SGPT-5.8B family, BASELINE configs[3]) and BLOOM (sgpt-bloom-7b1, configs[4]) encoders --------------------
@pytest.mark.parametrize("name", ["gptj_tiny", "bloom_tiny"])
def test_gptj_bloom_pooled_embeddings_vs_reference_fixture(golden_dir, name):
    """Tiny GPT-J (rotary q/k in the GEMM epilogue, parallel attn+MLP residual, hd 128) and BLOOM (ALiBi attention,
    embedding LayerNorm, per-head fused qkv regrouped at load) vs fixtures produced by HF GPTJModel / BloomModel +
    the reference's Pooling.py."""
    from oracle import bloom, gptj
    from sgpt_b200 import Encoder, ModelConfig

    z = np.load(os.path.join(golden_dir, name + ".npz"))
    a = [int(x) for x in z["spec"]]
    if name.startswith("gptj"):
        spec = gptj.GPTJSpec(n_layer=a[0], d_model=a[1], n_head=a[2], d_ff=a[3], vocab=a[4], max_pos=a[5], rotary_dim=a[6])
        w = gptj.init_weights(spec, seed=int(z["weight_seed"]))
        cfg = ModelConfig(arch="gptj", n_layer=a[0], d_model=a[1], n_head=a[2], d_ff=a[3], vocab=a[4], max_pos=a[5],
                          rotary_dim=a[6])
    else:
        spec = bloom.BloomSpec(n_layer=a[0], d_model=a[1], n_head=a[2], vocab=a[3])
        w = bloom.init_weights(spec, seed=int(z["weight_seed"]))
        cfg = ModelConfig(arch="bloom", n_layer=a[0], d_model=a[1], n_head=a[2], d_ff=4 * a[1], vocab=a[3], max_pos=1 << 20)
    enc = Encoder(cfg, w, device="cuda:0", max_tokens=2048, max_batch=16)
    ids, mask = z["input_ids"], z["attention_mask"]
    got = enc.encode_tokens(ids, mask, method="weightedmean").cpu()
    assert min_row_cosine(got, z["pooled_weightedmean"]) > 1 - COS_TOL
    got = enc.encode_tokens(ids, mask, method="mean").cpu()
    assert min_row_cosine(got, z["pooled_mean"]) > 1 - COS_TOL
    # all-hidden-state modes (BDR:243-257, 284-301) vs the executed reference pooling block
    sp = np.load(os.path.join(golden_dir, f"script_pooling_{name}.npz"))
    for method in ("meanmean", "lasttokenmean", "lasttoken"):
        got = enc.encode_tokens(ids, mask, method=method).cpu()
        assert min_row_cosine(got, sp["pooled_" + method]) > 1 - COS_TOL, method
    # per-token residual stream -> ln_f on the host vs HF's last hidden state
    enc.encode_tokens(ids, mask)
    resid = enc.last_residual().cpu()
    h = gpt_neo.layer_norm(resid, w["ln_f.weight"], w["ln_f.bias"], spec.ln_eps)
    ref = torch.from_numpy(z["hidden_states"][-1])[torch.from_numpy(mask).bool()]
    cos = torch.nn.functional.cosine_similarity(h.double(), ref.double(), dim=1)
    assert cos.min().item() > 1 - COS_TOL
    enc.close()


# --- full-width layers at reduced depth: the GEMM / attention shapes of the large configs ----------------------------
def test_wide_gpt_neo_hd128_long_sequences_vs_oracle():
    """SGPT-1.3B-width blocks (d 2048, 16 heads of 128, ff 8192) at depth 2, sequences up to 300 tokens: multi-tile
    attention (online softmax across key tiles) and the GPT-Neo local window (256 < 300) on the second layer."""
    from sgpt_b200 import Encoder

    spec = gpt_neo.NeoSpec(n_layer=2, d_model=2048, n_head=16, d_ff=8192, vocab=2000, max_pos=512, window=256)
    w = gpt_neo.init_weights(spec, seed=0)
    for k in list(w):  # keep the un-scaled GPT-Neo logits at a sane spread for the wider model
        if "q_proj" in k or "k_proj" in k:
            w[k] = (w[k] * (768 / 2048) ** 0.5 * 0.7).to(torch.bfloat16).float()
    enc = Encoder(_cfg_from_spec(spec), w, device="cuda:0", max_tokens=6 * 300, max_batch=6)
    ids, mask = ragged_batch(6, 300, spec.vocab, seed=5)
    mask[2] = 1  # a second full-length row
    with torch.no_grad():
        hs = gpt_neo.forward(spec, w, ids, mask)
    want = pooling.weighted_mean(hs[-1], mask)
    got = enc.encode_tokens(ids.numpy(), mask.numpy()).cpu()
    assert min_row_cosine(got, want) > 1 - COS_TOL
    enc.close()


def test_wide_gptj_hd256_and_bloom_hd128_vs_oracle():
    """GPT-J blocks with the real head_dim 256 / rotary_dim 64 and BLOOM blocks with head_dim 128, depth 2, S up to 300."""
    from oracle import bloom, gptj
    from sgpt_b200 import Encoder, ModelConfig

    js = gptj.GPTJSpec(n_layer=2, d_model=1024, n_head=4, d_ff=4096, vocab=2000, max_pos=512, rotary_dim=64)
    jw = gptj.init_weights(js, seed=1)
    enc = Encoder(ModelConfig(arch="gptj", n_layer=2, d_model=1024, n_head=4, d_ff=4096, vocab=2000, max_pos=512,
                              rotary_dim=64), jw, device="cuda:0", max_tokens=5 * 300, max_batch=5)
    ids, mask = ragged_batch(5, 300, js.vocab, seed=6)
    with torch.no_grad():
        want = pooling.weighted_mean(gptj.forward(js, jw, ids, mask)[-1], mask)
    got = enc.encode_tokens(ids.numpy(), mask.numpy()).cpu()
    assert min_row_cosine(got, want) > 1 - COS_TOL
    enc.close()

    bs = bloom.BloomSpec(n_layer=2, d_model=1024, n_head=8, vocab=2000)
    bw = bloom.init_weights(bs, seed=2)
    enc = Encoder(ModelConfig(arch="bloom", n_layer=2, d_model=1024, n_head=8, d_ff=4096, vocab=2000, max_pos=1 << 20),
                  bw, device="cuda:0", max_tokens=5 * 300, max_batch=5)
    ids, mask = ragged_batch(5, 300, bs.vocab, seed=7)
    with torch.no_grad():
        want = pooling.weighted_mean(bloom.forward(bs, bw, ids, mask)[-1], mask)
    got = enc.encode_tokens(ids.numpy(), mask.numpy()).cpu()
    assert min_row_cosine(got, want) > 1 - COS_TOL
    enc.close()


def test_semantic_search_matches_reference_util_and_shard_roundtrip(golden_dir, tmp_path):
    """`semantic_search` vs the hits the reference's own util.semantic_search produced for the scoring fixture
    (tests/golden/make_golden.py: run_scoring, chunk sizes 5/17, top_k 10), and CorpusShard.save/load reproduce the
    search bit for bit."""
    from sgpt_b200 import CorpusShard, semantic_search

    z = np.load(os.path.join(golden_dir, "scoring.npz"))
    q, c = torch.from_numpy(z["queries"]), torch.from_numpy(z["corpus"])
    # D = 100 is not a multiple of 8: pad with zero columns (changes neither dot products nor norms)
    pad = lambda x: torch.nn.functional.pad(x, (0, 4))  # noqa: E731
    hits = semantic_search(pad(q), pad(c), query_chunk_size=5, corpus_chunk_size=17, top_k=10)
    got_ids = np.array([[h["corpus_id"] for h in row] for row in hits])
    got_scores = np.array([[h["score"] for h in row] for row in hits], dtype=np.float32)
    # bf16 storage perturbs scores by ~1e-3: compare as sets with a tie band at the cut, scores within 5e-3
    for r in range(len(hits)):
        want = {int(i): float(s) for i, s in zip(z["hit_ids"][r], z["hit_scores"][r])}
        cut = min(want.values())
        for i, s in zip(got_ids[r], got_scores[r]):
            assert (int(i) in want and abs(want[int(i)] - s) < 5e-3) or abs(s - cut) < 5e-3, (r, i, s, cut)
        assert np.all(np.diff(got_scores[r]) <= 1e-7)  # best first
    shard = CorpusShard.from_embeddings(pad(c).cuda(), id_base=1000)
    s0, i0 = shard.search(pad(q).cuda(), 25, "dot")
    shard.save(str(tmp_path / "shard0"))
    again = CorpusShard.load(str(tmp_path / "shard0"), device="cuda:0")
    assert again.n == shard.n and again.id_base == 1000
    s1, i1 = again.search(pad(q).cuda(), 25, "dot")
    assert torch.equal(s0, s1) and torch.equal(i0, i1)


@pytest.mark.parametrize("k_hi", ["1", "24", "1001"])
def test_search_two_pass_front_and_back_lists(k_hi, monkeypatch):
    """The two-pass path keeps candidates above the upper threshold at the front of its lists and the rest at the back;
    the selection reads the back parts only when the front parts hold fewer than k entries.  SGPT_SEARCH_K_HI=1 puts the
    upper threshold at the sample's best score (front parts nearly empty: every query takes the back-list path), = k makes
    both thresholds equal (everything at the front); the result must be the oracle's either way.  130 k documents = the
    stride-8 sample of a shard with ~3 tiles per SM (the 125 k x 4096 shape of config 4 on 8 GPUs)."""
    from sgpt_b200 import CorpusShard

    monkeypatch.setenv("SGPT_SEARCH_K_HI", k_hi)
    nq, n, D, k = 37, 130001, 128, 1001
    q, c = planted_corpus(n, D, nq, seed=77)
    shard = CorpusShard.from_embeddings(c.cuda(), device="cuda:0", id_base=7)
    s, i = shard.search(q.cuda(), k, "cos_sim")
    full = _oracle_topk_on_stored(q, c, k, "cos_sim")
    _assert_same_topk(s, i, full, k, id_base=7)


def test_search_front_list_kernel_opt_in(monkeypatch):
    """SGPT_FRONT_SELECT=1: the final selection of the two-pass search by the front-list kernel (pack the entries above the
    upper threshold, sort all of them, take the first k) instead of the generic selection kernel — measured slower and off
    by default, but it must stay exact; queries it declines (front parts short) fall through to the generic kernel."""
    from sgpt_b200 import CorpusShard

    monkeypatch.setenv("SGPT_FRONT_SELECT", "1")
    nq, n, D, k = 37, 130001, 128, 1001
    q, c = planted_corpus(n, D, nq, seed=78)
    shard = CorpusShard.from_embeddings(c.cuda(), device="cuda:0", id_base=3)
    full = _oracle_topk_on_stored(q, c, k, "cos_sim")
    s, i = shard.search(q.cuda(), k, "cos_sim")
    _assert_same_topk(s, i, full, k, id_base=3)
    monkeypatch.setenv("SGPT_SEARCH_K_HI", "1")  # front parts nearly empty: every query is declined
    s, i = shard.search(q.cuda(), k, "cos_sim")
    _assert_same_topk(s, i, full, k, id_base=3)


def test_search_two_pass_with_massive_ties():
    """Two-pass filter path on a corpus with only 40 distinct vectors (every score value is shared by ~7750 documents):
    the admission threshold sits inside a tie group, which must not lose candidates."""
    from sgpt_b200 import CorpusShard

    g = torch.Generator().manual_seed(5)
    base = torch.randn(40, 64, generator=g)
    n = 310000
    c = base[torch.randint(0, 40, (n,), generator=g)]
    q = torch.randn(9, 64, generator=g)
    shard = CorpusShard.from_embeddings(c.cuda(), device="cuda:0")
    k = 1001
    s, i = shard.search(q.cuda(), k, "cos_sim")
    full = _oracle_topk_on_stored(q, c, k, "cos_sim")
    _assert_same_topk(s, i, full, k)
    for r in range(len(q)):
        assert len(set(i[r].tolist())) == k  # no document twice


def test_search_full_size_1m_docs_properties():
    """BASELINE size (128 queries x 1 M docs x 768, top-1001) through size-independent properties; torch on the GPU is
    used only as the checker: (a) descending scores, unique ids; (b) returned scores == cos_sim of the stored vectors;
    (c) exactness: fewer than k documents score above the returned k-th score; (d) planted near-duplicates rank first;
    (e) searching two half shards and merging == searching the whole shard."""
    from sgpt_b200 import CorpusShard
    from sgpt_b200.index import merge_topk

    dev, n, D, nq, k = torch.device("cuda:0"), 1_000_000, 768, 128, 1001
    g = torch.Generator(device=dev).manual_seed(99)
    q = torch.randn(nq, D, generator=g, device=dev)
    whole = CorpusShard(D, n, device=dev)
    for s0 in range(0, n, 100_000):
        c = torch.randn(100_000, D, generator=g, device=dev)
        idx = torch.arange(0, 100_000, 1000, device=dev)
        c[idx] = q[((s0 + idx) // 1000) % nq] + 0.3 * c[idx]  # doc 1000*j is a near-duplicate of query j % 128
        whole.add(c)
    del c
    s, i = whole.search(q, k, "cos_sim")
    assert torch.all(s[:, :-1] >= s[:, 1:])
    assert all(len(set(r)) == k for r in i.tolist())
    stored = whole.stored()
    qb = q.to(torch.bfloat16).float()
    qn = qb / qb.norm(dim=1, keepdim=True)
    # (b) recompute the returned scores from the stored rows
    rows = stored[i.reshape(-1)].float().reshape(nq, k, D)
    want = torch.einsum("qd,qkd->qk", qn, rows / rows.norm(dim=2, keepdim=True))
    assert (want - s).abs().max().item() < 2e-5
    # (c) exactness: count documents above the k-th returned score
    above = torch.zeros(nq, dtype=torch.int64, device=dev)
    for s0 in range(0, n, 100_000):
        blk = stored[s0:s0 + 100_000].float()
        sc = qn @ (blk / blk.norm(dim=1, keepdim=True)).T
        above += (sc > (s[:, -1:] + 2e-5)).sum(dim=1)
    assert int(above.max()) < k
    # (d) the planted near-duplicates of query j are documents 1000*m with m % 128 == j; the best hit must be one of them
    top1 = i[:, 0]
    assert torch.all(top1 % 1000 == 0) and torch.all((top1 // 1000) % nq == torch.arange(nq, device=dev))
    # (e) two half shards + merge
    half = n // 2
    a = CorpusShard.from_embeddings(stored[:half], device=dev, id_base=0)
    b = CorpusShard.from_embeddings(stored[half:], device=dev, id_base=half)
    sa, ia = a.search(q, k, "cos_sim")
    sb, ib = b.search(q, k, "cos_sim")
    sm, im = merge_topk(torch.stack([sa, sb]), torch.stack([ia, ib]))
    # a document's score does not depend on its shard, and ties resolve to the lowest ids: identical bits
    assert torch.equal(sm.view(torch.int32), s.view(torch.int32)) and torch.equal(im, i)
