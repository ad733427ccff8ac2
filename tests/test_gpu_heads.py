"""GPU parity tests of the rows added beside the hot path (SURVEY.md §8f rows 1–3; run with pytest -m gpu): learnt
position-weighted pooling, Dense / Asym / Normalize heads and the sentence-transformers directory loader against
embeddings produced by the REFERENCE's own module classes (tests/golden/make_st_model.py); the USEB-style encode; the
pickle embedding cache; the upstream-beir call convention of the exact search.  Everything runs through the C ABI."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN
from tests.helpers import min_row_cosine

pytestmark = pytest.mark.gpu

COS_TOL = 1e-3  # north_star tolerance on pooled embeddings


class IdTokenizer:
    """Texts are space-separated token ids: lets a test feed exact id sequences through the text-level API."""
    pad_token_id = 299
    model_max_length = 64

    def tokenize(self, text):
        return text.split()

    def convert_tokens_to_ids(self, tokens):
        return [int(t) for t in tokens]

    def encode(self, text, add_special_tokens=False):
        return [int(t) for t in text.split()]


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(GOLDEN, "st_tiny.npz"))


def _sentences(ref):
    return [" ".join(str(int(t)) for t, m in zip(row, mrow) if m) for row, mrow in zip(ref["ids"], ref["mask"])]


def test_pool_ex_learnt_position_weights_bit_level(ref):
    """sgpt_pool on the reference's fp32 token embeddings (x_bf16 = 0, no LayerNorm): same arithmetic as
    WeightedMeanPooling.forward, so fp32 agreement to rounding (1e-5), not just cosine."""
    from sgpt_b200 import _lib
    from sgpt_b200.encoder import pack_ragged

    tok, mask = ref["token_embeddings"], ref["mask"]
    B, S, d = tok.shape
    _, pos, cu, _ = pack_ragged(ref["ids"], mask)
    x = torch.from_numpy(tok.reshape(B * S, d)[mask.reshape(-1).astype(bool)]).cuda().contiguous()
    T = x.shape[0]
    pw = torch.from_numpy(ref["position_weights"]).cuda()
    out = torch.empty((B, d), dtype=torch.float32, device="cuda")
    ws = torch.empty(2 * T + B, dtype=torch.float32, device="cuda")
    pos_d, cu_d = torch.from_numpy(pos).cuda(), torch.from_numpy(cu).cuda()  # keep alive: raw pointers below
    rc = _lib.lib().sgpt_pool(x.data_ptr(), 0, pos_d.data_ptr(), cu_d.data_ptr(),
                              None, None, 1e-5, pw.data_ptr(), pw.numel(), out.data_ptr(), ws.data_ptr(), B, T, d,
                              _lib.POOL_WEIGHTEDMEAN, 1, 0, 0, 1.0, _lib.current_stream())
    _lib.check(rc, "sgpt_pool")
    assert np.abs(out.cpu().numpy() - ref["pooled_learnt"]).max() < 1e-5
    # a table needs the weightedmean mode
    rc = _lib.lib().sgpt_pool(x.data_ptr(), 0, None, None, None, None, 1e-5, pw.data_ptr(), pw.numel(), out.data_ptr(),
                              ws.data_ptr(), B, T, d, _lib.POOL_MEAN, 1, 0, 0, 1.0, _lib.current_stream())
    assert rc == 1


def test_dense_head_all_activations(ref):
    from sgpt_b200.heads import DenseHead

    x = torch.from_numpy(ref["pooled_learnt"]).cuda()
    w, b = torch.from_numpy(ref["dense_w"]), torch.from_numpy(ref["dense_b"])
    got = DenseHead(w, b, "torch.nn.modules.activation.Tanh")(x).cpu().numpy()
    assert np.abs(got - ref["dense_out"]).max() < 2e-6  # the reference Dense module's own output on the same input
    g = torch.Generator().manual_seed(3)
    for B, K, N in ((1, 8, 1), (37, 100, 33), (130, 768, 257)):  # ragged tile edges in every dimension
        x = torch.randn(B, K, generator=g)
        w = torch.randn(N, K, generator=g) / K ** 0.5
        b = torch.randn(N, generator=g)
        lin = x.double() @ w.double().T
        for act, fn in (("identity", lambda t: t), ("tanh", torch.tanh), ("relu", torch.relu), ("sigmoid", torch.sigmoid)):
            got = DenseHead(w, b, act)(x.cuda()).cpu().double()
            assert (got - fn(lin + b.double())).abs().max() < 5e-6, (B, K, N, act)
        got = DenseHead(w, None, "identity")(x.cuda()).cpu().double()
        assert (got - lin).abs().max() < 5e-6
    with pytest.raises(ValueError):
        DenseHead(w, b, "tanh")(torch.zeros(2, 5, device="cuda"))


def test_sentence_encoder_from_reference_written_directory(ref):
    """Transformer -> learnt WeightedMeanPooling -> Dense(Tanh) -> Normalize, loaded from the directory the reference
    classes saved, through SentenceTransformer.encode's signature; expected values from the reference modules."""
    from sgpt_b200 import SentenceEncoder, load_st_directory

    model = SentenceEncoder.from_spec(load_st_directory(os.path.join(GOLDEN, "st_tiny")), tokenizer=IdTokenizer(),
                                      batch_capacity=8)
    assert model.max_seq_length == 32 and model.get_sentence_embedding_dimension() == 48 and model.normalize
    sents = _sentences(ref)
    got = model.encode(sents, batch_size=4)  # two batches, length-sorted and un-sorted again
    assert got.shape == (6, 48) and isinstance(got, np.ndarray)
    assert min_row_cosine(got, ref["full"]) > 1 - COS_TOL
    assert np.abs(np.linalg.norm(got, axis=1) - 1).max() < 1e-5
    assert np.abs(got - ref["full"]).max() < 2e-2
    one = model.encode(sents[3], convert_to_tensor=True)
    assert one.shape == (48,) and one.is_cuda
    assert min_row_cosine(one[None].cpu(), ref["full"][3:4]) > 1 - COS_TOL
    # stages: learnt-weight pooling alone (encoder call) vs the reference WeightedMeanPooling output
    pooled = model.encoder.encode_tokens(ref["ids"], ref["mask"], method="weightedmean", clamp=True).cpu()
    assert min_row_cosine(pooled, ref["pooled_learnt"]) > 1 - COS_TOL
    # too long for the learnt table -> error like the reference's shape assert
    model.encoder.set_position_weights(torch.ones(4))
    with pytest.raises(RuntimeError, match="learnt position weights"):
        model.encoder.encode_tokens(ref["ids"], ref["mask"], method="weightedmean")
    model.encoder.set_position_weights(None)
    pooled = model.encoder.encode_tokens(ref["ids"], ref["mask"], method="weightedmean").cpu()
    assert min_row_cosine(pooled, ref["pooled_fixed"]) > 1 - COS_TOL  # back to the fixed i+1 weights
    model.encoder.close()


def test_asym_model_routes_queries_and_documents(ref):
    from sgpt_b200 import SentenceBERTAsym, SentenceEncoder

    model = SentenceEncoder.from_pretrained(os.path.join(GOLDEN, "st_tiny_asym"), tokenizer=IdTokenizer(), batch_capacity=8)
    assert model.pooling == "weightedmean" and model.asym is not None and not model.normalize
    wrap = SentenceBERTAsym(model)
    sents = _sentences(ref)
    q = wrap.encode_queries(sents, batch_size=8)
    assert q.shape == (6, 32) and min_row_cosine(q, ref["asym_qry"]) > 1 - COS_TOL
    d = wrap.encode_corpus([{"title": "", "text": s} for s in sents], batch_size=3, convert_to_tensor=True)
    assert min_row_cosine(d.cpu(), ref["asym_doc"]) > 1 - COS_TOL
    plain = model.encode(sents)  # no text key: no head (Asym allow_empty_key)
    assert plain.shape == (6, 128) and min_row_cosine(plain, ref["pooled_fixed"]) > 1 - COS_TOL
    normed = model.encode([{"QRY": s} for s in sents], normalize_embeddings=True)
    want = ref["asym_qry"] / np.linalg.norm(ref["asym_qry"], axis=1, keepdims=True)
    assert min_row_cosine(normed, want) > 1 - COS_TOL and np.abs(np.linalg.norm(normed, axis=1) - 1).max() < 1e-5
    model.encoder.close()


def test_useb_encode_and_pickle_cache_round_trip(ref, tmp_path, monkeypatch):
    from sgpt_b200 import CustomEmbedder, load_st_directory

    monkeypatch.chdir(tmp_path)
    path = os.path.join(GOLDEN, "st_tiny")
    spec = load_st_directory(path)
    emb = CustomEmbedder(model_name=path, batch_size=4, method="weightedmean", dataset="toy", save_emb=True,
                         config=spec.config, state_dict=spec.state_dict, tokenizer=IdTokenizer(), maxseqlen=32)
    sents = _sentences(ref)
    out = emb.encode(sents, method="learntmean")  # USEB flavour: List[List[float]], weights from 1_WeightedMeanPooling
    assert isinstance(out, list) and isinstance(out[0], list) and isinstance(out[0][0], float)
    assert min_row_cosine(np.array(out), ref["pooled_learnt"]) > 1 - COS_TOL
    out = emb.encode(sents, method="weightedmean")  # the table is removed again afterwards
    assert min_row_cosine(np.array(out), ref["pooled_fixed"]) > 1 - COS_TOL
    # pickle cache: first call computes + writes, second call must not touch the encoder
    queries = [(f"q{i}", s) for i, s in enumerate(sents)]
    first = emb.encode_queries(queries, batch_size=4)
    assert os.path.exists(f"embeddings/{os.path.basename(path)}/weightedmean/toy_queries.pickle")
    assert min_row_cosine(first, ref["pooled_fixed"]) > 1 - COS_TOL
    emb.encoder.close()
    again = emb.encode_queries(list(reversed(queries)), batch_size=4)
    assert np.array_equal(again, first[::-1])
    on_dev = emb.encode_queries(queries, batch_size=4, convert_to_tensor=True)
    assert on_dev.is_cuda and np.array_equal(on_dev.cpu().numpy(), first)


def test_exact_search_upstream_beir_convention(ref):
    """plain_lists=True: encode_queries(List[str]) / encode_corpus(List[dict]) as beir's own DRES calls the ST wrappers."""
    from sgpt_b200 import DenseRetrievalExactSearch, SentenceBERTBOSEOS, SentenceEncoder, load_st_directory

    spec = load_st_directory(os.path.join(GOLDEN, "st_tiny_asym"))
    spec.asym = {}
    model = SentenceEncoder.from_spec(spec, tokenizer=IdTokenizer(), batch_capacity=8)
    wrap = SentenceBERTBOSEOS(model)  # no specb/speca: plain texts
    wrap.device = model.device
    sents = _sentences(ref)
    corpus = {f"c{i}": {"title": "", "text": s} for i, s in enumerate(sents)}
    queries = {"qa": sents[2], "c4": sents[4]}  # second query id collides with a corpus id: self match is dropped
    dres = DenseRetrievalExactSearch(wrap, batch_size=4, corpus_chunk_size=4, plain_lists=True)
    res = dres.search(corpus, queries, top_k=3, score_function="cos_sim")
    assert max(res["qa"], key=res["qa"].get) == "c2" and abs(res["qa"]["c2"] - 1.0) < 1e-3
    assert "c4" not in res["c4"] and len(res["c4"]) <= 4
    e = torch.from_numpy(ref["pooled_fixed"]).to(torch.bfloat16).float()
    e = e / e.norm(dim=1, keepdim=True)
    want = (e[2] @ e.T)
    for cid, s in res["qa"].items():
        assert abs(s - want[int(cid[1:])].item()) < 5e-3
    model.encoder.close()
