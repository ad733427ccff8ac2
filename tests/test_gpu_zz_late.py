"""GPU tests added late in round 1 (GPT-J scorer, multi-row-tile scores GEMM, sharded DRES, IR evaluator).  They run last
(pytest orders files alphabetically and the driver runs with -x) so that a failure here could not hide the parity tests
above."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN
from tests.helpers import ToyTokenizer
from tests.test_gpu_cross_encoder import TOL_PER_TOKEN, _requests

pytestmark = pytest.mark.gpu


def test_gptj_untied_lm_head_with_bias_vs_executed_reference():
    """GPT-J scorer (rotary QKV epilogue, parallel residual, hd 128, untied lm_head + bias — the SGPT-CE 6.1B
    architecture) vs the reference functions executed on HF GPTJForCausalLM (tests/golden/make_ce.py)."""
    from oracle import gptj as ogptj
    from sgpt_b200 import ModelConfig
    from sgpt_b200.cross_encoder import LogLikelihoodScorer

    z = np.load(os.path.join(GOLDEN, "ce_gptj_tiny.npz"))
    L, d, H, ff, vocab, max_pos, rd = [int(x) for x in z["spec"]]
    spec = ogptj.GPTJSpec(n_layer=L, d_model=d, n_head=H, d_ff=ff, vocab=vocab, max_pos=max_pos, rotary_dim=rd)
    w = ogptj.init_weights(spec, int(z["weight_seed"]))
    g = torch.Generator().manual_seed(int(z["head_seed"]))  # same construction as make_ce.py:gptj_lm_head
    hw = (torch.randn(vocab, d, generator=g) * 0.05).to(torch.bfloat16).float()
    hb = (torch.randn(vocab, generator=g) * 0.5).float()
    sd = {"transformer." + k: v for k, v in w.items()}  # *ForCausalLM checkpoint naming
    sd["lm_head.weight"], sd["lm_head.bias"] = hw, hb
    cfg = ModelConfig(arch="gptj", n_layer=L, d_model=d, n_head=H, d_ff=ff, vocab=vocab, max_pos=max_pos, rotary_dim=rd)
    s = LogLikelihoodScorer(cfg, sd, max_tokens=1024, max_batch=8, rows_per_chunk=16)
    assert s.lm_bias is not None and s.vocab == vocab
    reqs = _requests(z)
    got = s.loglikelihood_tokens(reqs, int(z["max_length"]), batch_size=4, instruction_len=int(z["instruction_len"]))
    for gv, wv, (_, _, cont) in zip(got, z["loglik"], reqs):
        assert abs(gv - wv) < TOL_PER_TOKEN * len(cont), (gv, wv, len(cont))
    s.close()


def test_scores_gemm_with_more_than_one_row_tile():
    """sgpt_scores with nq > 128 (several M tiles of the CL=1 similarity GEMM): the LM head of the cross-encoder scorer
    runs it with rows_per_chunk rows; checked against fp64 matmul of the same bf16 inputs."""
    from sgpt_b200 import _lib

    g = torch.Generator().manual_seed(4)
    for nq, n, D in ((300, 1000, 128), (129, 50257, 64)):
        q = torch.randn(nq, D, generator=g).to(torch.bfloat16)
        c = torch.randn(n, D, generator=g).to(torch.bfloat16)
        lds = (n + 3) // 4 * 4
        out = torch.full((nq, lds), float("nan"), dtype=torch.float32, device="cuda")
        qd, cd = q.cuda(), c.cuda()
        _lib.check(_lib.lib().sgpt_scores(qd.data_ptr(), cd.data_ptr(), None, None, out.data_ptr(), lds, nq, n, D,
                                          _lib.current_stream()), "sgpt_scores")
        want = q.double() @ c.double().T
        assert (out[:, :n].cpu().double() - want).abs().max() < 1e-3 * D ** 0.5, (nq, n, D)


def test_sharded_dres_world1_equals_chunked_dres():
    """The multi-rank DRES class at world size 1 (one resident shard instead of 3 chunks, same kernels) returns the
    ranking of the chunked single-GPU DRES."""
    from oracle import gpt_neo
    from sgpt_b200 import CustomEmbedder, DenseRetrievalExactSearch, ModelConfig, ShardedDenseRetrievalExactSearch

    spec = gpt_neo.NeoSpec(n_layer=2, d_model=128, n_head=2, d_ff=512, vocab=500, max_pos=64, window=8)
    w = gpt_neo.init_weights(spec, seed=0)
    cfg = ModelConfig(arch="gpt_neo", n_layer=2, d_model=128, n_head=2, d_ff=512, vocab=500, max_pos=64, window=8)
    emb = CustomEmbedder("toy-gpt-neo", batch_size=16, device="cuda:0", method="weightedmean", specb=True, maxseqlen=40,
                         config=cfg, state_dict=w, tokenizer=ToyTokenizer(vocab=500))
    rs = np.random.RandomState(0)
    words = [f"w{i}" for i in range(300)]
    corpus = {f"d{i}": {"title": " ".join(rs.choice(words, 3)), "text": " ".join(rs.choice(words, rs.randint(1, 60)))}
              for i in range(130)}
    queries = {f"q{i}": " ".join(rs.choice(words, rs.randint(1, 12))) for i in range(9)}
    queries["d5"] = corpus["d5"]["text"]
    top_k = 20
    res = DenseRetrievalExactSearch(emb, batch_size=16, corpus_chunk_size=50).search(corpus, queries, top_k, "cos_sim")
    res1 = ShardedDenseRetrievalExactSearch(emb, batch_size=16, corpus_chunk_size=50).search(corpus, queries, top_k, "cos_sim")
    for qid in queries:
        assert "d5" not in res1["d5"]
        # both keep top_k+1 candidates per scan and drop the self match afterwards (XS:102-118), so a query that IS a corpus
        # document ends with top_k entries from one scan and top_k+1 from three: compare the top_k both must have
        r1 = sorted(res1[qid], key=res1[qid].get, reverse=True)[:top_k]
        r0 = sorted(res[qid], key=res[qid].get, reverse=True)[:top_k]
        assert len(res1[qid]) >= top_k and r1 == r0, qid
        assert max(abs(res1[qid][c] - res[qid][c]) for c in r1) < 2e-5


def test_information_retrieval_evaluator_on_corpus_shard():
    """InformationRetrievalEvaluator with its default search (CorpusShard on the GPU) == the same evaluator with the
    oracle's CPU search on the same bf16-rounded embeddings."""
    import json

    from oracle import search as osearch
    from sgpt_b200 import InformationRetrievalEvaluator

    with open(os.path.join(GOLDEN, "ir_eval.json")) as f:
        z = json.load(f)
    relevant = {k: set(v) for k, v in z["relevant"].items()}
    g = torch.Generator().manual_seed(2)
    table = torch.randn(100, 64, generator=g).to(torch.bfloat16).float()  # bf16-exact so both paths see the same vectors

    class StubModel:
        def __init__(self, dev):
            self.dev = dev

        def encode(self, sentences, batch_size=32, convert_to_tensor=True, **kw):
            return torch.stack([table[int(s.split()[-1])] for s in sentences]).to(self.dev)

    def cpu_search(q, c, k, fn):
        return osearch.topk_ids(osearch.SCORE_FUNCTIONS[fn](q.cpu(), c.cpu()), k)

    kw = dict(mrr_at_k=[10], ndcg_at_k=[10], accuracy_at_k=[1, 5], precision_recall_at_k=[3], map_at_k=[20])
    got = InformationRetrievalEvaluator(z["queries"], z["corpus"], relevant, **kw).compute_metrices(StubModel("cuda"))
    want = InformationRetrievalEvaluator(z["queries"], z["corpus"], relevant, search_fn=cpu_search, **kw).compute_metrices(
        StubModel("cpu"))
    for name in ("cos_sim", "dot_score"):
        for metric in want[name]:
            for k, v in want[name][metric].items():
                assert abs(got[name][metric][k] - v) < 1e-9, (name, metric, k)
