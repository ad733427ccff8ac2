"""SURVEY.md §8f row 1 / VERDICT r01 item 9: the flow of the reference's ``main`` (biencoder/beir/beir_dense_retriever.py:
352-498) — GenericDataLoader, empty-text filtering, DenseRetrievalExactSearch behind EvaluateRetrieval(k_values=[1, 3, 5,
10, 100, 1000]).retrieve/evaluate — on the stand-in ``beir`` package of sgpt_b200/compat must reproduce what the
reference's own ``main`` wrote for the same toy BEIR set: its result file and its metrics, stored in
tests/golden/reference_main_toyset.json by tests/golden/make_reference_main.py, which ran that ``main`` unmodified on the
stand-in packages.  The classes that launch CUDA kernels are CPU stand-ins with the same interfaces (a toy embedder with
CustomEmbedder's constructor keywords; the oracle's restatement of the search loop behind DenseRetrievalExactSearch's
``search``).  The same flow with the real classes is covered by tests/test_gpu_heads.py and
`python -m sgpt_b200.compat.run_reference`."""
import json
import os
import zlib

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_main_toyset.json")


class _ToyEmbedder:
    """CustomEmbedder's protocol (BDR:107-120, 316-348) with a deterministic bag-of-words embedding on the CPU."""

    def __init__(self, model_name, batch_size=250, device="cpu", save_emb=False, reinit=False, layeridx=-1, method="mean",
                 dataset="scifact", specb=False, maxseqlen=None, **kwargs):
        self.kw = dict(model_name=model_name, batch_size=batch_size, device=device, method=method, specb=specb,
                       layeridx=layeridx, maxseqlen=maxseqlen, save_emb=save_emb)
        self.device = torch.device("cpu")

    @staticmethod
    def _vec(text, dim=32):
        v = torch.zeros(dim)
        for w in text.lower().split():
            g = torch.Generator().manual_seed(zlib.crc32(w.encode()))
            v += torch.randn(dim, generator=g)
        return v

    def encode_queries(self, queries, batch_size=None, **kwargs):
        return torch.stack([self._vec(t) for _, t in queries])

    def encode_corpus(self, corpus, batch_size=None, **kwargs):
        return torch.stack([self._vec((d["title"] + " " + d["text"]).strip() if "title" in d else d["text"].strip())
                            for _, d in corpus])


class _CpuDRES:
    """DenseRetrievalExactSearch's interface (XS:22-42) on the oracle's restatement of XS:44-134."""

    def __init__(self, model, batch_size=128, corpus_chunk_size=50000, **kwargs):
        self.model, self.batch_size, self.corpus_chunk_size = model, batch_size, corpus_chunk_size
        self.results = {}

    def search(self, corpus, queries, top_k, score_function, return_sorted=False, **kwargs):
        from oracle import search as osearch

        if score_function not in ("cos_sim", "dot"):
            raise ValueError("score function: {} must be either (cos_sim) for cosine similarity or (dot) for dot product"
                             .format(score_function))
        qids = list(queries)
        cids = sorted(corpus, key=lambda k: len(corpus[k].get("title", "") + corpus[k].get("text", "")), reverse=True)
        q = self.model.encode_queries([(i, queries[i]) for i in qids], batch_size=self.batch_size)
        c = self.model.encode_corpus([(i, corpus[i]) for i in cids], batch_size=self.batch_size, batch_num=0)
        self.results = osearch.search_embeddings(qids, q, cids, c, top_k, score_function,
                                                 corpus_chunk_size=self.corpus_chunk_size)
        return self.results


def make_toy_beir(root):
    """Toy BEIR directory <root>/datasets/toyset: the relevant document of every query repeats the query's words."""
    rs = np.random.RandomState(0)
    words = [f"w{i}" for i in range(200)]
    root = os.path.join(root, "datasets", "toyset")
    os.makedirs(os.path.join(root, "qrels"))
    corpus = {f"d{i}": {"title": " ".join(rs.choice(words, 2)), "text": " ".join(rs.choice(words, rs.randint(3, 30)))}
              for i in range(60)}
    corpus["d_empty"] = {"title": "t", "text": ""}  # removed by main (BDR:382-388)
    queries = {f"q{i}": corpus[f"d{i}"]["text"] for i in range(8)}
    with open(os.path.join(root, "corpus.jsonl"), "w") as f:
        for k, v in corpus.items():
            f.write(json.dumps({"_id": k, **v}) + "\n")
    with open(os.path.join(root, "queries.jsonl"), "w") as f:
        for k, v in queries.items():
            f.write(json.dumps({"_id": k, "text": v}) + "\n")
    with open(os.path.join(root, "qrels", "test.tsv"), "w") as f:
        f.write("query-id\tcorpus-id\tscore\n")
        for i in range(8):
            f.write(f"q{i}\td{i}\t1\n")
    return root, queries


def test_stand_in_packages_reproduce_the_reference_main_on_a_toy_set(tmp_path, monkeypatch):
    from sgpt_b200 import compat

    monkeypatch.syspath_prepend(compat.COMPAT_DIR)
    import beir
    from beir.datasets.data_loader import GenericDataLoader
    from beir.retrieval.evaluation import EvaluateRetrieval

    assert os.path.dirname(os.path.dirname(beir.__file__)) == compat.COMPAT_DIR  # the stand-in, not an installed beir

    data_path, queries = make_toy_beir(str(tmp_path))
    corpus, qs, qrels = GenericDataLoader(data_path).load(split="test")
    for k in [k for k, v in corpus.items() if not v["text"]]:
        del corpus[k]
    model = _CpuDRES(_ToyEmbedder(model_name="toy/model", method="weightedmean", device="cpu", batch_size=16, specb=True))
    retriever = EvaluateRetrieval(model, k_values=[1, 3, 5, 10, 100, 1000])
    results = retriever.retrieve(corpus, qs)
    ndcg, _map, recall, precision = retriever.evaluate(qrels, results, retriever.k_values)

    want = json.load(open(GOLDEN))
    assert set(results) == set(queries) == set(want["results"])
    for q, docs in want["results"].items():
        assert set(results[q]) == set(docs), q
        for d, v in docs.items():
            assert abs(results[q][d] - v) <= 1e-5 * (1 + abs(v)), (q, d)
    for i in range(8):
        assert max(results[f"q{i}"], key=results[f"q{i}"].get) == f"d{i}"  # the planted document ranks first
        assert "d_empty" not in results[f"q{i}"]
    for name, got in (("ndcgs", ndcg), ("maps", _map), ("recalls", recall), ("precisions", precision)):
        ref = want["metrics"][name]["toy_model"]["toyset"]
        assert set(got) == set(ref), name
        for key, v in ref.items():
            assert abs(got[key] - v) <= 1e-9, (name, key)
