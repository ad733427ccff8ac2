"""``InformationRetrievalEvaluator`` on the CUDA exact search (SURVEY.md §8f row 3).

Same constructor, ``__call__`` / ``compute_metrices`` / ``compute_metrics`` contract and metric definitions as
sentence_transformers/evaluation/InformationRetrievalEvaluator.py:15-299 (Accuracy@k, Precision/Recall@k, MRR@k, NDCG@k
with binary gains, MAP@k with the ``min(k, #relevant)`` denominator), but the corpus is scanned by ``CorpusShard.search``
(one resident bf16 shard, fused top-k) instead of per-chunk ``score_function`` + ``torch.topk`` + Python lists (:152-170):
the top ``max_k`` hits of the union of per-chunk top-``max_k`` lists ARE the global top ``max_k``, so the metrics are
those of the reference.  ``model`` is anything with ``encode(sentences, batch_size=…, convert_to_tensor=True)``
(``SentenceEncoder``); score functions are named ``"cos_sim"`` / ``"dot_score"`` as in the reference's default dict.
"""
from __future__ import annotations

import logging
import os
import torch
from typing import Callable, Dict, List, Optional, Set

import numpy as np

logger = logging.getLogger(__name__)

_SCORE_NAMES = {"cos_sim": "cos_sim", "dot_score": "dot"}


class InformationRetrievalEvaluator:
    def __init__(self, queries: Dict[str, str], corpus: Dict[str, str], relevant_docs: Dict[str, Set[str]],
                 corpus_chunk_size: int = 50000, mrr_at_k: List[int] = (10,), ndcg_at_k: List[int] = (10,),
                 accuracy_at_k: List[int] = (1, 3, 5, 10), precision_recall_at_k: List[int] = (1, 3, 5, 10),
                 map_at_k: List[int] = (100,), show_progress_bar: bool = False, batch_size: int = 32, name: str = "",
                 write_csv: bool = True, score_functions=("cos_sim", "dot_score"), main_score_function: str = None,
                 search_fn: Optional[Callable] = None):
        self.queries_ids = [qid for qid in queries if qid in relevant_docs and len(relevant_docs[qid]) > 0]  # :42-45
        self.queries = [queries[qid] for qid in self.queries_ids]
        self.corpus_ids = list(corpus.keys())
        self.corpus = [corpus[cid] for cid in self.corpus_ids]
        self.relevant_docs = relevant_docs
        self.corpus_chunk_size = corpus_chunk_size
        self.mrr_at_k, self.ndcg_at_k, self.accuracy_at_k = list(mrr_at_k), list(ndcg_at_k), list(accuracy_at_k)
        self.precision_recall_at_k, self.map_at_k = list(precision_recall_at_k), list(map_at_k)
        self.show_progress_bar, self.batch_size, self.name, self.write_csv = show_progress_bar, batch_size, name, write_csv
        names = list(score_functions.keys()) if isinstance(score_functions, dict) else list(score_functions)
        for n in names:
            if n not in _SCORE_NAMES:
                raise ValueError(f"score function {n!r}: built: {sorted(_SCORE_NAMES)}")
        self.score_function_names = sorted(names)
        self.main_score_function = main_score_function
        self.search_fn = search_fn  # (query_emb, corpus_emb, k, "cos_sim"|"dot") -> (scores [Q,k], ids [Q,k]); tests inject one
        self.csv_file = "Information-Retrieval_evaluation" + ("_" + name if name else "") + "_results.csv"
        self.csv_headers = ["epoch", "steps"]
        for score_name in self.score_function_names:  # :73-88
            self.csv_headers += ["{}-Accuracy@{}".format(score_name, k) for k in self.accuracy_at_k]
            for k in self.precision_recall_at_k:
                self.csv_headers += ["{}-Precision@{}".format(score_name, k), "{}-Recall@{}".format(score_name, k)]
            self.csv_headers += ["{}-MRR@{}".format(score_name, k) for k in self.mrr_at_k]
            self.csv_headers += ["{}-NDCG@{}".format(score_name, k) for k in self.ndcg_at_k]
            self.csv_headers += ["{}-MAP@{}".format(score_name, k) for k in self.map_at_k]

    def __call__(self, model, output_path: str = None, epoch: int = -1, steps: int = -1, num_proc: int = None,
                 *args, **kwargs) -> float:
        scores = self.compute_metrices(model, *args, num_proc=num_proc, **kwargs)
        if output_path is not None and self.write_csv:  # :100-131
            csv_path = os.path.join(output_path, self.csv_file)
            new = not os.path.isfile(csv_path)
            with open(csv_path, mode="w" if new else "a", encoding="utf-8") as f:
                if new:
                    f.write(",".join(self.csv_headers) + "\n")
                row = [epoch, steps]
                for name in self.score_function_names:
                    row += [scores[name]["accuracy@k"][k] for k in self.accuracy_at_k]
                    for k in self.precision_recall_at_k:
                        row += [scores[name]["precision@k"][k], scores[name]["recall@k"][k]]
                    row += [scores[name]["mrr@k"][k] for k in self.mrr_at_k]
                    row += [scores[name]["ndcg@k"][k] for k in self.ndcg_at_k]
                    row += [scores[name]["map@k"][k] for k in self.map_at_k]
                f.write(",".join(map(str, row)) + "\n")
        if self.main_score_function is None:  # :133-136
            return max(scores[name]["map@k"][max(self.map_at_k)] for name in self.score_function_names)
        return scores[self.main_score_function]["map@k"][max(self.map_at_k)]

    def _search(self, q_emb, c_emb, k, score_function):
        if self.search_fn is not None:
            return self.search_fn(q_emb, c_emb, k, score_function)
        from .index import CorpusShard

        shard = c_emb if isinstance(c_emb, CorpusShard) else CorpusShard.from_embeddings(c_emb)
        return shard.search(q_emb.to(shard.device), k, score_function)

    def _encode_corpus(self, corpus_model, q_emb):
        """The corpus is encoded `corpus_chunk_size` documents at a time like the reference (:150-152), each chunk added
        to ONE bf16 shard and its fp32 embeddings dropped — a multi-million-document corpus never exists as an fp32
        [N, d] device tensor.  (With an injected search_fn the chunks are concatenated instead.)"""
        chunk = max(1, int(self.corpus_chunk_size))
        if self.search_fn is not None:
            parts = [corpus_model.encode(self.corpus[s0:s0 + chunk], show_progress_bar=False, batch_size=self.batch_size,
                                         convert_to_tensor=True) for s0 in range(0, len(self.corpus), chunk)]
            return torch.cat(parts) if parts else q_emb[:0]
        from .index import CorpusShard

        shard = CorpusShard(q_emb.shape[1], max(len(self.corpus), 1), device=q_emb.device)
        for s0 in range(0, len(self.corpus), chunk):
            shard.add(corpus_model.encode(self.corpus[s0:s0 + chunk], show_progress_bar=False, batch_size=self.batch_size,
                                          convert_to_tensor=True))
        return shard

    def compute_metrices(self, model, corpus_model=None, corpus_embeddings=None, num_proc: int = None) -> Dict[str, dict]:
        if corpus_model is None:
            corpus_model = model
        max_k = max(max(self.mrr_at_k), max(self.ndcg_at_k), max(self.accuracy_at_k), max(self.precision_recall_at_k),
                    max(self.map_at_k))
        q_emb = model.encode(self.queries, show_progress_bar=self.show_progress_bar, batch_size=self.batch_size,
                             convert_to_tensor=True)
        if corpus_embeddings is None:
            corpus_embeddings = self._encode_corpus(corpus_model, q_emb)
        k = min(max_k, len(self.corpus))
        scores = {}
        for name in self.score_function_names:
            s, i = self._search(q_emb, corpus_embeddings, k, _SCORE_NAMES[name])
            s, i = s.cpu().tolist(), i.cpu().tolist()
            result_list = [[{"corpus_id": self.corpus_ids[ci], "score": sc} for sc, ci in zip(srow, irow) if ci >= 0]
                           for srow, irow in zip(s, i)]
            scores[name] = self.compute_metrics(result_list)
        return scores

    def compute_metrics(self, queries_result_list: List[List[dict]]) -> Dict[str, dict]:
        """:177-260 — per query: hits sorted by score, then the six metric families."""
        num_hits_at_k = {k: 0 for k in self.accuracy_at_k}
        precisions_at_k = {k: [] for k in self.precision_recall_at_k}
        recall_at_k = {k: [] for k in self.precision_recall_at_k}
        mrr = {k: 0 for k in self.mrr_at_k}
        ndcg = {k: [] for k in self.ndcg_at_k}
        avep = {k: [] for k in self.map_at_k}
        for query_itr, hits in enumerate(queries_result_list):
            rel = self.relevant_docs[self.queries_ids[query_itr]]
            top = sorted(hits, key=lambda x: x["score"], reverse=True)
            is_rel = [h["corpus_id"] in rel for h in top]
            for k in self.accuracy_at_k:
                num_hits_at_k[k] += 1 if any(is_rel[:k]) else 0
            for k in self.precision_recall_at_k:
                c = sum(is_rel[:k])
                precisions_at_k[k].append(c / k)
                recall_at_k[k].append(c / len(rel))
            for k in self.mrr_at_k:
                for rank, r in enumerate(is_rel[:k]):
                    if r:
                        mrr[k] += 1.0 / (rank + 1)
                        break
            for k in self.ndcg_at_k:
                ndcg[k].append(self.compute_dcg_at_k([1 if r else 0 for r in is_rel[:k]], k) /
                               self.compute_dcg_at_k([1] * len(rel), k))
            for k in self.map_at_k:
                c, sp = 0, 0.0
                for rank, r in enumerate(is_rel[:k]):
                    if r:
                        c += 1
                        sp += c / (rank + 1)
                avep[k].append(sp / min(k, len(rel)))
        nq = len(self.queries)
        return {"accuracy@k": {k: v / nq for k, v in num_hits_at_k.items()},
                "precision@k": {k: float(np.mean(v)) for k, v in precisions_at_k.items()},
                "recall@k": {k: float(np.mean(v)) for k, v in recall_at_k.items()},
                "ndcg@k": {k: float(np.mean(v)) for k, v in ndcg.items()},
                "mrr@k": {k: v / nq for k, v in mrr.items()},
                "map@k": {k: float(np.mean(v)) for k, v in avep.items()}}

    @staticmethod
    def compute_dcg_at_k(relevances, k):
        return sum(relevances[i] / np.log2(i + 2) for i in range(min(len(relevances), k)))
