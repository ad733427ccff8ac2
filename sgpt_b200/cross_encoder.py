"""Continuation log-likelihood scoring with the CUDA encoder — the SGPT cross-encoder path (SURVEY.md §8f row 4).

``LogLikelihoodScorer.loglikelihood_tokens`` has the contract of ``_loglikelihood_tokens``
(crossencoder/beir/sgptce.py:150-262): requests ``(cache_key, context_enc, continuation_enc)`` in, one float per request
out — the sum of ``log p(continuation token | everything before it)``.  What changes is where the work happens:

* the batch is packed ragged (no right padding with token 0 as at :201-204; with causal attention the padding never
  influenced the real positions anyway), one ``sgpt_forward`` call per batch;
* only the rows that predict continuation tokens go through ln_f + the LM head (``sgpt_lm_logprobs``: wgmma GEMM
  against the tied/untied LM-head matrix, fused log-softmax-gather kernel); the ``[batch, seq, vocab]`` fp32
  log-softmax tensor of :221 and its ``.cpu()`` copy never exist;
* per-request sums are taken on the device (``sgpt_segment_sum``), one small D2H per batch.

``GPTRanker`` and ``Rerank`` mirror sgptce.py:265-330 and ``beir.reranking.Rerank`` (as used at sgptce.py:352, 382-384).
"""
from __future__ import annotations

import collections
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .config import ModelConfig
from .encoder import Encoder


def encode(requests: Sequence[Tuple[str, str]], tokenizer) -> List[Tuple[Tuple[str, str], List[int], List[int]]]:
    """sgptce.py:76-90: requests are (continuation, context) = (query, prompted document)."""
    new_reqs = []
    for continuation, context in requests:
        if context == "":
            context_enc = [tokenizer.eos_token_id]
        else:
            context_enc = list(tokenizer.encode(context, add_special_tokens=False))
        continuation_enc = list(tokenizer.encode(continuation, add_special_tokens=False))
        new_reqs.append(((context, continuation), context_enc, continuation_enc))
    return new_reqs


class LogLikelihoodScorer:
    """GPT forward + LM head on one GPU.  `state_dict` is an HF ``*ForCausalLM`` (or base-model) state dict; the LM head is
    ``lm_head.weight`` (+ ``lm_head.bias`` for GPT-J) when present, else the tied token embedding."""

    def __init__(self, cfg: ModelConfig, state_dict: Dict[str, torch.Tensor], device="cuda:0", max_tokens: int = 32768,
                 max_batch: int = 256, rows_per_chunk: int = 1024, precision: str = "bf16"):
        self.encoder = Encoder(cfg, state_dict, device=device, max_tokens=max_tokens, max_batch=max_batch,
                               precision=precision)
        self.cfg, self.device = cfg, self.encoder.device
        sd = {(k[len("transformer."):] if k.startswith("transformer.") else k): v for k, v in state_dict.items()}
        emb_key = "word_embeddings.weight" if cfg.arch == "bloom" else "wte.weight"
        head = sd.get("lm_head.weight", sd[emb_key])
        if head.shape[1] != cfg.d_model:
            raise ValueError(f"LM head shape {tuple(head.shape)} does not match d_model {cfg.d_model}")
        self.vocab = int(head.shape[0])
        self.lm_head = head.detach().to(self.device, torch.bfloat16).contiguous()
        bias = sd.get("lm_head.bias")
        self.lm_bias = None if bias is None else bias.detach().to(self.device, torch.float32).contiguous()
        self.rows_per_chunk = int(rows_per_chunk)
        self._lib = _lib.lib()
        need = self._lib.sgpt_lm_logprobs_workspace_bytes(cfg.d_model, self.vocab, self.rows_per_chunk)
        self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)

    def close(self):
        self.encoder.close()

    # ------------------------------------------------------------------------------------------------------------
    def score_batch(self, inputs: Sequence[Sequence[int]], continuations: Sequence[Sequence[int]],
                    return_greedy: bool = False):
        """inputs[b]: the model input of request b (already truncated, last token dropped); continuations[b]: its
        continuation tokens, predicted by the LAST len(continuations[b]) positions of inputs[b] (sgptce.py:196-200).
        Returns fp32 [B] sums on the device (and, optionally, whether greedy decoding reproduces each continuation)."""
        B = len(inputs)
        lens = np.array([len(x) for x in inputs], dtype=np.int64)
        clens = np.array([len(c) for c in continuations], dtype=np.int64)
        if B == 0:
            return torch.empty(0, dtype=torch.float32, device=self.device)
        if np.any(lens <= 0) or np.any(clens <= 0):
            raise ValueError("empty input or continuation")  # the reference asserts both (:175-176)
        if np.any(clens > lens):
            raise ValueError("continuation longer than the (truncated) model input")
        T = int(lens.sum())
        enc = self.encoder
        if T > enc.max_tokens or B > enc.max_batch:
            raise ValueError(f"batch of {B} requests / {T} tokens exceeds the workspace ({enc.max_batch} / {enc.max_tokens})")
        if self.cfg.arch != "bloom" and int(lens.max()) > self.cfg.max_pos:
            raise ValueError(f"input length {int(lens.max())} exceeds max_position_embeddings {self.cfg.max_pos}")
        cu = np.zeros(B + 1, dtype=np.int32)
        np.cumsum(lens, out=cu[1:])
        ids = np.concatenate([np.asarray(x, dtype=np.int32) for x in inputs])
        pos = np.concatenate([np.arange(n, dtype=np.int32) for n in lens])
        rows = np.concatenate([np.arange(cu[b + 1] - clens[b], cu[b + 1], dtype=np.int32) for b in range(B)])
        targets = np.concatenate([np.asarray(c, dtype=np.int32) for c in continuations])
        if targets.min() < 0 or targets.max() >= self.vocab or ids.min() < 0 or ids.max() >= self.cfg.vocab:
            raise ValueError("token id outside the vocabulary")
        offsets = np.zeros(B + 1, dtype=np.int32)
        np.cumsum(clens, out=offsets[1:])
        M = int(offsets[-1])
        host = np.concatenate([ids, pos, cu, rows, targets, offsets])
        dev = torch.from_numpy(host).to(self.device)  # one H2D copy
        o = np.cumsum([0, T, T, B + 1, M, M])
        d_ids, d_pos, d_cu, d_rows, d_tgt, d_off = (dev[o[i]:o[i] + n] for i, n in enumerate((T, T, B + 1, M, M, B + 1)))
        token_lp = torch.empty(M, dtype=torch.float32, device=self.device)
        greedy = torch.empty(M, dtype=torch.int32, device=self.device) if return_greedy else None
        sums = torch.empty(B, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            st = _lib.current_stream()
            _lib.check(self._lib.sgpt_forward(enc._handle, d_ids.data_ptr(), d_pos.data_ptr(), d_cu.data_ptr(), B, T,
                                              int(lens.max()), st), "sgpt_forward")
            _lib.check(self._lib.sgpt_lm_logprobs(enc._handle, self.lm_head.data_ptr(), _lib.ptr(self.lm_bias), self.vocab,
                                                  d_rows.data_ptr(), d_tgt.data_ptr(), M, token_lp.data_ptr(),
                                                  _lib.ptr(greedy), self._ws.data_ptr(), self._ws.numel(),
                                                  self.rows_per_chunk, st), "sgpt_lm_logprobs")
            _lib.check(self._lib.sgpt_segment_sum(token_lp.data_ptr(), d_off.data_ptr(), B, sums.data_ptr(), st),
                       "sgpt_segment_sum")
        if not return_greedy:
            return sums
        same = (greedy == d_tgt).cpu().numpy()
        is_greedy = [bool(same[offsets[b]:offsets[b + 1]].all()) for b in range(B)]
        return sums, is_greedy

    def loglikelihood_tokens(self, requests: Sequence[Tuple[object, Sequence[int], Sequence[int]]], max_length: int,
                             batch_size: int = 64, instruction_len: int = 0) -> List[float]:
        """sgptce.py:150-262.  Requests with identical (context + continuation) tokens are scored once (the reference's
        ``Reorderer`` groups them, :104-113), longest first (:164-166); results come back in the original order."""
        groups: Dict[tuple, List[int]] = collections.OrderedDict()
        for i, (_, ctx, cont) in enumerate(requests):
            if len(ctx) == 0 or len(cont) == 0:
                raise AssertionError("empty context or continuation")  # :175-176
            if len(cont) > max_length:
                raise AssertionError(f"Got {len(cont)} but max len is only {max_length}")  # :177
            groups.setdefault((-(len(ctx) + len(cont)), tuple(ctx) + tuple(cont), len(cont)), []).append(i)
        order = sorted(groups, key=lambda k: (k[0], k[1]))
        res: List[Optional[float]] = [None] * len(requests)
        max_tok = self.encoder.max_tokens
        start = 0
        while start < len(order):
            inputs, conts, members = [], [], []
            tokens = 0
            while start < len(order) and len(inputs) < min(batch_size, self.encoder.max_batch):
                key = order[start]
                i0 = groups[key][0]
                _, ctx, cont = requests[i0]
                ctx, cont = list(ctx), list(cont)
                # instruction + left-truncated rest, last token dropped (:186-193)
                inp = (ctx[:instruction_len] + (ctx[instruction_len:] + cont)[-(max_length + 1 - instruction_len):])[:-1]
                if inputs and tokens + len(inp) > max_tok:
                    break
                inputs.append(inp)
                conts.append(cont)
                members.append(groups[key])
                tokens += len(inp)
                start += 1
            sums = self.score_batch(inputs, conts).cpu().tolist()
            for idxs, v in zip(members, sums):
                for i in idxs:
                    res[i] = float(v)
        return res  # type: ignore[return-value]


class GPTRanker:
    """sgptce.py:265-330: log-probability of the query given the prompted document."""

    def __init__(self, scorer: LogLikelihoodScorer, tokenizer, max_length: Optional[int] = None, use_prompt: bool = True,
                 prompt_doc: str = "{}\n", prompt_doc_start: str = "{}\n{}\n", fewshots="", batch_size: int = 64):
        self.scorer, self.tokenizer = scorer, tokenizer
        self.max_length = max_length if max_length is not None else scorer.cfg.max_pos  # :290-299
        self.prompt_doc, self.use_prompt = prompt_doc, use_prompt
        self.instruction_len = len(tokenizer.tokenize(prompt_doc[:prompt_doc.index("{")]))  # :304
        self.fewshots = fewshots
        if self.fewshots:
            self.fewshots = prompt_doc_start.format(self.fewshots[0], self.fewshots[1])  # :310
            self.instruction_len += len(tokenizer.tokenize(self.fewshots))
        self.batch_size = batch_size

    def predict(self, sentences: List[Tuple[str, str]], batch_size: int = None, **kwargs) -> List[float]:
        """sentences: [query, document] -> log p(query | prompt(document)) (:314-330)."""
        if self.use_prompt:
            sentences = [(query, self.fewshots + self.prompt_doc.format(doc)) for (query, doc) in sentences]
        encoded = encode(sentences, self.tokenizer)
        return self.scorer.loglikelihood_tokens(encoded, self.max_length, batch_size=self.batch_size,
                                                instruction_len=self.instruction_len)


class Rerank:
    """``beir.reranking.Rerank`` as used at sgptce.py:352 (restated from beir 0.2.3; the package is absent offline):
    re-score the top_k first-stage hits of every query with ``model.predict([[query, title + " " + text], ...])``."""

    def __init__(self, model, batch_size: int = 128, **kwargs):
        self.cross_encoder = model
        self.batch_size = batch_size
        self.rerank_results: Dict[str, Dict[str, float]] = {}

    def rerank(self, corpus: Dict[str, Dict[str, str]], queries: Dict[str, str], results: Dict[str, Dict[str, float]],
               top_k: int) -> Dict[str, Dict[str, float]]:
        sentence_pairs, pair_ids = [], []
        for query_id in results:
            hits = results[query_id]
            doc_ids = ([d for d, _ in sorted(hits.items(), key=lambda item: item[1], reverse=True)[:top_k]]
                       if len(hits) > top_k else list(hits))
            for doc_id in doc_ids:
                pair_ids.append([query_id, doc_id])
                text = (corpus[doc_id].get("title", "") + " " + corpus[doc_id].get("text", "")).strip()
                sentence_pairs.append([queries[query_id], text])
        scores = [float(s) for s in self.cross_encoder.predict(sentence_pairs, batch_size=self.batch_size)]
        self.rerank_results = {query_id: {} for query_id in results}
        for (qid, did), score in zip(pair_ids, scores):
            self.rerank_results[qid][did] = score
        return self.rerank_results
