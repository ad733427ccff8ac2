"""Embedder plug-ins with the reference's call surface, running on the CUDA encoder.

* ``CustomEmbedder``  — drop-in for biencoder/beir/beir_dense_retriever.py:106-348 (script / HF path): same constructor
  keywords, ``embed_batcher``, ``encode_queries(List[(qid, text)], ...)``, ``encode_corpus(List[(cid, {title,text})], ...)``.
* ``SentenceEncoder`` — the ``SentenceTransformer.encode`` signature of the vendored fork
  (sentence_transformers/SentenceTransformer.py:107-215) incl. length-sorted batching and specb bracket rules of
  models/Transformer.py:131-153; ``SentenceBERTBOSEOS`` mirrors custommodels/sentence_bert_asym.py:21-79 on top of it.

Tokenisation stays on the host (it is outside the measured path, SURVEY.md §8a row T0); anything with the HF tokenizer
methods used by the reference (``tokenize``, ``convert_tokens_to_ids``, ``encode``) works, so tests can plug a tiny
deterministic tokenizer in where no pretrained files are reachable.
"""
from __future__ import annotations

import logging
import os
import pathlib
import pickle
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .config import ModelConfig
from .encoder import Encoder

logger = logging.getLogger(__name__)

SPECB_QUE_BOS, SPECB_QUE_EOS = "[", "]"   # beir_dense_retriever.py:100-101
SPECB_DOC_BOS, SPECB_DOC_EOS = "{", "}"   # beir_dense_retriever.py:103-104

METHODS = ("mean", "weightedmean", "lasttoken", "meanmean", "lasttokenmean")  # BDR:238-301
USEB_METHODS = METHODS + ("learntmean",)  # biencoder/useb/useb_dense_retriever.py:218-305
ST_POOLING = ("mean", "weightedmean", "lasttoken")  # single-hidden-state modes of ST/models/Pooling.py


def _pad_batch(seqs: Sequence[Sequence[int]], pad_id: int) -> Tuple[np.ndarray, np.ndarray]:
    """tokenizer.pad(..., padding=True) (BDR:201): right-pad with pad_id, mask 1 on real tokens."""
    S = max(len(s) for s in seqs)
    ids = np.full((len(seqs), S), pad_id, dtype=np.int64)
    mask = np.zeros((len(seqs), S), dtype=np.int64)
    for i, s in enumerate(seqs):
        ids[i, :len(s)] = s
        mask[i, :len(s)] = 1
    return ids, mask



def split_by_token_budget(lengths, max_tokens: int, max_rows: int) -> List[Tuple[int, int]]:
    """Greedy consecutive row ranges [lo, hi) whose token sums fit `max_tokens` and row counts `max_rows`.  A single row
    longer than the budget is an error (the workspace must at least hold max_seq_length tokens)."""
    out, lo, tok = [], 0, 0
    for r, n in enumerate(int(x) for x in lengths):
        if n > max_tokens:
            raise ValueError(f"a sequence of {n} tokens exceeds the encoder workspace of {max_tokens} tokens")
        if tok + n > max_tokens or r - lo >= max_rows:
            out.append((lo, r))
            lo, tok = r, 0
        tok += n
    if len(lengths) > lo:
        out.append((lo, len(lengths)))
    return out

class CustomEmbedder:
    def __init__(self, model_name: str = "EleutherAI/gpt-neo-1.3B", batch_size: int = 250, device: str = "cuda:0",
                 save_emb: bool = False, reinit: bool = False, layeridx: int = -1, method: str = "mean",
                 dataset: str = "scifact", specb: bool = False, maxseqlen: Optional[int] = None, *,
                 config: Optional[ModelConfig] = None, state_dict: Optional[Dict[str, torch.Tensor]] = None,
                 tokenizer=None, max_tokens: Optional[int] = None, **kwargs):
        """Keywords up to ``maxseqlen`` are the reference's (BDR:107-120).  ``config``/``state_dict``/``tokenizer`` let a
        caller hand the model over directly (no hub access offline); otherwise they are loaded with HF
        ``AutoConfig``/``AutoModel``/``AutoTokenizer`` from ``model_name`` exactly like BDR:123,138."""
        if method not in METHODS:
            raise NotImplementedError(f"pooling method {method!r}: built: {METHODS} (poolout needs a pooler head the "
                                      "GPT models of the reference do not have, BDR:303-304)")
        self.model_name = model_name
        self.save_emb = save_emb
        # BDR:155-156 (the reference creates the directory unconditionally; here only when something will be written)
        self.base_path = f"embeddings/{model_name.split('/')[-1]}/{method}/{dataset}"
        if save_emb:
            pathlib.Path(self.base_path).mkdir(parents=True, exist_ok=True)
        if state_dict is None:
            from transformers import AutoModel  # real checkpoint path

            hf = AutoModel.from_pretrained(model_name, **kwargs)
            if reinit:
                hf.init_weights()  # BDR:124-126
            config = ModelConfig.from_hf(hf.config)
            state_dict = hf.state_dict()
        if config is None:
            raise ValueError("config is required when state_dict is given")
        if tokenizer is None:
            from transformers import AutoTokenizer

            tokenizer = AutoTokenizer.from_pretrained(model_name)
            if "gpt" in model_name.lower():
                tokenizer.pad_token = tokenizer.eos_token  # BDR:140-141
        self.tokenizer = tokenizer
        self.config = config
        self.max_token_len = maxseqlen if maxseqlen else config.max_pos  # BDR:128
        if "bert" in model_name:
            self.max_token_len -= 2  # BDR:131-133
        if specb:
            self.max_token_len -= 2  # leave two tokens for the brackets, BDR:134-136
        self.batch_size = batch_size
        self.layeridx = layeridx
        self.method = method
        self.specb = specb
        if specb:
            self.bos_token_q = list(tokenizer.encode(SPECB_QUE_BOS))  # BDR:150-153
            self.eos_token_q = list(tokenizer.encode(SPECB_QUE_EOS))
            self.bos_token_d = list(tokenizer.encode(SPECB_DOC_BOS))
            self.eos_token_d = list(tokenizer.encode(SPECB_DOC_EOS))
        pad = getattr(tokenizer, "pad_token_id", None)
        self.pad_id = int(pad) if pad is not None else 0
        seq_cap = self.max_token_len + (2 if specb else 0)
        self.encoder = Encoder(config, state_dict, device=device,
                               max_tokens=max_tokens or max(batch_size * min(seq_cap, 512), 8192),
                               max_batch=max(batch_size, 1))
        self.device = self.encoder.device

    # ------------------------------------------------------------------------------------------------------------
    def tokenize_batch(self, batch: Sequence[str], is_query: bool) -> Tuple[np.ndarray, np.ndarray]:
        """Host token preparation of ``embed`` (BDR:164-201): newline -> space, tokenize, truncate to max_token_len,
        optional specb brackets with mask 1, right-pad."""
        seqs = []
        docs_truncated = toks_truncated = total = 0
        batch = [txt.replace("\n", " ") for txt in batch]  # BDR:166
        if getattr(self.tokenizer, "is_fast", False) and callable(self.tokenizer):
            # a fast tokenizer encodes the whole batch in one native call; same ids as tokenize + convert_tokens_to_ids
            all_tokens = self.tokenizer(list(batch), add_special_tokens=False)["input_ids"]
        else:
            all_tokens = [self.tokenizer.convert_tokens_to_ids(self.tokenizer.tokenize(txt)) for txt in batch]  # BDR:169-170
        for tokens in all_tokens:
            n = len(tokens)
            total += n
            if n > self.max_token_len:
                docs_truncated += 1
                toks_truncated += n - self.max_token_len
            elif n == 0:
                raise ValueError("Empty items should be cleaned prior to running")  # BDR:180-181
            ids = list(tokens[: self.max_token_len])  # GPT tokenizers add no special tokens in prepare_for_model
            if self.specb:
                ids = (self.bos_token_q + ids + self.eos_token_q) if is_query else (self.bos_token_d + ids + self.eos_token_d)
            seqs.append(ids)
        if docs_truncated:
            logger.warning(f"Truncated {docs_truncated} out of {len(batch)} documents by {toks_truncated} out of {total}.")
        return _pad_batch(seqs, self.pad_id)

    def embed_texts(self, sentences: Sequence[str], is_query: bool) -> torch.Tensor:
        """All sentences -> fp32 [n, D] on the device, in the given order (batches of self.batch_size, BDR:227-229)."""
        out = torch.empty((len(sentences), self.config.d_model), dtype=torch.float32, device=self.device)
        for i in range(0, len(sentences), self.batch_size):
            ids, mask = self.tokenize_batch(sentences[i:i + self.batch_size], is_query)
            # the reference simply runs whatever a batch holds (BDR:205); the workspace here is sized in tokens, so a
            # batch of long documents (DRES sorts longest first, XS:66-71) is cut greedily into sub-batches that fit
            for lo, hi in split_by_token_budget(mask.sum(axis=1), self.encoder.max_tokens, self.encoder.max_batch):
                out[i + lo:i + hi] = self.encoder.encode_tokens(ids[lo:hi], mask[lo:hi], method=self.method,
                                                                layer_idx=self.layeridx)
        return out

    def embed_batcher(self, texts: List[Tuple[str, str]], is_query: bool, out_name=None, **kwargs) -> Dict[str, np.ndarray]:
        """{id: embedding} like BDR:225-314 (one D2H copy for the whole list instead of per-row .numpy()); with
        save_emb the dict is pickled to `out_name` (BDR:311-312)."""
        ids, sentences = zip(*texts) if texts else ((), ())
        emb = self.embed_texts(list(sentences), is_query).cpu().numpy()
        all_embeddings = {i: e for i, e in zip(ids, emb)}
        assert len(texts) == len(all_embeddings)  # BDR:309 (duplicate ids collapse, exactly as upstream)
        if self.save_emb and out_name:
            with open(out_name, "wb") as f:
                pickle.dump(all_embeddings, f)
        return all_embeddings

    def _cached(self, path: str, ids: Sequence[str]) -> Optional[np.ndarray]:
        """The pickle-per-chunk embedding cache (BDR:319-323, 336-339): a {id: embedding} dict written by an earlier
        save_emb run is used whenever the file exists, whatever save_emb says now — like upstream."""
        if not os.path.exists(path):
            return None
        with open(path, "rb") as f:
            embeddings = pickle.load(f)
        return np.array([embeddings[i] for i in ids])  # order given, BDR:326 / :344

    def encode_queries(self, queries: List[Tuple[str, str]], batch_size: int = None, convert_to_tensor: bool = False,
                       **kwargs) -> Union[np.ndarray, torch.Tensor]:
        """BDR:316-330: rows in the order given.  convert_to_tensor=True keeps the result on the device."""
        path = f"{self.base_path}_queries.pickle"
        cached = self._cached(path, [qid for (qid, _) in queries])
        if cached is not None:
            emb = torch.from_numpy(cached).to(self.device) if convert_to_tensor else cached
        elif self.save_emb:
            d = self.embed_batcher(queries, is_query=True, out_name=path)
            emb = np.array([d[qid] for (qid, _) in queries])
            emb = torch.from_numpy(emb).to(self.device) if convert_to_tensor else emb
        else:
            emb = self.embed_texts([t for (_, t) in queries], is_query=True)
            emb = emb if convert_to_tensor else emb.cpu().numpy()
        logger.info(f"Produced embeddings of shape {tuple(emb.shape)}")
        return emb

    def encode_corpus(self, corpus: List[Tuple[str, Dict[str, str]]], batch_size: int = None, batch_num="",
                      convert_to_tensor: bool = False, **kwargs) -> Union[np.ndarray, torch.Tensor]:
        """BDR:332-348: text = (title + " " + text).strip() when a title key exists (BDR:341)."""
        path = f"{self.base_path}_corpus{batch_num}.pickle"
        cached = self._cached(path, [cid for (cid, _) in corpus])
        if cached is not None:
            emb = torch.from_numpy(cached).to(self.device) if convert_to_tensor else cached
        else:
            texts = [((d["title"] + " " + d["text"]).strip() if "title" in d else d["text"].strip()) for (_, d) in corpus]
            if self.save_emb:
                dd = self.embed_batcher(list(zip([cid for (cid, _) in corpus], texts)), is_query=False, out_name=path)
                emb = np.array([dd[cid] for (cid, _) in corpus])
                emb = torch.from_numpy(emb).to(self.device) if convert_to_tensor else emb
            else:
                emb = self.embed_texts(texts, is_query=False)
                emb = emb if convert_to_tensor else emb.cpu().numpy()
        logger.info(f"Produced embeddings of shape {tuple(emb.shape)}")
        return emb

    # ---- USEB flavour (biencoder/useb/useb_dense_retriever.py:76-309) ---------------------------------------------
    def encode(self, sentences: Sequence[str], method: str = "mean", show_progress_bar: bool = False,
               dataset_name=None, add_name: str = "", idx=None, **kwargs) -> List[List[float]]:
        """``CustomEmbedder.encode`` of the USEB script: plain sentences (no brackets), the pooling ``method`` chosen
        per call, result as a list of Python float lists (UDR:307).  ``learntmean`` (UDR:252-268) reads the learnt
        position weights from ``{model_name}/1_WeightedMeanPooling/pytorch_model.bin``.  The per-batch pickle of ALL
        hidden states (UDR:189-211) is not written: nothing downstream of this call ever needs them again."""
        if method not in USEB_METHODS:
            raise NotImplementedError(f"pooling method {method!r}: built: {USEB_METHODS}")
        if method == "learntmean":
            if getattr(self, "_learnt_weights", None) is None:
                from .st_loader import load_torch_weights

                self._learnt_weights = load_torch_weights(
                    os.path.join(self.model_name, "1_WeightedMeanPooling"))["position_weights"].float()
            self.encoder.set_position_weights(self._learnt_weights)
        out: List[List[float]] = []
        specb, self.specb = self.specb, False  # the USEB script has no bracket mode
        try:
            for i in range(0, len(sentences), self.batch_size):
                ids, mask = self.tokenize_batch(sentences[i:i + self.batch_size], is_query=True)
                emb = self.encoder.encode_tokens(ids, mask, method="weightedmean" if method == "learntmean" else method,
                                                 layer_idx=self.layeridx)
                out.extend(emb.cpu().numpy().tolist())
        finally:
            self.specb = specb
            if method == "learntmean":
                self.encoder.set_position_weights(None)
        assert len(sentences) == len(out)
        return out


class SentenceEncoder:
    """``SentenceTransformer.encode`` for a [Transformer -> Pooling | WeightedMeanPooling (-> Dense | Asym)* (-> Normalize)]
    SGPT model on the CUDA encoder (module pipeline of sentence_transformers/SentenceTransformer.py:98, run as one
    ``sgpt_encode`` call + ``sgpt_dense`` per head)."""

    def __init__(self, config: ModelConfig, state_dict: Dict[str, torch.Tensor], tokenizer, device: str = "cuda:0",
                 pooling: str = "weightedmean", max_seq_length: int = 300, batch_capacity: int = 256,
                 max_tokens: Optional[int] = None, position_weights: Optional[torch.Tensor] = None,
                 heads: Optional[Sequence] = None, asym=None, normalize: bool = False, do_lower_case: bool = False):
        if pooling not in ST_POOLING:
            raise NotImplementedError(f"pooling mode {pooling!r} not in {ST_POOLING}")
        if position_weights is not None and pooling != "weightedmean":
            raise ValueError("position_weights need pooling='weightedmean'")
        self.config, self.tokenizer, self.pooling = config, tokenizer, pooling
        self.max_seq_length = max_seq_length
        self.do_lower_case = do_lower_case
        self.encoder = Encoder(config, state_dict, device=device,
                               max_tokens=max_tokens or batch_capacity * max_seq_length, max_batch=batch_capacity)
        self.device = self.encoder.device
        if position_weights is not None:
            if position_weights.numel() < max_seq_length:
                raise ValueError(f"{position_weights.numel()} position weights < max_seq_length {max_seq_length}")
            self.encoder.set_position_weights(position_weights)
        self.heads = list(heads or [])   # DenseHead stack applied to every input (models/Dense.py)
        self.asym = asym                 # AsymHeads: stack chosen by the input dict key (models/Asym.py)
        self.normalize = bool(normalize)  # trailing models/Normalize.py module
        pad = getattr(tokenizer, "pad_token_id", None)
        self.pad_id = int(pad) if pad is not None else 0
        # specb/speca state installed by SentenceBERTBOSEOS (models/Transformer.py attributes of the same names)
        self.bos_spec_token_q = self.bos_spec_token_d = self.eos_spec_token_q = self.eos_spec_token_d = None
        self.bos_spec_token_q_rep = self.bos_spec_token_d_rep = None
        self.replace_bos = False

    # ---- construction from a saved sentence-transformers directory -----------------------------------------------
    @classmethod
    def from_spec(cls, spec, tokenizer=None, device: str = "cuda:0", batch_capacity: int = 256,
                  max_seq_length: Optional[int] = None, max_tokens: Optional[int] = None) -> "SentenceEncoder":
        """Build from ``st_loader.load_st_directory(path)``; the tokenizer defaults to ``AutoTokenizer`` of the model
        directory (models/Transformer.py:40)."""
        from .heads import AsymHeads, DenseHead

        if spec.state_dict is None:
            raise ValueError("spec has no transformer weights (load_weights=False?)")
        if tokenizer is None:
            from transformers import AutoTokenizer

            tokenizer = AutoTokenizer.from_pretrained(spec.hf_dir)
        msl = max_seq_length or spec.max_seq_length
        if msl is None:  # Transformer.py:43-46
            msl = min(spec.config.max_pos, getattr(tokenizer, "model_max_length", spec.config.max_pos))
        mk = lambda d: DenseHead(d.weight, d.bias, d.activation, device=device)  # noqa: E731
        heads = [mk(d) for d in spec.dense]
        asym = AsymHeads({k: [mk(d) for d in v] for k, v in spec.asym.items()}) if spec.asym else None
        return cls(spec.config, spec.state_dict, tokenizer, device=device, pooling=spec.pooling, max_seq_length=msl,
                   batch_capacity=batch_capacity, max_tokens=max_tokens, position_weights=spec.position_weights,
                   heads=heads, asym=asym, normalize=spec.normalize, do_lower_case=spec.do_lower_case)

    @classmethod
    def from_pretrained(cls, model_path: str, device: str = "cuda:0", **kwargs) -> "SentenceEncoder":
        """``SentenceTransformer(model_path)`` for a local model directory (SentenceTransformer.py:90-93): a
        ``modules.json`` directory is read module by module; a plain HF directory becomes Transformer + mean Pooling
        (``_load_auto_model``, :893-900)."""
        import os

        from . import st_loader

        if os.path.exists(os.path.join(model_path, "modules.json")):
            spec = st_loader.load_st_directory(model_path)
        else:
            from transformers import AutoConfig

            spec = st_loader.STModelSpec(hf_dir=model_path, pooling="mean",
                                         config=ModelConfig.from_hf(AutoConfig.from_pretrained(model_path)),
                                         state_dict=st_loader.load_torch_weights(model_path))
        return cls.from_spec(spec, device=device, **kwargs)

    def get_sentence_embedding_dimension(self) -> int:
        if self.heads:
            return self.heads[-1].out_features
        return self.config.d_model

    def _text_length(self, text) -> int:
        """SentenceTransformer.py:600-614: dict -> length of its first value; str -> len; list -> summed lengths."""
        if isinstance(text, dict):
            return len(next(iter(text.values())))
        if not hasattr(text, "__len__"):
            return 1
        if len(text) == 0 or isinstance(text, str) or isinstance(text[0], int):
            return len(text)
        return sum(len(t) for t in text)

    def tokenize(self, texts: Sequence) -> Tuple[np.ndarray, np.ndarray]:
        """models/Transformer.py:90-153: strip, (lower-case), tokenize with truncation, bracket rules, right-pad.
        ``{key: text}`` inputs contribute their text (the key selects the Asym stack in ``encode``)."""
        texts = [next(iter(t.values())) if isinstance(t, dict) else t for t in texts]
        texts = [str(s).strip() for s in texts]
        if self.do_lower_case:
            texts = [s.lower() for s in texts]  # :116-118
        spec = None not in (self.bos_spec_token_q, self.eos_spec_token_q, self.bos_spec_token_d, self.eos_spec_token_d)
        limit = self.max_seq_length - 2 if spec else self.max_seq_length  # :135
        if getattr(self.tokenizer, "is_fast", False) and callable(self.tokenizer):
            # one batched call like the reference (Transformer.py:127 / :132-135) — a fast tokenizer encodes the whole
            # batch in native code instead of one Python call per text
            batch_ids = [list(x) for x in self.tokenizer(texts, padding=False, truncation="longest_first",
                                                        max_length=limit)["input_ids"]]
        else:
            batch_ids = [list(self.tokenizer.encode(t))[:limit] for t in texts]
        seqs = []
        for t, ids in zip(texts, batch_ids):
            if spec:
                if ids and ids[0] == self.bos_spec_token_d:
                    if self.replace_bos:
                        ids[0] = self.bos_spec_token_d_rep
                    ids.append(self.eos_spec_token_d)
                elif ids and ids[0] == self.bos_spec_token_q:
                    if self.replace_bos:
                        ids[0] = self.bos_spec_token_q_rep
                    ids.append(self.eos_spec_token_q)
                else:
                    raise ValueError(f"Did not find BOS Token in sequence: {t[:40]!r}")  # :148
            seqs.append(ids)
        return _pad_batch(seqs, self.pad_id)

    @staticmethod
    def _text_key(sentence) -> Optional[str]:
        return next(iter(sentence.keys())) if isinstance(sentence, dict) else None

    def encode(self, sentences: Union[str, List[str]], batch_size: int = 32, show_progress_bar: bool = None,
               output_value: str = "sentence_embedding", convert_to_numpy: bool = True, convert_to_tensor: bool = False,
               device: str = None, normalize_embeddings: bool = False, num_proc=None):
        """SentenceTransformer.py:107-215: sort by -len, encode in batches, undo the sort; str in -> 1-D out."""
        if output_value != "sentence_embedding":
            raise NotImplementedError("only output_value='sentence_embedding' is built")
        if convert_to_tensor:
            convert_to_numpy = False
        input_was_string = isinstance(sentences, (str, dict)) or not hasattr(sentences, "__len__")
        if input_was_string:
            sentences = [sentences]
        post = bool(self.heads) or self.asym is not None
        # Normalize is the last module of the pipeline: it can only be fused into the pooling kernel when no head follows
        fuse_norm = (self.normalize or normalize_embeddings) and not post
        order = np.argsort([-self._text_length(s) for s in sentences], kind="stable")
        out = None
        for start in range(0, len(sentences), batch_size):
            idx = order[start:start + batch_size]
            batch = [sentences[i] for i in idx]
            ids, mask = self.tokenize(batch)
            # the learnt WeightedMeanPooling always clamps its denominator (:34), like Pooling.py:122
            emb = self.encoder.encode_tokens(ids, mask, method=self.pooling, clamp=True, normalize=fuse_norm)
            if post:
                from .heads import apply_heads, normalize_rows_

                emb = apply_heads(emb, self.heads)
                if self.asym is not None:
                    key = self._text_key(batch[0])  # Asym.py:50-52: text_keys[0] selects the stack for the batch
                    if key is not None:
                        emb = self.asym.apply(emb, key)
                if self.normalize or normalize_embeddings:
                    emb = normalize_rows_(emb.contiguous())  # SentenceTransformer.py:248-249
            if out is None:
                out = torch.empty((len(sentences), emb.shape[1]), dtype=torch.float32, device=self.device)
            elif out.shape[1] != emb.shape[1]:
                raise ValueError("inputs with different Asym text keys produce different embedding sizes; "
                                 "encode them in separate calls (Asym.py: mixed types cannot be encoded)")
            out[torch.as_tensor(idx, device=self.device)] = emb
        if out is None:
            out = torch.empty((0, self.get_sentence_embedding_dimension()), dtype=torch.float32, device=self.device)
        if convert_to_tensor:
            res = out
        elif convert_to_numpy:
            res = out.cpu().numpy()
        else:
            res = list(out)
        return res[0] if input_was_string else res


class SentenceBERTAsym:
    """custommodels/sentence_bert_asym.py:8-19: queries are passed as ``{'QRY': text}``, documents as
    ``{'DOCPOS': text}`` so that the model's Asym module applies the matching Dense stack."""

    def __init__(self, model: SentenceEncoder, sep: str = " "):
        self.model, self.sep = model, sep

    def encode_queries(self, queries: List[str], batch_size: int = 16, **kwargs):
        return self.model.encode([{"QRY": q} for q in queries], batch_size=batch_size, **kwargs)

    def encode_corpus(self, corpus: List[Dict[str, str]], batch_size: int = 8, **kwargs):
        # (the reference leaves title-less documents as bare strings, :18 — i.e. without a head; kept as is)
        sentences = [{"DOCPOS": (doc["title"] + self.sep + doc["text"]).strip()} if "title" in doc else doc["text"].strip()
                     for doc in corpus]
        return self.model.encode(sentences, batch_size=batch_size, **kwargs)


class SentenceBERTBOSEOS:
    """custommodels/sentence_bert_asym.py:21-79 on top of SentenceEncoder.  specb: the '[SOS]'/'{SOS}' markers are
    replaced by the bracket ids and the closing bracket is appended; speca: the markers are kept and '[EOS]'/'{EOS}'
    are appended (the four added tokens must exist in the tokenizer and the checkpoint's embedding matrix, :56-58)."""

    def __init__(self, model: SentenceEncoder, sep: str = " ", specb: bool = False, sos_q: int = None, sos_d: int = None,
                 speca: bool = False):
        self.model, self.sep, self.specb, self.speca = model, sep, specb, speca
        tok = model.tokenizer
        vocab = model.encoder.cfg.vocab

        def first(text, must_embed=False):
            """The id of a marker that must be ONE token (the reference registers the markers with add_tokens,
            sentence_bert_asym.py:36-38, 56-58; without that '[SOS]' would tokenize to '[' + ... and silently pass)."""
            ids = list(tok.encode(text, add_special_tokens=False))
            if len(ids) != 1:
                raise ValueError(f"{text!r} tokenizes to {len(ids)} ids {ids[:4]}; it must be a single (added) token")
            if must_embed and not 0 <= ids[0] < vocab:
                raise ValueError(f"token {text!r} has id {ids[0]} but the checkpoint's embedding matrix has {vocab} rows "
                                 "(speca needs a checkpoint trained with the added tokens, sentence_bert_asym.py:56-58)")
            return ids[0]

        if (specb or speca) and hasattr(tok, "add_tokens"):
            # sentence_bert_asym.py:36-37 / :56-57.  (resize_token_embeddings has no analogue: specb replaces the marker
            # ids before the embedding lookup, speca requires them inside the checkpoint's matrix — checked below.)
            tok.add_tokens(["[SOS]", "{SOS}"] if specb else ["[SOS]", "[EOS]", "{SOS}", "{EOS}"], special_tokens=True)
        if specb:
            model.bos_spec_token_q = sos_q if sos_q is not None else first("[SOS]")
            model.bos_spec_token_d = sos_d if sos_d is not None else first("{SOS}")
            model.bos_spec_token_q_rep = first("[")
            model.eos_spec_token_q = first("]")
            model.bos_spec_token_d_rep = first("{")
            model.eos_spec_token_d = first("}")
            model.replace_bos = True
        elif speca:
            model.bos_spec_token_q = sos_q if sos_q is not None else first("[SOS]", must_embed=True)
            model.eos_spec_token_q = first("[EOS]", must_embed=True)
            model.bos_spec_token_d = sos_d if sos_d is not None else first("{SOS}", must_embed=True)
            model.eos_spec_token_d = first("{EOS}", must_embed=True)

    def encode_queries(self, queries: List[str], batch_size: int = 16, **kwargs):
        if self.specb or self.speca:
            queries = ["[SOS]" + q for q in queries]
        return self.model.encode(queries, batch_size=batch_size, **kwargs)

    def encode_corpus(self, corpus: List[Dict[str, str]], batch_size: int = 8, **kwargs):
        pre = "{SOS}" if (self.specb or self.speca) else ""
        sentences = [(pre + doc["title"] + self.sep + doc["text"]).strip() if "title" in doc else pre + doc["text"].strip()
                     for doc in corpus]
        return self.model.encode(sentences, batch_size=batch_size, **kwargs)
