"""Reads a saved sentence-transformers model directory of the reference's fork into what the CUDA encoder needs.

Mirrors ``SentenceTransformer._load_sbert_model`` (sentence_transformers/SentenceTransformer.py:903-936): ``modules.json``
lists ``{idx, name, path, type}`` entries; each module directory is parsed the way that module's own ``load`` does —

* ``models.Transformer``   (models/Transformer.py:158-175): HF ``config.json`` + weights + ``sentence_bert_config.json``
* ``models.Pooling``       (models/Pooling.py:173-185): ``config.json`` with the ``pooling_mode_*`` flags
* ``models.WeightedMeanPooling`` (models/WeightedMeanPooling.py:45-60): ``config.json`` + ``pytorch_model.bin``
  holding ``position_weights``
* ``models.Dense``         (models/Dense.py:51-68): ``config.json`` + ``pytorch_model.bin`` (``linear.weight/bias``)
* ``models.Asym``          (models/Asym.py:62-117): ``config.json`` {types, structure, parameters} + sub-directories
* ``models.Normalize``     (models/Normalize.py): no state

Everything here is host-side parsing (no CUDA): the result is a plain ``STModelSpec`` that ``SentenceEncoder.from_spec``
turns into device buffers.  Module kinds the GPT bi-encoders of the reference never use (CNN, LSTM, WordEmbeddings, ...)
raise ``NotImplementedError`` by name.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

from .config import ModelConfig

_SBERT_CONFIG_NAMES = ("sentence_bert_config.json", "sentence_roberta_config.json", "sentence_distilbert_config.json",
                       "sentence_camembert_config.json", "sentence_albert_config.json",
                       "sentence_xlm-roberta_config.json", "sentence_xlnet_config.json")  # Transformer.py:168


@dataclass
class DenseSpec:
    weight: torch.Tensor            # fp32 [out, in]
    bias: Optional[torch.Tensor]    # fp32 [out] or None
    activation: str                 # class path as written by Dense.get_config_dict
    key_name: str = "sentence_embedding"


@dataclass
class STModelSpec:
    hf_dir: str                                     # directory with the HF config / weights / tokenizer files
    config: Optional[ModelConfig] = None
    state_dict: Optional[Dict[str, torch.Tensor]] = None
    max_seq_length: Optional[int] = None
    do_lower_case: bool = False
    pooling: str = "mean"                           # "mean" | "weightedmean" | "lasttoken"
    position_weights: Optional[torch.Tensor] = None  # learnt WeightedMeanPooling table, fp32 [n]
    dense: List[DenseSpec] = field(default_factory=list)
    asym: Dict[str, List[DenseSpec]] = field(default_factory=dict)
    normalize: bool = False
    modules: List[Tuple[str, str]] = field(default_factory=list)  # (type, path) in order, for diagnostics


def _read_json(path: str) -> dict:
    with open(path, encoding="utf8") as f:
        return json.load(f)


def load_torch_weights(directory: str) -> Dict[str, torch.Tensor]:
    """``pytorch_model.bin`` (torch.save of a state dict) or ``model.safetensors`` in `directory`; sharded HF
    checkpoints (``*.index.json``) are concatenated."""
    for index_name, loader in (("model.safetensors.index.json", "safetensors"), ("pytorch_model.bin.index.json", "torch")):
        idx = os.path.join(directory, index_name)
        if os.path.exists(idx):
            out: Dict[str, torch.Tensor] = {}
            for shard in sorted(set(_read_json(idx)["weight_map"].values())):
                out.update(_load_one(os.path.join(directory, shard), loader))
            return out
    st = os.path.join(directory, "model.safetensors")
    if os.path.exists(st):
        return _load_one(st, "safetensors")
    pt = os.path.join(directory, "pytorch_model.bin")
    if os.path.exists(pt):
        return _load_one(pt, "torch")
    raise FileNotFoundError(f"{directory}: neither model.safetensors nor pytorch_model.bin found")


def _load_one(path: str, kind: str) -> Dict[str, torch.Tensor]:
    if kind == "safetensors":
        from safetensors.torch import load_file  # ships with transformers

        return load_file(path, device="cpu")
    return torch.load(path, map_location="cpu", weights_only=True)


def pooling_mode_from_config(cfg: dict) -> str:
    """Pooling config flags (models/Pooling.py:36-56) -> the single mode string the CUDA pooling kernel runs."""
    flags = {"cls": cfg.get("pooling_mode_cls_token", False), "max": cfg.get("pooling_mode_max_tokens", False),
             "mean": cfg.get("pooling_mode_mean_tokens", False),
             "mean_sqrt_len_tokens": cfg.get("pooling_mode_mean_sqrt_len_tokens", False),
             "weightedmean": cfg.get("pooling_mode_weightedmean_tokens", False),
             "lasttoken": cfg.get("pooling_mode_lasttoken", False)}
    on = [k for k, v in flags.items() if v]
    if len(on) != 1:
        raise NotImplementedError(f"Pooling with modes {on}: exactly one pooling mode is supported (no concatenation)")
    if on[0] not in ("mean", "weightedmean", "lasttoken"):
        raise NotImplementedError(f"pooling mode {on[0]!r} is not used by the SGPT bi-encoders and is not built")
    return on[0]


def _dense_from_dir(path: str) -> DenseSpec:
    cfg = _read_json(os.path.join(path, "config.json"))
    sd = load_torch_weights(path)
    w = sd["linear.weight"].float()
    if tuple(w.shape) != (cfg["out_features"], cfg["in_features"]):
        raise ValueError(f"{path}: Dense weight {tuple(w.shape)} does not match config {cfg}")
    b = sd["linear.bias"].float() if cfg.get("bias", True) and "linear.bias" in sd else None
    return DenseSpec(weight=w, bias=b, activation=cfg.get("activation_function", "torch.nn.modules.activation.Tanh"),
                     key_name=cfg.get("key_name", "sentence_embedding"))


def load_st_directory(path: str, load_weights: bool = True) -> STModelSpec:
    """Parse a sentence-transformers model directory.  With ``load_weights=False`` the (large) transformer state dict
    is skipped — config, pooling and heads are still read."""
    modules_json = os.path.join(path, "modules.json")
    if not os.path.exists(modules_json):
        raise FileNotFoundError(f"{path}: no modules.json (not a sentence-transformers model directory)")
    spec = STModelSpec(hf_dir=path)
    seen_transformer = False
    for entry in sorted(_read_json(modules_json), key=lambda e: e.get("idx", 0)):
        kind = entry["type"].rsplit(".", 1)[-1]
        mdir = os.path.join(path, entry["path"]) if entry["path"] else path
        spec.modules.append((entry["type"], entry["path"]))
        if kind == "Transformer":
            if seen_transformer:
                raise NotImplementedError("more than one Transformer module")
            seen_transformer = True
            spec.hf_dir = mdir
            for name in _SBERT_CONFIG_NAMES:
                if os.path.exists(os.path.join(mdir, name)):
                    sb = _read_json(os.path.join(mdir, name))
                    spec.max_seq_length = sb.get("max_seq_length")
                    spec.do_lower_case = bool(sb.get("do_lower_case", False))
                    break
            from transformers import AutoConfig

            spec.config = ModelConfig.from_hf(AutoConfig.from_pretrained(mdir))
            if load_weights:
                spec.state_dict = load_torch_weights(mdir)
        elif kind == "Pooling":
            spec.pooling = pooling_mode_from_config(_read_json(os.path.join(mdir, "config.json")))
        elif kind == "WeightedMeanPooling":
            cfg = _read_json(os.path.join(mdir, "config.json"))
            pw = load_torch_weights(mdir)
            spec.pooling = "weightedmean"
            spec.position_weights = pw["position_weights"].float().contiguous()
            if cfg.get("position_start", 0) != 0:
                raise NotImplementedError("WeightedMeanPooling with position_start != 0")
        elif kind == "Dense":
            d = _dense_from_dir(mdir)
            if d.key_name != "sentence_embedding":
                raise NotImplementedError(f"Dense on key {d.key_name!r} (only the pooled sentence embedding is built)")
            spec.dense.append(d)
        elif kind == "Asym":
            cfg = _read_json(os.path.join(mdir, "config.json"))
            for key, ids in cfg["structure"].items():
                stack = []
                for model_id in ids:
                    mtype = cfg["types"][model_id].rsplit(".", 1)[-1]
                    if mtype != "Dense":
                        raise NotImplementedError(f"Asym sub-module {mtype!r} (only Dense is built)")
                    stack.append(_dense_from_dir(os.path.join(mdir, model_id)))
                spec.asym[key] = stack
        elif kind == "Normalize":
            spec.normalize = True
        else:
            raise NotImplementedError(f"sentence-transformers module {entry['type']!r} is not part of the SGPT "
                                      "bi-encoder path and is not built")
    if not seen_transformer:
        raise ValueError(f"{path}: modules.json has no Transformer module")
    return spec
