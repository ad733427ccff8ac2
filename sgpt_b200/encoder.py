"""Device-side encoder: HF-layout weights -> packed bf16 device buffers -> one C call per batch.

Replaces ``AutoModel.from_pretrained(...).to(device)`` + ``self.model(**batch_tokens, output_hidden_states=True)`` +
the pooling block of the reference (biencoder/beir/beir_dense_retriever.py:123, :205, :233-304; ST path:
sentence_transformers/models/Transformer.py:72 + models/Pooling.py:85-168).  PyTorch is used for device memory,
streams and host<->device copies only; all arithmetic runs in libsgpt_b200.so.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .config import ModelConfig

POOL_MODES = {"mean": _lib.POOL_MEAN, "weightedmean": _lib.POOL_WEIGHTEDMEAN, "lasttoken": _lib.POOL_LASTTOKEN,
              "meanmean": _lib.POOL_MEANMEAN, "lasttokenmean": _lib.POOL_LASTTOKENMEAN}


def pack_ragged(input_ids, attention_mask) -> Tuple[np.ndarray, np.ndarray, np.ndarray, int]:
    """[B,S] padded ids + mask (host) -> ragged layout: packed ids[T], padded-row index pos[T], cu_seqlens[B+1].

    `pos` is the index of the token inside its PADDED row: that is what both the position embedding
    (HF:gpt_neo/modeling_gpt_neo.py:455-463: position_ids = arange(S)) and the pooling weights
    (beir_dense_retriever.py:259-265: arange(1, S+1)) are functions of, for left- or right-padded rows alike.
    Each row's mask must be one contiguous run of ones (what tokenizer.pad produces, BDR:201).
    """
    ids = np.asarray(input_ids)
    mask = np.asarray(attention_mask).astype(bool)
    if ids.ndim != 2 or mask.shape != ids.shape:
        raise ValueError(f"input_ids / attention_mask must be [B,S] of equal shape, got {ids.shape} and {mask.shape}")
    B, S = ids.shape
    lens = mask.sum(axis=1)
    first = np.where(lens > 0, mask.argmax(axis=1), 0)
    last = np.where(lens > 0, S - 1 - mask[:, ::-1].argmax(axis=1), -1)
    if np.any((last - first + 1)[lens > 0] != lens[lens > 0]):
        raise ValueError("attention_mask rows must be contiguous runs of ones (left- or right-padded)")
    cu = np.zeros(B + 1, dtype=np.int32)
    np.cumsum(lens, out=cu[1:])
    flat = mask.reshape(-1)
    packed_ids = ids.reshape(-1)[flat].astype(np.int32)
    pos = np.broadcast_to(np.arange(S, dtype=np.int32), (B, S)).reshape(-1)[flat]
    return packed_ids, np.ascontiguousarray(pos), cu, int(lens.max()) if B else 0


class Encoder:
    """GPT encoder + pooling on one GPU.

    state_dict: tensors keyed like the HF base model's ``state_dict()`` for the architecture — ``GPTNeoModel``
    (``wte.weight``, ``h.0.attn.attention.q_proj.weight``, ...), ``GPTJModel`` (``h.0.attn.q_proj.weight``, ``mlp.fc_in``)
    or ``BloomModel`` (``word_embeddings.weight``, ``h.0.self_attention.query_key_value.weight``, ...); a
    ``transformer.`` prefix as in the ``*ForCausalLM`` checkpoints is accepted.  Linear weights are stored in bf16,
    LayerNorm parameters and biases in fp32.

    precision: ``"bf16"`` (default) or ``"fp8"``: every linear layer of every block runs as an e4m3 x e4m3 GEMM with
    per-output-channel weight scales and per-token activation scales (include/sgpt_b200.h, fp8 linear layers).  The bf16
    linear weights are quantized on the device by the library and only the e4m3 copies and their scales are kept.
    """

    def __init__(self, cfg: ModelConfig, state_dict: Dict[str, torch.Tensor], device="cuda:0", max_tokens: int = 32768,
                 max_batch: int = 1024, precision: str = "bf16"):
        if precision not in ("bf16", "fp8"):
            raise ValueError(f"precision must be 'bf16' or 'fp8', got {precision!r}")
        self.precision = precision
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("sgpt_b200.Encoder needs a CUDA device; there is no CPU path")
        self.max_tokens = int(max_tokens)
        self.max_batch = int(max_batch)
        self._lib = _lib.lib()
        self._keep = []  # device tensors the C handle borrows
        sd = {(k[len("transformer."):] if k.startswith("transformer.") else k): v for k, v in state_dict.items()}

        def dev(t, dtype):
            x = t.detach().to(device=self.device, dtype=dtype).contiguous()
            self._keep.append(x)
            return x

        def p32(name):
            return dev(sd[name], torch.float32).data_ptr() if name in sd else None

        def p16(t):
            return dev(t, torch.bfloat16).data_ptr()

        fp8 = precision == "fp8"
        fp8_layers = (_lib.Fp8LayerWeightsC * cfg.n_layer)()

        def plin(i, name, t):
            """Linear weight `name` of layer i: its bf16 device pointer, or with fp8 None after the bf16 values the bf16
            path would store have been quantized per output channel into fp8_layers[i].w_<name> / s_<name>."""
            if not fp8:
                return p16(t)
            w16 = t.detach().to(device=self.device, dtype=torch.bfloat16).contiguous()
            q = torch.empty(w16.shape, dtype=torch.uint8, device=self.device)
            sc = torch.empty(w16.shape[0], dtype=torch.float32, device=self.device)
            _lib.check(self._lib.sgpt_quantize_rows_fp8(w16.data_ptr(), q.data_ptr(), sc.data_ptr(), w16.shape[0],
                                                        w16.shape[1], _lib.current_stream()), "sgpt_quantize_rows_fp8")
            self._keep += [q, sc]
            setattr(fp8_layers[i], "w_" + name, q.data_ptr())
            setattr(fp8_layers[i], "s_" + name, sc.data_ptr())
            return None

        with torch.cuda.device(self.device):
            d, H, hd = cfg.d_model, cfg.n_head, cfg.head_dim
            layers = (_lib.LayerWeightsC * cfg.n_layer)()
            mw = _lib.ModelWeightsC()
            if cfg.arch == "gpt_neo":  # keys of HF GPTNeoModel.state_dict()
                wte, wpe = dev(sd["wte.weight"], torch.bfloat16), dev(sd["wpe.weight"], torch.bfloat16)
                if wte.shape != (cfg.vocab, d) or wpe.shape != (cfg.max_pos, d):
                    raise ValueError(f"embedding shapes {tuple(wte.shape)}, {tuple(wpe.shape)} do not match the config")
                mw.wte, mw.wpe = wte.data_ptr(), wpe.data_ptr()
                for i in range(cfg.n_layer):
                    p, lw = f"h.{i}.", layers[i]
                    a = p + "attn.attention."
                    lw.ln1_g, lw.ln1_b = p32(p + "ln_1.weight"), p32(p + "ln_1.bias")
                    lw.w_qkv = plin(i, "qkv", torch.cat([sd[a + "q_proj.weight"], sd[a + "k_proj.weight"],
                                                         sd[a + "v_proj.weight"]], 0))
                    if (a + "q_proj.bias") in sd:
                        lw.b_qkv = dev(torch.cat([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]], 0),
                                       torch.float32).data_ptr()
                    lw.w_o, lw.b_o = plin(i, "o", sd[a + "out_proj.weight"]), p32(a + "out_proj.bias")
                    lw.ln2_g, lw.ln2_b = p32(p + "ln_2.weight"), p32(p + "ln_2.bias")
                    lw.w_fc, lw.b_fc = plin(i, "fc", sd[p + "mlp.c_fc.weight"]), p32(p + "mlp.c_fc.bias")
                    lw.w_proj, lw.b_proj = plin(i, "proj", sd[p + "mlp.c_proj.weight"]), p32(p + "mlp.c_proj.bias")
                    lw.local_attention = 1 if cfg.attention_layers[i] == "local" else 0
                arch_id = _lib.ARCH_GPT_NEO
            elif cfg.arch == "gptj":  # keys of HF GPTJModel.state_dict(); no attention biases, single LayerNorm per block
                mw.wte = p16(sd["wte.weight"])
                for i in range(cfg.n_layer):
                    p, lw = f"h.{i}.", layers[i]
                    lw.ln1_g, lw.ln1_b = p32(p + "ln_1.weight"), p32(p + "ln_1.bias")
                    lw.w_qkv = plin(i, "qkv", torch.cat([sd[p + "attn.q_proj.weight"], sd[p + "attn.k_proj.weight"],
                                                         sd[p + "attn.v_proj.weight"]], 0))
                    lw.w_o = plin(i, "o", sd[p + "attn.out_proj.weight"])
                    lw.w_fc, lw.b_fc = plin(i, "fc", sd[p + "mlp.fc_in.weight"]), p32(p + "mlp.fc_in.bias")
                    lw.w_proj, lw.b_proj = plin(i, "proj", sd[p + "mlp.fc_out.weight"]), p32(p + "mlp.fc_out.bias")
                arch_id = _lib.ARCH_GPTJ
            else:  # bloom: keys of HF BloomModel.state_dict()
                mw.wte = p16(sd["word_embeddings.weight"])
                mw.emb_ln_g, mw.emb_ln_b = p32("word_embeddings_layernorm.weight"), p32("word_embeddings_layernorm.bias")
                for i in range(cfg.n_layer):
                    p, lw = f"h.{i}.", layers[i]
                    lw.ln1_g, lw.ln1_b = p32(p + "input_layernorm.weight"), p32(p + "input_layernorm.bias")
                    # fused query_key_value rows are ordered per head [q(hd) | k(hd) | v(hd)] (HF:bloom:211-215);
                    # regroup to [q_all | k_all | v_all], the layout the attention kernel reads
                    wq = sd[p + "self_attention.query_key_value.weight"].view(H, 3, hd, d)
                    bq = sd[p + "self_attention.query_key_value.bias"].view(H, 3, hd)
                    lw.w_qkv = plin(i, "qkv", wq.permute(1, 0, 2, 3).reshape(3 * d, d))
                    lw.b_qkv = dev(bq.permute(1, 0, 2).reshape(3 * d), torch.float32).data_ptr()
                    lw.w_o, lw.b_o = plin(i, "o", sd[p + "self_attention.dense.weight"]), p32(p + "self_attention.dense.bias")
                    lw.ln2_g, lw.ln2_b = (p32(p + "post_attention_layernorm.weight"),
                                          p32(p + "post_attention_layernorm.bias"))
                    lw.w_fc, lw.b_fc = plin(i, "fc", sd[p + "mlp.dense_h_to_4h.weight"]), p32(p + "mlp.dense_h_to_4h.bias")
                    lw.w_proj, lw.b_proj = (plin(i, "proj", sd[p + "mlp.dense_4h_to_h.weight"]),
                                            p32(p + "mlp.dense_4h_to_h.bias"))
                arch_id = _lib.ARCH_BLOOM
            mw.lnf_g, mw.lnf_b = p32("ln_f.weight"), p32("ln_f.bias")
            mw.layers = layers
            self._layers = layers
            mc = _lib.ModelConfigC(arch=arch_id, n_layer=cfg.n_layer, d_model=d, n_head=cfg.n_head, d_ff=cfg.d_ff,
                                   vocab=cfg.vocab, max_pos=cfg.max_pos, window=cfg.window, rotary_dim=cfg.rotary_dim,
                                   ln_eps=cfg.ln_eps, max_tokens=self.max_tokens, max_batch=self.max_batch)
            handle = C.c_void_p()
            if fp8:
                self._fp8_layers = fp8_layers
                _lib.check(self._lib.sgpt_model_create_fp8(C.byref(mc), C.byref(mw), fp8_layers, C.byref(handle)),
                           "sgpt_model_create_fp8")
            else:
                _lib.check(self._lib.sgpt_model_create(C.byref(mc), C.byref(mw), C.byref(handle)), "sgpt_model_create")
            self._handle = handle
        # two pinned staging buffers for [ids | pos | cu] and their device twins: one H2D copy per batch, and the
        # host may pack batch i+1 while the GPU still runs batch i
        cap = 2 * self.max_tokens + self.max_batch + 1
        self._stage_host = [torch.empty(cap, dtype=torch.int32, pin_memory=True) for _ in range(2)]
        self._stage_dev = [torch.empty(cap, dtype=torch.int32, device=self.device) for _ in range(2)]
        self._stage_evt = [torch.cuda.Event() for _ in range(2)]
        self._stage_idx = 0
        self.h2d_bytes_last = 0
        self._pos_weights: Optional[torch.Tensor] = None

    def close(self):
        if getattr(self, "_handle", None):
            self._lib.sgpt_model_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_position_weights(self, weights: Optional[torch.Tensor]) -> None:
        """Install (or, with None, remove) a learnt position-weight table for method="weightedmean": token at padded
        position i gets weight ``weights[i]`` instead of ``i+1`` (ST/models/WeightedMeanPooling.py:21-37)."""
        if weights is None:
            self._pos_weights = None
            _lib.check(self._lib.sgpt_model_set_position_weights(self._handle, None, 0))
            return
        w = weights.detach().to(self.device, torch.float32).contiguous().view(-1)
        if w.numel() == 0:
            raise ValueError("empty position-weight table")
        self._pos_weights = w  # borrowed by the C handle
        _lib.check(self._lib.sgpt_model_set_position_weights(self._handle, w.data_ptr(), w.numel()),
                   "sgpt_model_set_position_weights")

    @property
    def embedding_dim(self) -> int:
        return self.cfg.d_model

    def encode_packed(self, ids: torch.Tensor, pos: torch.Tensor, cu: torch.Tensor, B: int, T: int, max_seqlen: int,
                      method: str = "weightedmean", layer_idx: int = -1, clamp: bool = False, normalize: bool = False,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Ragged batch already on the device (int32 tensors) -> fp32 [B, d] embeddings on the device."""
        if method not in POOL_MODES:
            raise ValueError(f"pooling method {method!r} not in {sorted(POOL_MODES)}")
        if out is None:
            out = torch.empty((B, self.cfg.d_model), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            rc = self._lib.sgpt_encode(self._handle, ids.data_ptr(), pos.data_ptr(), cu.data_ptr(), B, T, max_seqlen,
                                       layer_idx, POOL_MODES[method], int(clamp), int(normalize), out.data_ptr(),
                                       _lib.current_stream())
        _lib.check(rc, "sgpt_encode")
        return out

    def encode_tokens(self, input_ids, attention_mask, method: str = "weightedmean", layer_idx: int = -1,
                      clamp: bool = False, normalize: bool = False) -> torch.Tensor:
        """Padded [B,S] ids + mask (numpy or CPU/GPU torch) -> fp32 [B, d] embeddings on the device.

        The padded batch is packed on the host (padding never reaches the GPU) and shipped with ONE pinned H2D copy.
        """
        if isinstance(input_ids, torch.Tensor):
            input_ids = input_ids.detach().cpu().numpy()
        if isinstance(attention_mask, torch.Tensor):
            attention_mask = attention_mask.detach().cpu().numpy()
        ids, pos, cu, max_len = pack_ragged(input_ids, attention_mask)
        B, T = len(cu) - 1, int(cu[-1])
        if T > self.max_tokens or B > self.max_batch:
            raise ValueError(f"batch of {B} rows / {T} tokens exceeds the encoder workspace "
                             f"({self.max_batch} rows / {self.max_tokens} tokens)")
        if T and (int(ids.min()) < 0 or int(ids.max()) >= self.cfg.vocab):
            # torch's embedding lookup raises on such ids (HF:gpt_neo:462); the gather kernel would otherwise clamp them
            raise IndexError(f"token id out of range [0, {self.cfg.vocab}): min {int(ids.min())}, max {int(ids.max())}")
        if self.cfg.arch != "bloom" and max_len > self.cfg.max_pos:
            raise ValueError(f"sequence length {max_len} exceeds max_position_embeddings {self.cfg.max_pos}")
        n = 2 * T + B + 1
        slot = self._stage_idx
        self._stage_idx ^= 1
        self._stage_evt[slot].synchronize()  # the copy that last used this pinned buffer has finished
        host = self._stage_host[slot][:n].numpy()
        host[:T] = ids
        host[T:2 * T] = pos
        host[2 * T:] = cu
        dev = self._stage_dev[slot]
        with torch.cuda.device(self.device):
            dev[:n].copy_(self._stage_host[slot][:n], non_blocking=True)
            self._stage_evt[slot].record()
        self.h2d_bytes_last = n * 4
        return self.encode_packed(dev[:T], dev[T:2 * T], dev[2 * T:n], B, T, max_len, method, layer_idx, clamp,
                                  normalize)

    def last_residual(self) -> torch.Tensor:
        """Residual stream of the last encode call widened to fp32 [T, d] (parity/debug tap), copied out of the workspace."""
        T, d = C.c_int32(), C.c_int32()
        buf = torch.empty(self.max_tokens * self.cfg.d_model, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.sgpt_model_read_residual(self._handle, buf.data_ptr(), buf.numel(), C.byref(T),
                                                          C.byref(d), _lib.current_stream()))
        return buf[:T.value * d.value].view(T.value, d.value)
