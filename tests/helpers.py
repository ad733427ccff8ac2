"""Shared test helpers: a tiny deterministic tokenizer (no pretrained files are reachable offline) and builders."""
import re
import zlib

import numpy as np
import torch


class ToyTokenizer:
    """Whitespace/bracket tokenizer with the HF methods the reference calls (tokenize, convert_tokens_to_ids, encode)."""

    SPECIAL = {"[": 58, "]": 60, "{": 90, "}": 92, "[SOS]": 997, "{SOS}": 998}  # GPT-2 BPE ids of the brackets

    def __init__(self, vocab=1000, pad_token_id=999):
        self.vocab = vocab
        self.pad_token_id = pad_token_id
        self.eos_token = "<|endoftext|>"
        self.pad_token = None

    def tokenize(self, text):
        return re.findall(r"\[SOS\]|\{SOS\}|[\[\]{}]|[^\s\[\]{}]+", text)

    def convert_tokens_to_ids(self, tokens):
        return [self.SPECIAL[t] if t in self.SPECIAL else 100 + zlib.crc32(t.encode()) % (self.vocab - 200) for t in tokens]

    def encode(self, text, add_special_tokens=False):
        return self.convert_tokens_to_ids(self.tokenize(text))


def ragged_batch(B, S, vocab, seed, pad_id=0):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, S + 1, (B,), generator=g)
    lens[0] = 1
    if B > 1:
        lens[1] = S
    ids = torch.randint(0, vocab, (B, S), generator=g)
    mask = (torch.arange(S).unsqueeze(0) < lens.unsqueeze(1)).long()
    ids = torch.where(mask.bool(), ids, torch.full_like(ids, pad_id))
    return ids, mask


def planted_corpus(n, D, nq, seed):
    """Random corpus with ~1% planted near-duplicates of the queries so the top of the ranking is meaningful."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(nq, D, generator=g)
    c = torch.randn(n, D, generator=g)
    idx = torch.arange(0, n, 97)
    c[idx] = q[idx // 97 % nq] + 0.5 * c[idx]
    return q, c


def min_row_cosine(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return torch.nn.functional.cosine_similarity(a, b, dim=1).min().item()


BF16_U = 2.0 ** -8  # unit roundoff of bf16 (8 significant bits, round to nearest): |bf16(x) - x| <= BF16_U |x|


def tensor_core_sum_bound(abs_sum, K):
    """Bound on the fp32 error of a K-term dot product accumulated by the GEMM on the tensor cores: at most K/16 + 16
    roundings (one per k16 step into the accumulator, plus the sum of the 16 products inside one step), each at most 2^-23
    (one ulp, so truncating adders are covered) of a partial sum, and every partial sum is at most
    abs_sum = sum_k |x_k w_k|."""
    return (K / 16 + 16) * 2.0 ** -23 * abs_sum


def topk_reference(scores, ids, k, exclude=None):
    """Exact top-k of candidate entries, the contract of include/sgpt_b200.h: per query the entries with id >= 0 and
    id != exclude[q], ordered by score descending with ties by ascending id (-0.0 equal to +0.0), the first k, the tail
    filled with (-inf, -1).  scores [nq, m] (any float dtype, values taken exactly), ids int64 [nq, m], exclude int64 [nq]
    or None.  Returns (fp64 scores [nq, k], int64 ids [nq, k])."""
    s = torch.as_tensor(scores).double().cpu().numpy()
    i = torch.as_tensor(ids).cpu().numpy().astype(np.int64)
    nq = s.shape[0]
    out_s = np.full((nq, k), -np.inf)
    out_i = np.full((nq, k), -1, dtype=np.int64)
    for q in range(nq):
        ok = i[q] >= 0
        if exclude is not None:
            ok &= i[q] != int(exclude[q])
        sq, iq = s[q][ok] + 0.0, i[q][ok]  # (+ 0.0 turns -0.0 into +0.0)
        order = np.lexsort((iq, -sq))[:k]  # last key primary: score descending, then id ascending
        out_s[q, :len(order)], out_i[q, :len(order)] = sq[order], iq[order]
    return torch.from_numpy(out_s), torch.from_numpy(out_i)


def rotary_cos_sin(max_pos, rotary_dim):
    """GPT-J's table in the layout of include/sgpt_b200.h: fp32[max_pos, rotary_dim/2, 2] = (cos, sin), from the oracle's
    create_sinusoidal_positions (oracle/gptj.py rotary_tables)."""
    from oracle.gptj import rotary_tables

    sin, cos = rotary_tables(max_pos, rotary_dim)
    return torch.stack([cos, sin], dim=-1).contiguous()


def rotary_reference(y, pos, cos_sin, d, head_dim, rotary_dim):
    """fp64 GPT-J rotary embedding of a fused projection y [M, 3d] = [q | k | v]: HF's rotate_every_two (oracle/gptj.py
    apply_rotary) on the first rotary_dim dims of every q and k head, with the (cos, sin) values of the table at pos."""
    from oracle.gptj import apply_rotary

    M = y.shape[0]
    cs = cos_sin.to(y.device).double()[pos.long()]  # [M, rd/2, 2]
    qk = y[:, :2 * d].reshape(M, 2 * d // head_dim, head_dim).clone()
    qk[..., :rotary_dim] = apply_rotary(qk[None, ..., :rotary_dim], cs[None, ..., 1], cs[None, ..., 0])[0]
    return torch.cat([qk.view(M, 2 * d), y[:, 2 * d:]], dim=1)


def rotary_abs_bound(e, pos, cos_sin, d, head_dim, rotary_dim):
    """Propagates a per-element error bound e >= 0 of y through the rotation: the pair (e0, e1) becomes
    (|c| e0 + |s| e1, |c| e1 + |s| e0) on the rotated dims; the other dims keep their bound."""
    M = e.shape[0]
    cs = cos_sin.to(e.device).double()[pos.long()].abs().repeat_interleave(2, dim=1)  # [M, rd, 2]
    qk = e[:, :2 * d].reshape(M, 2 * d // head_dim, head_dim).clone()
    r = qk[..., :rotary_dim]
    swapped = r.reshape(M, -1, rotary_dim // 2, 2).flip(-1).reshape(r.shape)
    qk[..., :rotary_dim] = r * cs[:, None, :, 0] + swapped * cs[:, None, :, 1]
    return torch.cat([qk.view(M, 2 * d), e[:, 2 * d:]], dim=1)


def left_padded_positions(M, max_pos, seed):
    """Positions of M packed rows taken from a left-padded batch: up to three runs of consecutive positions, none starting
    at 0, the last one ending at max_pos - 1 (int32)."""
    g = torch.Generator().manual_seed(seed)
    cuts = sorted(torch.randint(1, M, (2,), generator=g).tolist()) if M > 2 else []
    runs, prev = [], 0
    for c in cuts + [M]:
        if c > prev:
            runs.append(c - prev)
        prev = c
    pos = []
    for i, n in enumerate(runs):
        start = max_pos - n if i == len(runs) - 1 else int(torch.randint(1, max_pos - n + 1, (1,), generator=g))
        pos.append(torch.arange(start, start + n))
    return torch.cat(pos).to(torch.int32)


class LazyF32Weights(dict):
    """bf16/fp32 CPU tensors that are widened to fp32 only while an oracle expression uses them: the functional oracles
    index the state dict once per use, so a 6-7 B-parameter model never exists in fp32 as a whole (12-14 GB of bf16 on
    the host instead of 24-28 GB of fp32)."""

    def __getitem__(self, key):
        return dict.__getitem__(self, key).float()


def full_size_weights(arch, spec, seed, device="cuda:0", host_copy=True):
    """Random weights of a FULL-SIZE model (BASELINE.json configs[2..4]) drawn on the GPU (torch.randn on the CPU needs
    a minute per billion parameters), linear weights in bf16 — exactly the values the CUDA path stores — LayerNorm
    parameters and biases in fp32.  Key names follow the HF state_dict of the architecture (oracle/*.py:init_weights
    use the same construction at small sizes).  Returns (device dict for sgpt_b200.Encoder, LazyF32Weights for the CPU
    oracle holding the same values, or None with host_copy=False)."""
    import math

    g = torch.Generator(device=device).manual_seed(seed)
    bf, f32 = torch.bfloat16, torch.float32

    def rnd(*shape, sd=0.02, mean=0.0, dtype=bf):
        return (torch.randn(*shape, generator=g, device=device) * sd + mean).to(dtype)

    d, ff, L = spec.d_model, spec.d_ff, spec.n_layer
    hd = d // spec.n_head
    w = {}
    if arch == "gpt_neo":
        qk_sd = math.sqrt(2.5 / (d * math.sqrt(hd)))  # un-scaled q.k logits with a spread of ~2.5 (neither flat nor one-hot)
        w["wte.weight"], w["wpe.weight"] = rnd(spec.vocab, d), rnd(spec.max_pos, d, sd=0.01)
        for i in range(L):
            p = f"h.{i}."
            w[p + "ln_1.weight"], w[p + "ln_1.bias"] = rnd(d, sd=0.1, mean=1.0, dtype=f32), rnd(d, sd=0.05, dtype=f32)
            w[p + "attn.attention.q_proj.weight"], w[p + "attn.attention.k_proj.weight"] = rnd(d, d, sd=qk_sd), rnd(d, d, sd=qk_sd)
            w[p + "attn.attention.v_proj.weight"] = rnd(d, d)
            w[p + "attn.attention.out_proj.weight"], w[p + "attn.attention.out_proj.bias"] = rnd(d, d), rnd(d, dtype=f32)
            w[p + "ln_2.weight"], w[p + "ln_2.bias"] = rnd(d, sd=0.1, mean=1.0, dtype=f32), rnd(d, sd=0.05, dtype=f32)
            w[p + "mlp.c_fc.weight"], w[p + "mlp.c_fc.bias"] = rnd(ff, d), rnd(ff, dtype=f32)
            w[p + "mlp.c_proj.weight"], w[p + "mlp.c_proj.bias"] = rnd(d, ff), rnd(d, dtype=f32)
    elif arch == "gptj":
        qk_sd = math.sqrt(2.5 / (d * math.sqrt(hd))) * math.sqrt(math.sqrt(hd))  # logits / sqrt(hd) with spread ~2.5
        w["wte.weight"] = rnd(spec.vocab, d)
        for i in range(L):
            p = f"h.{i}."
            w[p + "ln_1.weight"], w[p + "ln_1.bias"] = rnd(d, sd=0.1, mean=1.0, dtype=f32), rnd(d, sd=0.05, dtype=f32)
            w[p + "attn.q_proj.weight"], w[p + "attn.k_proj.weight"] = rnd(d, d, sd=qk_sd), rnd(d, d, sd=qk_sd)
            w[p + "attn.v_proj.weight"], w[p + "attn.out_proj.weight"] = rnd(d, d), rnd(d, d)
            w[p + "mlp.fc_in.weight"], w[p + "mlp.fc_in.bias"] = rnd(ff, d), rnd(ff, dtype=f32)
            w[p + "mlp.fc_out.weight"], w[p + "mlp.fc_out.bias"] = rnd(d, ff), rnd(d, dtype=f32)
    elif arch == "bloom":
        qk_sd = math.sqrt(2.5 / (d * math.sqrt(hd))) * math.sqrt(math.sqrt(hd))
        w["word_embeddings.weight"] = rnd(spec.vocab, d)
        w["word_embeddings_layernorm.weight"] = rnd(d, sd=0.1, mean=1.0, dtype=f32)
        w["word_embeddings_layernorm.bias"] = rnd(d, sd=0.05, dtype=f32)
        for i in range(L):
            p = f"h.{i}."
            w[p + "input_layernorm.weight"], w[p + "input_layernorm.bias"] = rnd(d, sd=0.1, mean=1.0, dtype=f32), rnd(d, sd=0.05, dtype=f32)
            qkv = rnd(3 * d, d, sd=qk_sd).view(spec.n_head, 3, hd, d)  # per head [q | k | v] rows (HF:bloom:211-215)
            qkv[:, 2] = rnd(spec.n_head, hd, d)                         # v rows at the ordinary 0.02
            w[p + "self_attention.query_key_value.weight"] = qkv.view(3 * d, d)
            w[p + "self_attention.query_key_value.bias"] = rnd(3 * d, dtype=f32)
            w[p + "self_attention.dense.weight"], w[p + "self_attention.dense.bias"] = rnd(d, d), rnd(d, dtype=f32)
            w[p + "post_attention_layernorm.weight"] = rnd(d, sd=0.1, mean=1.0, dtype=f32)
            w[p + "post_attention_layernorm.bias"] = rnd(d, sd=0.05, dtype=f32)
            w[p + "mlp.dense_h_to_4h.weight"], w[p + "mlp.dense_h_to_4h.bias"] = rnd(ff, d), rnd(ff, dtype=f32)
            w[p + "mlp.dense_4h_to_h.weight"], w[p + "mlp.dense_4h_to_h.bias"] = rnd(d, ff), rnd(d, dtype=f32)
    else:
        raise ValueError(arch)
    w["ln_f.weight"], w["ln_f.bias"] = rnd(d, sd=0.1, mean=1.0, dtype=f32), rnd(d, sd=0.05, dtype=f32)
    return w, (LazyF32Weights({k: v.cpu() for k, v in w.items()}) if host_copy else None)
