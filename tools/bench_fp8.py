#!/usr/bin/env python
"""fp8 linear layers against bf16 on one GPU (random-init weights generated on the GPU, as tools/bench_models.py):

  accuracy   the fp8 GEMM's accumulation against fp64 on the dequantized operands, K = 768 ... 16384.  Columns k and
             k + K/2 cancel exactly (x equal, w negated), so the exact result is 0 while the partial sums grow like a
             random walk: the output IS the accumulation error, and max |out| / sum_k |x_k w_k| measures it.  The bf16
             GEMM on the same values is shown for comparison.
  encode     the four BASELINE configs, bf16 and fp8 timed alternately with device events over several rounds
             (median and spread), embeddings/s, linear-GEMM TFLOP/s against the data-sheet 1979 (fp8) / 989 (bf16),
             and the share of the step spent in the quantization kernels (a profiled run of its own).
  score      a GPT-J SGPT-CE scoring batch (sgpt_forward + LM-head log-probs), bf16 and fp8 alternately.
  quality    SGPT-125M random-init: cosine of fp8 (and bf16) embeddings to the pure fp32 oracle, and the top-10 overlap
             of a search over fp8- vs bf16-encoded documents.

    python tools/bench_fp8.py [--sections accuracy,encode,score,quality] [--rounds 5] [--steps 3]
Prints one JSON line per measurement; the card name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_models import SHAPES, rand_weights  # noqa: E402
from sgpt_b200 import Encoder, _lib, preset  # noqa: E402

DEV = torch.device("cuda:0")
CATS = ["embed", "layernorm", "linear_gemm", "attention", "pool", "similarity_gemm", "topk", "misc"]


def emit(**kw):
    print(json.dumps(kw), flush=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def quantize(x):
    n, K = x.shape
    q = torch.empty(n, K, dtype=torch.uint8, device=DEV)
    s = torch.empty(n, dtype=torch.float32, device=DEV)
    _lib.check(_lib.lib().sgpt_quantize_rows_fp8(x.data_ptr(), q.data_ptr(), s.data_ptr(), n, K, _lib.current_stream()))
    return q, s


def accuracy(ks):
    lib, st = _lib.lib(), _lib.current_stream()
    M, N = 512, 512
    for K in ks:
        g = torch.Generator(device=DEV).manual_seed(K)
        h = K // 2
        x = torch.randn(M, h, generator=g, device=DEV).to(torch.bfloat16)
        w = torch.randn(N, h, generator=g, device=DEV).to(torch.bfloat16)
        x, w = torch.cat([x, x], 1).contiguous(), torch.cat([w, -w], 1).contiguous()
        (xq, sx), (wq, sw) = quantize(x), quantize(w)
        # e4m3 x e4m3 products and their sums are exact in fp64, so the dot products are taken on q and scaled after
        qa, qb = xq.view(torch.float8_e4m3fn).double(), wq.view(torch.float8_e4m3fn).double()
        assert (qa @ qb.T).abs().max().item() == 0.0
        abs_sum = (qa.abs() @ qb.abs().T) * sx.double()[:, None] * sw.double()
        a, b = qa * sx.double()[:, None], qb * sw.double()[:, None]
        out = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        _lib.check(lib.sgpt_linear_fp8(xq.data_ptr(), K, sx.data_ptr(), wq.data_ptr(), K, sw.data_ptr(), None,
                                       out.data_ptr(), N, None, M, N, K, _lib.EPI_BF16, st))
        rel8 = out.double().abs() / abs_sum
        # the bf16 GEMM on the same values rounded to bf16 (the cancellation stays exact)
        ab, bb = a.to(torch.bfloat16), b.to(torch.bfloat16)
        abs16 = ab.double().abs() @ bb.double().abs().T
        o16 = torch.empty_like(out)
        _lib.check(lib.sgpt_linear(ab.data_ptr(), K, bb.data_ptr(), K, None, o16.data_ptr(), N, None, M, N, K,
                                   _lib.EPI_BF16, st))
        rel16 = o16.double().abs() / abs16
        emit(section="accuracy", K=K, fp8_max_err_over_abs_sum=rel8.max().item(),
             fp8_median_err_over_abs_sum=rel8.median().item(),
             fp8_max_err_over_sqrtK_2m23_abs_sum=(rel8 / (K ** 0.5 * 2.0 ** -23)).max().item(),
             bf16_max_err_over_abs_sum=rel16.max().item(), bf16_median_err_over_abs_sum=rel16.median().item())


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def profiled(fn, steps):
    lib = _lib.lib()
    ms_cat, n_cat = (ctypes.c_double * 8)(), (ctypes.c_int64 * 8)()
    lib.sgpt_profile_read(None, None, None)
    lib.sgpt_profile_enable(1)
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    lib.sgpt_profile_enable(0)
    lib.sgpt_profile_read(ms_cat, n_cat, None)
    return {c: ms_cat[i] / steps for i, c in enumerate(CATS) if ms_cat[i] > 0}


def alternate(fns, rounds, steps):
    """{name: [ms per step of each round]} with the candidates timed in turn inside every round."""
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            out[k].append(timed(fn, steps))
    return out


def encode(models, rounds, steps):
    for name in models:
        cfg = preset(name)
        B, S = SHAPES[name]
        sd = rand_weights(cfg, DEV)
        encs = {p: Encoder(cfg, sd, device=DEV, max_tokens=B * S, max_batch=B, precision=p) for p in ("bf16", "fp8")}
        del sd
        g = torch.Generator().manual_seed(1)
        ids = torch.randint(0, cfg.vocab, (B, S), generator=g).numpy()
        mask = np.ones((B, S), dtype=np.int8)
        fns = {p: (lambda e=e: e.encode_tokens(ids, mask)) for p, e in encs.items()}
        for fn in fns.values():
            fn(), fn()
        torch.cuda.synchronize()
        ms = alternate(fns, rounds, steps)
        L, d, ff = cfg.n_layer, cfg.d_model, cfg.d_ff
        lin_flops = B * S * 2 * L * (4 * d * d + 2 * d * ff)
        for p in ("bf16", "fp8"):
            prof = profiled(fns[p], steps)
            med = statistics.median(ms[p])
            gemm = prof.get("linear_gemm", float("nan"))
            emit(section="encode", model=name, precision=p, batch=B, seq_len=S, ms_median=med, ms_min=min(ms[p]),
                 ms_max=max(ms[p]), rounds=rounds, steps=steps, embeddings_per_s=B / (med / 1e3),
                 linear_gemm_ms=gemm, linear_gemm_tflops=lin_flops / (gemm / 1e3) / 1e12,
                 frac_of_datasheet=lin_flops / (gemm / 1e3) / 1e12 / (1979.0 if p == "fp8" else 989.0),
                 quant_ms=prof.get("misc", 0.0) if p == "fp8" else 0.0,
                 quant_share_of_step=(prof.get("misc", 0.0) / sum(prof.values())) if p == "fp8" else 0.0,
                 kernel_ms=prof)
        emit(section="encode", model=name, fp8_speedup=statistics.median(ms["bf16"]) / statistics.median(ms["fp8"]))
        for e in encs.values():
            e.close()
        del encs, fns
        torch.cuda.empty_cache()


def score(rounds, steps):
    from sgpt_b200.cross_encoder import LogLikelihoodScorer

    cfg = preset("sgpt-5.8b")
    sd = rand_weights(cfg, DEV)
    B, S, C = 32, 300, 16  # 32 (query, document) requests of 300 tokens, the last 16 are the scored query
    scs = {p: LogLikelihoodScorer(cfg, sd, device=DEV, max_tokens=B * S, max_batch=B, precision=p)
           for p in ("bf16", "fp8")}
    del sd
    g = torch.Generator().manual_seed(2)
    inputs = torch.randint(0, cfg.vocab, (B, S), generator=g).tolist()
    conts = [x[-C:] for x in inputs]
    fns = {p: (lambda s=s: s.score_batch(inputs, conts)) for p, s in scs.items()}
    for fn in fns.values():
        fn(), fn()
    torch.cuda.synchronize()
    ms = alternate(fns, rounds, steps)
    for p in ("bf16", "fp8"):
        prof = profiled(fns[p], steps)
        med = statistics.median(ms[p])
        emit(section="score", model="sgpt-5.8b", precision=p, requests=B, seq_len=S, ms_median=med, ms_min=min(ms[p]),
             ms_max=max(ms[p]), requests_per_s=B / (med / 1e3), quant_share_of_step=(
                 prof.get("misc", 0.0) / sum(prof.values())) if p == "fp8" else 0.0, kernel_ms=prof)
    for s in scs.values():
        s.close()
    del scs, fns
    torch.cuda.empty_cache()


def quality():
    from oracle import gpt_neo, pooling
    from sgpt_b200 import ModelConfig

    spec = gpt_neo.NeoSpec(**gpt_neo.SGPT_125M, vocab=2000, max_pos=128)
    cfg = ModelConfig(arch="gpt_neo", **gpt_neo.SGPT_125M, vocab=2000, max_pos=128, window=256)
    w = gpt_neo.init_weights(spec, seed=11)
    encs = {p: Encoder(cfg, w, device=DEV, max_tokens=256 * 64, max_batch=256, precision=p) for p in ("bf16", "fp8")}
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, spec.vocab, (32, 64), generator=g)
    lens = torch.randint(8, 65, (32,), generator=g)
    mask = (torch.arange(64)[None] < lens[:, None]).long()
    with torch.no_grad():
        want = pooling.weighted_mean(gpt_neo.forward(spec, w, ids, mask)[-1], mask).double()
    for p, e in encs.items():
        got = e.encode_tokens(ids.numpy(), mask.numpy(), method="weightedmean").cpu().double()
        cos = torch.nn.functional.cosine_similarity(got, want, dim=1)
        emit(section="quality", model="sgpt-125m random-init", precision=p, cos_to_fp32_oracle_min=cos.min().item(),
             cos_to_fp32_oracle_median=cos.median().item())
    # retrieval: 4096 documents and 256 queries, top-10 of cos_sim over fp8 vs bf16 embeddings of the same texts
    docs = torch.randint(0, spec.vocab, (4096, 64), generator=g)
    qs = torch.randint(0, spec.vocab, (256, 16), generator=g)
    emb = {}
    for p, e in encs.items():
        d = torch.cat([e.encode_tokens(docs[i:i + 256].numpy(), np.ones((256, 64), np.int8)) for i in range(0, 4096, 256)])
        q = e.encode_tokens(qs.numpy(), np.ones((256, 16), np.int8))
        emb[p] = (torch.nn.functional.normalize(q, dim=1), torch.nn.functional.normalize(d, dim=1))
    top = {p: (q @ d.T).topk(10, dim=1).indices.cpu() for p, (q, d) in emb.items()}
    overlap = [len(set(a.tolist()) & set(b.tolist())) / 10 for a, b in zip(top["fp8"], top["bf16"])]
    emit(section="quality", model="sgpt-125m random-init", top10_overlap_fp8_vs_bf16_mean=float(np.mean(overlap)),
         top10_overlap_min=float(np.min(overlap)))
    for e in encs.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sections", default="accuracy,encode,score,quality")
    ap.add_argument("--models", default="sgpt-125m,sgpt-1.3b,sgpt-5.8b,sgpt-bloom-7b1")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fp8.py measures on the GPU; there is nothing to measure without one"
    emit(section="card", card=card(), device=torch.cuda.get_device_name(0))
    sections = args.sections.split(",")
    if "accuracy" in sections:
        accuracy([768, 1024, 2048, 3072, 4096, 8192, 16384])
    if "encode" in sections:
        encode(args.models.split(","), args.rounds, args.steps)
    if "score" in sections:
        score(args.rounds, args.steps)
    if "quality" in sections:
        quality()


if __name__ == "__main__":
    main()
