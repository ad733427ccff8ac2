#!/usr/bin/env python
"""Range search, paraphrase mining and community detection timings; prints one JSON line.

    python tools/bench_mining.py [--docs 1000000] [--mining-docs 200000] [--ref-docs 20000]

* range search (sgpt_range_search through CorpusShard._range_call) on a docs x 768 bf16 shard with 256 queries, count
  only (cap = 0) and count + fill, at two thresholds: the median 10th and 1000th best cosine of the queries, so that
  about 10 and about 1000 documents per query are admitted.  Device-event time per call over --steps calls.
* all-pairs paraphrase_mining_embeddings (top_k 100, default chunk sizes) and community_detection (threshold 0.75,
  min_community_size 10) over mining-docs x 768 planted clusters, host clock around synchronised calls (they return
  host lists).
* the same two functions as the reference computes them (full score matrix, Python loops; oracle/mining.py restates
  util.py:129-189 and :385-448) on the CPU at ref-docs x 768, and the library at that size, in the same process.

Bytes and FLOPs come from the shapes: one scan of the shard per 256-query block (bf16 rows + fp32 norms) plus the
entries written, and 2 x queries x docs x 768 multiply-adds.  The share of peak is max(bytes / 3.35 TB/s,
flops / 989 TFLOP/s) over the measured time (H100 SXM data sheet, dense BF16, 700 W card).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sgpt_b200 import CorpusShard, community_detection, paraphrase_mining_embeddings  # noqa: E402

HBM, BF16 = 3.35e12, 989e12
DIM = 768


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out


def planted(n, cluster, noise, g, dev):
    """n documents in clusters of `cluster` noisy copies of random centres (within-cluster cosine ~ 1 / (1 + noise^2))."""
    centres = torch.randn(n // cluster + 1, DIM, generator=g, device=dev)
    x = centres.repeat_interleave(cluster, 0)[:n] + noise * torch.randn(n, DIM, generator=g, device=dev)
    return x[torch.randperm(n, generator=g, device=dev)]


def share(ms, nbytes, flops):
    floor = max(nbytes / HBM, flops / BF16)
    return round(floor / (ms / 1e3), 4), ("hbm" if nbytes / HBM >= flops / BF16 else "bf16")


def time_range(shard, qb, qs, threshold, cap, steps):
    nq = qb.shape[0]
    counts = torch.empty(nq, dtype=torch.int64, device=shard.device)
    s = torch.empty(max(cap, 1), dtype=torch.float32, device=shard.device)
    i = torch.empty(max(cap, 1), dtype=torch.int64, device=shard.device)
    c_scale = shard.inv_norms.data_ptr()
    for _ in range(3):
        shard._range_call(qb, qs, c_scale, threshold, counts, cap, s, i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        shard._range_call(qb, qs, c_scale, threshold, counts, cap, s, i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, int(counts.sum())


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=256)
    ap.add_argument("--mining-docs", type=int, default=200_000)
    ap.add_argument("--ref-docs", type=int, default=20_000)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mining.py measures the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    res = {"card": name, "power_limit": power, "dim": DIM}

    # ---- range search ----------------------------------------------------------------------------------------------
    g = torch.Generator(device=dev).manual_seed(1)
    n, nq = args.docs, args.queries
    shard = CorpusShard(DIM, n, device=dev)
    for s0 in range(0, n, 250_000):
        shard.add(torch.randn(min(250_000, n - s0), DIM, generator=g, device=dev))
    q = shard.stored()[torch.randint(0, n, (nq,), generator=g, device=dev)].float()
    q = q + 0.8 * torch.randn(q.shape, generator=g, device=dev)
    qb, qs, _ = shard._queries(q, "cos_sim")
    top, _ = shard.search(q, 1000, "cos_sim")
    scan_bytes = ((nq + 255) // 256) * (n * DIM * 2 + n * 4)
    flops = 2 * nq * n * DIM
    res["range"] = []
    for label, col in (("~10 per query", 9), ("~1000 per query", 999)):
        t = float(top[:, col].median())
        for mode in ("count", "fill"):
            cap = 0
            if mode == "fill":
                _, cap = time_range(shard, qb, qs, t, 0, 1)
            ms, total = time_range(shard, qb, qs, t, cap, args.steps)
            nbytes = scan_bytes + nq * 8 + (total * 12 if mode == "fill" else 0)
            frac, bound = share(ms, nbytes, flops)
            res["range"].append({"threshold": round(t, 5), "admitted": label, "mode": mode, "entries": total,
                                 "ms": round(ms, 4), "bytes": nbytes, "flops": flops, "share_of_peak": frac,
                                 "bound": bound})
    del shard, top
    torch.cuda.empty_cache()

    # ---- all-pairs mining over planted clusters -------------------------------------------------------------------
    m = args.mining_docs
    x = planted(m, 25, 0.4, g, dev)
    mshard = CorpusShard.from_embeddings(x)
    paraphrase_mining_embeddings(mshard.view(0, 20_000), top_k=100, max_pairs=10_000)  # warm-up of every shape class
    community_detection(mshard.view(0, 20_000), threshold=0.75, min_community_size=10)
    ms_pm, pairs = wall(lambda: paraphrase_mining_embeddings(mshard, top_k=100))
    ms_cd, comms = wall(lambda: community_detection(mshard, threshold=0.75, min_community_size=10))
    all_pairs_flops = 2 * m * m * DIM
    res["paraphrase_mining"] = {"docs": m, "top_k": 100, "ms": round(ms_pm, 1), "pairs": len(pairs),
                                "flops": all_pairs_flops,
                                "share_of_peak": share(ms_pm, -(-m // 256) * (m * DIM * 2 + m * 4), all_pairs_flops)[0]}
    res["community_detection"] = {"docs": m, "ms": round(ms_cd, 1), "communities": len(comms),
                                  "members": sum(len(c) for c in comms), "flops": all_pairs_flops}
    del mshard
    torch.cuda.empty_cache()

    # ---- the reference algorithms on the CPU and the library at the same size -------------------------------------
    from oracle import mining as omining

    r = args.ref_docs
    xr = planted(r, 25, 0.4, g, dev).to(torch.bfloat16).float()
    xc = xr.cpu()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    t0 = time.perf_counter()
    ref_pm = omining.paraphrase_mining_embeddings(xc, top_k=100)
    ms_ref_pm = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    ref_cd = omining.community_detection(xc, threshold=0.75, min_community_size=10)
    ms_ref_cd = (time.perf_counter() - t0) * 1e3
    ms_lib_pm, lib_pm = wall(lambda: paraphrase_mining_embeddings(xr, top_k=100))
    ms_lib_cd, lib_cd = wall(lambda: community_detection(xr, threshold=0.75, min_community_size=10))
    res["reference_cpu"] = {"docs": r, "cpu_threads": torch.get_num_threads(),
                            "paraphrase_mining_ms": round(ms_ref_pm, 1), "community_detection_ms": round(ms_ref_cd, 1),
                            "library_paraphrase_mining_ms": round(ms_lib_pm, 1),
                            "library_community_detection_ms": round(ms_lib_cd, 1),
                            "same_pairs": len(ref_pm) == len(lib_pm), "same_communities": len(ref_cd) == len(lib_cd)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
