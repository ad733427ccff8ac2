#!/usr/bin/env python
"""IVF range search against the exact range search, and paraphrase mining / community detection over an IVF index
against the exact all-pairs functions; prints one JSON line.

    python tools/bench_ivf_mining.py [--quick] [--parts range,mining] [--out result.json]

Data: the planted clusters of tools/bench_ivf.py (`nlist` randn centres, every row a centre plus unit-variance noise).
For mining every row is in addition one of a group of 25 near-duplicates (a parent drawn as above plus 0.4 x noise per
row, within-group cosine ~0.93), so that both functions have pairs and communities to find; the rows are shuffled.

* Range search: 1M x 768 bf16 and int8 indexes, nlist 4000; 1, 16 and 256 queries at nprobe 8 and 32; thresholds at the
  median 10th and 1000th best exact cosine of the queries (about 10 and 1000 documents per query).  Count-only (cap 0)
  and fill (cap = the total) are timed separately, each alternating with the exact range search of the same source shard
  (CUDA events, REPEATS rounds: median, min, max).  Probes and query rows are prepared once.  "host_issue_ms" is the host
  time to issue one IVF call (no synchronisation): when it reaches the device time, the call is launch-bound.
* Mining: paraphrase_mining_embeddings (top_k 100) and community_detection (0.75, 10) over a bf16 IVF index (nlist
  4 sqrt(n) rounded to a multiple of 8) at 200k and 1M rows against the exact functions on the same shard (nprobe 8 and
  32), and at 10M over the index only (nprobe 8).  Host clock around synchronised calls (they return host lists), as
  tools/bench_mining.py.  Recall: the share of the exact result's pairs (unordered) the IVF result contains, and the
  share of exact communities the IVF result reproduces exactly.

The card name and power limit are read in the same run, before and after."""
import argparse
import json
import math
import os
import statistics
import sys
import time

import torch

TOOLS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(TOOLS))
sys.path.insert(0, TOOLS)

from bench_ivf import card, planted  # noqa: E402

from sgpt_b200 import CorpusShard, IVFIndex, community_detection, paraphrase_mining_embeddings  # noqa: E402
from sgpt_b200.ivf import _rows_f32  # noqa: E402

DIM = 768
REPEATS = 5
NQS = (1, 16, 256)
NPROBES = (8, 32)


def time_calls(fn, steps):
    """(device ms per call, host ms to issue one call)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    host = (time.perf_counter() - t0) * 1e3 / steps
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, host


def alternate(fns):
    """{name: (median, min, max, host issue median) ms}: REPEATS rounds, every fn timed once per round in turn."""
    steps = {}
    for name, fn in fns.items():
        for _ in range(3):
            fn()
        steps[name] = max(3, min(500, int(50 / max(time_calls(fn, 3)[0], 1e-3))))
    dev, host = {n: [] for n in fns}, {n: [] for n in fns}
    for _ in range(REPEATS):
        for name, fn in fns.items():
            d, h = time_calls(fn, steps[name])
            dev[name].append(d)
            host[name].append(h)
    return {n: (statistics.median(dev[n]), min(dev[n]), max(dev[n]), statistics.median(host[n])) for n in fns}


def range_case(dtype, g, rows):
    n, nlist = 1_000_000, 4000
    src, _ = planted(n, DIM, nlist, dtype, g)
    index = IVFIndex.build(src, nlist, seed=0, train_size=40 * nlist)
    # queries: stored rows (dequantized) plus unit-variance noise
    q = _rows_f32(src, torch.randint(n, (max(NQS),), generator=g, device="cuda"))
    q += torch.randn(q.shape, generator=g, device="cuda")
    top, _ = src.search(q, 1000, "cos_sim")
    for label, col in (("~10", 9), ("~1000", 999)):
        t = float(top[:, col].median())
        for nq in NQS:
            qq = q[:nq].contiguous()
            qb, q_scale, c_scale = index.shard._queries(qq, "cos_sim")
            sb, s_scale, sc_scale = src._queries(qq, "cos_sim")
            counts = torch.empty(nq, dtype=torch.int64, device="cuda")
            for nprobe in NPROBES:
                probes = index.probe(qq, nprobe)
                mask = index.shard._mask(None, nq)
                index._range_call(qb, q_scale, c_scale, probes, t, mask, counts, 0, None, None)
                ivf_total = int(counts.sum())
                src._range_call(sb, s_scale, sc_scale, t, counts, 0, None, None)
                exact_total = int(counts.sum())
                cap = max(ivf_total, exact_total, 1)
                out_s = torch.empty(cap, dtype=torch.float32, device="cuda")
                out_i = torch.empty(cap, dtype=torch.int64, device="cuda")
                res = alternate({
                    "ivf_count": lambda: index._range_call(qb, q_scale, c_scale, probes, t, mask, counts, 0, None, None),
                    "exact_count": lambda: src._range_call(sb, s_scale, sc_scale, t, counts, 0, None, None),
                    "ivf_fill": lambda: index._range_call(qb, q_scale, c_scale, probes, t, mask, counts, cap, out_s,
                                                          out_i),
                    "exact_fill": lambda: src._range_call(sb, s_scale, sc_scale, t, counts, cap, out_s, out_i)})
                row = {"case": f"1M x {DIM} {dtype}", "nlist": nlist, "queries": nq, "nprobe": nprobe,
                       "admitted": label, "threshold": round(t, 5), "ivf_entries": ivf_total,
                       "exact_entries": exact_total, "recall": round(ivf_total / max(exact_total, 1), 4)}
                for name, (med, lo, hi, host) in res.items():
                    row[f"{name}_ms"] = round(med, 4)
                    row[f"{name}_ms_min_max"] = [round(lo, 4), round(hi, 4)]
                    if name.startswith("ivf"):
                        row[f"{name}_host_issue_ms"] = round(host, 4)
                for mode in ("count", "fill"):
                    row[f"{mode}_speedup_vs_exact"] = round(res[f"exact_{mode}"][0] / res[f"ivf_{mode}"][0], 2)
                rows.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
    del index, src
    torch.cuda.empty_cache()


def mining_data(n, nlist, g, slab=500_000):
    """Rows of bench_ivf's planted clusters, each one of 25 near-duplicates of a parent row, shuffled."""
    centres = torch.randn(nlist, DIM, generator=g, device="cuda")
    parents = centres[torch.randint(nlist, ((n + 24) // 25,), generator=g, device="cuda")]
    parents += torch.randn(parents.shape, generator=g, device="cuda")
    group = torch.randperm(n, generator=g, device="cuda") // 25  # the parent of every row
    shard = CorpusShard(DIM, n, device="cuda:0")
    for s0 in range(0, n, slab):
        m = min(slab, n - s0)
        shard.add(parents[group[s0:s0 + m]] + 0.4 * torch.randn(m, DIM, generator=g, device="cuda"))
    return shard


def pair_recall(exact, ivf):
    a = {(min(i, j), max(i, j)) for _, i, j in exact}
    b = {(min(i, j), max(i, j)) for _, i, j in ivf}
    return round(len(a & b) / max(len(a), 1), 4)


def community_recall(exact, ivf):
    b = {tuple(c) for c in ivf}
    return round(sum(tuple(c) in b for c in exact) / max(len(exact), 1), 4)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def mining_case(n, g, exact, nprobes):
    nlist = int(round(4 * math.sqrt(n) / 8)) * 8
    shard = mining_data(n, nlist, g)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    index = IVFIndex.build(shard, nlist, seed=0, train_size=min(n, 40 * nlist))
    torch.cuda.synchronize()
    out = {"docs": n, "nlist": nlist, "build_s": round(time.perf_counter() - t0, 2), "runs": []}
    want_pm = want_cd = None
    if exact:
        ms_pm, want_pm = wall(lambda: paraphrase_mining_embeddings(shard, top_k=100, corpus_chunk_size=n))
        ms_cd, want_cd = wall(lambda: community_detection(shard, threshold=0.75, min_community_size=10))
        out["exact"] = {"paraphrase_ms": round(ms_pm, 1), "pairs": len(want_pm), "community_ms": round(ms_cd, 1),
                        "communities": len(want_cd)}
    else:
        del shard
        torch.cuda.empty_cache()
    for nprobe in nprobes:
        ms_pm, pm = wall(lambda: paraphrase_mining_embeddings(index, top_k=100, nprobe=nprobe))
        ms_cd, cd = wall(lambda: community_detection(index, threshold=0.75, min_community_size=10, nprobe=nprobe))
        run = {"nprobe": nprobe, "paraphrase_ms": round(ms_pm, 1), "pairs": len(pm), "community_ms": round(ms_cd, 1),
               "communities": len(cd)}
        if exact:
            run["paraphrase_speedup"] = round(out["exact"]["paraphrase_ms"] / ms_pm, 2)
            run["community_speedup"] = round(out["exact"]["community_ms"] / ms_cd, 2)
            run["pair_recall"] = pair_recall(want_pm, pm)
            run["community_recall"] = community_recall(want_cd, cd)
        out["runs"].append(run)
        print(json.dumps(dict(run, docs=n)), file=sys.stderr, flush=True)
    del index
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="bf16 range search and the 200k mining case only")
    ap.add_argument("--parts", default="range,mining", help="comma-separated: range, mining")
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivf_mining measures the GPU; there is no CPU path"
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "dim": DIM, "range": [], "mining": []}
    parts = a.parts.split(",")
    if "range" in parts:
        for dtype in ("bf16",) if a.quick else ("bf16", "int8"):
            range_case(dtype, g, res["range"])
    if "mining" in parts:
        mining_case(20_000, g, True, NPROBES[:1])  # warm-up of every shape class of the mining paths
        cases = ((200_000, True, NPROBES),)
        if not a.quick:
            cases += ((1_000_000, True, NPROBES), (10_000_000, False, NPROBES[:1]))
        for n, exact, nprobes in cases:
            res["mining"].append(mining_case(n, g, exact, nprobes))
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
