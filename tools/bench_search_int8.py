"""bf16 vs int8 corpus shards: search time over the same documents, share of the HBM floor, and top-k overlap with fp32.

    python tools/bench_search_int8.py [--out result.json] [--quick]

The search reads the whole shard from HBM once per block of up to 256 queries, so its floor is the bytes of the shard:
n x D x (2 bytes bf16 | 1 byte int8) plus 4 bytes per document of scales.  Every case builds a bf16 and an int8 shard of
the same documents (int8 only at 10M x 4096, 82 GB in bf16) and times them alternately with CUDA events after warm-up
launches; the reported time is the median of the alternated repeats.  The overlap leg restates the planted corpus of
bench.py's fp32 overlap leg (200k x 768; every 100th document is a query plus 0.5 noise) and compares the top-k of each
shard type with exact fp32 cos_sim.  The card name and its power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sgpt_b200 import CorpusShard  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
K = 1001
REPEATS = 5


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        limit = f"unknown ({e})"
    return {"gpu": name, "power_limit": limit}


def fill(shards, n, D, q, g, slab=100_000):
    """The documents of bench.py's search leg: randn rows, every 100th a query plus 0.5 noise; added to every shard."""
    for s0 in range(0, n, slab):
        m = min(slab, n - s0)
        c = torch.randn(m, D, generator=g, device="cuda")
        idx = torch.arange(0, m, 100, device="cuda")
        c[idx] = q[((s0 + idx) // 100) % q.shape[0]] + 0.5 * c[idx]
        for sh in shards:
            sh.add(c)
        del c


def time_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def floor_ms(n, D, elem):
    return (n * D * elem + 4 * n) / HBM_BYTES_PER_S * 1e3


def alternate(fns, steps):
    """{name: median ms} over REPEATS rounds in which every fn is timed once, in turn, after warm-up launches."""
    for fn in fns.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {name: [] for name in fns}
    for _ in range(REPEATS):
        for name, fn in fns.items():
            times[name].append(time_ms(fn, steps))
    return {name: statistics.median(t) for name, t in times.items()}


def search_case(n, D, nqs, with_bf16, g):
    q = torch.randn(max(nqs), D, generator=g, device="cuda")
    shards = {"int8": CorpusShard(D, n, device="cuda:0", dtype="int8")}
    if with_bf16:
        shards["bf16"] = CorpusShard(D, n, device="cuda:0")
    fill(list(shards.values()), n, D, q, g)
    out = []
    for nq in nqs:
        qq = q[:nq].contiguous()
        steps = max(10, int(300 / (floor_ms(n, D, 2) / 0.6)))  # ~0.3 s per timed window
        t = alternate({k: (lambda sh=sh: sh.search(qq, K, "cos_sim")) for k, sh in shards.items()}, steps)
        row = {"case": f"{n // 10**6}M x {D}", "queries": nq, "k": K}
        for k, ms in t.items():
            row[f"{k}_ms"] = round(ms, 4)
            row[f"{k}_hbm_floor_ms"] = round(floor_ms(n, D, 2 if k == "bf16" else 1), 4)
            row[f"{k}_share_of_hbm_floor"] = round(floor_ms(n, D, 2 if k == "bf16" else 1) / ms, 3)
        if with_bf16:
            row["int8_speedup"] = round(t["bf16"] / t["int8"], 3)
        out.append(row)
        print(json.dumps(row), flush=True)
    del shards
    torch.cuda.empty_cache()
    return out


def range_case(g):
    n, D, nq = 1_000_000, 768, 256
    q = torch.randn(nq, D, generator=g, device="cuda")
    shards = {"bf16": CorpusShard(D, n, device="cuda:0"), "int8": CorpusShard(D, n, device="cuda:0", dtype="int8")}
    fill(list(shards.values()), n, D, q, g)
    s, _ = shards["int8"].search(q, 10, "cos_sim")
    thr = float(s[:, -1].median())  # about 10 documents per query
    t = alternate({k: (lambda sh=sh: sh.range_search(q, thr, "cos_sim")) for k, sh in shards.items()}, 100)
    per_q = float(shards["int8"].range_search(q, thr, "cos_sim")[0][-1]) / nq
    row = {"case": "range 1M x 768", "queries": nq, "threshold": thr, "int8_docs_per_query": round(per_q, 2)}
    for k, ms in t.items():
        row[f"{k}_ms"] = round(ms, 4)
        row[f"{k}_share_of_hbm_floor"] = round(floor_ms(n, D, 2 if k == "bf16" else 1) / ms, 3)
    print(json.dumps(row), flush=True)
    del shards
    torch.cuda.empty_cache()
    return row


def overlap_leg():
    """bench.py's planted 200k x 768 corpus; top-k of each shard type vs fp32 cos_sim + torch.topk of the raw vectors."""
    n, D, nq = 200_000, 768, 128
    g = torch.Generator(device="cuda").manual_seed(2024)
    q = torch.randn(nq, D, generator=g, device="cuda")
    c = torch.randn(n, D, generator=g, device="cuda")
    idx = torch.arange(0, n, 100, device="cuda")
    c[idx] = q[(idx // 100) % nq] + 0.5 * c[idx]
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    ref = torch.nn.functional.normalize(q, dim=1) @ torch.nn.functional.normalize(c, dim=1).T
    torch.backends.cuda.matmul.allow_tf32 = prev
    _, ri = torch.topk(ref, K, dim=1)
    ri = ri.tolist()
    out = {"case": "overlap vs fp32, planted 200k x 768", "queries": nq}
    for dtype in ("bf16", "int8"):
        _, i = CorpusShard.from_embeddings(c, device="cuda:0", dtype=dtype).search(q, K, "cos_sim")
        i = i.tolist()
        for kk in (10, 100, 1001):
            inter = sum(len(set(a[:kk]) & set(b[:kk])) for a, b in zip(i, ri))
            out[f"{dtype}_overlap_at_{kk}"] = round(inter / (nq * kk), 5)
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    ap.add_argument("--quick", action="store_true", help="only the 1M x 768 case and the overlap leg")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_search_int8 measures the GPU; there is no CPU path"
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "cases": []}
    print(json.dumps(res["card"]), flush=True)
    res["cases"] += search_case(1_000_000, 768, [128, 256], True, g)
    if not a.quick:
        res["cases"] += search_case(1_000_000, 2048, [128], True, g)
        res["cases"] += search_case(5_000_000, 4096, [128], True, g)
        res["cases"] += search_case(10_000_000, 4096, [128], False, g)
    res["cases"].append(range_case(g))
    res["overlap"] = overlap_leg()
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
