"""Graph index vs IVF and exact search: build time, time per search, recall and visited rows.

    python tools/bench_graph.py [--out result.json] [--big]

Datasets, generated on the device from seed 0, 1M x 768 bf16 each:
  clustered   4000 random centres (randn), every document a centre plus unit-variance noise (tools/bench_ivf.py's
              planted clusters at nlist = 4 sqrt(n)); queries are other draws around random centres.
  lowdim      G z + 0.1 eps, z ~ N(0, I_16), G a fixed random 768 x 16 matrix; queries from the same law.
The exact k-NN graph of the clustered data is likely disconnected between clusters, so hashed entry points can miss a
query's cluster: every cell reports hashed seeds and seeds from the IVF probe (the first itopk documents of the query's
best IVF list) side by side.

Build: GraphIndex.build's three phases timed apart (exact self k-NN lists of 64, detour pruning to degree 32, reverse-edge
merge).  Search cells: queries 1 / 16 / 128 / 1024 x itopk 32 / 64 / 128 / 256, k = min(100, itopk), default
max_iterations and num_seeds.  In each cell the graph search (both seedings), IVFIndex.search at nprobe 8 and 32 and the
exact search are timed alternately with CUDA events after warm-up (median of 5 rounds, with min and max).  Recall@10 /
@100 are against the exact search (@100 only where k = 100).  "visited_hbm_share" is the visited rows' bytes (row +
scale + 4 degree bytes of edges) at 3.35 TB/s (H100 SXM data sheet) over the hashed-seed search time.

--big adds 10M x 768 low-dimensional rows whose graph is built with GraphIndex.from_knn from IVFIndex.search of the rows
(nlist 12648, nprobe 8), timed the same way at itopk 64 and 128.  The card name and power limit are read in the same run."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sgpt_b200 import CorpusShard, GraphIndex, IVFIndex  # noqa: E402
from sgpt_b200.graph import default_max_iterations, merge_reverse, prune, self_knn  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
REPEATS = 5
NQS = (1, 16, 128, 1024)
ITOPKS = (32, 64, 128, 256)
DEGREE, KNN = 32, 64


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        limit = f"unknown ({e})"
    return {"gpu": name, "power_limit": limit}


def time_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def alternate(fns):
    """{name: (median, min, max) ms}: REPEATS rounds, every fn timed once per round in turn, ~40 ms per window."""
    steps = {}
    for name, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        steps[name] = max(2, min(1000, int(40 / max(time_ms(fn, 2), 1e-3))))
    times = {name: [] for name in fns}
    for _ in range(REPEATS):
        for name, fn in fns.items():
            times[name].append(time_ms(fn, steps[name]))
    return {name: (statistics.median(t), min(t), max(t)) for name, t in times.items()}


def clustered(n, D, nlist, nq, g, slab=500_000):
    centres = torch.randn(nlist, D, generator=g, device="cuda")
    shard = CorpusShard(D, n, device="cuda:0")
    for s0 in range(0, n, slab):
        m = min(slab, n - s0)
        c = centres[torch.randint(nlist, (m,), generator=g, device="cuda")]
        c += torch.randn(m, D, generator=g, device="cuda")
        shard.add(c)
        del c
    q = centres[torch.randint(nlist, (nq,), generator=g, device="cuda")]
    q += torch.randn(q.shape, generator=g, device="cuda")
    return shard, q


def lowdim(n, D, nq, g, slab=500_000):
    G = torch.randn(D, 16, generator=g, device="cuda")
    shard = CorpusShard(D, n, device="cuda:0")

    def draw(m):
        return torch.randn(m, 16, generator=g, device="cuda") @ G.T + 0.1 * torch.randn(m, D, generator=g, device="cuda")
    for s0 in range(0, n, slab):
        shard.add(draw(min(slab, n - s0)))
    return shard, draw(nq)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, round(time.perf_counter() - t0, 2)


def ivf_seeds(ivf, q, s):
    """The first s documents (global ids) of each query's best IVF list, -1 past the list's end."""
    lists = ivf.probe(q, 1)[:, 0].long()
    start = ivf.offsets[lists]
    length = ivf.offsets[lists + 1] - start
    j = torch.arange(s, device=q.device)
    pos = (start[:, None] + j).clamp(max=ivf.n - 1)
    return torch.where(j < length[:, None], ivf.ids[pos].long(), -1)


def recall(got, exact, kk):
    hit = sum(len(set(a[:kk]) & set(b[:kk])) for a, b in zip(got.tolist(), exact.tolist()))
    return round(hit / (exact.shape[0] * kk), 4)


def cells(name, shard, index, ivf, q, itopks=ITOPKS):
    row_bytes = shard.dim * 2 + 4 + 4 * index.degree
    rows = []
    for nq in NQS:
        qq = q[:nq].contiguous()
        _, exact_i = shard.search(qq, 100, "cos_sim")
        for itopk in itopks:
            k = min(100, itopk)

            def hashed():
                return index.search(qq, k, itopk=itopk)

            def seeded():
                return index.search(qq, k, itopk=itopk, seeds=ivf_seeds(ivf, qq, itopk))
            t = alternate({"graph_hashed": hashed, "graph_ivf_seeds": seeded,
                           "ivf_nprobe8": lambda: ivf.search(qq, k, 8), "ivf_nprobe32": lambda: ivf.search(qq, k, 32),
                           "exact": lambda: shard.search(qq, k, "cos_sim")})
            _, hi, hv = index.search(qq, k, itopk=itopk, return_visited=True)
            _, si, sv = index.search(qq, k, itopk=itopk, seeds=ivf_seeds(ivf, qq, itopk), return_visited=True)
            row = {"case": name, "queries": nq, "itopk": itopk, "k": k,
                   "max_iterations": default_max_iterations(itopk, 1, index.degree, itopk)}
            for fn, (med, lo, hi_) in t.items():
                row[f"{fn}_ms"] = round(med, 4)
                row[f"{fn}_ms_min_max"] = [round(lo, 4), round(hi_, 4)]
            for tag, ids, vis in (("hashed", hi, hv), ("ivf_seeds", si, sv)):
                row[f"recall_at_10_{tag}"] = recall(ids, exact_i, 10)
                row[f"recall_at_100_{tag}"] = recall(ids, exact_i, 100) if k == 100 else None
                row[f"mean_visited_{tag}"] = round(float(vis.double().mean()), 1)
            for ivf_np in (8, 32):
                _, ii = ivf.search(qq, k, ivf_np)
                row[f"recall_at_10_ivf_nprobe{ivf_np}"] = recall(ii, exact_i, 10)
            floor_ms = row["mean_visited_hashed"] * nq * row_bytes / HBM_BYTES_PER_S * 1e3
            row["visited_hbm_share"] = round(floor_ms / t["graph_hashed"][0], 4)
            row["speedup_hashed_vs_exact"] = round(t["exact"][0] / t["graph_hashed"][0], 2)
            row["speedup_hashed_vs_ivf_nprobe8"] = round(t["ivf_nprobe8"][0] / t["graph_hashed"][0], 2)
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def case_1m(name, shard, q):
    n = shard.n
    knn, t_knn = timed(lambda: self_knn(shard, KNN, "cos_sim"))
    pruned, t_prune = timed(lambda: prune(knn - shard.id_base, DEGREE))
    graph, t_merge = timed(lambda: merge_reverse(pruned))
    index = GraphIndex(shard, graph, "cos_sim")
    del knn, pruned
    nlist = int(round(4 * math.sqrt(n) / 8)) * 8
    ivf, t_ivf = timed(lambda: IVFIndex.build(shard, nlist, seed=0, train_size=min(n, 40 * nlist)))
    head = {"case": name, "n": n, "dim": shard.dim, "degree": DEGREE, "knn": KNN, "build_knn_s": t_knn,
            "build_prune_s": t_prune, "build_merge_s": t_merge, "ivf_nlist": nlist, "ivf_build_s": t_ivf,
            "graph_nbytes": index.nbytes}
    print(json.dumps(head), flush=True)
    rows = cells(name, shard, index, ivf, q)
    del index, ivf
    torch.cuda.empty_cache()
    return head, rows


def case_10m(g):
    n, D = 10_000_000, 768
    shard, q = lowdim(n, D, max(NQS), g)
    nlist = int(round(4 * math.sqrt(n) / 8)) * 8
    ivf, t_ivf = timed(lambda: IVFIndex.build(shard, nlist, seed=0, train_size=40 * nlist))

    def knn_from_ivf():
        out = torch.empty((n, KNN), dtype=torch.int64, device="cuda")
        for a in range(0, n, 65536):
            pos = torch.arange(a, min(a + 65536, n), device="cuda")
            ids = ivf.search(shard.vectors.index_select(0, pos), KNN + 1, 8)[1]
            own = (ids == pos[:, None]).to(torch.int8)
            out[a:a + len(pos)] = torch.gather(ids, 1, torch.sort(own, dim=1, stable=True)[1])[:, :KNN]
        return out
    knn, t_knn = timed(knn_from_ivf)
    index, t_graph = timed(lambda: GraphIndex.from_knn(shard, knn, DEGREE))
    del knn
    head = {"case": "lowdim 10M (from_knn of IVFIndex.search, nprobe 8)", "n": n, "ivf_nlist": nlist,
            "ivf_build_s": t_ivf, "build_knn_s": t_knn, "build_prune_merge_s": t_graph, "graph_nbytes": index.nbytes}
    print(json.dumps(head), flush=True)
    return head, cells("lowdim 10M", shard, index, ivf, q, itopks=(64, 128))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    ap.add_argument("--big", action="store_true", help="add the 10M x 768 leg built with from_knn")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_graph measures the GPU; there is no CPU path"
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "builds": [], "cells": []}
    print(json.dumps(res["card"]), flush=True)
    for name, make in (("clustered 1M", lambda: clustered(1_000_000, 768, 4000, max(NQS), g)),
                       ("lowdim 1M", lambda: lowdim(1_000_000, 768, max(NQS), g))):
        shard, q = make()
        head, rows = case_1m(name, shard, q)
        res["builds"].append(head)
        res["cells"] += rows
        del shard, q
        torch.cuda.empty_cache()
    if a.big:
        head, rows = case_10m(g)
        res["builds"].append(head)
        res["cells"] += rows
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
