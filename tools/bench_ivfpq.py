"""IVF-PQ index vs IVF index vs exact search on planted-cluster corpora: time per search, recall, bytes per document.

    python tools/bench_ivfpq.py [--out result.json] [--leg grid|scale|all]

Corpus: `nlist` random centres (randn), every document a centre plus unit-variance noise, every query another draw around
a random centre.  Grid: 1M x 768 with nlist 4000, m in {48, 96}, queries {1, 16, 128}, nprobe {8, 32, 128}, k = 100.  Per
cell the IVF-PQ search is split into probe (exact search over the centroids), tables (sgpt_pq_tables) and scan + select
(sgpt_ivfpq_search with tables precomputed), plus the refine pass (sgpt_rerank of k_refine = 10 k candidates) against the
bf16 and the int8 shard of the same rows; IVFIndex (bf16, int8) and the exact bf16 search run on the same data.  Every
function is timed with CUDA events after warm-up launches, alternately, median of REPEATS rounds with min and max.
Recall@10 / @100 are against the exact bf16 top-100.  "floor_bytes" are the codes and ids of the distinct probed lists
plus the candidate slots (8 bytes written by the scan and read by the selection per probed document), and
"scan_share_of_hbm_floor" their time at 3.35 TB/s (H100 SXM data sheet) over the scan + select time.

Scale leg: 50M x 768, m = 96, nlist 8192, built with train (262144 rows of the first chunk) + add of
1M-row chunks generated on the device; an int8 shard of the same rows (38 GB; bf16 would not fit next to it) is the exact
reference.  It reports the device memory peak (torch.cuda.max_memory_allocated), build time, search times and recall for
1 and 16 queries: the exact search's workspace for 128 queries over 50M documents (~48 GB) does not fit next to the shard.
The card name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sgpt_b200 import CorpusShard, IVFIndex, IVFPQIndex  # noqa: E402
from sgpt_b200.ivfpq import rerank  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
K = 100
REPEATS = 5
NQS = (1, 16, 128)
NPROBES = (8, 32, 128)
SCALE_NQS = (1, 16)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        limit = f"unknown ({e})"
    return {"gpu": name, "power_limit": limit}


def rows_of(centres, m, g):
    x = centres[torch.randint(centres.shape[0], (m,), generator=g, device="cuda")]
    x += torch.randn(x.shape, generator=g, device="cuda")
    return x


def time_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def alternate(fns):
    """{name: (median, min, max) ms}: REPEATS rounds, every fn timed once per round in turn, ~50 ms per window."""
    steps = {}
    for name, fn in fns.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        steps[name] = max(3, min(2000, int(50 / max(time_ms(fn, 3), 1e-3))))
    times = {name: [] for name in fns}
    for _ in range(REPEATS):
        for name, fn in fns.items():
            times[name].append(time_ms(fn, steps[name]))
    return {name: (statistics.median(t), min(t), max(t)) for name, t in times.items()}


def recall(got, exact, kk):
    return sum(len(set(a[:kk]) & set(b[:kk])) for a, b in zip(got.tolist(), exact.tolist())) / (exact.shape[0] * kk)


def put(row, t):
    for name, (med, lo, hi) in t.items():
        row[f"{name}_ms"] = round(med, 4)
        row[f"{name}_ms_min_max"] = [round(lo, 4), round(hi, 4)]


def grid():
    n, D, nlist = 1_000_000, 768, 4000
    g = torch.Generator(device="cuda").manual_seed(0)
    centres = torch.randn(nlist, D, generator=g, device="cuda")
    emb = rows_of(centres, n, g)
    q = rows_of(centres, max(NQS), g)
    src = {dt: CorpusShard.from_embeddings(emb, dtype=dt) for dt in ("bf16", "int8")}
    del emb
    ivf = {dt: IVFIndex.build(src[dt], nlist, seed=0, train_size=40 * nlist) for dt in ("bf16", "int8")}
    rows = []
    for m in (48, 96):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        index = IVFPQIndex.build(src["bf16"], nlist, m, seed=0, train_size=40 * nlist)
        torch.cuda.synchronize()
        head = {"case": f"1M x {D}", "nlist": nlist, "m": m, "build_s": round(time.perf_counter() - t0, 2),
                "bytes_per_doc": m + 8, "index_nbytes": index.nbytes, "max_list_len": index.max_list_len}
        print(json.dumps(head), flush=True)
        sizes = index.list_sizes.double()
        for nq in NQS:
            qq = q[:nq].contiguous()
            exact_i = src["bf16"].search(qq, K, "cos_sim")[1]
            for nprobe in NPROBES:
                probes = index.probe(qq, nprobe)
                lut, base = index.tables(qq, probes)
                cand = index.search(qq, 10 * K if 10 * K <= 4096 else 4096, nprobe)[1]
                t = alternate({
                    "exact": lambda: src["bf16"].search(qq, K, "cos_sim"),
                    "ivf_bf16": lambda: ivf["bf16"].search(qq, K, nprobe),
                    "ivf_int8": lambda: ivf["int8"].search(qq, K, nprobe),
                    "ivfpq": lambda: index.search(qq, K, nprobe),
                    "probe": lambda: index.probe(qq, nprobe),
                    "tables": lambda: index.tables(qq, probes),
                    "scan_select": lambda: index.scan(lut, base, probes, K),
                    "refine_bf16": lambda: rerank(src["bf16"], qq, cand, K),
                    "refine_int8": lambda: rerank(src["int8"], qq, cand, K)})
                pq_i = index.search(qq, K, nprobe)[1]
                ref_i = index.search(qq, K, nprobe, refine=src["bf16"], k_refine=10 * K)[1]
                ref8_i = index.search(qq, K, nprobe, refine=src["int8"], k_refine=10 * K)[1]
                lists = torch.unique(probes.long().cpu())
                probed_docs = int(sizes[probes.long().cpu()].sum())
                floor = int(sizes[lists].sum()) * (m + 4) + probed_docs * 16
                row = dict(head, queries=nq, nprobe=nprobe, k=K, k_refine=10 * K)
                put(row, t)
                row["floor_bytes"] = floor
                row["scan_share_of_hbm_floor"] = round(floor / HBM_BYTES_PER_S * 1e3 / t["scan_select"][0], 3)
                row["speedup_vs_exact"] = round(t["exact"][0] / t["ivfpq"][0], 2)
                for name, ids in (("pq", pq_i), ("refine_bf16", ref_i), ("refine_int8", ref8_i)):
                    row[f"recall_at_10_{name}"] = round(recall(ids, exact_i, 10), 4)
                    row[f"recall_at_100_{name}"] = round(recall(ids, exact_i, 100), 4)
                rows.append(row)
                print(json.dumps(row), flush=True)
        del index
    del ivf, src
    torch.cuda.empty_cache()
    return rows


def scale_leg():
    n, D, nlist, m, chunk = 50_000_000, 768, 8192, 96, 1_000_000
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device="cuda").manual_seed(1)
    centres = torch.randn(nlist, D, generator=g, device="cuda")
    q = rows_of(centres, max(NQS), g)
    shard = CorpusShard(D, n, device="cuda:0", dtype="int8")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    index = None
    for c0 in range(0, n, chunk):
        x = rows_of(centres, chunk, g)
        if index is None:
            sample = x[torch.randperm(chunk, device="cuda", generator=g)[:262144]]
            index = IVFPQIndex.train(sample, nlist, m, seed=0)
            del sample
            torch.cuda.synchronize()
            train_s = time.perf_counter() - t0
        index.add(x)
        shard.add(x)
        del x
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    head = {"case": f"50M x {D}", "nlist": nlist, "m": m, "train_s": round(train_s, 2),
            "build_s_incl_int8_shard": round(build_s, 2), "index_nbytes": index.nbytes,
            "int8_shard_bytes": n * (D + 8), "max_memory_allocated": torch.cuda.max_memory_allocated()}
    print(json.dumps(head), flush=True)
    rows = []
    for nq in SCALE_NQS:
        qq = q[:nq].contiguous()
        exact_i = shard.search(qq, K, "cos_sim")[1]
        for nprobe in (8, 32):
            t = alternate({"exact_int8": lambda: shard.search(qq, K, "cos_sim"),
                           "ivfpq": lambda: index.search(qq, K, nprobe),
                           "ivfpq_refine_int8": lambda: index.search(qq, K, nprobe, refine=shard, k_refine=10 * K)})
            row = dict(head, queries=nq, nprobe=nprobe, k=K)
            put(row, t)
            for name, ids in (("pq", index.search(qq, K, nprobe)[1]),
                              ("refine_int8", index.search(qq, K, nprobe, refine=shard, k_refine=10 * K)[1])):
                row[f"recall_at_10_{name}"] = round(recall(ids, exact_i, 10), 4)
                row[f"recall_at_100_{name}"] = round(recall(ids, exact_i, 100), 4)
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    ap.add_argument("--leg", choices=("grid", "scale", "all"), default="all", help="the 1M x 768 grid, the 50M leg or both")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivfpq measures the GPU; there is no CPU path"
    res = {"card": card()}
    print(json.dumps(res["card"]), flush=True)
    if a.leg in ("grid", "all"):
        res["grid"] = grid()
    if a.leg in ("scale", "all"):
        res["scale"] = scale_leg()
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
