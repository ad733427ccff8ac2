"""IVF index vs exact search on planted-cluster corpora: time per search, bytes scanned, recall, build time.

    python tools/bench_ivf.py [--out result.json] [--quick]

Corpus: `nlist` random centres (randn), every document a centre plus unit-variance noise, every query another draw around
a random centre; nlist = 4 sqrt(n) rounded to a multiple of 8.  Cases: 1M x 768 and 10M x 768, each as a bf16 and an int8
shard.  For every (queries, nprobe) cell the IVF search and the exact search of the same source shard are timed
alternately with CUDA events after warm-up launches (median of REPEATS rounds, with min and max); the IVF time is split
into the probe (exact search over the centroids) and the scan + select (sgpt_ivf_search with the probes precomputed).
"probed_list_bytes" are the bytes of the distinct lists the batch probes (rows + scales + ids), and
"share_of_hbm_floor" their time at 3.35 TB/s (H100 SXM data sheet) over the scan + select time.  Recall@10 / @100 are
against the exact top-100 of the same shard.  The card name and power limit are read in the same run."""
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

from sgpt_b200 import CorpusShard, IVFIndex, _lib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
K = 100
REPEATS = 5
NQS = (1, 16, 128)
NPROBES = (1, 8, 32, 128)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        limit = f"unknown ({e})"
    return {"gpu": name, "power_limit": limit}


def planted(n, D, nlist, dtype, g, slab=500_000):
    centres = torch.randn(nlist, D, generator=g, device="cuda")
    shard = CorpusShard(D, n, device="cuda:0", dtype=dtype)
    for s0 in range(0, n, slab):
        m = min(slab, n - s0)
        c = centres[torch.randint(nlist, (m,), generator=g, device="cuda")]
        c += torch.randn(m, D, generator=g, device="cuda")
        shard.add(c)
        del c
    q = centres[torch.randint(nlist, (max(NQS),), generator=g, device="cuda")]
    q += torch.randn(q.shape, generator=g, device="cuda")
    return shard, q


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


def scan_call(index, q, nprobe):
    """sgpt_ivf_search with the probes and query rows prepared once: the scan + select part of index.search."""
    probes = index.probe(q, nprobe)
    qb, q_scale, c_scale = index.shard._queries(q, index.score_function)
    nq = qb.shape[0]
    dt = index.shard._dtype_id()
    lib = _lib.lib()
    ws = torch.empty(lib.sgpt_ivf_search_workspace_bytes(dt, nq, index.nlist, nprobe, index.max_list_len, index.dim),
                     dtype=torch.uint8, device="cuda")
    out_s = torch.empty((nq, K), dtype=torch.float32, device="cuda")
    out_i = torch.empty((nq, K), dtype=torch.int64, device="cuda")
    stream = _lib.current_stream()

    def run():
        _lib.check(lib.sgpt_ivf_search(dt, qb.data_ptr(), index.shard.vectors.data_ptr(), _lib.ptr(q_scale), c_scale,
                                       nq, index.n, index.dim, index.offsets.data_ptr(), index.nlist, index.max_list_len,
                                       index.ids.data_ptr(), probes.data_ptr(), nprobe, K, None, out_s.data_ptr(),
                                       out_i.data_ptr(), ws.data_ptr(), ws.numel(), stream), "sgpt_ivf_search")
    return run, probes


def case(n, D, dtype, g):
    nlist = int(round(4 * math.sqrt(n) / 8)) * 8
    src, q = planted(n, D, nlist, dtype, g)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    index = IVFIndex.build(src, nlist, seed=0, train_size=min(n, 40 * nlist))
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    sizes = index.list_sizes.double()
    row_bytes = D * (1 if dtype == "int8" else 2) + 4 + 4  # row + scale + id
    head = {"case": f"{n // 10**6}M x {D} {dtype}", "nlist": nlist, "build_s": round(build_s, 2),
            "max_list_len": index.max_list_len, "mean_list_len": round(float(sizes.mean()), 1)}
    print(json.dumps(head), flush=True)
    rows = []
    for nq in NQS:
        qq = q[:nq].contiguous()
        _, exact_i = src.search(qq, K, "cos_sim")
        for nprobe in NPROBES:
            scan, probes = scan_call(index, qq, nprobe)
            t = alternate({"exact": lambda: src.search(qq, K, "cos_sim"),
                           "ivf": lambda: index.search(qq, K, nprobe),
                           "probe": lambda: index.probe(qq, nprobe),
                           "scan_select": scan})
            _, ivf_i = index.search(qq, K, nprobe)
            lists = torch.unique(probes.long())
            probed_bytes = int(sizes[lists.cpu()].sum()) * row_bytes
            rec = {}
            for kk in (10, 100):
                hit = sum(len(set(a[:kk]) & set(b[:kk])) for a, b in zip(ivf_i.tolist(), exact_i.tolist()))
                rec[kk] = hit / (nq * kk)
            row = dict(head, queries=nq, nprobe=nprobe, k=K)
            for name, (med, lo, hi) in t.items():
                row[f"{name}_ms"] = round(med, 4)
                row[f"{name}_ms_min_max"] = [round(lo, 4), round(hi, 4)]
            row["speedup_vs_exact"] = round(t["exact"][0] / t["ivf"][0], 2)
            row["probed_lists"] = int(lists.numel())
            row["probed_list_bytes"] = probed_bytes
            row["share_of_hbm_floor"] = round(probed_bytes / HBM_BYTES_PER_S * 1e3 / t["scan_select"][0], 3)
            row["recall_at_10"] = round(rec[10], 4)
            row["recall_at_100"] = round(rec[100], 4)
            rows.append(row)
            print(json.dumps(row), flush=True)
    del index, src
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    ap.add_argument("--quick", action="store_true", help="only the 1M x 768 cases")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivf measures the GPU; there is no CPU path"
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "cases": []}
    print(json.dumps(res["card"]), flush=True)
    shapes = [(1_000_000, 768)] + ([] if a.quick else [(10_000_000, 768)])
    for n, D in shapes:
        for dtype in ("bf16", "int8"):
            res["cases"] += case(n, D, dtype, g)
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
