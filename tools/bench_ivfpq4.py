"""4-bit against 8-bit IVF-PQ codes on a planted-cluster corpus: scan + select and table times, share of the HBM floor,
recall with and without refine.

    python tools/bench_ivfpq4.py [--out result.json]

Corpus: 1M x 768, `nlist` = 4000 random centres (randn), every document a centre plus unit-variance noise, every query
another draw around a random centre (tools/bench_ivfpq.py's grid data).  Three indexes are built from the same bf16
shard with the same seed and training rows, so they share their coarse centroids and every query's probes:
  4-bit m = 96 (56 bytes per document), 8-bit m = 48 (equal bytes: 56) and 8-bit m = 96 (equal m: 104).
Per queries {1, 16, 128} x nprobe {8, 32, 128}, k = 100, the three scans (``scan``: sgpt_ivfpq_search_nbits with the
tables precomputed) are timed alternately with CUDA events after warm-up, median of REPEATS rounds with min and max,
and so are the three table builds (``tables``: sgpt_pq_tables_nbits).  "floor_bytes" are the codes and ids of the distinct
probed lists plus the candidate slots (8 bytes written by the scan and read by the selection per probed document), and
"share_of_hbm_floor" their time at 3.35 TB/s (H100 SXM data sheet) over the scan + select time.  Recall@10 / @100 are
against the exact bf16 top-100, of the PQ pass alone and with refine against the bf16 shard (k_refine = 10 k).  The card
name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sgpt_b200 import CorpusShard, IVFPQIndex  # noqa: E402
from tools.bench_ivfpq import HBM_BYTES_PER_S, K, NPROBES, NQS, alternate, card, put, recall, rows_of  # noqa: E402

LEGS = (("pq4_m96", 96, 4), ("pq8_m48", 48, 8), ("pq8_m96", 96, 8))


def grid():
    n, D, nlist = 1_000_000, 768, 4000
    g = torch.Generator(device="cuda").manual_seed(0)
    centres = torch.randn(nlist, D, generator=g, device="cuda")
    emb = rows_of(centres, n, g)
    q = rows_of(centres, max(NQS), g)
    src = CorpusShard.from_embeddings(emb, dtype="bf16")
    del emb
    index, heads = {}, {}
    for name, m, nbits in LEGS:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        index[name] = IVFPQIndex.build(src, nlist, m, seed=0, train_size=40 * nlist, nbits=nbits)
        torch.cuda.synchronize()
        heads[name] = {"m": m, "nbits": nbits, "bytes_per_doc": m * nbits // 8 + 8,
                       "build_s": round(time.perf_counter() - t0, 2), "index_nbytes": index[name].nbytes}
        print(json.dumps(dict(heads[name], leg=name)), flush=True)
    first = index[LEGS[0][0]]
    assert all(torch.equal(first.centroids, index[nm].centroids) for nm, _, _ in LEGS)
    sizes = first.list_sizes.double()
    rows = []
    for nq in NQS:
        qq = q[:nq].contiguous()
        exact_i = src.search(qq, K, "cos_sim")[1]
        for nprobe in NPROBES:
            probes = first.probe(qq, nprobe)
            tabs = {nm: index[nm].tables(qq, probes) for nm, _, _ in LEGS}
            fns = {}
            for nm, _, _ in LEGS:
                fns[f"scan_{nm}"] = (lambda ix, t: lambda: ix.scan(t[0], t[1], probes, K))(index[nm], tabs[nm])
            for nm, _, _ in LEGS:
                fns[f"tables_{nm}"] = (lambda ix: lambda: ix.tables(qq, probes))(index[nm])
            t = alternate(fns)
            row = {"case": f"1M x {D}", "nlist": nlist, "queries": nq, "nprobe": nprobe, "k": K, "k_refine": 10 * K}
            put(row, t)
            lists = torch.unique(probes.long().cpu())
            probed_docs = int(sizes[probes.long().cpu()].sum())
            row["probed_docs"] = probed_docs
            for nm, m, nbits in LEGS:
                floor = int(sizes[lists].sum()) * (m * nbits // 8 + 4) + probed_docs * 16
                row[f"floor_bytes_{nm}"] = floor
                row[f"share_of_hbm_floor_{nm}"] = round(floor / HBM_BYTES_PER_S * 1e3 / t[f"scan_{nm}"][0], 3)
                row[f"scores_per_s_{nm}"] = round(probed_docs / (t[f"scan_{nm}"][0] * 1e-3), 0)
                pq_i = index[nm].search(qq, K, nprobe)[1]
                ref_i = index[nm].search(qq, K, nprobe, refine=src, k_refine=10 * K)[1]
                for what, ids in (("pq", pq_i), ("refine", ref_i)):
                    row[f"recall_at_10_{what}_{nm}"] = round(recall(ids, exact_i, 10), 4)
                    row[f"recall_at_100_{what}_{nm}"] = round(recall(ids, exact_i, 100), 4)
            row["scan_speedup_pq4_vs_pq8_m48"] = round(t["scan_pq8_m48"][0] / t["scan_pq4_m96"][0], 2)
            row["scan_speedup_pq4_vs_pq8_m96"] = round(t["scan_pq8_m96"][0] / t["scan_pq4_m96"][0], 2)
            rows.append(row)
            print(json.dumps(row), flush=True)
    return {"indexes": heads, "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivfpq4 measures the GPU; there is no CPU path"
    res = {"card": card()}
    print(json.dumps(res["card"]), flush=True)
    res["grid"] = grid()
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
