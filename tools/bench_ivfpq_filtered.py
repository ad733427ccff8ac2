"""Filtered IVF-PQ search (IVFPQIndex.search(allow=)): what a shared or per-query filter costs the scan and the whole
search, and the recall of the filtered search against the exact filtered search.

    python tools/bench_ivfpq_filtered.py [--out result.json]

Data: tools/bench_ivfpq.py's grid corpus, 1M x 768 planted clusters (4000 centres, unit noise), nlist 4000; one bf16
shard and two indexes built from it with the same seed (so with the same centroids and probes): 8-bit m = 48 and 4-bit
m = 96, 56 bytes per document each.  k = 100.

Scan: ``scan`` (scan + select) with the tables precomputed, at queries {1, 16, 128} x nprobe {8, 32}, for five filters,
timed alternately with device events, median of 5 rounds with min and max: none (deletions only, here none), shared
all-ones, shared 50 %, per-query all-ones and per-query 1 %.  The bitmaps are packed before timing.  "pq_ones_cost" is
the per-query all-ones median over the unfiltered one, minus 1: what reading one bitmap per query costs when it filters
nothing.

End to end: ``search`` (probe, tables, packing the filter, scan) unfiltered, with a shared 10 % filter and with a
per-query 10 % filter, same grid, same timing.

Recall: recall@10 at 128 queries against the exact filtered search (``CorpusShard.search(allow=)``) of the same shard,
for shared filters allowing 50 %, 10 % and 1 % of the documents, at nprobe 8 and 32, without and with refine (the bf16
shard, 1000 candidates).  The probes ignore the filter, so a selective filter leaves few allowed documents in the probed
lists.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sgpt_b200 import CorpusShard, IVFPQIndex  # noqa: E402
from tools.bench_ivfpq import K, NQS, alternate, card, put, recall, rows_of  # noqa: E402

NPROBES = (8, 32)
CODES = ((8, 48), (4, 96))  # (nbits, m): equal bytes per document
RECALL_SHARES = (0.5, 0.1, 0.01)


def filters(n, nq, g):
    """The scan leg's filters in document order (None: unfiltered)."""
    ones = torch.ones(n, dtype=torch.bool, device="cuda")
    return {"none": None, "shared_ones": ones, "shared_50": torch.rand(n, generator=g, device="cuda") < 0.5,
            "pq_ones": ones.expand(nq, n).contiguous(),
            "pq_1": torch.rand((nq, n), generator=g, device="cuda") < 0.01}


def spread(t):
    return round(max((hi - lo) / med for med, lo, hi in t.values()), 3)


def scan_cells(index, q, g):
    rows = []
    for nq in NQS:
        qq = q[:nq].contiguous()
        masks = {name: index._list_mask(a, nq) for name, a in filters(index.n, nq, g).items()}
        for nprobe in NPROBES:
            probes = index.probe(qq, nprobe)
            lut, base = index.tables(qq, probes)
            t = alternate({name: (lambda mk=mk: index.scan(lut, base, probes, K, mk)) for name, mk in masks.items()})
            row = {"leg": "scan", "nbits": index.nbits, "m": index.m, "queries": nq, "nprobe": nprobe, "k": K}
            put(row, t)
            row["pq_ones_cost"] = round(t["pq_ones"][0] / t["none"][0] - 1, 4)
            row["spread"] = spread(t)
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def search_cells(index, q, g):
    rows = []
    for nq in NQS:
        qq = q[:nq].contiguous()
        shared = torch.rand(index.n, generator=g, device="cuda") < 0.1
        per_query = torch.rand((nq, index.n), generator=g, device="cuda") < 0.1
        for nprobe in NPROBES:
            t = alternate({"none": lambda: index.search(qq, K, nprobe),
                           "shared_10": lambda: index.search(qq, K, nprobe, allow=shared),
                           "pq_10": lambda: index.search(qq, K, nprobe, allow=per_query)})
            row = {"leg": "search", "nbits": index.nbits, "m": index.m, "queries": nq, "nprobe": nprobe, "k": K}
            put(row, t)
            row["spread"] = spread(t)
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def recall_cells(index, src, q, g):
    rows = []
    for share in RECALL_SHARES:
        a = torch.rand(index.n, generator=g, device="cuda") < share
        exact = src.search(q, 10, "cos_sim", allow=a)[1]
        for nprobe in NPROBES:
            pq = index.search(q, K, nprobe, allow=a)[1]
            ref = index.search(q, K, nprobe, refine=src, k_refine=10 * K, allow=a)[1]
            row = {"leg": "recall", "nbits": index.nbits, "m": index.m, "queries": q.shape[0], "nprobe": nprobe,
                   "share": share, "recall_at_10_pq": round(recall(pq, exact, 10), 4),
                   "recall_at_10_refine_bf16": round(recall(ref, exact, 10), 4),
                   "mean_returned_pq": round(float((pq >= 0).sum(1).float().mean()), 1)}
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivfpq_filtered measures the GPU; there is no CPU path"
    res = {"card": card()}
    print(json.dumps(res["card"]), flush=True)
    n, D, nlist = 1_000_000, 768, 4000
    g = torch.Generator(device="cuda").manual_seed(0)
    centres = torch.randn(nlist, D, generator=g, device="cuda")
    src = CorpusShard.from_embeddings(rows_of(centres, n, g), dtype="bf16")
    q = rows_of(centres, max(NQS), g)
    res["rows"] = []
    for nbits, m in CODES:
        index = IVFPQIndex.build(src, nlist, m, seed=0, train_size=40 * nlist, nbits=nbits)
        gf = torch.Generator(device="cuda").manual_seed(1)
        res["rows"] += scan_cells(index, q, gf) + search_cells(index, q, gf) + recall_cells(index, src, q, gf)
        del index
    res["card_after"] = card()
    print(json.dumps(res["card_after"]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
