"""Cost of filters in the IVF search, and of growing an index with add(), on planted-cluster corpora.

    python tools/bench_ivf_masked.py [--out result.json]

Corpus and index as in tools/bench_ivf.py: 1M x 768, a bf16 and an int8 shard, nlist = 4 sqrt(n) rounded to a multiple
of 8.  For every (queries, nprobe) cell, nq in (1, 16, 128) and nprobe in (8, 32), the scan + select (the entry point
with the probes and query rows prepared once) is timed for five legs, alternately with CUDA events after warm-up launches
(median of REPEATS rounds, with min and max):
  unmasked       sgpt_ivf_search, no mask
  shared_ones    sgpt_ivf_search_masked, one all-ones bitmap (pitch 0)
  shared_50      one bitmap with a random half of the rows
  perq_ones      one all-ones bitmap per query (pitch ceil(n/32))
  perq_1pct      one bitmap per query with a random 1 % of the rows
"perq_ones_over_unmasked" is the per-query leg's median over the unmasked one: the cost of reading per-query bitmaps in
the scan.  add(): one warm-up add of 1 000 rows, then one timed add of 10 000 and one of 100 000 rows (host clock around
the call and a device synchronise; single runs).  The card name and power limit are read in the same run."""
import argparse
import json
import math
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_ivf import alternate, card, planted  # noqa: E402
from sgpt_b200 import IVFIndex, _lib  # noqa: E402
from sgpt_b200.index import pack_mask  # noqa: E402

K = 100
NQS = (1, 16, 128)
NPROBES = (8, 32)


def scan_calls(index, q, nprobe, masks):
    """{leg: fn}: the scan + select of index.search for each (mask, pitch) of `masks` (None: sgpt_ivf_search)."""
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
    common = (dt, qb.data_ptr(), index.shard.vectors.data_ptr(), _lib.ptr(q_scale), c_scale, nq, index.n, index.dim,
              index.offsets.data_ptr(), index.nlist, index.max_list_len, index.ids.data_ptr(), probes.data_ptr(), nprobe,
              K)
    tail = (out_s.data_ptr(), out_i.data_ptr(), ws.data_ptr(), ws.numel(), stream)

    def leg(m):
        if m is None:
            return lambda: _lib.check(lib.sgpt_ivf_search(*common, None, *tail), "sgpt_ivf_search")
        bits, pitch = m
        return lambda: _lib.check(lib.sgpt_ivf_search_masked(*common, bits.data_ptr(), pitch, *tail),
                                  "sgpt_ivf_search_masked")
    return {name: leg(m) for name, m in masks.items()}


def case(n, D, dtype, g):
    nlist = int(round(4 * math.sqrt(n) / 8)) * 8
    src, q = planted(n, D, nlist, dtype, g)
    index = IVFIndex.build(src, nlist, seed=0, train_size=min(n, 40 * nlist))
    del src
    torch.cuda.empty_cache()
    head = {"case": f"{n // 10**6}M x {D} {dtype}", "nlist": nlist, "max_list_len": index.max_list_len}
    print(json.dumps(head), flush=True)
    rows = []
    ones = torch.ones(n, dtype=torch.bool, device="cuda")
    for nq in NQS:
        qq = q[:nq].contiguous()
        words = (n + 31) // 32
        masks = {"unmasked": None,
                 "shared_ones": (pack_mask(ones), 0),
                 "shared_50": (pack_mask(torch.rand(n, generator=g, device="cuda") < 0.5), 0),
                 "perq_ones": (pack_mask(ones.expand(nq, n)), words),
                 "perq_1pct": (pack_mask(torch.rand(nq, n, generator=g, device="cuda") < 0.01), words)}
        for nprobe in NPROBES:
            t = alternate(scan_calls(index, qq, nprobe, masks))
            row = dict(head, queries=nq, nprobe=nprobe, k=K)
            for name, (med, lo, hi) in t.items():
                row[f"{name}_ms"] = round(med, 4)
                row[f"{name}_ms_min_max"] = [round(lo, 4), round(hi, 4)]
            row["perq_ones_over_unmasked"] = round(t["perq_ones"][0] / t["unmasked"][0], 3)
            rows.append(row)
            print(json.dumps(row), flush=True)
        del masks
    adds = []
    for m in (1000, 10_000, 100_000):
        x = q[torch.randint(q.shape[0], (m,), generator=g, device="cuda")]
        x += torch.randn(x.shape, generator=g, device="cuda")
        n0 = index.n
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        index.add(x)
        torch.cuda.synchronize()
        if m > 1000:  # the first add is the warm-up
            adds.append({"case": head["case"], "add_rows": m, "n_before": n0, "add_s": round(time.perf_counter() - t0, 3)})
            print(json.dumps(adds[-1]), flush=True)
        del x
    del index
    torch.cuda.empty_cache()
    return rows, adds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ivf_masked measures the GPU; there is no CPU path"
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "cases": [], "add": []}
    print(json.dumps(res["card"]), flush=True)
    for dtype in ("bf16", "int8"):
        rows, adds = case(1_000_000, 768, dtype, g)
        res["cases"] += rows
        res["add"] += adds
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
