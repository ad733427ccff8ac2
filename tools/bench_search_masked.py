"""Cost of the document mask: the unmasked search against masked searches of the same shard, alternated.

    python tools/bench_search_masked.py [--out result.json] [--quick]

128 queries over 1M x 768 and 1M x 4096 documents, on a bf16 and an int8 shard of the same documents (the corpus of
bench_search_int8.py: randn rows, every 100th a query plus noise).  Each round times, with CUDA events, the unmasked
entry point and the masked entry point with an all-ones shared mask, shared random masks at 50 % and 1 %, and per-query
random 1 % masks; the bitmaps are built before timing, so only the search is measured.  The reported time is the median
of the rounds.  The all-ones row answers whether the masked epilogue costs anything by itself (its results are checked
to equal the unmasked ones bit for bit); the selective rows show the price of fewer front-list survivors.  The card
name and its power limit are read in the same run."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sgpt_b200 import CorpusShard, _lib  # noqa: E402
from sgpt_b200.index import pack_mask  # noqa: E402
from tools.bench_search_int8 import card, fill, time_ms  # noqa: E402

K = 1001
NQ = 128
ROUNDS = 7


def masks(n, g):
    """name -> (bitmap or None, pitch)."""
    out = {"unmasked": (None, 0), "ones": (pack_mask(torch.ones(n, dtype=torch.bool, device="cuda")), 0)}
    for name, p in (("shared_50pct", 0.5), ("shared_1pct", 0.01)):
        out[name] = (pack_mask(torch.rand(n, generator=g, device="cuda") < p), 0)
    per = pack_mask(torch.rand((NQ, n), generator=g, device="cuda") < 0.01)
    out["per_query_1pct"] = (per, per.shape[1])
    return out


def case(n, D, g):
    q = torch.randn(NQ, D, generator=g, device="cuda")
    shards = {"bf16": CorpusShard(D, n, device="cuda:0"), "int8": CorpusShard(D, n, device="cuda:0", dtype="int8")}
    fill(list(shards.values()), n, D, q, g)
    ms = masks(n, g)
    lib = _lib.lib()
    rows = []
    for dtype, sh in shards.items():
        qb, q_scale, c_scale = sh._prepare(q, K, "cos_sim")
        dt = sh._dtype_id()
        out_s = torch.empty((NQ, K), dtype=torch.float32, device="cuda")
        out_i = torch.empty((NQ, K), dtype=torch.int64, device="cuda")

        def run(mask, pitch, masked=True):
            if masked:
                rc = lib.sgpt_search_masked(dt, qb.data_ptr(), sh.vectors.data_ptr(), _lib.ptr(q_scale), c_scale, NQ,
                                            sh.n, D, K, 0, _lib.ptr(mask), pitch, out_s.data_ptr(), out_i.data_ptr(),
                                            sh._ws.data_ptr(), sh._ws.numel(), _lib.current_stream())
            else:
                fn = lib.sgpt_search_i8 if dtype == "int8" else lib.sgpt_search
                rc = fn(qb.data_ptr(), sh.vectors.data_ptr(), _lib.ptr(q_scale), c_scale, NQ, sh.n, D, K, 0,
                        out_s.data_ptr(), out_i.data_ptr(), sh._ws.data_ptr(), sh._ws.numel(), _lib.current_stream())
            _lib.check(rc, "search")

        run(None, 0, masked=False)
        plain = (out_s.clone(), out_i.clone())
        run(*ms["ones"])
        same = torch.equal(out_s.view(torch.int32), plain[0].view(torch.int32)) and torch.equal(out_i, plain[1])
        fns = {"unmasked": lambda: run(None, 0, masked=False)}
        for name, (m, p) in ms.items():
            if name != "unmasked":
                fns[name] = lambda m=m, p=p: run(m, p)
        for fn in fns.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        steps = 20
        times = {name: [] for name in fns}
        for _ in range(ROUNDS):
            for name, fn in fns.items():
                times[name].append(time_ms(fn, steps))
        row = {"case": f"{n // 10**6}M x {D}", "dtype": dtype, "queries": NQ, "k": K,
               "all_ones_equals_unmasked": same}
        for name, t in times.items():
            row[f"{name}_ms"] = round(statistics.median(t), 4)
            row[f"{name}_spread_ms"] = round(max(t) - min(t), 4)
        print(json.dumps(row), flush=True)
        rows.append(row)
    del shards
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    ap.add_argument("--quick", action="store_true", help="only the 1M x 768 case")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_search_masked measures the GPU; there is no CPU path"
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card(), "cases": []}
    print(json.dumps(res["card"]), flush=True)
    res["cases"] += case(1_000_000, 768, g)
    if not a.quick:
        res["cases"] += case(1_000_000, 4096, g)
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
