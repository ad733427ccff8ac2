"""Binary corpus shards against bf16 and int8 ones on the same planted documents: search time (device events around each
whole call, the formats timed alternately round by round, median and spread of the rounds), how far the tie classes at
the k-th score reach past k, and recall against the exact top-k.

    python tools/bench_search_binary.py --sizes 1000000x768,1000000x4096 --queries 1,16,128 --k 100,1001 --rounds 5
    python tools/bench_search_binary.py --sizes 10000000x4096 --no-bf16
    python tools/bench_search_binary.py --sizes 50000000x4096 --binary-only --queries 1,16

The documents are generated in chunks of 256 k rows straight into every shard (``add``), so no format needs the corpus
as one tensor: a size is limited by the shards it builds.  They carry a large common offset (anisotropic, as mean-pooled
GPT embeddings are) and planted clusters around the queries; each chunk comes from its own seeded generator, so every
format and every run sees the same documents.  Prints the card name and power limit first.

Per (size, queries, k): bf16 / int8 / bits-only / rescore (kc = min(4096, 10 k)) / int8-refine milliseconds (cos_sim,
median thresholds), the bits-only search's share of the HBM floor (n D / 8 + 4 n bytes at 3.35 TB/s) and the spread of
the bits leg.  Ties: for the first 16 queries, the number of documents whose sign dot product is >= the k-th one's,
divided by k — every exact threshold filter admits at least these, so it bounds from below how much the tie classes at
the cut inflate the candidate lists (median and max over the queries).  Recall @10 / @100 of bits only, rescore and
int8 refine (kc = 1000), zero and median thresholds, against the exact bf16 top-100 (int8 with --no-bf16; none with
--binary-only).
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sgpt_b200 import CorpusShard, _lib  # noqa: E402
from sgpt_b200.index import binary_thresholds  # noqa: E402

CHUNK = 1 << 18


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


class Planted:
    """Documents offset + N(0, 1), the first 200 nq of them offset + center[i % nq] + 0.8 N(0, 1); queries offset +
    center + 0.8 N(0, 1).  chunk(i) regenerates rows [i CHUNK, (i + 1) CHUNK) from its own seed."""

    def __init__(self, n, D, nq, seed=0):
        self.n, self.D, self.nq, self.seed = n, D, nq, seed
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.offset = 3.0 * torch.rand(D, device="cuda", generator=g) + 1.0
        self.centers = torch.randn(nq, D, device="cuda", generator=g)
        self.queries = self.centers + 0.8 * torch.randn(nq, D, device="cuda", generator=g) + self.offset
        self.members = min(n, 200 * nq)

    def chunks(self):
        return range((self.n + CHUNK - 1) // CHUNK)

    def chunk(self, i):
        a, b = i * CHUNK, min(self.n, (i + 1) * CHUNK)
        g = torch.Generator(device="cuda").manual_seed(self.seed * 1000003 + i + 1)
        x = torch.randn(b - a, self.D, device="cuda", generator=g)
        m = max(0, min(b, self.members) - a)
        if m:
            x[:m] = self.centers[torch.arange(a, a + m, device="cuda") % self.nq] + 0.8 * x[:m]
        return x.add_(self.offset)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def recall(ids, truth, r):
    return sum(len(set(a[:r]) & set(b[:r])) for a, b in zip(ids.tolist(), truth.tolist())) / (truth.shape[0] * r)


def tie_reach(shard, q, k):
    """Per query: documents with s >= the k-th best s, over k (range search at that query's k-th sign dot product)."""
    s, _ = shard.search(q, k, "dot")
    out = []
    for j in range(q.shape[0]):
        off, _, _ = shard.range_search(q[j:j + 1], float(s[j, k - 1]), "dot")
        out.append(int(off[-1]) / k)
    out.sort()
    return out[len(out) // 2], out[-1]


def run_size(size, nqs, ks, args):
    """One corpus size: build its shards, time the legs, print the tables."""
    n, D = (int(x) for x in size.split("x"))
    data = Planted(n, D, max(nqs))
    thr = binary_thresholds(data.chunk(0)[:100_000])
    formats = {"binm": ("binary", thr)}
    if not args.binary_only:
        formats["bin0"] = ("binary", None)
        formats["int8"] = ("int8", None)
        if not args.no_bf16:
            formats["bf16"] = ("bf16", None)
    shards = {name: CorpusShard(D, n, dtype=dt, thresholds=t) for name, (dt, t) in formats.items()}
    for i in data.chunks():
        x = data.chunk(i)
        for sh in shards.values():
            sh.add(x)
        del x
    # one workspace for every shard (the calls run one after another on one stream)
    lib = _lib.lib()
    need = max(lib.sgpt_search_workspace_bytes(nq, n, kk) for nq in nqs for k in ks for kk in (k, min(4096, 10 * k)))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    for sh in shards.values():
        sh._ws = ws
    floor_ms = (n * D / 8 + 4 * n) / 3.35e12 * 1e3
    print(f"## {n} x {D}: binary {n * D / 8 / 1e9:.2f} GB, int8 {n * D / 1e9:.2f} GB, bf16 {2 * n * D / 1e9:.2f} GB "
          f"({', '.join(shards)} built); HBM floor of the bits {floor_ms:.3f} ms; "
          f"peak device memory {torch.cuda.max_memory_allocated() / 1e9:.1f} GB")
    print("| queries | k | bf16 ms | int8 ms | bits ms | rescore ms | int8 refine ms | bits / floor | spread bits |")
    print("|---|---|---|---|---|---|---|---|---|")
    binm = shards["binm"]
    for nq in nqs:
        q = data.queries[:nq]
        for k in ks:
            kc = min(4096, 10 * k)
            legs = {"bits": lambda: binm.search(q, k, "cos_sim"),
                    "rescore": lambda: binm.search(q, k, "cos_sim", rescore=kc)}
            if "int8" in shards:
                legs["refine"] = lambda: binm.search(q, k, "cos_sim", refine=shards["int8"], rescore=kc)
                legs["int8"] = lambda: shards["int8"].search(q, k, "cos_sim")
            if "bf16" in shards:
                legs["bf16"] = lambda: shards["bf16"].search(q, k, "cos_sim")
            for f in legs.values():
                f()
            res = {name: [] for name in legs}
            for _ in range(args.rounds):  # alternate the legs round by round
                for name, f in legs.items():
                    res[name].append(timed(f))
            med = {name: sorted(v)[len(v) // 2] for name, v in res.items()}
            cell = lambda name: f"{med[name]:.3f}" if name in med else "—"  # noqa: E731
            spread = max(res["bits"]) - min(res["bits"])
            print(f"| {nq} | {k} | {cell('bf16')} | {cell('int8')} | {cell('bits')} | {cell('rescore')} | "
                  f"{cell('refine')} | {floor_ms / med['bits']:.2f} | {spread:.3f} |")
    q16 = data.queries[:16]
    print("ties at the cut, median thresholds, 16 queries: documents with s >= the k-th s, over k (median / max): " +
          ", ".join("k = %d: %.2f / %.2f" % ((k,) + tie_reach(binm, q16, k)) for k in ks))
    if not args.binary_only:
        q = data.queries
        ref_name = "bf16" if "bf16" in shards else "int8"
        _, truth = shards[ref_name].search(q, 100, "cos_sim")
        print(f"recall against the exact {ref_name} top-100, {q.shape[0]} queries (kc = 1000):")
        print("| thresholds | bits @10 | bits @100 | rescore @10 | rescore @100 | int8 refine @10 | int8 refine @100 |")
        print("|---|---|---|---|---|---|---|")
        for name in ("bin0", "binm"):
            sh = shards[name]
            got = (sh.search(q, 100, "cos_sim")[1], sh.search(q, 100, "cos_sim", rescore=1000)[1],
                   sh.search(q, 100, "cos_sim", refine=shards["int8"], rescore=1000)[1])
            r = [recall(x, truth, rr) for x in got for rr in (10, 100)]
            print(f"| {'zero' if name == 'bin0' else 'median'} | " + " | ".join(f"{x:.3f}" for x in r) + " |")



def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000x768,1000000x4096")
    ap.add_argument("--queries", default="1,16,128")
    ap.add_argument("--k", default="100,1001")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-bf16", action="store_true", help="no bf16 shard (10 M x 4096: 82 GB)")
    ap.add_argument("--binary-only", action="store_true", help="the median-threshold binary shard alone (capacity legs)")
    args = ap.parse_args()
    print(f"# card: {card()}")
    print(f"# {' '.join(sys.argv)}")
    nqs = [int(x) for x in args.queries.split(",")]
    ks = [int(x) for x in args.k.split(",")]
    for size in args.sizes.split(","):
        run_size(size, nqs, ks, args)  # the shards are freed when it returns
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()


if __name__ == "__main__":
    main()
