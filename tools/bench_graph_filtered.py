"""Filtered graph search and GraphIndex.add: time, recall and fallback share, next to IVF and the exact search.

    python tools/bench_graph_filtered.py [--out result.json]

Data: tools/bench_graph.py's "lowdim" rows (G z + 0.1 eps, z ~ N(0, I_16), G a fixed random 768 x 16 matrix), 1M x 768
bf16 plus 100k more rows for the add leg, generated on the device from seed 0.  The graph is GraphIndex.build at degree
32 from 64-entry lists, the IVF index nlist 4000.

Filtered search cells: allowed shares 100 / 50 / 10 / 1 / 0.1 % of the shard (uniformly random), one filter shared by
all queries or one per query, 16 / 128 / 1024 queries, itopk 64 / 128, k = 10, default max_iterations and num_seeds.
Timed alternately with CUDA events after warm-up (median of 5 rounds, with min and max), as in tools/bench_graph.py:
  graph        GraphIndex.search(allow=) end to end: packing the filter, the filtered kernel, the host synchronisation
               and the exact-search fallback of the queries whose walk visited fewer than k allowed documents
  ivf32        IVFIndex.search(allow=) at nprobe 32
  exact        CorpusShard.search(allow=)
  kernel_filtered / kernel_plain   sgpt_graph_search_filtered on the packed filter and sgpt_graph_search (no mask) with
               the same arguments: the cost of keeping the allowed top-k next to the beam
Recall@10 is against the exact filtered search; "fallback" is the share of queries the exact search answered.

Add leg: GraphIndex.add of 1k / 10k / 100k rows into the 1M-row index (restored to 1M rows between sizes), timed with a
device synchronise; then, with the 100k rows added, recall@10 of 1024 queries drawn near the added rows for the grown
index and for GraphIndex.build over all 1.1M rows.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import torch

TOOLS = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(TOOLS))
sys.path.insert(0, TOOLS)

from bench_graph import alternate, card, recall, timed  # noqa: E402
from sgpt_b200 import CorpusShard, GraphIndex, IVFIndex, _lib  # noqa: E402
from sgpt_b200.graph import default_max_iterations  # noqa: E402

SHARES = (1.0, 0.5, 0.1, 0.01, 0.001)
NQS = (16, 128, 1024)
ITOPKS = (64, 128)
K, N, ADD = 10, 1_000_000, 100_000


def kernel(index, qb, q_scale, c_scale, itopk, mask, pitch, filtered, out_s, out_i):
    """One launch of sgpt_graph_search_filtered (or sgpt_graph_search without a mask) on prepared query rows."""
    nq = qb.shape[0]
    it = default_max_iterations(itopk, 1, index.degree, itopk)
    args = (index.shard._dtype_id(), qb.data_ptr(), index.shard.vectors.data_ptr(), _lib.ptr(q_scale), c_scale, nq,
            index.n, index.dim, index.id_base, index.graph.data_ptr(), index.degree, None, itopk, 0, itopk, 1, it, K)
    lib = _lib.lib()
    if filtered:
        rc = lib.sgpt_graph_search_filtered(*args, _lib.ptr(mask), pitch, out_s.data_ptr(), out_i.data_ptr(), None,
                                            _lib.current_stream())
    else:
        rc = lib.sgpt_graph_search(*args, None, out_s.data_ptr(), out_i.data_ptr(), None, _lib.current_stream())
    _lib.check(rc, "graph search")


def filtered_cells(shard, index, ivf, q):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1)
    for nq in NQS:
        qq = q[:nq].contiguous()
        qb, q_scale, c_scale = shard._queries(qq, "cos_sim")
        out_s = torch.empty((nq, K), device="cuda")
        out_i = torch.empty((nq, K), dtype=torch.int64, device="cuda")
        for per_query in (False, True):
            for share in SHARES:
                allow = torch.rand((nq, N) if per_query else (N,), generator=g, device="cuda") < share
                mask, pitch = shard._mask(allow, nq)
                _, exact = shard.search(qq, K, "cos_sim", allow=allow)
                for itopk in ITOPKS:
                    t = alternate({
                        "graph": lambda: index.search(qq, K, itopk=itopk, allow=allow),
                        "ivf32": lambda: ivf.search(qq, K, 32, allow=allow),
                        "exact": lambda: shard.search(qq, K, "cos_sim", allow=allow),
                        "kernel_filtered": lambda: kernel(index, qb, q_scale, c_scale, itopk, mask, pitch, True, out_s,
                                                          out_i),
                        "kernel_plain": lambda: kernel(index, qb, q_scale, c_scale, itopk, None, 0, False, out_s,
                                                       out_i)})
                    kernel(index, qb, q_scale, c_scale, itopk, mask, pitch, True, out_s, out_i)
                    fell = float((out_i[:, -1] < 0).float().mean())
                    walk = recall(out_i, exact, K)
                    _, gi = index.search(qq, K, itopk=itopk, allow=allow)
                    _, ii = ivf.search(qq, K, 32, allow=allow)
                    row = {"queries": nq, "filter": "per query" if per_query else "shared", "share": share,
                           "itopk": itopk, "fallback": round(fell, 4), "recall_at_10_graph": recall(gi, exact, K),
                           "recall_at_10_walk_only": walk, "recall_at_10_ivf32": recall(ii, exact, K)}
                    for fn, (med, lo, hi) in t.items():
                        row[f"{fn}_ms"] = round(med, 4)
                        row[f"{fn}_ms_min_max"] = [round(lo, 4), round(hi, 4)]
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                del allow, mask
    return rows


def add_leg(shard, index, extra, q_near):
    graph0, pruned0 = index.graph.clone(), index.pruned.clone()
    rows = []
    for m in (1_000, 10_000, 100_000):
        index.graph, index.pruned, index.n, shard.n = graph0.clone(), pruned0.clone(), N, N
        _, t = timed(lambda: index.add(extra[:m]))
        rows.append({"add_rows": m, "into": N, "seconds": t})
        print(json.dumps(rows[-1]), flush=True)
    _, exact = shard.search(q_near, K, "cos_sim")
    _, grown = index.search(q_near, K, itopk=128)
    rebuilt, t_build = timed(lambda: GraphIndex.build(shard))
    _, fresh = rebuilt.search(q_near, K, itopk=128)
    res = {"queries_near_added_rows": q_near.shape[0], "itopk": 128, "recall_at_10_build_1M_add_100k":
           recall(grown, exact, K), "recall_at_10_build_1.1M": recall(fresh, exact, K), "build_1.1M_s": t_build}
    print(json.dumps(res), flush=True)
    return rows, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_graph_filtered measures the GPU; there is no CPU path"
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"card": card()}
    print(json.dumps(res["card"]), flush=True)
    G = torch.randn(768, 16, generator=g, device="cuda")

    def draw(m):
        return torch.randn(m, 16, generator=g, device="cuda") @ G.T + 0.1 * torch.randn(m, 768, generator=g,
                                                                                         device="cuda")
    shard = CorpusShard(768, N + ADD, device="cuda:0")
    for s0 in range(0, N, 500_000):
        shard.add(draw(500_000))
    q = draw(max(NQS))
    extra = draw(ADD)
    q_near = extra[torch.randint(ADD, (1024,), generator=g, device="cuda")]
    q_near += 0.1 * torch.randn(q_near.shape, generator=g, device="cuda")
    index, t_graph = timed(lambda: GraphIndex.build(shard))
    ivf, t_ivf = timed(lambda: IVFIndex.build(shard, 4000, seed=0, train_size=160_000))
    res["build"] = {"n": N, "graph_build_s": t_graph, "ivf_build_s": t_ivf}
    print(json.dumps(res["build"]), flush=True)
    res["filtered"] = filtered_cells(shard, index, ivf, q)
    del ivf
    torch.cuda.empty_cache()
    res["add"], res["add_recall"] = add_leg(shard, index, extra, q_near)
    res["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
