#!/usr/bin/env python
"""Residual (reduce-add) GEMMs of every config with SGPT_GEMM_SPLITK forced to 0 / 2 / 3 / 4 and automatic, isolated
launches with the L2 flushed.  Usage: python tools/bench_splitk.py [--iters 20]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sgpt_b200 import _lib  # noqa: E402

# (label, M, N, K)
SHAPES = [("125m out_proj", 32768, 768, 768), ("125m c_proj", 32768, 768, 3072),
          ("1.3b out_proj", 16384, 2048, 2048), ("1.3b c_proj", 16384, 2048, 8192),
          ("5.8b out_proj", 9600, 4096, 4096), ("5.8b c_proj", 9600, 4096, 16384)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    L, lib = _lib, _lib.lib()
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    bf = torch.bfloat16
    st = L.current_stream()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timeit(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        tot = 0.0
        for _ in range(a.iters):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            tot += e0.elapsed_time(e1)
        return tot / a.iters

    for label, M, N, K in SHAPES:
        x = torch.randn(M, K, generator=g, device=dev).to(bf)
        w = (torch.randn(N, K, generator=g, device=dev) * 0.02).to(bf)
        bias = torch.randn(N, generator=g, device=dev) * 0.1
        r = torch.zeros(M, N, device=dev, dtype=bf)
        res = {"gemm": label, "M": M, "N": N, "K": K}
        for setting in ("0", "2", "3", "4", None):
            if setting is None:
                os.environ.pop("SGPT_GEMM_SPLITK", None)
            else:
                os.environ["SGPT_GEMM_SPLITK"] = setting
            t = timeit(lambda: L.check(lib.sgpt_linear(x.data_ptr(), K, w.data_ptr(), K, bias.data_ptr(), r.data_ptr(), N,
                                                       r.data_ptr(), M, N, K, L.EPI_RESID_BF16, st)))
            res["auto" if setting is None else "split" + setting] = {"us": round(1e3 * t, 1),
                                                                   "tflops": round(2.0 * M * N * K / t / 1e9, 1)}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
