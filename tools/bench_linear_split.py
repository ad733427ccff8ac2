#!/usr/bin/env python
"""Where the time of the SGPT-125M linear layers goes: for each of the four shapes of a block at M = 32768 tokens, the
product GEMM with its real epilogue, the same kernel with no global stores (sgpt_linear's profiling epilogue 100: the
mainloop and the epilogue arithmetic, no output written) and torch.nn.functional.linear (cuBLAS) on the same operands.
The variants alternate inside each round, every timed window is at least --window seconds of back-to-back launches
between two CUDA events, and the median and min-max over --rounds rounds are printed as one JSON line per shape.

Usage: python tools/bench_linear_split.py [--rounds 5] [--window 0.3]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sgpt_b200 import _lib  # noqa: E402

M = 32768
# (layer, N, K, epilogue): fused q/k/v (bias), attention out-projection (reduce-add into the residual stream),
# MLP c_fc (gelu_new + bias), MLP c_proj (reduce-add)
SHAPES = [("qkv", 2304, 768, "bf16"), ("out_proj", 768, 768, "resid"), ("c_fc", 3072, 768, "gelu"),
          ("c_proj", 768, 3072, "resid")]
EPI_NULL = 100  # gemm.cu: gemm_linear_kernel without its global stores


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the card name from torch is still worth reporting
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi": repr(e)[:200]}


def window_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.3, help="seconds per timed window")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_linear_split needs a GPU"
    L, lib = _lib, _lib.lib()
    dev = "cuda"
    st = L.current_stream()
    g = torch.Generator(device=dev).manual_seed(0)
    print(json.dumps({"card": card(), "M": M, "rounds": a.rounds, "window_s": a.window}), flush=True)
    for layer, N, K, epi in SHAPES:
        x = torch.randn(M, K, generator=g, device=dev).to(torch.bfloat16)
        w = (torch.randn(N, K, generator=g, device=dev) * 0.02).to(torch.bfloat16)
        bias = torch.randn(N, generator=g, device=dev) * 0.1
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        code = {"bf16": L.EPI_BF16, "gelu": L.EPI_GELU_BF16, "resid": L.EPI_RESID_BF16}[epi]
        rd = out.data_ptr() if epi == "resid" else None

        def product():
            L.check(lib.sgpt_linear(x.data_ptr(), K, w.data_ptr(), K, bias.data_ptr(), out.data_ptr(), N, rd, M, N, K,
                                    code, st))

        def mainloop():
            L.check(lib.sgpt_linear(x.data_ptr(), K, w.data_ptr(), K, None, out.data_ptr(), N, None, M, N, K, EPI_NULL,
                                    st))

        bias16 = bias.to(torch.bfloat16)

        def cublas():
            torch.nn.functional.linear(x, w, bias16)

        variants = {"product": product, "mainloop": mainloop, "torch_linear": cublas}
        iters = {}
        for name, fn in variants.items():  # warm up, then size each window to >= a.window seconds
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            t = window_ms(fn, 10) / 10
            iters[name] = max(10, int(a.window * 1e3 / t) + 1)
        times = {name: [] for name in variants}
        for _ in range(a.rounds):
            for name, fn in variants.items():
                times[name].append(1e3 * window_ms(fn, iters[name]) / iters[name])  # us per launch
        flop = 2.0 * M * N * K
        res = {"layer": layer, "M": M, "N": N, "K": K, "epilogue": epi}
        for name, ts in times.items():
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            res[name] = {"us_median": round(med, 2), "us_min": round(ts[0], 2), "us_max": round(ts[-1], 2),
                         "tflops_median": round(flop / med / 1e6, 1), "iters": iters[name]}
        res["product_over_mainloop"] = round(res["product"]["us_median"] / res["mainloop"]["us_median"], 3)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
