#!/usr/bin/env python
"""Device time of one sgpt_pool call on the two-kernel path: B sequences of S tokens, d > 1024, ln_f and weightedmean,
with and without the L2 normalisation.  Each timed window is back-to-back launches between two CUDA events, at least
--window seconds long; the median and min-max over --rounds windows are printed as one JSON line per variant, with the
card they ran on.  Point SGPT_B200_LIB at another build of the library to time it on the same inputs.

Usage: python tools/bench_pool.py [--B 256] [--S 128] [--d 4096] [--rounds 5] [--window 0.3]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sgpt_b200 import _lib  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:
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
    ap.add_argument("--B", type=int, default=256)
    ap.add_argument("--S", type=int, default=128)
    ap.add_argument("--d", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.3)
    a = ap.parse_args()
    lib = _lib.lib()
    B, S, d = a.B, a.S, a.d
    T = B * S
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn(T, d, generator=g, device="cuda") + 0.3).to(torch.bfloat16)
    pos = torch.arange(S, dtype=torch.int32, device="cuda").repeat(B)
    cu = torch.arange(0, T + 1, S, dtype=torch.int32, device="cuda")
    gamma = 1.0 + 0.1 * torch.randn(d, generator=g, device="cuda")
    beta = 0.05 * torch.randn(d, generator=g, device="cuda")
    out = torch.empty(B, d, device="cuda")
    ws = torch.empty(2 * T + B, device="cuda")
    stream = _lib.current_stream()
    res = []
    for normalize in (0, 1):
        def call():
            _lib.check(lib.sgpt_pool(x.data_ptr(), 1, pos.data_ptr(), cu.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                     1e-5, None, 0, out.data_ptr(), ws.data_ptr(), B, T, d, _lib.POOL_WEIGHTEDMEAN, 0,
                                     normalize, 0, 1.0, stream))

        call()
        one = window_ms(call, 10) / 10
        iters = max(10, int(a.window * 1e3 / max(one, 1e-3)))
        times = sorted(window_ms(call, iters) / iters * 1e3 for _ in range(a.rounds))
        res.append({"B": B, "S": S, "d": d, "normalize": normalize, "us_median": round(times[len(times) // 2], 2),
                    "us_min": round(times[0], 2), "us_max": round(times[-1], 2)})
    for r in res:
        print(json.dumps({**r, "lib": os.path.basename(_lib.LIB_PATH), "card": card()}))


if __name__ == "__main__":
    main()
