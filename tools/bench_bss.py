#!/usr/bin/env python
"""BSS Eval (ctn_bss_eval_sources, mir_eval's bss_eval_sources in fp64 on the GPU) at the tester's sizes: one JSON line.

    python tools/bench_bss.py [--reps 10] [--warmup 2] [--oracle-items 2] [--out result.json]

Cases: S = 2 and 3 sources, T = 40 000 samples (5 s at 8 kHz), K = 2 estimate sets (the estimates and the mixture repeated S
times, as the separation tester scores them), B = 1 (one test utterance) and B = 64.  References are low-pass filtered noise,
estimates FIR(reference) + cross-talk + noise (tests/bss_ref.py).  Per case, the median (min, max) of `reps` repetitions after
`warmup`, each bracketed by CUDA events and ended by a synchronise:
  call_ms         the C call alone (no host synchronisation inside)
  wrapper_ms      bss_eval_sources_batch from device tensors, including its read of the status word
  per_item_ms     call_ms / B;  launches: kernels one call enqueues
  oracle_ms_per_item  the fp64 numpy / scipy oracle (tests/bss_ref.py, mir_eval's route; not mir_eval itself) on the CPU, per item
                  and estimate set pair, over the first `oracle-items` items;  worst_err_db: largest |GPU - oracle| over their SDR,
                  SIR and SAR (the SAR of the mixture set, rounding noise on both sides, is left out)
The card's name and power limit are read in the same run; no device setting is changed."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bss_ref as R  # noqa: E402
from ctn_b200 import _native as N  # noqa: E402
from ctn_b200.utils.bss import bss_eval_sources_batch  # noqa: E402

T, K = 40000, 2


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def inputs(B, S):
    rng = np.random.default_rng(100 * S + B)
    refs, ests = zip(*(R.make_item(rng, S, T, coloured=True) for _ in range(B)))
    ref = np.stack(refs)
    est = np.stack([np.stack(ests), np.repeat(ref.sum(1, keepdims=True), S, axis=1)], 1)
    return torch.from_numpy(ref), torch.from_numpy(est)


def run_case(B, S, reps, warmup, oracle_items):
    ref_h, est_h = inputs(B, S)
    ref, est = ref_h.cuda(), est_h.cuda()
    dev = ref.device
    nbytes = C.c_size_t(0)
    N.check(N.ctn_bss_workspace_bytes(B, K, S, T, C.byref(nbytes)), "ctn_bss_workspace_bytes")
    ws = torch.empty(nbytes.value + 256, dtype=torch.uint8, device=dev)
    base, avail = N.aligned(ws)
    sdr, sir, sar = (torch.empty((B, K, S), dtype=torch.float64, device=dev) for _ in range(3))
    perm = torch.empty((B, K, S), dtype=torch.int32, device=dev)
    status = torch.empty(B, dtype=torch.int32, device=dev)
    st = N.stream_ptr(dev)

    def call():
        N.check(N.ctn_bss_eval_sources(ref.data_ptr(), est.data_ptr(), B, K, S, T, 1, sdr.data_ptr(), sir.data_ptr(), sar.data_ptr(),
                                       perm.data_ptr(), status.data_ptr(), base, avail, st), "ctn_bss_eval_sources")

    call_ms = median_ms(call, reps, warmup)
    launches = N.ctn_last_launch_count()
    assert int(status.abs().sum()) == 0
    wrapper_ms = median_ms(lambda: bss_eval_sources_batch(ref, est), reps, warmup)
    g = [t.cpu().numpy() for t in bss_eval_sources_batch(ref, est)]
    worst, t0, n = 0.0, time.perf_counter(), min(B, oracle_items)
    for b in range(n):
        for k in range(K):
            o = R.bss_eval_sources(ref_h[b].numpy(), est_h[b, k].numpy())
            for q in range(3 if k == 0 else 2):
                fin = np.isfinite(o[q])
                if fin.any():
                    worst = max(worst, float(np.max(np.abs(g[q][b, k][fin] - o[q][fin]))))
    oracle_ms = (time.perf_counter() - t0) * 1e3 / max(n, 1)
    del ws
    torch.cuda.empty_cache()
    return {"S": S, "B": B, "T": T, "K": K, "call_ms": call_ms[0], "call_ms_min_max": call_ms[1:], "wrapper_ms": wrapper_ms[0],
            "per_item_ms": call_ms[0] / B, "launches": launches, "workspace_bytes": nbytes.value,
            "oracle_ms_per_item": oracle_ms, "oracle_items": n, "worst_err_db": worst}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-items", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bss.py measures the GPU path and needs a CUDA device")
    name, power, clock = card()
    cases = [run_case(B, S, a.reps, a.warmup, a.oracle_items) for S in (2, 3) for B in (1, 64)]
    res = {"device": name, "power_limit": power, "max_sm_clock": clock, "cases": cases}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
