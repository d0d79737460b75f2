#!/usr/bin/env python
"""Fused vs generic ORPIT / SinkPIT (forward + backward w.r.t. the estimate), one JSON line per case.

    python tools/bench_pit_variants.py [--iters 20] [--warmup 5]

Both paths run the same NegSISDR criterion on CUDA tensors: the fused path through ORPIT / sinkpit (ctn_orpit_* /
ctn_sinkpit_*), the generic path through the reference's loops (_orpit_generic / _sinkpit_generic, whose criterion calls are
the native per-row SI-SDR).  Times come from CUDA events around `iters` calls after `warmup` calls; launches per call are
the CUDA kernels torch.profiler records for one call (a separate, untimed run).  The card's name and power limit are read in
the same run.  Cases: T = 32000, B = 8 (4 s of 8 kHz audio, the wsj0-mix recipes' training length), ORPIT with packed
n in {2, 3} (the "2+3" recipe), SinkPIT with S in {3, 10, 16} and K in {10, 200} (the tutorial recipe's K = 200)."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))

from ctn_b200.criterion import pit as PIT  # noqa: E402
from ctn_b200.criterion.sdr import NegSISDR  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def launches(fn):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memset" not in e.name
               and "Memcpy" not in e.name)


def orpit_case(B, n, T):
    g = torch.Generator().manual_seed(n)
    lens = [2 + (b % (n - 1)) for b in range(B)] if n > 2 else [2] * B
    tgt = torch.zeros(B, n, T)
    for b, nb in enumerate(lens):
        tgt[b, :nb] = torch.randn(nb, T, generator=g)
    est = torch.randn(B, 2, T, generator=g).cuda()
    packed = torch.nn.utils.rnn.pack_padded_sequence(tgt.cuda(), torch.tensor(lens), batch_first=True, enforce_sorted=False)
    padded, lengths = torch.nn.utils.rnn.pad_packed_sequence(packed, batch_first=True)
    crit = NegSISDR()

    def fused():
        x = est.clone().requires_grad_(True)
        loss, _ = PIT.ORPIT(crit)(x, packed)
        loss.backward()

    def generic():
        x = est.clone().requires_grad_(True)
        loss, _ = PIT._orpit_generic(crit, x, padded, lengths)
        loss.mean().backward()
    return dict(criterion="ORPIT", B=B, n=n, lens=sorted(set(lens)), T=T), fused, generic


def sink_case(B, S, K, T):
    g = torch.Generator().manual_seed(S)
    tgt = torch.randn(B, S, T, generator=g).cuda()
    est = (tgt[:, torch.randperm(S, generator=g)] + 0.5 * torch.randn(B, S, T, generator=g).cuda()).contiguous()
    crit = NegSISDR()

    def fused():
        x = est.clone().requires_grad_(True)
        loss, _ = PIT.sinkpit(crit, x, tgt, coldness=1.0, iteration=K)
        loss.backward()

    def generic():
        x = est.clone().requires_grad_(True)
        loss, _ = PIT._sinkpit_generic(crit, x, tgt, None, 1.0, K)
        loss.mean().backward()
    return dict(criterion="SinkPIT", B=B, S=S, K=K, T=T), fused, generic


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_pit_variants.py measures on a CUDA device; none is present")
    name, power = card()
    B, T = 8, 32000
    cases = [orpit_case(B, n, T) for n in (2, 3)] + [sink_case(B, S, K, T) for S in (3, 10, 16) for K in (10, 200)]
    for meta, fused, generic in cases:
        tf, tg = timed(fused, args.iters, args.warmup), timed(generic, args.iters, args.warmup)
        rec = dict(meta, fused_ms=round(tf, 4), generic_ms=round(tg, 4), speedup=round(tg / tf, 2),
                   fused_launches=launches(fused), generic_launches=launches(generic), gpu=name, power_limit=power)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
