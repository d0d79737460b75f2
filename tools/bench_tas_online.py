#!/usr/bin/env python
"""Online (chunk-by-chunk) LSTM-TasNet on one GPU: the wsj0-mix recipe shape made causal (plain encoder, N = 500, L = 40, stride 20,
H = 500, 2 blocks x 2 LSTM layers, sigmoid mask, 2 sources, 8 kHz), in the default numeric mode.

    python tools/bench_tas_online.py [--iters 50] [--warmup 10] [--out bench_tas_online.json]

For pushes of 20, 160, 320 and 800 samples and 1, 16 and 64 streams: the milliseconds of one push (median of CUDA-event timings of
single pushes after warm-up pushes, the state advancing as in a real stream), the real-time factor (push time / the audio one push
carries), the launches per push, and, from a separate torch.profiler pass over the same pushes, the share of the push's kernel time
spent in the recurrence.  The card's name and power limit are read in the same call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))
from ctn_b200 import _native as N  # noqa: E402
from ctn_b200.models.tasnet import TasNet  # noqa: E402

CFG = dict(n_basis=500, kernel_size=40, stride=20, H=500, blocks=2, layers=2, n_sources=2, sample_rate=8000)
PUSHES = (20, 160, 320, 800)
STREAMS = (1, 16, 64)


def build(dev):
    c = CFG
    m = TasNet(c["n_basis"], kernel_size=c["kernel_size"], stride=c["stride"], enc_basis="trainable", dec_basis="trainable",
               sep_num_blocks=c["blocks"], sep_num_layers=c["layers"], sep_hidden_channels=c["H"], mask_nonlinear="sigmoid", causal=True,
               rnn_type="lstm", n_sources=c["n_sources"])
    return m.to(dev).eval()


def push_ms(sep, x, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        sep.push(x)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def recurrence_share(sep, x, iters):
    """kernel milliseconds of `iters` pushes: the recurrence launches and everything"""
    from torch.autograd import DeviceType
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            sep.push(x)
        torch.cuda.synchronize()
    ks = [e for e in prof.events() if e.device_type == DeviceType.CUDA and e.time_range.elapsed_us() > 0]
    rec = sum(e.time_range.elapsed_us() for e in ks if "k_tas_lstm<" in e.name) / 1e3
    tot = sum(e.time_range.elapsed_us() for e in ks) / 1e3
    return rec / iters, tot / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tas_online needs a CUDA device")
    dev = torch.device("cuda", 0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        card = q.stdout.strip().splitlines()[0]
    except Exception:
        card = torch.cuda.get_device_name(0)
    torch.manual_seed(0)
    m = build(dev)
    rows = []
    with torch.no_grad():
        for B in STREAMS:
            for n in PUSHES:
                x = torch.randn(B, 1, n, device=dev)
                sep = m.online(batch_size=B, max_chunk=n)
                for _ in range(args.warmup):
                    sep.push(x)
                torch.cuda.synchronize()
                ms = push_ms(sep, x, args.iters)
                launches = sep.last_launches
                rec_ms, kern_ms = recurrence_share(m.online(batch_size=B, max_chunk=n), x, max(args.warmup, 10))
                audio_ms = 1e3 * n / CFG["sample_rate"]
                row = dict(streams=B, push_samples=n, push_frames=n // CFG["stride"], audio_ms=audio_ms, ms=round(ms, 4),
                           rtf=round(ms / audio_ms, 4), launches=launches, kernel_ms=round(kern_ms, 4), recurrence_ms=round(rec_ms, 4),
                           recurrence_share=round(rec_ms / max(kern_ms, 1e-9), 3), state_bytes=sep.state_bytes)
                rows.append(row)
                print(json.dumps(row))
    res = {"card": card, "cfg": CFG, "math": m.math or "default", "rows": rows}
    print(json.dumps({"card": card}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
