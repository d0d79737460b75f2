#!/usr/bin/env python
"""Online (chunk-by-chunk) inference of the paper-size causal Conv-TasNet: push latency, one JSON line per case.

    python tools/bench_online.py [--pushes 1000] [--warmup 50] [--out result.json]

Model: N = 512, L = 16, B = 128, H = 512, Sc = 128, P = 3, X = 8, R = 3, 2 sources, cLN, sigmoid mask, the default math mode,
random weights.  Cases: n in {8, 64, 256} samples per push, B in {1, 16, 128} streams, eager pushes and replays of one push
captured in a CUDA graph.  Every push is bracketed by CUDA events and followed by a synchronise, as a serving loop waiting
for each chunk's output would be; latencies are the medians and 99th percentiles of `pushes` pushes after `warmup`.
  rtf          = median latency / chunk duration (n / 8000 s): < 1 keeps up
  streams_rt   = B when the p99 latency fits in one chunk's duration, else 0 (the measured batch stays real-time)
  capacity     = B * chunk duration / median latency: streams one GPU could carry at this B and n, back to back
The offline causal forward on the same audio (B x 4 s) is timed for comparison, and the card's name and power limit are read
in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))

from ctn_b200.models.conv_tasnet import ConvTasNet  # noqa: E402

SR = 8000


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return name, power


def model():
    torch.manual_seed(0)
    m = ConvTasNet(512, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=512,
                   sep_bottleneck_channels=128, sep_skip_channels=128, sep_kernel_size=3, sep_num_blocks=3, sep_num_layers=8,
                   causal=True, n_sources=2)
    return m.cuda().eval()


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def run_case(m, B, n, graph, pushes, warmup):
    sep = m.online(batch_size=B, max_chunk=n)
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + n)
    xs = torch.randn(64, B, 1, n, device="cuda", generator=g) * 0.1
    static_x = xs[0].clone()
    for i in range(max(warmup, 4)):
        sep.push(xs[i % 64])
    launches = sep.last_launches
    step = lambda i: sep.push(xs[i % 64])  # noqa: E731
    if graph:
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, capture_error_mode="relaxed"):
            sep.push(static_x)
        for _ in range(warmup):
            gr.replay()

        def step(i):
            static_x.copy_(xs[i % 64])
            gr.replay()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(pushes)]
    for i in range(pushes):
        ev[i][0].record()
        step(i)
        ev[i][1].record()
        ev[i][1].synchronize()
    lat = [a.elapsed_time(b) for a, b in ev]
    med, p99 = pct(lat, 0.5), pct(lat, 0.99)
    chunk_ms = 1000.0 * n / SR
    return dict(case="online", mode="graph" if graph else "eager", B=B, n=n, pushes=pushes, median_ms=round(med, 4),
                p99_ms=round(p99, 4), rtf=round(med / chunk_ms, 4), streams_rt=B if p99 <= chunk_ms else 0,
                capacity=int(B * chunk_ms / med), launches_per_push=launches)


def offline_case(m, B, iters=20):
    x = torch.randn(B, 1, 4 * SR, device="cuda") * 0.1
    with torch.no_grad():
        for _ in range(3):
            m(x)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            m(x)
        b.record()
        torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    return dict(case="offline", B=B, seconds_of_audio=4 * B, ms=round(ms, 3), audio_s_per_s=round(4 * B / (ms / 1000.0), 1),
                launches=m.last_launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_online.py needs a CUDA device")
    name, power = card()
    m = model()
    rows = []
    for B in (1, 16, 128):
        for n in (8, 64, 256):
            for graph in (False, True):
                r = run_case(m, B, n, graph, args.pushes, args.warmup)
                r.update(card=name, power_limit=power)
                print(json.dumps(r), flush=True)
                rows.append(r)
        r = offline_case(m, B)
        r.update(card=name, power_limit=power)
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
