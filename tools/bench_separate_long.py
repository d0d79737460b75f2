#!/usr/bin/env python
"""ConvTasNet.separate_long on long recordings with the paper-size non-causal model: one JSON line.

    python tools/bench_separate_long.py [--minutes 10] [--reps 5] [--warmup 1] [--out result.json]

Model: N = 512, L = 16, B = 128, H = 512, Sc = 128, P = 3, X = 8, R = 3, 2 sources, gLN, sigmoid mask, the default math mode,
random weights.  Cases: 1 and 4 recordings of `minutes` at 8 kHz, chunk = 4 s, hop = 2 s, 16 chunks per forward.  Per case,
each the median of `reps` repetitions after `warmup`, every repetition bracketed by CUDA events and ended by a synchronise:
  call_ms         the whole separate_long call;  audio_s_per_s = recording seconds / call time
  post_ms         the work outside the forward -- the gather of every chunk batch, the alignment and the overlap-add, run
                  through their own entry points on a buffer of chunk estimates of the same shape;  post_share = post_ms / call_ms
  plain_ms        the plain forward on the same number of 4 s chunks as ordinary batches of 16 (what the call spends in the model);
                  plain_audio_s_per_s counts every chunk's 4 s, so with hop = chunk / 2 about half of it is the call's ceiling
  launches, workspace_bytes (what the call asks for), plain_workspace_bytes (the plain forward on the whole recording: not run)
The card's name and power limit are read in the same run; no device setting is changed."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))

from ctn_b200 import _native as N  # noqa: E402
from ctn_b200.models.conv_tasnet import ConvTasNet  # noqa: E402

SR, CHUNK, HOP, CHUNK_BATCH = 8000, 4 * 8000, 2 * 8000, 16


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def model():
    torch.manual_seed(0)
    m = ConvTasNet(512, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=512,
                   sep_bottleneck_channels=128, sep_skip_channels=128, sep_kernel_size=3, sep_num_blocks=3, sep_num_layers=8,
                   causal=False, n_sources=2)
    return m.cuda().eval()


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


def run_case(m, B, T, reps, warmup):
    S = m.n_sources
    dev = torch.device("cuda", torch.cuda.current_device())
    st = N.stream_ptr(dev)
    x = torch.randn(B, 1, T, device="cuda") * 0.1
    K = N.ctn_chunk_plan(T, CHUNK, HOP, None, 0)
    chunks = B * K
    with torch.no_grad():
        call = median_ms(lambda: m.separate_long(x, CHUNK, HOP, chunk_batch=CHUNK_BATCH), reps, warmup)
        launches = m.last_launches

        # the post-processing alone, on estimates of the same shape
        est = torch.randn(chunks, S, CHUNK, device="cuda") * 0.1
        xc = torch.empty(CHUNK_BATCH, 1, CHUNK, device="cuda")
        out = torch.empty(B, S, T, device="cuda")
        perms = torch.empty(B, K, S, dtype=torch.int32, device="cuda")
        nbytes = N.ctn_chunk_align_scratch_bytes(B, S, T, CHUNK, HOP)
        scratch = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device="cuda")

        def post():
            for g0 in range(0, chunks, CHUNK_BATCH):
                N.check(N.ctn_chunk_gather(x.data_ptr(), B, T, CHUNK, HOP, g0, min(CHUNK_BATCH, chunks - g0), xc.data_ptr(), st))
            N.check(N.ctn_chunk_align(est.data_ptr(), B, S, T, CHUNK, HOP, perms.data_ptr(), scratch.data_ptr(), nbytes, st))
            N.check(N.ctn_chunk_overlap_add(est.data_ptr(), perms.data_ptr(), B, S, T, CHUNK, HOP, out.data_ptr(), st))
        post_t = median_ms(post, reps, warmup)
        del est, out

        # the plain forward on as many 4 s chunks, as ordinary batches
        xb = torch.randn(CHUNK_BATCH, 1, CHUNK, device="cuda") * 0.1

        def plain():
            for g0 in range(0, chunks, CHUNK_BATCH):
                m(xb[:min(CHUNK_BATCH, chunks - g0)])
        plain_t = median_ms(plain, reps, warmup)
    cfg = m.native_config()
    need, whole = C.c_size_t(0), C.c_size_t(0)
    N.check(N.ctn_separate_long_workspace_bytes(C.byref(cfg), B, T, CHUNK, HOP, CHUNK_BATCH, C.byref(need)))
    N.check(N.ctn_workspace_bytes(C.byref(cfg), B, T, C.byref(whole)))
    audio_s = B * T / SR
    return dict(B=B, minutes=round(T / SR / 60.0, 3), chunks=chunks, call_ms=round(call[0], 2), call_min_ms=round(call[1], 2),
                call_max_ms=round(call[2], 2), audio_s_per_s=round(audio_s / (call[0] / 1e3), 1), post_ms=round(post_t[0], 3),
                post_share=round(post_t[0] / call[0], 5), plain_ms=round(plain_t[0], 2),
                plain_audio_s_per_s=round(chunks * CHUNK / SR / (plain_t[0] / 1e3), 1), launches=launches,
                workspace_bytes=need.value, plain_workspace_bytes=whole.value)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_separate_long.py needs a CUDA device")
    name, power, sm_clock = card()
    m = model()
    T = int(round(args.minutes * 60 * SR))
    result = dict(bench="separate_long", card=name, power_limit=power, max_sm_clock=sm_clock, chunk_s=CHUNK / SR, hop_s=HOP / SR,
                  chunk_batch=CHUNK_BATCH, reps=args.reps, warmup=args.warmup, cases=[run_case(m, B, T, args.reps, args.warmup) for B in (1, 4)])
    print(json.dumps(result), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
