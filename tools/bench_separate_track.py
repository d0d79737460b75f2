#!/usr/bin/env python
"""ConvTasNet.separate_track on one MUSDB18-length stereo track with the recipe's separator: one JSON line.

    python tools/bench_separate_track.py [--seconds 240] [--reps 5] [--warmup 1] [--out result.json]

Model: the MUSDB18 Conv-TasNet recipe's size, N = 256, L = 20, B = 256, H = 512, Sc = 128, P = 3, X = 10, R = 4, 4 stereo sources,
gLN, sigmoid mask, f16x3, random weights.  Input: one seeded stereo track of `seconds` at 44.1 kHz, 8 s segments.  Each time
is the median of `reps` repetitions after `warmup`, every repetition bracketed by CUDA events and ended by a synchronise:
  tester_ms        separate_track in the tester's layout (hop=None), the default chunk_batch;  audio_s_per_s = seconds / time
  crossfaded_ms    separate_track with hop = 4 s
  loop_ms          the recipe tester's loop restated on the native model: torch mean / std over each segment and channel,
                   one batch-1 forward per segment, std * estimate + mean, concatenate and crop
  steps_ms         statistics + every standardising gather + overlap-add through their own entry points, on buffers of the call's
                   shapes (tester layout);  steps_share = steps_ms / tester_ms
  launches, workspace_bytes, peak_bytes (torch's peak allocation over one call, workspace included)
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
from ctn_b200.models.conv_tasnet import ConvTasNet, TRACK_CHUNK_BATCH  # noqa: E402

SR, SEGMENT, HOP = 44100, 8 * 44100, 4 * 44100


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def model():
    torch.manual_seed(0)
    m = ConvTasNet(256, 20, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=512,
                   sep_bottleneck_channels=256, sep_skip_channels=128, sep_kernel_size=3, sep_num_blocks=4, sep_num_layers=10,
                   causal=False, n_sources=4, in_channels=2)
    m = m.cuda().eval()
    m.math = "f16x3"
    return m


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


def tester_loop(m, x, eps=1e-12):
    """x (1, 1, C, T): the recipe tester's steps around one batch-1 forward per segment"""
    T = x.size(-1)
    pad = (SEGMENT - T % SEGMENT) % SEGMENT
    seg = torch.nn.functional.pad(x, (0, pad)).reshape(1, x.size(2), -1, SEGMENT).permute(2, 0, 1, 3).contiguous()
    mean, std = seg.mean(dim=-1, keepdim=True), seg.std(dim=-1, keepdim=True)
    z = (seg - mean) / (std + eps)
    est = torch.stack([m(z[i:i + 1]).squeeze(0) for i in range(z.size(0))])
    y = std * est + mean                                           # (K, S, C, Lc)
    K, S, Cn, Lc = y.shape
    return y.permute(1, 2, 0, 3).reshape(S, Cn, K * Lc)[..., :T]


def steps(x, B, Cn, T, S, st, scratch, nbytes, xc, est, out, stream, eps=1e-12):
    K = N.ctn_track_plan(T, SEGMENT, 0, None, 0)
    N.check(N.ctn_track_stats(x.data_ptr(), B, Cn, T, SEGMENT, 0, st.data_ptr(), scratch.data_ptr(), nbytes, stream))
    nb = xc.size(0)
    for g0 in range(0, B * K, nb):
        n = min(nb, B * K - g0)
        N.check(N.ctn_track_gather(x.data_ptr(), st.data_ptr(), B, Cn, T, SEGMENT, 0, eps, g0, n, xc.data_ptr(), stream))
    N.check(N.ctn_track_overlap_add(est.data_ptr(), st.data_ptr(), B, S, Cn, T, SEGMENT, 0, out.data_ptr(), stream))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=240.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_separate_track needs a CUDA device")
    name, power, clock = card()
    m = model()
    T = int(a.seconds * SR)
    B, Cn, S = 1, 2, m.n_sources
    g = torch.Generator().manual_seed(1)
    x = (0.1 * torch.randn(B, 1, Cn, T, generator=g)).cuda()
    dev = torch.device("cuda", torch.cuda.current_device())
    stream = N.stream_ptr(dev)
    res = {"bench": "separate_track", "card": name, "power_limit": power, "max_sm_clock": clock, "seconds": a.seconds, "sr": SR,
           "segment_s": SEGMENT / SR, "chunk_batch": TRACK_CHUNK_BATCH, "math": "f16x3", "reps": a.reps}
    with torch.no_grad():
        res["tester_ms"] = median_ms(lambda: m.separate_track(x, SEGMENT), a.reps, a.warmup)
        res["launches"] = m.last_launches
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out_t = m.separate_track(x, SEGMENT)
        torch.cuda.synchronize()
        res["peak_bytes"] = torch.cuda.max_memory_allocated()
        res["peak_over_start_bytes"] = torch.cuda.max_memory_allocated() - base
        res["crossfaded_ms"] = median_ms(lambda: m.separate_track(x, SEGMENT, hop=HOP), a.reps, a.warmup)
        res["crossfaded_launches"] = m.last_launches
        c = m.native_config()
        need, need_x = C.c_size_t(0), C.c_size_t(0)
        N.check(N.ctn_separate_track_workspace_bytes(C.byref(c), B, T, SEGMENT, 0, TRACK_CHUNK_BATCH, C.byref(need)))
        N.check(N.ctn_separate_track_workspace_bytes(C.byref(c), B, T, SEGMENT, HOP, TRACK_CHUNK_BATCH, C.byref(need_x)))
        res["workspace_bytes"], res["crossfaded_workspace_bytes"] = need.value, need_x.value
        # the recipe tester's loop on the native model
        res["loop_ms"] = median_ms(lambda: tester_loop(m, x), a.reps, a.warmup)
        loop = tester_loop(m, x)
        res["loop_vs_call_maxabs"] = float((loop - out_t[0]).abs().max())
        res["out_maxabs"] = float(out_t.abs().max())
        # statistics + gathers + overlap-add alone
        K = N.ctn_track_plan(T, SEGMENT, 0, None, 0)
        nbytes = N.ctn_track_stats_scratch_bytes(B, Cn, T, SEGMENT, 0)
        st = torch.empty(B, K, Cn, 2, dtype=torch.float64, device="cuda")
        scratch = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device="cuda")
        xc = torch.empty(min(TRACK_CHUNK_BATCH, B * K), Cn, SEGMENT, device="cuda")
        est = torch.randn(B * K, S, Cn, SEGMENT, device="cuda")
        out = torch.empty(B, S, Cn, T, device="cuda")
        xf = x.reshape(B, Cn, T)
        res["steps_ms"] = median_ms(lambda: steps(xf, B, Cn, T, S, st, scratch, nbytes, xc, est, out, stream), a.reps, a.warmup)
        # the stats, gather and overlap-add bytes (read + write), for a rate
        moved = 4 * (B * Cn * T) + 4 * (B * K * Cn * SEGMENT) * 2 + 4 * (B * K * S * Cn * SEGMENT) + 4 * (B * S * Cn * T) + 4 * B * Cn * T
        res["steps_bytes"] = moved
    res["audio_s_per_s"] = a.seconds / (res["tester_ms"][0] / 1e3)
    res["crossfaded_audio_s_per_s"] = a.seconds / (res["crossfaded_ms"][0] / 1e3)
    res["loop_audio_s_per_s"] = a.seconds / (res["loop_ms"][0] / 1e3)
    res["steps_share"] = res["steps_ms"][0] / res["tester_ms"][0]
    res["steps_GB_per_s"] = res["steps_bytes"] / (res["steps_ms"][0] / 1e3) / 1e9
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
