#!/usr/bin/env python
"""The fused mask + decoder launch (ctn_pw(..., PRO_PRELU, EPI_MASKDEC, f16x3)) on its own, at the cfg2 and cfg5 shapes: one JSON line.

    python tools/bench_maskdec.py [--reps 30] [--warmup 5] [--configs cfg2,cfg5] [--out result.json]

Shapes (bench.py's workloads, paper hyper-parameters N = 512, Sc = 128, kernel 16 / stride 8):
  cfg2: 32 mixtures x 4 s @ 8 kHz, 2 sources -> B 32, frames 3999, M = S N = 1024, K = Sc = 128
  cfg5: 16 mixtures x 8 s @ 16 kHz, 4 sources -> B 16, frames 15999, M = 2048, K = 128
Inputs are seeded: the skip sum (B, Sc, pitch), mask weights and bias, the encoder output |w| (B, N, pitch), the decoder basis
(N, 16), with the operand scale at the top of its legal range, as the pipelines choose it.  Each call goes through the
verification hook (include/ctn_b200_probe.h), which also rebuilds the weight image, so the launch's own time comes from
torch.profiler's device-side kernel records: per call, the kernels that are not the weight-image builder.  Reported per shape:
  kernel_ms        median (min, max) over `reps` calls after `warmup`, from the profiler's kernel records
  call_ms          median of the whole hook call (image build + launch) between CUDA events, each ended by a synchronise
  floor            bytes (skip sum + w read once, estimates written once) and algorithmic flops (2 Sc S N frames B; the
                   3-piece split issues 3x that), and the time each takes at the H100 SXM data sheet's 3.35 TB/s and 989 TFLOP/s
The card's name, power limit and maximum SM clock are read in the same run; no device setting is changed."""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from ctn_b200 import _native as N  # noqa: E402
from test_pw_contraction_gpu import EPI, PRO, ProbeArgs, probe_pw, probe_wimg_bytes  # noqa: E402

SHAPES = {"cfg2": dict(B=32, T=32000, S=2), "cfg5": dict(B=16, T=128000, S=4)}
NB, SC, CROP = 512, 128, 4
HBM_BPS, F16_FLOPS = 3.35e12, 989e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def case(cfg):
    s = SHAPES[cfg]
    B, T, S = s["B"], s["T"], s["S"]
    frames = N.frames_of(T, 16, 8)[0]
    pitch = N.ctn_pitch(frames)
    M, K, T_out = S * NB, SC, 8 * frames + 8 - 2 * CROP
    g = torch.Generator().manual_seed(sum(map(ord, cfg)))
    dev = torch.device("cuda")
    t = {}
    t["A"] = torch.zeros(B, K, pitch)
    t["A"][..., :frames] = torch.randn(B, K, frames, generator=g) * 0.8 + 0.1
    t["W"] = torch.randn(M, K, generator=g) / math.sqrt(K)
    t["bias"] = torch.randn(M, generator=g) * 0.2
    t["wenc"] = torch.zeros(B, NB, pitch)
    t["wenc"][..., :frames] = torch.randn(B, NB, frames, generator=g).abs()
    t["dec"] = torch.randn(NB, 16, generator=g) * 0.3
    t["slope"] = torch.tensor([0.25])
    pmax = float(torch.where(t["A"] >= 0, t["A"], 0.25 * t["A"]).abs().max())
    t["scale"] = torch.tensor([2.0 ** (14 - math.floor(math.log2(pmax)))])
    t = {k: v.to(dev).contiguous() for k, v in t.items()}
    t["D"] = torch.zeros(B, S, T_out, device=dev)
    nbytes = probe_wimg_bytes(M, K, N.MATH_F16X3)
    t["wimg"] = torch.empty(nbytes // 4 + 64, device=dev)
    a = ProbeArgs()
    a.B, a.M, a.K, a.frames, a.pitch = B, M, K, frames, pitch
    a.A, a.W, a.D, a.bias, a.wenc, a.Nb = t["A"].data_ptr(), t["W"].data_ptr(), t["D"].data_ptr(), t["bias"].data_ptr(), t["wenc"].data_ptr(), NB
    a.dec_w, a.dec_crop_left, a.dec_T_out = t["dec"].data_ptr(), CROP, T_out
    a.pro_slope, a.act_scale = t["slope"].data_ptr(), t["scale"].data_ptr()
    stream = N.stream_ptr(dev)

    def call():
        st = probe_pw(C.byref(a), PRO["prelu"], EPI["maskdec"], N.MATH_F16X3, 0, t["wimg"].data_ptr(), nbytes, stream)
        if st != N.CTN_OK:
            raise RuntimeError(f"{cfg}: ctn_probe_pw status {st}")

    by = 4.0 * B * frames * (SC + NB) + 4.0 * B * S * T_out
    fl = 2.0 * SC * S * NB * frames * B
    return dict(B=B, S=S, frames=frames, pitch=pitch, M=M, K=K, T_out=T_out), call, t, by, fl


def stats(x):
    x = sorted(x)
    return x[len(x) // 2], x[0], x[-1]


def run(cfg, reps, warmup):
    shape, call, t, by, fl = case(cfg)
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    calls = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        e1.synchronize()
        calls.append(e0.elapsed_time(e1))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    kern = [e.time_range.elapsed_us() / 1e3 for e in prof.events()
            if e.device_type == torch.autograd.DeviceType.CUDA and "build_wimg" not in e.name and "emcpy" not in e.name
            and "emset" not in e.name]
    names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    if len(kern) != reps:
        raise RuntimeError(f"{cfg}: expected {reps} launch records, got {len(kern)}: {names}")
    k = stats(kern)
    return {"config": cfg, **shape, "kernel_ms": k[0], "kernel_ms_min_max": k[1:], "call_ms": stats(calls)[0], "kernels": names,
            "floor": {"bytes": by, "flops_algorithmic": fl, "flops_issued_3piece": 3 * fl, "hbm_ms": by / HBM_BPS * 1e3,
                      "tensor_ms_3piece": 3 * fl / F16_FLOPS * 1e3}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--configs", default="cfg2,cfg5")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.reps < 20:
        ap.error("--reps must be at least 20")
    if not torch.cuda.is_available():
        raise SystemExit("bench_maskdec.py measures the GPU launch and needs a CUDA device")
    name, power, clock = card()
    res = {"device": name, "power_limit": power, "max_sm_clock": clock,
           "cases": [run(c, a.reps, a.warmup) for c in a.configs.split(",")]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
