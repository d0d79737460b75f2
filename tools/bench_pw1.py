#!/usr/bin/env python
"""The TCN blocks' pw1 launch (ctn_pw(..., PRO_RES or PRO_NONE, EPI_H, f16x3)) on its own at the cfg2 and cfg5 shapes, and for the
record pw2 (PRO_DW, EPI_RAW) at the same shapes: one JSON line.

    python tools/bench_pw1.py [--reps 30] [--warmup 5] [--configs cfg2,cfg5] [--out result.json]

Shapes (bench.py's workloads, paper hyper-parameters N = 512, B_c = Sc = 128, H = 512):
  cfg2: 32 mixtures x 4 s @ 8 kHz -> B 32, frames 3999
  cfg5: 16 mixtures x 8 s @ 16 kHz -> B 16, frames 15999
Cases per shape: pw1_res (PRO_RES / EPI_H, blocks 1..23: M = H = 512, K = B_c = 128, the residual r with Mt = B_c + Sc rows),
pw1_none (PRO_NONE / EPI_H, block 0) and pw2 (PRO_DW / EPI_RAW, M = B_c + Sc = 256, K = H = 512, dilation 4).  Inputs are seeded,
with the operand scale at the top of its legal range, as the pipelines choose it.  Each call goes through the verification hook
(include/ctn_b200_probe.h), which also rebuilds the weight image, so the launch's own time comes from torch.profiler's
device-side kernel records: per call, the kernels that are not the weight-image builder.  Reported per case:
  kernel_ms        median (min, max) over `reps` calls after `warmup`, from the profiler's kernel records
  kernels          the kernel names the profiler saw (which path ran)
  floor            bytes (operand and r read once, h (and x_new) written once) and algorithmic flops (2 M K frames B; the 3-piece
                   split issues 3x that), and the time each takes at the H100 SXM data sheet's 3.35 TB/s and 989 TFLOP/s
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

SHAPES = {"cfg2": dict(B=32, T=32000), "cfg5": dict(B=16, T=128000)}
NB, BC, SC, H = 512, 128, 128, 512
HBM_BPS, F16_FLOPS = 3.35e12, 989e12
EPS = 1e-8


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def case(cfg, kind):
    s = SHAPES[cfg]
    B, T = s["B"], s["T"]
    frames = N.frames_of(T, 16, 8)[0]
    pitch = N.ctn_pitch(frames)
    M, K = (H, BC) if kind.startswith("pw1") else (BC + SC, H)
    g = torch.Generator().manual_seed(sum(map(ord, cfg + kind)))
    dev = torch.device("cuda")
    t = {}

    def padded(*shape, scale=1.0, shift=0.0):
        x = torch.zeros(*shape[:-1], pitch)
        x[..., :frames] = torch.randn(*shape[:-1], frames, generator=g) * scale + shift
        return x

    t["A"] = padded(B, K, frames, scale=0.8, shift=0.1)
    t["W"] = torch.randn(M, K, generator=g) / math.sqrt(K)
    t["D"] = torch.zeros(B, M, pitch)
    a = ProbeArgs()
    a.B, a.M, a.K, a.frames, a.pitch = B, M, K, frames, pitch
    if kind == "pw2":
        t["g1"], t["b1"] = torch.randn(K, generator=g) * 0.3 + 1.0, torch.randn(K, generator=g) * 0.1
        t["wd"], t["bd"] = torch.randn(K, 3, generator=g) * 0.5, torch.randn(K, generator=g) * 0.1
        t["slope"] = torch.tensor([-0.2])
        x = t["A"][..., :frames].double()
        t["stats_in"] = torch.stack([x.sum((1, 2)), (x * x).sum((1, 2))], 1)
        t["stats_out"] = torch.zeros(B, 2, dtype=torch.float64)
        # operand bound: |u| <= |PReLU(dwconv(gLN1(h)) + bd)|, taken from a CPU estimate with a margin
        mu = t["stats_in"][:, 0] / (K * frames)
        rstd = 1.0 / torch.sqrt(t["stats_in"][:, 1] / (K * frames) - mu * mu + EPS)
        hn = ((x - mu[:, None, None]) * rstd[:, None, None]).float() * t["g1"][None, :, None] + t["b1"][None, :, None]
        umax = float(hn.abs().amax()) * float(t["wd"].abs().sum(1).max()) * 1.25 + float(t["bd"].abs().max())
    else:
        t["bias"] = torch.randn(M, generator=g) * 0.2
        t["slope"] = torch.tensor([0.25])
        t["stats_out"] = torch.zeros(B, 2, dtype=torch.float64)
        umax = float(t["A"].abs().max())
        if kind == "pw1_res":
            Mt = BC + SC
            t["r"] = padded(B, Mt, frames, scale=2.0)
            t["v1"], t["v2"] = torch.randn(K, generator=g) * 0.2, torch.randn(K, generator=g) * 0.5
            y = torch.randn(B, H, frames, generator=g).double() * 1.5 + 0.2
            t["res_stats"] = torch.stack([y.sum((1, 2)), (y * y).sum((1, 2))], 1)
            t["xnew"] = torch.zeros(B, K, pitch)
            mu = t["res_stats"][:, 0] / (H * frames)
            rstd = 1.0 / torch.sqrt(t["res_stats"][:, 1] / (H * frames) - mu * mu + EPS)
            xn = (t["A"][..., :frames].double() + rstd[:, None, None] * t["r"][:, :K, :frames].double()
                  + t["v1"].double()[None, :, None] - (mu * rstd)[:, None, None] * t["v2"].double()[None, :, None])
            umax = float(xn.abs().max())
    t["scale"] = torch.tensor([2.0 ** (14 - math.floor(math.log2(umax)))])
    t = {k: v.to(dev).contiguous() for k, v in t.items()}
    a.A, a.W, a.D, a.act_scale = t["A"].data_ptr(), t["W"].data_ptr(), t["D"].data_ptr(), t["scale"].data_ptr()
    if kind == "pw2":
        a.pro_slope, a.dw_norm_g, a.dw_norm_b = t["slope"].data_ptr(), t["g1"].data_ptr(), t["b1"].data_ptr()
        a.dw_w, a.dw_b, a.dw_stats_in, a.dw_stats_out = t["wd"].data_ptr(), t["bd"].data_ptr(), t["stats_in"].data_ptr(), t["stats_out"].data_ptr()
        a.dw_dilation, a.dw_pad_left, a.dw_eps = 4, 4, EPS
        pro, epi = PRO["dw"], EPI["raw"]
        by = 4.0 * B * frames * (K + M)
    else:
        a.bias, a.slope, a.stats_out = t["bias"].data_ptr(), t["slope"].data_ptr(), t["stats_out"].data_ptr()
        pro, epi = (PRO["res"], EPI["h"]) if kind == "pw1_res" else (PRO["none"], EPI["h"])
        by = 4.0 * B * frames * (K + M)
        if kind == "pw1_res":
            a.res_r, a.res_Mt, a.res_v1, a.res_v2 = t["r"].data_ptr(), BC + SC, t["v1"].data_ptr(), t["v2"].data_ptr()
            a.res_stats, a.res_n, a.res_eps, a.res_x_out = t["res_stats"].data_ptr(), float(H * frames), EPS, t["xnew"].data_ptr()
            by += 4.0 * B * frames * 2 * K  # r[:Bc] read, x_new written
    nbytes = probe_wimg_bytes(M, K, N.MATH_F16X3)
    t["wimg"] = torch.empty(nbytes // 4 + 64, device=dev)
    stream = N.stream_ptr(dev)

    def call():
        st = probe_pw(C.byref(a), pro, epi, N.MATH_F16X3, 0, t["wimg"].data_ptr(), nbytes, stream)
        if st != N.CTN_OK:
            raise RuntimeError(f"{cfg} {kind}: ctn_probe_pw status {st}")

    fl = 2.0 * M * K * frames * B
    return dict(B=B, frames=frames, pitch=pitch, M=M, K=K), call, t, by, fl


def stats(x):
    x = sorted(x)
    return x[len(x) // 2], x[0], x[-1]


def run(cfg, kind, reps, warmup):
    shape, call, t, by, fl = case(cfg, kind)
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    kern = [e.time_range.elapsed_us() / 1e3 for e in prof.events()
            if e.device_type == torch.autograd.DeviceType.CUDA and "build_wimg" not in e.name and "emcpy" not in e.name
            and "emset" not in e.name]
    names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "build_wimg" not in e.name})
    if len(kern) != reps:
        raise RuntimeError(f"{cfg} {kind}: expected {reps} launch records, got {len(kern)}: {names}")
    k = stats(kern)
    return {"config": cfg, "case": kind, **shape, "kernel_ms": k[0], "kernel_ms_min_max": k[1:], "kernels": names,
            "floor": {"bytes": by, "flops_algorithmic": fl, "flops_issued_3piece": 3 * fl, "hbm_ms": by / HBM_BPS * 1e3,
                      "tensor_ms_3piece": 3 * fl / F16_FLOPS * 1e3},
            "share_of_hbm_floor": by / HBM_BPS * 1e3 / k[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--configs", default="cfg2,cfg5")
    ap.add_argument("--cases", default="pw1_res,pw1_none,pw2")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.reps < 20:
        ap.error("--reps must be at least 20")
    if not torch.cuda.is_available():
        raise SystemExit("bench_pw1.py measures the GPU launch and needs a CUDA device")
    name, power, clock = card()
    res = {"device": name, "power_limit": power, "max_sm_clock": clock,
           "cases": [run(c, k, a.reps, a.warmup) for c in a.configs.split(",") for k in a.cases.split(",")]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
