#!/usr/bin/env python
"""Native training step of the paper-size causal (cLN) Conv-TasNet: ms per forward / backward / step, one JSON line per case.

    python tools/bench_causal_train.py [--steps 7] [--out result.json]

Model: N = 512, L = 16, B = 128, H = 512, Sc = 128, P = 3, X = 8, R = 3, 2 sources, sigmoid mask, the default math mode, random
weights; PIT(NegSISDR) loss, clip + Adam on the flat gradient bucket.  Batches of 4 s at 8 kHz: 8, and the largest batch whose
training workspace fits in 60 % of the card's free memory (stated in its line).  Every shape is warmed up once; the figures are
medians over `steps` steps of CUDA-event intervals, each ended by a synchronise.  The non-causal (gLN) model of the same size
runs in the same call for context.
The three cLN-backward kernels (through ctn_probe_cln_bwd, one call = the three launches) and the causal depthwise backward are
timed on their own at (8, 512, 3999), with the bytes each must move computed from the shapes:
  cLN backward   : reads dy and pre, writes dpre in the apply pass; reads dy and pre in the frame-sum pass: 5 tensors
  causal dw bwd  : reads d_upre and h_pre, writes d_hn: 3 tensors (the shifted re-reads hit the caches)
so GB/s = bytes / time and the share of the 3.35 TB/s an H100 SXM's HBM3 is specified at.  Fails without a GPU."""
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
from ctn_b200.criterion.pit import PIT1d  # noqa: E402
from ctn_b200.criterion.sdr import NegSISDR  # noqa: E402
from ctn_b200.models.conv_tasnet import ConvTasNet  # noqa: E402
from ctn_b200.optim import FlatClipAdam  # noqa: E402

SR, HBM_PEAK = 8000, 3.35e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def model(causal):
    torch.manual_seed(0)
    m = ConvTasNet(512, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=512,
                   sep_bottleneck_channels=128, sep_skip_channels=128, sep_kernel_size=3, sep_num_blocks=3, sep_num_layers=8,
                   causal=causal, n_sources=2)
    m.causal_training = True
    return m.cuda().train()


def workspace_bytes(m, B, T):
    need = C.c_size_t(0)
    fn = N.ctn_causal_train_workspace_bytes if m.causal else N.ctn_train_workspace_bytes
    N.check(fn(C.byref(m.native_config()), B, T, C.byref(need)), "workspace bytes")
    return need.value


def median(v):
    return sorted(v)[len(v) // 2]


def step_case(m, B, steps):
    T = 4 * SR
    g = torch.Generator(device="cuda").manual_seed(B)
    mixture = torch.randn(B, 1, T, device="cuda", generator=g) * 0.1
    sources = torch.randn(B, 2, T, device="cuda", generator=g) * 0.1
    crit, opt = PIT1d(NegSISDR(), 2), FlatClipAdam(m, lr=1e-4, max_norm=5.0)
    fwd, bwd, tot = [], [], []
    for i in range(steps + 1):  # step 0 warms the shape up
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        opt.zero_grad()
        e[0].record()
        out = m(mixture)
        e[1].record()
        loss, _ = crit(out, sources)
        e[2].record()
        loss.backward()
        e[3].record()
        opt.step()
        end = torch.cuda.Event(enable_timing=True)
        end.record()
        end.synchronize()
        if i:
            fwd.append(e[0].elapsed_time(e[1]))
            bwd.append(e[2].elapsed_time(e[3]))
            tot.append(e[0].elapsed_time(end))
    del opt
    return dict(case="step", causal=bool(m.causal), B=B, seconds_of_audio=4 * B, steps=steps, forward_ms=round(median(fwd), 3),
                backward_ms=round(median(bwd), 3), step_ms=round(median(tot), 3), fwd_launches=m.last_launches,
                bwd_launches=m.last_bwd_launches, workspace_bytes=workspace_bytes(m, B, T))


def kernel_case(iters=20):
    B, Cc, frames = 8, 512, 3999
    pitch = N.ctn_pitch(frames)
    fp, i32 = C.c_void_p, C.c_int
    lib = N.lib
    for name, args in (("ctn_probe_cln_stats", [fp, fp, i32, i32, i32, i32, C.c_float, fp, fp, fp]),
                       ("ctn_probe_cln_bwd", [fp] * 6 + [C.c_float] + [fp] * 5 + [i32] * 4 + [fp]),
                       ("ctn_probe_cdw_bwd", [fp] * 9 + [i32] * 6 + [fp])):
        getattr(lib, name).restype, getattr(lib, name).argtypes = C.c_int, args
    pre = torch.zeros(B, Cc, pitch, device="cuda")
    pre[:, :, :frames] = torch.randn(B, Cc, frames, device="cuda")
    dy = torch.zeros_like(pre)
    dy[:, :, :frames] = torch.randn(B, Cc, frames, device="cuda")
    out = torch.empty_like(pre)
    gamma, beta, wd = torch.ones(Cc, device="cuda"), torch.zeros(Cc, device="cuda"), torch.randn(Cc, 3, device="cuda")
    slope = torch.full((1,), 0.25, device="cuda")
    st = torch.empty(B, frames, 2, dtype=torch.float64, device="cuda")
    mi = torch.empty(B, frames, 2, device="cuda")
    scratch = torch.empty(18 * B * frames, dtype=torch.float64, device="cuda")
    acc = torch.zeros(5, Cc * 3, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    N.check(lib.ctn_probe_cln_stats(pre.data_ptr(), slope.data_ptr(), B, Cc, frames, pitch, 1e-8, st.data_ptr(), mi.data_ptr(), s), "stats")

    def cln_bwd():
        N.check(lib.ctn_probe_cln_bwd(dy.data_ptr(), pre.data_ptr(), out.data_ptr(), slope.data_ptr(), gamma.data_ptr(), st.data_ptr(), 1e-8,
                                      scratch.data_ptr(), acc[0].data_ptr(), acc[1].data_ptr(), acc[2].data_ptr(), acc[3].data_ptr(), B, Cc,
                                      frames, pitch, s), "cln_bwd")

    def cdw_bwd():
        N.check(lib.ctn_probe_cdw_bwd(dy.data_ptr(), pre.data_ptr(), out.data_ptr(), mi.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                      slope.data_ptr(), wd.data_ptr(), acc[4].data_ptr(), B, Cc, frames, pitch, 3, 8, s), "cdw_bwd")

    tensor = 4 * B * Cc * frames
    rows = []
    for name, fn, nbytes in (("cln_bwd (3 kernels)", cln_bwd, 5 * tensor), ("causal_dw_bwd", cdw_bwd, 3 * tensor)):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        t = median(ms)
        rows.append(dict(case="kernel", kernel=name, shape=[B, Cc, frames], median_ms=round(t, 4), bytes=nbytes,
                         GBps=round(nbytes / t / 1e6, 1), share_of_3350GBps=round(nbytes / (t * 1e-3) / HBM_PEAK, 3)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_causal_train.py needs a CUDA device")
    if args.steps < 5:
        raise SystemExit("--steps must be at least 5")
    name, power = card()
    rows = []
    mc = model(True)
    free = torch.cuda.mem_get_info()[0]
    per8 = workspace_bytes(mc, 8, 4 * SR)
    bmax = max(8, int(0.6 * free / (per8 / 8)) // 8 * 8)
    for B in sorted({8, bmax}):
        rows.append(step_case(mc, B, args.steps))
        if B == bmax:
            rows[-1]["note"] = "largest batch whose workspace fits in 60 % of the free memory ({} MiB free)".format(free >> 20)
    del mc
    N.release_workspaces()
    torch.cuda.empty_cache()
    rows.append(step_case(model(False), 8, args.steps))
    rows += kernel_case()
    for r in rows:
        r.update(card=name, power_limit=power)
        print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
