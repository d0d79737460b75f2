#!/usr/bin/env python
"""The SDR training criterion: device-event timings and launch counts, one JSON line per case.

    python tools/bench_sdr_loss.py [--iters 20] [--warmup 5] [--steps 7]

Cases:
  * loss      fused PIT1d(NegSDR) forward + backward w.r.t. the estimate (ctn_sdr_pit_fwd / ctn_sdr_pit_bwd) against the reference's
              loop over the S! permutations through the differentiable NegSDR rows (ctn_sdr_fwd / ctn_sdr_bwd), S = 2 and 3,
              B = 32, 4 s at 8 kHz; the bytes each fused call must move: forward 2 B S T 4, backward 2 B S T 4 read + B S T 4 written;
  * wham      the gLN training step (the paper's separator: N = 512, L = 16, B = 128, H = 512, Sc = 128, P = 3, X = 8, R = 3) at the
              same batch under PIT1d(NegSDR) and under PIT1d(NegSISDR): forward + loss + backward;
  * musdb     the MUSDB18 recipe's step (tools/bench_multichannel_train.py's stereo model and batch: 4 x 8 s at 44.1 kHz,
              standardised by the mixture's mean and std) under NegSDR and under MeanSquaredError.
Loss timings are CUDA events around `iters` calls after `warmup`; step timings are medians over `steps` steps (one warm-up step
first), each ended by a synchronise.  Launches per call are the CUDA kernels torch.profiler records for one call.  The card's name
and power limit are read in the same run.  Fails without a GPU."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_pit_variants import card, launches, timed  # noqa: E402
import bench_multichannel_train as MC  # noqa: E402
from ctn_b200.criterion import pit as PIT  # noqa: E402
from ctn_b200.criterion.distance import MeanSquaredError  # noqa: E402
from ctn_b200.criterion.sdr import NegSDR, NegSISDR  # noqa: E402
from ctn_b200.models.conv_tasnet import ConvTasNet  # noqa: E402

B, T = 32, 32000
EPS = 1e-12


def loss_case(S, iters, warmup):
    g = torch.Generator(device="cuda").manual_seed(S)
    tgt = torch.randn(B, S, T, device="cuda", generator=g)
    est = (tgt[:, torch.randperm(S)] + 0.5 * torch.randn(B, S, T, device="cuda", generator=g)).contiguous()
    crit = PIT.PIT1d(NegSDR(), S)
    x = est.requires_grad_(True)

    def fused():
        x.grad = None
        loss, _ = crit(x, tgt)
        loss.backward()

    def generic():
        x.grad = None
        loss, _ = PIT._pit_generic(NegSDR(), x, tgt, patterns=crit.patterns)
        loss.backward()

    tf, tg = timed(fused, iters, warmup), timed(generic, iters, warmup)
    nbytes = 3 * B * S * T * 4 + 2 * B * S * T * 4
    return dict(case="loss", S=S, B=B, T=T, fused_ms=round(tf, 4), generic_ms=round(tg, 4), speedup=round(tg / tf, 2),
                fused_launches=launches(fused), generic_launches=launches(generic), fused_bytes=nbytes,
                fused_GBps=round(nbytes / (tf * 1e-3) / 1e9, 1))


def median(v):
    return sorted(v)[len(v) // 2]


def step_times(run, steps):
    out = []
    for i in range(steps + 1):  # step 0 warms the shape up
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        if i:
            out.append(a.elapsed_time(b))
    return round(median(out), 3)


def wham_case(steps):
    torch.manual_seed(0)
    m = ConvTasNet(512, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=512,
                   sep_bottleneck_channels=128, sep_skip_channels=128, sep_kernel_size=3, sep_num_blocks=3, sep_num_layers=8,
                   causal=False, n_sources=2).cuda().train()
    g = torch.Generator(device="cuda").manual_seed(7)
    sources = torch.randn(B, 2, T, device="cuda", generator=g)
    mixture = sources.sum(dim=1, keepdim=True)
    rec = dict(case="wham_step", B=B, T=T, S=2, steps=steps)
    for name, crit in (("NegSDR", PIT.PIT1d(NegSDR(), 2)), ("NegSISDR", PIT.PIT1d(NegSISDR(), 2))):
        def run():
            m.zero_grad(set_to_none=True)
            loss, _ = crit(m(mixture), sources)
            loss.backward()
        rec[name + "_step_ms"] = step_times(run, steps)
    return rec


def musdb_case(steps):
    m = MC.model(MC.CIN)
    g = torch.Generator(device="cuda").manual_seed(MC.CIN)
    sources = torch.randn((MC.BATCH, MC.S, MC.CIN, MC.T), device="cuda", generator=g) * 0.1
    mixture = sources.sum(dim=1, keepdim=True)
    mean, std = mixture.mean(dim=-1, keepdim=True), mixture.std(dim=-1, keepdim=True)
    mix_s, src_s = (mixture - mean) / (std + EPS), (sources - mean) / (std + EPS)
    rec = dict(case="musdb_step", B=MC.BATCH, T=MC.T, S=MC.S, C=MC.CIN, steps=steps)
    for name, crit in (("NegSDR", NegSDR()), ("MSE", MeanSquaredError(dim=-1, reduction="mean"))):
        def run():
            m.zero_grad(set_to_none=True)
            crit(m(mix_s), src_s).backward()
        rec[name + "_step_ms"] = step_times(run, steps)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_sdr_loss.py measures on a CUDA device; none is present")
    name, power = card()
    cases = [lambda: loss_case(2, args.iters, args.warmup), lambda: loss_case(3, args.iters, args.warmup),
             lambda: wham_case(args.steps), lambda: musdb_case(args.steps)]
    for case in cases:
        try:
            rec = case()
        except torch.cuda.OutOfMemoryError as e:  # reported, not hidden: the other cases still run
            rec = dict(case="out of memory", error=str(e).splitlines()[0])
        torch.cuda.empty_cache()
        rec.update(gpu=name, power_limit=power)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
