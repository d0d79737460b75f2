#!/usr/bin/env python
"""Native training step of the ORPIT recipe's softmax-mask Conv-TasNet: ms per forward / backward / step, one JSON line per case.

    python tools/bench_softmax_train.py [--steps 7] [--out result.json]

Model (egs/wsj0-mix/orpit_conv-tasnet/train.sh): N = 512, L = 16, stride 8, B = 128, H = 512, Sc = 128, P = 3, X = 8, R = 3, two
outputs (one and rest), gLN, softmax mask, the default math mode, random weights; batches of 4 x 4 s at 8 kHz (the recipe's) and
32 x 4 s, 3-speaker targets; ORPIT(NegSISDR()), clip 5 + Adam(lr=1e-3, weight_decay=1e-5) on the flat gradient bucket.  The
sigmoid-mask model of the same separator runs in the same call, its steps alternated with the softmax model's.  The recipe's
two-stage fine-tune step (finetune.sh: model, ORPIT, the 'rest' estimate back in as the mixture, model, ORPIT, one backward) is
timed at the recipe batch.  Each shape is warmed up once; the figures are medians over `steps` steps of CUDA-event intervals,
each ended by a synchronise; peak memory is torch.cuda.max_memory_allocated over the timed steps.
The softmax kernels of the step (k_softmax_mask forward, k_softmax_mask_bwd backward) are then timed by torch.profiler over a
few steps in a run of their own, with the bytes each must move computed from the shapes (M = 2 N channels, frames F, pitch P):
  k_softmax_mask     : reads logits (B, M, P) 3 times and w (B, N, P), writes mask and w_hat (B, M, P)
  k_softmax_mask_bwd : reads d_what, mask (B, M, P) twice and w (B, N, P) twice, writes d_wprod (B, N, P) and d_z (B, M, P)
so GB/s = bytes / time and the share of the 3.35 TB/s an H100 SXM's HBM3 is specified at.  Fails without a GPU."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))

from ctn_b200 import _native as N  # noqa: E402
from ctn_b200.criterion.pit import ORPIT  # noqa: E402
from ctn_b200.criterion.sdr import NegSISDR  # noqa: E402
from ctn_b200.models.conv_tasnet import ConvTasNet  # noqa: E402
from ctn_b200.optim import FlatClipAdam  # noqa: E402

SR, SECONDS, HBM_PEAK = 8000, 4, 3.35e12
T = SR * SECONDS
NB, L, STRIDE, S = 512, 16, 8, 2


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def model(mask):
    torch.manual_seed(0)
    m = ConvTasNet(NB, L, stride=STRIDE, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=512,
                   sep_bottleneck_channels=128, sep_skip_channels=128, sep_kernel_size=3, sep_num_blocks=3, sep_num_layers=8,
                   causal=False, n_sources=S, mask_nonlinear=mask)
    m.softmax_training = True
    return m.cuda().train()


def median(v):
    return sorted(v)[len(v) // 2]


def batch(B):
    g = torch.Generator(device="cuda").manual_seed(B)
    sources = torch.randn(B, 3, T, device="cuda", generator=g) * 0.1
    return sources.sum(dim=1, keepdim=True), sources


class Stepper:
    def __init__(self, m, B, finetune=False):
        self.m, self.B, self.finetune = m, B, finetune
        self.mixture, self.sources = batch(B)
        self.crit, self.opt = ORPIT(NegSISDR()), FlatClipAdam(m, lr=1e-3, weight_decay=1e-5, max_norm=5.0)
        self.fwd, self.bwd, self.tot = [], [], []

    def step(self, keep):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        self.opt.zero_grad()
        e[0].record()
        out = self.m(self.mixture)
        e[1].record()
        loss, idx = self.crit(out, self.sources)
        if self.finetune:  # stage 2: the targets other than the one taken, the 'rest' estimate as the mixture
            keep_ = torch.ones(self.B, 3, dtype=torch.bool, device="cuda")
            keep_[torch.arange(self.B, device="cuda"), idx] = False
            rest = self.sources[keep_].view(self.B, 2, T)
            loss = loss + self.crit(self.m(out[:, 1:]), rest)[0]
        e[2].record()
        loss.backward()
        e[3].record()
        self.opt.step()
        end = torch.cuda.Event(enable_timing=True)
        end.record()
        end.synchronize()
        if keep:
            self.fwd.append(e[0].elapsed_time(e[1]))
            self.bwd.append(e[2].elapsed_time(e[3]))
            self.tot.append(e[0].elapsed_time(end))

    def row(self, mask, steps):
        return dict(case="finetune-2-stage" if self.finetune else "step", mask=mask, B=self.B, T=T, steps=steps,
                    forward_ms=round(median(self.fwd), 3), backward_ms=round(median(self.bwd), 3), step_ms=round(median(self.tot), 3),
                    fwd_launches=self.m.last_launches, bwd_launches=self.m.last_bwd_launches)


def release():
    N.release_workspaces()
    torch.cuda.empty_cache()


def alternated(B, steps):
    soft, sig = Stepper(model("softmax"), B), Stepper(model("sigmoid"), B)
    for st in (soft, sig):
        st.step(False)
    torch.cuda.reset_peak_memory_stats()
    for _ in range(steps):
        soft.step(True)
        sig.step(True)
    peak = torch.cuda.max_memory_allocated()
    rows = [soft.row("softmax", steps), sig.row("sigmoid", steps)]
    for r in rows:
        r["peak_memory_bytes_both_models"] = peak
    rows[0]["softmax_over_sigmoid_step"] = round(rows[0]["step_ms"] / rows[1]["step_ms"], 4)
    return rows


def finetune(steps):
    ft = Stepper(model("softmax"), 4, finetune=True)
    ft.step(False)
    torch.cuda.reset_peak_memory_stats()
    for _ in range(steps):
        ft.step(True)
    r = ft.row("softmax", steps)
    r["peak_memory_bytes"] = torch.cuda.max_memory_allocated()
    return r


def kernels(bwd_ms, iters=5):
    st = Stepper(model("softmax"), 4)
    st.step(False)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            st.step(False)
        torch.cuda.synchronize()
    frames, _, _ = N.frames_of(T, L, STRIDE)
    P = N.ctn_pitch(frames)
    M, B = S * NB, 4
    nbytes = {"k_softmax_mask": 4 * B * P * (3 * M + NB + 2 * M), "k_softmax_mask_bwd": 4 * B * P * (4 * M + 2 * NB + NB + M)}
    rows = []
    for ev in prof.key_averages():
        for k in nbytes:
            if k in ev.key and (k + "_bwd" not in ev.key or k.endswith("_bwd")):
                t = ev.device_time_total / 1e3 / ev.count  # ms per call
                rows.append(dict(case="kernel", kernel=k, B=B, frames=frames, calls=ev.count, ms_per_call=round(t, 4), bytes=nbytes[k],
                                 GBps=round(nbytes[k] / t / 1e6, 1), share_of_3350GBps=round(nbytes[k] / (t * 1e-3) / HBM_PEAK, 3)))
                if k.endswith("_bwd"):
                    rows[-1]["share_of_backward"] = round(t / bwd_ms, 4)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_softmax_train.py needs a CUDA device")
    if args.steps < 3:
        raise SystemExit("--steps must be at least 3")
    name, power = card()
    rows = alternated(4, args.steps)
    release()
    rows += alternated(32, args.steps)
    release()
    rows.append(finetune(args.steps))
    release()
    rows += kernels(rows[0]["backward_ms"])
    for r in rows:
        r.update(card=name, power_limit=power)
        print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
