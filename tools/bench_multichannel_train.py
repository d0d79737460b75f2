#!/usr/bin/env python
"""Native training step of the MUSDB18 recipe's stereo Conv-TasNet: ms per forward / backward / step, one JSON line per case.

    python tools/bench_multichannel_train.py [--steps 7] [--out result.json]

Model (egs/musdb18/conv-tasnet): in_channels = 2, N = 256, L = 20, stride 10, B = 256, H = 512, Sc = 128, P = 3, X = 10, R = 4,
4 sources, gLN, sigmoid mask, the default math mode, random weights; batches of 4 x 8 s of stereo at 44.1 kHz (352 800 samples,
35 279 frames); MeanSquaredError(dim=-1, reduction='mean'), clip 5 + Adam on the flat gradient bucket.  The shape is warmed up
once; the figures are medians over `steps` steps of CUDA-event intervals, each ended by a synchronise; peak memory is
torch.cuda.max_memory_allocated over the timed steps.  The monaural model of the same separator at the same batch runs in the same
call for context.
The filter-bank kernels of the step are then timed alone at the recipe shape, with the bytes each must move computed from the shapes
(the filter banks and their windows stay in shared memory / L1 and are not counted):
  encoder          : reads x (B, 2, T), writes w (B, N, pitch)
  decoder          : reads w_hat (B*S, N, frames), writes y (B*S, 2, T)
  decoder adjoint  : the encoder over d_out: reads (B*S, 2, T), writes d_what (B*S, N, pitch)
  encoder dW       : reads d_w (B, N, frames) and x
  decoder dW       : reads w_hat (B*S, N, frames) and d_out (B*S, 2, T)
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
from ctn_b200.criterion.distance import MeanSquaredError  # noqa: E402
from ctn_b200.models.conv_tasnet import ConvTasNet  # noqa: E402
from ctn_b200.optim import FlatClipAdam  # noqa: E402

SR, SECONDS, BATCH, CIN, HBM_PEAK = 44100, 8, 4, 2, 3.35e12
T = SR * SECONDS
NB, L, STRIDE, S = 256, 20, 10, 4


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def model(in_channels):
    torch.manual_seed(0)
    m = ConvTasNet(NB, L, stride=STRIDE, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=512,
                   sep_bottleneck_channels=256, sep_skip_channels=128, sep_kernel_size=3, sep_num_blocks=4, sep_num_layers=10,
                   causal=False, n_sources=S, in_channels=in_channels)
    m.multichannel_training = True
    return m.cuda().train()


def median(v):
    return sorted(v)[len(v) // 2]


def step_case(m, steps):
    cin = m.in_channels
    g = torch.Generator(device="cuda").manual_seed(cin)
    shape = (BATCH, 1, cin, T) if cin > 1 else (BATCH, 1, T)
    sources = torch.randn((BATCH, S) + shape[2:], device="cuda", generator=g) * 0.1
    mixture = sources.sum(dim=1, keepdim=True)
    crit, opt = MeanSquaredError(dim=-1, reduction="mean"), FlatClipAdam(m, lr=3e-4, max_norm=5.0)
    fwd, bwd, tot = [], [], []
    for i in range(steps + 1):  # step 0 warms the shape up
        if i == 1:
            torch.cuda.reset_peak_memory_stats()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        opt.zero_grad()
        e[0].record()
        out = m(mixture)
        e[1].record()
        loss = crit(out, sources)
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
    return dict(case="step", in_channels=cin, B=BATCH, T=T, steps=steps, forward_ms=round(median(fwd), 3),
                backward_ms=round(median(bwd), 3), step_ms=round(median(tot), 3), fwd_launches=m.last_launches,
                bwd_launches=m.last_bwd_launches, peak_memory_bytes=torch.cuda.max_memory_allocated())


def kernel_case(iters=20):
    frames, pl, pr = N.frames_of(T, L, STRIDE)
    pitch = N.ctn_pitch(frames)
    BS = BATCH * S
    lib = N.lib
    lib.ctn_probe_encdec_wgrad_mc.restype = C.c_int
    lib.ctn_probe_encdec_wgrad_mc.argtypes = [C.c_void_p] * 3 + [C.c_int] * 9 + [C.c_void_p]
    dev = "cuda"
    x = torch.randn(BATCH, CIN, T, device=dev) * 0.3
    d_out = torch.randn(BS, CIN, T, device=dev)
    W = torch.randn(NB, CIN, L, device=dev) * 0.1
    w = torch.empty(BATCH, NB, pitch, device=dev)
    what = torch.zeros(BS, NB, pitch, device=dev)
    what[..., :frames] = torch.randn(BS, NB, frames, device=dev)
    dwhat = torch.empty(BS, NB, pitch, device=dev)
    y = torch.empty(BS, CIN, T, device=dev)
    dW = torch.zeros(NB, CIN, L, device=dev)
    stats = torch.zeros(BATCH, 2, dtype=torch.float64, device=dev)
    s = N.stream_ptr(torch.device(dev))
    f4 = 4

    def enc():
        N.check(N.ctn_encoder_mc_fwd(x.data_ptr(), W.data_ptr(), w.data_ptr(), BATCH, CIN, T, pl, pr, NB, L, STRIDE, 0, pitch,
                                     stats.data_ptr(), s), "encoder")

    def dec():
        N.check(N.ctn_decoder_mc_fwd(what.data_ptr(), W.data_ptr(), y.data_ptr(), BS, CIN, NB, frames, pitch, L, STRIDE, pl, T, s), "decoder")

    def adj():
        N.check(N.ctn_encoder_mc_fwd(d_out.data_ptr(), W.data_ptr(), dwhat.data_ptr(), BS, CIN, T, pl, pr, NB, L, STRIDE, 0, pitch, None, s),
                "adjoint")

    def wg_enc():
        N.check(lib.ctn_probe_encdec_wgrad_mc(what.data_ptr(), x.data_ptr(), dW.data_ptr(), BATCH, NB, CIN, frames, pitch, T, L, STRIDE,
                                              pl, s), "encoder dW")

    def wg_dec():
        N.check(lib.ctn_probe_encdec_wgrad_mc(what.data_ptr(), d_out.data_ptr(), dW.data_ptr(), BS, NB, CIN, frames, pitch, T, L, STRIDE,
                                              pl, s), "decoder dW")

    cases = (("encoder (k_encoder_v4_mc<20,10>)", enc, f4 * (BATCH * CIN * T + BATCH * NB * pitch)),
             ("decoder (k_decoder_mc_v<10,2>)", dec, f4 * (BS * NB * frames + BS * CIN * T)),
             ("decoder adjoint (k_encoder_v4_mc<20,10>)", adj, f4 * (BS * CIN * T + BS * NB * pitch)),
             ("encoder dW (k_encdec_wgrad, C = 2)", wg_enc, f4 * (BATCH * NB * frames + BATCH * CIN * T)),
             ("decoder dW (k_encdec_wgrad, C = 2)", wg_dec, f4 * (BS * NB * frames + BS * CIN * T)))
    rows = []
    for name, fn, nbytes in cases:
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
        rows.append(dict(case="kernel", kernel=name, frames=frames, median_ms=round(t, 4), bytes=nbytes, GBps=round(nbytes / t / 1e6, 1),
                         share_of_3350GBps=round(nbytes / (t * 1e-3) / HBM_PEAK, 3)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multichannel_train.py needs a CUDA device")
    if args.steps < 3:
        raise SystemExit("--steps must be at least 3")
    name, power = card()
    rows = [step_case(model(CIN), args.steps)]
    N.release_workspaces()
    torch.cuda.empty_cache()
    rows.append(step_case(model(1), args.steps))
    rows[-1]["note"] = "the monaural model of the same separator, for context"
    N.release_workspaces()
    torch.cuda.empty_cache()
    rows += kernel_case()
    for r in rows:
        r.update(card=name, power_limit=power)
        print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
