#!/usr/bin/env python
"""LSTM-TasNet forward on one GPU: the wsj0-mix recipe shape (gated encoder, N = 500, L = 40, stride 20, H = 500, 2 blocks x 2
bi-LSTM layers, sigmoid mask, 2 sources) at B = 1 x 4 s, B = 1 x 10 s and B = 4 x 4 s (8 kHz), against the same modules in torch
eager (cuDNN's LSTM, fp32, TF32 off).

    python tools/bench_lstm_tasnet.py [--iters 20] [--out bench_lstm_tasnet.json]

Reports per-call milliseconds (medians of CUDA-event timings), the kernel-time split between the input projections, the
recurrence and the rest (one torch.profiler pass of its own), microseconds per recurrence step, launches per call, peak memory,
FLOPs computed from the shapes here, and the card's name and power limit as read.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))
from ctn_b200 import _native as N  # noqa: E402
from ctn_b200.models.tasnet import TasNet  # noqa: E402

CFG = dict(n_basis=500, kernel_size=40, stride=20, H=500, blocks=2, layers=2, n_sources=2, dirs=2)


def frames_of(T):
    c = CFG
    L, s = c["kernel_size"], c["stride"]
    return (T + (s - (T - L) % s) % s - L) // s + 1


def flops(B, T):
    """2 x multiply-adds of the dense products, from the shapes"""
    c = CFG
    Tf, Nb, H, d = frames_of(T), c["n_basis"], c["H"], c["dirs"]
    n_layers = c["blocks"] * c["layers"]
    inproj = sum(2 * B * Tf * d * 4 * H * (Nb if i == 0 else d * H) for i in range(n_layers))
    rec = 2 * B * Tf * d * 4 * H * H * n_layers
    fc = 2 * B * Tf * d * H * c["n_sources"] * Nb
    enc = 2 * 2 * B * Tf * Nb * c["kernel_size"]
    dec = 2 * B * c["n_sources"] * Tf * Nb * c["kernel_size"]
    return dict(total=inproj + rec + fc + enc + dec, inproj=inproj, recurrence=rec, fc=fc, encoder=enc, decoder=dec,
                steps=n_layers * Tf)


def build(dev):
    c = CFG
    m = TasNet(c["n_basis"], kernel_size=c["kernel_size"], stride=c["stride"], enc_basis="trainableGated", dec_basis="trainable",
               sep_num_blocks=c["blocks"], sep_num_layers=c["layers"], sep_hidden_channels=c["H"], mask_nonlinear="sigmoid", causal=False,
               rnn_type="lstm", n_sources=c["n_sources"])
    return m.to(dev).eval()


def eager_forward(m, x):
    """the reference's forward in torch eager: the modules' own conv1d / nn.LSTM (cuDNN) / Linear"""
    sep = m.separator
    B, _, T = x.shape
    st, L = m.stride, m.kernel_size
    padding = (st - (T - L) % st) % st
    pl, pr = padding // 2, padding - padding // 2
    x = F_.pad(x, (pl, pr))
    x = x / (torch.linalg.norm(x, dim=2, keepdim=True) + m.encoder.eps)
    w = torch.relu(F_.conv1d(x, m.encoder.conv1d_U.weight, stride=st)) * torch.sigmoid(F_.conv1d(x, m.encoder.conv1d_V.weight, stride=st))
    mean = w.mean(dim=1, keepdim=True)
    var = (w ** 2).mean(dim=1, keepdim=True) - mean ** 2
    z = (sep.gamma * (w - mean) / (torch.sqrt(var) + sep.eps) + sep.beta).permute(0, 2, 1).contiguous()
    skip = 0
    for rnn in sep.rnn:
        z, _ = rnn(z)
        skip = z + skip
    y = sep.fc(skip).view(B, -1, m.n_sources, m.n_basis).permute(0, 2, 3, 1)
    what = (w.unsqueeze(1) * torch.sigmoid(y)).reshape(B * m.n_sources, m.n_basis, -1)
    out = F_.conv_transpose1d(what, m.decoder.conv_transpose1d.weight, stride=st).reshape(B, m.n_sources, -1)
    return out[..., pl:out.shape[-1] - pr]


def time_ms(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def split(fn):
    """kernel milliseconds of one call: the recurrence launches, the input-projection contractions (every k_pw launch but the
    last, which is fc, with their weight images), and the rest"""
    from torch.autograd import DeviceType
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ks = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and e.time_range.elapsed_us() > 0
                 and not e.name.startswith(("Memcpy", "Memset", "cuda"))), key=lambda e: e.time_range.start)
    pw = [i for i, e in enumerate(ks) if "k_pw" in e.name]
    tot = {"input_projections": 0.0, "recurrence": 0.0, "rest": 0.0}
    for i, e in enumerate(ks):
        ms = e.time_range.elapsed_us() / 1e3
        if "k_tas_lstm(" in e.name or e.name.endswith("k_tas_lstm"):
            tot["recurrence"] += ms
        elif ("k_pw" in e.name and i != pw[-1]) or "k_tas_lstm_prep" in e.name or ("k_build_wimg" in e.name and i < pw[-1] - 1):
            tot["input_projections"] += ms
        else:
            tot["rest"] += ms
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lstm_tasnet needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        card = q.stdout.strip().splitlines()[0]
    except Exception:
        card = torch.cuda.get_device_name(0)
    torch.manual_seed(0)
    m = build(dev)
    rows = []
    for B, secs in ((1, 4), (1, 10), (4, 4)):
        T = 8000 * secs
        x = torch.randn(B, 1, T, device=dev)
        fl = flops(B, T)
        with torch.no_grad():
            for _ in range(3):
                m(x)
                eager_forward(m, x)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            n0 = N.ctn_total_launch_count()
            m(x)
            torch.cuda.synchronize()
            launches = int(N.ctn_total_launch_count() - n0)
            peak = torch.cuda.max_memory_allocated() / 2 ** 20
            ms = time_ms(lambda: m(x), args.iters)
            ms_eager = time_ms(lambda: eager_forward(m, x), args.iters)
            ref = eager_forward(m, x)
            err = float((m(x) - ref).abs().max() / ref.abs().max())
            parts = split(lambda: m(x))
        row = dict(B=B, seconds=secs, frames=frames_of(T), ms=round(ms, 3), eager_ms=round(ms_eager, 3), speedup=round(ms_eager / ms, 2),
                   split_ms={k: round(v, 3) for k, v in parts.items()}, us_per_step=round(parts["recurrence"] * 1e3 / fl["steps"], 3),
                   launches=launches, peak_mib=round(peak, 1), gflop=round(fl["total"] / 1e9, 2),
                   gflop_inproj=round(fl["inproj"] / 1e9, 2), gflop_recurrence=round(fl["recurrence"] / 1e9, 2),
                   gflop_fc=round(fl["fc"] / 1e9, 2), gflop_enc=round(fl["encoder"] / 1e9, 3), gflop_dec=round(fl["decoder"] / 1e9, 3),
                   inproj_tflops=round(fl["inproj"] / max(parts["input_projections"], 1e-9) / 1e9, 2),
                   recurrence_tflops=round(fl["recurrence"] / max(parts["recurrence"], 1e-9) / 1e9, 3), rel_err_vs_eager=err)
        rows.append(row)
        print(json.dumps(row))
    res = {"card": card, "cfg": CFG, "rows": rows}
    print(json.dumps({"card": card}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
