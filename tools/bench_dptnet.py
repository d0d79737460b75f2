#!/usr/bin/env python
"""DPTNet forward on one GPU: the recipe shape (N = 64, L = 2, F = 64, K = 250, P = 125, 6 blocks, d_ff = 128, h = 4, 2 sources)
at B = 1 x 4 s, B = 1 x 10 s and B = 4 x 4 s (8 kHz), against the same modules in torch eager (fp32, TF32 off).

    python tools/bench_dptnet.py [--iters 20] [--out bench_dptnet.json]

Reports per-call milliseconds (medians of CUDA-event timings), the kernel-time split between attention, LSTM and the rest (one
torch.profiler pass of its own), launches per call, peak memory, achieved FLOP/s against the FLOPs computed from the shapes here,
and the card's name and power limit.
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
from ctn_b200.models.dptnet import DPTNet  # noqa: E402

CFG = dict(n_basis=64, kernel_size=2, F=64, d_ff=128, heads=4, K=250, P=125, blocks=6, n_sources=2)


def geometry(B, T):
    c = CFG
    frames = T - c["kernel_size"] + 1
    padding = (c["P"] - (frames - c["K"]) % c["P"]) % c["P"]
    S = (frames + padding - c["K"]) // c["P"] + 1
    return frames, S


def flops(B, T):
    """multiply-adds x 2 of the separator's dense products (attention, its projections, LSTM gates and projection, 1x1s)"""
    c = CFG
    frames, S = geometry(B, T)
    F, H, K = c["F"], c["d_ff"], c["K"]
    tok = B * S * K
    per_path = 0.0
    for n_seq, L in ((B * S, K), (B * K, S)):
        per_path += 2 * n_seq * L * F * 4 * F           # QKV + output projection
        per_path += 2 * 2 * n_seq * L * L * F           # QK^T and PV over all heads
        per_path += 2 * 2 * n_seq * L * 4 * H * (F + H)  # two LSTM directions, gates
        per_path += 2 * 2 * n_seq * L * H * F           # the Linear after the LSTM
    head_tail = 2 * B * frames * (c["n_basis"] * F + F * c["n_sources"] * c["n_basis"] + c["n_sources"] * 2 * c["n_basis"] ** 2)
    return c["blocks"] * per_path + head_tail, tok


def build(dev):
    c = CFG
    m = DPTNet(c["n_basis"], c["kernel_size"], stride=1, enc_basis="trainable", dec_basis="trainable", enc_nonlinear="relu",
               sep_bottleneck_channels=c["F"], sep_hidden_channels=c["d_ff"], sep_chunk_size=c["K"], sep_hop_size=c["P"],
               sep_num_blocks=c["blocks"], sep_num_heads=c["heads"], mask_nonlinear="relu", causal=False, n_sources=c["n_sources"])
    return m.to(dev).eval()


def eager_forward(m, x):
    """the reference's forward in torch eager (nn.MultiheadAttention, cuDNN LSTM, GroupNorm), channels-first like the reference"""
    sep = m.separator
    B, _, T = x.shape
    w = torch.relu(F_.conv1d(x, m.encoder.conv1d.weight, stride=m.stride))
    frames = w.shape[-1]
    K, P = sep.chunk_size, sep.hop_size
    padding = (P - (frames - K) % P) % P
    pl, pr = padding // 2, padding - padding // 2
    h = F_.pad(F_.conv1d(w, sep.bottleneck_conv1d.weight, sep.bottleneck_conv1d.bias), (pl, pr))
    z = h.unfold(2, K, P)
    z = F_.group_norm(z, 1, sep.norm2d.norm.weight, sep.norm2d.norm.bias, sep.eps)

    def improved(tr, x):  # x (T, n, F)
        a = tr.multihead_attn_block
        y, _ = a.multihead_attn(x, x, x)
        y = F_.group_norm((y + x).permute(1, 2, 0), 1, a.norm1d.norm.weight, a.norm1d.norm.bias, sep.eps).permute(2, 0, 1)
        f = tr.subnet
        r, _ = f.rnn(y)
        u = F_.linear(torch.relu(r), f.fc.weight, f.fc.bias) + y
        return F_.group_norm(u.permute(1, 2, 0), 1, f.norm1d.norm.weight, f.norm1d.norm.bias, sep.eps).permute(2, 0, 1)

    Bc = z.shape[1]
    S = z.shape[2]
    for blk in sep.dptransformer.net:
        q = z.permute(3, 0, 2, 1).reshape(K, B * S, Bc)
        q = improved(blk.intra_chunk_block.transformer, q).reshape(K, B, S, Bc)
        z = q.permute(1, 3, 2, 0)
        q = z.permute(2, 0, 3, 1).reshape(S, B * K, Bc)
        q = improved(blk.inter_chunk_block.transformer, q).reshape(S, B, K, Bc)
        z = q.permute(1, 3, 0, 2)
    y = F_.fold(z.permute(0, 1, 3, 2).reshape(B, Bc * K, S), (1, (S - 1) * P + K), kernel_size=(1, K), stride=(1, P)).reshape(B, Bc, -1)
    y = F_.prelu(y[..., pl:pl + frames], sep.prelu.weight)
    mk = F_.conv1d(y, sep.map.weight, sep.map.bias).reshape(B * m.n_sources, m.n_basis, frames)
    u = torch.tanh(F_.conv1d(mk, sep.gtu.map.weight, sep.gtu.map.bias)) * torch.sigmoid(F_.conv1d(mk, sep.gtu.map_gate.weight,
                                                                                                    sep.gtu.map_gate.bias))
    what = (w.unsqueeze(1) * torch.relu(u).reshape(B, m.n_sources, m.n_basis, frames)).reshape(B * m.n_sources, m.n_basis, frames)
    return F_.conv_transpose1d(what, m.decoder.conv_transpose1d.weight, stride=m.stride).reshape(B, m.n_sources, -1)


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
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {"attention": 0.0, "lstm": 0.0, "rest": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        k = e.key
        if "k_attn" in k or "k_rowproj" in k:
            tot["attention"] += us / 1e3
        elif "k_bilstm" in k or "k_lstm_build" in k:
            tot["lstm"] += us / 1e3
        elif not k.startswith("cuda") and not k.startswith("Memcpy") and not k.startswith("Memset"):
            tot["rest"] += us / 1e3
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dptnet needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    if hasattr(getattr(torch.backends.cudnn, "rnn", None), "fp32_precision"):
        torch.backends.cudnn.rnn.fp32_precision = "ieee"
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
        fl, _ = flops(B, T)
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
            err = float((m(x) - eager_forward(m, x)).abs().max() / eager_forward(m, x).abs().max())
            parts = split(lambda: m(x))
        frames, S = geometry(B, T)
        row = dict(B=B, seconds=secs, S=S, ms=round(ms, 3), eager_ms=round(ms_eager, 3), speedup=round(ms_eager / ms, 2),
                   split_ms={k: round(v, 3) for k, v in parts.items()}, launches=launches, peak_mib=round(peak, 1),
                   gflop=round(fl / 1e9, 2), tflops=round(fl / ms / 1e9, 2), rel_err_vs_eager=err)
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
