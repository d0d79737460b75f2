#!/usr/bin/env python
"""SepFormer forward on one GPU: the wsj0-mix recipe shape (N = F = 256, L = 16, stride 8, C = 250, P = 125, 2 blocks x (8 intra +
8 inter) layers, 8 heads, d_ff = 1024, 2 sources) at B = 1 x 4 s, B = 1 x 10 s and B = 4 x 4 s (8 kHz), against the same modules in
torch eager (fp32, TF32 off).

    python tools/bench_sepformer.py [--iters 20] [--out bench_sepformer.json]

Reports per-call milliseconds (medians of CUDA-event timings), the kernel-time split between the contractions, attention, norms and
the rest (one torch.profiler pass of its own), launches per call, peak memory, achieved FLOP/s against the FLOPs computed from the
shapes here, and the card's name and power limit as read.
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
from ctn_b200.models.sepformer import SepFormer  # noqa: E402

CFG = dict(n_basis=256, kernel_size=16, stride=8, F=256, d_ff=1024, heads=8, C=250, P=125, blocks=2, layers=8, n_sources=2)


def geometry(T):
    c = CFG
    frames = (T - c["kernel_size"] + (c["stride"] - (T - c["kernel_size"]) % c["stride"]) % c["stride"]) // c["stride"] + 1
    padding = (c["P"] - (frames - c["C"]) % c["P"]) % c["P"]
    S = (frames + padding - c["C"]) // c["P"] + 1
    return frames, S


def flops(B, T):
    """multiply-adds x 2 of the dense products: the four Linear layers and the attention of every layer, the head and tail 1x1s"""
    c = CFG
    frames, S = geometry(T)
    F, C, d_ff = c["F"], c["C"], c["d_ff"]
    tok = B * S * C
    linear = 2 * tok * F * (3 * F + F + 2 * d_ff)
    intra = 2 * 2 * (B * S) * C * C * F
    inter = 2 * 2 * (B * C) * S * S * F
    per_block = c["layers"] * (2 * linear + intra + inter)
    Nb, ns = c["n_basis"], c["n_sources"]
    head_tail = 2 * B * frames * (Nb * F + F * ns * Nb + ns * 3 * Nb * Nb)
    return dict(total=c["blocks"] * per_block + head_tail, linear=c["blocks"] * c["layers"] * 2 * linear,
                intra=c["blocks"] * c["layers"] * intra, inter=c["blocks"] * c["layers"] * inter)


def build(dev):
    c = CFG
    m = SepFormer(c["n_basis"], c["kernel_size"], stride=c["stride"], enc_basis="trainable", dec_basis="trainable", enc_nonlinear="relu",
                  sep_bottleneck_channels=c["F"], sep_chunk_size=c["C"], sep_hop_size=c["P"], sep_num_blocks=c["blocks"],
                  sep_num_layers_intra=c["layers"], sep_num_layers_inter=c["layers"], sep_num_heads_intra=c["heads"],
                  sep_num_heads_inter=c["heads"], sep_d_ff_intra=c["d_ff"], sep_d_ff_inter=c["d_ff"], mask_nonlinear="relu", causal=False,
                  n_sources=c["n_sources"])
    return m.to(dev).eval()


def eager_forward(m, x):
    """the reference's forward in torch eager: the modules' own nn.TransformerEncoderLayer, GroupNorm, conv1d / fold"""
    sep = m.separator
    B, _, T = x.shape
    st, L = m.stride, m.kernel_size
    padding = (st - (T - L) % st) % st
    pl0, pr0 = padding // 2, padding - padding // 2
    w = torch.relu(F_.conv1d(F_.pad(x, (pl0, pr0)), m.encoder.conv1d.weight, stride=st))
    frames = w.shape[-1]
    K, P = sep.chunk_size, sep.hop_size
    padding = (P - (frames - K) % P) % P
    pl, pr = padding // 2, padding - padding // 2
    h = F_.group_norm(w, 1, sep.norm1d.norm.weight, sep.norm1d.norm.bias, sep.eps)
    z = F_.pad(F_.conv1d(h, sep.bottleneck_conv1d_in.weight, sep.bottleneck_conv1d_in.bias), (pl, pr)).unfold(2, K, P)  # (B, F, S, K)

    def encoder(pt, q):  # q (T, n, F)
        res = q
        q = q + pt.positional_encoding(q)
        for layer in pt.transformer.layers:
            q = layer(q)
        g = pt.transformer.norm.norm1d.norm
        return F_.group_norm(q.permute(1, 2, 0), 1, g.weight, g.bias, sep.eps).permute(2, 0, 1) + res

    Bc, S = z.shape[1], z.shape[2]
    for blk in sep.dptransformer.net:
        q = encoder(blk.intra_transformer, z.permute(3, 0, 2, 1).reshape(K, B * S, Bc))
        z = q.reshape(K, B, S, Bc).permute(1, 3, 2, 0)
        q = encoder(blk.inter_transformer, z.permute(2, 0, 3, 1).reshape(S, B * K, Bc))
        z = q.reshape(S, B, K, Bc).permute(1, 3, 0, 2)
    y = F_.fold(z.permute(0, 1, 3, 2).reshape(B, Bc * K, S), (1, (S - 1) * P + K), kernel_size=(1, K), stride=(1, P)).reshape(B, Bc, -1)
    y = F_.prelu(y[..., pl:pl + frames], sep.prelu.weight)
    mk = F_.conv1d(y, sep.map.weight, sep.map.bias).reshape(B * m.n_sources, m.n_basis, frames)
    u = torch.tanh(F_.conv1d(mk, sep.gtu.map.weight, sep.gtu.map.bias)) * torch.sigmoid(F_.conv1d(mk, sep.gtu.map_gate.weight,
                                                                                                    sep.gtu.map_gate.bias))
    u = torch.relu(F_.conv1d(u, sep.bottleneck_conv1d_out.weight, sep.bottleneck_conv1d_out.bias))
    what = (w.unsqueeze(1) * u.reshape(B, m.n_sources, m.n_basis, frames)).reshape(B * m.n_sources, m.n_basis, frames)
    out = F_.conv_transpose1d(what, m.decoder.conv_transpose1d.weight, stride=st).reshape(B, m.n_sources, -1)
    return out[..., pl0:out.shape[-1] - pr0]


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
    tot = {"contractions": 0.0, "attention": 0.0, "norms": 0.0, "rest": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        k = e.key
        if "k_pw" in k or "k_build_wimg" in k:
            tot["contractions"] += us / 1e3
        elif "k_sfm_attn" in k:
            tot["attention"] += us / 1e3
        elif "k_token_ln" in k or "k_sfm_seq_norm" in k:
            tot["norms"] += us / 1e3
        elif not k.startswith("cuda") and not k.startswith("Memcpy") and not k.startswith("Memset"):
            tot["rest"] += us / 1e3
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sepformer needs a CUDA device")
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
        frames, S = geometry(T)
        row = dict(B=B, seconds=secs, S=S, tokens=S * CFG["C"], ms=round(ms, 3), eager_ms=round(ms_eager, 3), speedup=round(ms_eager / ms, 2),
                   split_ms={k: round(v, 3) for k, v in parts.items()}, launches=launches, peak_mib=round(peak, 1),
                   gflop=round(fl["total"] / 1e9, 1), gflop_linear=round(fl["linear"] / 1e9, 1), gflop_attn_intra=round(fl["intra"] / 1e9, 1),
                   gflop_attn_inter=round(fl["inter"] / 1e9, 1), tflops=round(fl["total"] / ms / 1e9, 2),
                   attn_tflops=round((fl["intra"] + fl["inter"]) / max(parts["attention"], 1e-9) / 1e9, 2),
                   contraction_tflops=round(fl["linear"] / max(parts["contractions"], 1e-9) / 1e9, 2), rel_err_vs_eager=err)
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
