#!/usr/bin/env python
"""GALRNet forward on one GPU: the wsj0-mix recipe shape (N = 64, L = 16, stride 8, H = 128, K = 100, P = 50, Q = 32, 6 blocks,
8 heads, 2 sources) at B = 1 x 4 s, B = 1 x 10 s and B = 4 x 4 s (8 kHz), against the same modules in torch eager (fp32, TF32 off,
cuDNN's LSTM in IEEE fp32; the positional encoding formed once per shape, not per call as the reference does).

    python tools/bench_galrnet.py [--iters 20] [--out bench_galrnet.json]

Reports per-call milliseconds (medians of CUDA-event timings after warm-up), the kernel-time split between the intra-chunk
LSTM blocks, the inter-chunk attentive blocks and the rest (one torch.profiler pass of its own), launches per call, peak memory,
achieved FLOP/s against the FLOPs computed from the shapes here, and the card's name and power limit.
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
from ctn_b200.models.galrnet import GALRNet  # noqa: E402

CFG = dict(n_basis=64, kernel_size=16, stride=8, H=128, K=100, P=50, Q=32, blocks=6, heads=8, n_sources=2)


def geometry(T):
    c = CFG
    frames = (T - c["kernel_size"]) // c["stride"] + 1
    padding = (c["P"] - (frames - c["K"]) % c["P"]) % c["P"]
    S = (frames + padding - c["K"]) // c["P"] + 1
    return frames, S


def flops(B, T):
    """multiply-adds x 2 of the dense products: LSTM gates and Linear, fc_map, attention and its projections, fc_inv, the tail's
    1x1s, encoder and decoder"""
    c = CFG
    frames, S = geometry(T)
    F, H, K, Q, ns = c["n_basis"], c["H"], c["K"], c["Q"], c["n_sources"]
    intra = 2 * 2 * B * S * K * 4 * H * (F + H) + 2 * B * S * K * 2 * H * F
    inter = 2 * B * S * Q * K * F + 2 * B * Q * S * 4 * F * F + 2 * 2 * B * Q * S * S * F + 2 * B * S * K * Q * F
    ends = 2 * B * frames * (F * ns * F + ns * 2 * F * F) + 2 * B * frames * F * c["kernel_size"] * (1 + ns)
    return c["blocks"] * (intra + inter) + ends, c["blocks"] * intra, c["blocks"] * inter


def build(dev):
    c = CFG
    m = GALRNet(c["n_basis"], c["kernel_size"], stride=c["stride"], enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None,
                sep_hidden_channels=c["H"], sep_chunk_size=c["K"], sep_hop_size=c["P"], sep_down_chunk_size=c["Q"],
                sep_num_blocks=c["blocks"], sep_num_heads=c["heads"], sep_norm=True, sep_dropout=0.1, mask_nonlinear="relu",
                low_dimension=True, causal=False, n_sources=c["n_sources"])
    return m.to(dev).eval()


_PE = {}


def eager_forward(m, x):
    """the reference's forward (galrnet.py:87-126, galr.py:161-197, dprnn.py:70-94) in torch eager, channels-first like it"""
    sep = m.separator
    B, _, T = x.shape
    L, st = m.kernel_size, m.stride
    padding = (st - (T - L) % st) % st
    pl0, pr0 = padding // 2, padding - padding // 2
    w = F_.conv1d(F_.pad(x, (pl0, pr0)), m.encoder.conv1d.weight, stride=st)
    frames = w.shape[-1]
    K, P, eps = sep.chunk_size, sep.hop_size, sep.eps
    padding = (P - (frames - K) % P) % P
    pl, pr = padding // 2, padding - padding // 2
    z = F_.group_norm(F_.pad(w, (pl, pr)).unfold(2, K, P), 1, sep.norm2d.norm.weight, sep.norm2d.norm.bias, eps)  # (B, F, S, K)
    Fc, S = z.shape[1], z.shape[2]
    for blk in sep.galr.net:
        ic, ib = blk.intra_chunk_block, blk.inter_chunk_block
        Q = ib.down_chunk_size
        r, _ = ic.rnn(z.permute(0, 2, 3, 1).reshape(B * S, K, Fc))
        y = F_.linear(r, ic.fc.weight, ic.fc.bias).reshape(B, S * K, Fc).permute(0, 2, 1)
        z = F_.group_norm(y, 1, ic.norm1d.norm.weight, ic.norm1d.norm.bias, eps).reshape(B, Fc, S, K) + z
        u = F_.linear(z, ib.fc_map.weight, ib.fc_map.bias)
        u = F_.layer_norm(u.permute(0, 2, 3, 1), (Fc,), ib.norm2d_in.norm.weight, ib.norm2d_in.norm.bias, eps).permute(0, 3, 1, 2)
        key = (S, Q, Fc)
        if key not in _PE:
            _PE[key] = ib.positional_encoding(S * Q, Fc).permute(1, 0).reshape(Fc, S, Q).to(x.device)
        u = (u + _PE[key]).permute(2, 0, 3, 1).reshape(S, B * Q, Fc)
        a, _ = ib.multihead_attn(u, u, u)
        a = (a + u).reshape(S, B, Q, Fc).permute(1, 3, 0, 2)
        a = F_.group_norm(a, 1, ib.norm2d_out.norm.weight, ib.norm2d_out.norm.bias, eps)
        z = F_.linear(a, ib.fc_inv.weight, ib.fc_inv.bias) + z
    y = F_.fold(z.permute(0, 1, 3, 2).reshape(B, Fc * K, S), (1, (S - 1) * P + K), kernel_size=(1, K), stride=(1, P)).reshape(B, Fc, -1)
    y = F_.prelu(y[..., pl:pl + frames], sep.prelu.weight)
    mk = F_.conv1d(y, sep.map.weight, sep.map.bias).reshape(B * m.n_sources, m.n_basis, frames)
    u = torch.tanh(F_.conv1d(mk, sep.gtu.map.weight, sep.gtu.map.bias)) * torch.sigmoid(F_.conv1d(mk, sep.gtu.map_gate.weight,
                                                                                                    sep.gtu.map_gate.bias))
    what = (w.unsqueeze(1) * torch.relu(u).reshape(B, m.n_sources, m.n_basis, frames)).reshape(B * m.n_sources, m.n_basis, frames)
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
    """kernel milliseconds of one call: intra (bi-LSTM + its gLN / residual), inter (down-map, attention, gLN statistics,
    up-map; the head's one gLN-statistics launch shares a kernel with it), rest"""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {"intra_lstm": 0.0, "inter_block": 0.0, "rest": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us <= 0:
            continue
        k = e.key
        if "k_bilstm" in k or "k_lstm_build" in k or "k_sample_stats2" in k or "k_norm_res2" in k:
            tot["intra_lstm"] += us / 1e3
        elif "k_galr" in k or "k_attn" in k or "k_rowproj" in k or "k_sample_part" in k:
            tot["inter_block"] += us / 1e3
        elif not k.startswith("cuda") and not k.startswith("Memcpy") and not k.startswith("Memset"):
            tot["rest"] += us / 1e3
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_galrnet needs a CUDA device")
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
        fl, fl_intra, fl_inter = flops(B, T)
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
        row = dict(B=B, seconds=secs, S=S, ms=round(ms, 3), eager_ms=round(ms_eager, 3), speedup=round(ms_eager / ms, 2),
                   split_ms={k: round(v, 3) for k, v in parts.items()}, launches=launches, peak_mib=round(peak, 1),
                   gflop=round(fl / 1e9, 2), gflop_intra=round(fl_intra / 1e9, 2), gflop_inter=round(fl_inter / 1e9, 2),
                   tflops=round(fl / ms / 1e9, 2), rel_err_vs_eager=err)
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
