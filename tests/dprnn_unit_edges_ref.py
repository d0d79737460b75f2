"""fp64 restatements, geometry, rows and per-unit bounds of the DPRNN-TasNet edge tests (test_dprnn_unit_edges_cpu.py and
test_dprnn_unit_edges_gpu.py).

Four sections, each with its own unit, so a loud unit in a batch cannot hide an error in a quiet one:
  A. k_bilstm through ctn_bilstm_proj_fwd and ctn_bilstm_relu_proj_fwd: a unit is one (sequence, direction).  h within the
     2e-5 absolute floor; each direction's partial projection within 1e-4 max|fp64 of the unit| + 1e-6.  The one exception is
     the x1e3 group of the loudness row (``fp32_groups``): it is held to H_C x the fp32 CPU recurrence's own worst error on it.
  B. the gLN + residual of a dual-path block, ctn_dprnn_norm_res2_fwd (Y = P0 + P1 + bias) and the fallback ctn_dprnn_norm_res_fwd
     (Y given): a unit is one sample, every element within NORM_C u scale, scale = (sum|parts of Y| + |mean|) rstd |gamma| +
     |beta| + |R|.  |mean| in the scale keeps the bound honest under a DC offset: the fp32 rounding of Y and of Y - mean is
     relative to it.  The statistics themselves must then be summed in double: fp32 partials lose the variance there.
  C. ctn_segment_fwd / ctn_overlap_add_fwd: copies and a plain fp32 sum in chunk order, compared bit for bit.
  D. the whole DPRNNTasNet: a unit is one (sample, source), within 1e-4 max|fp64| + 1e-6 (dual_path_edges_ref's bound).

``DEFECTS`` plants one known mistake per section; the CPU file shows each is rejected at the exact shape of the GPU row named in
``DEFECT_ROWS``.
"""
import collections
import math

import torch
import torch.nn.functional as F_

import dprnn_oracle as DO
import dual_path_edges_ref as D
from test_dprnn_edges_gpu import _ring

U = 2.0 ** -24
NORM_C = 8.0
H_FLOOR, H_C = 2e-5, 8.0          # A: the floor of test_lstm_gpu and the fp32-recurrence rule of test_dprnn_edges_gpu
LSEQ = 64                         # sequences per k_bilstm CTA
NAMES = ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0", "weight_ih_l0_reverse", "weight_hh_l0_reverse",
         "bias_ih_l0_reverse", "bias_hh_l0_reverse")
INSTANTIATIONS = [(F, H) for F in (32, 64, 128) for H in (32, 64, 128)]
GRID_LIMIT = 65535

DEFECTS = ("reverse_run_forwards", "last_cta_row_shifted", "relu_in_recurrence", "hout_after_relu", "gln_per_sequence",
           "stats_one_direction_missing", "pad_left_right_exchanged", "residual_after_swap", "fp32_partial_stats")


# ---- geometry ------------------------------------------------------------------------------------------------------------------------
def ring(F, H, proj=True):
    """(ring depth nst, weight slabs per step) of k_bilstm; without the projection a step streams H/32 slabs fewer"""
    nst, per_step = _ring(F, H)
    return nst, per_step - (0 if proj else H // 32)


def ctas(NSEQ):
    """(CTAs per direction, rows of the last CTA)"""
    n = -(-NSEQ // LSEQ)
    return n, NSEQ - LSEQ * (n - 1)


def residue(F, H, T, proj=True):
    """T per_step mod nst: the ring stage the call's last slab lands in is residue - 1 (mod nst)"""
    nst, per_step = ring(F, H, proj)
    return (T * per_step) % nst


def residue_steps(F, H):
    """for every residue of the ring depth the step counts T * per_step can reach (the multiples of gcd(per_step, nst)), the
    smallest T >= 3 that lands on it"""
    nst, per_step = ring(F, H)
    out = {}
    T = 3
    while len(out) < nst // math.gcd(per_step, nst):
        out.setdefault((T * per_step) % nst, T)
        T += 1
    return out


def segment_geometry(frames, K, P):
    """the padding rule of dprnn_tasnet.py:339-341 -> (pad_left, pad_right, S)"""
    return D.segment_geometry(frames, K, P)


# ---- A. the bi-LSTM ------------------------------------------------------------------------------------------------------------------
def lstm_rows():
    """name -> row; entry 'proj' (ctn_bilstm_proj_fwd) or 'relu' (ctn_bilstm_relu_proj_fwd); outs 'both', 'P' or 'h'"""
    rows = collections.OrderedDict()

    def add(entry, name, F, H, Fo, NSEQ, T, reaches, outs="both", scales=None, ih_scale=1.0, idx=None, fp32_groups=()):
        rows["{}:{}".format(entry, name)] = dict(entry=entry, F=F, H=H, Fo=Fo, NSEQ=NSEQ, T=T, outs=outs, scales=scales, ih_scale=ih_scale,
                                                 idx=idx, fp32_groups=fp32_groups, reaches=reaches)
    for entry in ("proj", "relu"):
        for F, H in INSTANTIATIONS:
            nst, per_step = ring(F, H)
            for T in [1, 2] + sorted(residue_steps(F, H).values()):
                add(entry, "F{}H{}-T{}".format(F, H, T), F, H, F, 65, T,
                    "k_bilstm<NCH={}, KSX={}>: nst={}, per_step={}, T per_step = {} = {} mod nst; NSEQ=65: a 1-row last CTA".format(
                        H // 32, F // 32, nst, per_step, T * per_step, (T * per_step) % nst))
        for NSEQ in (1, 63, 64, 65, 129):
            n, last = ctas(NSEQ)
            add(entry, "NSEQ{}".format(NSEQ), 64, 128, 64, NSEQ, 5, "NSEQ={}: {} CTA(s) per direction, the last with {} row(s)".format(NSEQ, n, last))
        for Fo in (32, 96, 128):
            add(entry, "Fo{}".format(Fo), 64, 128, Fo, 65, 4, "Fo={} != F=64: the o < Fo guard of the P store and {} projection "
                                                                   "columns of the 128-column slab".format(Fo, Fo))
        add(entry, "P-only", 64, 128, 64, 65, 6, "hout null: only the P store", outs="P")
        if entry == "proj":
            add(entry, "h-only", 64, 128, 64, 65, 6, "w_fc and P null: per_step without the projection slabs ({})".format(ring(64, 128, False)[1]),
                outs="h")
        else:
            add(entry, "h-raw", 32, 64, 32, 65, 9, "hout next to a ReLU projection: hout holds the raw h, P sees ReLU(h)")
        add(entry, "T3840", 64, 128, 64, 65, 3840, "T=3840: the inter-chunk recurrence of 60 s at L=2, K=250, P=125; {} slabs per CTA "
                                                    "through a ring of {}".format(3840 * 28, 3), idx=[0, 63, 64])
        add(entry, "loudness-wih8", 64, 128, 64, 68, 250, "sequences x0, x1e-3, x1, x1e3 in one launch, W_ih x8: gates saturated by the "
            "input, W_hh at its default scale so the quiet sequences stay well conditioned; x0, x1e-3, x1 hold the floors",
            scales=[0.0, 1e-3, 1.0, 1e3], ih_scale=8.0, fp32_groups=(3,))
    return rows


def lstm_weights(F, H, Fo, seed, ih_scale=1.0):
    """the state dict of one IntraChunkRNN's LSTM + fc (torch's default init scale; W_ih of both directions times ih_scale)"""
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / math.sqrt(H)
    sd = {}
    for n in NAMES:
        shape = (4 * H, F) if "weight_ih" in n else ((4 * H, H) if "weight_hh" in n else (4 * H,))
        sd["rnn." + n] = (torch.rand(shape, generator=g) * 2 - 1) * k * (ih_scale if "weight_ih" in n else 1.0)
    sd["fc.weight"] = (torch.rand(Fo, 2 * H, generator=g) * 2 - 1) / math.sqrt(2 * H)
    sd["fc.bias"] = (torch.rand(Fo, generator=g) * 2 - 1) / math.sqrt(2 * H)
    return sd


def lstm_case(r):
    """(state dict, z (NSEQ, T, F)) of a row"""
    sd = lstm_weights(r["F"], r["H"], r["Fo"], r["F"] + r["H"] + r["Fo"] + r["T"], r["ih_scale"])
    z = torch.randn(r["NSEQ"], r["T"], r["F"], generator=torch.Generator().manual_seed(r["NSEQ"] + r["T"])) * 1.5
    if r["scales"]:
        s = torch.tensor(r["scales"])
        z = z * s[torch.arange(r["NSEQ"]) % len(s)].view(-1, 1, 1)
    return sd, z


def lstm_loop(z, wih, whh, bias, reverse, relu_feedback=False):
    """one direction of nn.LSTM step by step (gates i, f, g, o); relu_feedback feeds ReLU(h) back (a planted mistake)"""
    NSEQ, T, _ = z.shape
    H = whh.shape[1]
    xw = z @ wih.t() + bias
    h = torch.zeros(NSEQ, H, dtype=z.dtype)
    c = torch.zeros(NSEQ, H, dtype=z.dtype)
    out = torch.empty(NSEQ, T, H, dtype=z.dtype)
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        g = xw[:, t] + (torch.relu(h) if relu_feedback else h) @ whh.t()
        i, f, gg, o = g.chunk(4, 1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
        out[:, t] = h
    return out


def bilstm(z, sd, defect=None):
    """(NSEQ, T, 2H) in z's dtype: DO._bilstm (torch.lstm), or the step loop when a recurrence mistake is planted"""
    if defect not in ("reverse_run_forwards", "relu_in_recurrence"):
        return DO._bilstm(z, sd, "rnn.")
    w = [sd["rnn." + n] for n in NAMES]
    fwd = lstm_loop(z, w[0], w[1], w[2] + w[3], False, defect == "relu_in_recurrence")
    rev = lstm_loop(z, w[4], w[5], w[6] + w[7], defect != "reverse_run_forwards", defect == "relu_in_recurrence")
    return torch.cat([fwd, rev], dim=2)


def lstm_answer(z, sd, relu, dtype=torch.float64, defect=None):
    """(hout (NSEQ, T, 2H), P (2, NSEQ, T, Fo)) as the entry defines them: P[d] = W_fc[:, dH:(d+1)H] act(h_d), no bias; act = ReLU
    for the ReLU entry.  hout is the raw h in both entries."""
    sdd = {k: v.to(dtype) for k, v in sd.items()}
    z = z.to(dtype)
    if defect == "last_cta_row_shifted":  # the last CTA's row r reads row r + 1's input, its last row reads past the batch (0)
        NSEQ = z.shape[0]
        s0 = LSEQ * (ctas(NSEQ)[0] - 1)
        z = z.clone()
        z[s0:NSEQ - 1] = z[s0 + 1:NSEQ].clone()
        z[NSEQ - 1] = 0
    h = bilstm(z, sdd, defect)
    H = h.shape[2] // 2
    hp = torch.relu(h) if relu else h
    W = sdd["fc.weight"]
    P = torch.stack([hp[..., d * H:(d + 1) * H] @ W[:, d * H:(d + 1) * H].t() for d in (0, 1)])
    return (torch.relu(h) if defect == "hout_after_relu" else h), P


def h_units(h):
    """(NSEQ, T, 2H) -> (NSEQ, 2, T, H): one unit per (sequence, direction)"""
    NSEQ, T, H2 = h.shape
    return h.reshape(NSEQ, T, 2, H2 // 2).permute(0, 2, 1, 3)


def h_unit_errors(h, h64):
    """the largest |h - h64| of each (sequence, direction) unit (infinite where h is not finite)"""
    err, _ = D.unit_errors(h_units(h), h_units(h64), 2)
    return err


def lstm_excess(h, P, h64, P64, rule32=None):
    """worst unit's error over its bound, h and P together (either may be None).  Every (sequence, direction) unit is held to the
    floors, except the sequences of rule32 = (mask over sequences, h32, P32): those are held to H_C x the largest error the fp32
    CPU recurrence makes on them, h and P alike, where that is larger than the floor."""
    ratio = 0.0
    if h is not None:
        eh = h_unit_errors(h, h64).view(-1, 2)
        bh = torch.full_like(eh, H_FLOOR)
        if rule32 is not None:
            m, h32, _ = rule32
            bh[m] = max(H_FLOOR, H_C * float(h_unit_errors(h32, h64).view(-1, 2)[m].max()))
        ratio = float((eh / bh).max())
    if P is not None:
        ep, mp = D.unit_errors(P.transpose(0, 1), P64.transpose(0, 1), 2)
        ep, bp = ep.view(-1, 2), (D.BOUND_REL * mp + D.BOUND_ABS).view(-1, 2)
        if rule32 is not None:
            m, _, P32 = rule32
            ep32, _ = D.unit_errors(P32.transpose(0, 1), P64.transpose(0, 1), 2)
            bp[m] = torch.clamp(bp[m], min=H_C * float(ep32.view(-1, 2)[m].max()))
        ratio = max(ratio, float((ep / bp).max()))
    return ratio


def fp32_mask(r, idx):
    """the checked sequences (idx) that belong to the row's fp32_groups: at x1e3 and W_ih x8 a pre-activation near 1e4 carries
    about 2^-24 of its sum of |terms| (some 1e5) in any fp32 arithmetic, and the recurrence carries that on: the fp32 CPU
    recurrence itself is some 6e-4 off in h there, 30x the floor.  The quieter groups of the same row stay near 1e-7 .. 2e-6."""
    if not r["fp32_groups"]:
        return None
    g = idx % len(r["scales"])
    return torch.tensor([int(x) in r["fp32_groups"] for x in g])


# ---- B. gLN + residual ---------------------------------------------------------------------------------------------------------------
def norm_rows():
    """name -> row; entries: which of 'res2' (ctn_dprnn_norm_res2_fwd) and 'res' (ctn_dprnn_norm_res_fwd) it runs on"""
    rows = collections.OrderedDict()

    def add(name, B, D1, D2, F, swap, reaches, dc=0.0, where="bias", amps=None, eps=DO.EPS, pscale=1.0, entries=("res2", "res")):
        rows[name] = dict(B=B, D1=D1, D2=D2, F=F, swap=swap, dc=dc, where=where, amps=amps, eps=eps, pscale=pscale, entries=entries,
                          reaches=reaches)
    for dc in (0.0, 1e1, 1e2, 1e3, 1e4):
        for where, swap in (("bias", 0), ("P", 1)):
            add("dc{:g}-{}".format(dc, where), 2, 16, 32, 64, swap, "DC offset {:g} in {}: n = 32768 per sample over {} stats CTAs; "
                "Y spread x0.4, so the offset is 2500 standard deviations at 1e3".format(dc, where, 8), dc=dc, where=where, pscale=0.4)
    add("loudness", 4, 8, 20, 64, 1, "samples x0, x1e-3, x1, x1e3 (P and R) in one call", amps=[0.0, 1e-3, 1.0, 1e3])
    add("eps~var", 2, 6, 25, 32, 0, "eps = 1e-3 comparable to the variance of Y (~5e-4)", eps=1e-3, pscale=0.02)
    add("swap0", 3, 7, 11, 32, 0, "swap = 0: out in the input layout (B, D1, D2, F)")
    add("swap1", 3, 7, 11, 32, 1, "swap = 1: out in the other path's layout (B, D2, D1, F)")
    add("F4", 2, 3, 5, 4, 1, "F=4: block (1, 256), one float4 per row")
    add("F12", 2, 3, 89, 12, 0, "F=12: block (3, 85) = 255 threads, a partial last warp in the absmax reduction")
    add("F1024", 2, 2, 3, 1024, 1, "F=1024: block (256, 1), TY = 1")
    add("F33-unaligned", 3, 5, 7, 33, 1, "F=33 (fallback only): n = 1155 odd, samples 1 and 2 start off a 16-byte boundary: "
        "the scalar k_sample_stats and k_norm_res", entries=("res",))
    add("F33-2mod4", 3, 21, 10, 33, 0, "F=33 (fallback only): n = 6930 = 2 mod 4, sample 1 starts 8 bytes off", entries=("res",))
    return rows


def norm_case(r):
    """(P (2, B, D1, D2, F), bias (F), R, gamma, beta) of a row"""
    B, D1, D2, F = r["B"], r["D1"], r["D2"], r["F"]
    g = torch.Generator().manual_seed(B * 1000 + D1 * 100 + D2 + F)
    P = (torch.randn(2, B, D1, D2, F, generator=g) * 0.8 + 0.3) * r["pscale"]
    bias = 0.2 * torch.randn(F, generator=g) * r["pscale"]
    R = torch.randn(B, D1, D2, F, generator=g)
    gamma = 1.0 + 0.2 * (torch.rand(F, generator=g) - 0.5)
    beta = 0.1 * (torch.rand(F, generator=g) - 0.5)
    if r["amps"]:
        a = torch.tensor(r["amps"]).view(-1, 1, 1, 1)
        P, R = P * a, R * a
    if r["where"] == "bias":
        bias = bias + r["dc"]
    else:
        P[0] = P[0] + r["dc"]
    return P, bias, R, gamma, beta


def fallback_y(P, bias):
    """the fallback entry's Y: the fp32 sum P0 + P1 + bias the fused entry forms"""
    return P[0] + P[1] + bias


def fp32_partial_sums(Y):
    """per sample (sum, sumsq) as k_sample_stats2 formed them before the fix: each thread added 4 float4s (16 values) in fp32
    ((x + y) + (z + w) per float4, the squares as one fmaf chain), then went to double"""
    B = Y.shape[0]
    v = Y.float().reshape(B, -1, 4, 4)
    s4 = (v[..., 0] + v[..., 1]) + (v[..., 2] + v[..., 3])
    ls = torch.zeros(v.shape[:2], dtype=torch.float32)
    lss = torch.zeros(v.shape[:2], dtype=torch.float32)
    for u in range(4):
        ls = ls + s4[..., u]
        for e in (3, 2, 1, 0):  # fmaf(x, x, fmaf(y, y, fmaf(z, z, fmaf(w, w, lss)))): one rounding per fma
            x = v[..., u, e].double()
            lss = (x * x + lss.double()).float()
    return ls.double().sum(1), lss.double().sum(1)


def norm_answer(parts, R, gamma, beta, eps, swap, defect=None):
    """parts: the fp32 tensors whose sum is Y ([P0, P1, bias] or [Y]) -> (out64, scale), both in the stored layout"""
    Y = sum(p.double() for p in parts)
    B = R.shape[0]
    n = Y[0].numel()
    if defect == "gln_per_sequence":
        flat = Y.reshape(B, R.shape[1], -1)
        mean = flat.mean(2).view(B, -1, 1, 1)
        var = flat.var(2, unbiased=False).view(B, -1, 1, 1)
    else:
        S = Y if defect != "stats_one_direction_missing" else parts[0].double() + parts[2].double()
        if defect == "fp32_partial_stats":
            s, ss = fp32_partial_sums(sum(parts))
        else:
            s, ss = S.reshape(B, -1).sum(1), (S.reshape(B, -1) ** 2).sum(1)
        mean = (s / n).view(B, 1, 1, 1)
        var = (ss / n).view(B, 1, 1, 1) - mean ** 2
        if defect is None:
            flat = Y.reshape(B, -1)
            mean = flat.mean(1).view(B, 1, 1, 1)
            var = flat.var(1, unbiased=False).view(B, 1, 1, 1)
    rstd = 1.0 / torch.sqrt(var.clamp_min(0.0) + eps)
    g, b = gamma.double(), beta.double()
    norm = (Y - mean) * rstd * g + b
    absparts = sum(p.double().abs() for p in parts)
    scale = (absparts + mean.abs()) * rstd * g.abs() + b.abs() + R.double().abs()
    if swap:
        norm, scale = norm.transpose(1, 2), scale.transpose(1, 2)
        Rs = R.double().reshape(norm.shape) if defect == "residual_after_swap" else R.double().transpose(1, 2)
        return (norm + Rs).contiguous(), scale.contiguous()
    return norm + R.double(), scale


def norm_excess(out, ref, scale):
    """the worst element's error over NORM_C u scale (infinite where out is not finite)"""
    err = (out.double() - ref).abs()
    err[~torch.isfinite(err)] = math.inf
    return float((err / (NORM_C * U * scale)).max())


# ---- C. segmentation and overlap-add -------------------------------------------------------------------------------------------------
def seg_rows():
    """name -> (B, F, frames, K, P, reaches): every padding remainder of a small hop and of P = 125, hop > chunk, hop = chunk and a
    hop that does not divide the chunk"""
    rows = collections.OrderedDict()
    for j in range(5):
        rows["K12P5-r{}".format(j)] = (2, 33, 3 * 12 + j, 12, 5, "K=12, P=5: (frames - K) mod P = {}".format((3 * 12 + j - 12) % 5))
    for j in range(125):
        rows["K250P125-r{}".format(j)] = (1, 8, 1000 + j, 250, 125, "K=250, P=125: (frames - K) mod P = {}".format((1000 + j - 250) % 125))
    rows["hop>chunk"] = (3, 64, 251, 20, 30, "P=30 > K=20: frames in the gaps, the cudaMemsetAsync branch; overlap-add writes 0 there")
    rows["hop=chunk"] = (2, 5, 200, 25, 25, "P=K=25: one chunk per frame")
    rows["hop∤chunk"] = (2, 33, 301, 40, 15, "P=15 does not divide K=40: up to 3 chunks per frame, some 2")
    rows["S1"] = (1, 33, 90, 100, 50, "frames < K: the padding makes one chunk")
    return rows


def segment(x, K, P, pl, pr, channels_last, defect=None):
    """x (B, F, frames) -> Z, (B, S, K, F) channels-last or (B, F, S, K); a copy, so exact in any dtype"""
    if defect == "pad_left_right_exchanged":
        pl, pr = pr, pl
    Z = DO.segment1d(F_.pad(x, (pl, pr)), K, P)
    return Z.permute(0, 2, 3, 1).contiguous() if channels_last else Z


def overlap_add(Z, K, P, crop_left, T_out, out_pitch, channels_last):
    """Z -> y (B, F, out_pitch) in fp32: each frame the sum of its chunks from 0 in increasing s (F.fold's order), columns
    [T_out, out_pitch) 0"""
    Zr = Z.permute(0, 3, 1, 2) if channels_last else Z
    y = DO.overlap_add1d(Zr.float(), K, P)
    out = torch.zeros(y.shape[0], y.shape[1], out_pitch, dtype=torch.float32)
    out[..., :T_out] = y[..., crop_left:crop_left + T_out]
    return out


# ---- D. the model ----------------------------------------------------------------------------------------------------------------------
RECIPE = dict(n_basis=64, kernel_size=2, sep_bottleneck_channels=64, sep_hidden_channels=128, sep_chunk_size=250, sep_hop_size=125,
              sep_num_blocks=6)
SMALL = dict(n_basis=16, kernel_size=2, sep_bottleneck_channels=32, sep_hidden_channels=32, sep_chunk_size=12, sep_hop_size=5,
             sep_num_blocks=2)


def model_rows():
    """name -> (cfg, batch, samples, amps, reaches)"""
    rows = collections.OrderedDict()

    def long_text(what, samples):
        S = segment_geometry(samples - 1, 250, 125)[2]
        return "{}: intra {} sequences of 250 steps, inter 250 sequences of {} steps".format(what, S, S)
    rows["recipe-4s"] = (RECIPE, 1, 32000, None, long_text("recipe (6 blocks, F=64, H=128) at 4 s", 32000))
    rows["recipe-10s"] = (RECIPE, 1, 80000, None, long_text("recipe at 10 s", 80000))
    rows["F32H32-60s"] = (dict(RECIPE, sep_bottleneck_channels=32, sep_hidden_channels=32, sep_num_blocks=2), 1, 480000, None,
                          long_text("F=H=32, 2 blocks at 60 s", 480000))
    for j in range(5):
        T = 3 * 12 + j + 1  # frames = T - 1 at L=2
        rows["small-r{}".format(j)] = (SMALL, 2, T, None, "K=12, P=5: (frames - K) mod P = {}".format((T - 1 - 12) % 5))
    rows["1src"] = (dict(SMALL, n_sources=1), 2, 203, None, "1 source")
    rows["4src"] = (dict(SMALL, n_sources=4), 2, 203, None, "4 sources")
    rows["fallback"] = (dict(n_basis=16, kernel_size=2, sep_bottleneck_channels=33, sep_hidden_channels=24, sep_chunk_size=10, sep_hop_size=5,
                             sep_num_blocks=2), 3, 108, None, "F=33, H=24: cuDNN LSTM + ctn_dprnn_norm_res_fwd")
    rows["loudness"] = (SMALL, 5, 803, [0.0, 1e-6, 1e-3, 1.0, 1e3], "samples x0, x1e-6, x1e-3, x1, x1e3 in one batch")
    return rows


def model_launches(cfg, mode):
    """launches of DPRNNTasNet.forward: encoder 1, separator head 2, segment 1, per block two paths of (ctn_bilstm_proj_fwd 2 +
    ctn_dprnn_norm_res2_fwd 2), overlap-add 1, separator tail 2; the tensor-core modes add one weight image each to head and tail"""
    return 1 + 2 + 1 + 8 * cfg["sep_num_blocks"] + 1 + 2 + 2 * (mode != "fp32")


def model_input(batch, samples, amps, seed):
    x = torch.randn(batch, 1, samples, generator=torch.Generator().manual_seed(seed))
    if amps:
        x = x * torch.tensor(amps).view(-1, 1, 1)
    return x


def model_answer(x, sd, cfg, dtype=torch.float64):
    sdd = {k: v.to(dtype) for k, v in sd.items()}
    out, _ = DO.dprnn_tasnet_fwd(x.to(dtype), sdd, DO.DPRNNConfig(**cfg))
    return out


# ---- the planted mistakes and the rows that catch them --------------------------------------------------------------------------------
DEFECT_ROWS = {
    "reverse_run_forwards": ("A", "proj:F64H128-T2"),
    "last_cta_row_shifted": ("A", "proj:NSEQ65"),
    "relu_in_recurrence": ("A", "relu:F64H128-T5"),
    "hout_after_relu": ("A", "relu:h-raw"),
    "gln_per_sequence": ("B", "swap0"),
    "stats_one_direction_missing": ("B", "dc0-bias"),
    "pad_left_right_exchanged": ("C", "K250P125-r2"),
    "residual_after_swap": ("B", "swap1"),
    "fp32_partial_stats": ("B", "dc1000-bias"),
}
