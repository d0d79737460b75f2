"""The edges of LSTM-TasNet's and GALRNet's kernels, shared by the CPU and the GPU edge tests: the recurrence's geometry restated
from ``ctn_tasnet.cu`` (U units per CTA, cpd CTAs per direction, the last CTA's nu units, the pass size), the rows chosen from it
for a device's SM count and opt-in shared memory, the rows of the encoder and GALR entries, and one planted mistake per edge.

The fp64 answers are the restatements of ``lstm_tasnet_ref`` (``lstm_ref``, ``enc_norm_ref``, ``tasnet_fwd``), ``galrnet_ref``
(``inter_block`` with its own gLN eps, ``head``, ``galrnet_fwd``, ``pe_table``) and ``tas_online_ref``; every comparison takes
``dual_path_edges_ref``'s bound per unit (a sequence and direction, a sample, a frame, a chunk), so a loud unit cannot hide an
error in a quiet one.  The planted mistakes go through a restatement of their own here (``recurrence``, ``gated_encoder``) that
equals the plain one when no mistake is planted (a CPU test holds it to that).
"""
import math

import torch
import torch.nn.functional as F_

import dual_path_edges_ref as D
import galrnet_ref as GR
import lstm_tasnet_ref as LR

check, excess, unit_errors, rel_of = D.check, D.excess, D.unit_errors, D.rel_of
MODES = ("fp32", "tf32x3", "f16x3", "tf32")
EPS = 1e-12
DEFECTS = ("last_cta_slice_dropped", "later_pass_carries_state", "prefetch_tile_stale", "gated_norm_frames_only",
           "batch_norm_instead_of_sample", "galr_eps_swapped", "galr_gln_eps_placement", "galr_down_last_pass_dropped",
           "galr_up_last_pass_dropped", "galr_position_q_major")

# the H100 SXM numbers DESIGN sections 16 and 18 state
H100_SMS, H100_SMEM_OPTIN = 132, 232448

# ---- the recurrence's geometry (ctn_tasnet.cu: lstm_smem_bytes, lstm_geo, ctn_tas_lstm_max_hidden) -------------------------------
TAS_THREADS, TAS_PF, TAS_GMAX = 256, 16, 16


def lstm_smem_bytes(H, U, gmax):
    """W_hh slice [4U][Hs], h [gmax][Hs], gate sums [4U][gmax], prefetch [2][4U][gmax][16] floats, Hs = H rounded up to 4"""
    Hs = (H + 3) & ~3
    return 4 * (4 * U * Hs + gmax * Hs + 4 * U * gmax + 2 * 4 * U * gmax * TAS_PF)


def lstm_geo(H, dirs, nsm, smem_optin):
    """dict(U, cpd, nu, group, smem) or None where H does not fit"""
    per_dir = nsm // dirs
    if H <= 0 or per_dir <= 0:
        return None
    U = -(-H // per_dir)
    cpd = -(-H // U)
    if U > TAS_THREADS:
        return None
    g = min(TAS_GMAX, TAS_THREADS // U)
    while g >= 1 and lstm_smem_bytes(H, U, g) > smem_optin:
        g -= 1
    if g < 1:
        return None
    return dict(U=U, cpd=cpd, nu=H - (cpd - 1) * U, group=g, smem=lstm_smem_bytes(H, U, g))


def lstm_max_hidden(dirs, nsm, smem_optin):
    lo, hi = 0, 1 << 16
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if lstm_geo(mid, dirs, nsm, smem_optin):
            lo = mid
        else:
            hi = mid - 1
    return lo


def u_steps(dirs, nsm, smem_optin):
    """the H values where U steps up (the first H of each U), up to the largest H"""
    hmax, out, prev = lstm_max_hidden(dirs, nsm, smem_optin), [], 0
    for H in range(1, hmax + 1):
        U = lstm_geo(H, dirs, nsm, smem_optin)["U"]
        if U != prev:
            out.append(H)
            prev = U
    return out


def hidden_rows(dirs, nsm, smem_optin):
    """(label, H): 1, 3, P, P + 1, 2P, 2P + 1, max - 1, max with P = SMs / dirs.  Where P + 1 or 2P + 1 leaves the last CTA more
    than one unit (P odd), the next H up whose last CTA owns exactly one is taken instead."""
    P, hmax = nsm // dirs, lstm_max_hidden(dirs, nsm, smem_optin)

    def one_unit(H):
        while lstm_geo(H, dirs, nsm, smem_optin)["nu"] != 1:
            H += 1
        return H
    return [("1", 1), ("3", 3), ("P", P), ("P+1", one_unit(P + 1)), ("2P", 2 * P), ("2P+1", one_unit(2 * P + 1)), ("max-1", hmax - 1),
            ("max", hmax)]


def lstm_rows(nsm, smem_optin):
    """the rows of ctn_tas_lstm_fwd: name -> dict(F, H, T, B, dirs, mode, skip, scales, alone).  Every H of hidden_rows for each
    dirs, with B in {1, 2, 3, 5, group, 2 group + 1}, T in {1, 15, 16, 17, 47, 48, 49} and F in {1, 7, 1001} cycled over them and
    every mode; then three passes at the largest H, a multi-pass row with skip_in / skip_out, a batch of sequences scaled 1e-3, 1
    and 1e3, and a three-pass batch whose sequences are each run alone too."""
    rows = {}
    Ts, Fs = (1, 15, 16, 17, 47, 48, 49), (1, 7, 1001)
    i = 0
    for dirs in (1, 2):
        for label, H in hidden_rows(dirs, nsm, smem_optin):
            g = lstm_geo(H, dirs, nsm, smem_optin)["group"]
            B = (1, 2, 3, 5, g, 2 * g + 1)[i % 6]
            rows["d{} H={}({}) B={} T={} F={}".format(dirs, label, H, B, Ts[i % 7], Fs[i % 3])] = dict(
                F=Fs[i % 3], H=H, T=Ts[i % 7], B=B, dirs=dirs, mode=MODES[i % 4], skip=False, scales=None, alone=False)
            i += 1
        hmax = lstm_max_hidden(dirs, nsm, smem_optin)
        g = lstm_geo(hmax, dirs, nsm, smem_optin)["group"]
        rows["d{} H=max({}) three passes".format(dirs, hmax)] = dict(F=7, H=hmax, T=17, B=2 * g + 1, dirs=dirs, mode="fp32", skip=False,
                                                                   scales=None, alone=False)
    dirs, H = 2, hidden_rows(2, nsm, smem_optin)[3][1]
    g = lstm_geo(H, dirs, nsm, smem_optin)["group"]
    rows["d2 H=P+1({}) three passes skip T=33".format(H)] = dict(F=7, H=H, T=33, B=2 * g + 1, dirs=2, mode="tf32x3", skip=True,
                                                                scales=None, alone=False)
    rows["d2 H=P+1({}) scaled 1e-3 1 1e3".format(H)] = dict(F=40, H=H, T=49, B=3, dirs=2, mode="fp32", skip=False,
                                                          scales=(1e-3, 1.0, 1e3), alone=False)
    rows["d2 H=P+1({}) three passes each alone".format(H)] = dict(F=24, H=H, T=20, B=2 * g + 1, dirs=2, mode="f16x3", skip=False,
                                                                 scales=None, alone=True)
    return rows


LSTM_DEFECT_ROWS = {"last_cta_slice_dropped": "d1 H=P+1(", "later_pass_carries_state": "d2 H=max(", "prefetch_tile_stale": "skip T=33"}


def lstm_defect_row(defect, nsm, smem_optin):
    """the name of the ctn_tas_lstm_fwd row each recurrence mistake is shown at: the last CTA owning one unit, three passes at
    the largest H, 33 steps (tiles of 16, 16 and 1) in both directions"""
    return next(n for n in lstm_rows(nsm, smem_optin) if LSTM_DEFECT_ROWS[defect] in n and
                (defect != "later_pass_carries_state" or "three passes" in n))


def lstm_weights(F, H, dirs, seed):
    """[w_ih, w_hh, b_ih, b_hh] per direction, U(-1/sqrt(H), 1/sqrt(H)) as nn.LSTM initialises them"""
    g = torch.Generator().manual_seed(seed)
    k = H ** -0.5
    ws = []
    for _ in range(dirs):
        ws += [(torch.rand(4 * H, F, generator=g) * 2 - 1) * k, (torch.rand(4 * H, H, generator=g) * 2 - 1) * k,
               (torch.rand(4 * H, generator=g) * 2 - 1) * k, (torch.rand(4 * H, generator=g) * 2 - 1) * k]
    return ws


def lstm_input(r, seed):
    """x (B, F, T) of a row, each sequence scaled by r['scales'] when given"""
    x = torch.randn(r["B"], r["F"], r["T"], generator=torch.Generator().manual_seed(seed))
    if r["scales"]:
        x = x * torch.tensor(r["scales"]).view(-1, 1, 1)
    return x


def recurrence(x, ws, dirs, geo, defect=None):
    """the recurrence entry in fp64 with one of the kernel's possible mistakes: x (B, F, T) -> (B, dirs H, T).  geo: U, cpd and
    the pass size (group) the kernel runs with.
    * last_cta_slice_dropped: units [(cpd - 1) U, H) are never updated (h and c stay 0);
    * later_pass_carries_state: sequence j of pass p > 0 starts from the final (h, c) of sequence j of pass p - 1;
    * prefetch_tile_stale: step s of a direction (its own order) with s % 16 == 0, s > 0, adds the projection of step s - 16."""
    B, _, T = x.shape
    xs = x.double().permute(0, 2, 1)
    outs = []
    for d in range(dirs):
        w_ih, w_hh, b_ih, b_hh = (t.double() for t in ws[4 * d:4 * d + 4])
        H = w_hh.shape[1]
        pre = (xs if d == 0 else torch.flip(xs, dims=(1,))) @ w_ih.t() + b_ih + b_hh   # (B, T, 4H), in the direction's order
        live = torch.ones(H, dtype=torch.float64)
        if defect == "last_cta_slice_dropped":
            live[(geo["cpd"] - 1) * geo["U"]:] = 0
        ys = torch.zeros(B, T, H, dtype=torch.float64)
        carry = None
        for b0 in range(0, B, geo["group"]):
            nb = min(geo["group"], B - b0)
            h = torch.zeros(nb, H, dtype=torch.float64)
            c = torch.zeros(nb, H, dtype=torch.float64)
            if defect == "later_pass_carries_state" and carry is not None:
                h, c = carry[0][:nb].clone(), carry[1][:nb].clone()
            for s in range(T):
                p = pre[b0:b0 + nb, s - TAS_PF if defect == "prefetch_tile_stale" and s >= TAS_PF and s % TAS_PF == 0 else s]
                i, f, gg, o = (p + h @ w_hh.t()).split(H, dim=1)
                c = (torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)) * live
                h = torch.sigmoid(o) * torch.tanh(c) * live
                ys[b0:b0 + nb, s] = h
            carry = (h, c)
        outs.append(ys if d == 0 else torch.flip(ys, dims=(1,)))
    return torch.cat(outs, dim=2).permute(0, 2, 1)


def lstm_answer(x, ws, dirs, geo, defect=None):
    return LR.lstm_ref(x, ws, dirs) if defect is None else recurrence(x, ws, dirs, geo, defect)


def lstm_units(y, B, dirs, H):
    """(B, dirs H, T) -> (B, dirs, H, T): one unit per (sequence, direction)"""
    return y.reshape(B, dirs, H, -1)


# ---- the gated encoder + frame norm (ctn_tas_enc_gated_fwd) and the frame norm alone (ctn_tas_frame_norm_fwd) -----------------
ENC_GEOMETRIES = ((40, 20), (16, 8), (2, 1), (4, 4), (20, 8))   # L / stride; 20 is not a multiple of 8
ENC_NS = (1, 31, 33, 500, 513)


def enc_smem_bytes(N, L, stride):
    nsamp = 7 * stride + L
    return 4 * (((nsamp + 3) & ~3) + 8 * N)


def enc_max_n(L, stride, smem_optin):
    """the most channels whose tile fits one CTA: the samples of 8 frames and an N x 8 tile"""
    return (max(smem_optin, 48 * 1024) // 4 - ((7 * stride + L + 3) & ~3)) // 8


def frame_norm_max_n(smem_optin):
    return max(smem_optin, 48 * 1024) // 32


def enc_rows():
    """the rows of ctn_tas_enc_gated_fwd: name -> dict(B, T, N, L, stride, pl, pr, amps, clicks).  Every remainder of
    (T + pl + pr - L) mod stride at every geometry (the ragged tail makes no frame but counts in the signal norm), N cycled over
    ENC_NS; then the loudness batch, and a click next to a near-silent recording.  (The largest N and the 1000 s recording are
    rows of their own in the GPU test.)"""
    rows, i = {}, 0
    for L, stride in ENC_GEOMETRIES:
        for rem in range(stride):
            pl, pr = i % 3, (i + 1) % 2
            T = L + 37 * stride + rem - pl - pr
            rows["{}/{} rem {} N={}".format(L, stride, rem, ENC_NS[i % 5])] = dict(B=2, T=T, N=ENC_NS[i % 5], L=L, stride=stride, pl=pl, pr=pr,
                                                                                  amps=None, clicks=())
            i += 1
    # ||x|| of the 1e-13 sample is about 1e-12, the encoder's eps
    rows["16/8 amplitudes 0 1e-13 1e-6 1 1e4"] = dict(B=5, T=101, N=33, L=16, stride=8, pl=1, pr=2, amps=(0.0, 1e-13, 1e-6, 1.0, 1e4),
                                                      clicks=())
    # a click (a single unit sample: the largest w any signal gives) next to a recording 1e-17 loud, whose norm is far below the
    # eps, so its w is about 1e-4 of the click's
    rows["2/1 click and 1e-17"] = dict(B=2, T=400, N=64, L=2, stride=1, pl=0, pr=0, amps=(1.0, 1e-17), clicks=(0,))
    return rows


ENC_DEFECT_ROWS = {"gated_norm_frames_only": "40/20 rem 19 N=513", "batch_norm_instead_of_sample": "2/1 click and 1e-17"}


def enc_params(N, L, seed):
    """U, V (N, 1, L) as the reference's Conv1d initialises them, gamma around 1, beta around 0 (1, N, 1)"""
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / math.sqrt(L)
    return {"encoder.conv1d_U.weight": (torch.rand(N, 1, L, generator=g) * 2 - 1) * k,
            "encoder.conv1d_V.weight": (torch.rand(N, 1, L, generator=g) * 2 - 1) * k,
            "separator.gamma": 1 + 0.1 * torch.randn(1, N, 1, generator=g), "separator.beta": 0.1 * torch.randn(1, N, 1, generator=g)}


def enc_input(r, seed):
    """x (B, 1, T) normals, sample b scaled by amps[b]; samples in `clicks` are one unit sample in the middle instead"""
    x = torch.randn(r["B"], 1, r["T"], generator=torch.Generator().manual_seed(seed))
    for b in r["clicks"]:
        x[b] = 0
        x[b, 0, r["T"] // 2] = 1.0
    if r["amps"]:
        x = x * torch.tensor(r["amps"]).view(-1, 1, 1)
    return x


def frame_norm(w, gamma, beta, eps):
    """w (B, N, frames) -> gamma (w - mean) / (sqrt(var) + eps) + beta over the N channels of each frame (tasnet.py:356-359)"""
    w = w.double()
    mean = w.mean(dim=1, keepdim=True)
    var = ((w - mean) ** 2).mean(dim=1, keepdim=True)
    return gamma.double() * (w - mean) / (torch.sqrt(var) + eps) + beta.double()


def signal_norm(x, L, stride, pl, pr, defect=None):
    """||x|| per sample (B, 1, 1) in fp64; the mistakes: the norm of the frames' samples only, and of the whole batch"""
    xp = F_.pad(x.double(), (pl, pr))
    if defect == "gated_norm_frames_only":
        frames = (xp.shape[-1] - L) // stride + 1
        xp = xp[..., :(frames - 1) * stride + L]
    if defect == "batch_norm_instead_of_sample":
        return torch.linalg.norm(xp).expand(x.shape[0], 1, 1)
    return torch.linalg.norm(xp, dim=2, keepdim=True)


def gated_encoder(x, p, L, stride, pl, pr, eps, defect=None):
    """(w, xn) of ctn_tas_enc_gated_fwd in fp64 with one of its possible mistakes in the signal norm"""
    xp = F_.pad(x.double(), (pl, pr)) / (signal_norm(x, L, stride, pl, pr, defect) + EPS)
    w = F_.conv1d(xp, p["encoder.conv1d_U.weight"].double(), stride=stride).relu() * \
        torch.sigmoid(F_.conv1d(xp, p["encoder.conv1d_V.weight"].double(), stride=stride))
    return w, frame_norm(w, p["separator.gamma"], p["separator.beta"], eps)


def enc_answer(x, p, L, stride, pl, pr, eps, defect=None):
    if defect is None:
        return LR.enc_norm_ref(x, p, dict(enc_basis="trainableGated", stride=stride, eps=eps), pl, pr)
    return gated_encoder(x, p, L, stride, pl, pr, eps, defect)


# ---- the globally attentive block (ctn_galr_inter_fwd) ---------------------------------------------------------------------------
GALR_FS = (32, 64, 128)


def galr_heads(F):
    """the head counts whose head dimension (8, 16, 32, 64) divides F"""
    return [F // d for d in (8, 16, 32, 64) if F % d == 0 and F // d >= 1 and F <= 128]


def galr_rows():
    """the rows of ctn_galr_inter_fwd: name -> dict(B, S, K, Q, F, heads, ln_eps, gn_eps, scale, amps).  For each F, Q and K
    around the pass of 2048 / F rows (P - 1, P, P + 1, and 2P + 1: three passes) and around the 32-row staging tile (31, 32, 33),
    each Q once with K = Q and once with the largest K; the head dimensions taken in turn.  Then the two eps told apart, the
    loudness batch, and the long attention sequences."""
    rows = {}
    for F in GALR_FS:
        P = GR.PASS_ELEMS // F
        vals = sorted({P - 1, P, P + 1, 2 * P + 1, 31, 32, 33})
        hs = galr_heads(F)
        i = 0
        for Q in vals:
            for K in sorted({Q, vals[-1]}):
                rows["F={} Q={} K={}".format(F, Q, K)] = dict(B=2, S=3, K=K, Q=Q, F=F, heads=hs[i % len(hs)], ln_eps=EPS, gn_eps=EPS, scale=1.0,
                                                           amps=None)
                i += 1
        # x scaled so LayerNorm's token variance is about 1e-3 and the gLN's about 1 (eps 1e-3 and 1e-1)
        rows["F={} eps 1e-3 1e-1".format(F)] = dict(B=2, S=5, K=P + 1, Q=P // 2 + 1, F=F, heads=hs[0], ln_eps=1e-3, gn_eps=1e-1, scale=0.05,
                                                    amps=None)
    rows["F=64 amplitudes 0 1e-3 1 1e3"] = dict(B=4, S=7, K=100, Q=32, F=64, heads=8, ln_eps=EPS, gn_eps=EPS, scale=1.0,
                                                amps=(0.0, 1e-3, 1.0, 1e3))
    rows["F=64 S=1200 Q=32"] = dict(B=1, S=1200, K=100, Q=32, F=64, heads=8, ln_eps=EPS, gn_eps=EPS, scale=1.0, amps=None)
    rows["F=32 S=2000 Q=64"] = dict(B=1, S=2000, K=100, Q=64, F=32, heads=4, ln_eps=EPS, gn_eps=EPS, scale=1.0, amps=None)
    return rows


GALR_DEFECT_ROWS = {"galr_eps_swapped": "F=64 eps 1e-3 1e-1", "galr_gln_eps_placement": "F=64 eps 1e-3 1e-1",
                    "galr_down_last_pass_dropped": "F=128 Q=17 K=17", "galr_up_last_pass_dropped": "F=128 Q=15 K=33",
                    "galr_position_q_major": "F=32 Q=33 K=129"}

INTER_KEYS = ("fc_map.weight", "fc_map.bias", "norm2d_in.norm.weight", "norm2d_in.norm.bias", "multihead_attn.in_proj_weight",
              "multihead_attn.in_proj_bias", "multihead_attn.out_proj.weight", "multihead_attn.out_proj.bias", "norm2d_out.norm.weight",
              "norm2d_out.norm.bias", "fc_inv.weight", "fc_inv.bias")


def inter_weights(F, K, Q, seed):
    shapes = {"fc_map.weight": (Q, K), "fc_map.bias": (Q,), "multihead_attn.in_proj_weight": (3 * F, F), "multihead_attn.in_proj_bias": (3 * F,),
              "multihead_attn.out_proj.weight": (F, F), "fc_inv.weight": (K, Q), "fc_inv.bias": (K,)}
    return GR.synth_state_dict([(k, shapes.get(k, (F,))) for k in INTER_KEYS], seed)


def inter_input(r, seed):
    x = torch.randn(r["B"], r["S"], r["K"], r["F"], generator=torch.Generator().manual_seed(seed)) * r["scale"]
    if r["amps"]:
        x = x * torch.tensor(r["amps"]).view(-1, 1, 1, 1)
    return x


def inter_answer(x, sd, heads, Q, ln_eps, gn_eps, defect=None):
    """galrnet_ref.inter_block with the LayerNorm's and the gLN's eps apart; the mistakes: the two eps exchanged, the position
    q S + s instead of s Q + q, and the in-block ones of galrnet_ref.EDGE_DEFECTS"""
    B, S, K, F = x.shape
    pe = GR.pe_table(S * Q, F)
    if defect == "galr_eps_swapped":
        ln_eps, gn_eps = gn_eps, ln_eps
    if defect == "galr_position_q_major":
        pe = pe.reshape(Q, S, F).transpose(0, 1).reshape(S * Q, F)
    return GR.inter_block(x.double(), sd, "", heads, Q, ln_eps, pe=pe, defect=defect if defect in GR.EDGE_DEFECTS else None,
                          gn_eps=gn_eps)


# ---- the separator head (ctn_galr_head_fwd) ---------------------------------------------------------------------------------------
def head_rows():
    """name -> dict(B, F, frames, K, P, amps): hops above, equal to and dividing the chunk and a hop of 1; K = 1; fewer frames
    than the chunk, made up by padding; the loudness batch"""
    rows = {}
    for i, (K, P) in enumerate(((16, 24), (16, 16), (16, 8), (16, 1), (1, 1), (1, 3), (100, 50))):
        for frames in sorted({max(1, K - 5), K, K + 21}):
            if GR.segment_geometry(frames, K, P)[2] < 1:        # a hop of 1 pads nothing: fewer frames than the chunk is refused
                continue
            rows["K={} P={} frames={}".format(K, P, frames)] = dict(B=2 + i % 2, F=(32, 64, 128)[i % 3], frames=frames, K=K, P=P, amps=None)
    rows["K=100 P=50 amplitudes 0 1e-3 1 1e3"] = dict(B=4, F=64, frames=499, K=100, P=50, amps=(0.0, 1e-3, 1.0, 1e3))
    return rows


def head_params(F, seed):
    g = torch.Generator().manual_seed(seed)
    return {"separator.norm2d.norm.weight": 1 + 0.1 * torch.randn(F, generator=g), "separator.norm2d.norm.bias": 0.1 * torch.randn(F, generator=g)}
