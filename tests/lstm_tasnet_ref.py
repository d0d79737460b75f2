"""fp64 restatement of LSTM-TasNet (src/models/tasnet.py:146-189, 324-381; src/models/filterbank.py:325-346), every stage written
out: the ConvTasNet padding, the gated (or plain) encoder, the per-frame norm, the (bi-)LSTM blocks with their skip sum, fc, the mask
over the sources and the transposed-conv decoder.  ``defect`` plants one known mistake, for the tests that show the bound rejects it.
"""
import math

import torch
import torch.nn.functional as F

EPS = 1e-12
BOUND_REL, BOUND_ABS = 1e-4, 1e-6  # |native - fp64| <= 1e-4 max|fp64| + 1e-6, as for DPTNet and SepFormer
DEFECTS = ("seg_norm", "norm_time", "no_flip", "skip_last", "swap_if", "no_bhh", "leak", "softmax_channels", "fc_ns")


def bound(ref):
    return BOUND_REL * float(ref.abs().max()) + BOUND_ABS


def synth_state_dict(keys_shapes, seed):
    """seeded weights for the reference's keys: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) like torch's defaults, gamma around 1, beta
    around 0"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in keys_shapes:
        shape = tuple(shape)
        if k.endswith("gamma"):
            v = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif k.endswith("beta"):
            v = 0.1 * torch.randn(shape, generator=g)
        else:
            if "rnn" in k:  # nn.LSTM: every tensor U(-1/sqrt(H), 1/sqrt(H)), first dim 4H
                fan_in = shape[0] // 4
            elif "conv_transpose1d" in k:
                fan_in = shape[1] * shape[2]
            elif len(shape) >= 2:
                fan_in = math.prod(shape[1:])
            else:
                fan_in = shape[0]
            b = 1.0 / math.sqrt(fan_in)
            v = (torch.rand(shape, generator=g) * 2 - 1) * b
        sd[k] = v.float()
    return sd


def lstm_layer(x, sd, prefix, layer, dirs, defect=None):
    """x (B, T, F) fp64 -> (B, T, dirs H): one nn.LSTM layer, zero initial state, gate order i, f, g, o"""
    B, T, _ = x.shape
    outs = []
    for d in range(dirs):
        sfx = "_l{}".format(layer) + ("_reverse" if d else "")
        w_ih, w_hh = sd[prefix + "weight_ih" + sfx].double(), sd[prefix + "weight_hh" + sfx].double()
        b = sd[prefix + "bias_ih" + sfx].double() + (0 if defect == "no_bhh" else sd[prefix + "bias_hh" + sfx].double())
        H = w_hh.shape[1]
        xs = x if d == 0 else torch.flip(x, dims=(1,))
        pre = xs @ w_ih.t() + b  # (B, T, 4H)
        h = torch.zeros(B, H, dtype=torch.float64)
        c = torch.zeros(B, H, dtype=torch.float64)
        hs = []
        for t in range(T):
            gts = pre[:, t] + h @ w_hh.t()
            i, f, gg, o = gts.split(H, dim=1)
            if defect == "swap_if":
                i, f = f, i
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            hs.append(h)
        y = torch.stack(hs, dim=1)
        if defect == "leak":  # run the batch as one long sequence instead
            return lstm_layer(x.reshape(1, B * T, -1), sd, prefix, layer, dirs).reshape(B, T, -1)
        if d == 1 and defect != "no_flip":
            y = torch.flip(y, dims=(1,))
        outs.append(y)
    return torch.cat(outs, dim=2)


def tasnet_fwd(x, sd, cfg, defect=None):
    """x (B, 1, T) -> (B, S, T) in fp64.  cfg: n_basis, kernel_size, stride, enc_basis, enc_nonlinear, sep_num_blocks,
    sep_num_layers, causal, mask_nonlinear, n_sources, eps"""
    x = x.double()
    L, stride = cfg["kernel_size"], cfg["stride"]
    Nb, S = cfg["n_basis"], cfg["n_sources"]
    eps = cfg.get("eps", EPS)
    B, _, T = x.shape
    padding = (stride - (T - L) % stride) % stride
    pl, pr = padding // 2, padding - padding // 2
    x = F.pad(x, (pl, pr))
    if cfg["enc_basis"] == "trainableGated":
        if defect == "seg_norm":  # each frame's segment normalised on its own
            seg = x.unfold(2, L, stride)  # (B, 1, T', L)
            seg = seg / (torch.linalg.norm(seg, dim=3, keepdim=True) + EPS)
            w = torch.einsum("bctl,ncl->bnt", seg, sd["encoder.conv1d_U.weight"].double()).relu() * \
                torch.sigmoid(torch.einsum("bctl,ncl->bnt", seg, sd["encoder.conv1d_V.weight"].double()))
        else:
            xn = x / (torch.linalg.norm(x, dim=2, keepdim=True) + EPS)  # the encoder's eps is always the default (tasnet.py:110)
            w = F.conv1d(xn, sd["encoder.conv1d_U.weight"].double(), stride=stride).relu() * \
                torch.sigmoid(F.conv1d(xn, sd["encoder.conv1d_V.weight"].double(), stride=stride))
    else:
        w = F.conv1d(x, sd["encoder.conv1d.weight"].double(), stride=stride)
        if cfg.get("enc_nonlinear") == "relu":
            w = w.relu()
    dim = 2 if defect == "norm_time" else 1
    mean = w.mean(dim=dim, keepdim=True)
    var = ((w - mean) ** 2).mean(dim=dim, keepdim=True)
    z = sd["separator.gamma"].double() * (w - mean) / (torch.sqrt(var) + eps) + sd["separator.beta"].double()
    z = z.permute(0, 2, 1)
    dirs = 1 if cfg["causal"] else 2
    skip = 0
    for blk in range(cfg["sep_num_blocks"]):
        for layer in range(cfg["sep_num_layers"]):
            z = lstm_layer(z, sd, "separator.rnn.{}.".format(blk), layer, dirs, defect)
        skip = z if defect == "skip_last" else z + skip
    y = skip @ sd["separator.fc.weight"].double().t() + sd["separator.fc.bias"].double()  # (B, T', S N)
    Tf = y.shape[1]
    if defect == "fc_ns":
        y = y.view(B, Tf, Nb, S).permute(0, 3, 2, 1)
    else:
        y = y.view(B, Tf, S, Nb).permute(0, 2, 3, 1)  # (B, S, N, T')
    if cfg["mask_nonlinear"] == "sigmoid":
        mask = torch.sigmoid(y)
    else:
        mask = torch.softmax(y, dim=2 if defect == "softmax_channels" else 1)
    what = (w.unsqueeze(1) * mask).reshape(B * S, Nb, Tf)
    out = F.conv_transpose1d(what, sd["decoder.conv_transpose1d.weight"].double(), stride=stride).view(B, S, -1)
    return out[..., pl:out.shape[-1] - pr]


def lstm_ref(x, ws, dirs):
    """the recurrence entry's contract in fp64: x (B, F, T) channel-first -> (B, dirs H, T); ws = [w_ih, w_hh, b_ih, b_hh] per
    direction"""
    sd = {}
    for d in range(dirs):
        sfx = "_l0" + ("_reverse" if d else "")
        for n, t in zip(("weight_ih", "weight_hh", "bias_ih", "bias_hh"), ws[4 * d:4 * d + 4]):
            sd[n + sfx] = t
    return lstm_layer(x.double().permute(0, 2, 1), sd, "", 0, dirs).permute(0, 2, 1)


def enc_norm_ref(x, sd, cfg, pl, pr):
    """(w, xn) of the encoder + frame norm in fp64: x (B, 1, T)"""
    x = F.pad(x.double(), (pl, pr))
    if cfg["enc_basis"] == "trainableGated":
        xn = x / (torch.linalg.norm(x, dim=2, keepdim=True) + EPS)
        w = F.conv1d(xn, sd["encoder.conv1d_U.weight"].double(), stride=cfg["stride"]).relu() * \
            torch.sigmoid(F.conv1d(xn, sd["encoder.conv1d_V.weight"].double(), stride=cfg["stride"]))
    else:
        w = F.conv1d(x, sd["encoder.conv1d.weight"].double(), stride=cfg["stride"])
        if cfg.get("enc_nonlinear") == "relu":
            w = w.relu()
    mean = w.mean(dim=1, keepdim=True)
    var = ((w - mean) ** 2).mean(dim=1, keepdim=True)
    z = sd["separator.gamma"].double() * (w - mean) / (torch.sqrt(var) + cfg.get("eps", EPS)) + sd["separator.beta"].double()
    return w, z
