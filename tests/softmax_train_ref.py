"""fp64 reference and error bounds of the softmax-mask backward k_softmax_mask_bwd (ctn_probe_softmax_mask_bwd), test
infrastructure only.  The mask is softmax over ALL M = S*N channels of a frame (conv_tasnet.py:345-357), w_hat[s][n] = w[n] *
m[s][n]; with g = d_what * w:

    d_wprod[n] = sum_s d_what[s][n] m[s][n]
    dot        = sum_c m_c g_c = sum_n w[n] d_wprod[n]
    d_z        = m * (g - dot)

Bounds (u = 2^-24; inputs are fp32 values, the reference is exact in fp64 from them).  Let A[n] = sum_s |d_what m|.
  * d_wprod: an fma chain over S sources, |err| <= S u A[n]; stated as (S + 1) u A[n].
  * dot: each of 8 warps runs an fma chain over its k = ceil(N / 8) channels, then the 8 parts are summed; with the d_wprod
    errors carried in, |err(dot)| <= E_dot = (k + S + 8 + 2) u sum_n |w[n]| A[n].
  * d_z: fma(d_what, w, -dot~) rounds once and the product with m once:
    |err| <= m (E_dot + 3 u (|g| + |dot|)).
The mutants show the bounds are tight: dropping dot, or summing it over source 0 only, moves d_z by m |dot| (or m times the
missing sources' share), orders of magnitude past m E_dot."""
import torch

U = 2.0 ** -24
WARPS = 8

# name: (B, S, N, frames, kind, reaches)
ROWS = {
    "SN7-F5": (1, 1, 7, 5, "rand", "S*N = 7: fewer channels than warps (warps 7 has no n), one partial 32-frame tile"),
    "2x64-F129": (2, 2, 64, 129, "rand", "129 frames: one frame into the fifth 32-frame tile; pad lanes in the same warp"),
    "2x512-F4000": (4, 2, 512, 4000, "rand", "the ORPIT recipe's head: S*N = 1024, B = 4, 4 s at 8 kHz with L = 16 (4000 frames)"),
    "5x64-F300": (2, 5, 64, 300, "rand", "S*N = 320, the SinkPIT tutorial's five outputs"),
    "5x512-F499": (2, 5, 512, 499, "rand", "S*N = 2560, the widest row of the forward edge tests"),
    "onehot": (2, 2, 64, 200, "onehot", "logits of +-100: near one-hot masks (m = 0 or 1 in fp32), d_z = 0 almost everywhere"),
    "uniform": (2, 2, 64, 200, "uniform", "near-uniform masks m ~ 1/M: g - dot of the size of its rounding"),
    "relu-zeros": (2, 2, 64, 200, "relu", "w = relu(.): half the encoder outputs exactly 0 (g = 0, d_z = -m dot)"),
    "B3": (3, 3, 40, 77, "rand", "B = 3, S = 3: the grid's sample index"),
}


def inputs(name, seed=0):
    """(dwhat (B, S, N, F), w (B, N, F), m (B, S, N, F)) as fp32 values in float64 tensors"""
    B, S, N, F, kind, _ = ROWS[name]
    g = torch.Generator().manual_seed(1000 + seed + sum(map(ord, name)))
    dwhat = torch.randn(B, S, N, F, generator=g, dtype=torch.float64)
    w = torch.randn(B, N, F, generator=g, dtype=torch.float64)
    if kind == "relu":
        w = torch.relu(w)
    if kind == "onehot":
        z = 100.0 * torch.sign(torch.randn(B, S * N, F, generator=g, dtype=torch.float64)) + torch.randn(B, S * N, F, generator=g,
                                                                                                         dtype=torch.float64)
    elif kind == "uniform":
        z = 1e-3 * torch.randn(B, S * N, F, generator=g, dtype=torch.float64)
    else:
        z = 2.0 * torch.randn(B, S * N, F, generator=g, dtype=torch.float64)
    m = torch.softmax(z, dim=1).view(B, S, N, F)
    return dwhat.float().double(), w.float().double(), m.float().double()


def softmax_mask_bwd(dwhat, w, m, mut=None):
    """{name: (value, bound)}: 'dz' (B, S, N, F) and 'dwprod' (B, N, F).  mut: None, 'no_dot' or 'dot_src0' (defects)."""
    S, N = dwhat.shape[1], dwhat.shape[2]
    dwprod = (dwhat * m).sum(1)
    A = (dwhat * m).abs().sum(1)
    if mut == "dot_src0":
        dot = (w * dwhat[:, 0] * m[:, 0]).sum(1, keepdim=True)
    else:
        dot = (w * dwprod).sum(1, keepdim=True)
    if mut == "no_dot":
        dot = torch.zeros_like(dot)
    g = dwhat * w[:, None]
    k = (N + WARPS - 1) // WARPS
    e_dot = (k + S + WARPS + 2) * U * (w.abs() * A).sum(1, keepdim=True)
    dz = m * (g - dot[:, None])
    dz_bound = m * (e_dot[:, None] + 3 * U * (g.abs() + dot.abs()[:, None]))
    return {"dz": (dz, dz_bound), "dwprod": (dwprod, (S + 1) * U * A)}


def autograd_softmax_mask(dwhat, w, z):
    """the same derivatives by torch autograd through softmax(z over all S*N channels) and w_hat = w * m: (d_z, d_w)"""
    B, S, N, F = dwhat.shape
    z = z.clone().requires_grad_(True)
    w = w.clone().requires_grad_(True)
    m = torch.softmax(z, dim=1).view(B, S, N, F)
    what = w[:, None] * m
    (what * dwhat).sum().backward()
    return z.grad.view(B, S, N, F), w.grad


def finetune_loss(model, mixture, sources, crit):
    """the ORPIT fine-tune step's loss (egs/wsj0-mix/orpit_conv-tasnet/src/adhoc_driver.py, FinetuneTrainer.run_one_epoch_train):
    n - 1 stages for n-speaker targets; each stage drops the target it took as 'one' and feeds its 'rest' estimate back in as the
    next stage's mixture.  model: mixture (B, 1, T) -> (B, 2, T); crit: (est, sources) -> (loss, indices).  Returns (loss, [est])."""
    n = sources.size(1)
    total, ests = 0, []
    for stage in range(n - 1):
        est = model(mixture)
        loss, idx = crit(est, sources)
        total = total + loss
        ests.append(est)
        idx = idx.cpu()
        keep = [[j for j in range(n - stage) if j != int(idx[b])] for b in range(sources.size(0))]
        sources = torch.stack([sources[b, keep[b]] for b in range(sources.size(0))])
        mixture = est[:, 1:]
    return total, ests
