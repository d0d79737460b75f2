"""fp64 restatement of online (chunk-by-chunk) LSTM-TasNet inference, the contract of ``TasNet.online``: each push of n samples
carries the encoder's last L - S input samples, (h, c) of every unidirectional LSTM layer and the decoder's last L/S - 1 frames, and
returns the n output samples D = L - S late.  With Y the concatenated push outputs and Z the flush, cat(Y[..., D:], Z) equals
``lstm_tasnet_ref.tasnet_fwd`` of the whole signal.  ``defect`` plants one known mistake, for the tests that show the bound rejects it.
"""
import torch
import torch.nn.functional as F

import lstm_tasnet_ref as R

DEFECTS = ("reset_state", "no_c", "delay", "no_hist", "count_incomplete")
# stream against the offline model in the same numeric mode: |stream - offline| <= 1e-6 |offline| + 1e-7 max|offline|
REL, ABS_OF_MAX = 1e-6, 1e-7


def frames_done(T, L, S):
    """frames complete after T samples (T a multiple of S): the Conv1d over the unpadded prefix"""
    return (T - L) // S + 1 if T >= L else 0


def _lstm_steps(z, sd, prefix, layer, h, c):
    """z (B, T, F) fp64, (h, c) (B, H) -> (B, T, H), (h, c) after the last step; gate order i, f, g, o"""
    sfx = "_l{}".format(layer)
    w_ih, w_hh = sd[prefix + "weight_ih" + sfx].double(), sd[prefix + "weight_hh" + sfx].double()
    b = sd[prefix + "bias_ih" + sfx].double() + sd[prefix + "bias_hh" + sfx].double()
    H = w_hh.shape[1]
    pre = z @ w_ih.t() + b
    hs = []
    for t in range(z.shape[1]):
        i, f, g, o = (pre[:, t] + h @ w_hh.t()).split(H, dim=1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        hs.append(h)
    y = torch.stack(hs, dim=1) if hs else z.new_zeros(z.shape[0], 0, H)
    return y, h, c


class Stream:
    """B streams of a causal, plain-encoder model in fp64.  cfg as for ``lstm_tasnet_ref.tasnet_fwd``."""

    def __init__(self, sd, cfg, batch, defect=None):
        assert cfg["causal"] and cfg["enc_basis"] == "trainable"
        self.sd, self.cfg, self.B, self.defect = sd, cfg, batch, defect
        self.L, self.S = cfg["kernel_size"], cfg["stride"]
        self.D, self.Rf = self.L - self.S, self.L // self.S
        self.Nb, self.Ns = cfg["n_basis"], cfg["n_sources"]
        self.H = sd["separator.rnn.0.weight_hh_l0"].shape[1]
        self.reset()

    def reset(self):
        B, H = self.B, self.H
        self.T0 = 0
        self.carry = torch.zeros(B, 1, self.D, dtype=torch.float64)
        self.hist = torch.zeros(B * self.Ns, self.Nb, self.Rf - 1, dtype=torch.float64)  # frames [F0 - (L/S - 1), F0)
        self.hc = {(blk, k): (torch.zeros(B, H, dtype=torch.float64), torch.zeros(B, H, dtype=torch.float64))
                   for blk in range(self.cfg["sep_num_blocks"]) for k in range(self.cfg["sep_num_layers"])}

    def _decode(self, window, F_first, g0, nout):
        """output samples [g0, g0 + nout) of the transposed conv over the frames `window` (B Ns, Nb, k) starting at frame F_first;
        samples before 0 are the delay's zeros"""
        y = torch.zeros(window.shape[0], nout, dtype=torch.float64)
        if window.shape[2] == 0:  # no frame yet, or the empty flush of a zero-delay model
            return y.view(self.B, self.Ns, nout)
        full = F.conv_transpose1d(window, self.sd["decoder.conv_transpose1d.weight"].double(), stride=self.S)
        for p in range(nout):
            g = g0 + p
            if g >= 0:
                y[:, p] = full[:, 0, g - F_first * self.S]
        return y.view(self.B, self.Ns, nout)

    def push(self, x):
        """x (B, 1, n) -> (B, Ns, n)"""
        sd, cfg, L, S, D = self.sd, self.cfg, self.L, self.S, self.D
        x = x.double()
        n = x.shape[-1]
        assert n > 0 and n % S == 0
        T0, T1 = self.T0, self.T0 + n
        F0, F1 = frames_done(T0, L, S), frames_done(T1, L, S)
        nv = F1 - F0
        xcat = torch.cat([self.carry, x], dim=2)  # samples [T0 - D, T1)
        base = F0 * S - (T0 - D)
        steps = nv
        if self.defect == "count_incomplete" and T0 == 0:  # the first push runs every column, windows zero-padded past T1
            steps = n // S
            xcat = F.pad(xcat, (0, L))
        seg = xcat[..., base:base + (steps - 1) * S + L] if steps else xcat[..., :0]
        w = F.conv1d(seg, sd["encoder.conv1d.weight"].double(), stride=S) if steps else torch.zeros(self.B, self.Nb, 0, dtype=torch.float64)
        if cfg.get("enc_nonlinear") == "relu":
            w = w.relu()
        mean = w.mean(dim=1, keepdim=True)
        var = ((w - mean) ** 2).mean(dim=1, keepdim=True)
        z = sd["separator.gamma"].double() * (w - mean) / (torch.sqrt(var) + cfg.get("eps", R.EPS)) + sd["separator.beta"].double()
        z = z.permute(0, 2, 1)
        skip = 0
        for blk in range(cfg["sep_num_blocks"]):
            for k in range(cfg["sep_num_layers"]):
                h, c = self.hc[(blk, k)]
                if self.defect == "reset_state":
                    h, c = torch.zeros_like(h), torch.zeros_like(c)
                if self.defect == "no_c":
                    c = torch.zeros_like(c)
                z, h, c = _lstm_steps(z, sd, "separator.rnn.{}.".format(blk), k, h, c)
                self.hc[(blk, k)] = (h, c)
            skip = z + skip
        skip, w = skip[:, :nv], w[..., :nv]
        y = skip @ sd["separator.fc.weight"].double().t() + sd["separator.fc.bias"].double()
        y = y.view(self.B, nv, self.Ns, self.Nb).permute(0, 2, 3, 1)
        mask = torch.sigmoid(y) if cfg["mask_nonlinear"] == "sigmoid" else torch.softmax(y, dim=1)
        what = (w.unsqueeze(1) * mask).reshape(self.B * self.Ns, self.Nb, nv)
        if self.defect == "no_hist":
            self.hist = torch.zeros_like(self.hist)
        window = torch.cat([self.hist, what], dim=2)  # frames [F0 - (L/S - 1), F1)
        out = self._decode(window, F0 - (self.Rf - 1), T0 - D, n)
        self.hist = window[..., window.shape[2] - (self.Rf - 1):]
        self.carry = xcat[..., n:n + D]
        self.T0 = T1
        return out

    def flush(self):
        """-> (B, Ns, D): the last D samples"""
        if self.T0 < self.L:
            raise ValueError("fewer than kernel_size samples pushed")
        F1 = frames_done(self.T0, self.L, self.S)
        return self._decode(self.hist, F1 - (self.Rf - 1), self.T0 - self.D, self.D)


def stream_fwd(x, sd, cfg, pushes, defect=None):
    """x (B, 1, T) pushed in chunks of `pushes` samples (sum = T) -> (B, Ns, T) = cat(Y[..., D:], Z), the offline output"""
    st = Stream(sd, cfg, x.shape[0], defect)
    ys, pos = [], 0
    for n in pushes:
        ys.append(st.push(x[..., pos:pos + n]))
        pos += n
    assert pos == x.shape[-1]
    Y = torch.cat(ys, dim=2)
    assert torch.all(Y[..., :st.D] == 0)
    if defect == "delay":  # the output one stride later than D
        Y = torch.cat([torch.zeros_like(Y[..., :st.S]), Y], dim=2)[..., :Y.shape[-1]]
    return torch.cat([Y[..., st.D:], st.flush()], dim=2)


def stream_bound(off):
    """the stream-vs-offline bound per element: 1e-6 |offline| + 1e-7 max|offline|"""
    return REL * off.abs() + ABS_OF_MAX * float(off.abs().max())
