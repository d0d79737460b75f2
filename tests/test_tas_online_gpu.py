"""Online LSTM-TasNet (TasNet.online, ctn_tas_online_*) on the GPU: every row streams a causal plain-encoder model chunk by chunk and
compares cat(Y[..., D:], flush()) with the offline GPU model in the same numeric mode, |stream - offline| <= 1e-6 |offline| + 1e-7
max|offline| per sample, and with the fp64 restatement (tests/lstm_tasnet_ref.py) under the offline path's bound.  The report prints
the bit-identical share of each row.  Bit for bit: two push patterns of one input, each stream against the others of its batch, a
reset stream against its first run, a CUDA-graph-captured push against eager pushes.  Also: the launches per push, a weight changed
after online(), flush before a frame and push after flush."""
import collections

import pytest
import torch

import lstm_tasnet_ref as R
import tas_online_ref as O
from ctn_b200 import _native as N
from ctn_b200.models.tasnet import TasNet

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
MODES = ("fp32", "tf32x3", "tf32", "f16x3")
Row = collections.namedtuple("Row", "n_basis L S H X R n_sources mask relu B T pushes mode lead_zeros")


def row(n_basis=32, L=16, S=8, H=32, X=2, R_=2, n_sources=2, mask="sigmoid", relu=False, B=1, T=800, pushes=(5,), mode="f16x3",
        lead_zeros=0):
    return Row(n_basis, L, S, H, X, R_, n_sources, mask, relu, B, T, pushes, mode, lead_zeros)


MIX = (1, 5, 128, 300, 2, 129)
ROWS = {
    "40/20": row(L=40, S=20, T=4000, pushes=(16,)),
    "16/8-mix": row(B=3, T=8 * 700, pushes=MIX, mode="fp32"),
    "8/4-one-frame": row(L=8, S=4, T=400, pushes=(1,)),
    "32/8-three-history": row(L=32, S=8, B=2, T=1200, pushes=(3, 7)),
    "L=S-zero-delay": row(L=8, S=8, T=640, pushes=(2, 1)),
    "129-frames": row(T=8 * 129 * 3, pushes=(129,), B=2),
    "X1R1": row(X=1, R_=1, T=8 * 500, pushes=MIX),
    "X3R2-skip": row(X=3, R_=2, B=2, T=1600, pushes=(4, 1)),
    "3src-softmax-relu": row(n_sources=3, mask="softmax", relu=True, B=3, T=1200, pushes=(6, 1, 13)),
    "B=group+1": row(H=64, B=-1, T=800, pushes=(5,)),
    "H=max": row(H=-1, X=1, R_=1, n_basis=16, T=8 * 48, pushes=(7,)),
    "1000-leading-zeros": row(T=1000 + 1200, pushes=(9,), lead_zeros=1000, B=2),
    "10s-320": row(L=40, S=20, T=80000, pushes=(16,)),
    "recipe-4s": row(n_basis=500, L=40, S=20, H=500, T=32000, pushes=(16,)),
}
for _m in MODES:
    ROWS["16/8-mix-" + _m] = ROWS["16/8-mix"]._replace(mode=_m, B=2)


def resolve(r):
    if r.H == -1:
        r = r._replace(H=N.ctn_tas_lstm_max_hidden(1))
    if r.B == -1:
        r = r._replace(B=N.ctn_tas_lstm_group(r.H, 1) + 1)
    return r


def build(r, seed=11):
    m = TasNet(r.n_basis, kernel_size=r.L, stride=r.S, enc_basis="trainable", dec_basis="trainable", enc_nonlinear="relu" if r.relu else None,
               sep_num_blocks=r.X, sep_num_layers=r.R, sep_hidden_channels=r.H, mask_nonlinear=r.mask, causal=True, rnn_type="lstm",
               n_sources=r.n_sources)
    sd = R.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed)
    m.load_state_dict(sd)
    m.math = r.mode
    cfg = dict(n_basis=r.n_basis, kernel_size=r.L, stride=r.S, enc_basis="trainable", enc_nonlinear="relu" if r.relu else None,
               sep_num_blocks=r.X, sep_num_layers=r.R, causal=True, mask_nonlinear=r.mask, n_sources=r.n_sources, eps=1e-12)
    return m.to(DEV).eval(), sd, cfg


def signal(r, seed=5):
    x = torch.randn(r.B, 1, r.T, generator=torch.Generator().manual_seed(seed))
    x[..., :r.lead_zeros] = 0
    return x


def sizes(T, S, pattern):
    out, i = [], 0
    while sum(out) < T:
        out.append(min(pattern[i % len(pattern)] * S, T - sum(out)))
        i += 1
    return out


def stream(m, x, ns, max_chunk=None):
    sep = m.online(batch_size=x.shape[0], max_chunk=max_chunk or max(ns))
    xd, ys, pos, launches = x.to(DEV), [], 0, set()
    for n in ns:
        ys.append(sep.push(xd[..., pos:pos + n]))
        launches.add(sep.last_launches)
        pos += n
    return sep, torch.cat(ys, 2), sep.flush(), launches


def whole(sep, Y, Z):
    D = sep.delay
    assert torch.all(Y[..., :D] == 0)
    return torch.cat([Y[..., D:], Z], 2)


@pytest.mark.parametrize("name", list(ROWS))
def test_stream_matches_offline_and_fp64(name):
    r = resolve(ROWS[name])
    m, sd, cfg = build(r)
    x = signal(r)
    sep, Y, Z, launches = stream(m, x, sizes(r.T, r.S, r.pushes))
    got = whole(sep, Y, Z)
    with torch.no_grad():
        off = m(x.to(DEV))
    torch.cuda.synchronize()
    excess = float(((got - off).abs() - O.stream_bound(off)).max())
    share = float((got == off).double().mean())
    print("[tas online] {:>22s} {:6s} B={} H={} T={} bit-identical {:.4%} worst excess {:.3g}".format(name, r.mode, r.B, r.H, r.T, share,
                                                                                                        excess))
    assert excess <= 0, (name, excess)
    assert launches == {4 + 2 * r.X * r.R + (r.mask == "softmax")}, launches
    ref = R.tasnet_fwd(x, sd, cfg)
    err = float((got.double().cpu() - ref).abs().max())
    assert err <= R.bound(ref), (name, err, R.bound(ref))


def test_two_push_patterns_give_the_same_bits():
    r = ROWS["16/8-mix"]._replace(mode="f16x3")
    m, _, _ = build(r)
    x = signal(r)
    a = whole(*stream(m, x, sizes(r.T, r.S, MIX))[:3])
    b = whole(*stream(m, x, sizes(r.T, r.S, (3, 64, 1)), max_chunk=300 * r.S)[:3])
    assert torch.equal(a, b)


def test_streams_are_independent():
    """changing one stream's input changes no bit of the others"""
    r = ROWS["3src-softmax-relu"]
    m, _, _ = build(r)
    x = signal(r)
    x2 = x.clone()
    x2[1] = torch.randn(1, r.T, generator=torch.Generator().manual_seed(99))
    ns = sizes(r.T, r.S, r.pushes)
    a = whole(*stream(m, x, ns)[:3])
    b = whole(*stream(m, x2, ns)[:3])
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]) and not torch.equal(a[1], b[1])


def test_reset_reproduces_the_first_run():
    r = ROWS["X3R2-skip"]
    m, _, _ = build(r)
    x = signal(r)
    ns = sizes(r.T, r.S, r.pushes)
    sep, Y, Z, _ = stream(m, x, ns)
    first = torch.cat([Y, Z], 2)
    sep.reset()
    xd, ys, pos = x.to(DEV), [], 0
    for n in ns:
        ys.append(sep.push(xd[..., pos:pos + n]))
        pos += n
    ys.append(sep.flush())
    assert torch.equal(torch.cat(ys, 2), first)


@pytest.mark.parametrize("mode", ["fp32", "f16x3"])
def test_graph_replay(mode):
    """a push captured in a CUDA graph and replayed equals eager pushes, bit for bit (the first replay completes no frame)"""
    r = ROWS["40/20"]._replace(mode=mode, B=2, T=20 * 16 * 30)
    m, _, _ = build(r)
    x = signal(r).to(DEV)
    n = 16 * r.S
    eager = m.online(batch_size=r.B, max_chunk=n)
    ref = [eager.push(x[..., i * n:(i + 1) * n]) for i in range(30)]
    sep = m.online(batch_size=r.B, max_chunk=n)
    static_x = torch.zeros(r.B, 1, n, device=DEV)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="relaxed"):
        static_y = sep.push(static_x)
    sep.reset()  # capturing ran nothing, but start from a clean state all the same
    for i in range(30):
        static_x.copy_(x[..., i * n:(i + 1) * n])
        g.replay()
        assert torch.equal(static_y, ref[i]), "replay {} differs from the eager push".format(i)


def test_early_pushes_complete_no_frame():
    """L = 2S: a first push of one stride completes nothing and returns zeros; flush needs kernel_size samples"""
    r = ROWS["16/8-mix"]._replace(mode="fp32")
    m, _, _ = build(r)
    x = signal(r).to(DEV)
    sep = m.online(batch_size=r.B, max_chunk=r.S)
    assert torch.all(sep.push(x[..., :r.S]) == 0)
    with pytest.raises(ValueError):
        sep.flush()
    sep.reset()
    sep.push(x[..., :r.S])
    sep.push(x[..., r.S:2 * r.S])
    sep.flush()
    with pytest.raises(RuntimeError):
        sep.push(x[..., :r.S])


def test_weight_change_is_loud():
    r = ROWS["X1R1"]
    m, _, _ = build(r)
    sep = m.online(batch_size=r.B, max_chunk=10 * r.S)
    sep.push(torch.zeros(r.B, 1, 4 * r.S, device=DEV))
    with torch.no_grad():
        m.separator.rnn[0].weight_hh_l0.mul_(1.0)  # in place: bumps the version, not the value
    with pytest.raises(RuntimeError):
        sep.push(torch.zeros(r.B, 1, 4 * r.S, device=DEV))


def test_state_bytes_is_exposed():
    r = ROWS["recipe-4s"]
    m, _, _ = build(r)
    sep = m.online(batch_size=1, max_chunk=320)
    assert sep.state_bytes > 16000 and sep.delay == 20
