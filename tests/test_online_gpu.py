"""Online inference of the causal Conv-TasNet (``ConvTasNet.online``, csrc/ctn_online.cu) on the GPU (``-m gpu``).

A stream of pushes must reproduce the offline causal forward: with Y the concatenated push outputs, Z = flush() and D the
delay, Y[..., :D] == 0 and cat(Y[..., D:], Z) == model(x).  Every row of ROWS names in `reaches` what its push pattern selects.

Bounds:
  vs the offline GPU model, same mode: |stream - offline| <= 1e-6 |offline| + 1e-7 max|offline| (the causality bound of
    test_forward_edges_gpu.py).  The online path runs the offline contractions column by column and keeps the offline order
    of every other sum, except the cLN prefix sums (double, other order).
  vs the fp64 oracle (O.conv_tasnet_fwd): rtol 1e-4 / atol 2e-5, and rtol 2e-2 / atol 5e-3 in 'tf32' (the forward-edge bounds).
  chunk-size invariance: two push patterns of the same input, the first bound.
  batch independence, reset, graph replay: bit for bit.
"""
import collections

import pytest
import torch

import convtasnet_oracle as O
from ctn_b200 import _native as N
from ctn_b200.models.conv_tasnet import ConvTasNet
from test_parity_gpu import MODES as PARITY_MODES

pytestmark = pytest.mark.gpu

MODES = PARITY_MODES + (["tf32"] if N.ctn_has_tcgen05() else [])
OUT_RTOL, OUT_ATOL = 1e-4, 2e-5
TF32_RTOL, TF32_ATOL = 2e-2, 5e-3
ON_RTOL, ON_ATOL = 1e-6, 1e-7   # atol as a share of max|offline|

_CACHE = {}


def _cfg(**kw):
    base = dict(n_basis=40, kernel_size=16, sep_bottleneck_channels=24, sep_hidden_channels=48, sep_skip_channels=20,
                sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=3, n_sources=2)
    base.update(kw)
    return O.OracleConfig(**base)


def _build(cfg, sd, mode):
    m = ConvTasNet(cfg.n_basis, cfg.kernel_size, stride=cfg.stride, enc_basis="trainable", dec_basis="trainable",
                   enc_nonlinear=cfg.enc_nonlinear, sep_hidden_channels=cfg.sep_hidden_channels,
                   sep_bottleneck_channels=cfg.sep_bottleneck_channels, sep_skip_channels=cfg.sep_skip_channels,
                   sep_kernel_size=cfg.sep_kernel_size, sep_num_blocks=cfg.sep_num_blocks, sep_num_layers=cfg.sep_num_layers,
                   mask_nonlinear=cfg.mask_nonlinear, causal=True, n_sources=cfg.n_sources, eps=cfg.eps)
    m.load_state_dict(sd, strict=True)
    m.math = mode
    return m.cuda().eval()


Row = collections.namedtuple("Row", "shape batch pushes zero_frames fp64 reaches")

PAPER = dict(n_basis=512, sep_bottleneck_channels=128, sep_hidden_channels=512, sep_skip_channels=128, sep_num_blocks=3,
             sep_num_layers=8)

ROWS = {
    "1-frame": Row({}, 2, [1] * 40, 0, True, "1 frame per push: every tap of d >= 1 reads the ring; the first push completes no "
                                              "frame and returns only the delay"),
    "7-frames-X4": Row(dict(sep_num_layers=4), 2, [7] * 30, 0, True, "7 frames per push, X=4 (d up to 8): taps straddle the ring "
                                                                     "and the chunk"),
    "128": Row({}, 2, [128] * 4, 0, True, "128 frames per push: one 128-column tile"),
    "129": Row({}, 2, [129] * 3, 0, True, "129 frames per push: two column tiles"),
    "mixed": Row({}, 2, [1, 5, 128, 300, 2, 129], 0, True, "pushes of 1, 5, 128, 300, 2 and 129 frames in one stream"),
    "P1-R2": Row(dict(n_basis=33, sep_bottleneck_channels=16, sep_hidden_channels=40, sep_skip_channels=13, sep_kernel_size=1,
                      sep_num_blocks=2), 2, [16] * 10, 0, True, "P=1: an empty ring; R=2: the last layer has no output head; "
                                                                  "N=33, Sc=13"),
    "P8-X13": Row(dict(n_basis=24, sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16, sep_kernel_size=8,
                       sep_num_layers=13), 1, [100] * 40, 0, True, "P=8, X=13: the last ring holds 7*4096 frames, more than the "
                                                                   "4000 pushed"),
    "P5-3src-relu": Row(dict(sep_kernel_size=5, sep_num_blocks=2, sep_num_layers=4, n_sources=3, enc_nonlinear="relu"), 2, [50] * 8,
                        0, True, "P=5, 3 sources, encoder ReLU"),
    "softmax": Row(dict(mask_nonlinear="softmax"), 2, [64] * 6, 0, True, "softmax mask over S*N channels"),
    "wide": Row(dict(n_basis=32, sep_bottleneck_channels=1040, sep_hidden_channels=1056, sep_skip_channels=24, sep_num_layers=2),
                2, [5] * 4, 0, True, "Bc=1040, H=1056: more rows than the 1024-CTA grids of the bias and residual kernels"),
    "B37": Row({}, 37, [32] * 8, 0, True, "37 streams"),
    "zeros": Row({}, 2, [256] * 8, 1500, True, "1500 leading frames of exact-zero input: var = 0 frames in every cLN"),
    "long": Row({}, 1, [256] * 782, 0, False, "200 192 frames in 2048-sample pushes: the carry across 782 pushes, many ring wraps"),
    "paper": Row(PAPER, 2, [32] * 125, 0, False, "paper sizes, 4 s at 8 kHz in 256-sample pushes"),
}


def _case(name):
    def fn():
        e = ROWS[name]
        cfg = _cfg(causal=True, **e.shape)
        sd = O.synth_state_dict(cfg, seed=701)
        T = sum(e.pushes) * cfg.stride
        x, _ = O.synth_batch(e.batch, cfg.n_sources, T, seed=702)
        if e.zero_frames:
            x[..., :e.zero_frames * cfg.stride] = 0.0
        return cfg, sd, x
    return _cached(("case", name), fn)


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def _stream(model, x, pushes, stride, B=None):
    """push x (B,1,T) chunk by chunk -> (list of push outputs, flush output)"""
    B = x.size(0) if B is None else B
    sep = model.online(batch_size=B, max_chunk=max(pushes) * stride)
    ys, t = [], 0
    xd = x.cuda()
    for f in pushes:
        ys.append(sep.push(xd[..., t:t + f * stride]))
        t += f * stride
    return ys, sep.flush(), sep


def _online_share(y, off):
    bound = ON_RTOL * off.double().abs() + ON_ATOL * float(off.abs().max())
    return float(((y.double() - off.double()).abs() / bound).max())


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(ROWS))
def test_stream_matches_offline(name, mode):
    """Checks 1-3: the stream against the offline GPU model (same mode) and the fp64 oracle; the delay and the lengths"""
    e = ROWS[name]
    cfg, sd, x = _case(name)
    model = _build(cfg, sd, mode)
    with torch.no_grad():
        off = model(x.cuda()).cpu()
    ys, z, sep = _stream(model, x, e.pushes, cfg.stride)
    D = cfg.kernel_size - cfg.stride
    assert sep.delay == D
    for f, y in zip(e.pushes, ys):
        assert y.shape == (e.batch, cfg.n_sources, f * cfg.stride)
    assert z.shape == (e.batch, cfg.n_sources, D)
    Y = torch.cat(ys, dim=2).cpu()
    assert torch.equal(Y[..., :D], torch.zeros_like(Y[..., :D])), "the first D samples are not exactly zero"
    if e.pushes[0] * cfg.stride <= D:
        assert torch.equal(ys[0].cpu(), torch.zeros_like(ys[0].cpu())), "the first push must return only the delay"
    s = torch.cat([Y[..., D:], z.cpu()], dim=2)
    assert s.shape == off.shape
    assert torch.isfinite(s).all()
    share = _online_share(s, off)
    assert share <= 1.0, "{} {}: stream vs offline at {:.3f} of the bound".format(name, mode, share)
    msg = "[online {} {}] vs offline {:.3g} of bound".format(name, mode, share)
    if e.fp64:
        def fn():
            return O.conv_tasnet_fwd(x.double(), {k: v.double() for k, v in sd.items()}, cfg)[0]
        ref = _cached(("fp64", name), fn)
        rtol, atol = (TF32_RTOL, TF32_ATOL) if mode == "tf32" else (OUT_RTOL, OUT_ATOL)
        torch.testing.assert_close(s.double(), ref, rtol=rtol, atol=atol, msg=lambda m: "{} {}: {}".format(name, mode, m))
        msg += "; vs fp64 {:.3g} of bound".format(float(((s.double() - ref).abs() / (atol + rtol * ref.abs())).max()))
    print(msg + " -- " + e.reaches)


INVARIANCE = {"1-frame": [3, 1, 7, 2, 27], "mixed": [17] * 33 + [4], "P8-X13": [1000, 3, 997, 2000], "B37": [1, 255]}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(INVARIANCE))
def test_chunk_size_invariance(name, mode):
    """Check 4: the same input pushed in another pattern gives the same stream within the offline bound"""
    e = ROWS[name]
    cfg, sd, x = _case(name)
    assert sum(INVARIANCE[name]) == sum(e.pushes)
    model = _build(cfg, sd, mode)
    a, za, _ = _stream(model, x, e.pushes, cfg.stride)
    b, zb, _ = _stream(model, x, INVARIANCE[name], cfg.stride)
    A, Bs = torch.cat(a + [za], 2).cpu(), torch.cat(b + [zb], 2).cpu()
    share = _online_share(Bs, A)
    assert share <= 1.0, "{} {}: {:.3f} of the bound".format(name, mode, share)
    print("[online invariance {} {}] {:.3g} of bound".format(name, mode, share))


@pytest.mark.parametrize("mode", MODES)
def test_batch_independence(mode):
    """Check 5: stream b of B equals stream b run alone, bit for bit"""
    e = ROWS["B37"]
    cfg, sd, x = _case("B37")
    model = _build(cfg, sd, mode)
    ys, z, _ = _stream(model, x, e.pushes, cfg.stride)
    full = torch.cat(ys + [z], 2).cpu()
    for b in (0, 17, 36):
        ys1, z1, _ = _stream(model, x[b:b + 1], e.pushes, cfg.stride)
        assert torch.equal(torch.cat(ys1 + [z1], 2).cpu(), full[b:b + 1]), "stream {} differs when run alone".format(b)


@pytest.mark.parametrize("mode", MODES)
def test_reset_is_a_fresh_start(mode):
    """Check 6: after reset() (and after a flush), the outputs are bit-identical to a fresh separator's"""
    e = ROWS["mixed"]
    cfg, sd, x = _case("mixed")
    model = _build(cfg, sd, mode)
    ys, z, sep = _stream(model, x, e.pushes, cfg.stride)
    with pytest.raises(RuntimeError):
        sep.push(x[..., :cfg.stride].cuda())
    sep.reset()
    xd, t, again = x.cuda(), 0, []
    for f in e.pushes:
        again.append(sep.push(xd[..., t:t + f * cfg.stride]))
        t += f * cfg.stride
    again.append(sep.flush())
    assert torch.equal(torch.cat(again, 2), torch.cat(ys + [z], 2))


@pytest.mark.parametrize("mode", MODES)
def test_graph_replay(mode):
    """Check 7: a steady-state push captured in a CUDA graph and replayed equals eager pushes, bit for bit"""
    cfg, sd, x = _case("7-frames-X4")
    model = _build(cfg, sd, mode)
    S, n, warm = cfg.stride, 7 * cfg.stride, 3
    xd = x.cuda()
    eager = model.online(batch_size=x.size(0), max_chunk=n)
    ref = [eager.push(xd[..., i * n:(i + 1) * n]) for i in range(20)]
    sep = model.online(batch_size=x.size(0), max_chunk=n)
    for i in range(warm):
        assert torch.equal(sep.push(xd[..., i * n:(i + 1) * n]), ref[i])
    static_x = xd[..., warm * n:(warm + 1) * n].clone()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="relaxed"):
        static_y = sep.push(static_x)
    for i in range(warm, 20):
        static_x.copy_(xd[..., i * n:(i + 1) * n])
        g.replay()
        assert torch.equal(static_y, ref[i]), "replay {} differs from the eager push".format(i)
    assert S * 20 * 7 <= x.size(-1)


def test_launch_count_is_fixed():
    """Check 8: every push launches the same kernels whatever its n, before and after L samples: 6 + 4 R X (+1 softmax)"""
    for name in ("mixed", "softmax"):
        cfg, sd, x = _case(name)
        model = _build(cfg, sd, "tf32x3")
        sep = model.online(batch_size=x.size(0), max_chunk=300 * cfg.stride)
        want = 6 + 4 * cfg.sep_num_blocks * cfg.sep_num_layers + (1 if cfg.mask_nonlinear == "softmax" else 0)
        xd, t = x.cuda(), 0
        for f in ([1, 1, 5, 300, 128, 2, 129] if name == "mixed" else ROWS[name].pushes):
            f = min(f, (x.size(-1) - t) // cfg.stride)
            if f <= 0:
                break
            sep.push(xd[..., t:t + f * cfg.stride])
            t += f * cfg.stride
            assert sep.last_launches == want, (name, f, sep.last_launches, want)
        print("[online launches {}] {} per push".format(name, want))


def test_weight_change_is_loud():
    """Check 9: changing a weight after online() makes the next push raise"""
    cfg, sd, x = _case("128")
    model = _build(cfg, sd, "fp32")
    sep = model.online(batch_size=x.size(0), max_chunk=128 * cfg.stride)
    sep.push(x[..., :cfg.stride * 4].cuda())
    with torch.no_grad():
        list(model.separator.tdcn.parameters())[3].mul_(1.0)  # in place: bumps the version, not the value
    with pytest.raises(RuntimeError):
        sep.push(x[..., cfg.stride * 4:cfg.stride * 8].cuda())


def test_flush_needs_a_frame():
    """flush() before L samples were pushed is a ValueError; push after flush raises until reset()"""
    cfg, sd, x = _case("1-frame")
    model = _build(cfg, sd, "fp32")
    sep = model.online(batch_size=x.size(0), max_chunk=cfg.stride)
    sep.push(x[..., :cfg.stride].cuda())
    with pytest.raises(ValueError):
        sep.flush()
    sep.reset()
    with pytest.raises(ValueError):
        sep.push(x[..., :cfg.stride + 1].cuda())
