"""Online inference (csrc/ctn_online.cu) at every filter-bank geometry and push size (``-m gpu``).

test_online_gpu.py varies the separator and the push pattern at one filter bank, kernel_size L = 16 / stride S = 8.  The
filter-bank carries depend on L and S alone, so each row here picks (L, S) and a push pattern for the branch of the carry
code its `reaches` names:
  - k_online_enc keeps the last D = L - S input samples.  A push of n < D samples takes part of the new carry from the old one.
  - k_online_dec keeps w_hat of the last R - 1 frames, R = L / S.  With R > 2 a push of fewer than R - 1 frames keeps part of
    the old history.  The decoder sums in k_decoder<S, 2>'s order (split into channel quarters) for L = 2S with
    S in {1, 2, 8, 10}, and in k_decoder_generic's order otherwise, as ctn_decoder_fwd chooses for the offline model.
  - L == S: D = 0, no carry, no history, and flush() returns (B, S, 0).
  - pushes above 12 k samples ask the encoder for more than 48 KB of dynamic shared memory; the state query caps it at 200 KiB.
Only kernel sizes that the offline encoder has (ctn_encoder_fwd: L in {2, 4, 8, 16, 20, 32, 40, 64}) are used, so every row
has an offline model to compare with.

Checks and bounds are those of test_online_gpu.py: Y[..., :D] == 0; cat(Y[..., D:], Z) against the offline GPU model of the
same mode at 1e-6 |offline| + 1e-7 max|offline|, and against the fp64 oracle at rtol 1e-4 / atol 2e-5 (2e-2 / 5e-3 in 'tf32').
No geometry reorders a sum against the offline kernels: k_online_enc sums k ascending with fmaf from 0 as k_encoder and
k_encoder_v4 do, and k_online_dec's two branches follow k_decoder<S, 2> and k_decoder_generic term by term.  So the offline
bound is not widened here.  Chunk-size invariance uses the same bound; reset and graph replay are bit for bit.

Every row also prints the share of output samples where the stream equals the offline model exactly, and
test_bit_identity_report prints it for the rows of test_online_gpu.py.  Neither asserts it: the cLN prefix sums are added in
another order, so equality is measured, not promised.  On an H100 80GB HBM3 (700 W) the share was 1 in every row and mode.
"""
import collections

import pytest
import torch

import convtasnet_oracle as O
from test_online_gpu import MODES, OUT_ATOL, OUT_RTOL, TF32_ATOL, TF32_RTOL, _build, _cfg, _online_share, _stream
from test_online_gpu import ROWS as BASE_ROWS
from test_online_gpu import _case as _base_case

pytestmark = pytest.mark.gpu

Row = collections.namedtuple("Row", "shape batch pushes reaches")

ROWS = {
    "L16S4-1f": Row(dict(kernel_size=16, stride=4), 2, [1] * 60,
                    "R=4, D=12, 1-frame pushes of 4 samples: generic decoder with 3 history frames; the encoder carry is 2/3 "
                    "old (n < D); the first 3 pushes complete no frame"),
    "L16S4-mixed": Row(dict(kernel_size=16, stride=4), 2, [1, 2, 3, 64, 129, 1, 2, 1, 1, 3, 30, 2],
                       "R=4: the history shifts by 1, 2 and >= R-1 frames in one stream"),
    "L32S8": Row(dict(n_basis=48, kernel_size=32, stride=8), 2, [1, 7] * 15,
                 "R=4, S=8: the generic decoder, not the split one S=8 takes at R=2; k_encoder<32>"),
    "L8S2-ring": Row(dict(n_basis=32, kernel_size=8, stride=2, sep_num_layers=10), 2, [37] * 60,
                     "R=4, P=3, X=10: rings of up to 1024 frames wrap many times at stride 2"),
    "L2S1": Row(dict(n_basis=24, kernel_size=2, stride=1), 2, [1] * 40 + [128, 129, 1, 1, 64],
                "split decoder S=1, D=1, 1-sample pushes; k_encoder_v4<2,1>"),
    "L4S2": Row(dict(kernel_size=4, stride=2), 2, [1] * 30 + [5, 128, 2, 129, 1, 3],
                "split decoder S=2, D=2: 1-frame pushes, then mixed"),
    "L20S10": Row(dict(kernel_size=20, stride=10), 2, [1, 2, 5, 128, 129, 1, 3, 64],
                  "split decoder S=10; offline k_encoder_v4<20,10>"),
    "L40S20": Row(dict(n_basis=24, kernel_size=40, stride=20), 2, [1, 2, 5, 128, 129, 1, 3, 64],
                  "R=2 but the generic decoder (S=20); offline k_encoder<40>"),
    "L64S2": Row(dict(n_basis=32, kernel_size=64, stride=2), 2, [1] * 80 + [5, 33],
                 "R=32, D=62: 31 history frames; pushes of 2 samples, far shorter than the carry"),
    "L16S16": Row(dict(kernel_size=16, stride=16), 2, [1] * 20 + [3, 128, 129, 2, 1],
                  "L == S, D=0: no carry, no history, the generic decoder over one frame; flush returns (B, S, 0)"),
    "L8S8-softmax-3src": Row(dict(kernel_size=8, stride=8, mask_nonlinear="softmax", n_sources=3, enc_nonlinear="relu"), 2,
                             [1, 4, 128, 129, 2, 1, 60], "D=0 with the softmax mask, 3 sources, encoder ReLU"),
    "big-push": Row(dict(kernel_size=16, stride=8), 2, [1600, 6399],
                    "L=16, S=8, pushes of 1600 and 6399 frames (max_chunk 6399 frames, pitch 6400): the encoder's dynamic "
                    "shared memory at 51 232 bytes, above 48 KB, then at exactly the 200 KiB limit"),
}

_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def _case(name):
    def fn():
        e = ROWS[name]
        cfg = _cfg(causal=True, **e.shape)
        sd = O.synth_state_dict(cfg, seed=711)
        x, _ = O.synth_batch(e.batch, cfg.n_sources, sum(e.pushes) * cfg.stride, seed=712)
        return cfg, sd, x
    return _cached(("case", name), fn)


def _bits(s, off):
    """share of output samples where the stream equals the offline model exactly"""
    return float((s == off).double().mean())


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(ROWS))
def test_stream_matches_offline(name, mode):
    """the delay, the push and flush shapes, Y[..., :D] == 0, and the stream against the offline model and the fp64 oracle"""
    e = ROWS[name]
    cfg, sd, x = _case(name)
    L, S = cfg.kernel_size, cfg.stride
    D = L - S
    model = _build(cfg, sd, mode)
    with torch.no_grad():
        off = model(x.cuda()).cpu()
    ys, z, sep = _stream(model, x, e.pushes, S)
    assert sep.delay == D
    for f, y in zip(e.pushes, ys):
        assert y.shape == (e.batch, cfg.n_sources, f * S)
    assert z.shape == (e.batch, cfg.n_sources, D)
    Y = torch.cat(ys, dim=2).cpu()
    assert torch.equal(Y[..., :D], torch.zeros_like(Y[..., :D])), "the first D samples are not exactly zero"
    s = torch.cat([Y[..., D:], z.cpu()], dim=2)
    assert s.shape == off.shape
    assert torch.isfinite(s).all()
    share = _online_share(s, off)
    assert share <= 1.0, "{} {}: stream vs offline at {:.3f} of the bound".format(name, mode, share)
    msg = "[online {} {}] vs offline {:.3g} of bound, bit-identical share {:.6f}".format(name, mode, share, _bits(s, off))

    def fn():
        return O.conv_tasnet_fwd(x.double(), {k: v.double() for k, v in sd.items()}, cfg)[0]
    ref = _cached(("fp64", name), fn)
    rtol, atol = (TF32_RTOL, TF32_ATOL) if mode == "tf32" else (OUT_RTOL, OUT_ATOL)
    torch.testing.assert_close(s.double(), ref, rtol=rtol, atol=atol, msg=lambda m: "{} {}: {}".format(name, mode, m))
    msg += "; vs fp64 {:.3g} of bound".format(float(((s.double() - ref).abs() / (atol + rtol * ref.abs())).max()))
    print(msg + " -- " + e.reaches)


INVARIANCE = {"L16S4-1f": [7, 1, 2, 3, 47], "L64S2": [2, 31, 1, 84], "L16S16": [1, 100, 182], "L2S1": [3, 300, 60]}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(INVARIANCE))
def test_chunk_size_invariance(name, mode):
    """the same input pushed in another pattern gives the same stream within the offline bound"""
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
@pytest.mark.parametrize("name", ["L16S4-mixed", "L16S16"])
def test_reset_is_a_fresh_start(name, mode):
    """after a flush and reset(), replaying the stream gives the same bits"""
    e = ROWS[name]
    cfg, sd, x = _case(name)
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
    """L = 16, S = 4: a captured one-frame push replayed 20 times equals eager pushes bit for bit.  Every replay shifts the
    3-frame decoder history and takes 8 of the 12 carried samples from the old carry."""
    cfg, sd, x = _case("L16S4-1f")
    model = _build(cfg, sd, mode)
    n, warm, reps = cfg.stride, 8, 20  # after 8 pushes (32 samples) the history holds 3 complete frames
    assert (warm + reps) * n <= x.size(-1)
    xd = x.cuda()
    eager = model.online(batch_size=x.size(0), max_chunk=n)
    ref = [eager.push(xd[..., i * n:(i + 1) * n]) for i in range(warm + reps)]
    sep = model.online(batch_size=x.size(0), max_chunk=n)
    for i in range(warm):
        assert torch.equal(sep.push(xd[..., i * n:(i + 1) * n]), ref[i])
    static_x = xd[..., warm * n:(warm + 1) * n].clone()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="relaxed"):
        static_y = sep.push(static_x)
    for i in range(warm, warm + reps):
        static_x.copy_(xd[..., i * n:(i + 1) * n])
        g.replay()
        assert torch.equal(static_y, ref[i]), "replay {} differs from the eager push".format(i)


@pytest.mark.parametrize("name", ["L16S4-mixed", "L8S8-softmax-3src"])
def test_launch_count_is_fixed(name):
    """every push launches 6 + 4 R X kernels (+1 softmax), R X the residual blocks, whatever the filter bank or n"""
    e = ROWS[name]
    cfg, sd, x = _case(name)
    model = _build(cfg, sd, "tf32x3")
    sep = model.online(batch_size=x.size(0), max_chunk=max(e.pushes) * cfg.stride)
    want = 6 + 4 * cfg.sep_num_blocks * cfg.sep_num_layers + (1 if cfg.mask_nonlinear == "softmax" else 0)
    xd, t = x.cuda(), 0
    for f in e.pushes:
        sep.push(xd[..., t:t + f * cfg.stride])
        t += f * cfg.stride
        assert sep.last_launches == want, (name, f, sep.last_launches, want)
    print("[online launches {}] {} per push".format(name, want))


def test_zero_delay_flush_checks_the_sample_count():
    """L == S: flush() before L samples is still a ValueError; after one frame it returns (B, S, 0)"""
    cfg, sd, x = _case("L16S16")
    model = _build(cfg, sd, "fp32")
    sep = model.online(batch_size=x.size(0), max_chunk=cfg.stride)
    with pytest.raises(ValueError):
        sep.flush()
    sep.reset()
    y = sep.push(x[..., :cfg.stride].cuda())
    assert y.shape == (x.size(0), cfg.n_sources, cfg.stride)
    z = sep.flush()
    assert z.shape == (x.size(0), cfg.n_sources, 0)


@pytest.mark.parametrize("mode", MODES)
def test_bit_identity_report(mode):
    """prints the share of bit-identical output samples for the rows of test_online_gpu.py (this file's rows print theirs in
    test_stream_matches_offline); asserts nothing beyond what those tests assert"""
    for name, e in BASE_ROWS.items():
        cfg, sd, x = _base_case(name)
        model = _build(cfg, sd, mode)
        with torch.no_grad():
            off = model(x.cuda()).cpu()
        ys, z, _ = _stream(model, x, e.pushes, cfg.stride)
        D = cfg.kernel_size - cfg.stride
        s = torch.cat([torch.cat(ys, 2)[..., D:], z], 2).cpu()
        print("[online-bits {} {}] bit-identical share {:.6f}, vs offline {:.3g} of bound".format(
            name, mode, _bits(s, off), _online_share(s, off)))
