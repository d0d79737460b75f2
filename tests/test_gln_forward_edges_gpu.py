"""Edge shapes of the non-causal (gLN), sigmoid-mask inference forward (``-m gpu``) against the oracle in float64: the path
bench.py measures, through every branch of run_tcn's block dispatch and run_separator's mask + decoder dispatch.

Rows, predicates, launch counts and references are in gln_forward_edges_ref.py; test_gln_forward_edges_cpu.py shows there that
each row reaches the branch its `reaches` text names and that the bound below rejects six plausible defects.
  * whole model: ctn_convtasnet_fwd without a latent (forward: k_maskdec where eligible) and with one (extract_latent: never
    k_maskdec), and model(x) / extract_latent giving the same bits as those calls;
  * ctn_separator_fwd at the sc129 and paper-short widths, ctn_tcn_fwd with inputs at |x| ~ 1e3 and 1e-3, ctn_tcn_blocks_fwd with
    explicit dilations (fused and stand-alone depthwise blocks alternating, with x_out, at 64 blocks), and its refusal of x_out
    when the last block has no output head.
Every call writes into NaN-filled outputs and a NaN-filled workspace, is repeated and must give the same bits, and must launch the
number of kernels the predicates derive for its branches.  The fp64 references are computed once per session (_CACHE).

Bound: rtol 1e-4 / atol 2e-5 of fp64 ('fp32', 'tf32x3', 'f16x3'), rtol 2e-2 / atol 5e-3 ('tf32').  In the silence row the model
is homogeneous in the input's amplitude, so each sample's atol is scaled by its peak output over the ordinary sample's; the
exact-zero sample's estimate and latent must be exactly 0.
"""
import ctypes as C
import time

import pytest
import torch

import convtasnet_oracle as O
import gln_forward_edges_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.tdcn import ResidualBlock1d, TimeDilatedConvNet, block_param_array
from test_forward_edges_gpu import _build

pytestmark = pytest.mark.gpu

MODES = ["fp32"] + (["tf32x3", "f16x3", "tf32"] if N.ctn_has_tcgen05() else [])
DEV = torch.device("cuda", 0)
_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        t0 = time.time()
        _CACHE[key] = fn()
        print("[fp64 reference {}] {:.1f} s".format(key, time.time() - t0))
    return _CACHE[key]


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _nan_ws(nbytes):
    """a workspace of all-ones bytes (NaN as float and as double) -> (buffer, base, nbytes); the caller holds the buffer until the
    call is enqueued, or the outputs allocated after it could take its memory"""
    buf = torch.full((int(nbytes) + 512,), 255, dtype=torch.uint8, device=DEV)
    return (buf,) + N.aligned(buf)


def _check(y, ref, rtol, atol, what, scale=None):
    """every cell within atol * scale + rtol |ref| of fp64 (scale per sample, broadcast over the rest); the worst share"""
    y, ref = y.cpu().double(), ref.double()
    assert y.shape == ref.shape, (what, tuple(y.shape), tuple(ref.shape))
    a = atol if scale is None else atol * scale.view(-1, *([1] * (ref.dim() - 1)))
    s = (y - ref).abs() / (a + rtol * ref.abs())
    worst = float(s.max())
    assert worst <= 1.0, "{}: {:.2f}x the bound at {} (|y - y64| = {:.3e})".format(
        what, worst, tuple(int(i) for i in torch.nonzero(s == s.max())[0]), float((y - ref).abs().max()))
    return worst


def _twice(fn):
    """fn() twice into fresh NaN buffers: the same bits and the same launch count both times -> (outputs, launches)"""
    a, n1 = fn()
    b, n2 = fn()
    for i, (u, v) in enumerate(zip(a, b)):
        if u is not None:
            assert torch.equal(u, v), "output {}: a second call gives other bits".format(i)
    assert n1 == n2, (n1, n2)
    return a, n1


# ---- whole model -----------------------------------------------------------------------------------------------------------
def _model_call(model, x, latent):
    """ctn_convtasnet_fwd as ConvTasNet._run calls it, into NaN-filled outputs and workspace -> ((out, latent), launches)"""
    cfg = model.native_config()
    params, keep = model.native_params(DEV)
    B, _, T = x.shape
    frames = N.frames_of(T, model.kernel_size, model.stride)[0]
    need = C.c_size_t(0)
    N.check(N.ctn_workspace_bytes(C.byref(cfg), B, T, C.byref(need)), "ctn_workspace_bytes")
    ws, base, nbytes = _nan_ws(need.value)
    out = _nan(B, model.n_sources, T)
    lat = _nan(B, model.n_sources, model.n_basis, frames) if latent else None
    N.check(N.ctn_convtasnet_fwd(C.byref(cfg), C.byref(params), x.data_ptr(), B, T, out.data_ptr(), N.ptr(lat), base, nbytes,
                                 N.stream_ptr(DEV)), "ctn_convtasnet_fwd")
    launches = N.ctn_last_launch_count()
    del ws
    return (out, lat), launches


def _scales(name, out64):
    """per-sample atol scale: 1, or in the silence row the sample's peak output over the ordinary sample's (the zero sample: 1,
    it is held to exact zero)"""
    if name != "silence":
        return None
    peak = out64.abs().flatten(1).max(1).values
    s = peak / peak[0]
    s[1] = 1.0
    return s


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(R.ROWS))
def test_model_vs_fp64(name, mode):
    r = R.ROWS[name]
    sd = R.state_dict(r)
    model = _build(r.cfg, sd, mode)
    rtol, atol = R.tol(mode)
    worst = 0.0
    for T in r.Ts:
        x = R.mixture(r, T, sd)
        out64, lat64 = _cached(("model", name, T), lambda: O.conv_tasnet_fwd(x.double(), {k: v.double() for k, v in sd.items()},
                                                                             r.cfg))
        xd = x.cuda()
        scale = _scales(name, out64)
        for latent in (False, True):
            (y, lat), n = _twice(lambda: _model_call(model, xd, latent))
            what = "{} T={} {} {}".format(name, T, mode, "extract_latent" if latent else "forward")
            want = R.model_launches(r.cfg, r.B, mode, latent)
            assert n == want, "{}: {} launches, the branches give {} (k_maskdec: {})".format(what, n, want,
                                                                                         R.maskdec(r.cfg, mode, latent))
            with torch.no_grad():
                api = model.extract_latent(xd) if latent else (model(xd), None)
            assert torch.equal(api[0], y) and (lat is None or torch.equal(api[1], lat)), what + ": the module gives other bits"
            if name == "silence":
                assert torch.equal(y[1].cpu(), torch.zeros_like(y[1].cpu())), what + ": the zero sample's estimate is not 0"
                if latent:
                    assert torch.equal(lat[1].cpu(), torch.zeros_like(lat[1].cpu())), what + ": the zero sample's latent is not 0"
            worst = max(worst, _check(y, out64, rtol, atol, what + " output", scale))
            if latent:
                lscale = None if scale is None else lat64.abs().flatten(1).max(1).values / lat64[0].abs().max()
                if lscale is not None:
                    lscale[1] = 1.0
                worst = max(worst, _check(lat, lat64, rtol, atol, what + " latent", lscale))
        if name == "b37":
            with torch.no_grad():
                batch = model(xd)
                for b in range(r.B):
                    alone = model(xd[b:b + 1].contiguous())
                    torch.testing.assert_close(alone[0], batch[b], rtol=rtol, atol=atol,
                                               msg=lambda m: "sample {} alone vs its row of the batch: {}".format(b, m))
    print("[gLN model {} {}] {:.3f} of bound -- {}".format(name, mode, worst, r.reaches))


# ---- ctn_separator_fwd -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(R.SEPARATORS))
def test_separator_vs_fp64(name, mode):
    cfg, B, frames, reaches = R.SEPARATORS[name]
    sd = O.synth_state_dict(cfg, seed=731)
    w = 0.3 * torch.randn(B, cfg.n_basis, frames, generator=torch.Generator().manual_seed(732)) + 0.05
    ref = _cached(("sep", name), lambda: O.separator_fwd(w.double(), {k: v.double() for k, v in sd.items()}, cfg))
    sep = _build(cfg, sd, mode).separator
    sep.math = mode
    ncfg = sep.native_config()
    params, keep = sep.native_params(DEV)
    wd = w.cuda()

    def call():
        need = C.c_size_t(0)
        N.check(N.ctn_workspace_bytes(C.byref(ncfg), B, frames, C.byref(need)), "ctn_workspace_bytes")
        ws, base, nbytes = _nan_ws(need.value + 4 * B * cfg.n_sources * cfg.n_basis * N.ctn_pitch(frames) + 1024)
        mask = _nan(B, cfg.n_sources, cfg.n_basis, frames)
        N.check(N.ctn_separator_fwd(C.byref(ncfg), C.byref(params), wd.data_ptr(), B, frames, mask.data_ptr(), base, nbytes,
                                    N.stream_ptr(DEV)), "ctn_separator_fwd")
        n = N.ctn_last_launch_count()
        del ws
        return (mask,), n
    (mask,), n = _twice(call)
    assert n == R.separator_launches(cfg, B, mode), n
    with torch.no_grad():
        assert torch.equal(sep(wd), mask)
    rtol, atol = R.tol(mode)
    worst = _check(mask, ref, rtol, atol, "separator {} {}".format(name, mode))
    print("[gLN separator {} {}] {:.3f} of bound -- {}".format(name, mode, worst, reaches))


# ---- ctn_tcn_fwd -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("amp", list(R.TCN_AMPS))
def test_tcn_amplitude_vs_fp64(amp, mode):
    """TimeDilatedConvNet (ctn_tcn_fwd) on x = amp randn: the f16x3 operand scales start from the measured max |x|
    (ctn_absmax_pitch), so pw1 of block 0 sees an operand scaled by ~1 / amp"""
    cfg, B, F = R.TCN_CFG, 2, R.TCN_FRAMES
    sd = O.synth_state_dict(cfg, seed=741)
    x = (R.TCN_AMPS[amp] * torch.randn(B, cfg.sep_bottleneck_channels, F, generator=torch.Generator().manual_seed(742))).float()
    kw = dict(kernel_size=3, num_blocks=cfg.sep_num_blocks, num_layers=cfg.sep_num_layers, dilated=True, causal=False,
              nonlinear=True, norm=True, eps=R.EPS)
    ref = _cached(("tcn", amp), lambda: O.tdcn_fwd(x.double(), {k: v.double() for k, v in sd.items()}, "separator.tdcn.", **kw))
    net = TimeDilatedConvNet(cfg.sep_bottleneck_channels, hidden_channels=cfg.sep_hidden_channels, skip_channels=cfg.sep_skip_channels,
                             kernel_size=3, num_blocks=cfg.sep_num_blocks, num_layers=cfg.sep_num_layers, dilated=True,
                             separable=True, causal=False, nonlinear="prelu", norm=True)
    net.load_state_dict({k[len("separator.tdcn."):]: v for k, v in sd.items() if k.startswith("separator.tdcn.")}, strict=True)
    net.math = mode
    net = net.cuda()
    ncfg = net.native_config()
    arr, keep = block_param_array(net.residual_blocks(), DEV)
    xd = x.cuda()

    def call():
        need = C.c_size_t(0)
        N.check(N.ctn_tcn_workspace_bytes(C.byref(ncfg), B, F, C.byref(need)), "ctn_tcn_workspace_bytes")
        ws, base, nbytes = _nan_ws(need.value)
        skip = _nan(B, cfg.sep_skip_channels, F)
        N.check(N.ctn_tcn_fwd(C.byref(ncfg), arr, xd.data_ptr(), skip.data_ptr(), B, F, base, nbytes, N.stream_ptr(DEV)), "ctn_tcn_fwd")
        n = N.ctn_last_launch_count()
        del ws
        return (skip,), n
    (skip,), n = _twice(call)
    assert n == R.tcn_fwd_launches(cfg.sep_bottleneck_channels, cfg.sep_hidden_channels, cfg.sep_skip_channels, 3,
                                   R.default_dils(cfg), mode, B), n
    with torch.no_grad():
        assert torch.equal(net(xd), skip)
    rtol, _ = R.tol(mode)
    worst = _check(skip, ref, rtol, _tcn_atol(mode, ref), "tcn {} {}".format(amp, mode))
    print("[gLN tcn {} {}] {:.3f} of bound".format(amp, mode, worst))


def _tcn_atol(mode, ref):
    """the model bound's atol; in 'tf32' relative to max |ref| when that is above 1: a skip sum of up to 64 blocks' one-pass tf32
    contractions (10-bit mantissa) carries an absolute error that grows with its terms, while cancellation can leave an entry
    near 0 (the softmax mask rows of test_forward_edges_gpu.py take atol x max|mask| the same way)"""
    _, atol = R.tol(mode)
    return atol * max(1.0, float(ref.abs().max())) if mode == "tf32" else atol


# ---- ctn_tcn_blocks_fwd ----------------------------------------------------------------------------------------------------
def _blocks(b, last_out=None):
    """the row's ResidualBlock1d modules on the GPU (their own dilation field is unused: the call passes b.dils)"""
    last_out = b.last_out if last_out is None else last_out
    n = len(b.dils)
    sd, prefixes = R.blocks_state_dict(n, b.Bc, b.H, b.Sc, b.P, b.last_out, b.seed)
    mods = []
    for i, pf in enumerate(prefixes):
        dual = i < n - 1 or last_out
        m = ResidualBlock1d(b.Bc, hidden_channels=b.H, skip_channels=b.Sc, kernel_size=b.P, stride=1, dilation=1, separable=True,
                            causal=False, nonlinear="prelu", norm=True, dual_head=dual)
        own = {k[len(pf):]: v for k, v in sd.items() if k.startswith(pf) and k[len(pf)].isalpha()}  # net.1. is not net.10.
        m.load_state_dict({k: v for k, v in own.items() if dual or "output_pointwise" not in k}, strict=True)
        mods.append(m.cuda())
    return sd, prefixes, mods


def _blocks_cfg(b, mode):
    cfg = N.Config()
    cfg.bottleneck, cfg.hidden, cfg.skip, cfg.sep_kernel, cfg.causal = b.Bc, b.H, b.Sc, b.P, 0
    cfg.num_blocks, cfg.num_layers = 1, len(b.dils)
    cfg.math = N.MATH_NAMES[mode]
    cfg.eps = cfg.eps_tcn = R.EPS
    return cfg


def _blocks_ws_bytes(cfg, B, frames):
    """ctn_tcn_workspace_bytes takes at most 20 layers per stage; the carve depends on the block count only"""
    n = cfg.num_layers
    q = N.Config.from_buffer_copy(cfg)
    q.num_layers = max(l for l in range(1, 21) if n % l == 0)
    q.num_blocks = n // q.num_layers
    need = C.c_size_t(0)
    N.check(N.ctn_tcn_workspace_bytes(C.byref(q), B, frames, C.byref(need)), "ctn_tcn_workspace_bytes")
    return need.value


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(R.BLOCKS))
def test_blocks_vs_fp64(name, mode):
    b = R.BLOCKS[name]
    sd, prefixes, mods = _blocks(b)
    x = torch.randn(b.B, b.Bc, b.frames, generator=torch.Generator().manual_seed(b.seed + 1))
    x64_out, skip64 = _cached(("blocks", name), lambda: R.chain(x.double(), {k: v.double() for k, v in sd.items()}, prefixes,
                                                                  b.dils, b.P, b.last_out))
    cfg = _blocks_cfg(b, mode)
    arr, keep = block_param_array(mods, DEV)
    dil = (C.c_int * len(b.dils))(*b.dils)
    xd = x.cuda()

    def call():
        ws, base, nbytes = _nan_ws(_blocks_ws_bytes(cfg, b.B, b.frames))
        skip = _nan(b.B, b.Sc, b.frames)
        xo = _nan(b.B, b.Bc, b.frames) if b.x_out else None
        N.check(N.ctn_tcn_blocks_fwd(C.byref(cfg), arr, len(b.dils), dil, xd.data_ptr(), N.ptr(xo), skip.data_ptr(), b.B, b.frames,
                                     base, nbytes, N.stream_ptr(DEV)), "ctn_tcn_blocks_fwd")
        n = N.ctn_last_launch_count()
        del ws
        return (skip, xo), n
    (skip, xo), n = _twice(call)
    assert n == R.tcn_fwd_launches(b.Bc, b.H, b.Sc, b.P, list(b.dils), mode, b.B, b.last_out, b.x_out), n
    rtol, atol = R.tol(mode)
    worst = _check(skip, skip64, rtol, _tcn_atol(mode, skip64), "blocks {} {} skip".format(name, mode))
    if b.x_out:
        worst = max(worst, _check(xo, x64_out, rtol, _tcn_atol(mode, x64_out), "blocks {} {} x_out".format(name, mode)))
    print("[gLN blocks {} {}] {:.3f} of bound -- {}".format(name, mode, worst, b.reaches))


def test_blocks_refuse_x_out_without_the_last_out_head():
    """x_out asked for while the last block has no output head: CTN_EINVAL, and nothing launched"""
    b = R.BLOCKS["mixed"]
    _, _, mods = _blocks(b, last_out=False)
    cfg = _blocks_cfg(b, "f16x3" if N.ctn_has_tcgen05() else "fp32")
    arr, keep = block_param_array(mods, DEV)
    dil = (C.c_int * len(b.dils))(*b.dils)
    ws, base, nbytes = _nan_ws(_blocks_ws_bytes(cfg, b.B, b.frames))
    x = torch.randn(b.B, b.Bc, b.frames, device=DEV)
    skip, xo = _nan(b.B, b.Sc, b.frames), _nan(b.B, b.Bc, b.frames)
    n0 = N.ctn_total_launch_count()
    st = N.ctn_tcn_blocks_fwd(C.byref(cfg), arr, len(b.dils), dil, x.data_ptr(), xo.data_ptr(), skip.data_ptr(), b.B, b.frames, base,
                              nbytes, N.stream_ptr(DEV))
    assert st == N.CTN_EINVAL and N.ctn_total_launch_count() == n0
    assert torch.isnan(skip).all() and torch.isnan(xo).all()
    del ws
