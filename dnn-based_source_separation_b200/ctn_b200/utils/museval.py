"""BSS Eval v4 of multichannel source images on sm_90a kernels: museval 0.4 ``evaluate(..., mode='v4')`` and ``eval_mus_track``,
which every MUSDB18 tester of the reference calls once per track.  Everything runs in fp64 on the GPU (ctn_bss_eval_images,
DESIGN §10): distortion filters of 512 taps over all sources and channels from the whole track, then SDR / ISR / SIR / SAR per
window.

Differences from museval: the inputs are rounded to float32 on the way in (the kernels widen them exactly; decoded PCM and model
outputs are float32 already); a Gram matrix that is not numerically positive definite raises ValueError where museval falls back to
a least-squares solve; at most 8 reference rows (sources x channels, e.g. 4 stems in stereo) are supported (NotImplementedError
beyond); ``mode='v3'`` (framewise filters) is not implemented."""
import warnings

import numpy as np
import torch

from .. import _native as N
from .bss import _on_device

METRICS = ("SDR", "ISR", "SIR", "SAR")


def bss_eval_images_v4(references, estimates, window=44100, hop=44100):
    """references, estimates (J, I, T) torch, J sources of I channels -> sdr, isr, sir, sar (J, nwin) float64,
    nwin = (T - window + hop) // hop.  Estimate j is scored against reference j.  CPU inputs are computed on the current CUDA
    device and the results come back to the CPU; CUDA inputs leave their results on their device."""
    if references.dim() != 3 or estimates.shape != references.shape:
        raise ValueError("references and estimates must both be (J, I, T), got {} and {}".format(
            tuple(references.shape), tuple(estimates.shape)))
    J, I, T = references.shape
    host = not references.is_cuda
    ref = _on_device(references).to(torch.float32).contiguous()
    est = estimates.to(device=ref.device, dtype=torch.float32).contiguous()
    dev = N.require_cuda(ref, est)
    nbytes = N.C.c_size_t(0)
    N.check(N.ctn_bss_images_workspace_bytes(J, I, T, int(window), int(hop), N.C.byref(nbytes)), "ctn_bss_images_workspace_bytes")
    nwin = (T - int(window) + int(hop)) // int(hop)
    base, avail = N.aligned(N.workspace(dev, nbytes.value + 256, "bss_images"))
    out = tuple(torch.empty((J, nwin), dtype=torch.float64, device=dev) for _ in range(4))
    status = torch.empty(1, dtype=torch.int32, device=dev)
    N.check(N.ctn_bss_eval_images(ref.data_ptr(), est.data_ptr(), J, I, T, int(window), int(hop), *(t.data_ptr() for t in out),
                                  status.data_ptr(), base, avail, N.stream_ptr(dev)), "ctn_bss_eval_images")
    if int(status.item()) & N.BSS_NOT_PD:
        why = ("the Gram matrix of the delayed references (or one of its per-source blocks) is not positive definite (museval "
               "would fall back to lstsq)")
        if J * I * 512 > T + 511:
            why += ": {} samples cannot separate {} x 512 filter taps".format(T, J * I)
        raise ValueError("bss_eval_images_v4: " + why)
    return tuple(t.cpu() for t in out) if host else out


def _as_nsi(x):
    """numpy or torch (nsrc, nsampl, nchan), or (nsrc, nsampl) for mono -> float32 torch (nsrc, nsampl, nchan)"""
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x))
    if t.dim() == 2:
        t = t[..., None]
    if t.dim() != 3:
        raise ValueError("expected (nsrc, nsampl, nchan), got shape {}".format(tuple(t.shape)))
    return t.to(torch.float32)


def pad_or_truncate(references, estimates):
    """museval.pad_or_truncate on (nsrc, nsampl, nchan): estimates cut to the references' length, or zero-padded at the end"""
    T, Te = references.shape[1], estimates.shape[1]
    if Te > T:
        estimates = estimates[:, :T]
    elif Te < T:
        estimates = torch.nn.functional.pad(estimates, (0, 0, 0, T - Te))
    return references, estimates


def evaluate(references, estimates, win=1 * 44100, hop=1 * 44100, mode='v4', padding=True):
    """museval.evaluate: references, estimates (nsrc, nsampl, nchan) numpy or torch -> SDR, ISR, SIR, SAR, numpy (nsrc, nwin)
    float64"""
    if mode != 'v4':
        raise NotImplementedError("mode={!r}: only museval's 'v4' (filters over the whole track) is implemented".format(mode))
    ref, est = _as_nsi(references), _as_nsi(estimates)
    if padding:
        ref, est = pad_or_truncate(ref, est)
    if est.shape != ref.shape:
        raise ValueError("references {} and estimates {} differ in shape".format(tuple(ref.shape), tuple(est.shape)))
    out = bss_eval_images_v4(ref.permute(0, 2, 1), est.permute(0, 2, 1), int(win), int(hop))
    return tuple(t.cpu().numpy() for t in out)


def eval_track(references, estimates, rate, win=1.0, hop=1.0, mode='v4'):
    """museval.eval_mus_track without musdb: references {target: (nsampl, nchan)} in the track's order (``{k: t.audio for k, t in
    track.targets.items()}``), estimates {target: (nsampl, nchan)} -> {target: {"SDR", "ISR", "SIR", "SAR": numpy (nwin,)}}.

    Targets are those of ``references`` that have an estimate.  With both 'vocals' and 'accompaniment' among them, accompaniment
    is left out of the call over the other targets and a second call scores vocals against accompaniment, which gives the
    reported vocals and accompaniment scores."""
    targets = [k for k in references if k in estimates]
    has_acc = all(k in targets for k in ("vocals", "accompaniment"))
    if has_acc:
        targets.remove("accompaniment")
    w, h = int(win * rate), int(hop * rate)
    scores = {}

    def run(names, skip=()):
        res = evaluate([np.asarray(references[k]) for k in names], [np.asarray(estimates[k]) for k in names], w, h, mode)
        for i, k in enumerate(names):
            if k not in skip:
                scores[k] = {m: res[q][i] for q, m in enumerate(METRICS)}

    if len(targets) >= 2:
        run(targets, skip=("vocals",) if has_acc else ())
    elif not has_acc:
        warnings.warn(UserWarning("Incorrect usage of BSSeval : at least two estimates must be provided. Target score will be empty."))
    if has_acc:
        run(["vocals", "accompaniment"])
    return scores


def frames_median(scores):
    """{target: {metric: (nwin,)}} -> {target: {metric: median over the windows, NaN windows skipped}}, as
    ``EvalStore(frames_agg='median')`` reports a track"""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)  # an all-NaN target is NaN, as in museval
        return {k: {m: float(np.nanmedian(v[m])) for m in METRICS} for k, v in scores.items()}
