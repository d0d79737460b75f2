"""BSS Eval on sm_90a kernels, mirroring src/utils/bss.py:4-30, the reference's wrapper of mir_eval 0.7
``mir_eval.separation.bss_eval_sources`` (filter length 512).  Everything runs in fp64 on the GPU (ctn_bss_eval_sources).

Differences from mir_eval: a Gram matrix of the references that is not numerically positive definite raises ValueError where
mir_eval falls back to a least-squares solve, and at most 4 sources are supported (NotImplementedError beyond)."""
import torch

from .. import _native as N

_REASONS = ((N.BSS_SILENT_REF, "a reference source is silent (all zeros)"),
            (N.BSS_SILENT_EST, "an estimated source is silent (all zeros)"),
            (N.BSS_NOT_PD, "the Gram matrix of the delayed references is not positive definite (mir_eval would fall back to lstsq)"))


def _on_device(t):
    if t.is_cuda:
        return t
    if not torch.cuda.is_available():
        raise RuntimeError("ctn_b200 runs on CUDA (sm_90a) tensors only; there is no CPU fallback")
    return t.to(torch.device("cuda", torch.cuda.current_device()))


def bss_eval_sources_batch(reference_sources, estimated_sources, compute_permutation=True):
    """reference_sources (B, S, T), estimated_sources (B, K, S, T) float32 -> sdr, sir, sar (B, K, S) float64 and perm (B, K, S)
    int64: set k of item b scored against the references of item b, as bss_eval_sources scores it.  Indexed by reference j: the
    estimate perm[b, k, j] is the one assigned to reference j.  CPU inputs are computed on the current CUDA device and the results
    come back to the CPU; CUDA inputs leave their results on their device."""
    if reference_sources.dim() != 3 or estimated_sources.dim() != 4:
        raise ValueError("reference_sources must be (B, S, T) and estimated_sources (B, K, S, T), got {} and {}".format(
            tuple(reference_sources.shape), tuple(estimated_sources.shape)))
    B, S, T = reference_sources.shape
    if estimated_sources.shape[0] != B or estimated_sources.shape[2:] != (S, T):
        raise ValueError("The shape of estimated sources and the true sources should match.  reference_sources.shape = {}, "
                         "estimated_sources.shape = {}".format(tuple(reference_sources.shape), tuple(estimated_sources.shape)))
    K = estimated_sources.shape[1]
    host = not reference_sources.is_cuda
    ref = _on_device(reference_sources).contiguous()
    est = estimated_sources.to(ref.device).contiguous()
    dev = N.require_cuda(ref, est)
    nbytes = N.C.c_size_t(0)
    N.check(N.ctn_bss_workspace_bytes(B, K, S, T, N.C.byref(nbytes)), "ctn_bss_workspace_bytes")
    base, avail = N.aligned(N.workspace(dev, nbytes.value + 256, "bss"))
    sdr, sir, sar = (torch.empty((B, K, S), dtype=torch.float64, device=dev) for _ in range(3))
    perm = torch.empty((B, K, S), dtype=torch.int32, device=dev)
    status = torch.empty(B, dtype=torch.int32, device=dev)
    N.check(N.ctn_bss_eval_sources(ref.data_ptr(), est.data_ptr(), B, K, S, T, int(bool(compute_permutation)), sdr.data_ptr(),
                                   sir.data_ptr(), sar.data_ptr(), perm.data_ptr(), status.data_ptr(), base, avail,
                                   N.stream_ptr(dev)), "ctn_bss_eval_sources")
    bad = status.cpu()
    for b in range(B):
        if int(bad[b]):
            raise ValueError("bss_eval_sources: item {}: {}".format(
                b, "; ".join(why for bit, why in _REASONS if int(bad[b]) & bit)))
    out = (sdr, sir, sar, perm.long())
    return tuple(t.cpu() for t in out) if host else out


def bss_eval_sources(reference_sources, estimated_sources, compute_permutation=True):
    """src/utils/bss.py:4-30.  reference_sources, estimated_sources (n_sources, T) or (T,) ->
    sdr, sir, sar (n_sources,) float64, perm (n_sources,) int64"""
    ref = reference_sources[None] if reference_sources.dim() == 1 else reference_sources
    est = estimated_sources[None] if estimated_sources.dim() == 1 else estimated_sources
    if ref.dim() != 2 or est.shape != ref.shape:
        raise ValueError("The shape of estimated sources and the true sources should match.  reference_sources.shape = {}, "
                         "estimated_sources.shape = {}".format(tuple(ref.shape), tuple(est.shape)))
    sdr, sir, sar, perm = bss_eval_sources_batch(ref[None], est[None, None], compute_permutation=compute_permutation)
    return sdr[0, 0], sir[0, 0], sar[0, 0], perm[0, 0]
