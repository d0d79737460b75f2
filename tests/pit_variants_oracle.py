"""CPU oracle for ORPIT and Sinkhorn PIT over SI-SDR (test infrastructure only): plain torch, any dtype, restating
src/criterion/pit.py:87-194 of the reference.  Pinned to the reference by tests/test_pit_variants_cpu.py against
tests/golden/pit_variants.pt (minted by tests/golden/make_pit_variants.py); the GPU tests run it in float64."""
import torch

from convtasnet_oracle import EPS, sisdr


def orpit(input, target, lengths=None, maximize=False, batch_mean=True, eps=EPS):
    """ORPIT.forward with criterion NegSISDR (maximize=False) or SISDR (maximize=True), src/criterion/pit.py:87-160.

    input (B, 2, T); target (B, n, T) padded, sample b using its first lengths[b] rows (None: all n).  The criterion sees
    2-D rows (:140-141), so its reduction does not enter.  Returns (loss, indices (B,) int64), first best candidate.
    """
    sign = 1.0 if maximize else -1.0
    losses, indices = [], []
    for b in range(input.shape[0]):
        n = target.shape[1] if lengths is None else int(lengths[b])
        t = target[b, :n]
        possible = []
        for i in range(n):
            rest = torch.sum(t * (torch.arange(n) != i).to(t.dtype).unsqueeze(-1), dim=0)  # :135-138
            one = sign * sisdr(input[b:b + 1, 0], t[i:i + 1], eps=eps)
            other = sign * sisdr(input[b:b + 1, 1], rest.unsqueeze(0), eps=eps)
            possible.append(one + other / (n - 1))  # :142
        possible = torch.cat(possible, dim=0)
        loss, idx = torch.max(possible, dim=0) if maximize else torch.min(possible, dim=0)  # :150-153
        losses.append(loss)
        indices.append(idx)
    loss = torch.stack(losses)
    if batch_mean:
        loss = loss.mean(dim=0)
    return loss, torch.stack(indices)


def sinkpit(input, target, coldness=1.0, iteration=10, maximize=False, batch_mean=True, eps=EPS):
    """sinkpit() with criterion NegSISDR (maximize=False) or SISDR (maximize=True), src/criterion/pit.py:162-194, on
    (B, S, T).  Returns (loss, P (B, S, S)); the gradient is that of the unrolled iterations."""
    B, S, T = input.shape
    possible = -sisdr(input.unsqueeze(2).expand(B, S, S, T), target.unsqueeze(1).expand(B, S, S, T), eps=eps)  # :169-178
    Z = -coldness * possible  # :180
    for _ in range(iteration):  # :182-184
        Z = Z - torch.logsumexp(Z, dim=1, keepdim=True)
        Z = Z - torch.logsumexp(Z, dim=2, keepdim=True)
    P = torch.exp(Z)
    loss = torch.sum((possible + Z / coldness) * P, dim=(1, 2))  # :187
    if maximize:
        loss = -loss
    if batch_mean:
        loss = loss.mean(dim=0)
    return loss, P
