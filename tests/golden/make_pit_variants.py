#!/usr/bin/env python
"""Mint tests/golden/pit_variants.pt from the UNMODIFIED reference (run in the build container only).

    python tests/golden/make_pit_variants.py

ORPIT (src/criterion/pit.py:87-160) and sinkpit (:162-194) of the reference, under NegSISDR and SISDR, with the autograd
gradients w.r.t. the estimate.  Estimates are noisy mixtures of the targets, so that candidates and pairs are separated.
The reference is imported as-is from /root/reference/src; nothing is copied from it.  /root/reference does not exist on
the GPU box: tests only read the committed .pt file.
"""
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference/src")
warnings.simplefilter("ignore")
from criterion.sdr import NegSISDR, SISDR  # noqa: E402  (reference)
from criterion.pit import ORPIT, sinkpit  # noqa: E402

torch.set_num_threads(8)


def main():
    from torch.nn.utils.rnn import pack_sequence
    g = torch.Generator().manual_seed(91)
    T = 203
    rec = {"orpit": [], "sinkpit": [], "sinkpit_inputs": {}}

    def orpit_inputs(lens):
        tgts = [torch.randn(n, T, generator=g) for n in lens]
        est = []
        for t in tgts:
            k = int(torch.randint(len(t), (1,), generator=g))
            rest = t.sum(dim=0) - t[k]
            est.append(torch.stack([t[k], rest]) + 0.3 * torch.randn(2, T, generator=g))
        return torch.stack(est), tgts

    est, tgts = orpit_inputs([3, 3, 3])
    cases = [("tensor_n3", est, torch.stack(tgts), None)]
    est, tgts = orpit_inputs([3, 2, 4])
    cases.append(("packed_3_2_4", est, tgts, [3, 2, 4]))
    for name, est, tgt, lens in cases:
        for crit_name, crit in (("NegSISDR", NegSISDR()), ("SISDR", SISDR())):
            x = est.clone().requires_grad_(True)
            target = tgt if lens is None else pack_sequence(tgt, enforce_sorted=False)
            loss, idx = ORPIT(crit)(x, target, batch_mean=True)
            loss.backward()
            with torch.no_grad():
                loss_b, _ = ORPIT(crit)(est, target, batch_mean=False)
            padded = tgt if lens is None else torch.nn.utils.rnn.pad_sequence(tgt, batch_first=True)
            rec["orpit"].append({"name": name, "criterion": crit_name, "input": est.clone(), "target": padded.clone(),
                                 "lengths": lens, "loss": loss.detach().clone(), "loss_b": loss_b.clone(),
                                 "indices": idx.clone(), "patterns": ORPIT(crit).patterns.clone(), "grad": x.grad.clone()})
    for S in (3, 10):
        tgt = torch.randn(2, S, T, generator=g)
        perm = torch.stack([torch.randperm(S, generator=g) for _ in range(2)])
        est = torch.stack([tgt[b, perm[b]] for b in range(2)]) + 0.5 * torch.randn(2, S, T, generator=g)
        rec["sinkpit_inputs"][S] = {"input": est.clone(), "target": tgt.clone()}
        for K in (10, 200):
            for c in (1.0, 10.0):
                for crit_name, crit in (("NegSISDR", NegSISDR()), ("SISDR", SISDR())):
                    x = est.clone().requires_grad_(True)
                    loss, P = sinkpit(crit, x, tgt, coldness=c, iteration=K, batch_mean=True)
                    loss.backward()
                    rec["sinkpit"].append({"S": S, "K": K, "coldness": c, "criterion": crit_name,
                                           "loss": loss.detach().clone(), "P": P.detach().clone(),
                                           "pattern": torch.argmax(P.detach(), dim=2), "grad": x.grad.clone()})
    path = os.path.join(HERE, "pit_variants.pt")
    torch.save(rec, path)
    print("pit_variants ->", os.path.getsize(path), "B")


if __name__ == "__main__":
    main()
